// Dense layer on the Hopper tensor cores (wgmma, sm_90a):
//     C[M,N] = act( A[M,K] @ W[N,K]^T + bias )          fp32 in, fp32 out, 3xTF32
// Row-loading policy of the persistent skeleton in tc_gemm.cuh: each producer thread owns one
// row of the 128-row tile, streams 32 consecutive K-values per k-block (8 x LDG.128, one of
// its k-blocks ahead) and hands them to the skeleton, which splits them into tf32 hi/lo and
// stores them into the shared-memory A ring.
// Replaces the nn.Linear call sites of the reference (model/lanczos_net.py:112,181,186;
// model/ada_lanczos_net.py:54-63 via :274).
#include "tc_gemm.cuh"

namespace {

struct RowLoadPolicy {
  static constexpr int kStagesB = 3;      // 96 KB of W tiles in flight per SM: the weight stream of a deep, narrow GEMM is HBM latency x bandwidth bound
  static constexpr int kStagesA = 2;      // 64 KB: one drain pass for the epilogue
  // groups > 1: block-diagonal ("grouped") layer -- column block g of A [M, groups*K] times
  // W_g [N, K] (stacked [groups*N, K]) into column block g of C [M, groups*N].
  struct Params {
    const float* A;
    const float* bias;
    float* C;
    int M, N, K, relu, groups;
    int dbg;                // debug experiment flags (LNB_DBG), 0 in production
    // split-K (few output tiles, deep K: the 4096-wide Ada filter MLP at M = batch): every tile is
    // computed by `splits` CTAs over disjoint k-block ranges; each writes its partial tile to `ws`
    // and the last one to arrive (per-tile counter) sums them, applies bias / ReLU and writes C.
    int splits;
    float* ws;              // [tiles][splits][128][128]
    int* counters;          // [tiles], zero on entry, zero again on exit
  };
  static __device__ __forceinline__ int tiles_per_group(const Params& p) { return (p.N + tcg::BN - 1) / tcg::BN; }
  static __device__ __forceinline__ int n_tiles(const Params& p) { return p.groups * tiles_per_group(p); }
  static __device__ __forceinline__ int num_tiles(const Params& p) {
    return ((p.M + tcg::BM - 1) / tcg::BM) * n_tiles(p);
  }
  static __device__ __forceinline__ int num_steps(const Params& p, int cta, int ncta) {
    const int t = num_tiles(p) * p.splits;
    return t > cta ? (t - cta + ncta - 1) / ncta : 0;
  }
  // sub = n-tile index + n_tiles * split
  static __device__ __forceinline__ void decode(const Params& p, int cta, int ncta, int it,
                                                int& m_tile, int& sub) {
    const int item = cta + it * ncta, nt = n_tiles(p);
    const int tile = item / p.splits, split = item - tile * p.splits;
    m_tile = tile / nt;
    sub = tile % nt + nt * split;
  }
  static __device__ __forceinline__ int kb_total(const Params& p) { return (p.K + tcg::BK - 1) / tcg::BK; }
  static __device__ __forceinline__ int kb_per_split(const Params& p) { return (kb_total(p) + p.splits - 1) / p.splits; }
  static __device__ __forceinline__ int kb_begin(const Params& p, int sub) { return (sub / n_tiles(p)) * kb_per_split(p); }
  static __device__ __forceinline__ int num_kblocks(const Params& p, int sub) {
    const int left = kb_total(p) - kb_begin(p, sub), per = kb_per_split(p);
    return left < per ? left : per;
  }
  static __device__ __forceinline__ int w_row0(const Params& p, int sub) {
    const int tpg = tiles_per_group(p), ns = sub % n_tiles(p);
    return (ns / tpg) * p.N + (ns % tpg) * tcg::BN;
  }
  static __device__ __forceinline__ void w_coords(const Params& p, int sub, int kb, int& col0, int& row0) {
    col0 = (kb_begin(p, sub) + kb) * tcg::BK;
    row0 = w_row0(p, sub);
  }

  const Params& p;
  const int r, grp;
  const int lda, ldc;
  const float* arow;
  bool row_ok;
  int row, kb0, tile;
  float cur[32];
  int* flag;                // shared: the split that arrived last reduces the tile

  __device__ RowLoadPolicy(const Params& p_, uint8_t* smem, int tid)
      : p(p_), r(tid & 127), grp(tid >> 7), lda(p_.groups * p_.K), ldc(p_.groups * p_.N),
        arow(nullptr), row_ok(false), row(0), kb0(0), tile(0), flag(reinterpret_cast<int*>(smem)) {}

  __device__ __forceinline__ void load(int kb, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = (kb0 + kb) * tcg::BK + 4 * j;
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row_ok && k < p.K) t = __ldg(reinterpret_cast<const float4*>(arow + k));
      v[4 * j + 0] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
    }
  }
  __device__ __forceinline__ void step_begin(int m_tile, int sub, int kb_first, tcg::PhaseTimer&) {
    row = m_tile * tcg::BM + r;
    row_ok = row < p.M;
    const int ns = sub % n_tiles(p);
    kb0 = kb_begin(p, sub);
    tile = m_tile * n_tiles(p) + ns;
    arow = p.A + (int64_t)(row_ok ? row : 0) * lda + (ns / tiles_per_group(p)) * p.K;
    load(kb_first, cur);
  }
  __device__ __forceinline__ void produce(int, int kb, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = cur[j];
    load(kb + tcg::ProducerGroups<RowLoadPolicy>::value, cur);   // this group's next k-block (zeros past K)
  }
  __device__ __forceinline__ void pre_epilogue(int) {}
  __device__ __forceinline__ void store(int sub, int col, const float (&x)[tcg::EW]) {
    if (p.splits > 1) {     // raw partial sums of this split
      float4* dst = reinterpret_cast<float4*>(
          p.ws + (((int64_t)tile * p.splits + sub / n_tiles(p)) * tcg::BM + r) * tcg::BN + col);
#pragma unroll
      for (int q = 0; q < tcg::EW / 4; ++q)
        __stcg(dst + q, make_float4(x[4 * q], x[4 * q + 1], x[4 * q + 2], x[4 * q + 3]));
      return;
    }
    const int left = p.N - ((sub % n_tiles(p)) % tiles_per_group(p)) * tcg::BN;
    const int w0 = w_row0(p, sub);
    tcg::store_row_chunk(row_ok ? p.C + (int64_t)row * ldc + w0 : nullptr,
                         left < tcg::BN ? left : tcg::BN, p.bias ? p.bias + w0 : nullptr,
                         p.relu != 0, col, x);
  }
  __device__ __forceinline__ void post_epilogue(int sub) {
    if (p.splits == 1) return;
    const int tid = grp * 128 + r;
    __threadfence();                       // this thread's partials are visible device-wide
    tcg::producers_sync<RowLoadPolicy>();
    if (tid == 0) {
      const int old = atomicAdd(p.counters + tile, 1);
      *flag = (old == p.splits - 1);
      if (old == p.splits - 1) p.counters[tile] = 0;      // ready for the next launch
    }
    tcg::producers_sync<RowLoadPolicy>();
    if (*flag) {
      __threadfence();
      const int ns = sub % n_tiles(p);
      const int m0 = (tile / n_tiles(p)) * tcg::BM;
      const int left = p.N - (ns % tiles_per_group(p)) * tcg::BN;
      const int ncols = left < tcg::BN ? left : tcg::BN;
      const int w0 = w_row0(p, sub);
      const float* base = p.ws + (int64_t)tile * p.splits * tcg::BM * tcg::BN;
      for (int e = tid; e < tcg::BM * tcg::BN / 4; e += tcg::producer_threads<RowLoadPolicy>) {
        const int rr = e / (tcg::BN / 4), c4 = (e - rr * (tcg::BN / 4)) * 4;
        if (m0 + rr >= p.M || c4 >= ncols) continue;
        float4 acc = __ldcg(reinterpret_cast<const float4*>(base + rr * tcg::BN + c4));
        for (int sp = 1; sp < p.splits; ++sp) {
          const float4 t = __ldcg(reinterpret_cast<const float4*>(base + ((int64_t)sp * tcg::BM + rr) * tcg::BN + c4));
          acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
        }
        float y[4] = {acc.x, acc.y, acc.z, acc.w};
        float* out = p.C + (int64_t)(m0 + rr) * ldc + w0 + c4;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (c4 + u < ncols) {
            if (p.bias) y[u] += __ldg(p.bias + w0 + c4 + u);
            if (p.relu) y[u] = fmaxf(y[u], 0.f);
            out[u] = y[u];
          }
        }
      }
    }
    tcg::producers_sync<RowLoadPolicy>();  // `flag` is rewritten by the next item
  }
};

constexpr size_t SMEM_BYTES = tcg::core_smem(RowLoadPolicy::kStagesB, RowLoadPolicy::kStagesA) + 1024 + 16;

}  // namespace

static int launch_linear(lnb_stream_t stream, const float* A, const float* W_hi, const float* W_lo,
                         const float* bias, int M, int N, int K, int groups, int relu, float* C,
                         const char* who, int splits = 1, float* ws = nullptr, int* counters = nullptr) {
  LNB_REQUIRE(A && W_hi && W_lo && C, "%s: null pointer", who);
  LNB_REQUIRE(M >= 0 && N >= 1 && K >= 1 && groups >= 1, "%s: bad dims M=%d N=%d K=%d groups=%d",
              who, M, N, K, groups);
  LNB_REQUIRE(K % 4 == 0, "%s: K=%d must be a multiple of 4 (16-byte rows)", who, K);
  LNB_REQUIRE(((uintptr_t)A & 15) == 0 && ((uintptr_t)W_hi & 15) == 0 && ((uintptr_t)W_lo & 15) == 0,
              "%s: A / W must be 16-byte aligned", who);
  if (M == 0) return LNB_OK;
  const int nkb = lnb::ceil_div(K, tcg::BK);
  LNB_REQUIRE(splits >= 1 && splits <= 16 && (splits == 1 || (ws && counters)),
              "%s: split-K needs 1 <= splits <= 16, a workspace and counters", who);
  LNB_REQUIRE(splits == 1 || lnb::ceil_div(nkb, splits) * (splits - 1) < nkb,
              "%s: %d splits leave an empty k range for K=%d", who, splits, K);
  RowLoadPolicy::Params p{A, bias, C, M, N, K, relu, groups, tcg::debug_flags(), splits, ws, counters};
  const int tiles = lnb::ceil_div(M, tcg::BM) * lnb::ceil_div(N, tcg::BN) * groups * splits;
  return tcg::launch<RowLoadPolicy>(stream, W_hi, W_lo, groups * N, K, SMEM_BYTES, tiles, p, who);
}

extern "C" {

int lnb_linear_tf32x3(lnb_stream_t stream, const float* A, const float* W_hi, const float* W_lo,
                      const float* bias, int M, int N, int K, int relu, float* C) {
  return launch_linear(stream, A, W_hi, W_lo, bias, M, N, K, 1, relu, C, "linear_tf32x3");
}

int lnb_linear_tf32x3_splitk(lnb_stream_t stream, const float* A, const float* W_hi, const float* W_lo,
                             const float* bias, int M, int N, int K, int relu, float* C, int splits,
                             float* workspace, int* counters) {
  return launch_linear(stream, A, W_hi, W_lo, bias, M, N, K, 1, relu, C, "linear_tf32x3_splitk", splits,
                       workspace, counters);
}

int lnb_linear_tf32x3_grouped(lnb_stream_t stream, const float* A, const float* W_hi,
                              const float* W_lo, const float* bias, int M, int groups, int N, int K,
                              int relu, float* C) {
  return launch_linear(stream, A, W_hi, W_lo, bias, M, N, K, groups, relu, C,
                       "linear_tf32x3_grouped");
}

}  // extern "C"
