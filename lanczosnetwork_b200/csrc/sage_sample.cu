// GraphSAGE's neighbour sampling on the device, from the bond-list records of lnb_graph_prepare_sparse.
//
// The reference's collate (dataset/qm8.py:137-166) draws, for every graph b, channel e and real node n,
// K neighbours among the non-zero columns of row n of the channel's L4 operator with numpy's
// RandomState: K distinct ones when there are at least K candidates, K with replacement otherwise.  One
// CTA per graph here rebuilds the candidates from the bond list (the adjacency bitmaps of
// batch_prepare_sparse_kernel plus the diagonal of L4) and draws from the same two distributions with
// a counter-based generator, so every draw is a pure function of (sample_key, b, n, e, i) and a CPU
// restatement reproduces it exactly (the rule is in include/lanczosnet_b200.h).  The key is read from
// device memory, so a captured CUDA graph draws new samples whenever the caller rewrites it.
//
// Outputs besides the samples: the ELL rows of the count-weighted operator M_e[n, m] = nonempty * count
// / K in lnb_graph_prepare's layout and slot order (diagonal first, then ascending column; values
// (float)count / (float)K as lnb_sage_operators rounds them), and optionally those of M_e^T, which the
// training adjoint reads.  The dense [B, N, N, E1] operator never exists.
#include "common.cuh"
#include "philox.cuh"

namespace {

constexpr int SS_THREADS = 256;
constexpr int SS_NW = LNB_MAX_N / 32;     // 32-bit words per adjacency row

struct SampleParams {
  const int32_t* sizes; const int32_t* node_ptr; const int32_t* node_feat;
  const int32_t* edge_ptr; const uint8_t* edges; const int64_t* key;
  int B, N, E1, K, flags;
  int64_t* node_ids; uint8_t* mask; float* nonempty;
  int32_t* nn_idx;                                            // [B,N,K,E1] or null
  float* ell_val; uint8_t* ell_idx; int32_t* ell_max; int32_t* gext;
  float* ellT_val; uint8_t* ellT_idx; int32_t* ellT_max; int32_t* gextT;
};

using lnb::philox4x32_10;

__device__ __forceinline__ uint32_t word(const uint4& x, int i) {
  return i == 0 ? x.x : i == 1 ? x.y : i == 2 ? x.z : x.w;
}

// number of set bits of the 128-bit mask below bit j
__device__ __forceinline__ int rank_below(const uint32_t* m, int j) {
  int r = 0;
#pragma unroll
  for (int w = 0; w < SS_NW; ++w) {
    const int lo = w << 5;
    const uint32_t keep = j >= lo + 32 ? 0xffffffffu : (j <= lo ? 0u : (1u << (j - lo)) - 1u);
    r += __popc(m[w] & keep);
  }
  return r;
}

// position of the j-th (0-based) set bit of the 128-bit mask
__device__ __forceinline__ int select_bit(const uint32_t* m, int j) {
  int pos = 0;
  bool found = false;
#pragma unroll
  for (int w = 0; w < SS_NW; ++w) {
    const int c = __popc(m[w]);
    if (!found && j < c) {
      uint32_t bits = m[w];
      for (int k = 0; k < j; ++k) bits &= bits - 1;
      pos = (w << 5) + __ffs(bits) - 1;
      found = true;
    }
    j -= c;
  }
  return pos;
}

__global__ void __launch_bounds__(SS_THREADS)
sage_sample_kernel(const SampleParams P) {
  extern __shared__ __align__(16) unsigned char ss_smem[];
  __shared__ int s_max[LNB_MAX_E1], s_maxT[LNB_MAX_E1];
  __shared__ int s_ne;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int N = P.N, E1 = P.E1, E = E1 - 1, K = P.K;
  const int nb = min(max(P.sizes[b], 0), N);
  const bool want_ell = P.flags & LNB_SAGE_SAMPLE_ELL, want_t = P.flags & LNB_SAGE_SAMPLE_ELL_T;
  uint32_t* adj = reinterpret_cast<uint32_t*>(ss_smem);                  // [E][N][NW] bonds per type
  uint32_t* pick = adj + (size_t)E * N * SS_NW;                           // [E1][N][NW] columns drawn
  uint32_t* scratch = pick + (size_t)E1 * N * SS_NW;                             // [N][THREADS]
  uint8_t* cnt_s = reinterpret_cast<uint8_t*>(scratch + (size_t)N * SS_THREADS);    // [N*E1]
  uint8_t* cntT_s = cnt_s + N * E1;                                                  // [N*E1]

  for (int i = tid; i < E * N * SS_NW; i += SS_THREADS) adj[i] = 0u;
  if (tid < LNB_MAX_E1) { s_max[tid] = 0; s_maxT[tid] = 0; }
  if (tid == 0) s_ne = 0;
  __syncthreads();
  // ---- adjacency from the bond list, as lnb_graph_prepare_sparse builds it -------------------------
  const int e0 = P.edge_ptr[b], e1 = P.edge_ptr[b + 1];
  for (int q = e0 + tid; q < e1; q += SS_THREADS) {
    const uchar4 ed = reinterpret_cast<const uchar4*>(P.edges)[q];
    const int u = ed.x, v = ed.y, c = ed.z;
    if (u < nb && v < nb && c < E) {
      atomicOr(&adj[(c * N + u) * SS_NW + (v >> 5)], 1u << (v & 31));
      atomicOr(&adj[(c * N + v) * SS_NW + (u >> 5)], 1u << (u & 31));
    }
  }
  __syncthreads();
  const uint32_t k0 = (uint32_t)P.key[0], k1 = (uint32_t)((uint64_t)P.key[0] >> 32);
  const uint32_t c2 = (uint32_t)P.key[1], c3 = (uint32_t)((uint64_t)P.key[1] >> 32);
  const float kf = (float)K;
  const int pairs = N * E1;
  uint32_t* sc = scratch + tid;                                // this thread's entry j at sc[j * THREADS]
  // ---- draws, one thread per (node, channel) -----------------------------------------------------
  for (int p = tid; p < pairs; p += SS_THREADS) {
    const int n = p / E1, e = p - n * E1;
    uint32_t cm[SS_NW], pk[SS_NW];                             // candidates, distinct columns drawn
    int L = 0;
#pragma unroll
    for (int w = 0; w < SS_NW; ++w) {
      uint32_t bits = 0u;
      if (n < nb) {
        if (e == 0) { for (int c = 0; c < E; ++c) bits |= adj[(c * N + n) * SS_NW + w]; }
        else bits = adj[((e - 1) * N + n) * SS_NW + w];
        if ((n >> 5) == w) bits |= 1u << (n & 31);             // the + I of L4
      }
      cm[w] = bits;
      pk[w] = 0u;
      L += __popc(bits);
    }
    const uint32_t r = (uint32_t)(((int64_t)b * N + n) * E1 + e);
    int32_t* out = P.nn_idx ? P.nn_idx + ((int64_t)(b * N + n) * K) * E1 + e : nullptr;
    const bool distinct = L >= K;
    if (distinct) {                                           // partial Fisher-Yates over the candidates
      int j = 0;
#pragma unroll
      for (int w = 0; w < SS_NW; ++w)
        for (uint32_t bits = cm[w]; bits; bits &= bits - 1) sc[(j++) * SS_THREADS] = (uint32_t)((w << 5) + __ffs(bits) - 1);
    } else {
      for (int j = 0; j < L; ++j) sc[j * SS_THREADS] = 0;     // draw counts per candidate
    }
    uint4 x = make_uint4(0u, 0u, 0u, 0u);
    for (int i = 0; i < K; ++i) {
      int s = 0;
      if (L > 0) {
        if ((i & 3) == 0) x = philox4x32_10(make_uint4((uint32_t)(i >> 2), r, c2, c3), k0, k1);
        const uint32_t xi = word(x, i & 3);
        if (distinct) {
          const int j = i + (int)__umulhi(xi, (uint32_t)(L - i));
          const uint32_t cj = sc[j * SS_THREADS];
          sc[j * SS_THREADS] = sc[i * SS_THREADS];
          sc[i * SS_THREADS] = cj;
          s = (int)cj;
        } else {
          const int j = (int)__umulhi(xi, (uint32_t)L);
          sc[j * SS_THREADS] += 1;
          s = select_bit(cm, j);
        }
#pragma unroll
        for (int w = 0; w < SS_NW; ++w) pk[w] |= (w == (s >> 5)) ? 1u << (s & 31) : 0u;
      }
      if (out) out[(int64_t)i * E1] = s;                      // L = 0: the collate's zero fill
    }
#pragma unroll
    for (int w = 0; w < SS_NW; ++w) pick[(e * N + n) * SS_NW + w] = pk[w];
    if (!want_ell) continue;
    // ---- ELL row n of M_e: diagonal first, then ascending column (lnb_graph_prepare's order) -------
    float* val = P.ell_val + ((int64_t)(b * E1 + e) * N) * N + n;
    uint8_t* idx = P.ell_idx + ((int64_t)(b * E1 + e) * N) * N + n;
    int cnt = 0, far = 0;
    auto emit = [&](int m) {
      const uint32_t count = distinct ? 1u : sc[rank_below(cm, m) * SS_THREADS];
      val[(int64_t)cnt * N] = (float)count / kf;
      idx[(int64_t)cnt * N] = (uint8_t)m;
      ++cnt;
      far = max(far, m + 1);
    };
    if ((pk[n >> 5] >> (n & 31)) & 1u) emit(n);
#pragma unroll
    for (int w = 0; w < SS_NW; ++w)
      for (uint32_t bits = pk[w] & ~((n >> 5) == w ? 1u << (n & 31) : 0u); bits; bits &= bits - 1)
        emit((w << 5) + __ffs(bits) - 1);
    cnt_s[p] = (uint8_t)cnt;
    if (cnt) {
      atomicMax(&s_max[e], cnt);
      atomicMax(&s_ne, max(n + 1, far));
    }
  }
  // ---- padded node ids, mask, nonempty: every real node is its own candidate in every channel -------
  const int r0 = P.node_ptr[b];
  for (int n = tid; n < N; n += SS_THREADS) {
    P.node_ids[(int64_t)b * N + n] = (n < nb) ? (int64_t)P.node_feat[r0 + n] : 0;
    P.mask[(int64_t)b * N + n] = (n < nb) ? 1 : 0;
    P.nonempty[(int64_t)b * N + n] = (n < nb) ? 1.f : 0.f;
  }
  if (!want_ell) return;
  __syncthreads();
  // ---- zero tails up to the channel maximum; the rows of M_e^T ---------------------------------------
  for (int p = tid; p < pairs; p += SS_THREADS) {
    const int n = p / E1, e = p - n * E1;
    float* val = P.ell_val + ((int64_t)(b * E1 + e) * N) * N + n;
    uint8_t* idx = P.ell_idx + ((int64_t)(b * E1 + e) * N) * N + n;
    for (int t = cnt_s[p]; t < s_max[e]; ++t) {
      val[(int64_t)t * N] = 0.f;
      idx[(int64_t)t * N] = 0;
    }
    if (!want_t) continue;
    // row m = n of M_e^T lists the rows that drew m: its own first, then ascending.  The value is the
    // one row q's ELL slot holds for column m (slots below cnt_s, which the tail fill does not touch).
    const int m = n;
    const uint32_t bit = 1u << (m & 31);
    const int wm = m >> 5;
    float* valT = P.ellT_val + ((int64_t)(b * E1 + e) * N) * N + m;
    uint8_t* idxT = P.ellT_idx + ((int64_t)(b * E1 + e) * N) * N + m;
    int cnt = 0;
    for (int t = -1; t < nb; ++t) {
      const int q = t < 0 ? m : t;
      if ((t >= 0 && q == m) || m >= nb) continue;
      const uint32_t* pq = pick + (e * N + q) * SS_NW;
      if (!(pq[wm] & bit)) continue;
      const int dq = (pq[q >> 5] >> (q & 31)) & 1u;
      const int slot = (q == m) ? 0 : dq + rank_below(pq, m) - ((dq && q < m) ? 1 : 0);
      valT[(int64_t)cnt * N] = P.ell_val[((int64_t)(b * E1 + e) * N + slot) * N + q];
      idxT[(int64_t)cnt * N] = (uint8_t)q;
      ++cnt;
    }
    cntT_s[p] = (uint8_t)cnt;
    if (cnt) atomicMax(&s_maxT[e], cnt);
  }
  if (tid < E1) P.ell_max[b * E1 + tid] = s_max[tid];
  if (tid == 0) { P.gext[b * 2] = s_ne; P.gext[b * 2 + 1] = 0; }
  if (!want_t) return;
  __syncthreads();
  for (int p = tid; p < pairs; p += SS_THREADS) {
    const int m = p / E1, e = p - m * E1;
    float* valT = P.ellT_val + ((int64_t)(b * E1 + e) * N) * N + m;
    uint8_t* idxT = P.ellT_idx + ((int64_t)(b * E1 + e) * N) * N + m;
    for (int t = cntT_s[p]; t < s_maxT[e]; ++t) {
      valT[(int64_t)t * N] = 0.f;
      idxT[(int64_t)t * N] = 0;
    }
  }
  // the non-zeros of M^T are those of M transposed, so the extent max(row, column) + 1 is the same
  if (tid < E1) P.ellT_max[b * E1 + tid] = s_maxT[tid];
  if (tid == 0) { P.gextT[b * 2] = s_ne; P.gextT[b * 2 + 1] = 0; }
}

}  // namespace

extern "C" {

int lnb_sage_sample_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* node_ptr,
                           const int32_t* node_feat, const int32_t* edge_ptr, const uint8_t* edges,
                           const int64_t* sample_key, int B, int N, int E1, int K, int flags,
                           int64_t* node_ids, uint8_t* mask, float* nonempty, int32_t* nn_idx,
                           float* ell_val, uint8_t* ell_idx, int32_t* ell_max, int32_t* gext,
                           float* ellT_val, uint8_t* ellT_idx, int32_t* ellT_max, int32_t* gextT) {
  if (!(B >= 0 && N >= 1 && N <= LNB_MAX_N && E1 >= 2 && E1 <= LNB_MAX_E1 && K >= 1 &&
        (int64_t)B * N * E1 < ((int64_t)1 << 31))) {
    lnb::set_err("sage_sample_sparse: B=%d N=%d E1=%d K=%d outside 1 <= N <= %d, 2 <= E1 <= %d, K >= 1, "
                 "B*N*E1 < 2^31", B, N, E1, K, LNB_MAX_N, LNB_MAX_E1);
    return LNB_ERR_UNSUPPORTED;
  }
  const int known = LNB_SAGE_SAMPLE_NN_IDX | LNB_SAGE_SAMPLE_ELL | LNB_SAGE_SAMPLE_ELL_T;
  LNB_REQUIRE((flags & ~known) == 0 && (!(flags & LNB_SAGE_SAMPLE_ELL_T) || (flags & LNB_SAGE_SAMPLE_ELL)),
              "sage_sample_sparse: flags %d (the transposed rows need LNB_SAGE_SAMPLE_ELL)", flags);
  if (B == 0) return LNB_OK;
  // edges may be NULL when the batch has no bonds: the kernel reads [edge_ptr[b], edge_ptr[b+1]) only
  LNB_REQUIRE(sizes && node_ptr && node_feat && edge_ptr && sample_key && node_ids && mask && nonempty,
              "sage_sample_sparse: null pointer");
  LNB_REQUIRE(!(flags & LNB_SAGE_SAMPLE_NN_IDX) || nn_idx, "sage_sample_sparse: null nn_idx");
  LNB_REQUIRE(!(flags & LNB_SAGE_SAMPLE_ELL) || (ell_val && ell_idx && ell_max && gext),
              "sage_sample_sparse: null ELL output");
  LNB_REQUIRE(!(flags & LNB_SAGE_SAMPLE_ELL_T) || (ellT_val && ellT_idx && ellT_max && gextT),
              "sage_sample_sparse: null transposed ELL output");
  SampleParams p;
  p.sizes = sizes; p.node_ptr = node_ptr; p.node_feat = node_feat; p.edge_ptr = edge_ptr; p.edges = edges;
  p.key = sample_key; p.B = B; p.N = N; p.E1 = E1; p.K = K; p.flags = flags;
  p.node_ids = node_ids; p.mask = mask; p.nonempty = nonempty;
  p.nn_idx = (flags & LNB_SAGE_SAMPLE_NN_IDX) ? nn_idx : nullptr;
  p.ell_val = ell_val; p.ell_idx = ell_idx; p.ell_max = ell_max; p.gext = gext;
  p.ellT_val = ellT_val; p.ellT_idx = ellT_idx; p.ellT_max = ellT_max; p.gextT = gextT;
  const size_t smem = (size_t)(2 * E1 - 1) * N * SS_NW * 4 + (size_t)N * SS_THREADS * 4 + (size_t)2 * N * E1;
  cudaStream_t s = (cudaStream_t)stream;
  if (smem > 48 * 1024)
    cudaFuncSetAttribute(sage_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  sage_sample_kernel<<<B, SS_THREADS, smem, s>>>(p);
  lnb::count_launch();
  return lnb::finish_launch("sage_sample_sparse");
}

}  // extern "C"
