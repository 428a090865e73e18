// One GGNN propagation step after the message MLPs (reference: model/ggnn.py:143-171):
//     h'[r, :] = GRUCell( [A_0 M_0 | ... | A_{E1-1} M_{E1-1}][r, :],  h[r, :] )
// with A_e the binarised operator of bond channel e (sum) or its row-normalised form
// A_e[n, m] / (nnz_e(n) + FLT_EPSILON) (avg), and M [B*N, E1*D] the per-channel messages.
//
// A policy of the persistent 3xTF32 wgmma skeleton (tc_gemm.cuh) over plain 128-row tiles of the
// B*N rows.  The GEMM is
//     G[r, :] = [agg(r) | h(r)] @ W^T,     W = the re-laid-out GRU weights [4D, (E1+1)*D]
// and its A operand is PRODUCED by the CUDA-core warps: the k-block of channel e of row (b, n) is the
// weighted sum of the M rows of node n's neighbours, gathered through the ELL rows of
// lnb_graph_prepare; the k-blocks past E1*D are the row of h.  The aggregated [B*N, E1*D] message
// matrix never exists in HBM.  W's rows hold the gate blocks r, z, n_in, n_h, interleaved so that a
// 16-column epilogue unit carries all four gates of 4 hidden units:
//     W row (u / 4) * 16 + g * 4 + u % 4 = gate g of hidden unit u
//     r:    [W_ir | W_hr]      z:    [W_iz | W_hz]      n_in: [W_in | 0]      n_h: [0 | W_hn]
// and the epilogue applies the GRU cell (the gate order of torch's CPU GRUCell):
//     r = sigmoid(G_r + b_r), z = sigmoid(G_z + b_z), n = tanh(G_nin + b_in + r * (G_nh + b_hn)),
//     h' = (h - n) * z + n
// Each row tile re-produces its A operand once per column tile (4D / 128 times); the column tiles of
// one row tile run on neighbouring CTAs at the same time, so the repeated gathers hit L2.
#include <float.h>

#include "tc_gemm.cuh"

namespace {

constexpr int GG_DMAX = 128, GG_NMAX = 255, GG_E1MAX = 16;

struct GgnnUpdatePolicy {
  static constexpr int kStagesB = 3;
  static constexpr int kStagesA = 2;
  struct Params {
    const float* M;          // [rows, E1*D]
    const float* h;          // [rows, D]
    const float* ell_val;    // [B, E1, N, N]  t-major ELL rows (lnb_graph_prepare)
    const uint8_t* ell_idx;  // [B, E1, N, N]
    const int32_t* ell_max;  // [B, E1]
    const float* bias;       // [4D] interleaved like the rows of W
    float* out;              // [rows, D]
    int rows, N, D, E1, avg;
    int dbg;
  };
  static __device__ __forceinline__ int n_tiles(const Params& p) { return 4 * p.D / tcg::BN; }
  static __device__ __forceinline__ int num_steps(const Params& p, int cta, int ncta) {
    const int t = ((p.rows + tcg::BM - 1) / tcg::BM) * n_tiles(p);
    return t > cta ? (t - cta + ncta - 1) / ncta : 0;
  }
  // consecutive items = the column tiles of one row tile: they run side by side and share the gathers in L2
  static __device__ __forceinline__ void decode(const Params& p, int cta, int ncta, int it, int& m_tile,
                                                int& sub) {
    const int item = cta + it * ncta, nt = n_tiles(p);
    m_tile = item / nt;
    sub = item - m_tile * nt;
  }
  static __device__ __forceinline__ int num_kblocks(const Params& p, int) {
    return (p.E1 + 1) * p.D / tcg::BK;
  }
  static __device__ __forceinline__ void w_coords(const Params&, int sub, int kb, int& col0, int& row0) {
    col0 = kb * tcg::BK;
    row0 = sub * tcg::BN;
  }

  const Params& p;
  const int r;
  int row, b, n;
  bool row_ok;

  __device__ GgnnUpdatePolicy(const Params& p_, uint8_t*, int tid)
      : p(p_), r(tid & 127), row(0), b(0), n(0), row_ok(false) {}

  __device__ __forceinline__ void step_begin(int m_tile, int, int, tcg::PhaseTimer&) {
    row = m_tile * tcg::BM + r;
    row_ok = row < p.rows;
    b = row_ok ? row / p.N : 0;
    n = row_ok ? row - b * p.N : 0;
  }

  __device__ __forceinline__ void produce(int, int kb, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = 0.f;
    if (!row_ok) return;
    const int c0 = kb * tcg::BK, e = c0 / p.D, j0 = c0 - e * p.D;
    if (e == p.E1) {                                   // the h columns
      const float4* src = reinterpret_cast<const float4*>(p.h + (int64_t)row * p.D + j0);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 t = __ldg(src + j);
        v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
      }
      return;
    }
    // row n of channel e: entries t < len, the non-zeros first (t-major, stride N), zero fill behind
    const int64_t line = ((int64_t)(b * p.E1 + e) * p.N) * p.N + n;
    const int len = __ldg(p.ell_max + b * p.E1 + e);
    int cnt = 0;
    while (cnt < len && __ldg(p.ell_val + line + (int64_t)cnt * p.N) != 0.f) ++cnt;
    // avg: the reference's L / (rowsum(L) + eps) on the 0/1 operator -- one correctly rounded reciprocal
    const float w = p.avg ? __frcp_rn((float)cnt + FLT_EPSILON) : 1.f;
    const int ldm = p.E1 * p.D;
    const float* mb = p.M + (int64_t)b * p.N * ldm + e * p.D + j0;
#pragma unroll 2
    for (int t = 0; t < cnt; ++t) {
      const int m = __ldg(p.ell_idx + line + (int64_t)t * p.N);
      const float4* src = reinterpret_cast<const float4*>(mb + (int64_t)m * ldm);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 x = __ldg(src + j);
        v[4 * j] = fmaf(w, x.x, v[4 * j]);
        v[4 * j + 1] = fmaf(w, x.y, v[4 * j + 1]);
        v[4 * j + 2] = fmaf(w, x.z, v[4 * j + 2]);
        v[4 * j + 3] = fmaf(w, x.w, v[4 * j + 3]);
      }
    }
  }

  __device__ __forceinline__ void pre_epilogue(int) {}

  static __device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

  __device__ __forceinline__ void store(int sub, int col, const float (&x)[tcg::EW]) {
    if (!row_ok) return;
    const int w0 = sub * tcg::BN + col;                // first W row of this unit
    const int u0 = w0 / 4;                             // its first hidden unit
    const float4 hv = __ldg(reinterpret_cast<const float4*>(p.h + (int64_t)row * p.D + u0));
    const float hp[4] = {hv.x, hv.y, hv.z, hv.w};
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float rg = sigmoid(x[i] + __ldg(p.bias + w0 + i));
      const float zg = sigmoid(x[4 + i] + __ldg(p.bias + w0 + 4 + i));
      const float gin = x[8 + i] + __ldg(p.bias + w0 + 8 + i);
      const float ghn = x[12 + i] + __ldg(p.bias + w0 + 12 + i);
      const float ng = tanhf(gin + rg * ghn);
      o[i] = (hp[i] - ng) * zg + ng;
    }
    *reinterpret_cast<float4*>(p.out + (int64_t)row * p.D + u0) = make_float4(o[0], o[1], o[2], o[3]);
  }

  __device__ __forceinline__ void post_epilogue(int) {}
};

constexpr size_t SMEM_BYTES = tcg::core_smem(GgnnUpdatePolicy::kStagesB, GgnnUpdatePolicy::kStagesA) + 1024 + 16;

// The phase-timer pointer lives in each translation unit's copy of tcg::g_prof: mirror the buffer
// registered with lnb_debug_set_prof into this one when it changes (profiling only).
unsigned long long* g_prof_mirrored = nullptr;

int sync_prof_buffer() {
  unsigned long long* buf = lnb::prof_buffer();
  if (buf == g_prof_mirrored) return LNB_OK;
  cudaError_t e = cudaMemcpyToSymbol(tcg::g_prof, &buf, sizeof(buf));
  if (e != cudaSuccess) { lnb::set_err("ggnn_update: %s", cudaGetErrorString(e)); return (int)e; }
  g_prof_mirrored = buf;
  return LNB_OK;
}

}  // namespace

extern "C" {

int lnb_ggnn_update(lnb_stream_t stream, const float* M, const float* h, const float* ell_val,
                    const uint8_t* ell_idx, const int32_t* ell_max, const float* W_hi, const float* W_lo,
                    const float* bias, int B, int N, int D, int E1, int avg, float* out) {
  LNB_REQUIRE(M && h && ell_val && ell_idx && ell_max && W_hi && W_lo && bias && out,
              "ggnn_update: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && D >= 1 && E1 >= 1, "ggnn_update: bad dims B=%d N=%d D=%d E1=%d", B, N, D,
              E1);
  if (N > GG_NMAX || D % 32 || D > GG_DMAX || E1 > GG_E1MAX) {
    lnb::set_err("ggnn_update: N=%d D=%d E1=%d outside the kernel (N <= %d, D %% 32 == 0, D <= %d, "
                 "E1 <= %d)", N, D, E1, GG_NMAX, GG_DMAX, GG_E1MAX);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE(((uintptr_t)M | (uintptr_t)h | (uintptr_t)out | (uintptr_t)W_hi | (uintptr_t)W_lo) % 16 == 0,
              "ggnn_update: M, h, out and W must be 16-byte aligned");
  LNB_REQUIRE(out != h, "ggnn_update: out must not alias h (the epilogue reads h after other tiles wrote)");
  LNB_REQUIRE((int64_t)B * N <= 0x7fffffff, "ggnn_update: B*N too large");
  const int rows = B * N;
  if (rows == 0) return LNB_OK;
  int rc = sync_prof_buffer();
  if (rc != LNB_OK) return rc;
  CUtensorMap map_hi, map_lo;
  rc = tcg::make_weight_map(&map_hi, W_hi, 4 * D, (E1 + 1) * D, "ggnn_update");
  if (rc != LNB_OK) return rc;
  rc = tcg::make_weight_map(&map_lo, W_lo, 4 * D, (E1 + 1) * D, "ggnn_update");
  if (rc != LNB_OK) return rc;
  auto kern = tcg::tc_gemm_kernel<GgnnUpdatePolicy>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES);
  GgnnUpdatePolicy::Params p{M, h, ell_val, ell_idx, ell_max, bias, out, rows, N, D, E1, avg ? 1 : 0,
                             tcg::debug_flags()};
  const int tiles = lnb::ceil_div(rows, tcg::BM) * (4 * D / tcg::BN);
  const int grid = tiles < tcg::sm_count() ? tiles : tcg::sm_count();
  kern<<<grid, tcg::THREADS, SMEM_BYTES, (cudaStream_t)stream>>>(map_hi, map_lo, p);
  lnb::count_launch();
  return lnb::finish_launch("ggnn_update");
}

}  // extern "C"
