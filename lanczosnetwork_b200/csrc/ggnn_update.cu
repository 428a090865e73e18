// One GGNN propagation step after the message MLPs (reference: model/ggnn.py:143-171):
//     h'[r, :] = GRUCell( [A_0 M_0 | ... | A_{E1-1} M_{E1-1}][r, :],  h[r, :] )
// with A_e the binarised operator of bond channel e (sum) or its row-normalised form
// A_e[n, m] / (nnz_e(n) + FLT_EPSILON) (avg), and M [B*N, E1*D] the per-channel messages.
//
// The GRU step of gru_step.cuh with E1*D/32 message k-blocks: the k-block of channel e of row (b, n) is
// the weighted sum of the M rows of node n's neighbours, gathered through the ELL rows of
// lnb_graph_prepare.  The aggregated [B*N, E1*D] message matrix never exists in HBM; W is the
// re-laid-out GRU weights [4D, (E1+1)*D].  Each row tile re-produces its A operand once per column
// tile (4D / 128 times); the column tiles of one row tile run on neighbouring CTAs at the same time,
// so the repeated gathers hit L2.
#include "gru_step.cuh"

namespace {


struct GgnnUpdateParams {
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

struct GgnnUpdatePolicy : gru::Step<GgnnUpdatePolicy, GgnnUpdateParams> {
  using Step::Step;
  static __device__ __forceinline__ int msg_kblocks(const Params& p) { return p.E1 * p.D / tcg::BK; }

  __device__ __forceinline__ void produce_msg(int kb, float (&v)[32]) {
    const int c0 = kb * tcg::BK, e = c0 / p.D, j0 = c0 - e * p.D;
    // row n of channel e: entries t < len, the non-zeros first (t-major, stride N), zero fill behind
    const int64_t line = ((int64_t)(b * p.E1 + e) * p.N) * p.N + n;
    const int cnt = gru::ell_count(p.ell_val, line, __ldg(p.ell_max + b * p.E1 + e), p.N);
    const float w = gru::row_weight(cnt, p.avg);
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
};

}  // namespace

extern "C" {

int lnb_ggnn_update(lnb_stream_t stream, const float* M, const float* h, const float* ell_val,
                    const uint8_t* ell_idx, const int32_t* ell_max, const float* W_hi, const float* W_lo,
                    const float* bias, int B, int N, int D, int E1, int avg, float* out) {
  LNB_REQUIRE(M && h && ell_val && ell_idx && ell_max && W_hi && W_lo && bias && out,
              "ggnn_update: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && D >= 1 && E1 >= 1, "ggnn_update: bad dims B=%d N=%d D=%d E1=%d", B, N, D,
              E1);
  if (N > LNB_MAX_N_ELL || D % 32 || D > LNB_MAX_WIDTH || E1 > LNB_MAX_E1) {
    lnb::set_err("ggnn_update: N=%d D=%d E1=%d outside the kernel (N <= %d, D %% 32 == 0, D <= %d, "
                 "E1 <= %d)", N, D, E1, LNB_MAX_N_ELL, LNB_MAX_WIDTH, LNB_MAX_E1);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE(((uintptr_t)M | (uintptr_t)h | (uintptr_t)out | (uintptr_t)W_hi | (uintptr_t)W_lo) % 16 == 0,
              "ggnn_update: M, h, out and W must be 16-byte aligned");
  LNB_REQUIRE(out != h, "ggnn_update: out must not alias h (the epilogue reads h after other tiles wrote)");
  LNB_REQUIRE((int64_t)B * N <= 0x7fffffff, "ggnn_update: B*N too large");
  const int rows = B * N;
  if (rows == 0) return LNB_OK;
  GgnnUpdatePolicy::Params p{M, h, ell_val, ell_idx, ell_max, bias, out, rows, N, D, E1, avg ? 1 : 0,
                             tcg::debug_flags()};
  return tcg::launch<GgnnUpdatePolicy>(stream, W_hi, W_lo, 4 * D, (E1 + 1) * D, GgnnUpdatePolicy::SMEM_BYTES,
                                       lnb::ceil_div(rows, tcg::BM) * (4 * D / tcg::BN), p, "ggnn_update");
}

}  // extern "C"
