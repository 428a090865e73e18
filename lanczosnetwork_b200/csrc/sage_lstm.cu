// One time step of GraphSAGE's LSTM aggregator (reference: model/graph_sage.py:37-41,131-140) for every
// sequence of a propagation layer at once:
//     x_t[s] = state[b*N + nn_idx[b, n, t, e]]        (a zero row for an id outside [0, N))
//     [i f g o] = x_t[s] W_ih^T + h[s] W_hh^T + b_ih + b_hh
//     c'[s] = sigmoid(f) c[s] + sigmoid(i) tanh(g),   h'[s] = sigmoid(o) tanh(c'[s])
// for the sequences s = (b*N + n)*E1 + e, i.e. the rows of h, h' and c are [B*N, E1*D] row-major: on
// the last step h' * nonempty is the message matrix that filter[ii] reads, column block e = channel e.
//
// A policy of the persistent 3xTF32 wgmma skeleton (tc_gemm.cuh), launched as sage_lstm_step_kernel, with
// the work split of gru_step.cuh:
// items are (128-row tile, column tile), column tiles innermost.  The A operand of row s is the D/32
// k-blocks of the gathered state row, then the D/32 k-blocks of h[s] (none at t = 0, where h = c = 0).
// W [4D, 2D] holds [W_ih | W_hh] with its rows interleaved so that a 16-column epilogue unit carries the
// gates i, f, g, o of 4 hidden units:
//     W row (u / 4) * 16 + g * 4 + u % 4 = gate g of hidden unit u       (torch's gate order i, f, g, o)
// and bias [4D] = b_ih + b_hh, interleaved the same way.  The epilogue applies the cell; exactly one
// thread reads and writes each element of c (in place).  h' goes to `out`, which must not alias h: the
// other column tiles of a row tile still read the old h.  A row with nonempty = 0 gathers nothing and
// runs no cell; its h' is left unwritten, except on the last step, where its message row is zero.
#include "gru_step.cuh"

namespace {


struct SageLstmParams {
  const float* state;      // [B*N, D]  the layer's input
  const int32_t* nn_idx;   // [B, N, K, E1]
  const float* nonempty;   // [B*N]
  const float* h;          // [R, D]    h of step t - 1 (unused at t = 0)
  float* c;                // [R, D]    c of step t - 1, overwritten with c of step t (not read at t = 0)
  const float* bias;       // [4D]      interleaved like the rows of W
  float* out;              // [R, D]    h of step t (times nonempty on the last step)
  int rows, N, K, E1, D, t, last;
  int dbg;
};

struct SageLstmPolicy {
  using Params = SageLstmParams;
  static constexpr int kStagesB = 3;
  static constexpr int kStagesA = 2;
  static constexpr size_t SMEM_BYTES = tcg::core_smem(kStagesB, kStagesA) + 1024 + 16;

  static __device__ __forceinline__ int n_tiles(const Params& p) { return 4 * p.D / tcg::BN; }
  static __device__ __forceinline__ int num_steps(const Params& p, int cta, int ncta) {
    const int t = ((p.rows + tcg::BM - 1) / tcg::BM) * n_tiles(p);
    return t > cta ? (t - cta + ncta - 1) / ncta : 0;
  }
  static __device__ __forceinline__ void decode(const Params& p, int cta, int ncta, int it, int& m_tile,
                                                int& sub) {
    const int item = cta + it * ncta, per = n_tiles(p);
    m_tile = item / per;
    sub = item - m_tile * per;
  }
  static __device__ __forceinline__ int num_kblocks(const Params& p, int) {
    return (p.t == 0 ? 1 : 2) * (p.D / tcg::BK);
  }
  static __device__ __forceinline__ void w_coords(const Params& p, int sub, int kb, int& col0, int& row0) {
    col0 = kb * tcg::BK;
    row0 = sub * tcg::BN;
  }

  const Params& p;
  const int r;
  int row;
  bool live;               // a real sequence of a node with nonempty != 0
  const float* x;          // its gathered state row, or null (an id outside [0, N))

  __device__ SageLstmPolicy(const Params& p_, uint8_t*, int tid)
      : p(p_), r(tid & 127), row(0), live(false), x(nullptr) {}

  __device__ __forceinline__ void step_begin(int m_tile, int, int, tcg::PhaseTimer&) {
    row = m_tile * tcg::BM + r;
    live = false;
    x = nullptr;
    if (row >= p.rows) return;
    const int node = row / p.E1, e = row - node * p.E1;     // node = b*N + n
    live = __ldg(p.nonempty + node) != 0.f;
    if (!live) return;
    const int b = node / p.N;
    const int m = __ldg(p.nn_idx + ((int64_t)node * p.K + p.t) * p.E1 + e);
    if (m >= 0 && m < p.N) x = p.state + ((int64_t)b * p.N + m) * p.D;
  }

  __device__ __forceinline__ void produce(int, int kb, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = 0.f;
    if (!live) return;
    const int xb = p.D / tcg::BK;
    const float* src = kb < xb ? x : p.h + (int64_t)row * p.D;
    if (src == nullptr) return;
    const float4* s4 = reinterpret_cast<const float4*>(src + (kb < xb ? kb : kb - xb) * tcg::BK);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 q = __ldg(s4 + j);
      v[4 * j] = q.x; v[4 * j + 1] = q.y; v[4 * j + 2] = q.z; v[4 * j + 3] = q.w;
    }
  }

  __device__ __forceinline__ void pre_epilogue(int) {}

  __device__ __forceinline__ void store(int sub, int col, const float (&x_)[tcg::EW]) {
    if (row >= p.rows) return;
    const int w0 = sub * tcg::BN + col;                     // first W row of this unit
    const int u0 = w0 / 4;                                  // its first hidden unit
    float4* orow = reinterpret_cast<float4*>(p.out + (int64_t)row * p.D + u0);
    if (!live) {
      if (p.last) *orow = make_float4(0.f, 0.f, 0.f, 0.f);
      return;
    }
    float4* crow = reinterpret_cast<float4*>(p.c + (int64_t)row * p.D + u0);
    float4 cv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.t > 0) cv = *crow;
    float cp[4] = {cv.x, cv.y, cv.z, cv.w}, o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float ig = gru::sigmoid(x_[i] + __ldg(p.bias + w0 + i));
      const float fg = gru::sigmoid(x_[4 + i] + __ldg(p.bias + w0 + 4 + i));
      const float gg = tanhf(x_[8 + i] + __ldg(p.bias + w0 + 8 + i));
      const float og = gru::sigmoid(x_[12 + i] + __ldg(p.bias + w0 + 12 + i));
      cp[i] = fg * cp[i] + ig * gg;
      o[i] = og * tanhf(cp[i]);
    }
    *crow = make_float4(cp[0], cp[1], cp[2], cp[3]);
    *orow = make_float4(o[0], o[1], o[2], o[3]);            // nonempty is 1 on a live row
  }

  __device__ __forceinline__ void post_epilogue(int) {}
};

// The skeleton's body under a name of its own, so profiles and SASS dumps name the LSTM step
__global__ void __launch_bounds__(tcg::cta_threads<SageLstmPolicy>, 1)
sage_lstm_step_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                      const SageLstmParams p) {
  tcg::tc_gemm_body<SageLstmPolicy, 0>(map_hi, map_lo, p);
}

// tcg::launch with sage_lstm_step_kernel as the production kernel (LNB_DBG bits 2 / 4 pick the skeleton's
// probe kernels, as there)
int launch_step(lnb_stream_t stream, const float* W_hi, const float* W_lo, int D, int items, const SageLstmParams& p) {
  const char* who = "sage_lstm_step";
  CUtensorMap map_hi, map_lo;
  int rc = tcg::make_weight_map(&map_hi, W_hi, 4 * D, 2 * D, who);
  if (rc != LNB_OK) return rc;
  rc = tcg::make_weight_map(&map_lo, W_lo, 4 * D, 2 * D, who);
  if (rc != LNB_OK) return rc;
  rc = tcg::sync_prof_buffer(who);
  if (rc != LNB_OK) return rc;
  const int skip = p.dbg & (tcg::SKIP_MMA | tcg::SKIP_TMA);
  auto kern = skip == 0                  ? sage_lstm_step_kernel
              : skip == tcg::SKIP_MMA    ? tcg::tc_gemm_probe_kernel<SageLstmPolicy, tcg::SKIP_MMA>
              : skip == tcg::SKIP_TMA    ? tcg::tc_gemm_probe_kernel<SageLstmPolicy, tcg::SKIP_TMA>
                                         : tcg::tc_gemm_probe_kernel<SageLstmPolicy, tcg::SKIP_MMA | tcg::SKIP_TMA>;
  const size_t smem = SageLstmPolicy::SMEM_BYTES;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  const int grid = tcg::persistent_grid(items);
  kern<<<grid, tcg::cta_threads<SageLstmPolicy>, smem, (cudaStream_t)stream>>>(map_hi, map_lo, p);
  lnb::count_launch();
  return lnb::finish_launch(who);
}

}  // namespace

extern "C" {

int lnb_sage_lstm_step(lnb_stream_t stream, const float* state, const int32_t* nn_idx, const float* nonempty,
                       const float* h, float* c, const float* W_hi, const float* W_lo, const float* bias, int B,
                       int N, int K, int E1, int D, int t, float* out) {
  LNB_REQUIRE(state && nn_idx && nonempty && c && W_hi && W_lo && bias && out, "sage_lstm_step: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && K >= 1 && E1 >= 1 && D >= 1, "sage_lstm_step: bad dims B=%d N=%d K=%d E1=%d D=%d",
              B, N, K, E1, D);
  LNB_REQUIRE(t >= 0 && t < K, "sage_lstm_step: step t=%d outside [0, K=%d)", t, K);
  if (D % 32 || D > LNB_MAX_WIDTH || E1 > LNB_MAX_E1) {
    lnb::set_err("sage_lstm_step: D=%d E1=%d outside the kernel (D %% 32 == 0, D <= %d, E1 <= %d)", D, E1, LNB_MAX_WIDTH,
                 LNB_MAX_E1);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE(t == 0 || h, "sage_lstm_step: h is null at step t=%d > 0", t);
  LNB_REQUIRE(((uintptr_t)state | (uintptr_t)h | (uintptr_t)c | (uintptr_t)out | (uintptr_t)W_hi |
               (uintptr_t)W_lo) % 16 == 0,
              "sage_lstm_step: state, h, c, out and W must be 16-byte aligned");
  LNB_REQUIRE(t == 0 || out != h, "sage_lstm_step: out must not alias h (other column tiles still read h)");
  LNB_REQUIRE(out != c, "sage_lstm_step: out must not alias c");
  LNB_REQUIRE((int64_t)B * N * E1 <= 0x7fffffff, "sage_lstm_step: B*N*E1 too large");
  const int rows = B * N * E1;
  if (rows == 0) return LNB_OK;
  SageLstmParams p{state, nn_idx, nonempty, h, c, bias, out, rows, N, K, E1, D, t, t == K - 1 ? 1 : 0,
                   tcg::debug_flags()};
  return launch_step(stream, W_hi, W_lo, D, lnb::ceil_div(rows, tcg::BM) * (4 * D / tcg::BN), p);
}

}  // extern "C"
