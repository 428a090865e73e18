// One GRU step as a policy of the persistent 3xTF32 wgmma skeleton (tc_gemm.cuh), shared by
// lnb_ggnn_update, lnb_mpnn_update and lnb_gpnn_partition_update.  They differ only in the message
// k-blocks their producers gather; Step supplies the rest of the skeleton contract.
//
// Work items are (row tile, part, column tile) over plain 128-row tiles of the B*N rows, column tiles
// innermost: the items of one row tile run on neighbouring CTAs at the same time, so they share the
// gathers in L2.  The GEMM is
//     G[r, :] = [msg(r) | h(r)] @ W^T,     W [4D, K]
// and its A operand is produced by the CUDA-core warps: the policy's message k-blocks, then the D/32
// k-blocks of the row of h.  W's rows hold the gate blocks r, z, n_in, n_h, interleaved so that a
// 16-column epilogue unit carries all four gates of 4 hidden units:
//     W row (u / 4) * 16 + g * 4 + u % 4 = gate g of hidden unit u
//     r:    [W_ir | W_hr]      z:    [W_iz | W_hz]      n_in: [W_in | 0]      n_h: [0 | W_hn]
// and the epilogue applies the GRU cell (the gate order of torch's CPU GRUCell):
//     r = sigmoid(G_r + b_r), z = sigmoid(G_z + b_z), n = tanh(G_nin + b_in + r * (G_nh + b_hn)),
//     h' = (h - n) * z + n
// and writes 4 contiguous h' values.
//
// A policy derives from Step<Policy, Params> (CRTP: the kernel's name keeps the policy's) and supplies
//   static int msg_kblocks(const Params&)         message k-blocks in front of the h blocks
//   void produce_msg(int kb, float (&v)[32])      message k-block kb of this thread's row; called for
//                                                 a live row only, with v zeroed
// It may replace (the default in brackets)
//   static int parts(const Params&)               parts per row tile [1]
//   static int col_tile(const Params&, int sub)   column tile of item sub [sub]
//   void begin_row(int sub)                       set-up after row, row_ok, b and n [nothing]
//   const float* h_row() const                    this thread's row of h [p.h, row stride D]
//   void write_row(int u0, const float (&o)[4], const float4& hv)
//                                                 h' of hidden units u0 .. u0 + 3 [p.out, row stride D]
// Params holds bias [4D] (interleaved like the rows of W), rows, N, D and dbg, and h and out unless
// h_row and write_row are replaced.
#pragma once
#include <float.h>

#include "tc_gemm.cuh"

namespace gru {

// non-zeros of ELL row `line` (t-major, stride N): the leading entries with a non-zero value
__device__ __forceinline__ int ell_count(const float* ell_val, int64_t line, int len, int N) {
  int cnt = 0;
  while (cnt < len && __ldg(ell_val + line + (int64_t)cnt * N) != 0.f) ++cnt;
  return cnt;
}

// avg: the reference's sum / (rowsum(A) + eps) on the 0/1 operator -- one correctly rounded reciprocal
__device__ __forceinline__ float row_weight(int cnt, int avg) {
  return avg ? __frcp_rn((float)cnt + FLT_EPSILON) : 1.f;
}

__device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

template <class Pol, class P>
struct Step {
  using Params = P;
  static constexpr int kStagesB = 3;
  static constexpr int kStagesA = 2;
  static constexpr size_t SMEM_BYTES = tcg::core_smem(kStagesB, kStagesA) + 1024 + 16;

  static __device__ __forceinline__ int parts(const Params&) { return 1; }
  static __device__ __forceinline__ int col_tile(const Params&, int sub) { return sub; }
  static __device__ __forceinline__ int n_tiles(const Params& p) { return 4 * p.D / tcg::BN; }
  static __device__ __forceinline__ int num_steps(const Params& p, int cta, int ncta) {
    const int t = ((p.rows + tcg::BM - 1) / tcg::BM) * Pol::parts(p) * n_tiles(p);
    return t > cta ? (t - cta + ncta - 1) / ncta : 0;
  }
  static __device__ __forceinline__ void decode(const Params& p, int cta, int ncta, int it, int& m_tile,
                                                int& sub) {
    const int item = cta + it * ncta, per = Pol::parts(p) * n_tiles(p);
    m_tile = item / per;
    sub = item - m_tile * per;
  }
  static __device__ __forceinline__ int num_kblocks(const Params& p, int) {
    return Pol::msg_kblocks(p) + p.D / tcg::BK;
  }
  static __device__ __forceinline__ void w_coords(const Params& p, int sub, int kb, int& col0, int& row0) {
    col0 = kb * tcg::BK;
    row0 = Pol::col_tile(p, sub) * tcg::BN;
  }

  const Params& p;
  const int r;
  int row, b, n;
  bool row_ok;

  __device__ Step(const Params& p_, uint8_t*, int tid)
      : p(p_), r(tid & 127), row(0), b(0), n(0), row_ok(false) {}

  __device__ __forceinline__ Pol& self() { return static_cast<Pol&>(*this); }

  __device__ __forceinline__ void begin_row(int) {}
  __device__ __forceinline__ const float* h_row() const { return p.h + (int64_t)row * p.D; }
  __device__ __forceinline__ void write_row(int u0, const float (&o)[4], const float4&) {
    *reinterpret_cast<float4*>(p.out + (int64_t)row * p.D + u0) = make_float4(o[0], o[1], o[2], o[3]);
  }

  __device__ __forceinline__ void step_begin(int m_tile, int sub, int, tcg::PhaseTimer&) {
    row = m_tile * tcg::BM + r;
    row_ok = row < p.rows;
    b = row_ok ? row / p.N : 0;
    n = row_ok ? row - b * p.N : 0;
    self().begin_row(sub);
  }

  __device__ __forceinline__ void produce(int, int kb, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = 0.f;
    if (!row_ok) return;
    const int hb = kb - Pol::msg_kblocks(p);
    if (hb >= 0) {                                     // the h columns
      const float4* src = reinterpret_cast<const float4*>(self().h_row() + hb * tcg::BK);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 t = __ldg(src + j);
        v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
      }
      return;
    }
    self().produce_msg(kb, v);
  }

  __device__ __forceinline__ void pre_epilogue(int) {}

  __device__ __forceinline__ void store(int sub, int col, const float (&x)[tcg::EW]) {
    if (!row_ok) return;
    const int w0 = Pol::col_tile(p, sub) * tcg::BN + col;   // first W row of this unit
    const int u0 = w0 / 4;                                  // its first hidden unit
    const float4 hv = __ldg(reinterpret_cast<const float4*>(self().h_row() + u0));
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
    self().write_row(u0, o, hv);
  }

  __device__ __forceinline__ void post_epilogue(int) {}
};

}  // namespace gru
