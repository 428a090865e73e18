// MPNN with the edge-network message function (reference: model/mpnn.py:131-191), receiver i,
// neighbour j, bond channel e, A_e = (L_e != 0):
//     agg_e[i] = w_i sum_j A_e[i, j] ( relu(W1a_e h_j + W1b_e h_i + b1_e) W2_e^T + b2_e )
// with w_i = 1 (sum) or 1 / (nnz_e(i) + FLT_EPSILON) (avg).  The second edge layer is linear, so it
// moves out of the sum:
//     agg_e[i] = S_e[i] W2_e^T + (w_i nnz_e(i)) b2_e,    S_e[i] = w_i sum_j A_e[i, j] relu(P_e[j] + Q_e[i])
// with P_e = h W1a_e^T and Q_e = h W1b_e^T + b1_e (64 wide, the edge network's hidden width), and the
// GRU input product folds W_ih into W2 and b2:
//     gi = [S_0 | ... | S_{E1-1} | deg] F^T + b_ih,   F = [W_ih,e W2_e]_e | [W_ih,e b2_e]_e,
//     deg[i, e] = w_i nnz_e(i)
//
// lnb_mpnn_update is the GRU step of gru_step.cuh with these k-blocks, produced by the CUDA-core warps:
//     k-blocks 0 .. 2 E1 - 1    32 columns of S_e (e = kb / 2): the producer thread of row i holds its own
//                               32 Q values and, for each non-zero j of its ELL row, adds P_e[j], applies
//                               the ReLU and accumulates with weight w_i
//     k-block 2 E1              the degree block: column e holds w_i nnz_e(i), the rest are zero
//     k-blocks past it          the row of h
// S never exists in HBM.  lnb_mpnn_edge_aggregate writes S with the same arithmetic for the training
// path, and lnb_mpnn_edge_aggregate_backward is its adjoint.
#include "gru_step.cuh"

namespace {

constexpr int MP_H = 64;                  // edge-network hidden width (model/mpnn.py:60)
constexpr int MP_PQ = 2 * MP_H;           // PQ columns per channel: 64 P, then 64 Q

struct MpnnUpdateParams {
  const float* PQ;         // [rows, E1*128]
  const float* h;          // [rows, D]
  const float* ell_val;    // [B, E1, N, N]  t-major ELL rows (lnb_graph_prepare)
  const uint8_t* ell_idx;  // [B, E1, N, N]
  const int32_t* ell_max;  // [B, E1]
  const float* bias;       // [4D] interleaved like the rows of W
  float* out;              // [rows, D]
  int rows, N, D, E1, avg;
  int dbg;
};

struct MpnnUpdatePolicy : gru::Step<MpnnUpdatePolicy, MpnnUpdateParams> {
  using Step::Step;
  static __device__ __forceinline__ int msg_kblocks(const Params& p) { return 2 * p.E1 + 1; }

  __device__ __forceinline__ void produce_msg(int kb, float (&v)[32]) {
    if (kb == 2 * p.E1) {                                 // degree block: w_i nnz_e(i)
      for (int e = 0; e < p.E1; ++e) {
        const int64_t line = ((int64_t)(b * p.E1 + e) * p.N) * p.N + n;
        const int cnt = gru::ell_count(p.ell_val, line, __ldg(p.ell_max + b * p.E1 + e), p.N);
#pragma unroll
        for (int j = 0; j < LNB_MAX_E1; ++j)
          if (j == e) v[j] = gru::row_weight(cnt, p.avg) * (float)cnt;
      }
      return;
    }
    const int e = kb >> 1, c0 = (kb & 1) * 32;
    const int64_t line = ((int64_t)(b * p.E1 + e) * p.N) * p.N + n;
    const int cnt = gru::ell_count(p.ell_val, line, __ldg(p.ell_max + b * p.E1 + e), p.N);
    if (cnt == 0) return;
    const float w = gru::row_weight(cnt, p.avg);
    const int ld = p.E1 * MP_PQ;
    float q[32];
    const float4* qs = reinterpret_cast<const float4*>(p.PQ + (int64_t)row * ld + e * MP_PQ + MP_H + c0);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 t = __ldg(qs + j);
      q[4 * j] = t.x; q[4 * j + 1] = t.y; q[4 * j + 2] = t.z; q[4 * j + 3] = t.w;
    }
    const float* pb = p.PQ + (int64_t)b * p.N * ld + e * MP_PQ + c0;
    for (int t = 0; t < cnt; ++t) {
      const int m = __ldg(p.ell_idx + line + (int64_t)t * p.N);
      const float4* src = reinterpret_cast<const float4*>(pb + (int64_t)m * ld);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 x = __ldg(src + j);
        v[4 * j] = fmaf(w, fmaxf(x.x + q[4 * j], 0.f), v[4 * j]);
        v[4 * j + 1] = fmaf(w, fmaxf(x.y + q[4 * j + 1], 0.f), v[4 * j + 1]);
        v[4 * j + 2] = fmaf(w, fmaxf(x.z + q[4 * j + 2], 0.f), v[4 * j + 2]);
        v[4 * j + 3] = fmaf(w, fmaxf(x.w + q[4 * j + 3], 0.f), v[4 * j + 3]);
      }
    }
  }
};

// ---- training path: S and its adjoint, one thread per (row, channel, hidden column) --------------
struct EdgeAggParams {
  const float* PQ;                  // [rows, E1*128]
  const float* ell_val;             // lnb_graph_prepare of the operators
  const uint8_t* ell_idx;
  const int32_t* ell_max;
  const float* ellT_val;            // lnb_graph_prepare of the transposed operators (backward only)
  const uint8_t* ellT_idx;
  const int32_t* ellT_max;
  const float* gS;                  // [rows, E1*64] (backward only)
  float* out;                       // S [rows, E1*64] (forward) or gPQ [rows, E1*128] (backward)
  int rows, N, E1, avg;
};

// S[i, e*64 + c] = sum over the ELL row of i, in ELL order, of fmaf(w_i, relu(P[j] + Q[i]), .):
// the producer's arithmetic of lnb_mpnn_update
__global__ void edge_aggregate_kernel(const EdgeAggParams p) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)p.rows * p.E1 * MP_H) return;
  const int c = (int)(idx % MP_H);
  const int e = (int)((idx / MP_H) % p.E1);
  const int row = (int)(idx / ((int64_t)MP_H * p.E1));
  const int b = row / p.N, n = row - b * p.N;
  const int ld = p.E1 * MP_PQ;
  const int64_t line = ((int64_t)(b * p.E1 + e) * p.N) * p.N + n;
  const int cnt = gru::ell_count(p.ell_val, line, __ldg(p.ell_max + b * p.E1 + e), p.N);
  const float w = gru::row_weight(cnt, p.avg);
  const float q = __ldg(p.PQ + (int64_t)row * ld + e * MP_PQ + MP_H + c);
  const float* pc = p.PQ + (int64_t)b * p.N * ld + e * MP_PQ + c;
  float v = 0.f;
  for (int t = 0; t < cnt; ++t) {
    const int m = __ldg(p.ell_idx + line + (int64_t)t * p.N);
    v = fmaf(w, fmaxf(__ldg(pc + (int64_t)m * ld) + q, 0.f), v);
  }
  p.out[(int64_t)row * p.E1 * MP_H + e * MP_H + c] = v;
}

// gQ[i] = sum_j A[i, j] w_i [P[j] + Q[i] > 0] gS[i]             (the ELL row of i)
// gP[j] = sum_i A[i, j] w_i [P[j] + Q[i] > 0] gS[i]             (the ELL row of j in the transposed pattern)
// Each output element is one thread's sum in ELL order: no atomics, deterministic.
__global__ void edge_aggregate_backward_kernel(const EdgeAggParams p) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)p.rows * p.E1 * MP_H) return;
  const int c = (int)(idx % MP_H);
  const int e = (int)((idx / MP_H) % p.E1);
  const int row = (int)(idx / ((int64_t)MP_H * p.E1));
  const int b = row / p.N, n = row - b * p.N;
  const int ld = p.E1 * MP_PQ, lds = p.E1 * MP_H;
  const int64_t base = ((int64_t)(b * p.E1 + e) * p.N) * p.N;
  const int len = __ldg(p.ell_max + b * p.E1 + e);
  const float* Pc = p.PQ + (int64_t)b * p.N * ld + e * MP_PQ + c;        // P column c of graph b
  const float* Qc = Pc + MP_H;
  const float* gc = p.gS + (int64_t)b * p.N * lds + e * MP_H + c;
  // gQ of row n
  const int cnt = gru::ell_count(p.ell_val, base + n, len, p.N);
  const float w = gru::row_weight(cnt, p.avg);
  const float qn = __ldg(Qc + (int64_t)n * ld), gn = __ldg(gc + (int64_t)n * lds);
  float gq = 0.f;
  for (int t = 0; t < cnt; ++t) {
    const int m = __ldg(p.ell_idx + base + n + (int64_t)t * p.N);
    if (__ldg(Pc + (int64_t)m * ld) + qn > 0.f) gq = fmaf(w, gn, gq);
  }
  // gP of row n: the receivers i with A[i, n] != 0
  const float pn = __ldg(Pc + (int64_t)n * ld);
  const int cntT = gru::ell_count(p.ellT_val, base + n, __ldg(p.ellT_max + b * p.E1 + e), p.N);
  float gp = 0.f;
  for (int t = 0; t < cntT; ++t) {
    const int i = __ldg(p.ellT_idx + base + n + (int64_t)t * p.N);
    if (pn + __ldg(Qc + (int64_t)i * ld) > 0.f) {
      const float wi = gru::row_weight(gru::ell_count(p.ell_val, base + i, len, p.N), p.avg);
      gp = fmaf(wi, __ldg(gc + (int64_t)i * lds), gp);
    }
  }
  float* o = p.out + (int64_t)row * ld + e * MP_PQ + c;
  o[0] = gp;
  o[MP_H] = gq;
}

int edge_aggregate_checks(const char* who, const float* PQ, const float* ell_val, const uint8_t* ell_idx,
                          const int32_t* ell_max, const float* out, int B, int N, int E1) {
  LNB_REQUIRE(PQ && ell_val && ell_idx && ell_max && out, "%s: null pointer", who);
  LNB_REQUIRE(B >= 0 && N >= 1 && E1 >= 1, "%s: bad dims B=%d N=%d E1=%d", who, B, N, E1);
  if (N > LNB_MAX_N_ELL || E1 > LNB_MAX_E1) {
    lnb::set_err("%s: N=%d E1=%d outside the kernel (N <= %d, E1 <= %d)", who, N, E1, LNB_MAX_N_ELL, LNB_MAX_E1);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE((int64_t)B * N * E1 * MP_PQ <= 0x7fffffff, "%s: B*N too large", who);
  return LNB_OK;
}

}  // namespace

extern "C" {

int lnb_mpnn_update(lnb_stream_t stream, const float* PQ, const float* h, const float* ell_val,
                    const uint8_t* ell_idx, const int32_t* ell_max, const float* W_hi, const float* W_lo,
                    const float* bias, int B, int N, int D, int E1, int avg, float* out) {
  LNB_REQUIRE(PQ && h && ell_val && ell_idx && ell_max && W_hi && W_lo && bias && out,
              "mpnn_update: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && D >= 1 && E1 >= 1, "mpnn_update: bad dims B=%d N=%d D=%d E1=%d", B, N, D,
              E1);
  if (N > LNB_MAX_N_ELL || D % 32 || D < 32 || D > LNB_MAX_WIDTH || E1 > LNB_MAX_E1) {
    lnb::set_err("mpnn_update: N=%d D=%d E1=%d outside the kernel (N <= %d, D %% 32 == 0, 32 <= D <= %d, "
                 "E1 <= %d)", N, D, E1, LNB_MAX_N_ELL, LNB_MAX_WIDTH, LNB_MAX_E1);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE(((uintptr_t)PQ | (uintptr_t)h | (uintptr_t)out | (uintptr_t)W_hi | (uintptr_t)W_lo) % 16 == 0,
              "mpnn_update: PQ, h, out and W must be 16-byte aligned");
  LNB_REQUIRE(out != h, "mpnn_update: out must not alias h (the epilogue reads h after other tiles wrote)");
  LNB_REQUIRE((int64_t)B * N * E1 * MP_PQ <= 0x7fffffff, "mpnn_update: B*N too large");
  const int rows = B * N;
  if (rows == 0) return LNB_OK;
  MpnnUpdatePolicy::Params p{PQ, h, ell_val, ell_idx, ell_max, bias, out, rows, N, D, E1, avg ? 1 : 0,
                             tcg::debug_flags()};
  return tcg::launch<MpnnUpdatePolicy>(stream, W_hi, W_lo, 4 * D, MP_H * E1 + 32 + D, MpnnUpdatePolicy::SMEM_BYTES,
                                       lnb::ceil_div(rows, tcg::BM) * (4 * D / tcg::BN), p, "mpnn_update");
}

int lnb_mpnn_edge_aggregate(lnb_stream_t stream, const float* PQ, const float* ell_val, const uint8_t* ell_idx,
                            const int32_t* ell_max, int B, int N, int E1, int avg, float* S) {
  const int rc = edge_aggregate_checks("mpnn_edge_aggregate", PQ, ell_val, ell_idx, ell_max, S, B, N, E1);
  if (rc != LNB_OK) return rc;
  const int64_t total = (int64_t)B * N * E1 * MP_H;
  if (total == 0) return LNB_OK;
  EdgeAggParams p{PQ, ell_val, ell_idx, ell_max, nullptr, nullptr, nullptr, nullptr, S, B * N, N, E1,
                  avg ? 1 : 0};
  edge_aggregate_kernel<<<lnb::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch("mpnn_edge_aggregate");
}

int lnb_mpnn_edge_aggregate_backward(lnb_stream_t stream, const float* PQ, const float* gS, const float* ell_val,
                                     const uint8_t* ell_idx, const int32_t* ell_max, const float* ellT_val,
                                     const uint8_t* ellT_idx, const int32_t* ellT_max, int B, int N, int E1,
                                     int avg, float* gPQ) {
  int rc = edge_aggregate_checks("mpnn_edge_aggregate_backward", PQ, ell_val, ell_idx, ell_max, gPQ, B, N, E1);
  if (rc != LNB_OK) return rc;
  LNB_REQUIRE(gS && ellT_val && ellT_idx && ellT_max, "mpnn_edge_aggregate_backward: null pointer");
  LNB_REQUIRE(gPQ != PQ && gPQ != gS, "mpnn_edge_aggregate_backward: gPQ must not alias PQ or gS");
  const int64_t total = (int64_t)B * N * E1 * MP_H;
  if (total == 0) return LNB_OK;
  EdgeAggParams p{PQ, ell_val, ell_idx, ell_max, ellT_val, ellT_idx, ellT_max, gS, gPQ, B * N, N, E1,
                  avg ? 1 : 0};
  edge_aggregate_backward_kernel<<<lnb::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch("mpnn_edge_aggregate_backward");
}

}  // extern "C"
