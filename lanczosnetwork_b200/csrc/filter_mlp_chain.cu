// Ritz-value filter MLPs of ALL layers in one persistent wgmma kernel
// (reference: model/lanczos_net.py:47-58 the per-layer Sequential, :109-113 its application to
// the B*K rows of Ritz-value powers).
//
// An item is (128-row tile, layer): four Linear stages S -> Hd -> Hd -> Hd -> S.
//   * The hidden stages are accumulator lifetimes ("steps") of the 3xTF32 skeleton in tc_gemm.cuh:
//     two per item for S <= 8, four for S > 8.
//   * The S-wide first stage (S <= 8 inputs) is evaluated by the CUDA cores in plain fp32 inside
//     produce(): k-block kb of stage 1 is columns [32 kb, 32 kb + 32) of ReLU(W1 t + b1), computed
//     in registers from the row's powers and written straight into the operand ring -- a tensor-core
//     step for K = 8 would cost a full accumulator hand-over for 2 % of the flops.  (S > 8 runs it
//     as an MMA step whose producers read the powers.)
//   * Every later hidden stage takes its operand from the previous step's accumulators: the
//     consumers apply bias + ReLU to their fragments and write the next step's k-blocks themselves
//     (operand_from_acc), so activations never leave the registers and the tensor cores' operand
//     ring.
//   * The S-wide output stage (S <= 8 outputs) runs in the epilogue of the last hidden stage: the
//     thread that owns a row applies bias + ReLU to each 16-column chunk of the drain and folds it
//     into its S dot products with the stage-3 weights, in ascending column order (a 128-wide MMA
//     for 8 columns would be another full hand-over).  (S > 8 runs it as an MMA step.)
#include "tc_gemm.cuh"

namespace {

constexpr int S0MAX = 8;                 // first / output stage widths the CUDA cores handle

struct ChainPolicy {
  static constexpr int kStagesB = 2;
  static constexpr int kStagesA = 4;     // one A stage per k-block of a 128-wide consumer-written operand
  struct Params {
    const float* table;     // [Rall, S]  powers of the Ritz values
    const int32_t* rowmap;  // [Rall]     compact list of rows to evaluate (nullptr: all rows)
    const int32_t* nrows;   // [1]        number of valid entries in rowmap (nullptr: Rall)
    const float* W_hi;      // [L * (3*Hd + S), Hd] split weights (the CUDA-core stages read hi + lo)
    const float* W_lo;
    const float* bias_all;  // [L * (3*Hd + S)]
    float* coeff;           // [L, Rall, S]
    int Rall, L, S, Hd;
    int dbg;                // debug experiment flags (LNB_DBG), 0 in production
  };
  // sub = layer * 4 + stage
  // S <= 8: stages 0 and 3 run on the CUDA cores, S > 8: all four stages are MMA steps
  static __device__ __forceinline__ bool mma0(const Params& p) { return p.S > S0MAX; }
  static __device__ __forceinline__ int first_stage(const Params& p) { return mma0(p) ? 0 : 1; }
  static __device__ __forceinline__ int steps_per_item(const Params& p) { return mma0(p) ? 4 : 2; }
  static __device__ __forceinline__ int rows(const Params& p) { return p.nrows ? __ldg(p.nrows) : p.Rall; }
  static __device__ __forceinline__ int ntile(const Params& p) { return (rows(p) + tcg::BM - 1) / tcg::BM; }
  // Items are numbered layer-major, and every CTA runs one contiguous range of them: a CTA's
  // consecutive items share the layer, so the CUDA-core stages' weights are staged once per
  // layer change (one or two per CTA) instead of at almost every item.  (All layers' weights sit
  // in L2 together.)
  static __device__ __forceinline__ void item_range(const Params& p, int cta, int ncta, int& first,
                                                    int& count) {
    const int items = ntile(p) * p.L, base = items / ncta, rem = items % ncta;
    count = base + (cta < rem ? 1 : 0);
    first = cta * base + min(cta, rem);
  }
  static __device__ __forceinline__ int num_steps(const Params& p, int cta, int ncta) {
    int first, count;
    item_range(p, cta, ncta, first, count);
    return count * steps_per_item(p);
  }
  static __device__ __forceinline__ void decode(const Params& p, int cta, int ncta, int it,
                                                int& m_tile, int& sub) {
    const int per = steps_per_item(p), nt = ntile(p);
    int first, count;
    item_range(p, cta, ncta, first, count);
    const int item = first + it / per;
    m_tile = item % nt;
    sub = (item / nt) * 4 + first_stage(p) + it % per;
  }
  static __device__ __forceinline__ int num_kblocks(const Params& p, int sub) {
    return (sub & 3) == 0 ? 1 : p.Hd / tcg::BK;
  }
  static __device__ __forceinline__ int w_row0(const Params& p, int layer, int stage) {
    return layer * (3 * p.Hd + p.S) + stage * p.Hd;
  }
  static __device__ __forceinline__ void w_coords(const Params& p, int sub, int kb, int& col0, int& row0) {
    col0 = kb * tcg::BK;
    row0 = w_row0(p, sub >> 2, sub & 3);
  }
  // Every hidden stage after the item's first MMA step multiplies the previous step's activations,
  // written into the A ring by the consumers: ReLU(acc + b), the operations the epilogue used to
  // apply before the producers read the row back.  b is the layer's bias of step sub's stage,
  // staged in shared memory by step_begin.
  static __device__ __forceinline__ bool operand_from_acc(const Params& p, int sub) {
    return (sub & 3) > first_stage(p);
  }
  static __device__ __forceinline__ float acc_operand(const Params&, const uint8_t* policy_smem, int sub, int col,
                                                      float x) {
    const float* bs = reinterpret_cast<const float*>(policy_smem) + BS_OFF;
    return fmaxf(x + bs[(sub & 3) * tcg::BN + col], 0.f);
  }

  const Params& p;
  const int tid, r;
  // shared memory (floats): W1s | W3s | bs | b3s
  static constexpr int BS_OFF = 2 * tcg::BN * S0MAX;
  float* W1s;               // [BN][S0MAX] first-stage weights (hi + lo)
  float* W3s;               // [BN][S0MAX] output-stage weights (hi + lo), transposed: W3s[c][s] = W3[s][c]
  float* bs;                // [3][BN]     biases of stages 0, 1, 2 (b1 = bs[0])
  float* b3s;               // [S0MAX]
  int src, cur_layer;
  float tv[S0MAX];          // this row's powers (first stage, S <= 8)
  float o[S0MAX];           // this row's output-stage sums (S <= 8)

  static size_t smem_bytes() {
    return (BS_OFF + 3 * tcg::BN + S0MAX) * 4;
  }

  __device__ ChainPolicy(const Params& p_, uint8_t* smem, int tid_)
      : p(p_), tid(tid_), r(tid_ & 127), src(-1), cur_layer(-1) {
    W1s = reinterpret_cast<float*>(smem);
    W3s = W1s + tcg::BN * S0MAX;
    bs = W1s + BS_OFF;
    b3s = bs + 3 * tcg::BN;
  }

  __device__ void step_begin(int m_tile, int sub, int, tcg::PhaseTimer& tm) {
    const int layer = sub >> 2;
    if ((sub & 3) != first_stage(p)) return;
    const int i = m_tile * tcg::BM + r;
    src = i < rows(p) ? (p.rowmap ? __ldg(p.rowmap + i) : i) : -1;
    // Stage this layer's hidden biases (read by the consumers' hand-overs and by store()) and, for
    // S <= 8, W1 and W3 (hi + lo) and b3.  The consumers read the previous layer's biases for the
    // last time before the drain these producers have read by now.
    if (layer != cur_layer) {
      tcg::producers_sync<ChainPolicy>();
      const int row0 = w_row0(p, layer, 0), row3 = w_row0(p, layer, 3);
      if (!mma0(p)) {
#pragma unroll 4
        for (int e = tid; e < p.Hd * S0MAX; e += tcg::producer_threads<ChainPolicy>) {
          const int c = e / S0MAX, k = e - c * S0MAX;
          const int64_t o1 = (int64_t)(row0 + c) * p.Hd + k;
          W1s[e] = (k < p.S) ? __ldg(p.W_hi + o1) + __ldg(p.W_lo + o1) : 0.f;
          const int64_t o3 = (int64_t)(row3 + k) * p.Hd + c;
          W3s[e] = (k < p.S) ? __ldg(p.W_hi + o3) + __ldg(p.W_lo + o3) : 0.f;
        }
        if (tid < S0MAX) b3s[tid] = tid < p.S ? __ldg(p.bias_all + row3 + tid) : 0.f;
      }
      for (int e = tid; e < 3 * tcg::BN; e += tcg::producer_threads<ChainPolicy>) {
        const int st = e / tcg::BN, c = e - st * tcg::BN;
        bs[e] = c < p.Hd ? __ldg(p.bias_all + row0 + st * p.Hd + c) : 0.f;
      }
      tcg::producers_sync<ChainPolicy>();
      cur_layer = layer;
      tm.lap(1);
    }
    if (mma0(p)) return;
#pragma unroll
    for (int k = 0; k < S0MAX; ++k)
      tv[k] = (src >= 0 && k < p.S) ? __ldg(p.table + (int64_t)src * p.S + k) : 0.f;
  }

  __device__ __forceinline__ void produce(int sub, int kb, float (&v)[32]) {
    if ((sub & 3) == 0) {                                 // S > 8: the MMA first stage reads the powers
#pragma unroll
      for (int j = 0; j < 32; ++j)
        v[j] = (src >= 0 && j < p.S) ? __ldg(p.table + (int64_t)src * p.S + j) : 0.f;
      return;
    }
    // ---- first stage on the CUDA cores (S <= 8): columns [32 kb, 32 kb + 32) of ReLU(W1 t + b1) ----
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int c = kb * tcg::BK + j;
      const float4* wr = reinterpret_cast<const float4*>(W1s + c * S0MAX);
      const float4 wa = wr[0], wb = wr[1];
      float a = bs[c];
      a = fmaf(tv[0], wa.x, a); a = fmaf(tv[1], wa.y, a); a = fmaf(tv[2], wa.z, a); a = fmaf(tv[3], wa.w, a);
      a = fmaf(tv[4], wb.x, a); a = fmaf(tv[5], wb.y, a); a = fmaf(tv[6], wb.z, a); a = fmaf(tv[7], wb.w, a);
      v[j] = fmaxf(a, 0.f);
    }
  }
  __device__ __forceinline__ void pre_epilogue(int) {}
  __device__ __forceinline__ void post_epilogue(int) {}

  // Only the item's last step is drained: stage 3 (S > 8) or stage 2 (S <= 8).
  __device__ __forceinline__ void store(int sub, int col, const float (&x)[tcg::EW]) {
    const int layer = sub >> 2, stage = sub & 3;
    if (stage == 3) {
      if (src < 0 || col >= p.S) return;
      const float* bias = p.bias_all + w_row0(p, layer, stage);
      float* dst = p.coeff + ((int64_t)layer * p.Rall + src) * p.S;
#pragma unroll
      for (int j = 0; j < tcg::EW; ++j)
        if (col + j < p.S) dst[col + j] = x[j] + __ldg(bias + col + j);
      return;
    }
    // ---- output stage on the CUDA cores (S <= 8): coeff = W3 ReLU(acc + b2) + b3 ------------------
    // The chunks arrive in ascending column order, so every sum runs over the columns in order.
    if (col >= p.Hd) return;
    const float* b2 = bs + 2 * tcg::BN;
    if (col == 0) {
#pragma unroll
      for (int s = 0; s < S0MAX; ++s) o[s] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < tcg::EW; ++j) {
      const float y = fmaxf(x[j] + b2[col + j], 0.f);
      const float4* wr = reinterpret_cast<const float4*>(W3s + (col + j) * S0MAX);
      const float4 wa = wr[0], wb = wr[1];
      o[0] = fmaf(y, wa.x, o[0]); o[1] = fmaf(y, wa.y, o[1]);
      o[2] = fmaf(y, wa.z, o[2]); o[3] = fmaf(y, wa.w, o[3]);
      o[4] = fmaf(y, wb.x, o[4]); o[5] = fmaf(y, wb.y, o[5]);
      o[6] = fmaf(y, wb.z, o[6]); o[7] = fmaf(y, wb.w, o[7]);
    }
    if (col + tcg::EW < p.Hd || src < 0) return;
    float* dst = p.coeff + ((int64_t)layer * p.Rall + src) * p.S;
#pragma unroll
    for (int s = 0; s < S0MAX; ++s)
      if (s < p.S) dst[s] = o[s] + b3s[s];
  }
};

// Compact list of the (graph, k) rows whose Ritz vector is not identically zero.  The forward runs it
// between the prepare pass and the chain, so the list is written coalesced: a warp writes the k_eff
// consecutive entries of one graph (a thread writing its own graph's entries stores 32 scattered
// words per instruction and took 15 us at B = 1024 on an H100 at 700 W, against 7 us now).
__global__ void __launch_bounds__(1024)
ritz_rowmap_kernel(const int32_t* __restrict__ gext, int B, int K, int32_t* __restrict__ rowmap,
                   int32_t* __restrict__ nrows) {
  __shared__ int warp_sums[32];
  __shared__ int gbase[1024], gk[1024];
  __shared__ int running;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) running = 0;
  __syncthreads();
  for (int b0 = 0; b0 < B; b0 += 1024) {
    const int b = b0 + tid;
    int k = (b < B) ? min(gext[b * 2 + 1], K) : 0;
    int incl = k;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = warp_sums[lane], wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += t;
      }
      warp_sums[lane] = wi - w;          // exclusive prefix of the warp totals
    }
    __syncthreads();
    const int base = running + warp_sums[warp] + incl - k;
    gbase[tid] = base;
    gk[tid] = k;
    __syncthreads();
    if (tid == 1023) running = base + k;
    for (int j = warp; j < 1024 && b0 + j < B; j += 32)
      for (int i = lane; i < gk[j]; i += 32) rowmap[gbase[j] + i] = (b0 + j) * K + i;
    __syncthreads();
  }
  if (tid == 0) nrows[0] = running;
}

}  // namespace

extern "C" {

int lnb_ritz_rowmap(lnb_stream_t stream, const int32_t* gext, int B, int K, int32_t* rowmap,
                    int32_t* nrows) {
  LNB_REQUIRE(gext && rowmap && nrows, "ritz_rowmap: null pointer");
  LNB_REQUIRE(B >= 0 && K >= 1, "ritz_rowmap: bad dims");
  ritz_rowmap_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(gext, B, K, rowmap, nrows);
  lnb::count_launch();
  return lnb::finish_launch("ritz_rowmap");
}

int lnb_ritz_filter_mlp(lnb_stream_t stream, const float* table, const int32_t* rowmap,
                        const int32_t* nrows, const float* W_hi, const float* W_lo,
                        const float* bias_all, int Rall, int L, int S, int Hd, float* coeff) {
  return lnb_ritz_filter_mlp_ctas(stream, table, rowmap, nrows, W_hi, W_lo, bias_all, Rall, L, S, Hd,
                                  coeff, 0);
}

int lnb_ritz_filter_mlp_ctas(lnb_stream_t stream, const float* table, const int32_t* rowmap,
                             const int32_t* nrows, const float* W_hi, const float* W_lo,
                             const float* bias_all, int Rall, int L, int S, int Hd, float* coeff,
                             int ctas) {
  LNB_REQUIRE(table && W_hi && W_lo && bias_all && coeff, "ritz_filter_mlp: null pointer");
  LNB_REQUIRE((rowmap == nullptr) == (nrows == nullptr), "ritz_filter_mlp: rowmap and nrows go together");
  LNB_REQUIRE(Rall >= 0 && L >= 1 && S >= 1 && Hd >= 1 && ctas >= 0, "ritz_filter_mlp: bad dims");
  if (S > LNB_FILTER_MLP_MAX_S || Hd % 32 != 0 || Hd > LNB_MAX_WIDTH) {
    lnb::set_err("ritz_filter_mlp: unsupported shape S=%d hidden=%d (needs S<=32, hidden%%32==0, hidden<=128)", S, Hd);
    return LNB_ERR_UNSUPPORTED;
  }
  if (Rall == 0) return LNB_OK;
  const size_t smem = tcg::core_smem(ChainPolicy::kStagesB, ChainPolicy::kStagesA) + 1024 + ChainPolicy::smem_bytes();
  ChainPolicy::Params p{table, rowmap, nrows, W_hi, W_lo, bias_all, coeff, Rall, L, S, Hd, tcg::debug_flags()};
  return tcg::launch<ChainPolicy>(stream, W_hi, W_lo, L * (3 * Hd + S), Hd, smem, lnb::ceil_div(Rall, tcg::BM) * L, p,
                                  "ritz_filter_mlp", ctas);
}

}  // extern "C"
