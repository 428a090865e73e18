// Set2Vec readout of MPNN (reference: model/set2set.py:8-100, model/mpnn.py:198-207) for every graph of
// the batch, followed by output_func, in one launch.  Per graph, with X the node states of its set (the
// masked nodes, or all N nodes without a mask), hidden = 0 [2D], mem = 0 [D], and per step:
//     f, i, o = sigmoid(Wg_{f,i,o} hidden + bg_{f,i,o}),  c = tanh(Wg_m hidden + bg_m)   (Set2SetLSTM)
//     mem = f * mem + i * c,  h = o * tanh(mem)
//     u = h W_1                                          (W_1 [D, D] used as [in, out])
//     e_n = tanh(u + x_n) . W_2                          over the nodes n of the set
//     a = softmax(e) (max subtracted),  read = sum_n a_n x_n  (0 for an empty set)
//     hidden = [h | read]
// and finally score = hidden W_out^T + b_out.
//
// fp32 on the CUDA cores.  A CTA owns G graphs and stages their node states in shared memory; the gate
// weights (4D x 2D, 512 KB at D = 128) do not fit on chip and are streamed from L2 once per step for all
// G graphs, transposed ([2D, 4D]) so consecutive threads read consecutive gate rows.  Every sum runs in
// a fixed order: repeated launches are bit-identical.
#include <float.h>
#include <math.h>

#include "common.cuh"

namespace {

constexpr int S2V_GMAX = 8;
constexpr int S2V_THREADS = 512;
constexpr size_t S2V_SMEM_MAX = 200 * 1024;

struct S2vParams {
  const float* X;          // [B, N, D]
  const uint8_t* mask;     // [B, N] or null
  const float* WgT;        // [2D, 4D]: column r = gate row r (forget, input, output, memory blocks)
  const float* bg;         // [4D]
  const float* W1;         // [D, D]
  const float* W2;         // [D]
  const float* Wout;       // [P, 2D]
  const float* bout;       // [P]
  float* score;            // [B, P]
  int B, N, D, P, steps, G;
};

__host__ __device__ inline size_t s2v_smem_floats(int N, int D, int G) {
  // x [G][N][D], hidden [G][2D], mem [G][D], gates [G][4D], u [G][D], energy / weight [G][N], in-set [G][N]
  return (size_t)G * ((size_t)N * D + 8 * D + 2 * N);
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

__global__ void __launch_bounds__(S2V_THREADS) set2vec_kernel(const S2vParams p) {
  extern __shared__ __align__(16) float sm[];
  const int N = p.N, D = p.D, G = p.G, D2 = 2 * D, D4 = 4 * D;
  float* xs = sm;                                   // [G][N][D]
  float* hid = xs + (size_t)G * N * D;              // [G][2D]
  float* mem = hid + G * D2;                        // [G][D]
  float* gate = mem + G * D;                        // [G][4D]
  float* us = gate + G * D4;                        // [G][D]
  float* en = us + G * D;                           // [G][N]
  float* ins = en + G * N;                          // [G][N]  1 = node in the set
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = S2V_THREADS / 32;
  const int g0 = blockIdx.x * G;
  const int ng = min(G, p.B - g0);

  for (int i = tid; i < ng * N * D; i += S2V_THREADS) xs[i] = __ldg(p.X + (int64_t)g0 * N * D + i);
  for (int i = tid; i < ng * N; i += S2V_THREADS)
    ins[i] = (p.mask == nullptr || __ldg(p.mask + (int64_t)g0 * N + i) != 0) ? 1.f : 0.f;
  for (int i = tid; i < G * D2; i += S2V_THREADS) hid[i] = 0.f;
  for (int i = tid; i < G * D; i += S2V_THREADS) mem[i] = 0.f;
  __syncthreads();

  for (int step = 0; step < p.steps; ++step) {
    // gate pre-activations: thread r owns gate row r for all graphs of the CTA
    for (int r = tid; r < D4; r += S2V_THREADS) {
      float acc[S2V_GMAX];
      const float br = __ldg(p.bg + r);
#pragma unroll
      for (int g = 0; g < S2V_GMAX; ++g) acc[g] = br;
      for (int k = 0; k < D2; ++k) {
        const float w = __ldg(p.WgT + (int64_t)k * D4 + r);
#pragma unroll
        for (int g = 0; g < S2V_GMAX; ++g)
          if (g < ng) acc[g] = fmaf(w, hid[g * D2 + k], acc[g]);
      }
#pragma unroll
      for (int g = 0; g < S2V_GMAX; ++g)
        if (g < ng) gate[g * D4 + r] = acc[g];
    }
    __syncthreads();
    // LSTM cell: h goes to the first half of hidden
    for (int i = tid; i < ng * D; i += S2V_THREADS) {
      const int g = i / D, d = i - g * D;
      const float* z = gate + g * D4;
      const float ft = sigmoidf_(z[d]), it = sigmoidf_(z[D + d]), ot = sigmoidf_(z[2 * D + d]);
      const float ct = tanhf(z[3 * D + d]);
      const float m = ft * mem[i] + it * ct;
      mem[i] = m;
      hid[g * D2 + d] = ot * tanhf(m);
    }
    __syncthreads();
    // u = h W_1
    for (int i = tid; i < ng * D; i += S2V_THREADS) {
      const int g = i / D, k = i - g * D;
      const float* hg = hid + g * D2;
      float acc = 0.f;
      for (int d = 0; d < D; ++d) acc = fmaf(hg[d], __ldg(p.W1 + d * D + k), acc);
      us[i] = acc;
    }
    __syncthreads();
    // energies: one warp per (graph, node), lanes over the features, fixed reduction tree
    for (int it = warp; it < ng * N; it += nwarps) {
      const int g = it / N, n = it - g * N;
      float acc = 0.f;
      if (ins[it] != 0.f) {
        const float* xn = xs + ((size_t)g * N + n) * D;
        const float* ug = us + g * D;
        for (int k = lane; k < D; k += 32) acc = fmaf(tanhf(ug[k] + xn[k]), __ldg(p.W2 + k), acc);
        acc = lnb::warp_sum(acc);
      }
      if (lane == 0) en[it] = acc;
    }
    __syncthreads();
    // softmax over the set: one warp per graph, nodes in order
    for (int g = warp; g < ng; g += nwarps) {
      float mx = -FLT_MAX;
      int any = 0;
      for (int n = lane; n < N; n += 32)
        if (ins[g * N + n] != 0.f) { mx = fmaxf(mx, en[g * N + n]); any = 1; }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      any = __any_sync(0xffffffffu, any);
      if (lane == 0) {
        float s = 0.f;
        for (int n = 0; n < N; ++n)
          if (ins[g * N + n] != 0.f) {
            const float ex = expf(en[g * N + n] - mx);
            en[g * N + n] = ex;
            s += ex;
          } else {
            en[g * N + n] = 0.f;
          }
        const float inv = any ? 1.f / s : 0.f;     // empty set: every weight 0, read = 0
        for (int n = 0; n < N; ++n) en[g * N + n] *= inv;
      }
    }
    __syncthreads();
    // read = sum_n a_n x_n -> second half of hidden
    for (int i = tid; i < ng * D; i += S2V_THREADS) {
      const int g = i / D, d = i - g * D;
      const float* a = en + g * N;
      const float* xg = xs + (size_t)g * N * D + d;
      float acc = 0.f;
      for (int n = 0; n < N; ++n) acc = fmaf(a[n], xg[(size_t)n * D], acc);
      hid[g * D2 + D + d] = acc;
    }
    __syncthreads();
  }
  // output_func
  for (int i = tid; i < ng * p.P; i += S2V_THREADS) {
    const int g = i / p.P, q = i - g * p.P;
    const float* hg = hid + g * D2;
    const float* w = p.Wout + (int64_t)q * D2;
    float acc = 0.f;
    for (int k = 0; k < D2; ++k) acc = fmaf(hg[k], __ldg(w + k), acc);
    p.score[(int64_t)(g0 + g) * p.P + q] = acc + __ldg(p.bout + q);
  }
}

}  // namespace

extern "C" {

int lnb_set2vec(lnb_stream_t stream, const float* X, const uint8_t* mask, const float* WgT, const float* bg,
                const float* W1, const float* W2, const float* W_out, const float* b_out, int B, int N, int D,
                int P, int steps, float* score) {
  LNB_REQUIRE(X && WgT && bg && W1 && W2 && W_out && b_out && score, "set2vec: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && D >= 1 && P >= 1 && steps >= 0, "set2vec: bad dims B=%d N=%d D=%d P=%d steps=%d",
              B, N, D, P, steps);
  if (N > LNB_MAX_N || D % 32 || D > LNB_MAX_WIDTH || P > LNB_SET2VEC_MAX_P) {
    lnb::set_err("set2vec: N=%d D=%d P=%d outside the kernel (N <= %d, D %% 32 == 0, D <= %d, P <= %d)", N, D,
                 P, LNB_MAX_N, LNB_MAX_WIDTH, LNB_SET2VEC_MAX_P);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  // graphs per CTA: enough CTAs to cover the SMs, as many graphs as shared memory holds, at most 8
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int G = lnb::ceil_div(B, sms > 0 ? sms : 132);
  if (G > S2V_GMAX) G = S2V_GMAX;
  while (G > 1 && s2v_smem_floats(N, D, G) * sizeof(float) > S2V_SMEM_MAX) --G;
  const size_t shm = s2v_smem_floats(N, D, G) * sizeof(float);
  S2vParams p{X, mask, WgT, bg, W1, W2, W_out, b_out, score, B, N, D, P, steps, G};
  cudaFuncSetAttribute(set2vec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S2V_SMEM_MAX);
  set2vec_kernel<<<lnb::ceil_div(B, G), S2V_THREADS, shm, (cudaStream_t)stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch("set2vec");
}

}  // extern "C"
