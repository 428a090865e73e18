// GraphSAGE (reference: model/graph_sage.py) on the machinery of the convolution stack.
//
// With the Mean aggregator the message of channel e is linear in the state: the mean over the K
// neighbours drawn with replacement (dataset/qm8.py:137-166) is M_e X with
//     M_e[n, m] = nonempty[n] * count_e(n, m) / K,
// a layer-invariant operator.  lnb_sage_operators writes it in the dense channel-innermost layout
// lnb_graph_prepare reads, so the unchanged prepare pass produces the ELL lists, extents and tile
// schedule, and the stack kernel runs the whole model (lnb_sage_stack_forward in
// spectral_conv_fused.cu).  The Max aggregator reads the same ELL lists: the non-zeros of row n of
// M_e are exactly the distinct neighbours drawn.  lnb_neighbour_max is its unfused form for the
// training path: the max plus the argmax that routes the gradient back.
#include "common.cuh"

namespace {

constexpr int SAGE_THREADS = 128;

// One CTA per (graph, node): counts of the K samples of every channel in shared memory, then the
// node's N x E1 operator entries written out (zeros included), contiguous in [m, e] order.
__global__ void __launch_bounds__(SAGE_THREADS)
sage_operator_kernel(const int64_t* __restrict__ nn_idx, const float* __restrict__ nonempty, int N,
                     int K, int E1, float* __restrict__ out) {
  extern __shared__ int cnt[];                       // [N * E1]
  const int64_t bn = blockIdx.x;                     // b * N + n
  const int tid = threadIdx.x, per = N * E1;
  for (int i = tid; i < per; i += SAGE_THREADS) cnt[i] = 0;
  __syncthreads();
  const bool live = __ldg(nonempty + bn) != 0.f;
  if (live) {
    const int64_t* src = nn_idx + bn * K * E1;       // [K, E1]
    for (int i = tid; i < K * E1; i += SAGE_THREADS) {
      const int64_t m = __ldg(src + i);
      if (m >= 0 && m < N) atomicAdd(&cnt[(int)m * E1 + i % E1], 1);   // out-of-range ids: no entry
    }
  }
  __syncthreads();
  float* dst = out + bn * per;
  const float kf = (float)K;
  for (int i = tid; i < per; i += SAGE_THREADS) dst[i] = live ? (float)cnt[i] / kf : 0.f;
}

// Thread per (b, n, e, f): max over the ELL entries of row n of channel e of X[b, i, f]; ties go to
// the lowest node index; a row without entries gives 0 and argmax -1.
__global__ void __launch_bounds__(256)
neighbour_max_kernel(const float* __restrict__ X, const float* __restrict__ ell_val,
                     const uint8_t* __restrict__ ell_idx, const int32_t* __restrict__ ell_max, int B,
                     int N, int E1, int D, float* __restrict__ out, int32_t* __restrict__ argmax) {
  const int64_t total = (int64_t)B * N * E1 * D;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int f = (int)(i % D);
    int64_t q = i / D;
    const int e = (int)(q % E1);
    q /= E1;
    const int n = (int)(q % N);
    const int64_t b = q / N;
    const int64_t line = ((b * E1 + e) * N) * N + n;   // entry t at line + t * N
    const int len = __ldg(ell_max + b * E1 + e);
    const float* xb = X + b * N * D + f;
    float best = 0.f;
    int arg = -1;
    for (int t = 0; t < len; ++t) {
      if (__ldg(ell_val + line + (int64_t)t * N) == 0.f) continue;   // fill up to the longest row
      const int m = __ldg(ell_idx + line + (int64_t)t * N);
      const float x = __ldg(xb + (int64_t)m * D);
      if (arg < 0 || x > best || (x == best && m < arg)) { best = x; arg = m; }
    }
    out[i] = best;
    argmax[i] = arg;
  }
}

}  // namespace

extern "C" {

int lnb_sage_operators(lnb_stream_t stream, const int64_t* nn_idx, const float* nonempty, int B, int N,
                       int K, int E1, float* out) {
  LNB_REQUIRE(nn_idx && nonempty && out, "sage_operators: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && K >= 1 && E1 >= 1, "sage_operators: bad dims B=%d N=%d K=%d E1=%d",
              B, N, K, E1);
  const size_t shm = (size_t)N * E1 * sizeof(int);
  if (shm > lnb::SMEM_MAX) {
    lnb::set_err("sage_operators: N=%d, E1=%d need %zu B of shared memory", N, E1, shm);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE((int64_t)B * N <= 0x7fffffff, "sage_operators: B*N too large");
  if (B == 0) return LNB_OK;
  if (shm > 48 * 1024)
    cudaFuncSetAttribute(sage_operator_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
  sage_operator_kernel<<<(unsigned)((int64_t)B * N), SAGE_THREADS, shm, (cudaStream_t)stream>>>(
      nn_idx, nonempty, N, K, E1, out);
  lnb::count_launch();
  return lnb::finish_launch("sage_operators");
}

int lnb_neighbour_max(lnb_stream_t stream, const float* X, const float* ell_val, const uint8_t* ell_idx,
                      const int32_t* ell_max, int B, int N, int E1, int D, float* out, int32_t* argmax) {
  LNB_REQUIRE(X && ell_val && ell_idx && ell_max && out && argmax, "neighbour_max: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && N <= LNB_MAX_N_ELL && E1 >= 1 && D >= 1,
              "neighbour_max: bad dims B=%d N=%d E1=%d D=%d", B, N, E1, D);
  const int64_t total = (int64_t)B * N * E1 * D;
  if (total == 0) return LNB_OK;
  const int64_t blocks = (total + 255) / 256;
  neighbour_max_kernel<<<(unsigned)(blocks < 65536 * 16 ? blocks : 65536 * 16), 256, 0,
                         (cudaStream_t)stream>>>(X, ell_val, ell_idx, ell_max, B, N, E1, D, out, argmax);
  lnb::count_launch();
  return lnb::finish_launch("neighbour_max");
}

}  // extern "C"
