// AdaLanczosNet's spectral filter on the Lanczos tridiagonal T (lanczos_fused.cu produces T): the powers
// of T (model/ada_lanczos_net.py:262-270) and the symmetrisation of the learned filters (:278).
#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------
// Powers of the tridiagonal: P_{p+1} = P_p T using only the three diagonals of T.
// ------------------------------------------------------------------------------------------
struct PowerList { int v[32]; };

__global__ void __launch_bounds__(128)
tridiag_powers_kernel(const float* __restrict__ T, int B, int K, PowerList pw,
                      int S, float* __restrict__ out) {
  const int* powers = pw.v;
  extern __shared__ float smem[];
  float* P0 = smem;            // K x K
  float* P1 = P0 + K * K;      // K x K
  float* dg = P1 + K * K;      // K
  float* up = dg + K;          // K : T[c-1][c]
  float* lo = up + K;          // K : T[c+1][c]
  const int g = blockIdx.x, tid = threadIdx.x;
  const float* Tg = T + (int64_t)g * K * K;
  for (int e = tid; e < K * K; e += blockDim.x) P0[e] = Tg[e];
  for (int c = tid; c < K; c += blockDim.x) {
    dg[c] = Tg[c * K + c];
    up[c] = c > 0 ? Tg[(c - 1) * K + c] : 0.f;
    lo[c] = c < K - 1 ? Tg[(c + 1) * K + c] : 0.f;
  }
  __syncthreads();
  float* cur = P0;
  float* nxt = P1;
  int s = 0;
  const int pmax = powers[S - 1];
  for (int p = 1; p <= pmax; ++p) {
    if (p == powers[s]) {
      for (int e = tid; e < K * K; e += blockDim.x) {
        int r = e / K, c = e % K;
        out[(((int64_t)g * K + r) * S + s) * K + c] = cur[e];
      }
      ++s;
      if (s == S) break;
    }
    for (int e = tid; e < K * K; e += blockDim.x) {
      int r = e / K, c = e % K;
      float v = cur[r * K + c] * dg[c];
      if (c > 0) v = fmaf(cur[r * K + c - 1], up[c], v);
      if (c < K - 1) v = fmaf(cur[r * K + c + 1], lo[c], v);
      nxt[e] = v;
    }
    __syncthreads();
    float* t = cur; cur = nxt; nxt = t;
  }
}

__global__ void symmetrize_filters_kernel(const float* __restrict__ Y, int B, int K, int S,
                                          float* __restrict__ G) {
  int64_t total = (int64_t)B * S * K * K;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % K);
    int r = (int)((i / K) % K);
    int s = (int)((i / ((int64_t)K * K)) % S);
    int64_t b = i / ((int64_t)K * K * S);
    const float* Yb = Y + b * (int64_t)K * K * S;
    G[i] = (Yb[((int64_t)r * K + c) * S + s] + Yb[((int64_t)c * K + r) * S + s]) * 0.5f;
  }
}

}  // namespace

extern "C" {

int lnb_tridiag_powers(lnb_stream_t stream, const float* T, int B, int K, const int* powers, int S,
                       float* out) {
  LNB_REQUIRE(T && powers && out, "tridiag_powers: null pointer");
  LNB_REQUIRE(B >= 0 && K >= 1 && S >= 1 && S <= LNB_TRIDIAG_POWERS_MAX_S, "tridiag_powers: bad dims B=%d K=%d S=%d",
              B, K, S);
  for (int i = 0; i < S; ++i)
    LNB_REQUIRE(powers[i] >= 1 && (i == 0 || powers[i] > powers[i - 1]),
                "tridiag_powers: powers must be positive and strictly increasing");
  if (B == 0) return LNB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  PowerList pw;
  for (int i = 0; i < S; ++i) pw.v[i] = powers[i];
  size_t shm = ((size_t)2 * K * K + 3 * K) * sizeof(float);
  LNB_REQUIRE(shm <= lnb::SMEM_MAX, "tridiag_powers: K=%d too large", K);
  if (shm > 48 * 1024)
    cudaFuncSetAttribute(tridiag_powers_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)shm);
  tridiag_powers_kernel<<<B, 128, shm, s>>>(T, B, K, pw, S, out);
  lnb::count_launch();
  return lnb::finish_launch("tridiag_powers");
}

int lnb_symmetrize_filters(lnb_stream_t stream, const float* Y, int B, int K, int S, float* G) {
  LNB_REQUIRE(Y && G, "symmetrize_filters: null pointer");
  LNB_REQUIRE(B >= 0 && K >= 1 && S >= 1, "symmetrize_filters: bad dims");
  int64_t total = (int64_t)B * S * K * K;
  if (total == 0) return LNB_OK;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  symmetrize_filters_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(Y, B, K, S, G);
  lnb::count_launch();
  return lnb::finish_launch("symmetrize_filters");
}

}  // extern "C"
