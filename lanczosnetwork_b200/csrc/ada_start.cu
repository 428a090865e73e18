// AdaLanczosNet's Lanczos start vector drawn on the device (the reference draws torch.randn(B, N, 1) on
// the CPU generator every call, model/ada_lanczos_net.py:161, which a CUDA graph cannot replay).  Every
// entry is a pure function of (start_key, b, n), the rule in include/lanczosnet_b200.h, so a CPU
// restatement reproduces it and a captured graph draws anew whenever the key in device memory changes.
#include "common.cuh"
#include "philox.cuh"

namespace {

constexpr int AS_THREADS = 256;

__global__ void __launch_bounds__(AS_THREADS)
ada_start_vector_kernel(const int64_t* __restrict__ key, int B, int N, float* __restrict__ q1) {
  const uint64_t seed = (uint64_t)key[0], ctr = (uint64_t)key[1];
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  const uint32_t c2 = (uint32_t)ctr, c3 = (uint32_t)(ctr >> 32);
  const int half = (N + 1) >> 1;
  const int64_t total = (int64_t)B * half;
  for (int64_t i = blockIdx.x * (int64_t)AS_THREADS + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * AS_THREADS) {
    const int b = (int)(i / half), m = (int)(i - (int64_t)b * half);
    const uint4 x = lnb::philox4x32_10(make_uint4((uint32_t)m, (uint32_t)b, c2, c3), k0, k1);
    const float u1 = ((float)x.x + 1.0f) * 0x1p-32f;        // (0, 1]
    const float u2 = (float)x.y * 0x1p-32f;                 // [0, 1]
    const float r = sqrtf(-2.0f * logf(u1));
    float sn, cs;
    sincospif(2.0f * u2, &sn, &cs);
    float* row = q1 + (int64_t)b * N;
    const int n = 2 * m;
    row[n] = r * cs;
    if (n + 1 < N) row[n + 1] = r * sn;
  }
}

}  // namespace

extern "C" {

int lnb_ada_start_vector(lnb_stream_t stream, const int64_t* start_key, int B, int N, float* q1) {
  LNB_REQUIRE(B >= 0 && N >= 1, "ada_start_vector: bad dims B=%d N=%d", B, N);
  if (B == 0) return LNB_OK;
  LNB_REQUIRE(start_key && q1, "ada_start_vector: null pointer");
  const int64_t total = (int64_t)B * ((N + 1) >> 1);
  int blocks = lnb::ceil_div(total, AS_THREADS);
  if (blocks > 132 * 8) blocks = 132 * 8;
  ada_start_vector_kernel<<<blocks, AS_THREADS, 0, (cudaStream_t)stream>>>(start_key, B, N, q1);
  lnb::count_launch();
  return lnb::finish_launch("ada_start_vector");
}

}  // extern "C"
