// Shared helpers for liblanczosnet_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/lanczosnet_b200.h"

namespace lnb {

// dynamic shared memory one CTA may opt in to on sm_90a
constexpr int SMEM_MAX = 227 * 1024;

// the reference's Lanczos constants, shared by the inference and training kernels
constexpr float LANCZOS_EPS = 1.1920928955078125e-07f;  // np.finfo(np.float32).eps (ada_lanczos_net.py:8)
constexpr float LANCZOS_BETA_LOWER_BOUND = 1.0e-4f;     // ada_lanczos_net.py:169

// thread-local error text + launch counter (no other global mutable state)
char* err_buf();
void set_err(const char* fmt, ...);
void count_launch(int n = 1);
unsigned long long* prof_buffer();          // profiling aid (lnb_debug_set_prof), nullptr = off
void set_prof_buffer(unsigned long long* p);
int debug_max_ctas();                       // testing aid (lnb_debug_set_max_ctas), 0 = no cap

void launch_tile_assign(cudaStream_t s, const int32_t* gext, int B, int K, int32_t* tiles,
                        int32_t* rowmap, int32_t* nrows);   // spectral_conv_fused.cu
// after a prepare kernel: the tile assignment (with the row list), or with LNB_PREP_DEFER_TILES in
// flags only the row list (lnb_ritz_rowmap); counts its launch and checks the launches
int launch_tiles_or_rowmap(cudaStream_t s, int flags, const int32_t* gext, int B, int K,
                           int32_t* tiles, int32_t* rowmap, int32_t* nrows, const char* who);

inline int finish_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_err("%s: %s", what, cudaGetErrorString(e));
    return (int)e;
  }
  return LNB_OK;
}

#define LNB_REQUIRE(cond, ...)            \
  do {                                    \
    if (!(cond)) {                        \
      lnb::set_err(__VA_ARGS__);          \
      return LNB_ERR_ARG;                 \
    }                                     \
  } while (0)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

static inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

}  // namespace lnb
