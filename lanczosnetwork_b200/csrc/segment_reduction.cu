// unsorted_segment_sum forward / backward.
// Replaces operators/src/cuda/segment_reduction.cu:39-95 (reference).  Semantics are the
// *intended* ones: output is [B, num_segments, dim2] with batch stride num_segments*dim2
// (the reference kernel hard-codes dim1*dim2, segment_reduction.cu:48, which only agrees
// when num_segments == dim1).  Out-of-range ids are ignored instead of writing out of bounds.
// The forward adds with fp32 atomics; lnb_unsorted_segment_sum_exact is its exact, order-independent twin.
#include "common.cuh"

namespace {

// One thread per 4 consecutive features when dim2 % 4 == 0 (vector path), else scalar.
template <int VEC>
__global__ void segsum_fwd_kernel(const float* __restrict__ data,
                                  const int64_t* __restrict__ ids, int64_t total, int dim1,
                                  int dim2v, int num_segments, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int x = (int)(i % dim2v);
    int64_t row = i / dim2v;  // b*dim1 + c
    int64_t b = row / dim1;
    int64_t seg = ids[row];
    if (seg < 0 || seg >= num_segments) continue;
    float* dst = out + ((b * num_segments + seg) * dim2v + x) * VEC;
    if (VEC == 4) {
      // one 16-byte reduction (red.global.add.v4.f32, sm_90+) instead of four scalar atomics;
      // dst is 16-byte aligned on this path (dim2 % 4 == 0 and an aligned output base)
      const float4 v = reinterpret_cast<const float4*>(data)[i];
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(v.x), "f"(v.y),
                   "f"(v.z), "f"(v.w) : "memory");
    } else {
      atomicAdd(dst, data[i]);
    }
  }
}

template <int VEC>
__global__ void segsum_bwd_kernel(const float* __restrict__ gout,
                                  const int64_t* __restrict__ ids, int64_t total, int dim1,
                                  int dim2v, int num_segments, float* __restrict__ gdata) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int x = (int)(i % dim2v);
    int64_t row = i / dim2v;
    int64_t b = row / dim1;
    int64_t seg = ids[row];
    bool ok = seg >= 0 && seg < num_segments;
    if (VEC == 4) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ok) v = reinterpret_cast<const float4*>(gout)[(b * num_segments + seg) * dim2v + x];
      reinterpret_cast<float4*>(gdata)[i] = v;
    } else {
      gdata[i] = ok ? gout[(b * num_segments + seg) * dim2v + x] : 0.f;
    }
  }
}

int grid_for(int64_t total) {
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = 132 * 16;  // 132 SMs x 16 resident 256-thread blocks, grid-stride beyond
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Exact, order-independent twin of segsum_fwd_kernel (lnb_unsorted_segment_sum_exact).  Every output
// element owns an int32 exponent word, an int32 flag word and an int64 accumulator, zeroed by the caller,
// and only integer atomics touch them, so the result has the same bits for any row order, grid or schedule:
//   pass 1: ex = max ilogb|x| + EXACT_BIAS over the finite nonzero terms (0: none); fl = NaN / +Inf / -Inf;
//   pass 2: acc += rint(x * 2^k), k = 61 - H - ilogb_max, H = bit length of dim1 (exact in double and int64);
//   pass 3: out += NaN | +-Inf | ldexpf(float(acc), -k) | 0.
constexpr int EXACT_BIAS = 150;   // ilogb of the smallest subnormal is -149, so a stored 0 means "no term"
constexpr int EXACT_NAN = 1, EXACT_PINF = 2, EXACT_NINF = 4;

__device__ __forceinline__ int exact_ilogb(float x) {   // x finite and nonzero, plus EXACT_BIAS
  const unsigned u = __float_as_uint(x) & 0x7fffffffu;
  const int e = (int)(u >> 23);
  return (e ? e - 127 : 31 - __clz(u) - 149) + EXACT_BIAS;
}

__device__ __forceinline__ int exact_scale(int ex, int H) { return 61 - H - (ex - EXACT_BIAS); }

template <int VEC, bool SCALE>
__global__ void segsum_exact_terms_kernel(const float* __restrict__ data, const int64_t* __restrict__ ids,
                                          int64_t total, int dim1, int dim2v, int num_segments, int H,
                                          int* __restrict__ ex, int* __restrict__ fl,
                                          unsigned long long* __restrict__ acc) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % dim2v);
    const int64_t row = i / dim2v;
    const int64_t b = row / dim1;
    const int64_t seg = ids[row];
    if (seg < 0 || seg >= num_segments) continue;
    const int64_t o = ((b * num_segments + seg) * dim2v + x) * VEC;
    float v[VEC];
    if constexpr (VEC == 4) {
      const float4 t = reinterpret_cast<const float4*>(data)[i];
      v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
      v[0] = data[i];
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float t = v[j];
      if (!SCALE) {
        if (isnan(t)) {
          atomicOr(fl + o + j, EXACT_NAN);
        } else if (isinf(t)) {
          atomicOr(fl + o + j, t > 0.f ? EXACT_PINF : EXACT_NINF);
        } else if (t != 0.f) {
          // the word only grows, so a term at or below the L2 copy cannot raise it
          const int e = exact_ilogb(t);
          if (e > __ldcg(ex + o + j)) atomicMax(ex + o + j, e);
        }
      } else if (t != 0.f && isfinite(t)) {
        // 2^k as a double (k lies in [-97, 209]); x * 2^k is exact and |rint| <= 2^(62 - H)
        const double scale = __hiloint2double((exact_scale(ex[o + j], H) + 1023) << 20, 0);
        atomicAdd(acc + o + j, (unsigned long long)__double2ll_rn((double)t * scale));
      }
    }
  }
}

__global__ void segsum_exact_finish_kernel(int64_t n, int H, const int* __restrict__ ex,
                                           const int* __restrict__ fl, const long long* __restrict__ acc,
                                           float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int f = fl[i];
    float s;
    if ((f & EXACT_NAN) || (f & (EXACT_PINF | EXACT_NINF)) == (EXACT_PINF | EXACT_NINF)) {
      s = __int_as_float(0x7fffffff);
    } else if (f) {
      s = __int_as_float(f == EXACT_PINF ? 0x7f800000 : 0xff800000);
    } else if (ex[i] == 0) {
      s = 0.f;
    } else {
      s = ldexpf(__ll2float_rn(acc[i]), -exact_scale(ex[i], H));
    }
    out[i] += s;
  }
}

}  // namespace

extern "C" {

int lnb_unsorted_segment_sum_forward(lnb_stream_t stream, const float* data,
                                     const int64_t* segment_ids, const int* data_shape,
                                     int num_segments, float* output) {
  LNB_REQUIRE(data_shape, "segment_sum_forward: null shape");
  int B = data_shape[0], d1 = data_shape[1], d2 = data_shape[2];
  if ((int64_t)B * d1 * d2 == 0) return LNB_OK;   // empty input: nothing to add
  LNB_REQUIRE(data && segment_ids && output, "segment_sum_forward: null pointer");
  LNB_REQUIRE(B >= 0 && d1 >= 0 && d2 >= 0 && num_segments > 0,
              "segment_sum_forward: bad shape [%d,%d,%d] S=%d", B, d1, d2, num_segments);
  int64_t n = (int64_t)B * d1 * d2;
  if (n == 0) return LNB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  if (d2 % 4 == 0 && aligned16(data) && aligned16(output)) {
    int64_t t = n / 4;
    segsum_fwd_kernel<4><<<grid_for(t), 256, 0, s>>>(data, segment_ids, t, d1, d2 / 4,
                                                      num_segments, output);
  } else {
    segsum_fwd_kernel<1><<<grid_for(n), 256, 0, s>>>(data, segment_ids, n, d1, d2, num_segments,
                                                      output);
  }
  lnb::count_launch();
  return lnb::finish_launch("segment_sum_forward");
}

int lnb_unsorted_segment_sum_backward(lnb_stream_t stream, const float* grad_output,
                                      const int64_t* segment_ids, const int* data_shape,
                                      int num_segments, float* grad_data) {
  LNB_REQUIRE(data_shape, "segment_sum_backward: null shape");
  int B = data_shape[0], d1 = data_shape[1], d2 = data_shape[2];
  if ((int64_t)B * d1 * d2 == 0) return LNB_OK;
  LNB_REQUIRE(grad_output && segment_ids && grad_data, "segment_sum_backward: null pointer");
  LNB_REQUIRE(B >= 0 && d1 >= 0 && d2 >= 0 && num_segments > 0,
              "segment_sum_backward: bad shape [%d,%d,%d] S=%d", B, d1, d2, num_segments);
  int64_t n = (int64_t)B * d1 * d2;
  if (n == 0) return LNB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  if (d2 % 4 == 0 && aligned16(grad_output) && aligned16(grad_data)) {
    int64_t t = n / 4;
    segsum_bwd_kernel<4><<<grid_for(t), 256, 0, s>>>(grad_output, segment_ids, t, d1, d2 / 4,
                                                      num_segments, grad_data);
  } else {
    segsum_bwd_kernel<1><<<grid_for(n), 256, 0, s>>>(grad_output, segment_ids, n, d1, d2,
                                                      num_segments, grad_data);
  }
  lnb::count_launch();
  return lnb::finish_launch("segment_sum_backward");
}

int lnb_unsorted_segment_sum_exact(lnb_stream_t stream, const float* data, const int64_t* segment_ids,
                                   const int* data_shape, int num_segments, int64_t* acc, int32_t* exp,
                                   int32_t* flags, float* output) {
  LNB_REQUIRE(data_shape, "segment_sum_exact: null shape");
  int B = data_shape[0], d1 = data_shape[1], d2 = data_shape[2];
  if ((int64_t)B * d1 * d2 == 0) return LNB_OK;   // empty input: nothing to add
  LNB_REQUIRE(data && segment_ids && acc && exp && flags && output, "segment_sum_exact: null pointer");
  LNB_REQUIRE(B >= 0 && d1 >= 0 && d2 >= 0 && num_segments > 0,
              "segment_sum_exact: bad shape [%d,%d,%d] S=%d", B, d1, d2, num_segments);
  const int64_t n = (int64_t)B * d1 * d2, n_out = (int64_t)B * num_segments * d2;
  const int H = 32 - __builtin_clz((unsigned)d1);
  auto* acc_u = reinterpret_cast<unsigned long long*>(acc);
  cudaStream_t s = (cudaStream_t)stream;
  if (d2 % 4 == 0 && aligned16(data)) {
    const int64_t t = n / 4;
    segsum_exact_terms_kernel<4, false><<<grid_for(t), 256, 0, s>>>(data, segment_ids, t, d1, d2 / 4,
                                                                     num_segments, H, exp, flags, acc_u);
    segsum_exact_terms_kernel<4, true><<<grid_for(t), 256, 0, s>>>(data, segment_ids, t, d1, d2 / 4,
                                                                    num_segments, H, exp, flags, acc_u);
  } else {
    segsum_exact_terms_kernel<1, false><<<grid_for(n), 256, 0, s>>>(data, segment_ids, n, d1, d2,
                                                                     num_segments, H, exp, flags, acc_u);
    segsum_exact_terms_kernel<1, true><<<grid_for(n), 256, 0, s>>>(data, segment_ids, n, d1, d2,
                                                                    num_segments, H, exp, flags, acc_u);
  }
  segsum_exact_finish_kernel<<<grid_for(n_out), 256, 0, s>>>(n_out, H, exp, flags,
                                                              reinterpret_cast<const long long*>(acc), output);
  lnb::count_launch(3);
  return lnb::finish_launch("segment_sum_exact");
}

}  // extern "C"
