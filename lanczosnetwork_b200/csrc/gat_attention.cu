// Graph-attention aggregation of the GAT baseline (model/gat.py:145-180) on the CUDA cores, fp32.
//
// The per-head projection Wh_c = X W_c^T runs before this kernel as ONE 3xTF32 dense layer over all
// heads of all bond channels; this kernel does the rest of a layer for every channel c = jj*heads + ii:
//   s1 = Wh_c a1_c + c1_c,  s2 = Wh_c a2_c + c2_c                          (att_net_1 / att_net_2)
//   att[i,k] = softmax over i of ( leaky_relu(s1[i] + s2[k], 0.2) + bias[i,k,jj] )   (column softmax)
//   h_c = att Wh_c + state_bias_c
// hidden layer: out[:, c*F:(c+1)*F] = ELU(h_c);  last layer: out = mean over c of h_c.
//
// Work split.  Hidden layer: one CTA per (graph, bond channel jj, group of heads), so the CTAs of a
// graph are adjacent in launch order and its channel-strided bias block is fetched from HBM once and
// served from L2 afterwards.  Last layer: one CTA per graph walks every channel in order c = 0..C-1
// and keeps the running sum in the graph's own output rows (same thread, same element each time:
// deterministic, no atomics).  A group of G heads shares the staged bias: Wh columns of the group are
// one contiguous G*F-float piece of every row.
#include "common.cuh"

namespace {

constexpr int GAT_THREADS = 256;
constexpr int GAT_NMAX = 128, GAT_FMAX = 128, GAT_E1MAX = 16, GAT_HEADSMAX = 32;
constexpr size_t GAT_SMEM_TARGET = 48 * 1024;     // head groups are sized to this when possible
constexpr size_t GAT_SMEM_MAX = 227 * 1024;

struct GatParams {
  const float* Wh;          // [B, N, C*F]
  const float* bias;        // [B, N, N, E1]
  const float* a1; const float* a2;    // [C, F]
  const float* c1; const float* c2;    // [C]
  const float* sb;          // [C, F]
  float* out;               // [B, N, C*F] (hidden) or [B, N, F] (last)
  int N, F, E1, heads, G, ngroups, last;
};

// leaky_relu(s1 + s2, 0.2) + bias, rounded op by op like the reference (no contraction)
__device__ __forceinline__ float gat_logit(float s1, float s2, float b) {
  float x = __fadd_rn(s1, s2);
  x = x > 0.f ? x : __fmul_rn(x, 0.2f);
  return __fadd_rn(x, b);
}

__device__ __forceinline__ float elu(float x) { return x > 0.f ? x : expm1f(x); }

__global__ void __launch_bounds__(GAT_THREADS)
gat_attention_kernel(GatParams p) {
  extern __shared__ __align__(16) float smem[];
  const int N = p.N, F = p.F, E1 = p.E1, heads = p.heads, G = p.G;
  const int C = E1 * heads;
  const int tid = threadIdx.x;
  const int64_t row = (int64_t)C * F;                 // Wh / hidden-output row stride
  float* Ws = smem;                                   // [N][gcnt*F]   Wh of the head group
  float* As = Ws + (size_t)N * G * F;                 // [G][N][N]     logits, then weights
  float* Bs = As + (size_t)G * N * N;                 // [N][N]        bias of channel jj
  float* S1 = Bs + (size_t)N * N;                     // [G][N]
  float* S2 = S1 + (size_t)G * N;                     // [G][N]

  int b, it0, it1;
  if (p.last) {
    b = blockIdx.x;
    it0 = 0;
    it1 = E1 * p.ngroups;
  } else {
    b = blockIdx.x / (E1 * p.ngroups);
    it0 = blockIdx.x % (E1 * p.ngroups);
    it1 = it0 + 1;
  }
  const float* Whb = p.Wh + (int64_t)b * N * row;
  int staged_jj = -1;
  for (int it = it0; it < it1; ++it) {
    const int jj = it / p.ngroups;
    const int h0 = (it % p.ngroups) * G;
    const int gcnt = min(G, heads - h0);
    const int c0 = jj * heads + h0;                   // first channel of the group
    const int gf = gcnt * F;
    __syncthreads();                                  // the previous group is fully consumed
    const int q = gf >> 2;
    for (int e = tid; e < N * q; e += GAT_THREADS) {
      const int r = e / q, v = e - r * q;
      const float4 x = __ldg(reinterpret_cast<const float4*>(Whb + r * row + (int64_t)c0 * F) + v);
      reinterpret_cast<float4*>(Ws + r * gf)[v] = x;
    }
    if (jj != staged_jj) {
      const float* bb = p.bias + (int64_t)b * N * N * E1 + jj;
      for (int e = tid; e < N * N; e += GAT_THREADS) Bs[e] = __ldg(bb + (int64_t)e * E1);
      staged_jj = jj;
    }
    __syncthreads();
    // attention logits of every node: fp32 dots in feature order, then the bias
    for (int e = tid; e < gcnt * N; e += GAT_THREADS) {
      const int g = e / N, k = e - g * N;
      const float* w = Ws + k * gf + g * F;
      const float* v1 = p.a1 + (int64_t)(c0 + g) * F;
      const float* v2 = p.a2 + (int64_t)(c0 + g) * F;
      float d1 = 0.f, d2 = 0.f;
      for (int f = 0; f < F; ++f) {
        d1 = fmaf(w[f], __ldg(v1 + f), d1);
        d2 = fmaf(w[f], __ldg(v2 + f), d2);
      }
      S1[e] = __fadd_rn(d1, __ldg(p.c1 + c0 + g));
      S2[e] = __fadd_rn(d2, __ldg(p.c2 + c0 + g));
    }
    __syncthreads();
    // softmax over the row index i of every column k (dim=1 of the reference): one thread per column
    for (int e = tid; e < gcnt * N; e += GAT_THREADS) {
      const int g = e / N, k = e - g * N;
      const float* s1 = S1 + g * N;
      const float s2 = S2[e];
      float* A = As + (size_t)g * N * N + k;
      float m = -INFINITY;
      for (int i = 0; i < N; ++i) {
        const float x = gat_logit(s1[i], s2, Bs[i * N + k]);
        A[i * N] = x;
        m = fmaxf(m, x);
      }
      float z = 0.f;
      for (int i = 0; i < N; ++i) {
        const float ex = expf(A[i * N] - m);
        A[i * N] = ex;
        z += ex;
      }
      for (int i = 0; i < N; ++i) A[i * N] = A[i * N] / z;
    }
    __syncthreads();
    // aggregation h = att Wh + state_bias, four features per thread
    const int q4 = F >> 2;
    if (!p.last) {
      for (int e = tid; e < N * gcnt * q4; e += GAT_THREADS) {
        const int i = e / (gcnt * q4), rem = e - i * (gcnt * q4);
        const int g = rem / q4, v = rem - g * q4;
        const float* A = As + ((size_t)g * N + i) * N;
        const float* w = Ws + g * F + 4 * v;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int k = 0; k < N; ++k) {
          const float a = A[k];
          const float4 x = *reinterpret_cast<const float4*>(w + k * gf);
          acc.x = fmaf(a, x.x, acc.x);
          acc.y = fmaf(a, x.y, acc.y);
          acc.z = fmaf(a, x.z, acc.z);
          acc.w = fmaf(a, x.w, acc.w);
        }
        const float4 s = __ldg(reinterpret_cast<const float4*>(p.sb + (int64_t)(c0 + g) * F) + v);
        float4 o;
        o.x = elu(acc.x + s.x);
        o.y = elu(acc.y + s.y);
        o.z = elu(acc.z + s.z);
        o.w = elu(acc.w + s.w);
        reinterpret_cast<float4*>(p.out + ((int64_t)b * N + i) * row + (int64_t)(c0 + g) * F)[v] = o;
      }
    } else {
      const bool first = (it == 0), final_ = (it == it1 - 1);
      const float fC = (float)C;
      for (int e = tid; e < N * q4; e += GAT_THREADS) {
        const int i = e / q4, v = e - i * q4;
        float4* dst = reinterpret_cast<float4*>(p.out + ((int64_t)b * N + i) * F) + v;
        float4 sum = first ? make_float4(0.f, 0.f, 0.f, 0.f) : *dst;
        for (int g = 0; g < gcnt; ++g) {                // channels in ascending order
          const float* A = As + ((size_t)g * N + i) * N;
          const float* w = Ws + g * F + 4 * v;
          float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int k = 0; k < N; ++k) {
            const float a = A[k];
            const float4 x = *reinterpret_cast<const float4*>(w + k * gf);
            acc.x = fmaf(a, x.x, acc.x);
            acc.y = fmaf(a, x.y, acc.y);
            acc.z = fmaf(a, x.z, acc.z);
            acc.w = fmaf(a, x.w, acc.w);
          }
          const float4 s = __ldg(reinterpret_cast<const float4*>(p.sb + (int64_t)(c0 + g) * F) + v);
          sum.x += acc.x + s.x;
          sum.y += acc.y + s.y;
          sum.z += acc.z + s.z;
          sum.w += acc.w + s.w;
        }
        if (final_) {
          sum.x /= fC;
          sum.y /= fC;
          sum.z /= fC;
          sum.w /= fC;
        }
        *dst = sum;
      }
    }
  }
}

size_t gat_smem_floats(int N, int F, int G) {
  return (size_t)N * G * F + (size_t)G * N * N + (size_t)N * N + 2 * (size_t)G * N;
}

}  // namespace

extern "C" {

int lnb_gat_attention(lnb_stream_t stream, const float* Wh, const float* bias, const float* a1,
                      const float* a2, const float* c1, const float* c2, const float* state_bias,
                      int B, int N, int E1, int heads, int F, int last, float* out) {
  LNB_REQUIRE(Wh && bias && a1 && a2 && c1 && c2 && state_bias && out, "gat_attention: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && E1 >= 1 && heads >= 1 && F >= 1, "gat_attention: bad dims");
  if (N > GAT_NMAX || F % 4 || F > GAT_FMAX || E1 > GAT_E1MAX || heads > GAT_HEADSMAX) {
    lnb::set_err("gat_attention: N=%d F=%d E1=%d heads=%d outside the kernel (N <= %d, F %% 4 == 0, "
                 "F <= %d, E1 <= %d, heads <= %d)", N, F, E1, heads, GAT_NMAX, GAT_FMAX, GAT_E1MAX,
                 GAT_HEADSMAX);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE(((uintptr_t)Wh | (uintptr_t)state_bias | (uintptr_t)out) % 16 == 0,
              "gat_attention: Wh, state_bias and out must be 16-byte aligned");
  if (B == 0) return LNB_OK;
  // heads per group: as many as fit the occupancy target, at least one (fits 227 KB in the envelope)
  int G = heads;
  while (G > 1 && gat_smem_floats(N, F, G) * sizeof(float) > GAT_SMEM_TARGET) --G;
  const size_t shm = gat_smem_floats(N, F, G) * sizeof(float);
  LNB_REQUIRE(shm <= GAT_SMEM_MAX, "gat_attention: %zu bytes of shared memory", shm);
  const int ngroups = (heads + G - 1) / G;
  const int64_t grid = last ? (int64_t)B : (int64_t)B * E1 * ngroups;
  LNB_REQUIRE(grid <= 0x7fffffff, "gat_attention: B=%d too large", B);
  if (shm > 48 * 1024)
    cudaFuncSetAttribute(gat_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
  GatParams p;
  p.Wh = Wh; p.bias = bias; p.a1 = a1; p.a2 = a2; p.c1 = c1; p.c2 = c2; p.sb = state_bias; p.out = out;
  p.N = N; p.F = F; p.E1 = E1; p.heads = heads; p.G = G; p.ngroups = ngroups; p.last = last ? 1 : 0;
  gat_attention_kernel<<<(unsigned)grid, GAT_THREADS, shm, (cudaStream_t)stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch("gat_attention");
}

}  // extern "C"
