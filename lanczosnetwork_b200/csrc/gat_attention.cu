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
//
// The training path's adjoint, gat_attention_backward_kernel, is at the end of this file.
#include "common.cuh"
#include "gat_dropout.cuh"

namespace {

constexpr int GAT_THREADS = 256;
constexpr size_t GAT_SMEM_TARGET = 48 * 1024;     // head groups are sized to this when possible

struct GatParams {
  const float* Wh;          // [B, N, C*F]
  const float* bias;        // [B, N, N, E1]
  const float* a1; const float* a2;    // [C, F]
  const float* c1; const float* c2;    // [C]
  const float* sb;          // [C, F]
  float* out;               // [B, N, C*F] (hidden) or [B, N, F] (last)
  int N, F, E1, heads, G, ngroups, last;
};

// Helpers of the forward and the backward kernel: the backward recomputes the forward's scores and
// attention weights with the same operations in the same order, so it differentiates exactly the att
// the forward applied (it is never saved: [B, C, N, N] floats would be 10 MB per layer at B = 64).

// leaky_relu(s1 + s2, 0.2) + bias, rounded op by op like the reference (no contraction)
__device__ __forceinline__ float gat_logit(float s1, float s2, float b) {
  float x = __fadd_rn(s1, s2);
  x = x > 0.f ? x : __fmul_rn(x, 0.2f);
  return __fadd_rn(x, b);
}

// s1 = w . v1 + *u1, s2 = w . v2 + *u2 of one node row w of a channel (v = its a1 / a2 row, u = its
// c1 / c2): fp32 dots in feature order
__device__ __forceinline__ void gat_scores(const float* w, const float* v1, const float* v2, const float* u1,
                                           const float* u2, int F, float& s1, float& s2) {
  float d1 = 0.f, d2 = 0.f;
  for (int f = 0; f < F; ++f) {
    d1 = fmaf(w[f], __ldg(v1 + f), d1);
    d2 = fmaf(w[f], __ldg(v2 + f), d2);
  }
  s1 = __fadd_rn(d1, __ldg(u1));
  s2 = __fadd_rn(d2, __ldg(u2));
}

// softmax over the row index i of one column k (dim=1 of the reference), written to A[i * N];
// bias_at(i) is bias[i, k].  Returns the column max m and the sum z: att[i,k] = gat_weight(logit, m, z).
// The forward kernel spells out the same three loops inline (as a call, the same source schedules
// differently there); the backward uses this function.
template <class BiasAt>
__device__ __forceinline__ void gat_column_softmax(float* A, const float* s1, float s2, int N, BiasAt bias_at,
                                                   float& m_out, float& z_out) {
  float m = -INFINITY;
  for (int i = 0; i < N; ++i) {
    const float x = gat_logit(s1[i], s2, bias_at(i));
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
  m_out = m;
  z_out = z;
}

// one attention weight from its logit and the column's max and sum: the value gat_column_softmax wrote
__device__ __forceinline__ float gat_weight(float x, float m, float z) { return expf(x - m) / z; }

__device__ __forceinline__ float elu(float x) { return x > 0.f ? x : expm1f(x); }

// The dropout kernels' masks of one head group, in place in shared memory once the scores are taken:
// Ws [N][gcnt*F] (Wh of channels c0 .. c0+gcnt-1) becomes Wh' = Wh * M_wh s and As [gcnt][N][N] (att)
// becomes att' = att * M_att s.  One Philox call per four elements of a site: a Wh quad is four features
// of one node (F % 4 == 0); the [N, N] block of graph b starts at element b*N*N of its site, so its first
// and last quads may be shared with the neighbouring graphs.
__device__ __forceinline__ void gat_drop_group(const lnb::GatDrop& d, int b, int N, int F, int c0, int gcnt,
                                               float* Ws, float* As, int nthreads) {
  const lnb::GatDropKey key = lnb::gat_drop_key(d);
  const int gf = gcnt * F, q4 = F >> 2;
  for (int e = threadIdx.x; e < N * gcnt * q4; e += nthreads) {
    const int n = e / (gcnt * q4), rem = e - n * (gcnt * q4);
    const int g = rem / q4, v = rem - g * q4;
    const uint64_t q = (((uint64_t)b * N + n) * F + 4 * v) >> 2;
    const uint4 w = lnb::gat_drop_words(key, q, lnb::gat_site(d.layer, c0 + g, lnb::GAT_SITE_WH));
    float4* x = reinterpret_cast<float4*>(Ws + n * gf + g * F) + v;
    *x = lnb::gat_drop4(*x, w, d);
  }
  const uint64_t base = (uint64_t)b * N * N;
  const uint64_t qlo = base >> 2;
  const int nq = (int)(((base + (uint64_t)N * N - 1) >> 2) - qlo + 1);
  for (int e = threadIdx.x; e < gcnt * nq; e += nthreads) {
    const int g = e / nq;
    const uint64_t q = qlo + (e - g * nq);
    const uint4 w = lnb::gat_drop_words(key, q, lnb::gat_site(d.layer, c0 + g, lnb::GAT_SITE_ATT));
    float* A = As + (size_t)g * N * N;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t i = (int64_t)(4 * q + j) - (int64_t)base;
      if (i >= 0 && i < (int64_t)N * N) A[i] = lnb::gat_drop(A[i], lnb::gat_word(w, j), d);
    }
  }
}

// DROP: the training forward with the reference's dropout (lnb_gat_attention_dropout): after the softmax,
// att' = att * M_att s and Wh' = Wh * M_wh s replace att and Wh in the aggregation; the scores read Wh.
// DROP = false is lnb_gat_attention (d unused).
template <bool DROP>
__device__ __forceinline__ void gat_attention_body(GatParams p, lnb::GatDrop d) {
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
      gat_scores(Ws + k * gf + g * F, p.a1 + (int64_t)(c0 + g) * F, p.a2 + (int64_t)(c0 + g) * F,
                 p.c1 + c0 + g, p.c2 + c0 + g, F, S1[e], S2[e]);
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
    if constexpr (DROP) {
      gat_drop_group(d, b, N, F, c0, gcnt, Ws, As, GAT_THREADS);
      __syncthreads();
    }
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

__global__ void __launch_bounds__(GAT_THREADS)
gat_attention_kernel(GatParams p) {
  gat_attention_body<false>(p, lnb::GatDrop{});
}

__global__ void __launch_bounds__(GAT_THREADS)
gat_attention_dropout_kernel(GatParams p, lnb::GatDrop d) {
  gat_attention_body<true>(p, d);
}

size_t gat_smem_floats(int N, int F, int G) {
  return (size_t)N * G * F + (size_t)G * N * N + (size_t)N * N + 2 * (size_t)G * N;
}

// ------------------------------------------------------------------------------------------------
// Backward.  Per channel c of a layer, with gh = dL/dh_c (hidden: gout_c * ELU'(h_c); last: gout / C for
// every channel).  ELU'(h) = exp(h) for h <= 0 is taken from h = att Wh_c + state_bias_c, recomputed
// with the forward's arithmetic: out + 1 would lose it where out rounds towards -1.
//   gWh[k]  = sum_i att[i,k] gh[i] + gs1[k] a1_c + gs2[k] a2_c
//   gAtt[i,k] = gh[i] . Wh[k];   gE[i,k] = att[i,k] (gAtt[i,k] - sum_i' att[i',k] gAtt[i',k])
//   gX[i,k] = gE[i,k] * (s1[i] + s2[k] > 0 ? 1 : 0.2);   gs1[i] = sum_k gX[i,k],  gs2[k] = sum_i gX[i,k]
//   per-graph partials: ga1 = sum_k gs1[k] Wh[k], ga2 = sum_k gs2[k] Wh[k], gsb = sum_i gh[i],
//   gc1 = sum gs1, gc2 = sum gs2   -> gpar[b, c, :] = [ga1 | ga2 | gsb | gc1 | gc2]   (3F + 2 floats)
// One CTA per (graph, bond channel, head group) in both layers: the channels of the last layer are
// independent in the backward.  Every output element is one thread's sum in a fixed order: no atomics,
// repeated launches are bit-identical.  The recomputed h and gAtt = gh Wh^T accumulate in fp32; att^T gh,
// the softmax adjoint and the O(N) reductions behind gs1, gs2 and the parameter partials accumulate in
// fp64: sum_i gE[i,k] is zero up to the leaky-ReLU kink, so gs2 is mostly cancellation, and fp32 row-order
// sums of it land several times further from the exact value than fp32 autograd's tree reductions.  Shared memory: Wh and gh of the group, one [N, N] matrix per
// channel (att, then gAtt, then gX) and six [N] vectors; the bias is read through L2 (staging it too
// would not fit the N = F = 128 corner).
struct GatBwdParams {
  const float* gout;        // [B, N, C*F] (hidden) or [B, N, F] (last)
  const float* sb;          // [C, F]
  const float* Wh; const float* bias;
  const float* a1; const float* a2; const float* c1; const float* c2;
  float* gWh;               // [B, N, C*F]
  float* gpar;              // [B, C, 3F+2]
  int N, F, E1, heads, G, ngroups, last;
};

// DROP: the adjoint of the dropout forward (lnb_gat_attention_dropout_backward).  The masks are drawn again:
// Ws and As hold Wh' and att' from the softmax on, gWh's aggregation term is M_wh s (att'^T gh), the softmax
// adjoint reads gAtt = M_att s (gh Wh'^T), and the score terms ga1 / ga2 read the undropped Wh from memory.
template <bool DROP>
__device__ __forceinline__ void gat_attention_backward_body(const GatBwdParams& p, const lnb::GatDrop& dr) {
  extern __shared__ __align__(16) float smem[];
  const int N = p.N, F = p.F, E1 = p.E1, heads = p.heads, G = p.G;
  const int C = E1 * heads;
  const int tid = threadIdx.x;
  const int64_t row = (int64_t)C * F;
  const int b = blockIdx.x / (E1 * p.ngroups);
  const int it = blockIdx.x % (E1 * p.ngroups);
  const int jj = it / p.ngroups;
  const int h0 = (it % p.ngroups) * G;
  const int gcnt = min(G, heads - h0);
  const int c0 = jj * heads + h0;
  const int gf = gcnt * F;
  const int q = gf >> 2, q4 = F >> 2;
  float* Ws = smem;                                   // [N][gf]      Wh of the head group
  float* Gs = Ws + (size_t)N * G * F;                 // [N][gf]      gh
  float* As = Gs + (size_t)N * G * F;                 // [G][N][N]    att, then gAtt, then gX
  float* S1 = As + (size_t)G * N * N;                 // [G][N]
  float* S2 = S1 + (size_t)G * N;
  float* Mx = S2 + (size_t)G * N;                     // column max of the logits
  float* Zs = Mx + (size_t)G * N;                     // column sum of the exponentials
  float* R1 = Zs + (size_t)G * N;                     // gs1
  float* R2 = R1 + (size_t)G * N;                     // gs2
  const float* bb = p.bias + (int64_t)b * N * N * E1 + jj;
  const float* Whb = p.Wh + (int64_t)b * N * row + (int64_t)c0 * F;

  for (int e = tid; e < N * q; e += GAT_THREADS) {
    const int r = e / q, v = e - r * q;
    reinterpret_cast<float4*>(Ws + r * gf)[v] = __ldg(reinterpret_cast<const float4*>(Whb + r * row) + v);
    float4 g;
    if (!p.last) {                                    // ELU' applied below, once h is known
      g = __ldg(reinterpret_cast<const float4*>(p.gout + ((int64_t)b * N + r) * row + (int64_t)c0 * F) + v);
    } else {
      const float fC = (float)C;
      g = __ldg(reinterpret_cast<const float4*>(p.gout + ((int64_t)b * N + r) * F) + v % q4);
      g.x /= fC;
      g.y /= fC;
      g.z /= fC;
      g.w /= fC;
    }
    reinterpret_cast<float4*>(Gs + r * gf)[v] = g;
  }
  __syncthreads();
  for (int e = tid; e < gcnt * N; e += GAT_THREADS) {
    const int g = e / N, k = e - g * N;
    gat_scores(Ws + k * gf + g * F, p.a1 + (int64_t)(c0 + g) * F, p.a2 + (int64_t)(c0 + g) * F,
               p.c1 + c0 + g, p.c2 + c0 + g, F, S1[e], S2[e]);
  }
  __syncthreads();
  for (int e = tid; e < gcnt * N; e += GAT_THREADS) {
    const int g = e / N, k = e - g * N;
    gat_column_softmax(As + (size_t)g * N * N + k, S1 + g * N, S2[e], N,
                       [=](int i) { return __ldg(bb + (int64_t)(i * N + k) * E1); }, Mx[e], Zs[e]);
  }
  __syncthreads();
  if constexpr (DROP) {
    gat_drop_group(dr, b, N, F, c0, gcnt, Ws, As, GAT_THREADS);
    __syncthreads();
  }
  if (!p.last) {
    // h = att Wh + state_bias as the forward's aggregation computes it, then gh = gout * ELU'(h)
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
      const float4 sv = __ldg(reinterpret_cast<const float4*>(p.sb + (int64_t)(c0 + g) * F) + v);
      float4* gp = reinterpret_cast<float4*>(Gs + i * gf + g * F) + v;
      float4 gh = *gp;
      const float hx = acc.x + sv.x, hy = acc.y + sv.y, hz = acc.z + sv.z, hw = acc.w + sv.w;
      gh.x = hx > 0.f ? gh.x : gh.x * expf(hx);
      gh.y = hy > 0.f ? gh.y : gh.y * expf(hy);
      gh.z = hz > 0.f ? gh.z : gh.z * expf(hz);
      gh.w = hw > 0.f ? gh.w : gh.w * expf(hw);
      *gp = gh;
    }
    __syncthreads();
  }
  // aggregation adjoint att^T gh, four features per thread; the score terms are added below by the
  // same thread to the same elements
  float* gWhb = p.gWh + (int64_t)b * N * row + (int64_t)c0 * F;
  for (int e = tid; e < N * gcnt * q4; e += GAT_THREADS) {
    const int k = e / (gcnt * q4), rem = e - k * (gcnt * q4);
    const int g = rem / q4, v = rem - g * q4;
    const float* A = As + (size_t)g * N * N + k;
    const float* h = Gs + g * F + 4 * v;
    double ax = 0.0, ay = 0.0, az = 0.0, aw = 0.0;
    for (int i = 0; i < N; ++i) {
      const double a = A[i * N];
      const float4 x = *reinterpret_cast<const float4*>(h + i * gf);
      ax = fma(a, (double)x.x, ax);
      ay = fma(a, (double)x.y, ay);
      az = fma(a, (double)x.z, az);
      aw = fma(a, (double)x.w, aw);
    }
    float4 o = make_float4((float)ax, (float)ay, (float)az, (float)aw);
    if constexpr (DROP) {
      const uint64_t q = (((uint64_t)b * N + k) * F + 4 * v) >> 2;
      o = lnb::gat_drop4(o, lnb::gat_drop_words(lnb::gat_drop_key(dr), q,
                                                lnb::gat_site(dr.layer, c0 + g, lnb::GAT_SITE_WH)), dr);
    }
    reinterpret_cast<float4*>(gWhb + k * row + g * F)[v] = o;
  }
  __syncthreads();
  // gAtt[i,k] = gh[i] . Wh[k] over the features, in order
  for (int e = tid; e < gcnt * N * N; e += GAT_THREADS) {
    const int g = e / (N * N), rem = e - g * (N * N);
    const int i = rem / N, k = rem - i * N;
    const float4* x = reinterpret_cast<const float4*>(Gs + i * gf + g * F);
    const float4* w = reinterpret_cast<const float4*>(Ws + k * gf + g * F);
    float d = 0.f;
    for (int v = 0; v < q4; ++v) {
      const float4 a = x[v], c = w[v];
      d = fmaf(a.x, c.x, d);
      d = fmaf(a.y, c.y, d);
      d = fmaf(a.z, c.z, d);
      d = fmaf(a.w, c.w, d);
    }
    if constexpr (DROP) {
      const uint64_t i_el = ((uint64_t)b * N + i) * N + k;
      const uint4 w = lnb::gat_drop_words(lnb::gat_drop_key(dr), i_el >> 2,
                                          lnb::gat_site(dr.layer, c0 + g, lnb::GAT_SITE_ATT));
      d = lnb::gat_drop(d, lnb::gat_word(w, (int)(i_el & 3)), dr);
    }
    As[e] = d;
  }
  __syncthreads();
  // softmax and leaky-ReLU adjoints, one thread per column; att recomputed from the column's m and z
  for (int e = tid; e < gcnt * N; e += GAT_THREADS) {
    const int g = e / N, k = e - g * N;
    const float* s1 = S1 + g * N;
    const float s2 = S2[e], m = Mx[e], z = Zs[e];
    float* A = As + (size_t)g * N * N + k;
    // dot = sum_i att gAtt / sum_i att: the fp32 weights sum to 1 only to rounding, and dividing by their
    // sum keeps sum_i gE[i,k] = 0 exactly instead of adding dot * (sum - 1) to every column
    double dot = 0.0, asum = 0.0;
    for (int i = 0; i < N; ++i) {
      const float a = gat_weight(gat_logit(s1[i], s2, __ldg(bb + (int64_t)(i * N + k) * E1)), m, z);
      dot = fma((double)a, (double)A[i * N], dot);
      asum += (double)a;
    }
    dot /= asum;
    double r2 = 0.0;
    for (int i = 0; i < N; ++i) {
      const float a = gat_weight(gat_logit(s1[i], s2, __ldg(bb + (int64_t)(i * N + k) * E1)), m, z);
      double gx = (double)a * ((double)A[i * N] - dot);
      gx = __fadd_rn(s1[i], s2) > 0.f ? gx : gx * 0.2;
      A[i * N] = (float)gx;
      r2 += gx;
    }
    R2[e] = (float)r2;
  }
  __syncthreads();
  for (int e = tid; e < gcnt * N; e += GAT_THREADS) {
    const int g = e / N, i = e - g * N;
    const float* A = As + ((size_t)g * N + i) * N;
    double r1 = 0.0;
    for (int k = 0; k < N; ++k) r1 += (double)A[k];
    R1[e] = (float)r1;
  }
  __syncthreads();
  for (int e = tid; e < N * gcnt * q4; e += GAT_THREADS) {
    const int k = e / (gcnt * q4), rem = e - k * (gcnt * q4);
    const int g = rem / q4, v = rem - g * q4;
    float4* dst = reinterpret_cast<float4*>(gWhb + k * row + g * F) + v;
    const float4 v1 = __ldg(reinterpret_cast<const float4*>(p.a1 + (int64_t)(c0 + g) * F) + v);
    const float4 v2 = __ldg(reinterpret_cast<const float4*>(p.a2 + (int64_t)(c0 + g) * F) + v);
    const float r1 = R1[g * N + k], r2 = R2[g * N + k];
    float4 acc = *dst;
    acc.x = fmaf(r2, v2.x, fmaf(r1, v1.x, acc.x));
    acc.y = fmaf(r2, v2.y, fmaf(r1, v1.y, acc.y));
    acc.z = fmaf(r2, v2.z, fmaf(r1, v1.z, acc.z));
    acc.w = fmaf(r2, v2.w, fmaf(r1, v1.w, acc.w));
    *dst = acc;
  }
  // this graph's share of the parameter gradients, summed over B on the host
  const int P = 3 * F + 2;
  for (int e = tid; e < gcnt * P; e += GAT_THREADS) {
    const int g = e / P, j = e - g * P;
    double acc = 0.0;
    if (j < 2 * F) {                                  // ga1, ga2
      const float* r = (j < F ? R1 : R2) + g * N;
      if constexpr (DROP) {                           // Ws holds Wh': the scores read Wh
        const float* w = Whb + g * F + (j < F ? j : j - F);
        for (int k = 0; k < N; ++k) acc = fma((double)r[k], (double)__ldg(w + k * row), acc);
      } else {
        const float* w = Ws + g * F + (j < F ? j : j - F);
        for (int k = 0; k < N; ++k) acc = fma((double)r[k], (double)w[k * gf], acc);
      }
    } else if (j < 3 * F) {                           // gsb
      const float* h = Gs + g * F + (j - 2 * F);
      for (int i = 0; i < N; ++i) acc += (double)h[i * gf];
    } else {                                          // gc1, gc2
      const float* r = (j == 3 * F ? R1 : R2) + g * N;
      for (int k = 0; k < N; ++k) acc += (double)r[k];
    }
    p.gpar[((int64_t)b * C + c0 + g) * P + j] = (float)acc;
  }
}

__global__ void __launch_bounds__(GAT_THREADS)
gat_attention_backward_kernel(GatBwdParams p) {
  gat_attention_backward_body<false>(p, lnb::GatDrop{});
}

__global__ void __launch_bounds__(GAT_THREADS)
gat_attention_dropout_backward_kernel(GatBwdParams p, lnb::GatDrop d) {
  gat_attention_backward_body<true>(p, d);
}

size_t gat_bwd_smem_floats(int N, int F, int G) {
  return 2 * (size_t)N * G * F + (size_t)G * N * N + 6 * (size_t)G * N;
}

bool gat_shape_ok(int N, int F, int E1, int heads) {
  return N <= LNB_MAX_N && F % 4 == 0 && F <= LNB_GAT_MAX_WIDTH && E1 <= LNB_MAX_E1 && heads <= LNB_GAT_MAX_HEADS;
}

// the launches of lnb_gat_attention(_backward) and of their dropout forms (drop != nullptr); `who` prefixes
// the error text
int launch_gat_attention(cudaStream_t stream, const char* who, const float* Wh, const float* bias,
                         const float* a1, const float* a2, const float* c1, const float* c2,
                         const float* state_bias, int B, int N, int E1, int heads, int F, int last, float* out,
                         const lnb::GatDrop* drop) {
  LNB_REQUIRE(Wh && bias && a1 && a2 && c1 && c2 && state_bias && out, "%s: null pointer", who);
  LNB_REQUIRE(B >= 0 && N >= 1 && E1 >= 1 && heads >= 1 && F >= 1, "%s: bad dims", who);
  if (!gat_shape_ok(N, F, E1, heads)) {
    lnb::set_err("%s: N=%d F=%d E1=%d heads=%d outside the kernel (N <= %d, F %% 4 == 0, "
                 "F <= %d, E1 <= %d, heads <= %d)", who, N, F, E1, heads, LNB_MAX_N, LNB_GAT_MAX_WIDTH, LNB_MAX_E1,
                 LNB_GAT_MAX_HEADS);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE(((uintptr_t)Wh | (uintptr_t)state_bias | (uintptr_t)out) % 16 == 0,
              "%s: Wh, state_bias and out must be 16-byte aligned", who);
  if (B == 0) return LNB_OK;
  // heads per group: as many as fit the occupancy target, at least one (fits 227 KB in the envelope)
  int G = heads;
  while (G > 1 && gat_smem_floats(N, F, G) * sizeof(float) > GAT_SMEM_TARGET) --G;
  const size_t shm = gat_smem_floats(N, F, G) * sizeof(float);
  LNB_REQUIRE(shm <= lnb::SMEM_MAX, "%s: %zu bytes of shared memory", who, shm);
  const int ngroups = (heads + G - 1) / G;
  const int64_t grid = last ? (int64_t)B : (int64_t)B * E1 * ngroups;
  LNB_REQUIRE(grid <= 0x7fffffff, "%s: B=%d too large", who, B);
  if (shm > 48 * 1024) {
    if (drop)
      cudaFuncSetAttribute(gat_attention_dropout_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
    else
      cudaFuncSetAttribute(gat_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
  }
  GatParams p;
  p.Wh = Wh; p.bias = bias; p.a1 = a1; p.a2 = a2; p.c1 = c1; p.c2 = c2; p.sb = state_bias; p.out = out;
  p.N = N; p.F = F; p.E1 = E1; p.heads = heads; p.G = G; p.ngroups = ngroups; p.last = last ? 1 : 0;
  if (drop)
    gat_attention_dropout_kernel<<<(unsigned)grid, GAT_THREADS, shm, stream>>>(p, *drop);
  else
    gat_attention_kernel<<<(unsigned)grid, GAT_THREADS, shm, stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch(who);
}

int launch_gat_attention_backward(cudaStream_t stream, const char* who, const float* gout, const float* Wh,
                                  const float* bias, const float* a1, const float* a2, const float* c1,
                                  const float* c2, const float* state_bias, int B, int N, int E1, int heads,
                                  int F, int last, float* gWh, float* gpar, const lnb::GatDrop* drop) {
  LNB_REQUIRE(gout && Wh && bias && a1 && a2 && c1 && c2 && state_bias && gWh && gpar, "%s: null pointer", who);
  LNB_REQUIRE(B >= 0 && N >= 1 && E1 >= 1 && heads >= 1 && F >= 1, "%s: bad dims", who);
  if (!gat_shape_ok(N, F, E1, heads)) {
    lnb::set_err("%s: N=%d F=%d E1=%d heads=%d outside the kernel (N <= %d, F %% 4 == 0, "
                 "F <= %d, E1 <= %d, heads <= %d)", who, N, F, E1, heads, LNB_MAX_N, LNB_GAT_MAX_WIDTH, LNB_MAX_E1,
                 LNB_GAT_MAX_HEADS);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE(((uintptr_t)gout | (uintptr_t)Wh | (uintptr_t)a1 | (uintptr_t)a2 | (uintptr_t)state_bias |
               (uintptr_t)gWh) % 16 == 0,
              "%s: gout, Wh, a1, a2, state_bias and gWh must be 16-byte aligned", who);
  if (B == 0) return LNB_OK;
  int G = heads;
  while (G > 1 && gat_bwd_smem_floats(N, F, G) * sizeof(float) > GAT_SMEM_TARGET) --G;
  const size_t shm = gat_bwd_smem_floats(N, F, G) * sizeof(float);
  LNB_REQUIRE(shm <= lnb::SMEM_MAX, "%s: %zu bytes of shared memory", who, shm);
  const int ngroups = (heads + G - 1) / G;
  const int64_t grid = (int64_t)B * E1 * ngroups;
  LNB_REQUIRE(grid <= 0x7fffffff, "%s: B=%d too large", who, B);
  if (shm > 48 * 1024) {
    if (drop)
      cudaFuncSetAttribute(gat_attention_dropout_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)shm);
    else
      cudaFuncSetAttribute(gat_attention_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
  }
  GatBwdParams p;
  p.gout = gout; p.sb = state_bias; p.Wh = Wh; p.bias = bias; p.a1 = a1; p.a2 = a2; p.c1 = c1; p.c2 = c2;
  p.gWh = gWh; p.gpar = gpar;
  p.N = N; p.F = F; p.E1 = E1; p.heads = heads; p.G = G; p.ngroups = ngroups; p.last = last ? 1 : 0;
  if (drop)
    gat_attention_dropout_backward_kernel<<<(unsigned)grid, GAT_THREADS, shm, stream>>>(p, *drop);
  else
    gat_attention_backward_kernel<<<(unsigned)grid, GAT_THREADS, shm, stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch(who);
}

// the dropout forms' own checks: the key, p in [0, 1], and the site words of the rule
int check_gat_drop(const char* who, const int64_t* key, double p, int t, int C, int64_t elements) {
  LNB_REQUIRE(key, "%s: null dropout_key", who);
  LNB_REQUIRE(p >= 0.0 && p <= 1.0, "%s: p=%g outside [0, 1]", who, p);
  if (t < 0 || t >= (1 << 16) || C > (1 << 14) || elements >= (int64_t(1) << 34)) {
    lnb::set_err("%s: layer %d, %d channels or %lld elements per site outside the mask rule "
                 "(t < 2^16, C <= 2^14, < 2^34 elements)", who, t, C, (long long)elements);
    return LNB_ERR_UNSUPPORTED;
  }
  return LNB_OK;
}

}  // namespace

extern "C" {

int lnb_gat_attention(lnb_stream_t stream, const float* Wh, const float* bias, const float* a1,
                      const float* a2, const float* c1, const float* c2, const float* state_bias,
                      int B, int N, int E1, int heads, int F, int last, float* out) {
  return launch_gat_attention((cudaStream_t)stream, "gat_attention", Wh, bias, a1, a2, c1, c2, state_bias, B, N,
                              E1, heads, F, last, out, nullptr);
}

int lnb_gat_attention_backward(lnb_stream_t stream, const float* gout, const float* Wh, const float* bias,
                               const float* a1, const float* a2, const float* c1, const float* c2,
                               const float* state_bias, int B, int N, int E1, int heads, int F, int last,
                               float* gWh, float* gpar) {
  return launch_gat_attention_backward((cudaStream_t)stream, "gat_attention_backward", gout, Wh, bias, a1, a2, c1,
                                       c2, state_bias, B, N, E1, heads, F, last, gWh, gpar, nullptr);
}

int lnb_gat_attention_dropout(lnb_stream_t stream, const float* Wh, const float* bias, const float* a1,
                              const float* a2, const float* c1, const float* c2, const float* state_bias,
                              int B, int N, int E1, int heads, int F, int last, const int64_t* dropout_key,
                              double p, int t, float* out) {
  const char* who = "gat_attention_dropout";
  const int64_t per_site = (int64_t)B * N * (N > F ? N : F);
  const int rc = check_gat_drop(who, dropout_key, p, t, E1 * heads, per_site);
  if (rc != LNB_OK) return rc;
  const lnb::GatDrop d = gat_drop_params(dropout_key, p, t);
  return launch_gat_attention((cudaStream_t)stream, who, Wh, bias, a1, a2, c1, c2, state_bias, B, N, E1, heads,
                              F, last, out, &d);
}

int lnb_gat_attention_dropout_backward(lnb_stream_t stream, const float* gout, const float* Wh, const float* bias,
                                       const float* a1, const float* a2, const float* c1, const float* c2,
                                       const float* state_bias, int B, int N, int E1, int heads, int F, int last,
                                       const int64_t* dropout_key, double p, int t, float* gWh, float* gpar) {
  const char* who = "gat_attention_dropout_backward";
  const int64_t per_site = (int64_t)B * N * (N > F ? N : F);
  const int rc = check_gat_drop(who, dropout_key, p, t, E1 * heads, per_site);
  if (rc != LNB_OK) return rc;
  const lnb::GatDrop d = gat_drop_params(dropout_key, p, t);
  return launch_gat_attention_backward((cudaStream_t)stream, who, gout, Wh, bias, a1, a2, c1, c2, state_bias, B, N,
                                       E1, heads, F, last, gWh, gpar, &d);
}

}  // extern "C"
