// GAT's per-head input dropout fused into the per-head projection (model/gat.py:149-152), fp32 FFMA:
//   Wh[:, c*F:(c+1)*F] = (X * M_c s) W_c^T          for every channel c of a layer,
// and its adjoint.  The reference draws a fresh [B, N, Din] mask for every channel, which rules out the
// one stacked projection of the inference path: here each channel has its own masked A operand, built in
// the operand producer from X and the channel's mask words (gat_dropout.cuh) and never stored.  At the
// reference's hidden layer (C = 56 channels, Din = 896) that is C*M*Din mask words per pass, a quarter as
// many Philox calls, and they, not the FLOPs, bound these kernels.
//
// Forward: one CTA per (block of PJ_BM rows, channel), k-blocks of PJ_BK features; the masked X tile
// and W_c's tile go through shared memory, each thread holds rt rows x 4 columns of the [PJ_BM, F] tile.
// Backward: one CTA per (row slab, 32-feature block) walks the slab's row blocks and, for each, every
// channel in order: gX of the block accumulates in registers over the channels, X * M_c s goes through
// shared memory once per channel for gW_c, whose slab partial the CTA alone owns in the workspace.  A
// second launch sums the slabs in order.  Every sum runs in a fixed order, no atomics.
#include "common.cuh"
#include "gat_dropout.cuh"

namespace {

constexpr int PJ_THREADS = 256;
constexpr int PJ_BM = 128, PJ_BK = 32, PJ_RTMAX = 16;
constexpr int PB_BM = 64, PB_BD = 32;
constexpr int64_t PB_WORK_FLOATS = 16 << 20;        // slabs are capped so the partials stay within 64 MB

__global__ void __launch_bounds__(PJ_THREADS)
gat_dropout_project_kernel(const float* __restrict__ X, const float* __restrict__ W, int M, int Din, int C,
                           int F, lnb::GatDrop d, float* __restrict__ Wh) {
  __shared__ __align__(16) float Xs[PJ_BK][PJ_BM + 4];       // X * M_c s, transposed
  __shared__ __align__(16) float Ws[PJ_BK][LNB_GAT_MAX_WIDTH];         // W_c^T
  const int tid = threadIdx.x;
  const int c = blockIdx.y;
  const int m0 = blockIdx.x * PJ_BM;
  const int q4 = F >> 2;
  const int rs = PJ_THREADS / q4;                            // row groups
  const int rt = (PJ_BM + rs - 1) / rs;                      // rows per thread
  const int rg = tid / q4, v = tid - rg * q4;
  const bool active = rg < rs;
  const lnb::GatDropKey key = lnb::gat_drop_key(d);
  const uint32_t site = lnb::gat_site(d.layer, c, lnb::GAT_SITE_INPUT);
  const float* Wc = W + (int64_t)c * F * Din;
  float4 acc[PJ_RTMAX];
#pragma unroll
  for (int j = 0; j < PJ_RTMAX; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);

  for (int k0 = 0; k0 < Din; k0 += PJ_BK) {
    // masked X tile: one Philox call per four features of a row (Din % 4 == 0: they share i >> 2)
    for (int e = tid; e < PJ_BM * (PJ_BK / 4); e += PJ_THREADS) {
      const int r = e / (PJ_BK / 4), dq = e - r * (PJ_BK / 4);
      const int m = m0 + r, dd = k0 + 4 * dq;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m < M && dd < Din) {
        const int64_t i = (int64_t)m * Din + dd;
        x = lnb::gat_drop4(__ldg(reinterpret_cast<const float4*>(X + i)),
                           lnb::gat_drop_words(key, (uint64_t)i >> 2, site), d);
      }
      Xs[4 * dq + 0][r] = x.x;
      Xs[4 * dq + 1][r] = x.y;
      Xs[4 * dq + 2][r] = x.z;
      Xs[4 * dq + 3][r] = x.w;
    }
    for (int e = tid; e < F * (PJ_BK / 4); e += PJ_THREADS) {
      const int f = e / (PJ_BK / 4), dq = e - f * (PJ_BK / 4);
      const int dd = k0 + 4 * dq;
      const float4 w = dd < Din ? __ldg(reinterpret_cast<const float4*>(Wc + (int64_t)f * Din + dd))
                                : make_float4(0.f, 0.f, 0.f, 0.f);
      Ws[4 * dq + 0][f] = w.x;
      Ws[4 * dq + 1][f] = w.y;
      Ws[4 * dq + 2][f] = w.z;
      Ws[4 * dq + 3][f] = w.w;
    }
    __syncthreads();
    if (active) {
#pragma unroll 4
      for (int kk = 0; kk < PJ_BK; ++kk) {
        const float4 w = *reinterpret_cast<const float4*>(&Ws[kk][4 * v]);
#pragma unroll
        for (int j = 0; j < PJ_RTMAX; ++j) {
          const int r = rg + j * rs;
          if (j < rt && r < PJ_BM) {
            const float a = Xs[kk][r];
            acc[j].x = fmaf(a, w.x, acc[j].x);
            acc[j].y = fmaf(a, w.y, acc[j].y);
            acc[j].z = fmaf(a, w.z, acc[j].z);
            acc[j].w = fmaf(a, w.w, acc[j].w);
          }
        }
      }
    }
    __syncthreads();
  }
  if (!active) return;
  const int64_t row = (int64_t)C * F;
#pragma unroll
  for (int j = 0; j < PJ_RTMAX; ++j) {
    const int r = rg + j * rs;
    if (j < rt && r < PJ_BM && m0 + r < M)
      reinterpret_cast<float4*>(Wh + (int64_t)(m0 + r) * row + (int64_t)c * F)[v] = acc[j];
  }
}

// row slabs of the backward: as many as keep ~1024 CTAs in flight, at most one per row block, and the
// partials within PB_WORK_FLOATS -- a function of the shape only, so the bits do not depend on the device
int project_slabs(int M, int Din, int C, int F) {
  const int64_t rblocks = (M + PB_BM - 1) / PB_BM, dblocks = (Din + PB_BD - 1) / PB_BD;
  int64_t s = 1024 / dblocks;
  const int64_t cap = PB_WORK_FLOATS / ((int64_t)C * F * Din);
  if (s > cap) s = cap;
  if (s > rblocks) s = rblocks;
  return (int)(s < 1 ? 1 : s);
}

size_t project_bwd_smem_floats(int F) {
  return 2 * (size_t)PB_BM * PB_BD + (size_t)PB_BM * F + (size_t)F * PB_BD;
}

__global__ void __launch_bounds__(PJ_THREADS)
gat_dropout_project_backward_kernel(const float* __restrict__ X, const float* __restrict__ W,
                                    const float* __restrict__ gWh, int M, int Din, int C, int F, int rb_per_slab,
                                    lnb::GatDrop d, float* __restrict__ gX, float* __restrict__ work) {
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem;                                   // [PB_BM][PB_BD]   X of the row block
  float* Xm = Xs + PB_BM * PB_BD;                     // [PB_BM][PB_BD]   X * M_c s
  float* Gs = Xm + PB_BM * PB_BD;                     // [PB_BM][F]       gWh_c
  float* Ws = Gs + PB_BM * F;                         // [F][PB_BD]       W_c
  const int tid = threadIdx.x;
  const int slab = blockIdx.x;
  const int d0 = blockIdx.y * PB_BD;
  const int q4 = F >> 2;
  const int64_t row = (int64_t)C * F;
  const lnb::GatDropKey key = lnb::gat_drop_key(d);
  constexpr int DQ = PB_BD / 4;                        // feature quads of a block
  constexpr int GQ = PB_BM * DQ / PJ_THREADS;         // gX quads per thread
  const int nrb = (M + PB_BM - 1) / PB_BM;
  const int rb0 = slab * rb_per_slab, rb1 = min(nrb, rb0 + rb_per_slab);
  float* part = work + (int64_t)slab * row * Din;

  for (int rb = rb0; rb < rb1; ++rb) {
    const int m0 = rb * PB_BM;
    __syncthreads();                                  // the previous block's Xs is consumed
    for (int e = tid; e < PB_BM * DQ; e += PJ_THREADS) {
      const int r = e / DQ, dq = e - r * DQ;
      const int m = m0 + r, dd = d0 + 4 * dq;
      const float4 x = (m < M && dd < Din) ? __ldg(reinterpret_cast<const float4*>(X + (int64_t)m * Din + dd))
                                           : make_float4(0.f, 0.f, 0.f, 0.f);
      reinterpret_cast<float4*>(Xs)[e] = x;
    }
    float4 gacc[GQ];
#pragma unroll
    for (int j = 0; j < GQ; ++j) gacc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c = 0; c < C; ++c) {
      const uint32_t site = lnb::gat_site(d.layer, c, lnb::GAT_SITE_INPUT);
      for (int e = tid; e < PB_BM * q4; e += PJ_THREADS) {
        const int r = e / q4, v = e - r * q4;
        const int m = m0 + r;
        reinterpret_cast<float4*>(Gs)[e] =
            m < M ? __ldg(reinterpret_cast<const float4*>(gWh + (int64_t)m * row + (int64_t)c * F) + v)
                  : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      for (int e = tid; e < F * DQ; e += PJ_THREADS) {
        const int f = e / DQ, dq = e - f * DQ;
        const int dd = d0 + 4 * dq;
        reinterpret_cast<float4*>(Ws)[e] =
            dd < Din ? __ldg(reinterpret_cast<const float4*>(W + ((int64_t)c * F + f) * Din + dd))
                     : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      __syncthreads();
      // gX += M_c s * (gWh_c W_c) on this thread's quads, and X * M_c s for gW_c: one Philox call per quad
#pragma unroll
      for (int j = 0; j < GQ; ++j) {
        const int e = tid + j * PJ_THREADS;
        const int r = e / DQ, dq = e - r * DQ;
        const int m = m0 + r, dd = d0 + 4 * dq;
        float4 xm = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m < M && dd < Din) {
          const float* g = Gs + r * F;
          const float4* w = reinterpret_cast<const float4*>(Ws) + dq;
          float4 pr = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int f = 0; f < F; ++f) {
            const float a = g[f];
            const float4 b = w[f * DQ];
            pr.x = fmaf(a, b.x, pr.x);
            pr.y = fmaf(a, b.y, pr.y);
            pr.z = fmaf(a, b.z, pr.z);
            pr.w = fmaf(a, b.w, pr.w);
          }
          const uint4 mw = lnb::gat_drop_words(key, ((uint64_t)m * Din + dd) >> 2, site);
          pr = lnb::gat_drop4(pr, mw, d);
          gacc[j].x += pr.x;
          gacc[j].y += pr.y;
          gacc[j].z += pr.z;
          gacc[j].w += pr.w;
          xm = lnb::gat_drop4(reinterpret_cast<const float4*>(Xs)[e], mw, d);
        }
        reinterpret_cast<float4*>(Xm)[e] = xm;
      }
      __syncthreads();
      // gW_c partial of the slab: sum over the block's rows in order, added to the slab's running sum
      for (int e = tid; e < F * DQ; e += PJ_THREADS) {
        const int f = e / DQ, dq = e - f * DQ;
        const int dd = d0 + 4 * dq;
        if (dd >= Din) continue;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int r = 0; r < PB_BM; ++r) {
          const float a = Gs[r * F + f];
          const float4 x = reinterpret_cast<const float4*>(Xm)[r * DQ + dq];
          s.x = fmaf(a, x.x, s.x);
          s.y = fmaf(a, x.y, s.y);
          s.z = fmaf(a, x.z, s.z);
          s.w = fmaf(a, x.w, s.w);
        }
        float4* dst = reinterpret_cast<float4*>(part + ((int64_t)c * F + f) * Din + dd);
        if (rb != rb0) {
          const float4 o = *dst;
          s.x += o.x;
          s.y += o.y;
          s.z += o.z;
          s.w += o.w;
        }
        *dst = s;
      }
      __syncthreads();                                // Gs, Ws, Xm are rewritten by the next channel
    }
#pragma unroll
    for (int j = 0; j < GQ; ++j) {
      const int e = tid + j * PJ_THREADS;
      const int r = e / DQ, dq = e - r * DQ;
      const int m = m0 + r, dd = d0 + 4 * dq;
      if (m < M && dd < Din) reinterpret_cast<float4*>(gX + (int64_t)m * Din + dd)[0] = gacc[j];
    }
  }
}

__global__ void __launch_bounds__(PJ_THREADS)
gat_dropout_slab_sum_kernel(const float4* __restrict__ work, int64_t n4, int slabs, float4* __restrict__ gW) {
  for (int64_t i = blockIdx.x * (int64_t)PJ_THREADS + threadIdx.x; i < n4; i += (int64_t)gridDim.x * PJ_THREADS) {
    float4 s = work[i];
    for (int k = 1; k < slabs; ++k) {
      const float4 x = work[(int64_t)k * n4 + i];
      s.x += x.x;
      s.y += x.y;
      s.z += x.z;
      s.w += x.w;
    }
    gW[i] = s;
  }
}

int check_project(const char* who, const void* X, const void* W, const void* out, int M, int Din, int C, int F,
                  const int64_t* key, double p, int t) {
  LNB_REQUIRE(X && W && out && key, "%s: null pointer", who);
  LNB_REQUIRE(M >= 0 && Din >= 1 && C >= 1 && F >= 1, "%s: bad dims M=%d Din=%d C=%d F=%d", who, M, Din, C, F);
  LNB_REQUIRE(p >= 0.0 && p <= 1.0, "%s: p=%g outside [0, 1]", who, p);
  if (Din % 4 || F % 4 || F > LNB_GAT_MAX_WIDTH || t < 0 || t >= (1 << 16) || C > (1 << 14) ||
      (int64_t)M * Din >= (int64_t(1) << 34) || (int64_t)C * F > 0x7fffffff) {
    lnb::set_err("%s: Din=%d F=%d C=%d t=%d M=%d outside the kernel (Din %% 4 == 0, F %% 4 == 0, F <= %d) or the "
                 "mask rule (t < 2^16, C <= 2^14, M*Din < 2^34)", who, Din, F, C, t, M, LNB_GAT_MAX_WIDTH);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE(((uintptr_t)X | (uintptr_t)W | (uintptr_t)out) % 16 == 0, "%s: X, W and the output must be 16-byte "
              "aligned", who);
  return LNB_OK;
}

}  // namespace

extern "C" {

int lnb_gat_dropout_project(lnb_stream_t stream, const float* X, const float* W, int M, int Din, int C, int F,
                            const int64_t* dropout_key, double p, int t, float* Wh) {
  const int rc = check_project("gat_dropout_project", X, W, Wh, M, Din, C, F, dropout_key, p, t);
  if (rc != LNB_OK) return rc;
  if (M == 0) return LNB_OK;
  LNB_REQUIRE(C <= 65535, "gat_dropout_project: C=%d channels exceed the grid", C);
  const dim3 grid((unsigned)lnb::ceil_div(M, PJ_BM), (unsigned)C);
  gat_dropout_project_kernel<<<grid, PJ_THREADS, 0, (cudaStream_t)stream>>>(X, W, M, Din, C, F,
                                                                            gat_drop_params(dropout_key, p, t), Wh);
  lnb::count_launch();
  return lnb::finish_launch("gat_dropout_project");
}

int lnb_gat_dropout_project_slabs(int M, int Din, int C, int F) {
  if (M < 0 || Din < 1 || C < 1 || F < 1) return 0;
  return project_slabs(M, Din, C, F);
}

int lnb_gat_dropout_project_backward(lnb_stream_t stream, const float* X, const float* W, const float* gWh,
                                     int M, int Din, int C, int F, const int64_t* dropout_key, double p, int t,
                                     float* gX, float* gW, float* work) {
  const char* who = "gat_dropout_project_backward";
  const int rc = check_project(who, X, W, gX, M, Din, C, F, dropout_key, p, t);
  if (rc != LNB_OK) return rc;
  LNB_REQUIRE(gWh && gW && work, "%s: null pointer", who);
  LNB_REQUIRE(((uintptr_t)gWh | (uintptr_t)gW | (uintptr_t)work) % 16 == 0,
              "%s: gWh, gW and work must be 16-byte aligned", who);
  const int64_t n4 = (int64_t)C * F * Din / 4;
  if (M == 0) {
    cudaMemsetAsync(gW, 0, (size_t)n4 * 16, (cudaStream_t)stream);
    return lnb::finish_launch(who);
  }
  const int slabs = project_slabs(M, Din, C, F);
  const int nrb = lnb::ceil_div(M, PB_BM);
  const int per = lnb::ceil_div(nrb, slabs);
  const int used = lnb::ceil_div(nrb, per);          // every used slab holds at least one row block
  const size_t shm = project_bwd_smem_floats(F) * sizeof(float);
  if (shm > 48 * 1024)
    cudaFuncSetAttribute(gat_dropout_project_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
  const dim3 grid((unsigned)used, (unsigned)lnb::ceil_div(Din, PB_BD));
  gat_dropout_project_backward_kernel<<<grid, PJ_THREADS, shm, (cudaStream_t)stream>>>(
      X, W, gWh, M, Din, C, F, per, gat_drop_params(dropout_key, p, t), gX, work);
  int blocks = lnb::ceil_div(n4, PJ_THREADS);
  if (blocks > 132 * 8) blocks = 132 * 8;
  gat_dropout_slab_sum_kernel<<<blocks, PJ_THREADS, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(work), n4, used, reinterpret_cast<float4*>(gW));
  lnb::count_launch(2);
  return lnb::finish_launch(who);
}

}  // extern "C"
