// Fused batched Lanczos -> tridiagonal QL -> Ritz vectors: ONE kernel, one group of TPG threads per
// graph, everything after the single read of the operator stays in shared memory / registers.
//
//   1. compress: the padded dense operator A_g [N,N] is read from HBM exactly once (warp per row,
//      coalesced streaming loads) and its non-zeros are packed into a CSR pool in shared memory.
//      Graph operators are sparse (QM8 molecules: degree <= 4; G(N, 8/N) of the sweep: ~9 per row),
//      exact zeros contribute nothing to A q, so the K matvecs run from the on-chip copy.  A graph
//      whose non-zeros do not fit the pool streams its dense rows from global memory / L2 in every
//      iteration instead (correct for any density; status bit 1 reports it).
//   2. Lanczos with the reference's rules (model/ada_lanczos_net.py:139-247): thread t owns nodes
//      t, t+TPG, ...; Krylov basis in shared memory; two block Gram-Schmidt passes per iteration
//      with the reference's 1/(q_j.q_j + EPS) scaling; cumulative validity from beta >= 1e-4,
//      idx = min(#valid, #real nodes), masked alpha / beta / Q columns and rows, zero padding to K.
//   3. QL with implicit shifts on (alpha, beta) held in shared memory, rotations applied to the rows
//      of a K x K identity by one warp (lane = row), Ritz values ranked by descending |theta|.
//   4. V = Q S as a register-tiled product straight over the basis in shared memory (in place),
//      then one coalesced write of V (and Q, T, alpha, beta, idx when asked for).
//
// Differences from the reference that stay inside the stated tolerances (tests/test_gpu_kernels.py):
// block (classical, twice) instead of sequential modified Gram-Schmidt; q_{i+1}.q_{i+1} reduced
// together with alpha_{i+1}.
#include "common.cuh"
#include <float.h>
#include <stdlib.h>

namespace {

constexpr unsigned kFull = 0xffffffffu;

struct FusedParams {
  const float* A; const uint8_t* mask; const float* q1;
  int B, N, K, flags;
  float* T; float* Q; float* alpha; float* beta; int32_t* idx;
  float* theta; float* V; int32_t* status;
  int cap;            // CSR pool capacity per graph (entries)
  int pool_words;     // 4-byte words reserved for the pool / the QL scratch that aliases it
  int per_graph;      // 4-byte words of shared memory per graph
  int zw;             // words of the zs / partial-projection region
  unsigned long long* prof;   // profiling aid (lnb_debug_set_prof): per-phase clock64 totals, [8] = graphs
};

template <int TPG>
__device__ __forceinline__ void gbar(int grp) {
  if (TPG == 32) __syncwarp();
  else asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "n"(TPG) : "memory");
}

// producer / consumer hand-over between the two QL warps of a group (named barriers, 64 threads)
__device__ __forceinline__ void pair_sync(int id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void pair_arrive(int id) { asm volatile("bar.arrive %0, 64;" ::"r"(id) : "memory"); }

// sums of two values over the TPG threads of a graph; identical result (same order) in every thread
template <int TPG>
__device__ __forceinline__ float2 gsum2(float a, float b, float* red, int& flip, int grp, int wg,
                                        int lane) {
  a = lnb::warp_sum(a);
  b = lnb::warp_sum(b);
  if (TPG == 32) return make_float2(a, b);
  float* buf = red + flip * 64;
  flip ^= 1;
  if (lane == 0) { buf[2 * wg] = a; buf[2 * wg + 1] = b; }
  gbar<TPG>(grp);
  float sa = 0.f, sb = 0.f;
#pragma unroll
  for (int w = 0; w < TPG / 32; ++w) { sa += buf[2 * w]; sb += buf[2 * w + 1]; }
  return make_float2(sa, sb);
}

// Sum NV (8 or 32) per-lane values across the warp with NV-1 (+ log2(32/NV)) shuffles: at every stage
// the lanes whose bit `o` is set keep the upper half of the remaining values.  On return v[0] of lane
// L is the warp total of value L * NV / 32.
template <int NV>
__device__ __forceinline__ void multi_reduce(float (&v)[NV], int lane) {
#pragma unroll
  for (int s = 0; s < 5; ++s) {
    const int o = 16 >> s;
    const int n = NV >> (s + 1);                // values kept after this stage
    if (n >= 1) {
      const bool up = (lane & o) != 0;
#pragma unroll
      for (int k = 0; k < n; ++k) {
        const float send = up ? v[k] : v[k + n];
        const float keep = up ? v[k + n] : v[k];
        v[k] = keep + __shfl_xor_sync(kFull, send, o);
      }
    } else {
      v[0] += __shfl_xor_sync(kFull, v[0], o);
    }
  }
}

template <int TPG, int NPT, int KB>
__global__ void __launch_bounds__((TPG > 128 ? TPG : 128))
lanczos_ritz_kernel(const FusedParams P) {
  constexpr int CTA = TPG > 128 ? TPG : 128;
  constexpr int NP = TPG * NPT;                 // padded node count
  constexpr int NS = NP + 1;                    // basis row stride (odd: transposed reads conflict-free)
  constexpr int NWG = TPG / 32;                 // warps per graph
  constexpr int NCH = NP / 32;                  // 32-column chunks of an operator row
  extern __shared__ __align__(16) float smem_f[];
  const int tid = threadIdx.x, grp = tid / TPG, t = tid % TPG;
  const int lane = tid & 31, wg = t >> 5;
  const int g = blockIdx.x * (CTA / TPG) + grp;
  if (g >= P.B) return;                         // whole groups leave together (no CTA-wide barrier below)
  const int N = P.N, K = P.K;
  const int iters = N < K ? N : K;
  const int K4 = (K + 3) & ~3;

  float* base = smem_f + (size_t)grp * P.per_graph;     // 16-byte aligned (per_graph % 4 == 0)
  float* cs = base;                             // K4          projection coefficients (float4 reads)
  float* al = cs + K4;                          // K4
  float* be = al + K4;                          // K4
  float* iq = be + K4;                          // K4 + 4   1 / (q_j . q_j + EPS)
  float* red = iq + K4 + 4;                     // 128: two flip buffers x (2 values x up to 32 warps)
  int* ctl = reinterpret_cast<int*>(red + 128); // 4  : cursor, overflow
  uint32_t* rinfo = reinterpret_cast<uint32_t*>(ctl + 4);    // NP : start | len << 16
  float* zs = reinterpret_cast<float*>(rinfo + NP);          // ZW   z of the streamed matvec; aliased by
  float* part = zs;                                          //      the per-warp partial projections [NWG][K4]
  float* pval = zs + P.zw;                      // pool: cap values, then cap 16-bit columns (16-byte aligned)
  uint16_t* pcol = reinterpret_cast<uint16_t*>(pval + P.cap);
  float* Qs = pval + P.pool_words;              // K x NS      Krylov basis, row i = q_i
  int flip = 0;
  long long tph = P.prof ? clock64() : 0;
#define LNB_PHASE(k)                                                          \
  if (P.prof && t == 0) {                                                     \
    const long long now_ = clock64();                                         \
    atomicAdd(&P.prof[k], (unsigned long long)(now_ - tph));                  \
    tph = now_;                                                               \
  }

  // ---- 0. init ----------------------------------------------------------------------------------
  if (t < 4) ctl[t] = 0;
  for (int n = t; n < NP; n += TPG) rinfo[n] = 0;
  gbar<TPG>(grp);

  // ---- 1. compress: dense rows (HBM, read once) -> CSR pool --------------------------------------
  const float* Ag = P.A + (size_t)g * N * N;
  if (NCH >= 4 && (N & 3) == 0 && (reinterpret_cast<uintptr_t>(P.A) & 15) == 0) {
    // 16-byte row loads: lane l holds columns 4l..4l+3 (+128 per chunk) of RB rows; the row's non-zeros
    // are packed lane-major (deterministic), offsets from one shuffle scan of the per-lane counts
    constexpr int NC4 = NCH >= 4 ? NCH / 4 : 1;
    constexpr int RB = NC4 >= 4 ? 2 : 4;
    int cursor = 0;
    // rows of the iterations after next are pulled into L2 while this one is packed (one bulk prefetch
    // per row, no registers): the 16-byte loads below then wait for L2, not for HBM
    constexpr int PF = 2;
    const unsigned row_bytes = (unsigned)N * 4u;
    if (NC4 >= 2 && lane < RB * PF) {
      const int r = wg + (lane / RB) * NWG * RB + (lane % RB) * NWG;
      if (r < N) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(Ag + (size_t)r * N), "r"(row_bytes) : "memory");
    }
    for (int r0 = wg; r0 < N; r0 += NWG * RB) {
      float4 v[RB][NC4];
      if (NC4 >= 2 && lane < RB) {
        const int r = r0 + PF * NWG * RB + lane * NWG;
        if (r < N) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(Ag + (size_t)r * N), "r"(row_bytes) : "memory");
      }
#pragma unroll
      for (int b = 0; b < RB; ++b) {
        const int r = r0 + b * NWG;
        const float4* row = reinterpret_cast<const float4*>(Ag + (size_t)r * N);
#pragma unroll
        for (int k = 0; k < NC4; ++k) {
          const int c = 4 * lane + 128 * k;
          v[b][k] = (r < N && c < N) ? __ldcs(row + lane + 32 * k) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int b = 0; b < RB; ++b) {
        const int r = r0 + b * NWG;
        if (r >= N) break;                       // warp-uniform
        int mine = 0;
#pragma unroll
        for (int k = 0; k < NC4; ++k)
          mine += (v[b][k].x != 0.f) + (v[b][k].y != 0.f) + (v[b][k].z != 0.f) + (v[b][k].w != 0.f);
        int incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int up = __shfl_up_sync(kFull, incl, o);
          if (lane >= o) incl += up;
        }
        const int cnt = __shfl_sync(kFull, incl, 31);
        int start;
        if constexpr (TPG == 32) {
          start = cursor;
          cursor += cnt;
        } else {
          start = 0;
          if (lane == 0) start = atomicAdd(&ctl[0], cnt);
          start = __shfl_sync(kFull, start, 0);
        }
        if (start + cnt <= P.cap) {
          int p = start + incl - mine;
#pragma unroll
          for (int k = 0; k < NC4; ++k) {
            const int c = 4 * lane + 128 * k;
            const float vv[4] = {v[b][k].x, v[b][k].y, v[b][k].z, v[b][k].w};
#pragma unroll
            for (int u = 0; u < 4; ++u)
              if (vv[u] != 0.f) { pval[p] = vv[u]; pcol[p] = (uint16_t)(c + u); ++p; }
          }
          if (lane == 0) rinfo[r] = (uint32_t)start | ((uint32_t)cnt << 16);
        } else if (lane == 0) {
          ctl[1] = 1;
        }
      }
    }
  } else {
    // RB rows per warp in flight (RB * NCH independent coalesced loads) before any is consumed
    constexpr int RB = NCH >= 16 ? 2 : (NCH >= 8 ? 4 : 8);
    int cursor = 0;                              // single-warp groups allocate from a register
    for (int r0 = wg; r0 < N; r0 += NWG * RB) {
      float v[RB][NCH];
#pragma unroll
      for (int b = 0; b < RB; ++b) {
        const int r = r0 + b * NWG;
        const float* row = Ag + (size_t)r * N;
#pragma unroll
        for (int k = 0; k < NCH; ++k) {
          const int c = lane + 32 * k;
          v[b][k] = (r < N && c < N) ? __ldcs(row + c) : 0.f;
        }
      }
#pragma unroll
      for (int b = 0; b < RB; ++b) {
        const int r = r0 + b * NWG;
        if (r >= N) break;                       // warp-uniform
        int cnt = 0;
#pragma unroll
        for (int k = 0; k < NCH; ++k) cnt += __popc(__ballot_sync(kFull, v[b][k] != 0.f));
        int start;
        if constexpr (TPG == 32) {
          start = cursor;
          cursor += cnt;
        } else {
          start = 0;
          if (lane == 0) start = atomicAdd(&ctl[0], cnt);
          start = __shfl_sync(kFull, start, 0);
        }
        if (start + cnt <= P.cap) {
          int off = start;
#pragma unroll
          for (int k = 0; k < NCH; ++k) {
            const unsigned m = __ballot_sync(kFull, v[b][k] != 0.f);
            if (v[b][k] != 0.f) {
              const int p = off + __popc(m & ((1u << lane) - 1u));
              pval[p] = v[b][k];
              pcol[p] = (uint16_t)(lane + 32 * k);
            }
            off += __popc(m);
          }
          if (lane == 0) rinfo[r] = (uint32_t)start | ((uint32_t)cnt << 16);
        } else if (lane == 0) {
          ctl[1] = 1;
        }
      }
    }
  }
  LNB_PHASE(0)
  // ---- start vector (ada_lanczos_net.py:159-167) --------------------------------------------------
  float q[NPT], qp[NPT], z[NPT];
  float cnt_real = 0.f, psum = 0.f;
#pragma unroll
  for (int kk = 0; kk < NPT; ++kk) {
    const int n = t + kk * TPG;
    float mk = 0.f, v = 0.f;
    if (n < N) {
      mk = P.mask ? (P.mask[(size_t)g * N + n] ? 1.f : 0.f) : 1.f;
      v = P.q1[(size_t)g * N + n] * mk;
    }
    q[kk] = v; qp[kk] = 0.f;
    psum += v * v; cnt_real += mk;
  }
  float2 r0 = gsum2<TPG>(psum, cnt_real, red, flip, grp, wg, lane);   // also orders the pool writes
  const float nrm = sqrtf(r0.x);
  const int nreal = (int)(r0.y + 0.5f);
#pragma unroll
  for (int kk = 0; kk < NPT; ++kk) {
    q[kk] = q[kk] / nrm;
    if (t + kk * TPG >= N) q[kk] = 0.f;
    Qs[t + kk * TPG] = q[kk];
  }
  gbar<TPG>(grp);
  const bool dense = ctl[1] != 0;               // pool overflow: stream the dense rows instead

  LNB_PHASE(1)
  // ---- 2. Lanczos ----------------------------------------------------------------------------------
  float beta_prev = 0.f, valid = 1.f;
  int count = 0;
  for (int i = 0; i < iters; ++i) {
    const float* qi = Qs + (size_t)i * NS;
    if (!dense) {
#pragma unroll
      for (int kk = 0; kk < NPT; ++kk) {
        const uint32_t ri = rinfo[t + kk * TPG];
        const int s = ri & 0xffffu, len = ri >> 16;
        float a0 = 0.f, a1 = 0.f;
        int p = 0;
        for (; p + 1 < len; p += 2) {
          a0 = fmaf(pval[s + p], qi[pcol[s + p]], a0);
          a1 = fmaf(pval[s + p + 1], qi[pcol[s + p + 1]], a1);
        }
        if (p < len) a0 = fmaf(pval[s + p], qi[pcol[s + p]], a0);
        z[kk] = a0 + a1;
      }
    } else {
      for (int r = wg; r < N; r += NWG) {
        const float* row = Ag + (size_t)r * N;
        float s = 0.f;
        for (int c = lane; c < N; c += 32) s = fmaf(__ldg(row + c), qi[c], s);
        s = lnb::warp_sum(s);
        if (lane == 0) zs[r] = s;
      }
      gbar<TPG>(grp);
#pragma unroll
      for (int kk = 0; kk < NPT; ++kk) z[kk] = (t + kk * TPG < N) ? zs[t + kk * TPG] : 0.f;
    }
    float pa = 0.f, pq = 0.f;
#pragma unroll
    for (int kk = 0; kk < NPT; ++kk) { pa = fmaf(q[kk], z[kk], pa); pq = fmaf(q[kk], q[kk], pq); }
    const float2 aq = gsum2<TPG>(pa, pq, red, flip, grp, wg, lane);
    const float alpha = aq.x;
    if (t == 0) iq[i] = 1.f / (aq.y + lnb::LANCZOS_EPS);    // first read by the projections of step i+1
#pragma unroll
    for (int kk = 0; kk < NPT; ++kk) z[kk] = z[kk] - alpha * q[kk] - beta_prev * qp[kk];
    if (i > 0) {
      for (int pass = 0; pass < 2; ++pass) {
        // Projections c_j = (z . q_j) / (q_j . q_j + EPS), all j < i at once: every thread forms the
        // partial products over its own nodes, a butterfly of select-and-add shuffle stages leaves
        // lane L of each warp with the warp total of coefficient jb + L (31 shuffles for 32 values
        // instead of 5 per value, and no serial chain over j).
#pragma unroll 1
        for (int jb = 0; jb < i; jb += 32) {
          if (i - jb > 8) {
            float v[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              float a = 0.f;
              if (jb + j < i) {
#pragma unroll
                for (int kk = 0; kk < NPT; ++kk) a = fmaf(z[kk], Qs[(size_t)(jb + j) * NS + t + kk * TPG], a);
              }
              v[j] = a;
            }
            multi_reduce<32>(v, lane);
            if (jb + lane < i) {
              if constexpr (TPG == 32) cs[jb + lane] = v[0] * iq[jb + lane];
              else part[wg * K4 + jb + lane] = v[0];
            }
          } else {
            float v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              float a = 0.f;
              if (jb + j < i) {
#pragma unroll
                for (int kk = 0; kk < NPT; ++kk) a = fmaf(z[kk], Qs[(size_t)(jb + j) * NS + t + kk * TPG], a);
              }
              v[j] = a;
            }
            multi_reduce<8>(v, lane);
            const int j = jb + (lane >> 2);
            if ((lane & 3) == 0 && j < i) {
              if constexpr (TPG == 32) cs[j] = v[0] * iq[j];
              else part[wg * K4 + j] = v[0];
            }
          }
        }
        if constexpr (TPG == 32) {
          __syncwarp();
        } else {
          gbar<TPG>(grp);
          for (int j = t; j < i; j += TPG) {
            float sum = 0.f;
#pragma unroll
            for (int w = 0; w < NWG; ++w) sum += part[w * K4 + j];
            cs[j] = sum * iq[j];
          }
          gbar<TPG>(grp);
        }
        // z -= sum_j cs[j] q_j
        {
          float s0[NPT], s1[NPT];
#pragma unroll
          for (int kk = 0; kk < NPT; ++kk) { s0[kk] = 0.f; s1[kk] = 0.f; }
          int j = 0;
          for (; j + 3 < i; j += 4) {
            const float4 c4 = *reinterpret_cast<const float4*>(cs + j);
#pragma unroll
            for (int kk = 0; kk < NPT; ++kk) {
              const int n = t + kk * TPG;
              s0[kk] = fmaf(c4.x, Qs[(size_t)(j + 0) * NS + n], s0[kk]);
              s1[kk] = fmaf(c4.y, Qs[(size_t)(j + 1) * NS + n], s1[kk]);
              s0[kk] = fmaf(c4.z, Qs[(size_t)(j + 2) * NS + n], s0[kk]);
              s1[kk] = fmaf(c4.w, Qs[(size_t)(j + 3) * NS + n], s1[kk]);
            }
          }
          for (; j < i; ++j) {
            const float c = cs[j];
#pragma unroll
            for (int kk = 0; kk < NPT; ++kk) s0[kk] = fmaf(c, Qs[(size_t)j * NS + t + kk * TPG], s0[kk]);
          }
#pragma unroll
          for (int kk = 0; kk < NPT; ++kk) z[kk] -= s0[kk] + s1[kk];
        }
        if constexpr (TPG == 32) __syncwarp();  // cs is rewritten by the next pass
      }
    }
    float pb = 0.f;
#pragma unroll
    for (int kk = 0; kk < NPT; ++kk) pb = fmaf(z[kk], z[kk], pb);
    const float beta = sqrtf(gsum2<TPG>(pb, 0.f, red, flip, grp, wg, lane).x);
    valid = (beta >= lnb::LANCZOS_BETA_LOWER_BOUND) ? valid : 0.f;
    count += (valid != 0.f) ? 1 : 0;
    if (t == 0) { al[i] = alpha; be[i] = beta; }
#pragma unroll
    for (int kk = 0; kk < NPT; ++kk) {
      const float qn = (z[kk] * valid) / (beta + lnb::LANCZOS_EPS);
      qp[kk] = q[kk]; q[kk] = qn;
      if (i + 1 < iters) Qs[(size_t)(i + 1) * NS + t + kk * TPG] = qn;
    }
    beta_prev = beta;
    gbar<TPG>(grp);
  }

  LNB_PHASE(2)
  // ---- 3. masking rules + tridiagonal outputs (ada_lanczos_net.py:207-245) ------------------------
  // reference rules: idx = min(#valid, #real nodes) directions AND node rows are kept, the alpha of
  // the breakdown step is dropped while the beta in front of it stays (ada_lanczos_net.py:207-237).
  // LNB_LANCZOS_PROPER: the textbook Krylov factorisation instead -- m = #valid + 1 basis vectors
  // (q_0 and one per accepted beta), T_m with all m alphas and m-1 betas, no row masking -- whose
  // Ritz values are eigenvalues of the operator (what an online (D, V) provider needs).
  const bool proper = (P.flags & 1) != 0;
  int idx = count < nreal ? count : nreal;
  int kcols = idx, nrows_keep = idx, nbeta = idx < iters - 1 ? idx : iters - 1;
  if (proper) {
    idx = count + 1 < iters ? count + 1 : iters;
    if (idx > nreal) idx = nreal;                // a Krylov space cannot outgrow the graph
    if (idx < 1) idx = nreal > 0 ? 1 : 0;
    kcols = idx; nrows_keep = NP; nbeta = idx - 1;
  }
  if (kcols > iters) kcols = iters;
  for (int k = 0; k < K; ++k) {
#pragma unroll
    for (int kk = 0; kk < NPT; ++kk) {
      const int n = t + kk * TPG;
      if (!(k < kcols && n < nrows_keep)) Qs[(size_t)k * NS + n] = 0.f;
    }
  }
  gbar<TPG>(grp);                                // every al / be write of the loop is visible
  for (int k = t; k < K; k += TPG) {
    const float av = (k < kcols) ? al[k] : 0.f;
    const float bv = (k < nbeta) ? be[k] : 0.f;
    cs[k] = av;                                  // staged: al / be are read by other threads below
    iq[k] = bv;
  }
  gbar<TPG>(grp);
  for (int k = t; k < K; k += TPG) {
    al[k] = cs[k]; be[k] = iq[k];
    P.alpha[(size_t)g * K + k] = cs[k];
    P.beta[(size_t)g * K + k] = iq[k];
  }
  if (t == 0) P.idx[g] = idx;
  gbar<TPG>(grp);
  if (P.T) {
    float* Tg = P.T + (size_t)g * K * K;
    for (int e = t; e < K * K; e += TPG) {
      const int r = e / K, c = e - r * K;
      float v = 0.f;
      if (r == c) v = al[r];
      else if (c == r + 1) v = be[r];
      else if (r == c + 1) v = be[c];
      Tg[e] = v;
    }
  }
  if (P.Q) {
    float* Qg = P.Q + (size_t)g * N * K;
    for (int e = t; e < N * K; e += TPG) {
      const int n = e / K, k = e - n * K;
      Qg[e] = Qs[(size_t)k * NS + n];
    }
  }
  LNB_PHASE(3)
  if (!P.theta) {
    if (P.prof && t == 0) atomicAdd(&P.prof[8], 1ull);
    return;
  }

  // ---- 4. QL with implicit shifts on (al, be); rotations on the rows of a K x K identity ------------
  // scratch aliases the pool (the operator is dead): Zt[i][k] (column i of Z over rows k), then
  // Zr[k][rank] re-laid out with 16-byte aligned rows for the product.
  float* Zt = pval;                              // K x KR
  const int KR = K | 1;
  float* Zr = Zt + (((size_t)K * KR + 3) & ~(size_t)3);   // K x K4, 16-byte aligned rows
  int* rank = reinterpret_cast<int*>(Zr + (size_t)K * K4);   // K4
  // groups of >= 2 warps split the eigensolve: warp 0 carries the scalar recurrence and publishes the
  // rotations (s, c) of a sweep; warp 1 applies them to Z one sweep behind (double-buffered ring)
  constexpr bool kSplitQL = TPG >= 64;
  float2* scr = reinterpret_cast<float2*>(rank + K4);         // [2][K] rotations of a sweep, indexed by row
  int* sdesc = reinterpret_cast<int*>(scr + 2 * (size_t)K);   // [2][2] {m, first rotated row}; m < 0: done
  const int bar0 = 4 + 4 * grp;                               // FULL[0..1] = bar0 + b, EMPTY[0..1] = bar0 + 2 + b
  for (int e = t; e < K * KR; e += TPG) {
    const int i = e / KR, k = e - i * KR;
    Zt[e] = (i == k) ? 1.f : 0.f;
  }
  gbar<TPG>(grp);
  int fail = 0;
  if (wg == 0) {
    // All lanes carry the scalar recurrence redundantly (it is warp-uniform); lane 0 stores d / e.
    // The dependent chain of one rotation is kept to ~8 instructions: rsqrt + one Newton step
    // instead of sqrt and two divisions, d / e of the next rotation prefetched, the search for the
    // small sub-diagonal done by the whole warp at once.
    // Within a sweep every read of d / e is of a value from BEFORE the sweep, so lane 0 stores the new
    // values into shadow rows (the dead projection scratch) and the warp commits them after the sweep:
    // no lane can ever read an entry another lane has already overwritten, without a barrier per rotation.
    float* d = al;
    float* e = be;                               // e[K-1] = 0 by construction
    float* d2 = cs;
    float* e2 = iq;
    const bool act0 = lane < K, act1 = lane + 32 < K;
    int nsw = 0;                                 // sweeps published so far (split mode)
    for (int l = 0; l < K; ++l) {
      int sweeps = 0;
      while (true) {
        int m = K - 1;
        for (int m0 = l; m0 < K - 1; m0 += 32) {
          const int mm = m0 + lane;
          bool small = true;                     // lanes past K-2 terminate the search at K-1
          if (mm < K - 1) small = fabsf(e[mm]) <= FLT_EPSILON * (fabsf(d[mm]) + fabsf(d[mm + 1]));
          const unsigned hit = __ballot_sync(kFull, small);
          if (hit) { m = m0 + __ffs(hit) - 1; break; }
        }
        if (m > K - 1) m = K - 1;
        if (m == l) break;
        if (++sweeps > 60) { fail = 1; break; }
        const float dl = d[l], el = e[l];
        float gq = (d[l + 1] - dl) / (2.f * el);
        float r = sqrtf(gq * gq + 1.f);
        gq = d[m] - dl + el / (gq + copysignf(r, gq));
        float s = 1.f, c = 1.f, p = 0.f;
        int i = m - 1;
        bool underflow = false;
        float d_ip1 = d[m], d_i = d[m - 1], e_i = e[m - 1];
        // rows k = lane (+32) of Z: the value of column i+1 travels in a register between rotations
        float hi0 = 0.f, hi1 = 0.f;
        const int buf = nsw & 1;
        if constexpr (kSplitQL) {
          if (nsw >= 2) pair_sync(bar0 + 2 + buf);            // the consumer is done with sweep nsw - 2
        } else {
          hi0 = act0 ? Zt[(size_t)m * KR + lane] : 0.f;
          hi1 = act1 ? Zt[(size_t)m * KR + lane + 32] : 0.f;
        }
        for (; i >= l; --i) {
          const float d_n = (i > l) ? d[i - 1] : 0.f;       // prefetch for rotation i-1
          const float e_n = (i > l) ? e[i - 1] : 0.f;
          const float f = s * e_i;
          const float b = c * e_i;
          const float r2 = fmaf(f, f, gq * gq);
          if (r2 < 1.0e-36f) {                   // f = g = 0 up to underflow: the reference QL's r == 0 exit
            if (lane == 0) { e2[i + 1] = 0.f; d2[i + 1] = d_ip1 - p; e2[m] = 0.f; }
            underflow = true;
            break;
          }
          float rinv;                            // MUFU.RSQ without the denormal pre-scaling + one Newton step
          asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(rinv) : "f"(r2));
          rinv = rinv * fmaf(-0.5f * r2, rinv * rinv, 1.5f);
          s = f * rinv;
          c = gq * rinv;
          const float g2 = d_ip1 - p;
          const float rr = fmaf(2.f * c, b, (d_i - g2) * s);
          p = s * rr;
          gq = fmaf(c, rr, -b);
          if (lane == 0) { e2[i + 1] = r2 * rinv; d2[i + 1] = g2 + p; }
          if constexpr (kSplitQL) {
            if (lane == 0) scr[(size_t)buf * K + i] = make_float2(s, c);
          } else {
            const float lo0 = act0 ? Zt[(size_t)i * KR + lane] : 0.f;
            if (act0) Zt[(size_t)(i + 1) * KR + lane] = fmaf(s, lo0, c * hi0);
            hi0 = fmaf(c, lo0, -s * hi0);
            if (K > 32) {
              const float lo1 = act1 ? Zt[(size_t)i * KR + lane + 32] : 0.f;
              if (act1) Zt[(size_t)(i + 1) * KR + lane + 32] = fmaf(s, lo1, c * hi1);
              hi1 = fmaf(c, lo1, -s * hi1);
            }
          }
          d_ip1 = d_i; d_i = d_n; e_i = e_n;
        }
        if constexpr (kSplitQL) {
          if (lane == 0) { sdesc[2 * buf] = m; sdesc[2 * buf + 1] = i + 1; }
          pair_arrive(bar0 + buf);               // sweep nsw is published (rows i+1 .. m-1 were rotated)
          ++nsw;
        } else {
          // column i+1 (= l after a complete sweep) still lives in the register
          if (act0) Zt[(size_t)(i + 1) * KR + lane] = hi0;
          if (act1) Zt[(size_t)(i + 1) * KR + lane + 32] = hi1;
        }
        if (!underflow && lane == 0) { d2[l] = d_ip1 - p; e2[l] = gq; e2[m] = 0.f; }
        __syncwarp();
        for (int j = i + 1 + lane; j <= m; j += 32) { d[j] = d2[j]; e[j] = e2[j]; }   // rows [i+1, m] changed
        __syncwarp();
      }
      if (fail) break;
    }
    if constexpr (kSplitQL) {
      const int buf = nsw & 1;
      if (nsw >= 2) pair_sync(bar0 + 2 + buf);
      if (lane == 0) sdesc[2 * buf] = -1;
      pair_arrive(bar0 + buf);                   // "done"
      if (nsw >= 1) pair_sync(bar0 + 2 + (buf ^ 1));          // the last sweep's release
    }
    __syncwarp();
    // rank by descending |theta|; ties: ascending signed value, then ascending index
    for (int j = lane; j < K; j += 32) {
      const float dj = d[j], aj = fabsf(dj);
      int rk = 0;
      for (int i = 0; i < K; ++i) {
        const float di = d[i], ai = fabsf(di);
        rk += ((ai > aj) || (ai == aj && (di < dj || (di == dj && i < j)))) ? 1 : 0;
      }
      rank[j] = rk;
      P.theta[(size_t)g * K + rk] = dj;
    }
    if (lane == 0) P.status[g] = fail | (dense ? 2 : 0);
  } else if (kSplitQL && wg == 1) {
    // consumer: the rotations of sweep n on the rows of Z (column k = lane, lane + 32), one sweep behind
    const bool act0 = lane < K, act1 = lane + 32 < K;
    for (int n = 0;; ++n) {
      const int buf = n & 1;
      pair_sync(bar0 + buf);
      const int m = sdesc[2 * buf], i_end = sdesc[2 * buf + 1];
      if (m < 0) break;
      float hi0 = act0 ? Zt[(size_t)m * KR + lane] : 0.f;
      float hi1 = act1 ? Zt[(size_t)m * KR + lane + 32] : 0.f;
      const float2* sc = scr + (size_t)buf * K;
      for (int i = m - 1; i >= i_end; --i) {
        const float2 r = sc[i];
        const float lo0 = act0 ? Zt[(size_t)i * KR + lane] : 0.f;
        if (act0) Zt[(size_t)(i + 1) * KR + lane] = fmaf(r.x, lo0, r.y * hi0);
        hi0 = fmaf(r.y, lo0, -r.x * hi0);
        if (K > 32) {
          const float lo1 = act1 ? Zt[(size_t)i * KR + lane + 32] : 0.f;
          if (act1) Zt[(size_t)(i + 1) * KR + lane + 32] = fmaf(r.x, lo1, r.y * hi1);
          hi1 = fmaf(r.y, lo1, -r.x * hi1);
        }
      }
      if (act0) Zt[(size_t)i_end * KR + lane] = hi0;
      if (act1) Zt[(size_t)i_end * KR + lane + 32] = hi1;
      pair_arrive(bar0 + 2 + buf);
    }
  }
  gbar<TPG>(grp);
  LNB_PHASE(4)
  for (int e = t; e < K * K; e += TPG) {
    const int k = e / K, j = e - k * K;
    Zr[(size_t)k * K4 + rank[j]] = Zt[(size_t)j * KR + k];
  }
  if (K4 != K)
    for (int k = t; k < K; k += TPG)
      for (int j = K; j < K4; ++j) Zr[(size_t)k * K4 + j] = 0.f;
  gbar<TPG>(grp);

  // ---- 5. V = Q Z, one node at a time, written over the node's basis column ------------------------
#pragma unroll 1
  for (int kk = 0; kk < NPT; ++kk) {
    const int n = t + kk * TPG;
    float acc[KB];
#pragma unroll
    for (int j = 0; j < KB; ++j) acc[j] = 0.f;
    for (int k = 0; k < K; ++k) {
      const float qv = Qs[(size_t)k * NS + n];
      const float4* zr = reinterpret_cast<const float4*>(Zr + (size_t)k * K4);
#pragma unroll
      for (int j4 = 0; j4 < KB / 4; ++j4) {
        if (4 * j4 < K) {
          const float4 zv = zr[j4];
          acc[4 * j4 + 0] = fmaf(qv, zv.x, acc[4 * j4 + 0]);
          acc[4 * j4 + 1] = fmaf(qv, zv.y, acc[4 * j4 + 1]);
          acc[4 * j4 + 2] = fmaf(qv, zv.z, acc[4 * j4 + 2]);
          acc[4 * j4 + 3] = fmaf(qv, zv.w, acc[4 * j4 + 3]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < KB; ++j)
      if (j < K) Qs[(size_t)j * NS + n] = acc[j];
  }
  gbar<TPG>(grp);
  LNB_PHASE(5)
  {
    float* Vg = P.V + (size_t)g * N * K;
    for (int e = t; e < N * K; e += TPG) {
      const int n = e / K, k = e - n * K;
      Vg[e] = Qs[(size_t)k * NS + n];
    }
  }
  LNB_PHASE(6)
  if (P.prof && t == 0) atomicAdd(&P.prof[8], 1ull);
#undef LNB_PHASE
}

struct FusedPlan {
  int tpg, npt, kb;
  int cta, gpc;
  FusedParams p;
  size_t smem;
};

// shared-memory plan: the pool takes what is left of an SM share after the basis
static bool plan_fused(int N, int K, int tpg, int npt, FusedPlan& pl) {
  const int NP = tpg * npt, NS = NP + 1, K4 = (K + 3) & ~3;
  const int cta = tpg > 128 ? tpg : 128, gpc = cta / tpg;
  const int nwg = tpg / 32;
  int zw = nwg * K4 > NP ? nwg * K4 : NP;
  zw = (zw + 3) & ~3;
  const int fixed = K * NS + NP + zw + 4 * K4 + 4 + 128 + 4;
  const int ql_words = ((K * (K | 1) + 3) & ~3) + K * K4 + K4 + 4 * K + 8;   // Zt, Zr, rank, rotation ring, descriptors
  // target capacity: every entry of a dense operator while that is cheap (N <= 48: <= 13.5 KB),
  // else 12 non-zeros per row
  long want = (long)N * N;
  const long sparse_want = (long)N * 12;
  if (N > 48 && want > sparse_want) want = sparse_want;
  if (want > 65535) want = 65535;
  auto pool_words_for = [&](long cap) { long w = (cap * 6 + 3) / 4; return (int)(w > ql_words ? w : ql_words); };
  int pool_words = pool_words_for(want);
  long per_graph = ((long)fixed + pool_words + 3) & ~3L;
  long cap = want;
  if (per_graph * gpc * 4 > lnb::SMEM_MAX) {
    // shrink the pool to what fits one CTA per SM (still at least 4 per row), else give up
    const long room = lnb::SMEM_MAX / 4 / gpc - fixed - 4;
    if (room < ql_words) return false;
    cap = room * 4 / 6;
    if (cap > 65535) cap = 65535;
    if (cap < (long)N * 4) return false;
    pool_words = pool_words_for(cap);
    if (pool_words > room) { pool_words = (int)room; cap = (long)room * 4 / 6; }
    per_graph = ((long)fixed + pool_words + 3) & ~3L;
  } else {
    // use the slack of the SM share (k CTAs per SM) for a larger pool
    const long bytes = per_graph * gpc * 4;
    int ctas = (int)(lnb::SMEM_MAX / (bytes + 1024));
    if (ctas < 1) ctas = 1;
    if (ctas > 8) ctas = 8;
    const long share_words = (lnb::SMEM_MAX / ctas - 1024) / 4 / gpc;
    const long room = share_words - fixed - 4;
    if (room > pool_words) {
      long c2 = room * 4 / 6;
      if (c2 > (long)N * N) c2 = (long)N * N;
      if (c2 > 65535) c2 = 65535;
      if (c2 > cap) { cap = c2; pool_words = pool_words_for(cap); }
      per_graph = ((long)fixed + pool_words + 3) & ~3L;
    }
  }
  pl.tpg = tpg; pl.npt = npt; pl.cta = cta; pl.gpc = gpc;
  pl.p.cap = (int)cap; pl.p.pool_words = pool_words; pl.p.per_graph = (int)per_graph;
  pl.p.zw = zw;
  pl.smem = (size_t)per_graph * gpc * 4;
  return pl.smem <= (size_t)lnb::SMEM_MAX;
}

template <int TPG, int NPT, int KB>
static int launch_fused(cudaStream_t s, const FusedPlan& pl) {
  auto kern = lanczos_ritz_kernel<TPG, NPT, KB>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem);
  if (e != cudaSuccess) { lnb::set_err("lanczos_ritz: smem attribute: %s", cudaGetErrorString(e)); return (int)e; }
  kern<<<lnb::ceil_div(pl.p.B, pl.gpc), pl.cta, pl.smem, s>>>(pl.p);
  return LNB_OK;
}

template <int TPG, int NPT>
static int launch_fused_k(cudaStream_t s, const FusedPlan& pl) {
  if (pl.p.K <= 32) return launch_fused<TPG, NPT, 32>(s, pl);
  return launch_fused<TPG, NPT, 64>(s, pl);
}

}  // namespace

extern "C" {

int lnb_lanczos_ritz(lnb_stream_t stream, const float* A, const uint8_t* mask, const float* q1,
                     int B, int N, int K, int flags, float* T, float* Q, float* alpha, float* beta,
                     int32_t* idx, float* theta, float* ritz_vec, int32_t* status) {
  LNB_REQUIRE(B >= 0 && N >= 1 && K >= 1, "lanczos_ritz: bad dims B=%d N=%d K=%d", B, N, K);
  if (B == 0) return LNB_OK;
  LNB_REQUIRE(A && q1 && alpha && beta && idx, "lanczos_ritz: null pointer");
  LNB_REQUIRE((theta == nullptr) == (ritz_vec == nullptr) && (theta == nullptr) == (status == nullptr),
              "lanczos_ritz: theta, ritz_vec and status are given (or omitted) together");
  if (N > LNB_LANCZOS_FUSED_MAX_N || K > LNB_LANCZOS_MAX_K) {
    lnb::set_err("lanczos_ritz: N=%d K=%d outside the fused kernel (N <= 1024, K <= 64)", N, K);
    return LNB_ERR_UNSUPPORTED;
  }
  // (a 1024-thread group was measured at N = 1024: 49.8 ms against 39.7 ms -- 32-warp barriers and
  // a 64-register cap cost more than the extra parallelism buys)
  static const int cfgs[][2] = {{32, 1}, {32, 2}, {64, 2}, {128, 2}, {256, 2}, {512, 2}};
  FusedPlan pl;
  int sel = -1;
  const char* force = getenv("LNB_LANCZOS_TPG");     // profiling aid: force a thread-group size
  for (int c = 0; c < 6; ++c) {
    if (cfgs[c][0] * cfgs[c][1] < N) continue;
    if (force && atoi(force) != cfgs[c][0]) continue;
    if (plan_fused(N, K, cfgs[c][0], cfgs[c][1], pl)) { sel = c; break; }
  }
  if (sel < 0) {
    lnb::set_err("lanczos_ritz: Krylov basis (N=%d, K=%d) does not fit shared memory", N, K);
    return LNB_ERR_UNSUPPORTED;
  }
  pl.p.A = A; pl.p.mask = mask; pl.p.q1 = q1; pl.p.B = B; pl.p.N = N; pl.p.K = K; pl.p.flags = flags;
  pl.p.T = T; pl.p.Q = Q; pl.p.alpha = alpha; pl.p.beta = beta; pl.p.idx = idx;
  pl.p.theta = theta; pl.p.V = ritz_vec; pl.p.status = status;
  pl.p.prof = lnb::prof_buffer();
  cudaStream_t s = (cudaStream_t)stream;
  int rc = LNB_OK;
  switch (sel) {
    case 0: rc = launch_fused_k<32, 1>(s, pl); break;
    case 1: rc = launch_fused_k<32, 2>(s, pl); break;
    case 2: rc = launch_fused_k<64, 2>(s, pl); break;
    case 3: rc = launch_fused_k<128, 2>(s, pl); break;
    case 4: rc = launch_fused_k<256, 2>(s, pl); break;
    default: rc = launch_fused_k<512, 2>(s, pl); break;
  }
  if (rc != LNB_OK) return rc;
  lnb::count_launch();
  return lnb::finish_launch("lanczos_ritz");
}

}  // extern "C"
