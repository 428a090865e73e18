// Batched Lanczos tridiagonalisation for DENSE operators (two-launch path: lnb_lanczos_tridiag, then
// lnb_tridiag_ritz), tridiagonal QL eigensolve (Ritz pairs) and tridiagonal powers.  lnb_lanczos_tridiag
// is the fused kernel of lanczos_fused.cu without its QL stage wherever that kernel fits (N <= 1024,
// K <= 64, basis in shared memory); the CTA-per-graph kernel below is the fallback for everything else
// (operator staged in shared memory when it fits, streamed otherwise).
//
// Reference behaviour reproduced (model/ada_lanczos_net.py:139-247), including its masking
// rules: cumulative validity from beta >= 1e-4 (:193-199), idx = min(#valid, #real nodes)
// (:207-211), alpha/beta/Q columns zeroed past idx and Q *rows* >= idx zeroed (:213-237),
// zero padding to K when N < K (:240-245), and the always-on double Gram-Schmidt with the
// 1/(q.q + EPS) normalisation (:177-189).
#include "common.cuh"
#include <float.h>

namespace {

constexpr float kEps = 1.1920928955078125e-07f;  // np.finfo(np.float32).eps (ada_lanczos_net.py:8)
constexpr float kBetaLowerBound = 1.0e-4f;       // ada_lanczos_net.py:169

// ------------------------------------------------------------------------------------------
// CTA-per-graph kernel, any N.  Krylov basis in shared memory; the operator is staged in
// shared memory when it fits, otherwise streamed (coalesced, L2-resident across iterations).
// Re-orthogonalisation is done as two *block* Gram-Schmidt passes (all projections of a pass
// from the same z): identical to the sequential order up to O(eps * |q_l.q_j|), i.e. second
// order, and needs 2 barriers per pass instead of 2(i-1).
// ------------------------------------------------------------------------------------------
constexpr int CTA_THREADS = 256;

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = lnb::warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < CTA_THREADS / 32) ? red[lane] : 0.f;
  t = lnb::warp_sum(t);
  __syncthreads();
  return t;
}

__global__ void __launch_bounds__(CTA_THREADS)
lanczos_cta_kernel(const float* __restrict__ A, const uint8_t* __restrict__ mask,
                   const float* __restrict__ q1, int B, int N, int K, int stage_A,
                   float* __restrict__ T, float* __restrict__ Q, float* __restrict__ alpha_out,
                   float* __restrict__ beta_out, int32_t* __restrict__ idx_out) {
  extern __shared__ float smem[];
  const int g = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nwarps = CTA_THREADS / 32;
  const int iters = N < K ? N : K;
  const int NP = (N + 3) & ~3;
  float* Qs = smem;                         // (iters+1) x NP
  float* zs = Qs + (int64_t)(iters + 1) * NP;  // NP
  float* al = zs + NP;                      // K
  float* be = al + K;                       // K
  float* qq = be + K;                       // K+1
  float* cs = qq + (K + 1);                 // K
  float* red = cs + K;                      // 32
  float* As = red + 32;                     // N x (N+1) if staged
  const int lda = stage_A ? (N + 1) : N;

  const float* Ag = A + (int64_t)g * N * N;
  if (stage_A) {
    for (int e = tid; e < N * N; e += CTA_THREADS) As[(e / N) * lda + (e % N)] = Ag[e];
  }
  const float* Aop = stage_A ? As : Ag;

  float part = 0.f, cnt = 0.f;
  for (int n = tid; n < N; n += CTA_THREADS) {
    float mk = mask ? (mask[(int64_t)g * N + n] ? 1.f : 0.f) : 1.f;
    float v = q1[(int64_t)g * N + n] * mk;
    Qs[n] = v;
    part += v * v;
    cnt += mk;
  }
  __syncthreads();
  float nrm = sqrtf(block_sum(part, red));
  const int nreal = (int)(block_sum(cnt, red) + 0.5f);
  part = 0.f;
  for (int n = tid; n < N; n += CTA_THREADS) {
    float v = Qs[n] / nrm;
    Qs[n] = v;
    part += v * v;
  }
  float qq0 = block_sum(part, red);
  if (tid == 0) qq[0] = qq0;
  __syncthreads();

  float beta_prev = 0.f, valid = 1.f;
  int count = 0;
  for (int i = 0; i < iters; ++i) {
    const float* qi = Qs + (int64_t)i * NP;
    const float* qp = i > 0 ? Qs + (int64_t)(i - 1) * NP : nullptr;
    if (!stage_A && (N & 3) == 0) {
      // z = A q_i with the operator streamed from HBM / L2: a warp takes 4 rows at a time and
      // reads them as 16-byte vectors, two column blocks in flight -> 4 KB of loads in flight per
      // warp (the scalar row-at-a-time loop kept ~8 KB in flight per SM: latency bound at 18 % of HBM)
      const float4* q4 = reinterpret_cast<const float4*>(qi);
      const int nv = N >> 2;
      for (int r0 = warp * 4; r0 < N; r0 += nwarps * 4) {
        const float4* rows[4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
          rows[u] = reinterpret_cast<const float4*>(Ag + (int64_t)min(r0 + u, N - 1) * N);
        float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 2
        for (int m = lane; m < nv; m += 32) {
          const float4 q = q4[m];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float4 a = __ldcs(rows[u] + m);
            s[u] = fmaf(a.x, q.x, s[u]); s[u] = fmaf(a.y, q.y, s[u]);
            s[u] = fmaf(a.z, q.z, s[u]); s[u] = fmaf(a.w, q.w, s[u]);
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float t = lnb::warp_sum(s[u]);
          if (lane == 0 && r0 + u < N) zs[r0 + u] = t;
        }
      }
    } else {
      // z = A q_i : one warp per row, lanes stride the row (coalesced / conflict-free)
      for (int r = warp; r < N; r += nwarps) {
        const float* row = Aop + (int64_t)r * lda;
        float s = 0.f;
        for (int m = lane; m < N; m += 32) s = fmaf(row[m], qi[m], s);
        s = lnb::warp_sum(s);
        if (lane == 0) zs[r] = s;
      }
    }
    __syncthreads();
    part = 0.f;
    for (int n = tid; n < N; n += CTA_THREADS) part += qi[n] * zs[n];
    float alpha = block_sum(part, red);
    for (int n = tid; n < N; n += CTA_THREADS) {
      float v = zs[n] - alpha * qi[n];
      if (qp) v -= beta_prev * qp[n];
      zs[n] = v;
    }
    __syncthreads();
    if (i > 0) {
      for (int pass = 0; pass < 2; ++pass) {
        for (int j = warp; j < i; j += nwarps) {
          const float* qj = Qs + (int64_t)j * NP;
          float s = 0.f;
          for (int n = lane; n < N; n += 32) s = fmaf(zs[n], qj[n], s);
          s = lnb::warp_sum(s);
          if (lane == 0) cs[j] = s / (qq[j] + kEps);
        }
        __syncthreads();
        for (int n = tid; n < N; n += CTA_THREADS) {
          float v = zs[n];
          for (int j = 0; j < i; ++j) v -= cs[j] * Qs[(int64_t)j * NP + n];
          zs[n] = v;
        }
        __syncthreads();
      }
    }
    part = 0.f;
    for (int n = tid; n < N; n += CTA_THREADS) part += zs[n] * zs[n];
    float beta = sqrtf(block_sum(part, red));
    valid = (beta >= kBetaLowerBound) ? valid : 0.f;
    count += (valid != 0.f) ? 1 : 0;
    float* qn = Qs + (int64_t)(i + 1) * NP;
    part = 0.f;
    for (int n = tid; n < N; n += CTA_THREADS) {
      float v = (zs[n] * valid) / (beta + kEps);
      qn[n] = v;
      part += v * v;
    }
    float qqn = block_sum(part, red);
    if (tid == 0) { al[i] = alpha; be[i] = beta; qq[i + 1] = qqn; }
    __syncthreads();
    beta_prev = beta;
  }

  const int idx = count < nreal ? count : nreal;
  if (tid == 0) idx_out[g] = idx;
  for (int k = tid; k < K; k += CTA_THREADS) {
    alpha_out[(int64_t)g * K + k] = (k < iters && k < idx) ? al[k] : 0.f;
    beta_out[(int64_t)g * K + k] = (k < iters - 1 && k < idx) ? be[k] : 0.f;
  }
  float* Tg = T + (int64_t)g * K * K;
  for (int e = tid; e < K * K; e += CTA_THREADS) {
    int r = e / K, c = e % K;
    float v = 0.f;
    if (r == c) v = (r < iters && r < idx) ? al[r] : 0.f;
    else if (c == r + 1) v = (r < iters - 1 && r < idx) ? be[r] : 0.f;
    else if (r == c + 1) v = (c < iters - 1 && c < idx) ? be[c] : 0.f;
    Tg[e] = v;
  }
  float* Qg = Q + (int64_t)g * N * K;
  for (int64_t e = tid; e < (int64_t)N * K; e += CTA_THREADS) {
    int n = (int)(e / K), k = (int)(e % K);
    float v = 0.f;
    if (k < iters && k < idx && n < idx) v = Qs[(int64_t)k * NP + n];
    Qg[e] = v;
  }
}

// ------------------------------------------------------------------------------------------
// Ritz pairs: implicit-shift QL on the symmetric tridiagonal (alpha, beta), Givens rotations
// applied to the rows of Z (initialised to Q) so the result is V = Q S directly.
// One group of GW warps per graph; every warp redundantly carries the (tiny) scalar
// recurrence on its private copy of (d, e) so no cross-warp traffic is needed; each thread
// owns rows n = t, t + 32*GW, ... of Z.
// ------------------------------------------------------------------------------------------
template <int GW>
__global__ void __launch_bounds__(128)
tridiag_ritz_kernel(const float* __restrict__ alpha, const float* __restrict__ beta,
                    const float* __restrict__ Q, int B, int N, int K,
                    float* __restrict__ theta, float* __restrict__ V,
                    int32_t* __restrict__ status) {
  extern __shared__ float smem[];
  constexpr int GPC = 4 / GW;                 // graphs per 128-thread CTA
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = warp / GW, wg = warp % GW;
  const int g = blockIdx.x * GPC + grp;
  const int KP = K | 1;                       // odd row stride -> conflict-free column access
  const int zrows = (GW == 1) ? 32 : N;
  const int per_graph = zrows * KP + 4 * 2 * K;  // Z + (d,e) per warp (up to 4 warps)
  float* Zs = smem + grp * per_graph;
  float* d = Zs + zrows * KP + (wg * 2) * K;
  float* e = d + K;
  if (g >= B) return;
  const int tg = wg * 32 + lane;              // thread index inside the graph group
  const int gthreads = GW * 32;

  for (int k = lane; k < K; k += 32) {
    d[k] = alpha[(int64_t)g * K + k];
    e[k] = (k < K - 1) ? beta[(int64_t)g * K + k] : 0.f;
  }
  for (int n = tg; n < N; n += gthreads)
    for (int k = 0; k < K; ++k) Zs[n * KP + k] = Q[((int64_t)g * N + n) * K + k];
  __syncwarp();

  int fail = 0;
  for (int l = 0; l < K; ++l) {
    int sweeps = 0;
    while (true) {
      int m = l;
      for (; m < K - 1; ++m) {
        float dd = fabsf(d[m]) + fabsf(d[m + 1]);
        if (fabsf(e[m]) <= FLT_EPSILON * dd) break;
      }
      if (m == l) break;
      if (++sweeps > 60) { fail = 1; break; }
      float gq = (d[l + 1] - d[l]) / (2.f * e[l]);
      float r = sqrtf(gq * gq + 1.f);
      gq = d[m] - d[l] + e[l] / (gq + copysignf(r, gq));
      float s = 1.f, c = 1.f, p = 0.f;
      int i = m - 1;
      bool underflow = false;
      for (; i >= l; --i) {
        // every lane carries the recurrence; lane 0 alone stores, after all lanes have read this row
        const float ei = e[i], di1 = d[i + 1], di = d[i];
        __syncwarp();
        float f = s * ei;
        float b = c * ei;
        r = sqrtf(f * f + gq * gq);
        if (r == 0.f) {
          if (lane == 0) { e[i + 1] = r; d[i + 1] = di1 - p; e[m] = 0.f; }
          underflow = true;
          break;
        }
        s = f / r;
        c = gq / r;
        gq = di1 - p;
        const float rr = (di - gq) * s + 2.f * c * b;
        p = s * rr;
        if (lane == 0) { e[i + 1] = r; d[i + 1] = gq + p; }
        gq = c * rr - b;
        for (int n = tg; n < N; n += gthreads) {
          float z1 = Zs[n * KP + i + 1], z0 = Zs[n * KP + i];
          Zs[n * KP + i + 1] = s * z0 + c * z1;
          Zs[n * KP + i] = c * z0 - s * z1;
        }
      }
      if (!underflow) {
        const float dl = d[l];
        __syncwarp();
        if (lane == 0) { d[l] = dl - p; e[l] = gq; e[m] = 0.f; }
      }
      __syncwarp();
    }
    if (fail) break;
  }
  __syncwarp();
  // order by descending |theta|; ties: ascending signed value, then ascending index
  // (every warp fills its private copy of the permutation; warp 0 of the group writes theta)
  for (int j = lane; j < K; j += 32) {
    float dj = d[j], aj = fabsf(dj);
    int rank = 0;
    for (int i = 0; i < K; ++i) {
      float di = d[i], ai = fabsf(di);
      bool before = (ai > aj) || (ai == aj && (di < dj || (di == dj && i < j)));
      rank += before ? 1 : 0;
    }
    e[j] = __int_as_float(rank);   // e is dead after QL: reuse as the permutation
    if (wg == 0) theta[(int64_t)g * K + rank] = dj;
  }
  __syncwarp();
  if (tg == 0) status[g] = fail;
  for (int n = tg; n < N; n += gthreads)
    for (int k = 0; k < K; ++k)
      V[((int64_t)g * N + n) * K + __float_as_int(e[k])] = Zs[n * KP + k];
}

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

int lnb_lanczos_tridiag(lnb_stream_t stream, const float* A, const uint8_t* mask, const float* q1,
                        int B, int N, int K, float* T, float* Q, float* alpha, float* beta,
                        int32_t* idx) {
  LNB_REQUIRE(A && q1 && T && Q && alpha && beta && idx, "lanczos_tridiag: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && K >= 1, "lanczos_tridiag: bad dims B=%d N=%d K=%d", B, N, K);
  if (B == 0) return LNB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int iters = N < K ? N : K;
  if (N <= LNB_LANCZOS_FUSED_MAX_N && K <= LNB_LANCZOS_MAX_K) {
    // the fused kernel without its QL stage: operator rows loaded coalesced ONCE and packed on chip,
    // butterfly projections (it replaced the round-1 warp / resident-operator kernels at every size)
    const int rc = lnb_lanczos_ritz(stream, A, mask, q1, B, N, K, 0, T, Q, alpha, beta, idx, nullptr, nullptr, nullptr);
    if (rc != LNB_ERR_UNSUPPORTED) return rc;
  }
  {
    const int NP = (N + 3) & ~3;
    size_t base = ((size_t)(iters + 1) * NP + NP + 4 * (size_t)K + 1 + 32) * sizeof(float);
    size_t stage = (size_t)N * (N + 1) * sizeof(float);
    int stage_A = (base + stage <= 220 * 1024) ? 1 : 0;
    size_t shm = base + (stage_A ? stage : 0);
    LNB_REQUIRE(shm <= lnb::SMEM_MAX,
                "lanczos_tridiag: Krylov basis (N=%d, K=%d) does not fit shared memory", N, K);
    cudaFuncSetAttribute(lanczos_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)shm);
    lanczos_cta_kernel<<<B, CTA_THREADS, shm, s>>>(A, mask, q1, B, N, K, stage_A, T, Q, alpha,
                                                    beta, idx);
  }
  lnb::count_launch();
  return lnb::finish_launch("lanczos_tridiag");
}

int lnb_tridiag_ritz(lnb_stream_t stream, const float* alpha, const float* beta, const float* Q,
                     int B, int N, int K, float* theta, float* ritz_vec, int32_t* status) {
  LNB_REQUIRE(alpha && beta && Q && theta && ritz_vec && status, "tridiag_ritz: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && K >= 1, "tridiag_ritz: bad dims B=%d N=%d K=%d", B, N, K);
  if (B == 0) return LNB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int KP = K | 1;
  if (N <= 32) {
    size_t shm = (size_t)4 * (32 * KP + 8 * K) * sizeof(float);
    LNB_REQUIRE(shm <= lnb::SMEM_MAX, "tridiag_ritz: K=%d too large", K);
    if (shm > 48 * 1024)
      cudaFuncSetAttribute(tridiag_ritz_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)shm);
    tridiag_ritz_kernel<1><<<lnb::ceil_div(B, 4), 128, shm, s>>>(alpha, beta, Q, B, N, K, theta,
                                                                  ritz_vec, status);
  } else {
    size_t shm = ((size_t)N * KP + 8 * K) * sizeof(float);
    LNB_REQUIRE(shm <= lnb::SMEM_MAX, "tridiag_ritz: N=%d K=%d does not fit shared memory", N, K);
    cudaFuncSetAttribute(tridiag_ritz_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)shm);
    tridiag_ritz_kernel<4><<<B, 128, shm, s>>>(alpha, beta, Q, B, N, K, theta, ritz_vec, status);
  }
  lnb::count_launch();
  return lnb::finish_launch("tridiag_ritz");
}

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
