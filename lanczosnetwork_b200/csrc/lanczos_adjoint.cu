// Training kernels of AdaLanczosNet's Lanczos layer, for sm_90a, one CTA per graph, no atomics:
//   * lnb_lanczos_tridiag_train / lnb_lanczos_tridiag_backward: the K-step recurrence of train._lanczos_train
//     (below) and its exact adjoint;
//   * lnb_tridiag_powers_backward: the adjoint of lnb_tridiag_powers.
//
// Adjoint of lnb_tridiag_powers (AdaLanczosNet's powers of the tridiagonal T, the input of its learned
// spectral filter) for the training path: one CTA per graph, no atomics.
//
// The forward is P_1 = T (every entry) and P_{p+1} = P_p Tri(T), where Tri(T) keeps the three diagonals
// of T (lnb_tridiag_powers reads only those), with out[:, :, s, :] = P_{powers[s]}.  Its adjoint, with
// G_p = gOut[:, :, s, :] when p = powers[s] and 0 otherwise:
//   H_pmax = G_pmax;  for p = pmax-1 .. 1:  gTri += (P_p^T H_{p+1}) on the three diagonals,
//                                           H_p = G_p + H_{p+1} Tri(T)^T;
//   gT = H_1 + gTri.
// The CTA recomputes P_1 .. P_{pmax-1} with the forward's arithmetic and keeps them in shared memory,
// then runs the reverse sweep; each entry of gTri is owned by one thread, which sums its dot products
// over p in a fixed order (deterministic).  This replaces ~pmax forward and ~2 pmax backward GEMM
// launches of the bmm chain.
#include "common.cuh"

namespace {

constexpr int TPB_THREADS = 256;

struct PowerList { int v[32]; };

__global__ void __launch_bounds__(TPB_THREADS)
tridiag_powers_backward_kernel(const float* __restrict__ T, const float* __restrict__ gOut, int K,
                               PowerList pw, int S, float* __restrict__ gT) {
  extern __shared__ float smem[];
  const int g = blockIdx.x, tid = threadIdx.x;
  const int KK = K * K, pmax = pw.v[S - 1];
  float* dg = smem;              // K  : T[c][c]
  float* up = dg + K;            // K  : T[c-1][c]
  float* lo = up + K;            // K  : T[c+1][c]
  float* acc = lo + K;           // 3K : gTri, [0,K) diagonal, [K,2K) T[m][m+1], [2K,3K) T[m+1][m]
  float* H0 = acc + 3 * K;       // K x K
  float* H1 = H0 + KK;           // K x K
  float* P = H1 + KK;            // (pmax - 1) x K x K : P_1 .. P_{pmax-1}
  const float* Tg = T + (int64_t)g * KK;
  const float* Gg = gOut + (int64_t)g * K * S * K;   // [K, S, K]

  for (int c = tid; c < K; c += TPB_THREADS) {
    dg[c] = Tg[c * K + c];
    up[c] = c > 0 ? Tg[(c - 1) * K + c] : 0.f;
    lo[c] = c < K - 1 ? Tg[(c + 1) * K + c] : 0.f;
  }
  for (int e = tid; e < 3 * K; e += TPB_THREADS) acc[e] = 0.f;
  if (pmax > 1)
    for (int e = tid; e < KK; e += TPB_THREADS) P[e] = Tg[e];
  __syncthreads();
  // forward recompute, the arithmetic of tridiag_powers_kernel
  for (int p = 1; p + 1 < pmax; ++p) {
    const float* cur = P + (size_t)(p - 1) * KK;
    float* nxt = P + (size_t)p * KK;
    for (int e = tid; e < KK; e += TPB_THREADS) {
      const int r = e / K, c = e - r * K;
      float v = cur[r * K + c] * dg[c];
      if (c > 0) v = fmaf(cur[r * K + c - 1], up[c], v);
      if (c < K - 1) v = fmaf(cur[r * K + c + 1], lo[c], v);
      nxt[e] = v;
    }
    __syncthreads();
  }

  // reverse sweep: H = H_{p+1} on entry of step p
  int s = S - 1;
  for (int e = tid; e < KK; e += TPB_THREADS) {
    const int r = e / K, c = e - r * K;
    H0[e] = Gg[((int64_t)r * S + s) * K + c];
  }
  --s;
  __syncthreads();
  float* H = H0;
  float* Hn = H1;
  for (int p = pmax - 1; p >= 1; --p) {
    const float* Pp = P + (size_t)(p - 1) * KK;
    // gTri[m][c] += sum_r P_p[r][m] H[r][c], |m - c| <= 1
    for (int e = tid; e < 3 * K; e += TPB_THREADS) {
      const int kind = e / K, m = e - kind * K;
      const int c = kind == 0 ? m : (kind == 1 ? m + 1 : m);
      const int mm = kind == 2 ? m + 1 : m;
      if (c < K && mm < K) {
        float a = 0.f;
        for (int r = 0; r < K; ++r) a = fmaf(Pp[r * K + mm], H[r * K + c], a);
        acc[e] += a;
      }
    }
    // H_p[r][m] = G_p[r][m] + sum_c H[r][c] Tri[m][c]
    const bool sel = s >= 0 && pw.v[s] == p;
    for (int e = tid; e < KK; e += TPB_THREADS) {
      const int r = e / K, m = e - r * K;
      float v = H[r * K + m] * dg[m];
      if (m + 1 < K) v = fmaf(H[r * K + m + 1], up[m + 1], v);   // Tri[m][m+1]
      if (m > 0) v = fmaf(H[r * K + m - 1], lo[m - 1], v);       // Tri[m][m-1]
      if (sel) v += Gg[((int64_t)r * S + s) * K + m];
      Hn[e] = v;
    }
    if (sel) --s;
    __syncthreads();
    float* t = H; H = Hn; Hn = t;
  }

  float* gTg = gT + (int64_t)g * KK;
  for (int e = tid; e < KK; e += TPB_THREADS) {
    const int r = e / K, c = e - r * K;
    float v = H[e];
    if (c == r) v += acc[r];
    else if (c == r + 1) v += acc[K + r];
    else if (r == c + 1) v += acc[2 * K + c];
    gTg[e] = v;
  }
}

size_t powers_backward_smem(int K, int pmax) {
  return ((size_t)6 * K + (size_t)(pmax + 1) * K * K) * sizeof(float);
}


// ------------------------------------------------------------------------------------------------------
// The Lanczos recurrence of train._lanczos_train (the reference's rules, model/ada_lanczos_net.py:139-247,
// with the inference kernel's two classical block Gram-Schmidt passes):
//   q_0 = (q1 . m) / ||q1 . m||;  for i < iters = min(N, K):
//     z = A q_i,  a_i = q_i . z,  z0 = z - a_i q_i - b_{i-1} q_{i-1}
//     two passes (i > 0):  c_j = (q_j . z_in) s_j,  s_j = 1 / (q_j . q_j + EPS),  z_out = z_in - sum_j c_j q_j
//     b_i = ||z2||,  ok_i = ok_{i-1} & (b_i >= 1e-4),  q_{i+1} = z2 ok_i / (b_i + EPS)
//   idx = min(#ok, #real nodes); column k is kept when ok_k and k < idx, node rows when n < idx.
// One CTA of 128 threads per graph, thread n owns node n (N <= 128): the operator, the basis, the adjoints
// of the basis and the operator's gradient live in shared memory.  Both entries run the same forward code
// (fixed reduction order, deterministic), so the backward differentiates, bit for bit, the tape the
// training forward returned.  The backward then sweeps i = iters-1 .. 0, recomputing the step's
// intermediates (z, z0, z1, z2, the projections) from the basis, and accumulates
//   dA += zbar q_i^T  in the order of the sweep.  Acceptance, idx and the masks are data (no gradient).
// ------------------------------------------------------------------------------------------------------
constexpr int LZ_THREADS = 128;
static_assert(LNB_LANCZOS_TRAIN_MAX_N <= LZ_THREADS, "thread n owns node n");

__device__ __forceinline__ float lz_block_sum(float v, float* red) {
  v = lnb::warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < LZ_THREADS / 32; ++w) t += red[w];
  __syncthreads();
  return t;
}

// out[j] = vec . q_j for j < i (one warp per j, fixed order); ends with a barrier
__device__ __forceinline__ void lz_project(const float* vec, const float* Qs, int N, int i, float* out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = warp; j < i; j += LZ_THREADS / 32) {
    float s = 0.f;
    for (int m = lane; m < N; m += 32) s = fmaf(vec[m], Qs[j * N + m], s);
    s = lnb::warp_sum(s);
    if (lane == 0) out[j] = s;
  }
  __syncthreads();
}

struct LzStep { float z, z0, z1, z2, a, b; };

// step i of the recurrence for node n (every thread calls it); pr1 / pr2: the raw projections of the passes
__device__ LzStep lz_step(int i, int n, int N, const float* As, int lda, const float* Qs, const float* iqs,
                          float bprev, float* zs, float* pr1, float* pr2, float* red) {
  const bool act = n < N;
  const float* qi = Qs + i * N;
  LzStep st;
  float z = 0.f;
  if (act)
    for (int m = 0; m < N; ++m) z = fmaf(As[n * lda + m], qi[m], z);
  const float qn = act ? qi[n] : 0.f;
  st.z = z;
  st.a = lz_block_sum(qn * z, red);
  float z0 = 0.f;
  if (act) {
    z0 = z - st.a * qn;
    if (i > 0) z0 -= bprev * Qs[(i - 1) * N + n];
  }
  st.z0 = z0;
  float z1 = z0, z2 = z0;
  if (i > 0) {
    if (act) zs[n] = z0;
    __syncthreads();
    lz_project(zs, Qs, N, i, pr1);
    if (act) {
      float t = 0.f;
      for (int j = 0; j < i; ++j) t = fmaf(pr1[j] * iqs[j], Qs[j * N + n], t);
      z1 = z0 - t;
    }
    __syncthreads();
    if (act) zs[n] = z1;
    __syncthreads();
    lz_project(zs, Qs, N, i, pr2);
    if (act) {
      float t = 0.f;
      for (int j = 0; j < i; ++j) t = fmaf(pr2[j] * iqs[j], Qs[j * N + n], t);
      z2 = z1 - t;
    }
  }
  st.z1 = z1;
  st.z2 = z2;
  st.b = sqrtf(lz_block_sum(z2 * z2, red));
  return st;
}

struct LzParams {
  const float* A; const uint8_t* mask; const float* q1; int N, K;
  const float* gT; const float* gQ; float* gA;                    // backward (gA != null)
  float* T; float* Q; float* alpha; float* beta; int32_t* idx;    // forward outputs (each may be null)
};

__global__ void __launch_bounds__(LZ_THREADS) lanczos_train_kernel(const LzParams P) {
  extern __shared__ float smem[];
  const int g = blockIdx.x, n = threadIdx.x, N = P.N, K = P.K;
  const int iters = N < K ? N : K;
  const int lda = N + 1;
  const bool act = n < N;
  float* As = smem;                          // N x (N+1)
  float* Qs = As + N * lda;                  // (K+1) x N basis
  float* iqs = Qs + (K + 1) * N;             // K+1
  float* al = iqs + K + 1;                   // K
  float* be = al + K;                        // K
  float* okf = be + K;                       // K
  float* vcol = okf + K;                     // K
  float* pr1 = vcol + K;                     // K
  float* pr2 = pr1 + K;                      // K
  float* cb = pr2 + K;                       // K
  float* red = cb + K;                       // 32
  float* zs = red + 32;                      // N
  float* gAs = zs + N;                       // backward: N x (N+1)
  float* Qb = gAs + N * lda;                 // backward: (K+1) x N adjoints of the basis
  float* abar = Qb + (K + 1) * N;            // K
  float* bbar = abar + K;                    // K
  float* sbar = bbar + K;                    // K+1

  const float* Ag = P.A + (size_t)g * N * N;
  for (int e = threadIdx.x; e < N * N; e += LZ_THREADS) As[(e / N) * lda + e % N] = Ag[e];
  float mk = 0.f, v = 0.f;
  if (act) {
    mk = P.mask ? (P.mask[(size_t)g * N + n] ? 1.f : 0.f) : 1.f;
    v = P.q1[(size_t)g * N + n] * mk;
  }
  const float nrm = sqrtf(lz_block_sum(v * v, red));
  const int nreal = (int)(lz_block_sum(mk, red) + 0.5f);
  const float q0 = v / nrm;
  if (act) Qs[n] = q0;
  const float qq0 = lz_block_sum(act ? q0 * q0 : 0.f, red);
  if (n == 0) iqs[0] = 1.f / (qq0 + lnb::LANCZOS_EPS);

  float bprev = 0.f, okv = 1.f;
  int count = 0;
  for (int i = 0; i < iters; ++i) {
    const LzStep st = lz_step(i, n, N, As, lda, Qs, iqs, bprev, zs, pr1, pr2, red);
    okv = (st.b >= lnb::LANCZOS_BETA_LOWER_BOUND) ? okv : 0.f;
    count += (okv != 0.f) ? 1 : 0;
    const float qn = act ? (st.z2 * okv) / (st.b + lnb::LANCZOS_EPS) : 0.f;
    if (act) Qs[(i + 1) * N + n] = qn;
    const float qq = lz_block_sum(qn * qn, red);
    if (n == 0) { iqs[i + 1] = 1.f / (qq + lnb::LANCZOS_EPS); al[i] = st.a; be[i] = st.b; okf[i] = okv; }
    bprev = st.b;
    __syncthreads();
  }
  const int idx = count < nreal ? count : nreal;
  for (int k = n; k < K; k += LZ_THREADS) vcol[k] = (k < iters && okf[k] != 0.f && k < idx) ? 1.f : 0.f;
  __syncthreads();

  if (P.idx && n == 0) P.idx[g] = idx;
  for (int k = n; k < K; k += LZ_THREADS) {
    if (P.alpha) P.alpha[(size_t)g * K + k] = k < iters ? al[k] * vcol[k] : 0.f;
    if (P.beta) P.beta[(size_t)g * K + k] = k < iters - 1 ? be[k] * vcol[k] : 0.f;
  }
  if (P.T) {
    float* Tg = P.T + (size_t)g * K * K;
    for (int e = n; e < K * K; e += LZ_THREADS) {
      const int r = e / K, c = e - r * K;
      float t = 0.f;
      if (r == c && r < iters) t = al[r] * vcol[r];
      else if (c == r + 1 && r < iters - 1) t = be[r] * vcol[r];
      else if (r == c + 1 && c < iters - 1) t = be[c] * vcol[c];
      Tg[e] = t;
    }
  }
  if (P.Q) {
    float* Qg = P.Q + (size_t)g * N * K;
    for (int e = n; e < N * K; e += LZ_THREADS) {
      const int r = e / K, k = e - r * K;
      Qg[e] = k < iters ? Qs[k * N + r] * (vcol[k] * (r < idx ? 1.f : 0.f)) : 0.f;
    }
  }
  if (!P.gA) return;

  // ---- reverse sweep ------------------------------------------------------------------------------------
  const float* gTg = P.gT + (size_t)g * K * K;
  for (int k = n; k < K; k += LZ_THREADS) {
    abar[k] = k < iters ? gTg[k * K + k] * vcol[k] : 0.f;
    bbar[k] = k < iters - 1 ? (gTg[k * K + k + 1] + gTg[(k + 1) * K + k]) * vcol[k] : 0.f;
  }
  for (int k = n; k <= K; k += LZ_THREADS) sbar[k] = 0.f;
  for (int e = threadIdx.x; e < N * lda; e += LZ_THREADS) gAs[e] = 0.f;
  if (act) {
    const float rk = n < idx ? 1.f : 0.f;
    for (int k = 0; k <= K; ++k)
      Qb[k * N + n] = k < iters ? P.gQ[((size_t)g * N + n) * K + k] * (vcol[k] * rk) : 0.f;
  }
  __syncthreads();
  for (int i = iters - 1; i >= 0; --i) {
    const float bp = i > 0 ? be[i - 1] : 0.f;
    const LzStep st = lz_step(i, n, N, As, lda, Qs, iqs, bp, zs, pr1, pr2, red);
    const float qi = act ? Qs[i * N + n] : 0.f;
    const float qnext = act ? Qs[(i + 1) * N + n] : 0.f;
    // q_{i+1} is final: add the gradient through s_{i+1} = 1 / (q.q + EPS)
    const float sn = iqs[i + 1];
    const float qbn = act ? Qb[(i + 1) * N + n] - 2.f * sn * sn * sbar[i + 1] * qnext : 0.f;
    const float ok = okf[i], inv = 1.f / (st.b + lnb::LANCZOS_EPS);
    float zb = qbn * ok * inv;
    const float t = lz_block_sum(qbn * st.z2, red);
    const float bb = bbar[i] - ok * t * inv * inv;
    if (st.b > 0.f) zb += bb * st.z2 / st.b;
    if (i > 0) {
      // pass 2 (z1 -> z2), then pass 1 (z0 -> z1)
      for (int pass = 1; pass >= 0; --pass) {
        const float* pr = pass ? pr2 : pr1;
        const float zin = pass ? st.z1 : st.z0;
        if (act) zs[n] = zb;
        __syncthreads();
        lz_project(zs, Qs, N, i, cb);                  // cb_j = q_j . zbar_out
        float zin_b = zb;
        if (act) {
          for (int j = 0; j < i; ++j) {
            const float d = -cb[j] * iqs[j];
            Qb[j * N + n] += -(pr[j] * iqs[j]) * zb + d * zin;
            zin_b = fmaf(d, Qs[j * N + n], zin_b);
          }
        }
        if (n == 0)
          for (int j = 0; j < i; ++j) sbar[j] += -cb[j] * pr[j];
        zb = zin_b;
        __syncthreads();
      }
    }
    // three-term step
    const float ab = abar[i] - lz_block_sum(qi * zb, red);
    if (i > 0) {
      const float tb = lz_block_sum(act ? Qs[(i - 1) * N + n] * zb : 0.f, red);
      if (n == 0) bbar[i - 1] += -tb;
      if (act) Qb[(i - 1) * N + n] += -bp * zb;
    }
    const float zbar = zb + ab * qi;
    if (act) {
      Qb[i * N + n] += -st.a * zb + ab * st.z;
      for (int m = 0; m < N; ++m) gAs[n * lda + m] = fmaf(zbar, Qs[i * N + m], gAs[n * lda + m]);
      zs[n] = zbar;
    }
    __syncthreads();
    if (act) {
      float s = 0.f;
      for (int m = 0; m < N; ++m) s = fmaf(As[m * lda + n], zs[m], s);
      Qb[i * N + n] += s;
    }
    __syncthreads();
  }
  float* gAg = P.gA + (size_t)g * N * N;
  for (int e = threadIdx.x; e < N * N; e += LZ_THREADS) gAg[e] = gAs[(e / N) * lda + e % N];
}

size_t lanczos_train_smem(int N, int K, bool backward) {
  const size_t lda = (size_t)N + 1;
  size_t w = (size_t)N * lda + (size_t)(K + 1) * N + (K + 1) + 8 * (size_t)K + 32 + N;
  if (backward) w += (size_t)N * lda + (size_t)(K + 1) * N + 3 * (size_t)K + 1;
  return w * sizeof(float);
}

int launch_lanczos_train(lnb_stream_t stream, const LzParams& p, int B, const char* who) {
  if (!(p.N >= 1 && p.N <= LNB_LANCZOS_TRAIN_MAX_N && p.K >= 1 && p.K <= LNB_LANCZOS_MAX_K &&
        lanczos_train_smem(p.N, p.K, true) <= lnb::SMEM_MAX)) {
    lnb::set_err("%s: N=%d K=%d outside 1 <= N <= 128, 1 <= K <= 64", who, p.N, p.K);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE(B >= 0, "%s: bad B=%d", who, B);
  if (B == 0) return LNB_OK;
  LNB_REQUIRE(p.A && p.q1, "%s: null pointer", who);
  const size_t shm = lanczos_train_smem(p.N, p.K, p.gA != nullptr);
  cudaFuncSetAttribute(lanczos_train_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
  lanczos_train_kernel<<<B, LZ_THREADS, shm, (cudaStream_t)stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch(who);
}

}  // namespace

extern "C" {
int lnb_lanczos_tridiag_train(lnb_stream_t stream, const float* A, const uint8_t* mask, const float* q1, int B,
                              int N, int K, float* T, float* Q, float* alpha, float* beta, int32_t* idx) {
  LzParams p = {A, mask, q1, N, K, nullptr, nullptr, nullptr, T, Q, alpha, beta, idx};
  return launch_lanczos_train(stream, p, B, "lanczos_tridiag_train");
}

int lnb_lanczos_tridiag_backward(lnb_stream_t stream, const float* A, const uint8_t* mask, const float* q1,
                                 int B, int N, int K, const float* gT, const float* gQ, float* gA, float* T,
                                 float* Q) {
  if (B > 0) LNB_REQUIRE(gT && gQ && gA, "lanczos_tridiag_backward: null pointer");
  LzParams p = {A, mask, q1, N, K, gT, gQ, gA, T, Q, nullptr, nullptr, nullptr};
  return launch_lanczos_train(stream, p, B, "lanczos_tridiag_backward");
}


int lnb_tridiag_powers_backward(lnb_stream_t stream, const float* T, const float* gOut, int B, int K,
                                const int* powers, int S, float* gT) {
  LNB_REQUIRE(powers, "tridiag_powers_backward: null powers");
  LNB_REQUIRE(B >= 0 && K >= 1 && S >= 1 && S <= LNB_TRIDIAG_POWERS_MAX_S,
              "tridiag_powers_backward: bad dims B=%d K=%d S=%d",
              B, K, S);
  for (int i = 0; i < S; ++i)
    LNB_REQUIRE(powers[i] >= 1 && (i == 0 || powers[i] > powers[i - 1]),
                "tridiag_powers_backward: powers must be positive and strictly increasing");
  const size_t shm = powers_backward_smem(K, powers[S - 1]);
  if (shm > lnb::SMEM_MAX) {
    lnb::set_err("tridiag_powers_backward: K=%d with powers up to %d needs %zu bytes of shared memory "
                 "(limit 227 KB)", K, powers[S - 1], shm);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  LNB_REQUIRE(T && gOut && gT, "tridiag_powers_backward: null pointer");
  PowerList pw;
  for (int i = 0; i < S; ++i) pw.v[i] = powers[i];
  if (shm > 48 * 1024)
    cudaFuncSetAttribute(tridiag_powers_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
  tridiag_powers_backward_kernel<<<B, TPB_THREADS, shm, (cudaStream_t)stream>>>(T, gOut, K, pw, S, gT);
  lnb::count_launch();
  return lnb::finish_launch("tridiag_powers_backward");
}

}  // extern "C"
