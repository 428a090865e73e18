// Device routines of the fp64 symmetric eigensolver (graph_eigs.cu), shared by lnb_sym_eigs,
// lnb_graph_eigs_sparse and lnb_spectral_partition.
//
//   1. Householder tridiagonalisation of the leading n x n block (lower triangle, packed in shared
//      memory; the reflectors overwrite the columns they annihilate, as LAPACK's dsptrd does),
//   2. implicit-shift QL on the tridiagonal with the rotations accumulated into Z (the QL stage of
//      lanczos_fused.cu, in fp64),
//   3. the reference's ordering: descending |lambda|, ties by ascending lambda (np.argsort(-|w|,
//      kind='mergesort') over eigh's ascending order), then the first kk,
//   4. the back-transform Q Z of only those columns.
//
// Work unit: a group of W warps per graph (W = 1: one warp, W = 4: one 128-thread CTA); a thread owns
// one row of A and of Z.  Every reduction has a fixed order: repeated launches are bit-identical.
#pragma once

#include <float.h>

#include "common.cuh"

namespace eigs {

constexpr int GE_THREADS = 128;
constexpr int GE_SWEEPS = 60;    // QL sweeps per eigenvalue before status bit 0 is set

// packed lower triangle, row-major: element (i, j), i >= j
__device__ __forceinline__ int tri(int i, int j) { return i * (i + 1) / 2 + j; }

__host__ __device__ constexpr int tri_doubles(int N) { return (N * (N + 1) / 2 + 1) & ~1; }

// per graph: packed A, Z [N][N|1], (d, e) per warp, tau / sub / v / w / scale, reduction slots, perm
__host__ __device__ constexpr size_t graph_doubles(int N, int W) {
  return (size_t)tri_doubles(N) + (size_t)N * (N | 1) + (size_t)W * 2 * N + 5 * (size_t)N + 8 + (N + 1) / 2;
}

template <int W>
__device__ __forceinline__ void gsync() {
  if (W == 1) __syncwarp(); else __syncthreads();
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// sum over the graph's threads in a fixed order (every thread gets the same bits)
template <int W>
__device__ __forceinline__ double group_sum(double v, double* red) {
  v = warp_sum_d(v);
  if (W == 1) return v;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = red[0];
#pragma unroll
  for (int w = 1; w < W; ++w) s += red[w];
  return s;
}

// The shared-memory layout of one graph (graph_doubles(N, W) doubles from base).  The pointers are
// computed where they are used, so they hold no registers across the solver's loops.
struct Work {
  double* base;
  int N, W, wg, ZS;

  __device__ __forceinline__ Work(double* base_, int N_, int W_, int wg_)
      : base(base_), N(N_), W(W_), wg(wg_), ZS(N_ | 1) {}
  __device__ __forceinline__ double* Ap() const { return base; }                  // packed A, then reflectors
  __device__ __forceinline__ double* Z() const { return base + tri_doubles(N); }  // [N][ZS] rotations / vectors
  __device__ __forceinline__ double* d0() const { return Z() + (size_t)N * ZS; }  // warp 0's eigenvalues
  __device__ __forceinline__ double* dq() const { return d0() + (size_t)wg * 2 * N; }   // this warp's (d, e)
  __device__ __forceinline__ double* eq() const { return dq() + N; }
  __device__ __forceinline__ double* taus() const { return d0() + (size_t)W * 2 * N; }
  __device__ __forceinline__ double* sub() const { return taus() + N; }          // subdiagonal
  __device__ __forceinline__ double* hv() const { return taus() + 2 * N; }       // reflector v (v[j+1] = 1)
  __device__ __forceinline__ double* hw() const { return taus() + 3 * N; }       // w = p - (tau/2)(p.v) v
  __device__ __forceinline__ double* sc() const { return taus() + 4 * N; }       // deg^-1/2 (producers)
  __device__ __forceinline__ double* red() const { return taus() + 5 * N; }
  __device__ __forceinline__ int* perm() const {                                  // perm[r]: column of pair r
    return reinterpret_cast<int*>(taus() + 5 * N + 8);
  }
};

// ---- Householder tridiagonalisation: column j's reflector maps A[j+2:, j] to zero ----------------
template <int W>
__device__ __forceinline__ void tridiagonalize(const Work& w, int n, int t) {
  double* Ap = w.Ap();
  for (int j = 0; j + 2 < n; ++j) {
    const double xi = (t > j + 1 && t < n) ? Ap[tri(t, j)] : 0.0;
    const double sigma = group_sum<W>(xi * xi, w.red());
    const double alpha = Ap[tri(j + 1, j)];
    if (sigma == 0.0) {                         // already reduced: H = I
      if (t == 0) { w.taus()[j] = 0.0; w.sub()[j] = alpha; }
      gsync<W>();
      continue;
    }
    const double beta = -copysign(sqrt(alpha * alpha + sigma), alpha);
    const double tau = (beta - alpha) / beta;
    const double scal = 1.0 / (alpha - beta);
    const double vi = (t == j + 1) ? 1.0 : xi * scal;
    if (t < n) w.hv()[t] = (t > j) ? vi : 0.0;
    gsync<W>();
    // p = tau A22 v over the trailing block; row t reads its own row left of the diagonal and its
    // column below it
    double p = 0.0;
    if (t > j && t < n) {
      for (int k = j + 1; k <= t; ++k) p = fma(Ap[tri(t, k)], w.hv()[k], p);
      for (int k = t + 1; k < n; ++k) p = fma(Ap[tri(k, t)], w.hv()[k], p);
      p *= tau;
    }
    const double pv = group_sum<W>(p * ((t > j && t < n) ? vi : 0.0), w.red());
    const double wi = p - 0.5 * tau * pv * vi;
    if (t > j && t < n) w.hw()[t] = wi;
    gsync<W>();
    if (t > j && t < n) {
      for (int k = j + 1; k <= t; ++k) Ap[tri(t, k)] -= vi * w.hw()[k] + wi * w.hv()[k];
      if (t > j + 1) Ap[tri(t, j)] = vi;        // keep the reflector where x was
    }
    if (t == 0) { w.taus()[j] = tau; w.sub()[j] = beta; }
    gsync<W>();
  }
}

// ---- (d, e) into every warp's private copy, Z = I, then implicit-shift QL; every warp carries the
// scalar recurrence, thread t rotates row t of Z.  Returns 1 when the sweeps ran out.
// An off-diagonal splits below eps * ||T|| (EISPACK tql2's test), not below eps * (|d_m| + |d_m+1|):
// where a whole eigenspace sits at the rounding level (the complete graph's eigenvalue 0, n - 1 times)
// the pairwise test never fires.  Eigenvalues stay within eps * ||T|| of exact.
template <int W>
__device__ __forceinline__ int tridiag_ql(const Work& w, int n, int t, int lane) {
  const double* Ap = w.Ap();
  double* dq = w.dq();
  double* eq = w.eq();
  double* Z = w.Z();
  const int ZS = w.ZS;
  for (int i = lane; i < n; i += 32) {
    dq[i] = Ap[tri(i, i)];
    eq[i] = (i + 2 < n) ? w.sub()[i] : (i + 1 < n ? Ap[tri(i + 1, i)] : 0.0);
  }
  gsync<W>();
  if (t < n)
    for (int k = 0; k < n; ++k) Z[(size_t)t * ZS + k] = (t == k) ? 1.0 : 0.0;
  gsync<W>();

  double tnorm = 0.0;
  for (int i = lane; i < n; i += 32) tnorm = fmax(tnorm, fabs(dq[i]) + fabs(eq[i]) + (i ? fabs(eq[i - 1]) : 0.0));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) tnorm = fmax(tnorm, __shfl_xor_sync(0xffffffffu, tnorm, o));
  const double etol = DBL_EPSILON * tnorm;
  int fail = 0;
  for (int l = 0; l < n; ++l) {
    int sweeps = 0;
    while (true) {
      int m = l;
      for (; m < n - 1; ++m)
        if (fabs(eq[m]) <= etol) break;
      if (m == l) break;
      if (++sweeps > GE_SWEEPS) { fail = 1; break; }
      double g = (dq[l + 1] - dq[l]) / (2.0 * eq[l]);
      double r = sqrt(g * g + 1.0);
      g = dq[m] - dq[l] + eq[l] / (g + copysign(r, g));
      double s = 1.0, c = 1.0, p = 0.0;
      bool underflow = false;
      for (int i = m - 1; i >= l; --i) {
        // every lane carries the recurrence; lane 0 alone stores, after all lanes have read this row
        const double ei = eq[i], di1 = dq[i + 1], di = dq[i];
        __syncwarp();
        const double f = s * ei;
        const double bb = c * ei;
        r = sqrt(f * f + g * g);
        if (r == 0.0) {
          if (lane == 0) { eq[i + 1] = r; dq[i + 1] = di1 - p; eq[m] = 0.0; }
          underflow = true;
          break;
        }
        const double ir = 1.0 / r;
        s = f * ir;
        c = g * ir;
        g = di1 - p;
        const double rr = (di - g) * s + 2.0 * c * bb;
        p = s * rr;
        if (lane == 0) { eq[i + 1] = r; dq[i + 1] = g + p; }
        g = c * rr - bb;
        if (t < n) {
          double* zr = Z + (size_t)t * ZS;
          const double z1 = zr[i + 1], z0 = zr[i];
          zr[i + 1] = s * z0 + c * z1;
          zr[i] = c * z0 - s * z1;
        }
      }
      if (!underflow) {
        const double dl = dq[l];
        __syncwarp();
        if (lane == 0) { dq[l] = dl - p; eq[l] = g; eq[m] = 0.0; }
      }
      __syncwarp();
    }
    if (fail) break;
  }
  gsync<W>();
  return fail;
}

// ---- the reference's order: descending |lambda|, then ascending lambda, then index; perm[0, kk) -----
template <int W>
__device__ __forceinline__ void order_pairs(const Work& w, int n, int kk, int t) {
  constexpr int GT = W * 32;
  const double* d0 = w.d0();
  for (int r = t; r < kk; r += GT) w.perm()[r] = r;  // only a NaN operator leaves a rank unfilled
  gsync<W>();
  for (int j = t; j < n; j += GT) {
    const double dj = d0[j], aj = fabs(dj);
    int rank = 0;
    for (int i = 0; i < n; ++i) {
      const double di = d0[i], ai = fabs(di);
      rank += ((ai > aj) || (ai == aj && (di < dj || (di == dj && i < j)))) ? 1 : 0;
    }
    if (rank < kk) w.perm()[rank] = j;
  }
  gsync<W>();
}

// ---- back-transform of the kept columns perm[0, kk) only: z <- H_0 ... H_{n-3} z ------------------
template <int W>
__device__ __forceinline__ void back_transform(const Work& w, int n, int kk, int t) {
  constexpr int GT = W * 32;
  const double* Ap = w.Ap();
  double* Z = w.Z();
  const int ZS = w.ZS;
  for (int r = t; r < kk; r += GT) {
    const int col = w.perm()[r];
    for (int j = n - 3; j >= 0; --j) {
      const double tau = w.taus()[j];
      if (tau == 0.0) continue;
      double s = Z[(size_t)(j + 1) * ZS + col];
      for (int i = j + 2; i < n; ++i) s = fma(Ap[tri(i, j)], Z[(size_t)i * ZS + col], s);
      s *= tau;
      Z[(size_t)(j + 1) * ZS + col] -= s;
      for (int i = j + 2; i < n; ++i) Z[(size_t)i * ZS + col] -= s * Ap[tri(i, j)];
    }
  }
  gsync<W>();
}

}  // namespace eigs
