// Exact eigenpairs of one small symmetric operator per graph, in fp64: the reference's offline
// preprocessing (utils/data_helper.py:169-226 dense eigh branch, called from
// dataset/get_qm8_data.py:63-83 and truncated / zero padded to K at collate, dataset/qm8.py:265-291)
// on the device.
//
//   1. Householder tridiagonalisation of the leading n x n block (lower triangle, packed in shared
//      memory; the reflectors overwrite the columns they annihilate, as LAPACK's dsptrd does),
//   2. implicit-shift QL on the tridiagonal with the rotations accumulated into Z (the pattern of
//      tridiag_ritz_kernel, in fp64),
//   3. the reference's ordering: descending |lambda|, ties by ascending lambda (np.argsort(-|w|,
//      kind='mergesort') over eigh's ascending order), then the first min(n, K),
//   4. the back-transform Q Z of only those columns, one rounding to fp32 on the way out.
//
// Work unit: one warp per graph for N <= 32 (four graphs per CTA), one 128-thread CTA per graph
// above; a thread owns one row of A and of Z.  Every reduction has a fixed order: repeated launches
// are bit-identical.  Eigenvectors are determined up to sign (and up to a rotation inside a repeated
// eigenvalue's eigenspace), which no consumer sees: they read V diag(g(D)) V^T.
#include <float.h>

#include "common.cuh"

namespace {

constexpr int GE_THREADS = 128;
constexpr int GE_NMAX = 128;     // same limit as lnb_graph_prepare_sparse
constexpr int GE_KMAX = 128;
constexpr int GE_EMAX = 32;      // bond types of the sparse producer (one bit each)
constexpr int GE_SWEEPS = 60;    // QL sweeps per eigenvalue before status bit 0 is set

struct EigParams {
  // dense producer: A[((b * N + i) * N + j) * es], lower triangle read (eigh's default UPLO='L')
  const float* A; int64_t es;
  // sparse producer: bond lists + the fp64 deg^-1/2 table, as lnb_graph_prepare_sparse
  const int32_t* node_ptr; const int32_t* edge_ptr; const uint8_t* edges; const double* inv_sqrt_deg;
  int E;
  const int32_t* sizes;
  int B, N, K;
  float* D; float* V; int32_t* status;     // V: [B,N,K] (dense) or [node_ptr[B],K] rows (sparse)
};

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

template <int W, bool SPARSE>
__global__ void __launch_bounds__(GE_THREADS)
graph_eigs_kernel(const EigParams P) {
  extern __shared__ __align__(16) double ge_smem[];
  constexpr int GPC = 4 / W;                 // graphs per CTA
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = warp / W, wg = warp % W;
  const int t = wg * 32 + lane;              // row owned by this thread
  const int GT = W * 32;
  const int N = P.N, K = P.K, ZS = N | 1;
  const int b = blockIdx.x * GPC + grp;

  double* Ap = ge_smem + (size_t)grp * graph_doubles(N, W);
  double* Z = Ap + tri_doubles(N);
  double* dq = Z + (size_t)N * ZS + (size_t)wg * 2 * N;   // this warp's private (d, e) of the QL
  double* eq = dq + N;
  double* taus = Z + (size_t)N * ZS + (size_t)W * 2 * N;
  double* sub = taus + N;                     // subdiagonal of the tridiagonal
  double* hv = sub + N;                      // current reflector v (v[j+1] = 1)
  double* hw = hv + N;                        // w = p - (tau/2)(p.v) v
  double* sc = hw + N;                        // deg^-1/2 (sparse producer)
  double* red = sc + N;
  int* perm = reinterpret_cast<int*>(red + 8);   // perm[r] = column of Z holding the r-th pair
  if (b >= P.B) return;                       // whole groups only: a CTA-wide group has b < B

  const int n = min(max(P.sizes[b], 0), N);

  // ---- the fp64 operator: lower triangle, packed ----------------------------------------------
  if (SPARSE) {
    // bond-type bitmask per node pair (in Z's storage, free until QL): a bond listed twice with one
    // type counts once, as in lnb_graph_prepare_sparse's adjacency bitmaps
    uint32_t* mk = reinterpret_cast<uint32_t*>(Z);
    for (int i = t; i < n * n; i += GT) mk[i] = 0u;
    gsync<W>();
    const int e0 = P.edge_ptr[b], e1 = P.edge_ptr[b + 1];
    for (int e = e0 + t; e < e1; e += GT) {
      const uchar4 ed = reinterpret_cast<const uchar4*>(P.edges)[e];
      const int u = ed.x, v = ed.y, c = ed.z;
      if (u < n && v < n && c < P.E) {
        atomicOr(&mk[u * n + v], 1u << c);
        atomicOr(&mk[v * n + u], 1u << c);
      }
    }
    gsync<W>();
    if (t < n) {
      int deg = 1;                                        // the + I of L4
      for (int j = 0; j < n; ++j) deg += __popc(mk[t * n + j]);
      sc[t] = P.inv_sqrt_deg[deg < 255 ? deg : 255];
    }
    gsync<W>();
    if (t < n) {
      // the reference's (scale_i * m_ij) * scale_j with i the row: what eigh reads below the diagonal
      const double si = sc[t];
      for (int j = 0; j <= t; ++j) {
        const int m = (t == j ? 1 : 0) + __popc(mk[t * n + j]);
        Ap[tri(t, j)] = m ? (si * (double)m) * sc[j] : 0.0;
      }
    }
  } else {
    if (t < n) {
      const float* Ab = P.A + (int64_t)b * N * N * P.es;
      for (int j = 0; j <= t; ++j) Ap[tri(t, j)] = (double)Ab[((int64_t)t * N + j) * P.es];
    }
  }
  gsync<W>();

  // ---- Householder tridiagonalisation: column j's reflector maps A[j+2:, j] to zero ----------------
  for (int j = 0; j + 2 < n; ++j) {
    const double xi = (t > j + 1 && t < n) ? Ap[tri(t, j)] : 0.0;
    const double sigma = group_sum<W>(xi * xi, red);
    const double alpha = Ap[tri(j + 1, j)];
    if (sigma == 0.0) {                         // already reduced: H = I
      if (t == 0) { taus[j] = 0.0; sub[j] = alpha; }
      gsync<W>();
      continue;
    }
    const double beta = -copysign(sqrt(alpha * alpha + sigma), alpha);
    const double tau = (beta - alpha) / beta;
    const double scal = 1.0 / (alpha - beta);
    const double vi = (t == j + 1) ? 1.0 : xi * scal;
    if (t < n) hv[t] = (t > j) ? vi : 0.0;
    gsync<W>();
    // p = tau A22 v over the trailing block; row t reads its own row left of the diagonal and its
    // column below it
    double p = 0.0;
    if (t > j && t < n) {
      for (int k = j + 1; k <= t; ++k) p = fma(Ap[tri(t, k)], hv[k], p);
      for (int k = t + 1; k < n; ++k) p = fma(Ap[tri(k, t)], hv[k], p);
      p *= tau;
    }
    const double pv = group_sum<W>(p * ((t > j && t < n) ? vi : 0.0), red);
    const double wi = p - 0.5 * tau * pv * vi;
    if (t > j && t < n) hw[t] = wi;
    gsync<W>();
    if (t > j && t < n) {
      for (int k = j + 1; k <= t; ++k) Ap[tri(t, k)] -= vi * hw[k] + wi * hv[k];
      if (t > j + 1) Ap[tri(t, j)] = vi;        // keep the reflector where x was
    }
    if (t == 0) { taus[j] = tau; sub[j] = beta; }
    gsync<W>();
  }

  // ---- tridiagonal (d, e) into every warp's private copy; Z = I ----------------------------------
  for (int i = lane; i < n; i += 32) {
    dq[i] = Ap[tri(i, i)];
    eq[i] = (i + 2 < n) ? sub[i] : (i + 1 < n ? Ap[tri(i + 1, i)] : 0.0);
  }
  gsync<W>();
  if (t < n)
    for (int k = 0; k < n; ++k) Z[(size_t)t * ZS + k] = (t == k) ? 1.0 : 0.0;
  gsync<W>();

  // ---- implicit-shift QL; every warp carries the scalar recurrence, thread t rotates row t of Z ----
  // an off-diagonal splits below eps * ||T|| (EISPACK tql2's test), not below eps * (|d_m| + |d_m+1|):
  // where a whole eigenspace sits at the rounding level (the complete graph's eigenvalue 0, n - 1 times)
  // the pairwise test never fires.  Eigenvalues stay within eps * ||T|| of exact.
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

  // ---- the reference's order: descending |lambda|, then ascending lambda, then index --------------
  const int kk = min(n, K);
  const double* d0 = Z + (size_t)N * ZS;         // warp 0's eigenvalues (all copies are identical)
  for (int r = t; r < kk; r += GT) perm[r] = r;  // only a NaN operator leaves a rank unfilled
  gsync<W>();
  for (int j = t; j < n; j += GT) {
    const double dj = d0[j], aj = fabs(dj);
    int rank = 0;
    for (int i = 0; i < n; ++i) {
      const double di = d0[i], ai = fabs(di);
      rank += ((ai > aj) || (ai == aj && (di < dj || (di == dj && i < j)))) ? 1 : 0;
    }
    if (rank < kk) perm[rank] = j;
  }
  gsync<W>();

  // ---- back-transform of the kept columns only: z <- H_0 ... H_{n-3} z ----------------------------
  for (int r = t; r < kk; r += GT) {
    const int col = perm[r];
    for (int j = n - 3; j >= 0; --j) {
      const double tau = taus[j];
      if (tau == 0.0) continue;
      double s = Z[(size_t)(j + 1) * ZS + col];
      for (int i = j + 2; i < n; ++i) s = fma(Ap[tri(i, j)], Z[(size_t)i * ZS + col], s);
      s *= tau;
      Z[(size_t)(j + 1) * ZS + col] -= s;
      for (int i = j + 2; i < n; ++i) Z[(size_t)i * ZS + col] -= s * Ap[tri(i, j)];
    }
  }
  gsync<W>();

  // ---- fp32 outputs, zero padded ----------------------------------------------------------------
  for (int r = t; r < K; r += GT) P.D[(int64_t)b * K + r] = (r < kk) ? __double2float_rn(d0[perm[r]]) : 0.f;
  if (SPARSE) {
    float* Vb = P.V + (int64_t)P.node_ptr[b] * K;
    for (int i = t; i < n * K; i += GT) {
      const int row = i / K, r = i - row * K;
      Vb[i] = (r < kk) ? __double2float_rn(Z[(size_t)row * ZS + perm[r]]) : 0.f;
    }
  } else {
    float* Vb = P.V + (int64_t)b * N * K;
    for (int i = t; i < N * K; i += GT) {
      const int row = i / K, r = i - row * K;
      Vb[i] = (row < n && r < kk) ? __double2float_rn(Z[(size_t)row * ZS + perm[r]]) : 0.f;
    }
  }
  if (t == 0) P.status[b] = fail;
}

template <bool SPARSE>
int launch(lnb_stream_t stream, const EigParams& p, const char* what) {
  cudaStream_t s = (cudaStream_t)stream;
  if (p.N <= 32) {
    const size_t shm = 4 * graph_doubles(p.N, 1) * sizeof(double);
    if (shm > 48 * 1024)
      cudaFuncSetAttribute(graph_eigs_kernel<1, SPARSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
    graph_eigs_kernel<1, SPARSE><<<lnb::ceil_div(p.B, 4), GE_THREADS, shm, s>>>(p);
  } else {
    const size_t shm = graph_doubles(p.N, 4) * sizeof(double);
    if (shm > 48 * 1024)
      cudaFuncSetAttribute(graph_eigs_kernel<4, SPARSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
    graph_eigs_kernel<4, SPARSE><<<p.B, GE_THREADS, shm, s>>>(p);
  }
  lnb::count_launch();
  return lnb::finish_launch(what);
}

static_assert(sizeof(double) * graph_doubles(GE_NMAX, 4) <= 227 * 1024,
              "graph_eigs: N = 128 must fit one CTA's shared memory");
static_assert(4 * sizeof(double) * graph_doubles(32, 1) <= 227 * 1024, "graph_eigs: four N = 32 graphs per CTA");

}  // namespace

extern "C" {

int lnb_graph_eigs_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* node_ptr,
                          const int32_t* edge_ptr, const uint8_t* edges, const double* inv_sqrt_deg, int B,
                          int N, int E, int K, float* D, float* V_rows, int32_t* status) {
  if (!(B >= 0 && N >= 1 && N <= GE_NMAX && K >= 1 && K <= GE_KMAX && E >= 1 && E <= GE_EMAX)) {
    lnb::set_err("graph_eigs_sparse: B=%d N=%d E=%d K=%d outside 1 <= N <= %d, 1 <= K <= %d, 1 <= E <= %d",
                 B, N, E, K, GE_NMAX, GE_KMAX, GE_EMAX);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  // edges may be NULL when the batch has no bonds: the kernel reads [edge_ptr[b], edge_ptr[b+1]) only
  LNB_REQUIRE(sizes && node_ptr && edge_ptr && inv_sqrt_deg && D && V_rows && status,
              "graph_eigs_sparse: null pointer");
  EigParams p = {};
  p.node_ptr = node_ptr; p.edge_ptr = edge_ptr; p.edges = edges; p.inv_sqrt_deg = inv_sqrt_deg; p.E = E;
  p.sizes = sizes; p.B = B; p.N = N; p.K = K; p.D = D; p.V = V_rows; p.status = status;
  return launch<true>(stream, p, "graph_eigs_sparse");
}

int lnb_sym_eigs(lnb_stream_t stream, const float* A, int64_t elem_stride, const int32_t* sizes, int B, int N,
                 int K, float* D, float* V, int32_t* status) {
  if (!(B >= 0 && N >= 1 && N <= GE_NMAX && K >= 1 && K <= GE_KMAX && elem_stride >= 1)) {
    lnb::set_err("sym_eigs: B=%d N=%d K=%d stride=%lld outside 1 <= N <= %d, 1 <= K <= %d", B, N, K,
                 (long long)elem_stride, GE_NMAX, GE_KMAX);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  LNB_REQUIRE(A && sizes && D && V && status, "sym_eigs: null pointer");
  EigParams p = {};
  p.A = A; p.es = elem_stride; p.sizes = sizes; p.B = B; p.N = N; p.K = K; p.D = D; p.V = V; p.status = status;
  return launch<false>(stream, p, "sym_eigs");
}

}  // extern "C"
