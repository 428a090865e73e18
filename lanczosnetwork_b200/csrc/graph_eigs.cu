// Exact eigenpairs of one small symmetric operator per graph, in fp64: the reference's offline
// preprocessing (utils/data_helper.py:169-226 dense eigh branch, called from
// dataset/get_qm8_data.py:63-83 and truncated / zero padded to K at collate, dataset/qm8.py:265-291)
// on the device.  The solver's stages (Householder, QL, the reference's order, the back-transform of the
// first min(n, K) columns) are the device routines of graph_eigs.cuh; this file builds the operator and
// rounds the kept pairs to fp32 on the way out.
//
// Work unit: one warp per graph for N <= 32 (four graphs per CTA), one 128-thread CTA per graph
// above; a thread owns one row of A and of Z.  Every reduction has a fixed order: repeated launches
// are bit-identical.  Eigenvectors are determined up to sign (and up to a rotation inside a repeated
// eigenvalue's eigenspace), which no consumer sees: they read V diag(g(D)) V^T.
#include "graph_eigs.cuh"

namespace {

using namespace eigs;

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

  const Work w(ge_smem + (size_t)grp * graph_doubles(N, W), N, W, wg);
  double* Ap = w.Ap();
  double* Z = w.Z();
  double* sc = w.sc();
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
      sc[t] = P.inv_sqrt_deg[min(deg, LNB_INV_SQRT_DEG_LEN - 1)];
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

  tridiagonalize<W>(w, n, t);
  const int fail = tridiag_ql<W>(w, n, t, lane);
  const int kk = min(n, K);
  order_pairs<W>(w, n, kk, t);
  back_transform<W>(w, n, kk, t);
  const double* d0 = w.d0();
  const int* perm = w.perm();

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

static_assert(sizeof(double) * graph_doubles(LNB_MAX_N, 4) <= lnb::SMEM_MAX,
              "graph_eigs: N = 128 must fit one CTA's shared memory");
static_assert(4 * sizeof(double) * graph_doubles(32, 1) <= lnb::SMEM_MAX, "graph_eigs: four N = 32 graphs per CTA");

}  // namespace

extern "C" {

int lnb_graph_eigs_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* node_ptr,
                          const int32_t* edge_ptr, const uint8_t* edges, const double* inv_sqrt_deg, int B,
                          int N, int E, int K, float* D, float* V_rows, int32_t* status) {
  if (!(B >= 0 && N >= 1 && N <= LNB_MAX_N && K >= 1 && K <= LNB_EIGS_MAX_K && E >= 1 && E <= LNB_EIGS_MAX_E)) {
    lnb::set_err("graph_eigs_sparse: B=%d N=%d E=%d K=%d outside 1 <= N <= %d, 1 <= K <= %d, 1 <= E <= %d",
                 B, N, E, K, LNB_MAX_N, LNB_EIGS_MAX_K, LNB_EIGS_MAX_E);
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
  if (!(B >= 0 && N >= 1 && N <= LNB_MAX_N && K >= 1 && K <= LNB_EIGS_MAX_K && elem_stride >= 1)) {
    lnb::set_err("sym_eigs: B=%d N=%d K=%d stride=%lld outside 1 <= N <= %d, 1 <= K <= %d", B, N, K,
                 (long long)elem_stride, LNB_MAX_N, LNB_EIGS_MAX_K);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  LNB_REQUIRE(A && sizes && D && V && status, "sym_eigs: null pointer");
  EigParams p = {};
  p.A = A; p.es = elem_stride; p.sizes = sizes; p.B = B; p.N = N; p.K = K; p.D = D; p.V = V; p.status = status;
  return launch<false>(stream, p, "sym_eigs");
}

}  // extern "C"
