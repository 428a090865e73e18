// GPNN's graph partition on the device: the reference collate's spectral_clustering (P eigenvectors of
// largest |lambda| of the padded simple-graph L4, then scikit-learn's KMeans with random_state = seed)
// and get_L_cluster_cut (utils/spectral_graph_partition.py:10-50, called per graph from
// dataset/qm8.py:123-136), one graph per warp (N <= 32, four graphs per CTA) or per CTA (N > 32).
//
//   1. operator: the fp64 L4 s_i s_j of channel 0's off-diagonal non-zero pattern (s = deg^-1/2 from
//      the host's table, deg = 1 + row count); a node with a zero diagonal is padding and keeps a zero
//      row.  When the fp32 rounding of that matrix is not channel 0 bit for bit (a weighted operator),
//      the widened fp32 values are decomposed instead and status bit 3 is set;
//   2. the eigensolver of graph_eigs.cuh on the whole padded N x N, back-transforming the first P
//      columns of the reference's order; bit 1 when |lambda_P| and |lambda_P+1| are within 1e-9;
//   3. k-means in fp64 by the graph's first warp, with scikit-learn >= 1.4's defaults: centring, the
//      k-means++ seeding with 2 + floor(ln P) local trials fed by the host's RandomState draws, Lloyd
//      with the strict-convergence / centre-shift tolerance test, up to 300 iterations (bit 2 when
//      they run out), empty clusters relocated to the farthest points;
//   4. canonical labels (no edge: -1, the rest numbered by first appearance) and L_cluster / L_cut,
//      fp32 of the fp64 L4 of the within-cluster and the cut adjacency (every node keeps its self-loop).
// Every reduction has a fixed order: repeated launches are bit-identical.
//
// The sparse entry (lnb_spectral_partition_sparse) differs in step 1 only: it reads the bond lists of
// lnb_graph_prepare_sparse and forms the fp64 L4 with graph_eigs_sparse's products, (s_i m_ij) s_j with m
// the bond multiplicity, so padded rows are zero exactly as the dense entry sees them.  The bond pattern
// stays in a bitmap behind the k-means scratch for step 4, which may write L_cluster / L_cut and writes
// their ELL rows in lnb_graph_prepare's layout and slot order (diagonal, then ascending column).
#include "graph_eigs.cuh"

namespace {

using namespace eigs;

constexpr int SP_ITERS = 300;                 // KMeans' max_iter
constexpr double SP_TIE = 1e-9;

struct PartParams {
  const float* L; int64_t es;                 // channel 0: L[((b * N + i) * N + j) * es]
  // sparse entry: the records of lnb_graph_prepare_sparse, bond types < E
  const int32_t* sizes; const int32_t* edge_ptr; const uint8_t* edges; int E;
  const double* inv_sqrt_deg;                 // [LNB_INV_SQRT_DEG_LEN]
  const double* draws;                        // [1 + (P - 1) * T]
  int B, N, P, T;
  int32_t* labels; float* L_cluster; float* L_cut; int32_t* status;   // L_cluster / L_cut may be null
  float* ell_val; uint8_t* ell_idx; int32_t* ell_max; int32_t* gext;  // ELL rows of [L_cluster, L_cut]
};

// k-means scratch behind the eigensolver's: C, Cn [P][P], cn2, wic [P], dist, xx [N], misc [8],
// then the ints lab, lab_old, linked [N]
__host__ __device__ constexpr size_t km_doubles(int N, int P) {
  return 2 * (size_t)P * P + 2 * (size_t)P + 2 * (size_t)N + 8 + (3 * (size_t)N + 1) / 2;
}

// the sparse entry's bond pattern: N rows of ceil(N / 32) words
__host__ __device__ constexpr size_t adj_doubles(int N) {
  return ((size_t)N * ((N + 31) / 32) + 1) / 2;
}

__host__ __device__ constexpr size_t part_doubles(int N, int W, int P, bool sparse = false) {
  return graph_doubles(N, W) + km_doubles(N, P) + (sparse ? adj_doubles(N) : 0);
}

template <int W>
__device__ __forceinline__ int group_any(int v) {
  if (W == 1) return __any_sync(0xffffffffu, v);
  return __syncthreads_or(v);
}

template <int W>
__device__ __forceinline__ int group_max(int v, int* red) {
  v = __reduce_max_sync(0xffffffffu, v);
  if (W == 1) return v;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int m = red[0];
#pragma unroll
  for (int w = 1; w < W; ++w) m = max(m, red[w]);
  return m;
}

struct Kmeans {
  const Work& w;
  const int N, P, lane;
  double *C, *Cn, *cn2, *wic, *dist, *xx, *misc;
  int *lab, *lab_old;

  __device__ __forceinline__ double X(int i, int k) const { return w.Z()[(size_t)i * w.ZS + w.perm()[k]]; }
  __device__ __forceinline__ double& Xr(int i, int k) const { return w.Z()[(size_t)i * w.ZS + w.perm()[k]]; }

  // _euclidean_distances(X[c], X, squared=True): max((-2 x_c.x_i + |x_c|^2) + |x_i|^2, 0)
  __device__ __forceinline__ double dist_pt(int c, int i) const {
    double d = 0.0;
    for (int k = 0; k < P; ++k) d = fma(X(c, k), X(i, k), d);
    return fmax(__dadd_rn(__dadd_rn(-2.0 * d, xx[c]), xx[i]), 0.0);
  }

  // argmin_j |c_j|^2 - 2 x_i.c_j (first minimum), sklearn's _update_chunk_dense
  __device__ __forceinline__ int nearest(int i) const {
    int best = 0;
    double bd = 0.0;
    for (int j = 0; j < P; ++j) {
      double d = 0.0;
      for (int k = 0; k < P; ++k) d = fma(X(i, k), C[j * P + k], d);
      const double pd = fma(-2.0, d, cn2[j]);
      if (j == 0 || pd < bd) { bd = pd; best = j; }
    }
    return best;
  }

  __device__ __forceinline__ void centre_norms() const {
    if (lane < P) {
      double s = 0.0;
      for (int k = 0; k < P; ++k) s = fma(C[lane * P + k], C[lane * P + k], s);
      cn2[lane] = s;
    }
    __syncwarp();
  }

  // returns status bit 2 when the iterations ran out
  __device__ int run(const double* draws, int T) {
    // centring, tolerance mean(var(X, 0)) * 1e-4, row norms
    if (lane < P) {
      double s = 0.0;
      for (int i = 0; i < N; ++i) s += X(i, lane);
      cn2[lane] = s / (double)N;
    }
    __syncwarp();
    for (int i = lane; i < N; i += 32)
      for (int k = 0; k < P; ++k) Xr(i, k) -= cn2[k];
    __syncwarp();
    if (lane < P) {
      double s = 0.0;
      for (int i = 0; i < N; ++i) s += X(i, lane);
      const double m = s / (double)N;
      double v = 0.0;
      for (int i = 0; i < N; ++i) { const double d = X(i, lane) - m; v += d * d; }
      wic[lane] = v / (double)N;
    }
    for (int i = lane; i < N; i += 32) {
      double s = 0.0;
      for (int k = 0; k < P; ++k) s = fma(X(i, k), X(i, k), s);
      xx[i] = s;
    }
    __syncwarp();
    double tol = 0.0;
    for (int k = 0; k < P; ++k) tol += wic[k];
    tol = tol / (double)P * 1e-4;

    // ---- k-means++ ----------------------------------------------------------------------------
    int* ids = reinterpret_cast<int*>(misc);
    const int c0 = min(max((int)draws[0], 0), N - 1);
    if (lane < P) C[lane] = X(c0, lane);
    double pot = 0.0;
    for (int i = lane; i < N; i += 32) { dist[i] = dist_pt(c0, i); pot += dist[i]; }
    pot = warp_sum_d(pot);
    __syncwarp();
    for (int c = 1; c < P; ++c) {
      if (lane == 0) {
        // searchsorted(cumsum(dist), u * pot), clipped to N - 1
        double rv[4];
        for (int r = 0; r < T; ++r) { rv[r] = draws[1 + (c - 1) * T + r] * pot; ids[r] = N - 1; }
        int open = (1 << T) - 1;
        double acc = 0.0;
        for (int i = 0; i < N && open; ++i) {
          acc += dist[i];
          for (int r = 0; r < T; ++r)
            if ((open >> r & 1) && acc >= rv[r]) { ids[r] = i; open &= ~(1 << r); }
        }
      }
      __syncwarp();
      int best = 0;
      double bpot = 0.0;
      for (int r = 0; r < T; ++r) {
        const int cand = ids[r];
        double s = 0.0;
        for (int i = lane; i < N; i += 32) s += fmin(dist[i], dist_pt(cand, i));
        s = warp_sum_d(s);
        if (r == 0 || s < bpot) { bpot = s; best = r; }
      }
      const int cand = ids[best];
      pot = bpot;
      for (int i = lane; i < N; i += 32) dist[i] = fmin(dist[i], dist_pt(cand, i));
      if (lane < P) C[c * P + lane] = X(cand, lane);
      __syncwarp();
    }

    // ---- Lloyd --------------------------------------------------------------------------------
    for (int i = lane; i < N; i += 32) lab_old[i] = -1;
    bool strict = false;
    int it = 0;
    for (; it < SP_ITERS; ++it) {
      centre_norms();
      for (int j = lane; j < P * P; j += 32) Cn[j] = 0.0;
      if (lane < P) wic[lane] = 0.0;
      for (int i = lane; i < N; i += 32) lab[i] = nearest(i);
      __syncwarp();
      if (lane < P) {                        // sums in point order, one lane per feature
        for (int i = 0; i < N; ++i) Cn[lab[i] * P + lane] += X(i, lane);
      } else if (lane == 31) {
        for (int i = 0; i < N; ++i) wic[lab[i]] += 1.0;
      }
      __syncwarp();
      if (lane == 0) relocate_empty();
      __syncwarp();
      if (lane < P) {
        if (wic[lane] > 0.0) {
          const double a = 1.0 / wic[lane];
          for (int k = 0; k < P; ++k) Cn[lane * P + k] *= a;
        }
        double s = 0.0;
        for (int k = 0; k < P; ++k) { const double d = Cn[lane * P + k] - C[lane * P + k]; s += d * d; }
        dist[lane] = sqrt(s);
      }
      __syncwarp();
      double* tmp = C; C = Cn; Cn = tmp;
      bool same = true;
      for (int i = lane; i < N; i += 32) same = same && lab[i] == lab_old[i];
      if (__all_sync(0xffffffffu, same)) { strict = true; break; }
      double tot = 0.0;
      for (int j = 0; j < P; ++j) tot += dist[j] * dist[j];
      if (tot <= tol) break;
      for (int i = lane; i < N; i += 32) lab_old[i] = lab[i];
      __syncwarp();
    }
    if (!strict) {
      centre_norms();
      for (int i = lane; i < N; i += 32) lab[i] = nearest(i);
      __syncwarp();
    }
    return it == SP_ITERS ? 4 : 0;
  }

  // _relocate_empty_clusters_dense: each empty cluster (ascending) takes the next point farthest from
  // its centre (descending distance, ties by the lower index), which leaves its old cluster
  __device__ void relocate_empty() {
    int far[LNB_PARTITION_MAX_P];
    int taken = 0;
    for (int j = 0; j < P; ++j) {
      if (wic[j] != 0.0) continue;
      int pick = -1;
      double pd = -1.0;
      for (int i = 0; i < N; ++i) {
        bool used = false;
        for (int q = 0; q < taken; ++q) used = used || far[q] == i;
        if (used) continue;
        double d = 0.0;
        for (int k = 0; k < P; ++k) { const double e = X(i, k) - C[lab[i] * P + k]; d += e * e; }
        if (d > pd) { pd = d; pick = i; }
      }
      if (pick < 0) break;
      far[taken++] = pick;
      const int old = lab[pick];
      for (int k = 0; k < P; ++k) {
        Cn[old * P + k] -= X(pick, k);
        Cn[j * P + k] = X(pick, k);
      }
      wic[j] = 1.0;
      wic[old] -= 1.0;
    }
  }
};

template <int W, bool SPARSE>
__global__ void __launch_bounds__(GE_THREADS)
spectral_partition_kernel(const PartParams p) {
  extern __shared__ __align__(16) double sp_smem[];
  constexpr int GPC = 4 / W;                 // graphs per CTA
  constexpr int GT = W * 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = warp / W, wg = warp % W;
  const int t = wg * 32 + lane;              // row owned by this thread
  const int N = p.N, P = p.P;
  const int b = blockIdx.x * GPC + grp;
  double* base = sp_smem + (size_t)grp * part_doubles(N, W, P, SPARSE);
  const Work w(base, N, W, wg);
  if (b >= p.B) return;                       // whole groups only: a CTA-wide group has b < B

  double* km = base + graph_doubles(N, W);
  int* ibase = reinterpret_cast<int*>(km + 2 * (size_t)P * P + 2 * P + 2 * N + 8);
  int* lab = ibase;
  int* canon = ibase + N;                    // lab_old of the k-means, then the canonical labels
  int* linked = ibase + 2 * N;
  const int NW = (N + 31) >> 5;
  uint32_t* adj = reinterpret_cast<uint32_t*>(base + graph_doubles(N, W) + km_doubles(N, P));
  const float* Lb = SPARSE ? nullptr : p.L + (int64_t)b * N * N * p.es;
  auto at = [&](int i, int j) { return __ldg(Lb + ((int64_t)i * N + j) * p.es); };
  // an off-diagonal entry of the pattern
  auto edge = [&](int i, int j) {
    if (SPARSE) return (adj[i * NW + (j >> 5)] >> (j & 31) & 1u) != 0u;
    return j != i && at(i, j) != 0.f;
  };

  // ---- 1. the operator --------------------------------------------------------------------------
  int weighted = 0;
  if (SPARSE) {
    // graph_eigs_sparse's producer: bond-type bitmask per node pair in Z's storage (free until QL), a
    // bond listed twice with one type counts once; the pattern bitmap outlives the solver
    const int n = min(max(p.sizes[b], 0), N);
    uint32_t* mk = reinterpret_cast<uint32_t*>(w.Z());
    for (int i = t; i < n * n; i += GT) mk[i] = 0u;
    for (int i = t; i < N * NW; i += GT) adj[i] = 0u;
    gsync<W>();
    const int e0 = p.edge_ptr[b], e1 = p.edge_ptr[b + 1];
    for (int e = e0 + t; e < e1; e += GT) {
      const uchar4 ed = reinterpret_cast<const uchar4*>(p.edges)[e];
      const int u = ed.x, v = ed.y, c = ed.z;
      if (u < n && v < n && c < p.E) {
        atomicOr(&mk[u * n + v], 1u << c);
        atomicOr(&mk[v * n + u], 1u << c);
        if (u != v) {
          atomicOr(&adj[u * NW + (v >> 5)], 1u << (v & 31));
          atomicOr(&adj[v * NW + (u >> 5)], 1u << (u & 31));
        }
      }
    }
    gsync<W>();
    if (t < N) {
      int deg = 1, any = 0;                             // the + I of L4
      for (int j = 0; j < n && t < n; ++j) deg += __popc(mk[t * n + j]);
      for (int k = 0; k < NW; ++k) any |= adj[t * NW + k] != 0u;
      linked[t] = any;
      w.sc()[t] = t < n ? p.inv_sqrt_deg[min(deg, LNB_INV_SQRT_DEG_LEN - 1)] : 0.0;   // padding: a zero row
    }
    gsync<W>();
    if (t < N) {
      const double si = w.sc()[t];
      for (int j = 0; j <= t; ++j) {
        const int m = t < n ? (t == j ? 1 : 0) + __popc(mk[t * n + j]) : 0;
        w.Ap()[tri(t, j)] = m ? (si * (double)m) * w.sc()[j] : 0.0;
      }
    }
  } else {
    if (t < N) {
      int deg = 1;                                        // the + I of L4
      for (int j = 0; j < N; ++j) deg += (j != t && at(t, j) != 0.f) ? 1 : 0;
      linked[t] = deg > 1;
      w.sc()[t] = at(t, t) != 0.f ? p.inv_sqrt_deg[deg] : 0.0;   // padding: a zero row
    }
    gsync<W>();
    if (t < N) {
      const double si = w.sc()[t];
      for (int j = 0; j < N; ++j) {
        const float a = at(t, j);
        // the reference's (s_i * 1) * s_j on the pattern and the diagonal
        const double v = (j == t || a != 0.f) ? si * w.sc()[j] : 0.0;
        weighted |= __float_as_uint(__double2float_rn(v)) != __float_as_uint(a);
        if (j <= t) w.Ap()[tri(t, j)] = v;
      }
    }
    weighted = group_any<W>(weighted);
    if (weighted && t < N)
      for (int j = 0; j <= t; ++j) w.Ap()[tri(t, j)] = (double)at(t, j);
  }
  gsync<W>();

  // ---- 2. eigenvectors: the first P of the reference's order (and the P+1-th eigenvalue) ----------
  tridiagonalize<W>(w, N, t);
  const int fail = tridiag_ql<W>(w, N, t, lane);
  order_pairs<W>(w, N, P + 1, t);
  back_transform<W>(w, N, P, t);
  const int tie = fabs(fabs(w.d0()[w.perm()[P - 1]]) - fabs(w.d0()[w.perm()[P]])) < SP_TIE;

  // ---- 3. k-means on the first warp ------------------------------------------------------------
  if (wg == 0) {
    Kmeans k{w, N, P, lane, km, km + P * P, km + 2 * P * P, km + 2 * P * P + P, km + 2 * P * P + 2 * P,
             km + 2 * P * P + 2 * P + N, km + 2 * P * P + 2 * P + 2 * N, lab, canon};
    const int iters = k.run(p.draws, p.T);
    if (lane == 0) {
      int map[LNB_PARTITION_MAX_P], next = 0;
      for (int j = 0; j < P; ++j) map[j] = -1;
      for (int i = 0; i < N; ++i) {
        if (!linked[i]) { canon[i] = -1; continue; }
        if (map[lab[i]] < 0) map[lab[i]] = next++;
        canon[i] = map[lab[i]];
      }
      p.status[b] = fail | tie << 1 | iters | (weighted ? 8 : 0);
    }
  }
  gsync<W>();

  // ---- 4. outputs: labels, then the L4 of the within-cluster and of the cut adjacency --------------
  double* s_cl = w.hv();
  double* s_ct = w.hw();
  if (t < N) {
    p.labels[(int64_t)b * N + t] = canon[t];
    int dc = 1, dt = 1;
    for (int j = 0; j < N; ++j) {
      if (!edge(t, j)) continue;
      if (lab[j] == lab[t]) ++dc; else ++dt;
    }
    s_cl[t] = p.inv_sqrt_deg[dc];
    s_ct[t] = p.inv_sqrt_deg[dt];
  }
  gsync<W>();
  if (p.L_cluster) {
    float* Oc = p.L_cluster + (int64_t)b * N * N;
    float* Ot = p.L_cut + (int64_t)b * N * N;
    for (int idx = t; idx < N * N; idx += GT) {
      const int r = idx / N, c = idx - r * N;
      const bool e = edge(r, c);
      const bool same = lab[r] == lab[c];
      Oc[idx] = (r == c || (e && same)) ? __double2float_rn(s_cl[r] * s_cl[c]) : 0.f;
      Ot[idx] = (r == c || (e && !same)) ? __double2float_rn(s_ct[r] * s_ct[c]) : 0.f;
    }
  }
  if (SPARSE) {
    // lnb_graph_prepare of stack([L_cluster, L_cut], 3) with a zero Q: row t of channel ch holds the
    // diagonal, then its part's edges by ascending column, zero-filled to the channel's longest row.
    // Every row keeps its self-loop, so the graph's extent is (N, 0).
    int cnt[2] = {0, 0};
#pragma unroll
    for (int ch = 0; ch < 2; ++ch) {
      const double* sv = ch ? s_ct : s_cl;
      float* val = p.ell_val + ((int64_t)(b * 2 + ch) * N) * N + t;
      uint8_t* idx = p.ell_idx + ((int64_t)(b * 2 + ch) * N) * N + t;
      if (t < N) {
        val[0] = __double2float_rn(sv[t] * sv[t]);
        idx[0] = (uint8_t)t;
        int c = 1;
        for (int j = 0; j < N; ++j) {
          if (!edge(t, j) || (lab[j] == lab[t]) != (ch == 0)) continue;
          val[(int64_t)c * N] = __double2float_rn(sv[t] * sv[j]);
          idx[(int64_t)c * N] = (uint8_t)j;
          ++c;
        }
        cnt[ch] = c;
      }
    }
    int* red = reinterpret_cast<int*>(w.red());
    const int m0 = group_max<W>(cnt[0], red);
    const int m1 = group_max<W>(cnt[1], red + 4);
#pragma unroll
    for (int ch = 0; ch < 2; ++ch) {
      if (t >= N) break;
      float* val = p.ell_val + ((int64_t)(b * 2 + ch) * N) * N + t;
      uint8_t* idx = p.ell_idx + ((int64_t)(b * 2 + ch) * N) * N + t;
      for (int s = cnt[ch]; s < (ch ? m1 : m0); ++s) {
        val[(int64_t)s * N] = 0.f;
        idx[(int64_t)s * N] = 0;
      }
    }
    if (t == 0) {
      p.ell_max[b * 2] = m0;
      p.ell_max[b * 2 + 1] = m1;
      p.gext[b * 2] = N;
      p.gext[b * 2 + 1] = 0;
    }
  }
}

static_assert(sizeof(double) * part_doubles(LNB_MAX_N, 4, LNB_PARTITION_MAX_P, true) <= lnb::SMEM_MAX,
              "spectral_partition: N = 128, P = 16 must fit one CTA's shared memory");
static_assert(4 * sizeof(double) * part_doubles(32, 1, LNB_PARTITION_MAX_P, true) <= lnb::SMEM_MAX,
              "spectral_partition: four N = 32 graphs per CTA");

template <bool SPARSE>
int launch(lnb_stream_t stream, const PartParams& p, const char* what) {
  cudaStream_t s = (cudaStream_t)stream;
  if (p.N <= 32) {
    const size_t shm = 4 * part_doubles(p.N, 1, p.P, SPARSE) * sizeof(double);
    if (shm > 48 * 1024)
      cudaFuncSetAttribute(spectral_partition_kernel<1, SPARSE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)shm);
    spectral_partition_kernel<1, SPARSE><<<lnb::ceil_div(p.B, 4), GE_THREADS, shm, s>>>(p);
  } else {
    const size_t shm = part_doubles(p.N, 4, p.P, SPARSE) * sizeof(double);
    if (shm > 48 * 1024)
      cudaFuncSetAttribute(spectral_partition_kernel<4, SPARSE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)shm);
    spectral_partition_kernel<4, SPARSE><<<p.B, GE_THREADS, shm, s>>>(p);
  }
  lnb::count_launch();
  return lnb::finish_launch(what);
}

}  // namespace

extern "C" {

int lnb_spectral_partition_draws(int P) {
  if (P < LNB_PARTITION_MIN_P || P > LNB_PARTITION_MAX_P) return 0;
  return 1 + (P - 1) * (2 + (int)log((double)P));
}

int lnb_spectral_partition(lnb_stream_t stream, const float* L, int64_t elem_stride, int B, int N, int P,
                           const double* inv_sqrt_deg, const double* draws, int32_t* labels, float* L_cluster,
                           float* L_cut, int32_t* status) {
  if (!(B >= 0 && N >= 1 && N <= LNB_MAX_N && P >= LNB_PARTITION_MIN_P && P <= LNB_PARTITION_MAX_P && P < N &&
        elem_stride >= 1)) {
    lnb::set_err("spectral_partition: B=%d N=%d P=%d stride=%lld outside 1 <= N <= %d, %d <= P <= %d, P < N",
                 B, N, P, (long long)elem_stride, LNB_MAX_N, LNB_PARTITION_MIN_P, LNB_PARTITION_MAX_P);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  LNB_REQUIRE(L && inv_sqrt_deg && draws && labels && L_cluster && L_cut && status,
              "spectral_partition: null pointer");
  PartParams p = {};
  p.L = L; p.es = elem_stride; p.inv_sqrt_deg = inv_sqrt_deg; p.draws = draws;
  p.B = B; p.N = N; p.P = P; p.T = 2 + (int)log((double)P);
  p.labels = labels; p.L_cluster = L_cluster; p.L_cut = L_cut; p.status = status;
  return launch<false>(stream, p, "spectral_partition");
}

int lnb_spectral_partition_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* edge_ptr,
                                  const uint8_t* edges, const double* inv_sqrt_deg, int B, int N, int E, int P,
                                  const double* draws, int32_t* labels, int32_t* status, float* ell_val,
                                  uint8_t* ell_idx, int32_t* ell_max, int32_t* gext, float* L_cluster,
                                  float* L_cut) {
  if (!(B >= 0 && N >= 1 && N <= LNB_MAX_N && P >= LNB_PARTITION_MIN_P && P <= LNB_PARTITION_MAX_P && P < N &&
        E >= 1 && E <= LNB_EIGS_MAX_E)) {
    lnb::set_err("spectral_partition_sparse: B=%d N=%d E=%d P=%d outside 1 <= N <= %d, %d <= P <= %d, P < N, "
                 "1 <= E <= 32", B, N, E, P, LNB_MAX_N, LNB_PARTITION_MIN_P, LNB_PARTITION_MAX_P);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  // edges may be NULL when the batch has no bonds: the kernel reads [edge_ptr[b], edge_ptr[b+1]) only
  LNB_REQUIRE(sizes && edge_ptr && inv_sqrt_deg && draws && labels && status && ell_val && ell_idx && ell_max &&
                  gext && (L_cluster == nullptr) == (L_cut == nullptr),
              "spectral_partition_sparse: null pointer");
  PartParams p = {};
  p.sizes = sizes; p.edge_ptr = edge_ptr; p.edges = edges; p.E = E;
  p.inv_sqrt_deg = inv_sqrt_deg; p.draws = draws;
  p.B = B; p.N = N; p.P = P; p.T = 2 + (int)log((double)P);
  p.labels = labels; p.L_cluster = L_cluster; p.L_cut = L_cut; p.status = status;
  p.ell_val = ell_val; p.ell_idx = ell_idx; p.ell_max = ell_max; p.gext = gext;
  return launch<true>(stream, p, "spectral_partition_sparse");
}

}  // extern "C"
