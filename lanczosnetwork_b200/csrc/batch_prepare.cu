// GPU-side batch construction (SURVEY 8f2): from per-molecule SPARSE records -- node ids, bond list
// (u, v, bond type), Ritz pairs of the real nodes -- straight to what the convolution kernels
// consume.  Replaces, on the device, the reference's host pipeline
//   utils/data_helper.py:92-116,155-156   L4 = D^-1/2 (A + I) D^-1/2 per bond channel + simple graph
//   dataset/qm8.py:57-90,220-291          zero padding / stacking of node_feat, node_mask, L, (D, V)
// and lnb_graph_prepare's pass over the dense operators: the dense [B,N,N,E+1] tensor (21.8 MB per
// 1024 QM8 molecules, ~4 % non-zero) is never built unless the caller asks for it, and never crosses
// PCIe.
//
// Bit-exactness: the reference normalises in fp64 -- scale = deg^-1/2, value = (scale_i * m_ij) *
// scale_j -- and casts to fp32 at collate (dataset/qm8.py:262).  Degrees are integers, so the host
// passes an fp64 table of numpy's deg^-1/2 covering every degree of the envelope (LNB_INV_SQRT_DEG_LEN);
// the kernel forms the same two fp64 products in the same order and rounds once (__double2float_rn):
// identical bits by construction.
// Masks, ids, ELL indices and extents are integer logic.
#include "common.cuh"

namespace {

constexpr int BP_THREADS = 256;
constexpr int BP_NW = LNB_MAX_N / 32;   // 32-bit adjacency words per row

struct SparseBatchParams {
  const int32_t* sizes;        // [B] real nodes per graph
  const int32_t* node_ptr;     // [B+1] prefix sums of sizes (rows of V_rows)
  const int32_t* node_feat;    // [node_ptr[B]] atom ids of the real nodes
  const int32_t* edge_ptr;     // [B+1]
  const uint8_t* edges;        // [edge_ptr[B]][4] = {u, v, bond type, 0}, undirected, listed once
  const float* V_rows;         // [node_ptr[B], K] Ritz vectors, rows of real nodes only
  const double* inv_sqrt_deg;  // [LNB_INV_SQRT_DEG_LEN] deg^-1/2 in fp64 (entry 0 = 0)
  const uint8_t* blob;         // packed batch (lnb_graph_prepare_sparse_packed / _features_packed): the pointers
                               // above, and node_x, are derived from its header on the device, so ONE H2D copy
                               // ships a whole batch
  int B, N, E1, K, flags;
  float* ell_val; uint8_t* ell_idx; int32_t* ell_max; int32_t* gext;
  int64_t* node_ids; uint8_t* mask; float* V;     // padded [B,N], [B,N], [B,N,K]
  float* L;                                        // optional dense [B,N,N,E1]
  int32_t* rowmap; int32_t* nrows;                 // written here when the packed batch carries krow_ptr
  // feature variant (lnb_graph_prepare_sparse_features): float rows instead of atom ids
  const float* node_x;                             // [node_ptr[B], F] features of the real nodes
  float* X;                                        // padded [B,N,F]
  int F;
};

// multiplicity of entry (i, j) of channel ch (0 = simple graph = sum over bond types)
__device__ __forceinline__ int entry_mult(const uint32_t* rowmask, int E, int ch, int i, int j) {
  const int w = j >> 5;
  const uint32_t bit = 1u << (j & 31);
  int m = (i == j) ? 1 : 0;                        // the + I of L4
  if (ch == 0) {
    for (int c = 0; c < E; ++c) m += (rowmask[(c * LNB_MAX_N + i) * BP_NW + w] & bit) ? 1 : 0;
  } else {
    m += (rowmask[((ch - 1) * LNB_MAX_N + i) * BP_NW + w] & bit) ? 1 : 0;
  }
  return m;
}

// Graph b's padded feature rows X[b] [N,F]: the real rows copied bit for bit, the padded rows zero.
// 16-byte copies when F and both pointers allow (every row then starts 16-byte aligned), else scalar.
__device__ __forceinline__ void copy_feature_rows(const float* __restrict__ src, float* __restrict__ dst,
                                                  int nb, int N, int F, int tid) {
  const int real = nb * F, total = N * F;
  if ((F & 3) == 0 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int i = tid; i < total / 4; i += BP_THREADS)
      d4[i] = i < real / 4 ? __ldg(s4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
    for (int i = tid; i < total; i += BP_THREADS) dst[i] = i < real ? __ldg(src + i) : 0.f;
  }
}

// kFeat = false: atom ids -> node_ids (lnb_graph_prepare_sparse / _packed); kFeat = true: float feature rows
// -> X (lnb_graph_prepare_sparse_features / _features_packed).  Everything else is the same code.
template <bool kFeat>
__global__ void __launch_bounds__(BP_THREADS)
batch_prepare_sparse_kernel(const SparseBatchParams P) {
  extern __shared__ __align__(16) unsigned char bp_smem[];
  __shared__ int s_max[LNB_MAX_E1];
  __shared__ int s_ke;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int N = P.N, E1 = P.E1, E = E1 - 1, K = P.K;
  const int32_t* sizes = P.sizes; const int32_t* node_ptr = P.node_ptr; const int32_t* node_feat = P.node_feat;
  const int32_t* edge_ptr = P.edge_ptr; const uint8_t* edges = P.edges; const float* V_rows = P.V_rows;
  bool other_width = false;                      // a feature batch of another F: read as empty graphs
  if (P.blob) {                                  // header: byte offsets of the segments (see the C header)
    const int32_t* header = reinterpret_cast<const int32_t*>(P.blob);
    sizes = reinterpret_cast<const int32_t*>(P.blob + header[LNB_PACK_HDR_SIZES]);
    node_ptr = reinterpret_cast<const int32_t*>(P.blob + header[LNB_PACK_HDR_NODE_PTR]);
    edge_ptr = reinterpret_cast<const int32_t*>(P.blob + header[LNB_PACK_HDR_EDGE_PTR]);
    if (kFeat) other_width = header[LNB_PACK_HDR_F] != P.F;   // node_x is derived where it is read
    else node_feat = reinterpret_cast<const int32_t*>(P.blob + header[LNB_PACK_HDR_NODE_FEAT]);
    V_rows = reinterpret_cast<const float*>(P.blob + header[LNB_PACK_HDR_V_ROWS]);
    edges = P.blob + header[LNB_PACK_HDR_EDGES];
    if ((P.flags & LNB_PACKED_HOST_TILES) && header[LNB_PACK_HDR_KROW] > 0 && P.rowmap) {
      // compact Ritz row list {b*K + k : k < k_eff(b)} from the host's prefix sums (the host also ships
      // the tile table, so no tile-assignment launch follows)
      const int32_t* krow = reinterpret_cast<const int32_t*>(P.blob + header[LNB_PACK_HDR_KROW]);
      const int k0 = krow[b], k1 = krow[b + 1];
      for (int i = threadIdx.x; i < k1 - k0; i += BP_THREADS) P.rowmap[k0 + i] = b * P.K + i;
      if (b == 0 && threadIdx.x == 0) P.nrows[0] = krow[P.B];
    }
  }
  const int nb = other_width ? 0 : min(max(sizes[b], 0), N);
  uint32_t* rowmask = reinterpret_cast<uint32_t*>(bp_smem);              // [E][NMAX][NW]
  double* scale = reinterpret_cast<double*>(rowmask + (size_t)E * LNB_MAX_N * BP_NW);   // [E1][NMAX]
  uint8_t* cnt_s = reinterpret_cast<uint8_t*>(scale + (size_t)E1 * LNB_MAX_N);          // [N*E1]

  for (int i = tid; i < E * LNB_MAX_N * BP_NW; i += BP_THREADS) rowmask[i] = 0u;
  if (tid < LNB_MAX_E1) s_max[tid] = 0;
  if (tid == 0) s_ke = 0;
  __syncthreads();
  // ---- adjacency bitmaps from the bond list (idempotent: duplicates do not double count) ----------
  const int e0 = edge_ptr[b], e1 = edge_ptr[b + 1];
  for (int e = e0 + tid; e < e1; e += BP_THREADS) {
    const uchar4 ed = reinterpret_cast<const uchar4*>(edges)[e];
    const int u = ed.x, v = ed.y, c = ed.z;
    if (u < nb && v < nb && c < E) {
      atomicOr(&rowmask[(c * LNB_MAX_N + u) * BP_NW + (v >> 5)], 1u << (v & 31));
      atomicOr(&rowmask[(c * LNB_MAX_N + v) * BP_NW + (u >> 5)], 1u << (u & 31));
    }
  }
  __syncthreads();
  // ---- degrees of A + I per channel -> deg^-1/2 (fp64 table) ---------------------------------------
  for (int p = tid; p < E1 * N; p += BP_THREADS) {
    const int ch = p / N, i = p - ch * N;
    double sc = 0.0;
    if (i < nb) {
      int deg = 1;
      if (ch == 0) {
        for (int c = 0; c < E; ++c)
          for (int w = 0; w < BP_NW; ++w) deg += __popc(rowmask[(c * LNB_MAX_N + i) * BP_NW + w]);
      } else {
        for (int w = 0; w < BP_NW; ++w) deg += __popc(rowmask[((ch - 1) * LNB_MAX_N + i) * BP_NW + w]);
      }
      sc = P.inv_sqrt_deg[min(deg, LNB_INV_SQRT_DEG_LEN - 1)];
    }
    scale[ch * LNB_MAX_N + i] = sc;
  }
  __syncthreads();
  // ---- ELL rows, same order as lnb_graph_prepare: diagonal first, then ascending column ------------
  const int binarize = P.flags & 1;
  const int pairs = N * E1;
  for (int p = tid; p < pairs; p += BP_THREADS) {
    const int n = p / E1, ch = p - n * E1;
    float* val = P.ell_val + ((int64_t)(b * E1 + ch) * N) * N + n;
    uint8_t* idx = P.ell_idx + ((int64_t)(b * E1 + ch) * N) * N + n;
    int cnt = 0;
    if (n < nb) {
      const double sn = scale[ch * LNB_MAX_N + n];
      {
        const int m = entry_mult(rowmask, E, ch, n, n);
        const float v = __double2float_rn((sn * (double)m) * sn);
        if (v != 0.f) { val[0] = binarize ? 1.f : v; idx[0] = (uint8_t)n; cnt = 1; }
      }
      for (int w = 0; w < BP_NW; ++w) {
        uint32_t bits = 0u;
        if (ch == 0) { for (int c = 0; c < E; ++c) bits |= rowmask[(c * LNB_MAX_N + n) * BP_NW + w]; }
        else bits = rowmask[((ch - 1) * LNB_MAX_N + n) * BP_NW + w];
        while (bits) {
          const int j = (w << 5) + __ffs(bits) - 1;
          bits &= bits - 1;
          if (j == n) continue;
          const int m = entry_mult(rowmask, E, ch, n, j);
          const float v = __double2float_rn((sn * (double)m) * scale[ch * LNB_MAX_N + j]);
          if (v != 0.f) {
            val[(int64_t)cnt * N] = binarize ? 1.f : v;
            idx[(int64_t)cnt * N] = (uint8_t)j;
            ++cnt;
          }
        }
      }
    }
    cnt_s[p] = (uint8_t)cnt;
    if (cnt) atomicMax(&s_max[ch], cnt);
  }
  // ---- padded node ids, mask, Ritz vectors; k_eff ---------------------------------------------------
  const int r0 = node_ptr[b];
  for (int n = tid; n < N; n += BP_THREADS) {
    if (!kFeat) P.node_ids[(int64_t)b * N + n] = (n < nb) ? (int64_t)node_feat[r0 + n] : 0;
    P.mask[(int64_t)b * N + n] = (n < nb) ? 1 : 0;
  }
  if (kFeat) {
    const float* node_x = P.blob ? reinterpret_cast<const float*>(
        P.blob + reinterpret_cast<const int32_t*>(P.blob)[LNB_PACK_HDR_NODE_FEAT]) : P.node_x;
    copy_feature_rows(node_x + (int64_t)r0 * P.F, P.X + (int64_t)b * N * P.F, nb, N, P.F, tid);
  }
  int ke = 0;
  for (int i = tid; i < N * K; i += BP_THREADS) {
    const int n = i / K, k = i - n * K;
    float v = 0.f;
    if (n < nb) v = V_rows[(int64_t)(r0 + n) * K + k];
    P.V[(int64_t)b * N * K + i] = v;
    if (v != 0.f) ke = max(ke, k + 1);
  }
  if (ke) atomicMax(&s_ke, ke);
  __syncthreads();
  for (int pr = tid; pr < pairs; pr += BP_THREADS) {
    const int n = pr / E1, ch = pr - n * E1;
    float* val = P.ell_val + ((int64_t)(b * E1 + ch) * N) * N + n;
    uint8_t* idx = P.ell_idx + ((int64_t)(b * E1 + ch) * N) * N + n;
    for (int t = cnt_s[pr]; t < s_max[ch]; ++t) {
      val[(int64_t)t * N] = 0.f;
      idx[(int64_t)t * N] = 0;
    }
  }
  if (tid < E1) P.ell_max[b * E1 + tid] = s_max[tid];
  if (tid == 0) { P.gext[b * 2] = nb; P.gext[b * 2 + 1] = s_ke; }
  // ---- optional dense operators [N,N,E1] exactly as the reference's collate pads them -------------
  if (P.L) {
    float* Lg = P.L + (int64_t)b * N * N * E1;
    const int total = N * N * E1;
    for (int i = tid; i < total; i += BP_THREADS) {
      const int ch = i % E1, ij = i / E1, r = ij / N, c = ij - r * N;
      float v = 0.f;
      if (r < nb && c < nb) {
        const int m = entry_mult(rowmask, E, ch, r, c);
        if (m) v = __double2float_rn((scale[ch * LNB_MAX_N + r] * (double)m) * scale[ch * LNB_MAX_N + c]);
      }
      Lg[i] = v;
    }
  }
}

// GAT's additive attention bias (data.gat_bias of the collated operators) from the bond lists: -0.0 on the
// diagonal (padded nodes included) and on every bond of the channel (channel 0: any bond type < E), -1e9
// elsewhere.  One CTA per graph: the fill, then the bonds overwrite their entries.
__global__ void __launch_bounds__(BP_THREADS)
gat_bias_sparse_kernel(const int32_t* __restrict__ sizes, const int32_t* __restrict__ edge_ptr,
                       const uint8_t* __restrict__ edges, int N, int E1, float* __restrict__ out) {
  const int b = blockIdx.x, tid = threadIdx.x;
  const int nb = min(max(sizes[b], 0), N);
  float* ob = out + (int64_t)b * N * N * E1;
  const int total = N * N * E1;
  for (int i = tid; i < total; i += BP_THREADS) {
    const int ij = i / E1, r = ij / N, c = ij - r * N;
    ob[i] = r == c ? -0.0f : -1e9f;
  }
  __syncthreads();
  const int e0 = edge_ptr[b], e1 = edge_ptr[b + 1];
  for (int e = e0 + tid; e < e1; e += BP_THREADS) {
    const uchar4 ed = reinterpret_cast<const uchar4*>(edges)[e];
    const int u = ed.x, v = ed.y, c = ed.z;
    if (u < nb && v < nb && c < E1 - 1) {
      ob[((int64_t)u * N + v) * E1] = -0.0f;
      ob[((int64_t)v * N + u) * E1] = -0.0f;
      ob[((int64_t)u * N + v) * E1 + c + 1] = -0.0f;
      ob[((int64_t)v * N + u) * E1 + c + 1] = -0.0f;
    }
  }
}

template <bool kFeat>
static int launch_sparse(lnb_stream_t stream, SparseBatchParams p, int32_t* tiles, int32_t* rowmap,
                         int32_t* nrows) {
  p.rowmap = rowmap; p.nrows = nrows;
  const size_t smem = (size_t)(p.E1 - 1) * LNB_MAX_N * BP_NW * 4 + (size_t)p.E1 * LNB_MAX_N * 8 +
                       (size_t)p.N * p.E1 + 16;
  cudaStream_t s = (cudaStream_t)stream;
  if (smem > 48 * 1024)
    cudaFuncSetAttribute(batch_prepare_sparse_kernel<kFeat>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  batch_prepare_sparse_kernel<kFeat><<<p.B, BP_THREADS, smem, s>>>(p);
  lnb::count_launch(1);
  if (p.blob && (p.flags & LNB_PACKED_HOST_TILES))  // tile table + row-list offsets came with the batch
    return lnb::finish_launch("graph_prepare_sparse");
  return lnb::launch_tiles_or_rowmap(s, p.flags, p.gext, p.B, p.K, tiles, rowmap, nrows,
                                     "graph_prepare_sparse");
}

}  // namespace

extern "C" {

int lnb_graph_prepare_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* node_ptr,
                             const int32_t* node_feat, const int32_t* edge_ptr, const uint8_t* edges,
                             const float* V_rows, const double* inv_sqrt_deg, int B, int N, int E1,
                             int K, int flags, float* ell_val, uint8_t* ell_idx, int32_t* ell_max,
                             int32_t* gext, int32_t* tiles, int32_t* rowmap, int32_t* nrows,
                             int64_t* node_ids, uint8_t* mask, float* V, float* L_dense) {
  LNB_REQUIRE(B >= 0 && N >= 1 && N <= LNB_MAX_N && E1 >= 2 && E1 <= LNB_MAX_E1 && K >= 1,
              "graph_prepare_sparse: bad dims B=%d N=%d E1=%d K=%d (N <= %d, 2 <= E1 <= %d)", B, N, E1,
              K, LNB_MAX_N, LNB_MAX_E1);
  if (B == 0) return LNB_OK;
  // edges may be NULL when the batch has no bonds: the kernel reads [edge_ptr[b], edge_ptr[b+1]) only
  LNB_REQUIRE(sizes && node_ptr && node_feat && edge_ptr && V_rows && inv_sqrt_deg &&
                  ell_val && ell_idx && ell_max && gext && tiles && node_ids && mask && V,
              "graph_prepare_sparse: null pointer");
  LNB_REQUIRE((rowmap == nullptr) == (nrows == nullptr), "graph_prepare_sparse: rowmap and nrows go together");
  SparseBatchParams p;
  p.sizes = sizes; p.node_ptr = node_ptr; p.node_feat = node_feat; p.edge_ptr = edge_ptr;
  p.edges = edges; p.V_rows = V_rows; p.inv_sqrt_deg = inv_sqrt_deg; p.blob = nullptr;
  p.B = B; p.N = N; p.E1 = E1; p.K = K; p.flags = flags;
  p.ell_val = ell_val; p.ell_idx = ell_idx; p.ell_max = ell_max; p.gext = gext;
  p.node_ids = node_ids; p.mask = mask; p.V = V; p.L = L_dense;
  p.node_x = nullptr; p.X = nullptr; p.F = 0;
  return launch_sparse<false>(stream, p, tiles, rowmap, nrows);
}

int lnb_graph_prepare_sparse_packed(lnb_stream_t stream, const uint8_t* blob, const double* inv_sqrt_deg,
                                    int B, int N, int E1, int K, int flags, float* ell_val,
                                    uint8_t* ell_idx, int32_t* ell_max, int32_t* gext, int32_t* tiles,
                                    int32_t* rowmap, int32_t* nrows, int64_t* node_ids, uint8_t* mask,
                                    float* V, float* L_dense) {
  LNB_REQUIRE(B >= 0 && N >= 1 && N <= LNB_MAX_N && E1 >= 2 && E1 <= LNB_MAX_E1 && K >= 1,
              "graph_prepare_sparse_packed: bad dims B=%d N=%d E1=%d K=%d", B, N, E1, K);
  if (B == 0) return LNB_OK;
  LNB_REQUIRE(blob && inv_sqrt_deg && ell_val && ell_idx && ell_max && gext &&
                  (tiles || (flags & LNB_PACKED_HOST_TILES)) && node_ids && mask && V,
              "graph_prepare_sparse_packed: null pointer");
  LNB_REQUIRE((reinterpret_cast<uintptr_t>(blob) & 15) == 0, "graph_prepare_sparse_packed: blob must be 16-byte aligned");
  LNB_REQUIRE((rowmap == nullptr) == (nrows == nullptr), "graph_prepare_sparse_packed: rowmap and nrows go together");
  SparseBatchParams p;
  p.sizes = nullptr; p.node_ptr = nullptr; p.node_feat = nullptr; p.edge_ptr = nullptr;
  p.edges = nullptr; p.V_rows = nullptr; p.inv_sqrt_deg = inv_sqrt_deg; p.blob = blob;
  p.B = B; p.N = N; p.E1 = E1; p.K = K; p.flags = flags;
  p.ell_val = ell_val; p.ell_idx = ell_idx; p.ell_max = ell_max; p.gext = gext;
  p.node_ids = node_ids; p.mask = mask; p.V = V; p.L = L_dense;
  p.node_x = nullptr; p.X = nullptr; p.F = 0;
  return launch_sparse<false>(stream, p, tiles, rowmap, nrows);
}

int lnb_graph_prepare_sparse_features(lnb_stream_t stream, const int32_t* sizes, const int32_t* node_ptr,
                                      const float* node_x, const int32_t* edge_ptr, const uint8_t* edges,
                                      const float* V_rows, const double* inv_sqrt_deg, int B, int N, int E1,
                                      int K, int F, int flags, float* ell_val, uint8_t* ell_idx,
                                      int32_t* ell_max, int32_t* gext, int32_t* tiles, int32_t* rowmap,
                                      int32_t* nrows, float* X, uint8_t* mask, float* V, float* L_dense) {
  if (!(B >= 0 && N >= 1 && N <= LNB_MAX_N && E1 >= 2 && E1 <= LNB_MAX_E1 && K >= 1 && F >= 1 &&
        F <= LNB_PREPARE_MAX_F)) {
    lnb::set_err("graph_prepare_sparse_features: B=%d N=%d E1=%d K=%d F=%d outside 1 <= N <= %d, "
                 "2 <= E1 <= %d, K >= 1, 1 <= F <= 4096", B, N, E1, K, F, LNB_MAX_N, LNB_MAX_E1);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  // edges may be NULL when the batch has no bonds, as in lnb_graph_prepare_sparse
  LNB_REQUIRE(sizes && node_ptr && node_x && edge_ptr && V_rows && inv_sqrt_deg && ell_val &&
                  ell_idx && ell_max && gext && tiles && X && mask && V,
              "graph_prepare_sparse_features: null pointer");
  LNB_REQUIRE((rowmap == nullptr) == (nrows == nullptr),
              "graph_prepare_sparse_features: rowmap and nrows go together");
  SparseBatchParams p;
  p.sizes = sizes; p.node_ptr = node_ptr; p.node_feat = nullptr; p.edge_ptr = edge_ptr;
  p.edges = edges; p.V_rows = V_rows; p.inv_sqrt_deg = inv_sqrt_deg; p.blob = nullptr;
  p.B = B; p.N = N; p.E1 = E1; p.K = K; p.flags = flags & ~LNB_PACKED_HOST_TILES;
  p.ell_val = ell_val; p.ell_idx = ell_idx; p.ell_max = ell_max; p.gext = gext;
  p.node_ids = nullptr; p.mask = mask; p.V = V; p.L = L_dense;
  p.node_x = node_x; p.X = X; p.F = F;
  return launch_sparse<true>(stream, p, tiles, rowmap, nrows);
}

int lnb_graph_prepare_sparse_features_packed(lnb_stream_t stream, const uint8_t* blob, const double* inv_sqrt_deg,
                                             int B, int N, int E1, int K, int F, int flags, float* ell_val,
                                             uint8_t* ell_idx, int32_t* ell_max, int32_t* gext, int32_t* tiles,
                                             int32_t* rowmap, int32_t* nrows, float* X, uint8_t* mask, float* V,
                                             float* L_dense) {
  if (!(B >= 0 && N >= 1 && N <= LNB_MAX_N && E1 >= 2 && E1 <= LNB_MAX_E1 && K >= 1 && F >= 1 &&
        F <= LNB_PREPARE_MAX_F)) {
    lnb::set_err("graph_prepare_sparse_features_packed: B=%d N=%d E1=%d K=%d F=%d outside 1 <= N <= %d, "
                 "2 <= E1 <= %d, K >= 1, 1 <= F <= %d", B, N, E1, K, F, LNB_MAX_N, LNB_MAX_E1, LNB_PREPARE_MAX_F);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  LNB_REQUIRE(blob && inv_sqrt_deg && ell_val && ell_idx && ell_max && gext &&
                  (tiles || (flags & LNB_PACKED_HOST_TILES)) && X && mask && V,
              "graph_prepare_sparse_features_packed: null pointer");
  LNB_REQUIRE((reinterpret_cast<uintptr_t>(blob) & 15) == 0,
              "graph_prepare_sparse_features_packed: blob must be 16-byte aligned");
  LNB_REQUIRE((rowmap == nullptr) == (nrows == nullptr),
              "graph_prepare_sparse_features_packed: rowmap and nrows go together");
  SparseBatchParams p;
  p.sizes = nullptr; p.node_ptr = nullptr; p.node_feat = nullptr; p.edge_ptr = nullptr;
  p.edges = nullptr; p.V_rows = nullptr; p.inv_sqrt_deg = inv_sqrt_deg; p.blob = blob;
  p.B = B; p.N = N; p.E1 = E1; p.K = K; p.flags = flags;
  p.ell_val = ell_val; p.ell_idx = ell_idx; p.ell_max = ell_max; p.gext = gext;
  p.node_ids = nullptr; p.mask = mask; p.V = V; p.L = L_dense;
  p.node_x = nullptr; p.X = X; p.F = F;
  return launch_sparse<true>(stream, p, tiles, rowmap, nrows);
}

int lnb_gat_bias_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* edge_ptr, const uint8_t* edges,
                        int B, int N, int E1, float* bias) {
  if (!(B >= 0 && N >= 1 && N <= LNB_MAX_N && E1 >= 2 && E1 <= LNB_MAX_E1)) {
    lnb::set_err("gat_bias_sparse: B=%d N=%d E1=%d outside 1 <= N <= %d, 2 <= E1 <= %d", B, N, E1, LNB_MAX_N,
                 LNB_MAX_E1);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  // edges may be NULL when the batch has no bonds: the kernel reads [edge_ptr[b], edge_ptr[b+1]) only
  LNB_REQUIRE(sizes && edge_ptr && bias, "gat_bias_sparse: null pointer");
  gat_bias_sparse_kernel<<<B, BP_THREADS, 0, (cudaStream_t)stream>>>(sizes, edge_ptr, edges, N, E1, bias);
  lnb::count_launch();
  return lnb::finish_launch("gat_bias_sparse");
}

}  // extern "C"
