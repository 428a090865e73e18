// A packed batch (data.pack_sparse / data.PackedMolecules) split back into the bond-list records of
// data.sparse_collate, on the device, in one launch (lnb_records_unpack).  The records producers
// (lnb_graph_prepare_sparse, lnb_gat_bias_sparse, lnb_spectral_partition_sparse, lnb_sage_sample_sparse,
// lnb_graph_eigs_sparse) then run unchanged behind it, so every drop-in with a records entry takes the
// one-H2D-copy format at the cost of one D2D copy of the blob's bytes.  lnb_records_unpack_labels also
// copies the label segment [B, P] of a training batch (the same launch, an eighth segment);
// lnb_records_unpack_features reads a batch of float feature rows, whose node segment is 4 F bytes per node.
//
// The segment offsets change from batch to batch, so they are read here, on the device: one captured
// graph serves every batch of a (B, N, K) whose rows fit the capacities.  Every block validates the
// header on its own (a handful of loads) and reaches the same verdict, so no block copies anything from
// a batch another block refuses.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int RU_THREADS = 256;
constexpr int RU_SEGS = 8;          // sizes, node_ptr, edge_ptr, node_feat (ids or rows), edges, D, V_rows, label

struct UnpackParams {
  const uint8_t* blob;
  int64_t blob_bytes;
  int B, K;
  int64_t cap_rows, cap_edges;
  int F;                               // width of the node rows: 0 = atom ids, F > 0 = float feature rows
  int32_t* sizes; int32_t* node_ptr; uint8_t* node_feat; int32_t* edge_ptr; uint8_t* edges;
  float* D; float* V_rows;
  int P; float* label;                 // label [B, P] of lnb_records_unpack_labels, else 0 / NULL
  int32_t* status;
};

// [off, off + bytes) inside the body [LNB_PACK_HDR_BYTES, total) of the blob, 16-byte aligned
__device__ __forceinline__ bool seg_ok(int64_t off, int64_t bytes, int64_t total) {
  return off >= LNB_PACK_HDR_BYTES && (off & 15) == 0 && bytes >= 0 && off + bytes <= total;
}

__global__ void __launch_bounds__(RU_THREADS) records_unpack_kernel(const UnpackParams P) {
  __shared__ int s_status;
  __shared__ int64_t s_src[RU_SEGS], s_units[RU_SEGS + 1], s_vec[RU_SEGS];
  __shared__ uint8_t* s_dst[RU_SEGS];
  if (threadIdx.x == 0) {
    const int32_t* header = reinterpret_cast<const int32_t*>(P.blob);
    const int64_t B = P.B, K = P.K;
    int st = 0;
    if (header[LNB_PACK_HDR_MAGIC] != LNB_PACK_MAGIC) st |= LNB_UNPACK_BAD_MAGIC;
    if (header[LNB_PACK_HDR_B] != P.B || header[LNB_PACK_HDR_K] != P.K) st |= LNB_UNPACK_BAD_SHAPE;
    if (header[LNB_PACK_HDR_F] != P.F) st |= LNB_UNPACK_BAD_FEATURES;
    const int64_t row_bytes = 4 * (int64_t)(P.F ? P.F : 1);    // one atom id or F floats per node
    const int64_t total = header[LNB_PACK_HDR_TOTAL];
    int64_t rows = 0, nedge = 0;
    const bool eigs = header[LNB_PACK_HDR_D] != 0 || header[LNB_PACK_HDR_V_ROWS] != 0;
    if (!st) {
      if (total < LNB_PACK_HDR_BYTES || total > P.blob_bytes || (total & 15) ||
          !seg_ok(header[LNB_PACK_HDR_SIZES], 4 * B, total) ||
          !seg_ok(header[LNB_PACK_HDR_NODE_PTR], 4 * (B + 1), total) ||
          !seg_ok(header[LNB_PACK_HDR_EDGE_PTR], 4 * (B + 1), total)) {
        st |= LNB_UNPACK_BAD_SEGMENT;
      } else {
        const int32_t* np_ = reinterpret_cast<const int32_t*>(P.blob + header[LNB_PACK_HDR_NODE_PTR]);
        const int32_t* ep_ = reinterpret_cast<const int32_t*>(P.blob + header[LNB_PACK_HDR_EDGE_PTR]);
        rows = np_[B];
        nedge = ep_[B];
        if (np_[0] != 0 || ep_[0] != 0 || rows < 0 || nedge < 0 ||
            !seg_ok(header[LNB_PACK_HDR_NODE_FEAT], row_bytes * rows, total) ||
            !seg_ok(header[LNB_PACK_HDR_EDGES], 4 * nedge, total))
          st |= LNB_UNPACK_BAD_SEGMENT;
        else if (eigs && (!seg_ok(header[LNB_PACK_HDR_D], 4 * B * K, total) ||
                          !seg_ok(header[LNB_PACK_HDR_V_ROWS], 4 * rows * K, total)))
          st |= LNB_UNPACK_BAD_SEGMENT;              // present eigenpairs come as both segments
      }
    }
    if (!st && rows > P.cap_rows) st |= LNB_UNPACK_ROWS_OVER;
    if (!st && nedge > P.cap_edges) st |= LNB_UNPACK_EDGES_OVER;
    if (!st && !eigs && (P.D || P.V_rows)) st |= LNB_UNPACK_NO_EIGS;
    if (!st && P.label && (header[LNB_PACK_HDR_P] != P.P || !seg_ok(header[LNB_PACK_HDR_LABEL], 4 * B * P.P, total)))
      st |= LNB_UNPACK_NO_LABELS;
    s_status = st;
    if (!st) {
      // a label segment is read only when asked for: lnb_records_unpack ignores it
      const int64_t src[RU_SEGS] = {header[LNB_PACK_HDR_SIZES], header[LNB_PACK_HDR_NODE_PTR],
                                    header[LNB_PACK_HDR_EDGE_PTR], header[LNB_PACK_HDR_NODE_FEAT],
                                    header[LNB_PACK_HDR_EDGES], header[LNB_PACK_HDR_D],
                                    header[LNB_PACK_HDR_V_ROWS], P.label ? header[LNB_PACK_HDR_LABEL] : 0};
      const int64_t bytes[RU_SEGS] = {4 * B, 4 * (B + 1), 4 * (B + 1), row_bytes * rows, 4 * nedge,
                                      P.D ? 4 * B * K : 0, P.V_rows ? 4 * rows * K : 0,
                                      P.label ? 4 * B * P.P : 0};
      uint8_t* dst[RU_SEGS] = {reinterpret_cast<uint8_t*>(P.sizes), reinterpret_cast<uint8_t*>(P.node_ptr),
                               reinterpret_cast<uint8_t*>(P.edge_ptr), P.node_feat,
                               P.edges, reinterpret_cast<uint8_t*>(P.D), reinterpret_cast<uint8_t*>(P.V_rows),
                               reinterpret_cast<uint8_t*>(P.label)};
      // every segment is a whole number of 4-byte words: 16-byte vectors, then up to three words
      s_units[0] = 0;
      for (int s = 0; s < RU_SEGS; ++s) {
        s_src[s] = src[s];
        s_dst[s] = dst[s];
        s_vec[s] = bytes[s] >> 4;
        s_units[s + 1] = s_units[s] + s_vec[s] + ((bytes[s] & 15) >> 2);
      }
    }
  }
  __syncthreads();
  const int st = s_status;
  if (st) {                                          // every graph empty: the producers read nothing
    if (blockIdx.x == 0) {
      for (int i = threadIdx.x; i < P.B; i += RU_THREADS) P.sizes[i] = 0;
      for (int i = threadIdx.x; i <= P.B; i += RU_THREADS) P.node_ptr[i] = P.edge_ptr[i] = 0;
      if (threadIdx.x == 0) P.status[0] = st;
    }
    return;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) P.status[0] = 0;
  const int64_t n_units = s_units[RU_SEGS];
  int s = 0;
  for (int64_t u = (int64_t)blockIdx.x * RU_THREADS + threadIdx.x; u < n_units;
       u += (int64_t)gridDim.x * RU_THREADS) {
    while (u >= s_units[s + 1]) ++s;               // units rise along the grid stride: s never goes back
    const int64_t i = u - s_units[s];
    const uint8_t* src = P.blob + s_src[s];
    uint8_t* dst = s_dst[s];
    if (i < s_vec[s]) {
      reinterpret_cast<uint4*>(dst)[i] = __ldg(reinterpret_cast<const uint4*>(src) + i);
    } else {
      const int64_t w = 4 * s_vec[s] + (i - s_vec[s]);
      reinterpret_cast<int32_t*>(dst)[w] = __ldg(reinterpret_cast<const int32_t*>(src) + w);
    }
  }
}

int launch_unpack(lnb_stream_t stream, const uint8_t* blob, int64_t blob_bytes, int B, int K, int F, int64_t cap_rows,
                  int64_t cap_edges, int32_t* sizes, int32_t* node_ptr, void* node_feat, int32_t* edge_ptr,
                  uint8_t* edges, float* D, float* V_rows, int P, float* label, int32_t* status) {
  LNB_REQUIRE(B >= 1 && K >= 1 && cap_rows >= 0 && cap_edges >= 0 && blob_bytes >= LNB_PACK_HDR_BYTES,
              "records_unpack: bad dims B=%d K=%d cap_rows=%lld cap_edges=%lld blob_bytes=%lld", B, K,
              (long long)cap_rows, (long long)cap_edges, (long long)blob_bytes);
  LNB_REQUIRE(blob && sizes && node_ptr && edge_ptr && status && (node_feat || cap_rows == 0) &&
                  (edges || cap_edges == 0),
              "records_unpack: null pointer");
  const void* ptrs[] = {blob, sizes, node_ptr, node_feat, edge_ptr, edges, D, V_rows, label};
  for (const void* p : ptrs)
    LNB_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15) == 0, "records_unpack: buffers must be 16-byte aligned");
  UnpackParams p;
  p.blob = blob; p.blob_bytes = blob_bytes; p.B = B; p.K = K; p.cap_rows = cap_rows; p.cap_edges = cap_edges;
  p.F = F; p.sizes = sizes; p.node_ptr = node_ptr; p.node_feat = static_cast<uint8_t*>(node_feat);
  p.edge_ptr = edge_ptr; p.edges = edges;
  p.D = D; p.V_rows = V_rows; p.P = P; p.label = label; p.status = status;
  // the grid depends on the capacities only (a captured launch serves every batch that fits them)
  const int64_t max_bytes = 12 * (int64_t)B + 8 + 4 * (int64_t)(F ? F : 1) * cap_rows + 4 * cap_edges +
                            (D ? 4 * (int64_t)B * K : 0) + (V_rows ? 4 * cap_rows * K : 0) +
                            (label ? 4 * (int64_t)B * P : 0);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(lnb::ceil_div(max_bytes, 16 * RU_THREADS) + 1,
                                                               4 * (int64_t)sms));
  records_unpack_kernel<<<grid, RU_THREADS, 0, (cudaStream_t)stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch("records_unpack");
}

}  // namespace

extern "C" {

int lnb_records_unpack(lnb_stream_t stream, const uint8_t* blob, int64_t blob_bytes, int B, int K,
                       int64_t cap_rows, int64_t cap_edges, int32_t* sizes, int32_t* node_ptr,
                       int32_t* node_feat, int32_t* edge_ptr, uint8_t* edges, float* D, float* V_rows,
                       int32_t* status) {
  return launch_unpack(stream, blob, blob_bytes, B, K, 0, cap_rows, cap_edges, sizes, node_ptr, node_feat, edge_ptr,
                       edges, D, V_rows, 0, nullptr, status);
}

int lnb_records_unpack_labels(lnb_stream_t stream, const uint8_t* blob, int64_t blob_bytes, int B, int K,
                              int64_t cap_rows, int64_t cap_edges, int32_t* sizes, int32_t* node_ptr,
                              int32_t* node_feat, int32_t* edge_ptr, uint8_t* edges, float* D, float* V_rows,
                              int32_t* status, int P, float* label) {
  LNB_REQUIRE(P >= 1 && label, "records_unpack_labels: P=%d, label %p", P, (const void*)label);
  return launch_unpack(stream, blob, blob_bytes, B, K, 0, cap_rows, cap_edges, sizes, node_ptr, node_feat, edge_ptr,
                       edges, D, V_rows, P, label, status);
}

int lnb_records_unpack_features(lnb_stream_t stream, const uint8_t* blob, int64_t blob_bytes, int B, int K, int F,
                                int64_t cap_rows, int64_t cap_edges, int32_t* sizes, int32_t* node_ptr,
                                float* node_x, int32_t* edge_ptr, uint8_t* edges, float* D, float* V_rows,
                                int32_t* status, int P, float* label) {
  LNB_REQUIRE(F >= 1 && F <= LNB_PREPARE_MAX_F && P >= 0 && (P == 0) == (label == nullptr),
              "records_unpack_features: F=%d (1 <= F <= %d), P=%d, label %p", F, LNB_PREPARE_MAX_F, P,
              (const void*)label);
  return launch_unpack(stream, blob, blob_bytes, B, K, F, cap_rows, cap_edges, sizes, node_ptr, node_x, edge_ptr,
                       edges, D, V_rows, P, label, status);
}

}  // extern "C"
