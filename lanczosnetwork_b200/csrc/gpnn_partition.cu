// GPNN propagation within clusters and across cuts (reference: model/gpnn.py:192-225), both partition
// operators in one launch.  For part p in {cluster, cut} with valued operator L_p [B, N, N]:
//     h'_p[r, :] = GRUCell( (W_p M_p)[r, :],  h_p[r, :] )
// with W_p = L_p (sum) or L_p[n, m] / (rowsum_n(L_p) + FLT_EPSILON) (avg), M_p [B*N, H] the messages of
// msg_func[0] and the GRU weights of update_func_partition (input width H).  Unlike lnb_ggnn_update the
// operator VALUES enter: the partition operators are L4 Laplacians D^-1/2 (I + A_part) D^-1/2.
//
// The GRU step of gru_step.cuh with H/32 message k-blocks, over work items (row tile, part, column
// tile): the items of one row tile run on neighbouring CTAs at the same time, so the gathers of both
// parts share L2.  W is the gru_gate_matrix of update_func_partition [4H, 2H].  The message k-blocks
// are the weighted sum of the M_p rows of node n's neighbours, gathered through the ELL rows of
// lnb_graph_prepare over stack([L_cluster, L_cut], 3) (not binarised).  The output of part p goes to
// out_p with row stride ldo (a column block of the [B*N, 3H] input of state_func), and the first
// active part can copy its h row into h_copy (block 0 of that input) from the values its epilogue
// already loads.
#include "gru_step.cuh"

namespace {

constexpr int GP_PARTS = 2;                   // cluster, cut

struct GpnnPartitionParams {
  const float* M[GP_PARTS];    // [rows, ldm] messages of part slot s (may alias between slots)
  const float* h[GP_PARTS];    // [rows, ldh] state of part slot s (may alias between slots)
  float* out[GP_PARTS];        // [rows, ldo]
  int op[GP_PARTS];            // operator channel (0 cluster, 1 cut) of part slot s
  const float* ell_val;        // [B, 2, N, N]  t-major ELL rows (lnb_graph_prepare)
  const uint8_t* ell_idx;      // [B, 2, N, N]
  const int32_t* ell_max;      // [B, 2]
  const float* bias;           // [4H] interleaved like the rows of W
  float* h_copy;               // [rows, ldo] or null: slot 0 writes its h row here
  int rows, N, D, avg, nparts, ldm, ldh, ldo;   // D = H
  int dbg;
};

struct GpnnPartitionPolicy : gru::Step<GpnnPartitionPolicy, GpnnPartitionParams> {
  using Step::Step;
  static __device__ __forceinline__ int parts(const Params& p) { return p.nparts; }
  // sub = slot * n_tiles + column tile
  static __device__ __forceinline__ int col_tile(const Params& p, int sub) { return sub % n_tiles(p); }
  static __device__ __forceinline__ int msg_kblocks(const Params& p) { return p.D / tcg::BK; }

  int slot = 0, cnt = 0;
  int64_t line = 0;
  float denom = 1.f;

  __device__ __forceinline__ void begin_row(int sub) {
    slot = sub / n_tiles(p);
    cnt = 0;
    denom = 1.f;
    if (!row_ok) return;
    // row n of the operator: entries t < len, the non-zeros first (diagonal, then ascending column)
    const int e = p.op[slot];
    line = ((int64_t)(b * GP_PARTS + e) * p.N) * p.N + n;
    const int len = __ldg(p.ell_max + b * GP_PARTS + e);
    float sum = 0.f;
    while (cnt < len) {
      const float v = __ldg(p.ell_val + line + (int64_t)cnt * p.N);
      if (v == 0.f) break;
      sum += v;
      ++cnt;
    }
    // avg: the reference's L / (rowsum(L) + eps), one correctly rounded division per entry
    denom = sum + FLT_EPSILON;
  }

  __device__ __forceinline__ const float* h_row() const { return p.h[slot] + (int64_t)row * p.ldh; }

  __device__ __forceinline__ void produce_msg(int kb, float (&v)[32]) {
    const float* mb = p.M[slot] + (int64_t)b * p.N * p.ldm + kb * tcg::BK;
#pragma unroll 2
    for (int t = 0; t < cnt; ++t) {
      const float val = __ldg(p.ell_val + line + (int64_t)t * p.N);
      const float w = p.avg ? __fdiv_rn(val, denom) : val;
      const int m = __ldg(p.ell_idx + line + (int64_t)t * p.N);
      const float4* src = reinterpret_cast<const float4*>(mb + (int64_t)m * p.ldm);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 x = __ldg(src + j);
        v[4 * j] = fmaf(w, x.x, v[4 * j]);
        v[4 * j + 1] = fmaf(w, x.y, v[4 * j + 1]);
        v[4 * j + 2] = fmaf(w, x.z, v[4 * j + 2]);
        v[4 * j + 3] = fmaf(w, x.w, v[4 * j + 3]);
      }
    }
  }

  __device__ __forceinline__ void write_row(int u0, const float (&o)[4], const float4& hv) {
    const int64_t off = (int64_t)row * p.ldo + u0;
    *reinterpret_cast<float4*>(p.out[slot] + off) = make_float4(o[0], o[1], o[2], o[3]);
    if (slot == 0 && p.h_copy) *reinterpret_cast<float4*>(p.h_copy + off) = hv;
  }
};

// Do the element sets {a + i*lda + j} and {b + i*ldb + j} (0 <= i < rows, 0 <= j < width) intersect?
// Exact for equal strides (column blocks of one matrix), conservative otherwise.
bool blocks_overlap(const float* a, int64_t lda, const float* b, int64_t ldb, int64_t rows, int64_t width) {
  const uintptr_t a0 = (uintptr_t)a, b0 = (uintptr_t)b;
  const uintptr_t a1 = a0 + ((rows - 1) * lda + width) * sizeof(float);
  const uintptr_t b1 = b0 + ((rows - 1) * ldb + width) * sizeof(float);
  if (a1 <= b0 || b1 <= a0) return false;
  const int64_t d = (int64_t)(a0 - b0);
  if (lda != ldb || d % (int64_t)sizeof(float) != 0) return true;
  const int64_t ld = lda, m = (((d / (int64_t)sizeof(float)) % ld) + ld) % ld;   // column offset of a in b's rows
  return m < width || ld - m < width;
}

}  // namespace

extern "C" {

int lnb_gpnn_partition_update(lnb_stream_t stream, const float* M0, const float* h0, float* out0,
                              const float* M1, const float* h1, float* out1, const float* ell_val,
                              const uint8_t* ell_idx, const int32_t* ell_max, const float* W_hi,
                              const float* W_lo, const float* bias, float* h_copy, int B, int N, int H,
                              int ldm, int ldh, int ldo, int avg) {
  LNB_REQUIRE(ell_val && ell_idx && ell_max && W_hi && W_lo && bias, "gpnn_partition_update: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && H >= 1, "gpnn_partition_update: bad dims B=%d N=%d H=%d", B, N, H);
  const float* Ms[GP_PARTS] = {M0, M1};
  const float* hs[GP_PARTS] = {h0, h1};
  float* outs[GP_PARTS] = {out0, out1};
  GpnnPartitionPolicy::Params p{};
  int np = 0;
  for (int e = 0; e < GP_PARTS; ++e) {
    if (!Ms[e] && !hs[e] && !outs[e]) continue;      // a null part is skipped
    LNB_REQUIRE(Ms[e] && hs[e] && outs[e], "gpnn_partition_update: part %d has a null M, h or out", e);
    p.M[np] = Ms[e]; p.h[np] = hs[e]; p.out[np] = outs[e]; p.op[np] = e;
    ++np;
  }
  LNB_REQUIRE(np > 0 || !h_copy, "gpnn_partition_update: h_copy needs an active part");
  if (N > LNB_MAX_N_ELL || H % 32 || H < 32 || H > LNB_MAX_WIDTH) {
    lnb::set_err("gpnn_partition_update: N=%d H=%d outside the kernel (N <= %d, H %% 32 == 0, 32 <= H <= %d)",
                 N, H, LNB_MAX_N_ELL, LNB_MAX_WIDTH);
    return LNB_ERR_UNSUPPORTED;
  }
  uintptr_t al = (uintptr_t)W_hi | (uintptr_t)W_lo | (uintptr_t)h_copy;
  for (int s = 0; s < np; ++s) al |= (uintptr_t)p.M[s] | (uintptr_t)p.h[s] | (uintptr_t)p.out[s];
  if (al % 16 || ldm % 4 || ldh % 4 || ldo % 4 || ldm < H || ldh < H || ldo < H) {
    lnb::set_err("gpnn_partition_update: M, h, out, h_copy and W must be 16-byte aligned and ldm=%d, ldh=%d, "
                 "ldo=%d multiples of 4 and >= H=%d", ldm, ldh, ldo, H);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE((int64_t)B * N <= 0x7fffffff, "gpnn_partition_update: B*N too large");
  const int rows = B * N;
  if (rows == 0 || np == 0) return LNB_OK;
  // the epilogue reads h after other tiles wrote their outputs: no output may overlap any h
  for (int s = 0; s < np; ++s) {
    for (int q = 0; q < np; ++q) {
      if (blocks_overlap(p.out[s], ldo, p.h[q], ldh, rows, H) ||
          (h_copy && blocks_overlap(h_copy, ldo, p.h[q], ldh, rows, H))) {
        lnb::set_err("gpnn_partition_update: out / h_copy must not overlap any h");
        return LNB_ERR_UNSUPPORTED;
      }
      if (q != s && blocks_overlap(p.out[s], ldo, p.out[q], ldo, rows, H)) {
        lnb::set_err("gpnn_partition_update: the outputs of the two parts overlap");
        return LNB_ERR_UNSUPPORTED;
      }
    }
    if (h_copy && blocks_overlap(h_copy, ldo, p.out[s], ldo, rows, H)) {
      lnb::set_err("gpnn_partition_update: h_copy overlaps an output");
      return LNB_ERR_UNSUPPORTED;
    }
  }
  p.ell_val = ell_val; p.ell_idx = ell_idx; p.ell_max = ell_max; p.bias = bias; p.h_copy = h_copy;
  p.rows = rows; p.N = N; p.D = H; p.avg = avg ? 1 : 0; p.nparts = np;
  p.ldm = ldm; p.ldh = ldh; p.ldo = ldo; p.dbg = tcg::debug_flags();
  return tcg::launch<GpnnPartitionPolicy>(stream, W_hi, W_lo, 4 * H, 2 * H, GpnnPartitionPolicy::SMEM_BYTES,
                                          lnb::ceil_div(rows, tcg::BM) * np * (4 * H / tcg::BN), p,
                                          "gpnn_partition_update");
}

}  // extern "C"
