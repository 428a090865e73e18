/*
 * lanczosnet_b200.h -- C ABI of liblanczosnet_b200.so (sm_90a only).
 *
 * Drop-in boundary for the LanczosNet spectral-convolution forward path of
 * lrjconan/LanczosNetwork.  Conventions follow the reference's own native interface
 * (operators/src/cuda/segment_reduction.h:8-12): the CUDA stream comes first, inputs are
 * const device pointers to contiguous row-major buffers, dimensions are plain ints,
 * outputs come last.  Differences, on purpose:
 *   - every entry point returns an int status (0 = ok, <0 = argument error, >0 = cudaError_t)
 *     instead of calling exit(-1) on a launch failure (segment_reduction.cu:28-36);
 *   - the library owns no tensor memory and never synchronises; workspace is caller-provided;
 *   - no global mutable state besides a thread-local error string (re-entrant under
 *     nn.DataParallel's one-thread-per-device execution, runner/qm8_runner.py:291-292).
 *
 * All pointers are DEVICE pointers unless stated otherwise.  There is no CPU fallback.
 */
#ifndef LANCZOSNET_B200_H_
#define LANCZOSNET_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* lnb_stream_t; /* cudaStream_t */

#define LNB_OK 0
#define LNB_ERR_ARG (-1)
#define LNB_ERR_UNSUPPORTED (-2)

/* Shape limits: an entry point returns LNB_ERR_UNSUPPORTED outside its envelope, which the comments below
 * state in these names.  Kernels that feed one another share a name. */
#define LNB_MAX_N 128               /* padded nodes per graph of the records producers, the ELL messages, the
                                       eigensolver, the partition, the convolution stack, GAT and Set2Vec */
#define LNB_MAX_N_ELL 255           /* nodes a uint8 ELL column index addresses: lnb_graph_prepare and the
                                       kernels that read only its ELL rows (GRU updates, neighbour max) */
#define LNB_MAX_E1 16               /* operator channels E1 = bond types + 1 */
#define LNB_MAX_WIDTH 128           /* feature width of the tensor-core kernels: one 128-column wgmma tile */
#define LNB_PREPARE_MAX_F 4096      /* float node features of lnb_graph_prepare_sparse_features */
#define LNB_CONV_MAX_K 32           /* Ritz pairs of the fused convolution */
#define LNB_CONV_MAX_LAYERS 8       /* layers of one lnb_spectral_stack_forward (lnb_spectral_stack.Din) */
#define LNB_FILTER_MLP_MAX_S 32     /* long scales of the Ritz power table and the filter-MLP chain */
#define LNB_GAT_MAX_WIDTH 128       /* GAT head width F */
#define LNB_GAT_MAX_HEADS 32
#define LNB_SET2VEC_MAX_P 128       /* Set2Vec outputs */
#define LNB_CHAIN_MAX_N 32          /* nodes of the one-launch operator chain and its walk */
#define LNB_CHAIN_MAX_STEPS 64      /* steps of that chain, and short-walk steps of lnb_graph_messages */
#define LNB_MESSAGES_MAX_N 32       /* lnb_graph_messages */
#define LNB_MESSAGES_MAX_K 32
#define LNB_MESSAGES_MAX_S 8
#define LNB_LANCZOS_FUSED_MAX_N 1024 /* lnb_lanczos_ritz */
#define LNB_LANCZOS_MAX_K 64        /* Lanczos steps of the fused kernel and of the training path */
#define LNB_LANCZOS_TRAIN_MAX_N 128 /* lnb_lanczos_tridiag_train / _backward: one thread per node */
#define LNB_TRIDIAG_POWERS_MAX_S 32 /* powers of lnb_tridiag_powers and its adjoint */
#define LNB_EIGS_MAX_K 128          /* eigenpairs of lnb_graph_eigs_sparse / lnb_sym_eigs */
#define LNB_EIGS_MAX_E 32           /* bond types the sparse eigensolver and partition read (one bit each) */
#define LNB_PARTITION_MIN_P 2       /* clusters of lnb_spectral_partition(_sparse) */
#define LNB_PARTITION_MAX_P 16

/* ABI version (bumped on any signature change) and last error text of the calling thread. */
int lnb_abi_version(void);
const char* lnb_last_error(void);
/* Number of kernels this library has launched from the calling thread (bench.py's
 * gpu_launches evidence). */
int64_t lnb_launch_count(void);

/* ---------------------------------------------------------------------------------------
 * operators/segment_reduction  (replaces operators/src/cuda/segment_reduction.h:8-12 and the
 * four python-visible names of operators/src/segment_reduction{,_cuda}.h:1-6)
 * data [B, dim1, dim2] fp32, segment_ids [B, dim1] int64, output [B, num_segments, dim2].
 * forward:  output[b, ids[b,c], :] += data[b, c, :]       (output pre-zeroed by the caller,
 *                                                          operators/functions/unsorted_segment_sum.py:20-27)
 * backward: grad_data[b, c, :] = grad_output[b, ids[b,c], :]
 * data_shape = host pointer to {B, dim1, dim2} like the reference launcher.
 * ------------------------------------------------------------------------------------- */
int lnb_unsorted_segment_sum_forward(lnb_stream_t stream, const float* data,
                                     const int64_t* segment_ids, const int* data_shape,
                                     int num_segments, float* output);
int lnb_unsorted_segment_sum_backward(lnb_stream_t stream, const float* grad_output,
                                      const int64_t* segment_ids, const int* data_shape,
                                      int num_segments, float* grad_data);

/* The forward's sum made exact and order-independent: the same arguments and semantics (output
 * accumulated into, batch stride num_segments*dim2, ids outside [0, num_segments) skipped, empty data:
 * nothing launched), but the result's bits do not depend on row order, grid size or scheduling, so
 * repeated runs are bit-identical.  lnb_unsorted_segment_sum_forward adds with fp32 atomics instead.
 * Workspace, one word of each per output element [B, num_segments, dim2], zeroed by the caller:
 * acc int64, exp int32, flags int32.  Three launches, integer atomics only.  For each output element
 * with terms x_i (out_in: its value on entry):
 *   1. e_max = the largest ilogb|x_i| over the finite nonzero terms; flags record NaN, +Inf, -Inf;
 *   2. k = 61 - H - e_max, H = the bit length of dim1;  acc = sum of rint(x_i * 2^k) (ties to even),
 *      each product exact in double and the sum exact in int64 (|acc| < 2^62);
 *   3. out = out_in + s, with s = NaN if a NaN or both infinities occurred, else +-Inf if one sign of
 *      infinity occurred, else 0 if there was no finite nonzero term, else
 *      ldexpf(__ll2float_rn(acc), -k): acc rounded to float, then scaled by 2^-k (correctly rounded).
 * Against the exact sum of c terms, s errs by at most c * 2^(e_max - 62 + H) plus its final rounding:
 * below half an ulp of the largest term whenever c * 2^H < 2^38. */
int lnb_unsorted_segment_sum_exact(lnb_stream_t stream, const float* data, const int64_t* segment_ids,
                                   const int* data_shape, int num_segments, int64_t* acc, int32_t* exp,
                                   int32_t* flags, float* output);

/* ---------------------------------------------------------------------------------------
 * Generic strided batched fp32 GEMM
 *     C[b,z] = act( alpha * (A[b,z] * kscale[b,z]) @ B[b,z] + beta * D[b,z] + bias )
 * (the torch.bmm / nn.Linear call sites of model/lanczos_net.py:112-121,167-181; the addend D is
 * the Chebyshev recurrence 2 L s_{k-1} - s_{k-2} of model/cheby_net.py:91-93).
 * Strides are in elements.  kscale (optional) multiplies column k of A; bias (optional) has
 * N entries; relu != 0 applies max(.,0); alpha == 0 is read as 1 (zero-initialised descriptors
 * keep their old meaning); addend == NULL skips the beta term.  CUDA-core FFMA path for
 * arbitrary shapes/strides.
 * ------------------------------------------------------------------------------------- */
typedef struct lnb_gemm_desc {
  const float* A; int64_t a_sb, a_sz, a_sm, a_sk;
  const float* B; int64_t b_sb, b_sz, b_sk, b_sn;
  float* C;       int64_t c_sb, c_sz, c_sm, c_sn;
  const float* kscale; int64_t s_sb, s_sz, s_sk;
  const float* bias; int64_t bias_sz;   /* bias[z*bias_sz + n] */
  int32_t batch, nz, M, N, K, relu;
  float alpha, beta;
  const float* addend; int64_t d_sb, d_sz, d_sm, d_sn;
} lnb_gemm_desc;
int lnb_batched_gemm(lnb_stream_t stream, const lnb_gemm_desc* desc /* host */);

/* ---------------------------------------------------------------------------------------
 * Dense layer on the Hopper tensor cores (wgmma):  C[M,N] = act(A[M,K] @ W[N,K]^T + bias)
 * (nn.Linear of model/lanczos_net.py:181 and the 4096-wide MLP of ada_lanczos_net.py:54-63).
 * fp32 in/out; computed as 3xTF32 split products (hi*hi + hi*lo + lo*hi) with fp32
 * accumulation -> fp32-grade accuracy.  W_hi / W_lo are the tf32 split of W produced once by
 * lnb_split_tf32.  Requirements: K % 4 == 0 and 16-byte aligned operands; any M, N.
 * Two accumulators (A_hi*W_hi and the two correction products) are summed in fp32 by the
 * epilogue so the small terms do not add truncation steps to the large accumulator.
 * ------------------------------------------------------------------------------------- */
int lnb_split_tf32(lnb_stream_t stream, const float* x, int64_t n, float* hi, float* lo);
int lnb_linear_tf32x3(lnb_stream_t stream, const float* A, const float* W_hi, const float* W_lo,
                      const float* bias, int M, int N, int K, int relu, float* C);
/* Split-K variant for few output tiles and a deep K (the 4096-wide learned filter MLP of
 * model/ada_lanczos_net.py:54-63 at M = batch): every 128 x 128 output tile is computed by `splits`
 * CTAs over disjoint K ranges, so 2 x 32 tiles fill 128 SMs instead of 64 and the weight stream uses
 * the whole HBM bandwidth.  workspace: ceil(M/128)*ceil(N/128)*splits*128*128 floats; counters:
 * ceil(M/128)*ceil(N/128) ints, zero on entry (the kernel leaves them zero). */
int lnb_linear_tf32x3_splitk(lnb_stream_t stream, const float* A, const float* W_hi, const float* W_lo,
                             const float* bias, int M, int N, int K, int relu, float* C, int splits,
                             float* workspace, int* counters);

/* Block-diagonal ("grouped") variant: C[:, g*N:(g+1)*N] = act(A[:, g*K:(g+1)*K] @ W_g^T + b_g)
 * with A [M, groups*K], W stacked [groups*N, K], bias [groups*N], C [M, groups*N].  Used to run
 * the per-layer Ritz-filter MLPs of all layers (model/lanczos_net.py:47-58,109-113) in one launch
 * per MLP stage. */
int lnb_linear_tf32x3_grouped(lnb_stream_t stream, const float* A, const float* W_hi,
                              const float* W_lo, const float* bias, int M, int groups, int N, int K,
                              int relu, float* C);

/* ---------------------------------------------------------------------------------------
 * Fused spectral graph-convolution layer (model/lanczos_net.py:157-182):
 *   out[b,n,:] = act( cat_c(M_c X_b)[n,:] W^T + bias ),  channels c = S long scales
 *   (V diag(coeff[:,:,s]) V^T) followed by the E1 edge-type operators L[...,e].
 * One persistent wgmma kernel; no intermediate of the reference (N x N filters, [B*N, C*D]
 * messages) exists in HBM.  lnb_graph_prepare runs once per forward (the operators are layer
 * invariant):
 *   ell_val/ell_idx [B,E1,N,N]  t-major ELL rows of every operator channel, ell_max [B,E1];
 *   gext [B,2] = {n_eff, k_eff}: operators / Q are identically zero beyond these extents;
 *   tiles [4B+2]: tiles[0] = T, tiles[1+t] = first graph of packed tile t (next-fit:
 *                sum n_eff <= 128, sum ceil4(k_eff) <= 128, <= 32 graphs), tiles[1+T] = B;
 *                for B >= 2 the tile SCHEDULE the fused kernels run follows at S = tiles + B + 2
 *                (at most 2B + 2 ints; the rest of [B+2, 4B+2) is scratch): S[0] = T',
 *                S[1+t] = first slot of tile t, S[1+T'] = B, S[T'+2+slot] = graph id.  Rule:
 *                first-fit decreasing -- graphs by n_eff descending, k_eff descending, index
 *                ascending, each into the lowest tile where sum n_eff <= 128, sum k_eff <= 128
 *                (unpadded) and <= 32 graphs still hold (data.host_tile_schedule).  Shapes the
 *                fused kernels do not run (K > 32, n_eff > 128) and batches of more than 7113
 *                graphs (beyond the assignment kernel's shared memory) get the next-fit tiles in
 *                graph order instead; with B <= 1 the fused kernels run the table;
 *   rowmap [B*K], nrows [1] (both optional, NULL to skip): the compact Ritz row list of
 *                lnb_ritz_rowmap, produced by the same pass;
 *   flags bit 0: store 1.0 for every non-zero (the `L[L != 0] = 1.0` of model/gcnfp.py:83);
 *   flags bit 2 (LNB_PREP_DEFER_TILES): build the row list (a one-CTA lnb_ritz_rowmap launch) but
 *                leave `tiles` unwritten; the caller writes it with lnb_tile_assign, on any stream,
 *                before a fused kernel reads it.  The filter-MLP chain needs only the row list, so
 *                the placement can run beside the chain instead of in front of it.
 * lnb_tile_assign: the tile table and schedule of `tiles` from gext alone, exactly as the pass
 * above writes them (one CTA).
 * Skipping exact zeros / padded rows is exact.  write_pad != 0 also writes the constant rows
 * act(bias) of padded nodes (needed when the full [B,N,H] tensor is read afterwards).
 * Requirements of the fused kernel: N <= LNB_MAX_N, Din % 32 == 0, K % 4 == 0, K <= LNB_CONV_MAX_K,
 * H % 4 == 0, H <= LNB_MAX_WIDTH, E1 <= LNB_MAX_E1; W is [H, (S+E1)*Din].  Returns LNB_ERR_UNSUPPORTED
 * otherwise (callers use the unfused ops).
 * ------------------------------------------------------------------------------------- */
int lnb_graph_prepare(lnb_stream_t stream, const float* L, const float* Q, int B, int N, int E1,
                      int K, float* ell_val, uint8_t* ell_idx, int32_t* ell_max, int32_t* gext,
                      int32_t* tiles, int32_t* rowmap, int32_t* nrows, int flags);
#define LNB_PREP_DEFER_TILES 4
int lnb_tile_assign(lnb_stream_t stream, const int32_t* gext, int B, int K, int32_t* tiles);
int lnb_spectral_conv_fused(lnb_stream_t stream, const float* X, const float* Q, const float* coeff,
                            const float* ell_val, const uint8_t* ell_idx, const int32_t* ell_max,
                            const int32_t* gext, const int32_t* tiles, const float* W_hi,
                            const float* W_lo, const float* bias, int B, int N, int Din, int E1,
                            int K, int S, int H, int relu, int write_pad, float* out);

/* Length of the fp64 table inv_sqrt_deg that the normalising sparse producers take (lnb_graph_prepare_sparse
 * and its variants, lnb_graph_eigs_sparse, lnb_spectral_partition(_sparse)): entry d is numpy's
 * np.power(d, -0.5), entry 0 is 0.  It covers every simple-graph degree of their envelope, deg = 1 + the
 * multiplicities summed over bond types, at most 1 + 32 * 128 (32 bond types, self-loops included, on 128
 * nodes). */
#define LNB_INV_SQRT_DEG_LEN 4098

/* ---------------------------------------------------------------------------------------
 * GPU-side batch construction from SPARSE per-molecule records (replaces, on the device, the host
 * pipeline utils/data_helper.py:92-116,155-156 (L4 = D^-1/2 (A + I) D^-1/2 of every bond channel and
 * of the simple graph) + dataset/qm8.py:57-90,220-291 (zero padding / stacking of node_feat,
 * node_mask, L, (D, V)) and the dense pass of lnb_graph_prepare).  Inputs, all device pointers:
 *   sizes [B] real nodes per graph; node_ptr [B+1] their prefix sums; node_feat [node_ptr[B]] atom
 *   ids of the real nodes; edge_ptr [B+1]; edges [edge_ptr[B]][4] bytes {u, v, bond type, 0}
 *   (undirected bonds listed once, local node indices); V_rows [node_ptr[B], K] Ritz vectors of the
 *   real nodes; inv_sqrt_deg [LNB_INV_SQRT_DEG_LEN] fp64 table of deg^-1/2 (entry 0 = 0) from the
 *   host's numpy, so the fp64 products (scale_i * m_ij) * scale_j and their single rounding to fp32 are
 *   bit-identical to the reference's preprocessing.
 * Outputs: everything lnb_graph_prepare emits (same layouts, same bits: ell_val / ell_idx / ell_max /
 * gext / tiles / rowmap / nrows), the padded node_ids [B,N] int64, mask [B,N] uint8 and
 * V [B,N,K] that lnb_spectral_stack_forward reads, and -- only when L_dense != NULL -- the padded dense
 * operators [B,N,N,E1] exactly as the reference's collate builds them.  flags as lnb_graph_prepare
 * (LNB_PREP_DEFER_TILES included).
 * Limits: N <= LNB_MAX_N, 2 <= E1 <= LNB_MAX_E1.
 * ------------------------------------------------------------------------------------- */
int lnb_graph_prepare_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* node_ptr,
                             const int32_t* node_feat, const int32_t* edge_ptr, const uint8_t* edges,
                             const float* V_rows, const double* inv_sqrt_deg, int B, int N, int E1,
                             int K, int flags, float* ell_val, uint8_t* ell_idx, int32_t* ell_max,
                             int32_t* gext, int32_t* tiles, int32_t* rowmap, int32_t* nrows,
                             int64_t* node_ids, uint8_t* mask, float* V, float* L_dense);

/* Packed variant: the whole sparse batch in ONE contiguous, 16-byte aligned device buffer, so a step
 * costs a single H2D copy of exactly the bytes present (eight ranks issuing seven small copies each
 * were host-bound).  Layout: an int32 header hdr[16] of LNB_PACK_HDR_BYTES, its slots named below (the
 * rest 0), then the body [LNB_PACK_HDR_BYTES, TOTAL): the segments, at byte offsets that are multiples of
 * 16.  SIZES, NODE_PTR, EDGE_PTR, D,
 * TILES and KROW depend on (B, K) only, so D and the tiles sit at fixed addresses of a reused buffer
 * (lnb_ritz_power_table and lnb_spectral_stack_forward read them there).
 * D, V_ROWS, TILES and KROW are 0 when the batch carries no eigenpairs (data.pack_sparse of
 * data.sparse_collate(..., eigs=False) records, data.PackedMolecules(..., eigs=False)): without the Ritz
 * rows the host cannot know k_eff.  Such a batch is read through lnb_records_unpack, never by this kernel.
 * LABEL and P: the labels of a training batch (data.pack_sparse(..., label=True),
 * data.PackedMolecules(..., labels=True)), the last segment, behind the bonds; every other offset is that
 * of the same batch without labels, and TOTAL counts the segment.  Both are 0 when the batch carries no
 * labels.  Only lnb_records_unpack_labels reads the segment.
 * F: the width of the node rows.  0 = atom ids, NODE_FEAT is int32 [sum n]; F > 0 = float feature rows
 * (LanczosNetGeneral's GraphData records), NODE_FEAT is float32 [sum n, F], 4 F bytes per node.  Every other
 * segment and offset rule is the same for both.  Atom-id batches are read by lnb_graph_prepare_sparse_packed
 * and lnb_records_unpack(_labels), feature batches by lnb_graph_prepare_sparse_features_packed and
 * lnb_records_unpack_features. */
#define LNB_PACK_MAGIC 0x4c4e4231   /* "LNB1" */
#define LNB_PACK_HDR_BYTES 64
#define LNB_PACK_HDR_MAGIC 0        /* LNB_PACK_MAGIC */
#define LNB_PACK_HDR_B 1
#define LNB_PACK_HDR_K 2
#define LNB_PACK_HDR_SIZES 3        /* offset of sizes [B] i32 */
#define LNB_PACK_HDR_NODE_PTR 4     /* offset of node_ptr [B+1] i32 */
#define LNB_PACK_HDR_EDGE_PTR 5     /* offset of edge_ptr [B+1] i32 */
#define LNB_PACK_HDR_D 6            /* offset of D [B,K] f32 */
#define LNB_PACK_HDR_NODE_FEAT 7    /* offset of node_feat [sum n] i32 */
#define LNB_PACK_HDR_V_ROWS 8       /* offset of V_rows [sum n, K] f32 */
#define LNB_PACK_HDR_EDGES 9        /* offset of edges [sum E][4] u8 */
#define LNB_PACK_HDR_TOTAL 10       /* total bytes */
#define LNB_PACK_HDR_TILES 11       /* offset of tiles [3B+4] i32: next-fit table [B+2], tile schedule [2B+2] */
#define LNB_PACK_HDR_KROW 12        /* offset of krow_ptr [B+1] i32 */
#define LNB_PACK_HDR_LABEL 13       /* offset of label [B, P] f32 */
#define LNB_PACK_HDR_P 14
#define LNB_PACK_HDR_F 15           /* width of the node rows: 0 = atom ids, F > 0 = float32 [sum n, F] */
/* The kernel derives its input pointers from the header on the device.  flags bit 1
 * (LNB_PACKED_HOST_TILES): the host knows every graph's extents, so it ships the tiles (the same
 * next-fit table and first-fit-decreasing schedule as lnb_graph_prepare, in the same layout) and the
 * prefix sums krow_ptr of k_eff; the kernel expands the Ritz row list itself and NO tile-assignment
 * launch follows (the `tiles` argument is then unused: pass the blob's segment to the stack kernel). */
#define LNB_PACKED_HOST_TILES 2
int lnb_graph_prepare_sparse_packed(lnb_stream_t stream, const uint8_t* blob, const double* inv_sqrt_deg,
                                    int B, int N, int E1, int K, int flags, float* ell_val,
                                    uint8_t* ell_idx, int32_t* ell_max, int32_t* gext, int32_t* tiles,
                                    int32_t* rowmap, int32_t* nrows, int64_t* node_ids, uint8_t* mask,
                                    float* V, float* L_dense);

/* A packed batch (layout above, with or without eigenpairs) split back into the records of
 * lnb_graph_prepare_sparse, in ONE launch: the header is read on the device and every segment present is
 * copied into fixed-capacity buffers -- sizes [B], node_ptr [B+1], edge_ptr [B+1], node_feat [cap_rows],
 * edges [cap_edges][4], and, when not NULL, D [B,K] and V_rows [cap_rows, K].  Offsets change from batch to
 * batch, so one captured launch serves every batch of the same (B, K) that fits the capacities.  Copies
 * are 16-byte vectors (then up to three 4-byte words per segment), grid-stride; the grid depends on the
 * capacities only.  Nothing past the header's TOTAL is read, nothing past a capacity is written; rows past
 * node_ptr[B] / edge_ptr[B] keep their old contents.
 * blob_bytes: the allocation behind blob (>= LNB_PACK_HDR_BYTES); every buffer is 16-byte aligned.
 * status [1]: 0 = copied; otherwise nothing but sizes, node_ptr and edge_ptr is written, all three zero
 * (every graph empty, so the producers behind read no row), and status is a set of the bits below. */
#define LNB_UNPACK_BAD_MAGIC 1
#define LNB_UNPACK_BAD_SHAPE 2      /* B or K differs from the header */
#define LNB_UNPACK_BAD_SEGMENT 4    /* a segment unaligned or outside the body, or TOTAL > blob_bytes */
#define LNB_UNPACK_ROWS_OVER 8      /* node_ptr[B] > cap_rows */
#define LNB_UNPACK_EDGES_OVER 16    /* edge_ptr[B] > cap_edges */
#define LNB_UNPACK_NO_EIGS 32       /* D or V_rows requested from a batch without eigenpairs */
#define LNB_UNPACK_NO_LABELS 64     /* lnb_records_unpack_labels: no label segment of that P in the body */
#define LNB_UNPACK_BAD_FEATURES 128 /* the header's F differs from the caller's (0 for the atom-id entries) */
int lnb_records_unpack(lnb_stream_t stream, const uint8_t* blob, int64_t blob_bytes, int B, int K,
                       int64_t cap_rows, int64_t cap_edges, int32_t* sizes, int32_t* node_ptr,
                       int32_t* node_feat, int32_t* edge_ptr, uint8_t* edges, float* D, float* V_rows,
                       int32_t* status);

/* lnb_records_unpack that also copies the label segment (LABEL, P) into label [B, P] (16-byte
 * aligned), in the same launch.  A batch without the segment, with another P or with the segment outside
 * the body adds LNB_UNPACK_NO_LABELS, with every graph empty and nothing copied, as the other failures do.
 * lnb_records_unpack ignores a label segment. */
int lnb_records_unpack_labels(lnb_stream_t stream, const uint8_t* blob, int64_t blob_bytes, int B, int K,
                              int64_t cap_rows, int64_t cap_edges, int32_t* sizes, int32_t* node_ptr,
                              int32_t* node_feat, int32_t* edge_ptr, uint8_t* edges, float* D, float* V_rows,
                              int32_t* status, int P, float* label);

/* The same split of a batch of float feature rows (header slot F > 0): node_x [cap_rows, F] float32 takes the
 * NODE_FEAT segment, 4 F bytes per node, in place of node_feat; P >= 1 also copies the labels into label
 * [B, P], as lnb_records_unpack_labels does, and P = 0 (label NULL) leaves them.  A header whose F is not the
 * caller's adds LNB_UNPACK_BAD_FEATURES, with every graph empty and nothing copied.  One launch of the kernel
 * of lnb_records_unpack.  Limits: 1 <= F <= LNB_PREPARE_MAX_F. */
int lnb_records_unpack_features(lnb_stream_t stream, const uint8_t* blob, int64_t blob_bytes, int B, int K, int F,
                                int64_t cap_rows, int64_t cap_edges, int32_t* sizes, int32_t* node_ptr,
                                float* node_x, int32_t* edge_ptr, uint8_t* edges, float* D, float* V_rows,
                                int32_t* status, int P, float* label);

/* Float-feature variant (LanczosNetGeneral's GraphData records, node features instead of atom ids): the
 * same records and outputs as lnb_graph_prepare_sparse, except that node_x [node_ptr[B], F] fp32 holds the
 * feature rows of the real nodes in place of node_feat, and X [B,N,F] receives the padded feature tensor in
 * place of node_ids: real rows copied bit for bit, padded rows 0 (the reference's GraphData collate followed
 * by .float()).  The copy takes 16-byte vectors when F % 4 == 0 and node_x and X are 16-byte aligned, scalar
 * loads otherwise; the bits are the same either way.  Same kernel as lnb_graph_prepare_sparse (a
 * compile-time variant), one launch plus the tile assignment unless LNB_PREP_DEFER_TILES.
 * Limits: 1 <= N <= LNB_MAX_N, 2 <= E1 <= LNB_MAX_E1, K >= 1, 1 <= F <= LNB_PREPARE_MAX_F
 * (LNB_ERR_UNSUPPORTED otherwise, nothing launched). */
int lnb_graph_prepare_sparse_features(lnb_stream_t stream, const int32_t* sizes, const int32_t* node_ptr,
                                      const float* node_x, const int32_t* edge_ptr, const uint8_t* edges,
                                      const float* V_rows, const double* inv_sqrt_deg, int B, int N, int E1,
                                      int K, int F, int flags, float* ell_val, uint8_t* ell_idx,
                                      int32_t* ell_max, int32_t* gext, int32_t* tiles, int32_t* rowmap,
                                      int32_t* nrows, float* X, uint8_t* mask, float* V, float* L_dense);

/* lnb_graph_prepare_sparse_features on a packed batch of float feature rows with eigenpairs (header slot
 * F > 0): the input pointers come from the header on the device, as in lnb_graph_prepare_sparse_packed, and
 * flags takes LNB_PACKED_HOST_TILES the same way (the tiles and krow_ptr come with the batch, the kernel
 * expands the Ritz row list and no tile-assignment launch follows).  Outputs as
 * lnb_graph_prepare_sparse_features: X [B,N,F], mask, V, the ELL rows and, when L_dense != NULL, the dense
 * operators.  A batch whose header slot F is not the caller's F is read as B empty graphs.  Same kernel as
 * lnb_graph_prepare_sparse_features.  Limits: those of lnb_graph_prepare_sparse_features. */
int lnb_graph_prepare_sparse_features_packed(lnb_stream_t stream, const uint8_t* blob, const double* inv_sqrt_deg,
                                             int B, int N, int E1, int K, int F, int flags, float* ell_val,
                                             uint8_t* ell_idx, int32_t* ell_max, int32_t* gext, int32_t* tiles,
                                             int32_t* rowmap, int32_t* nrows, float* X, uint8_t* mask, float* V,
                                             float* L_dense);

/* ---------------------------------------------------------------------------------------
 * The whole convolution stack (and optionally the embedding gather in front and the readout
 * behind it) in ONE persistent kernel: every CTA keeps its packed tile's state in shared memory
 * across layers, so between layers nothing touches HBM.  Layer l uses rows [l*H, (l+1)*H) of
 * the stacked split weights W_hi / W_lo [num_layers*H, Kw] (columns beyond (S+E1)*Din[l] zero),
 * bias + l*H and coeff + l*coeff_layer_stride.  Input: X [B,N,Din[0]] or node_ids [B,N] +
 * emb_table [emb_rows, Din[0]] (model/lanczos_net.py:154).  Outputs: out_state [B,N,H] (may be
 * NULL) and / or score [B,P] from the fused readout (model/lanczos_net.py:185-194; mask may be
 * NULL = mean over all N nodes; P <= 48).  Same shape limits as lnb_spectral_conv_fused, plus
 * Din[l>0] == H, num_layers <= LNB_CONV_MAX_LAYERS and a 16-byte aligned bias.
 * ------------------------------------------------------------------------------------- */
typedef struct lnb_spectral_stack {
  const float* X; const int64_t* node_ids; const float* emb_table;
  const float* Q; const float* coeff; int64_t coeff_layer_stride;
  const float* ell_val; const uint8_t* ell_idx; const int32_t* ell_max; const int32_t* gext;
  const int32_t* tiles;
  const float* W_hi; const float* W_lo; const float* bias;
  float* out_state;
  const float* W_out; const float* b_out; const float* w_att; const float* b_att;
  const uint8_t* mask; float* score;
  int32_t Din[8];
  int32_t num_layers, Kw, emb_rows, P, write_pad;
  int32_t B, N, E1, K, S, H, relu;
} lnb_spectral_stack;
int lnb_spectral_stack_forward(lnb_stream_t stream, const lnb_spectral_stack* desc /* host */);

/* ---------------------------------------------------------------------------------------
 * GraphSAGE (model/graph_sage.py:98-175) on the convolution stack.  With the Mean aggregator the
 * message of channel e is M_e X with the layer-invariant, count-weighted operator
 *   M_e[b, n, m] = (nonempty[b, n] != 0) * count(nn_idx[b, n, :, e] == m) / K
 * lnb_sage_operators writes it dense, [B, N, N, E1] channel innermost (every entry, zeros
 * included): the layout lnb_graph_prepare reads.  nn_idx [B, N, K, E1] int64 (the collate's
 * neighbour samples), nonempty [B, N] fp32 (one flag per node).  Ids outside [0, N) contribute
 * nothing.  Limit: N * E1 ints within shared memory (LNB_ERR_UNSUPPORTED otherwise).
 *
 * lnb_sage_stack_forward runs the descriptor of lnb_spectral_stack_forward (same fields, same
 * shape limits, S must be 0; LNB_ERR_UNSUPPORTED and nothing launched otherwise) with two changes:
 * every finished layer row y = act(. + b) is replaced by y / (||y||_2 + FLT_EPSILON) (the padded
 * nodes' constant rows of write_pad and of the readout likewise), and with LNB_SAGE_MAX in flags the
 * edge messages are the elementwise max over the ELL entries of each row (values ignored, a row
 * without entries gives 0) instead of the weighted sum.
 *
 * lnb_neighbour_max: the Max messages on their own (the training path),
 *   out[b, n, e*D + f] = max over the ELL entries m of row n of channel e of X[b, m, f]
 *   argmax[b, n, e, f] = that m (ties: lowest m), -1 for a row without entries (out = 0).
 * X [B, N, D]; ell_* from lnb_graph_prepare on the operators above; N <= LNB_MAX_N_ELL.
 * ------------------------------------------------------------------------------------- */
#define LNB_SAGE_MAX 1
int lnb_sage_operators(lnb_stream_t stream, const int64_t* nn_idx, const float* nonempty, int B, int N,
                       int K, int E1, float* out /* [B,N,N,E1] */);
int lnb_sage_stack_forward(lnb_stream_t stream, const lnb_spectral_stack* desc /* host */, int flags);
int lnb_neighbour_max(lnb_stream_t stream, const float* X, const float* ell_val, const uint8_t* ell_idx,
                      const int32_t* ell_max, int B, int N, int E1, int D, float* out /* [B,N,E1*D] */,
                      int32_t* argmax /* [B,N,E1,D] */);

/* ---------------------------------------------------------------------------------------
 * GraphSAGE's neighbour samples drawn on the device from the SPARSE records of
 * lnb_graph_prepare_sparse (sizes, node_ptr, node_feat, edge_ptr, edges; same layouts, bond types
 * >= E1 - 1 ignored), one CTA per graph.  The rule, for graph b, node n < sizes[b] and channel e:
 *   candidates c[0..L): the non-zero columns of row n of channel e of the padded L4 operator
 *     (channel 0 the simple graph, e >= 1 bond type e - 1), ascending -- n itself and its bonded
 *     neighbours;
 *   x_i = word i % 4 of Philox4x32-10 (Random123's constants) at key (seed lo, seed hi) and counter
 *     (i / 4, r, ctr lo, ctr hi), r = (b*N + n)*E1 + e, where (seed, ctr) = sample_key[0..1] (int64,
 *     DEVICE memory: a captured graph draws anew when the caller rewrites the key);
 *   L >= K: a partial Fisher-Yates, for i < K: j = i + floor(x_i (L - i) / 2^32), swap c[i], c[j],
 *     sample i = c[i] (a uniform ordered K-subset, numpy's choice(replace=False));
 *   1 <= L < K: sample i = c[floor(x_i L / 2^32)] (choice(replace=True));
 *   L = 0 and padded rows: every sample is 0 (the reference collate's zero fill).
 * nonempty[b, n] = 1 iff some channel has L >= 1, i.e. n < sizes[b].  The multiply-high mapping is
 * biased by at most L / 2^32 per draw.
 * Outputs: node_ids [B,N] int64, mask [B,N] uint8 and nonempty [B,N] fp32 always; with
 *   LNB_SAGE_SAMPLE_NN_IDX nn_idx [B,N,K,E1] int32 (the collate's layout, what lnb_sage_lstm_step reads);
 *   LNB_SAGE_SAMPLE_ELL the ELL rows, ell_max and gext that lnb_graph_prepare writes for the operator
 *     of lnb_sage_operators on these samples with a zero Q (same values, same slot order; slots past
 *     ell_max unwritten; no tile table: lnb_tile_assign builds it from gext);
 *   LNB_SAGE_SAMPLE_ELL_T (needs LNB_SAGE_SAMPLE_ELL) the same for the transposed operator M_e^T
 *     (ellT_*, gextT), which the training adjoint reads: M is not symmetric.
 * Limits: 1 <= N <= LNB_MAX_N, 2 <= E1 <= LNB_MAX_E1, K >= 1, B*N*E1 < 2^31 (LNB_ERR_UNSUPPORTED otherwise,
 * nothing launched).  edges may be NULL for a batch without bonds.
 * ------------------------------------------------------------------------------------- */
#define LNB_SAGE_SAMPLE_NN_IDX 1
#define LNB_SAGE_SAMPLE_ELL 2
#define LNB_SAGE_SAMPLE_ELL_T 4
int lnb_sage_sample_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* node_ptr,
                           const int32_t* node_feat, const int32_t* edge_ptr, const uint8_t* edges,
                           const int64_t* sample_key, int B, int N, int E1, int K, int flags,
                           int64_t* node_ids, uint8_t* mask, float* nonempty, int32_t* nn_idx,
                           float* ell_val, uint8_t* ell_idx, int32_t* ell_max, int32_t* gext,
                           float* ellT_val, uint8_t* ellT_idx, int32_t* ellT_max, int32_t* gextT);

/* ---------------------------------------------------------------------------------------
 * Embedding rows (model/lanczos_net.py:154): out[r, :] = table[idx[r], :].
 * ------------------------------------------------------------------------------------- */
int lnb_embedding_rows(lnb_stream_t stream, const int64_t* idx, const float* table,
                       int64_t rows, int num_embeddings, int dim, float* out);

/* ---------------------------------------------------------------------------------------
 * Ritz-value power table (model/lanczos_net.py:146-149): table[b,k,s] = D[b,k] ** powers[s],
 * correctly rounded from a double-precision pow.  The per-layer filter MLP
 * (model/lanczos_net.py:109-113) is then four lnb_batched_gemm / lnb_linear_tf32x3 calls over
 * the B*K rows, batched over all layers at once because the input does not depend on the
 * layer state.  powers: host pointer to S ints (S <= LNB_FILTER_MLP_MAX_S).
 * ------------------------------------------------------------------------------------- */
int lnb_ritz_power_table(lnb_stream_t stream, const float* D, int64_t rows, const int* powers,
                         int S, float* table /* [rows, S] */);

/* ---------------------------------------------------------------------------------------
 * Ritz-value filter MLPs of all layers in one persistent wgmma kernel
 * (model/lanczos_net.py:47-58,109-113): coeff[l, r, :] = MLP_l(table[r, :]) for the rows r listed
 * in rowmap (nrows[0] entries; both NULL = all Rall rows).  The four Linear stages of a
 * (row tile, layer) item run back to back with the 128 x hidden activations kept in shared
 * memory.  W_hi/W_lo: tf32 split of the stacked weights [L*(3*hidden+S), hidden]: per layer the
 * rows of stage 0 (input columns zero-padded from S to hidden), stage 1, stage 2, stage 3
 * (S rows); bias_all uses the same row indexing.  lnb_ritz_rowmap builds the compact row list
 * {b*K + k : k < k_eff(b)} from the extents of lnb_graph_prepare (rows of zero-padded Ritz pairs
 * multiply zero Ritz vectors downstream and are skipped; their coeff entries stay unwritten).
 * Requirements: S <= LNB_FILTER_MLP_MAX_S, hidden % 32 == 0, hidden <= LNB_MAX_WIDTH (else
 * LNB_ERR_UNSUPPORTED).
 * lnb_ritz_filter_mlp_ctas: the same with at most `ctas` persistent CTAs (0: one per SM), e.g. one
 * SM fewer while lnb_tile_assign holds an SM beside it, so no CTA waits for that SM.  An item's
 * arithmetic does not depend on the CTA that runs it: coeff is bit-identical for every `ctas`.
 * ------------------------------------------------------------------------------------- */
int lnb_ritz_rowmap(lnb_stream_t stream, const int32_t* gext, int B, int K, int32_t* rowmap,
                    int32_t* nrows);
int lnb_ritz_filter_mlp(lnb_stream_t stream, const float* table, const int32_t* rowmap,
                        const int32_t* nrows, const float* W_hi, const float* W_lo,
                        const float* bias_all, int Rall, int L, int S, int Hd, float* coeff);
int lnb_ritz_filter_mlp_ctas(lnb_stream_t stream, const float* table, const int32_t* rowmap,
                             const int32_t* nrows, const float* W_hi, const float* W_lo,
                             const float* bias_all, int Rall, int L, int S, int Hd, float* coeff,
                             int ctas);

/* ---------------------------------------------------------------------------------------
 * Readout (model/lanczos_net.py:185-194, ada_lanczos_net.py:350-361):
 *   y[b,n,:] = (W_out state[b,n,:] + b_out) * sigmoid(w_att . state[b,n,:] + b_att)
 *   score[b,:] = mean over n with mask[b,n] != 0 (mask == NULL -> all n)
 * ------------------------------------------------------------------------------------- */
int lnb_readout(lnb_stream_t stream, const float* state, const float* W_out, const float* b_out,
                const float* w_att, const float* b_att, const uint8_t* mask, int B, int N, int H,
                int P, float* score /* [B,P] */);

/* ---------------------------------------------------------------------------------------
 * Graph attention of the GAT baseline (model/gat.py:145-180), everything of a layer after the
 * per-head projection.  Channel c = jj*heads + ii (bond channel jj, head ii), C = E1*heads:
 *   s1[k] = Wh_c[k,:] . a1[c,:] + c1[c],   s2[k] = Wh_c[k,:] . a2[c,:] + c2[c]
 *   att[i,k] = softmax over i (the ROW index, per column k) of
 *              leaky_relu(s1[i] + s2[k], 0.2) + bias[b,i,k,jj]
 *   h_c = att Wh_c + state_bias[c,:]
 *   last == 0: out[b,n,c*F:(c+1)*F] = ELU(h_c[n,:])           out [B,N,C*F]
 *   last != 0: out[b,n,:] = (sum over c = 0..C-1 of h_c[n,:]) / C   out [B,N,F]
 * Wh [B,N,C*F] (column block c = Wh_c), bias [B,N,N,E1] channel innermost (the additive mask the
 * reference collate builds, dataset/qm8.py:196-219), a1/a2/state_bias [C,F], c1/c2 [C].  fp32 dots in
 * feature order, max-subtracted softmax with expf, ELU with expm1f; the channel sum runs in a fixed
 * order, so repeated launches are bit-identical.  Wh, state_bias and out 16-byte aligned.
 * Envelope: N <= LNB_MAX_N, F % 4 == 0, F <= LNB_GAT_MAX_WIDTH, E1 <= LNB_MAX_E1, heads <= LNB_GAT_MAX_HEADS
 * (LNB_ERR_UNSUPPORTED otherwise, nothing launched).
 * ------------------------------------------------------------------------------------- */
int lnb_gat_attention(lnb_stream_t stream, const float* Wh, const float* bias, const float* a1,
                      const float* a2, const float* c1, const float* c2, const float* state_bias,
                      int B, int N, int E1, int heads, int F, int last, float* out);

/* Adjoint of lnb_gat_attention for the training path.  Inputs: the forward's Wh, bias, a1, a2, c1, c2,
 * state_bias and gout = dL/dout (the shape of the forward's out).  Per channel c, with att and
 * h_c = att Wh_c + state_bias_c recomputed exactly as the forward computes them, and gh = gout_c * ELU'(h_c)
 * (hidden; ELU'(h) = exp(h) for h <= 0) or gout / C (last):
 *   gWh[b,k,c*F:(c+1)*F] = sum_i att[i,k] gh[i] + gs1[k] a1[c] + gs2[k] a2[c]        gWh [B,N,C*F]
 *   gX[i,k] = att[i,k] (gh[i].Wh[k] - sum_i' att[i',k] gh[i'].Wh[k]) * (s1[i] + s2[k] > 0 ? 1 : 0.2)
 *   gs1[i] = sum_k gX[i,k],  gs2[k] = sum_i gX[i,k]
 *   gpar[b,c,:] = [sum_k gs1[k] Wh[k] (F) | sum_k gs2[k] Wh[k] (F) | sum_i gh[i] (F) | sum gs1 | sum gs2]
 * gpar [B, C, 3F+2] holds each graph's share of the gradients of a1, a2, state_bias, c1 and c2: the caller
 * sums it over B.  The bias gets no gradient.  One CTA per (graph, bond channel, head group); every sum
 * in a fixed order, no atomics: repeated launches are bit-identical.  gout, Wh, a1, a2, state_bias, gWh
 * 16-byte aligned.  Envelope: that of lnb_gat_attention (LNB_ERR_UNSUPPORTED otherwise, nothing launched).
 */
int lnb_gat_attention_backward(lnb_stream_t stream, const float* gout, const float* Wh, const float* bias,
                               const float* a1, const float* a2, const float* c1, const float* c2,
                               const float* state_bias, int B, int N, int E1, int heads, int F, int last,
                               float* gWh, float* gpar);

/* ---------------------------------------------------------------------------------------
 * GAT dropout masks (model/gat.py:149-163; the KeyedGAT training forward).  Layer t, channel
 * c = jj*heads + ii (C channels of F features, layer input width Din, M = B*N node rows) has three
 * sites sigma, each with its own mask of the same p:
 *   sigma = 0, input:     the layer input X seen by channel c, element i = (b*N + n)*Din + d
 *   sigma = 1, attention: att[b, i_row, k] (softmax over i_row), element i = (b*N + i_row)*N + k
 *   sigma = 2, Wh:        Wh_c = the channel's projection, element i = (b*N + n)*F + f
 * Element i of a site is decided by
 *   word = word (i & 3), in the order x, y, z, w, of Philox4x32-10 (Random123's constants) at key
 *     (seed lo, seed hi) and counter (i >> 2, site, ctr lo, ctr hi), where site = (t << 16) | (c << 2) | sigma
 *     and (seed, ctr) = dropout_key[0..1] (int64, DEVICE memory: a captured graph draws anew whenever the
 *     key changes);
 *   kept iff word >= thr, thr = floor(p * 2^32) computed in fp64 and held as a uint64 (p = 1 keeps nothing);
 *   a kept value is x * s with s = (float)(1 / (1 - p)) (one fp32 multiply), a dropped value is 0.
 * One training forward uses one key for every layer, channel and site.  Needs t < 2^16, C <= 2^14 and fewer
 * than 2^34 elements per site (LNB_ERR_UNSUPPORTED otherwise, nothing launched).  The draws are not
 * torch's: same distribution, different masks.
 * ------------------------------------------------------------------------------------- */

/* lnb_gat_attention with the reference's attention and Wh dropout of layer t: att' = att * M_att s and
 * Wh' = Wh_c * M_wh s replace att and Wh_c in h_c = att' Wh' + state_bias_c; the scores s1, s2 read the
 * undropped Wh.  Same arguments, layouts, envelope and determinism as lnb_gat_attention, plus dropout_key,
 * p in [0, 1] and t (the mask rule above). */
int lnb_gat_attention_dropout(lnb_stream_t stream, const float* Wh, const float* bias, const float* a1,
                              const float* a2, const float* c1, const float* c2, const float* state_bias,
                              int B, int N, int E1, int heads, int F, int last, const int64_t* dropout_key,
                              double p, int t, float* out);

/* Adjoint of lnb_gat_attention_dropout, with its masks drawn again (nothing of the forward is saved):
 *   gWh[b,k,c] = M_wh s * (sum_i att'[i,k] gh[i]) + gs1[k] a1[c] + gs2[k] a2[c]
 *   gX[i,k] = att[i,k] (gAtt[i,k] - sum_i' att[i',k] gAtt[i',k]) * (s1[i] + s2[k] > 0 ? 1 : 0.2),
 *     gAtt = M_att s * (gh Wh'^T)
 * and h (for ELU') = att' Wh' + state_bias; ga1, ga2 read the undropped Wh.  Arguments, outputs (gpar
 * per graph, summed by the caller), envelope and determinism as lnb_gat_attention_backward. */
int lnb_gat_attention_dropout_backward(lnb_stream_t stream, const float* gout, const float* Wh, const float* bias,
                                       const float* a1, const float* a2, const float* c1, const float* c2,
                                       const float* state_bias, int B, int N, int E1, int heads, int F, int last,
                                       const int64_t* dropout_key, double p, int t, float* gWh, float* gpar);

/* The per-channel input dropout and projection of GAT layer t:
 *   Wh[m, c*F:(c+1)*F] = (X[m,:] * M_c[m,:] s) W_c^T      for every channel c < C and row m < M
 * X [M, Din], W [C*F, Din] (channel c's weight = rows c*F .. c*F+F-1), Wh [M, C*F]; M_c the input-site
 * mask of (t, c) (the rule above).  No masked copy of X exists: each mask word is drawn once per
 * (row, feature, channel) as the operand tile is loaded.  FFMA in fp32, the sum over d in order.
 * Envelope: Din % 4 == 0, F % 4 == 0, F <= LNB_GAT_MAX_WIDTH; X, W, Wh 16-byte aligned (LNB_ERR_UNSUPPORTED /
 * LNB_ERR_ARG otherwise, nothing launched). */
int lnb_gat_dropout_project(lnb_stream_t stream, const float* X, const float* W, int M, int Din, int C, int F,
                            const int64_t* dropout_key, double p, int t, float* Wh);

/* Row slabs of lnb_gat_dropout_project_backward's gW partials for a shape (a function of the shape
 * only); its workspace holds slabs * C*F*Din floats. */
int lnb_gat_dropout_project_slabs(int M, int Din, int C, int F);

/* Adjoint of lnb_gat_dropout_project, with the masks drawn again:
 *   gX = s sum_{c = 0..C-1} M_c * (gWh_c W_c)              gX [M, Din]
 *   gW_c = s gWh_c^T (X * M_c)                             gW [C*F, Din]
 * One launch walks every (row block, 32-feature block) over the channels in order and draws each mask
 * word once; it writes gX and one gW partial per row slab into `work` [slabs, C*F, Din]; a second launch
 * sums the slabs in order.  No atomics: repeated launches are bit-identical.  Envelope and alignment of
 * lnb_gat_dropout_project, plus gWh, gX, gW, work 16-byte aligned. */
int lnb_gat_dropout_project_backward(lnb_stream_t stream, const float* X, const float* W, const float* gWh,
                                     int M, int Din, int C, int F, const int64_t* dropout_key, double p, int t,
                                     float* gX, float* gW, float* work);

/* ---------------------------------------------------------------------------------------
 * GGNN propagation step after the message MLPs (model/ggnn.py:143-171), one persistent 3xTF32 wgmma
 * launch over all B*N rows:
 *   agg[b,n, e*D:(e+1)*D] = sum over the non-zeros m of row n of channel e of  w * M[b*N+m, e*D:(e+1)*D]
 *                           w = 1 (avg == 0, 'sum') or 1 / (nnz + FLT_EPSILON) (avg != 0, 'avg')
 *   G = [agg | h] W^T + bias;   r = sigmoid(G_r), z = sigmoid(G_z), n = tanh(G_nin + r * G_nh)
 *   out = (h - n) * z + n                                                 (torch's GRUCell)
 * The operators enter only through their non-zero pattern (A_e = L_e != 0, the reference's in-place
 * binarisation): ell_* are the ELL rows of lnb_graph_prepare over L [B,N,N,E1].  The aggregated
 * messages are computed in the producer warps of the GEMM and never written out.
 * M [B*N, E1*D] (column block e = channel e), h and out [B*N, D] (out must not alias h).
 * W_hi / W_lo: tf32 split of the re-laid-out gate matrix [4D, (E1+1)*D] whose row (u/4)*16 + g*4 + u%4
 * is gate g of hidden unit u, g = r, z, n_in, n_h:  r = [W_ir | W_hr], z = [W_iz | W_hz],
 * n_in = [W_in | 0], n_h = [0 | W_hn] (weight_ih / weight_hh of torch.nn.GRUCell); bias [4D] in the same
 * order: b_ir + b_hr, b_iz + b_hz, b_in, b_hn.  M, h, out, W 16-byte aligned.
 * Envelope: 1 <= N <= LNB_MAX_N_ELL, D % 32 == 0, 32 <= D <= LNB_MAX_WIDTH, 1 <= E1 <= LNB_MAX_E1
 * (LNB_ERR_UNSUPPORTED otherwise, nothing launched).  Summation order is fixed: repeated launches are
 * bit-identical.
 * ------------------------------------------------------------------------------------- */
int lnb_ggnn_update(lnb_stream_t stream, const float* M, const float* h, const float* ell_val,
                    const uint8_t* ell_idx, const int32_t* ell_max, const float* W_hi, const float* W_lo,
                    const float* bias, int B, int N, int D, int E1, int avg, float* out);

/* ---------------------------------------------------------------------------------------
 * One time step t of GraphSAGE's LSTM aggregator (model/graph_sage.py:131-140) for all R = B*N*E1
 * sequences of a layer, one persistent 3xTF32 wgmma launch.  Sequence s = (b*N + n)*E1 + e:
 *   x = state[b*N + m] with m = nn_idx[b, n, t, e]  (a zero row when m is outside [0, N))
 *   [i f g o] = [x | h[s]] W^T + bias;  c[s] = sigmoid(f) c[s] + sigmoid(i) tanh(g)
 *   out[s] = sigmoid(o) tanh(c[s])                                       (torch's LSTMCell)
 * At t = 0, h = c = 0: h is not read (may be null) and c is only written.  On the last step
 * (t == K - 1) out[s] is multiplied by nonempty[b*N + n], so out read as [B*N, E1*D] is the layer's
 * message matrix (column block e = channel e).  A sequence of a node with nonempty == 0 gathers nothing
 * and runs no cell: its out row is written (zero) on the last step only, its c row never.
 * state [B*N, D], nn_idx int32 [B, N, K, E1], nonempty [B*N], h / c / out [R, D]; c is updated in place,
 * out must alias neither h (for t > 0) nor c.
 * W_hi / W_lo: tf32 split of [W_ih | W_hh] [4D, 2D] (torch.nn.LSTMCell) with row (u/4)*16 + g*4 + u%4 =
 * gate g of hidden unit u, g = i, f, g, o; bias [4D] = b_ih + b_hh in the same order.  state, h, c, out
 * and W 16-byte aligned.
 * Envelope: D % 32 == 0, 32 <= D <= LNB_MAX_WIDTH, 1 <= E1 <= LNB_MAX_E1, K >= 1, 0 <= t < K (LNB_ERR_UNSUPPORTED for
 * D / E1 outside it, nothing launched).  Summation order is fixed: repeated launches are bit-identical.
 * ------------------------------------------------------------------------------------- */
int lnb_sage_lstm_step(lnb_stream_t stream, const float* state, const int32_t* nn_idx, const float* nonempty,
                       const float* h, float* c, const float* W_hi, const float* W_lo, const float* bias, int B,
                       int N, int K, int E1, int D, int t, float* out);

/* ---------------------------------------------------------------------------------------
 * GPNN propagation within clusters and across cuts (model/gpnn.py:192-225), both partition operators in
 * one persistent 3xTF32 wgmma launch over all B*N rows.  For each active part p (0 = cluster, 1 = cut):
 *   agg_p[b,n, :] = sum over the non-zeros m of row n of operator p of  w * M_p[b*N+m, :]
 *                   w = val (avg == 0, 'sum') or val / (rowsum_n + FLT_EPSILON) (avg != 0, 'avg'; the row
 *                   sum runs over the row's entries in ELL order, the division is correctly rounded)
 *   G = [agg_p | h_p] W^T + bias, then the GRU cell of lnb_ggnn_update: out_p = (h_p - n) * z + n.
 * The operator VALUES enter (the L4 partition Laplacians); ell_* are the ELL rows of lnb_graph_prepare
 * over stack([L_cluster, L_cut], 3) [B,N,N,2], not binarised.  Every one of the B*N rows is computed.
 * M_p [B*N rows, stride ldm], h_p [stride ldh] and out_p [stride ldo], H columns each.  A part whose
 * M, h and out are all null is skipped; M and h may alias between the parts.  h_copy [stride ldo] or
 * null: the first active part also writes its h rows there (block 0 of the [B*N, 3H] input of
 * state_func, whose blocks 1 and 2 are the outputs).
 * W_hi / W_lo: tf32 split of gru_gate_matrix of the partition GRUCell, [4H, 2H] (layout of
 * lnb_ggnn_update with E1 = 1); bias [4H].
 * Envelope: 1 <= N <= LNB_MAX_N_ELL, H % 32 == 0, 32 <= H <= LNB_MAX_WIDTH; pointers 16-byte aligned and ldm, ldh, ldo
 * multiples of 4, at least H; no output (nor h_copy) may share an element with any h or with each other.
 * Outside it: LNB_ERR_UNSUPPORTED, nothing launched.  Summation order is fixed: repeated launches are
 * bit-identical.
 * ------------------------------------------------------------------------------------- */
int lnb_gpnn_partition_update(lnb_stream_t stream, const float* M0, const float* h0, float* out0,
                              const float* M1, const float* h1, float* out1, const float* ell_val,
                              const uint8_t* ell_idx, const int32_t* ell_max, const float* W_hi,
                              const float* W_lo, const float* bias, float* h_copy, int B, int N, int H,
                              int ldm, int ldh, int ldo, int avg);

/* ---------------------------------------------------------------------------------------
 * MPNN propagation step with the edge-network messages (model/mpnn.py:131-191), one persistent 3xTF32
 * wgmma launch over all B*N rows.  Receiver i, neighbour j, channel e, A_e = (L_e != 0):
 *   S_e[i]  = w_i * sum over the non-zeros j of row i of channel e of relu(P_e[j] + Q_e[i])   (64 wide)
 *   deg[i,e] = w_i * nnz_e(i)           w_i = 1 (avg == 0, 'sum') or 1 / (nnz_e(i) + FLT_EPSILON) (avg != 0)
 *   G = [S_0 | ... | S_{E1-1} | deg, zero padded to 32 | h] W^T + bias, then the GRU cell of
 *   lnb_ggnn_update: out = (h - n) * z + n.
 * PQ [B*N, E1*128]: per channel the 64 columns of P_e = h W1a_e^T, then the 64 of Q_e = h W1b_e^T + b1_e
 * (the first edge layer split at the neighbour / receiver halves of its input [h_j | h_i]).
 * W_hi / W_lo: tf32 split of the gate matrix [4D, 64*E1 + 32 + D] laid out as in lnb_ggnn_update, whose
 * input part is the folded F = [W_ih,e W2_e]_e | [W_ih,e b2_e]_e (zero padded to 64*E1 + 32 columns).
 * ell_*: lnb_graph_prepare of L [B,N,N,E1].  h and out [B*N, D] (out must not alias h).  PQ, h, out, W
 * 16-byte aligned.  S is computed in the producer warps and never written out.
 * Envelope: 1 <= N <= LNB_MAX_N_ELL, D % 32 == 0, 32 <= D <= LNB_MAX_WIDTH, 1 <= E1 <= LNB_MAX_E1
 * (LNB_ERR_UNSUPPORTED otherwise, nothing launched).  Summation order is fixed: repeated launches are
 * bit-identical.
 * ------------------------------------------------------------------------------------- */
int lnb_mpnn_update(lnb_stream_t stream, const float* PQ, const float* h, const float* ell_val,
                    const uint8_t* ell_idx, const int32_t* ell_max, const float* W_hi, const float* W_lo,
                    const float* bias, int B, int N, int D, int E1, int avg, float* out);

/* ---------------------------------------------------------------------------------------
 * Training path of lnb_mpnn_update: S [B*N, E1*64] (column block e = S_e) with the producer's
 * arithmetic, and its adjoint
 *   gQ_e[i] = w_i sum_j A_e[i,j] [P_e[j] + Q_e[i] > 0] gS_e[i]
 *   gP_e[j] = sum_i A_e[i,j] w_i [P_e[j] + Q_e[i] > 0] gS_e[i]
 * written as gPQ [B*N, E1*128] in the layout of PQ.  ellT_* are lnb_graph_prepare of the transposed
 * operators L.transpose(1, 2) (operators need not be symmetric).  One thread per output element, sums
 * in ELL order, no atomics: deterministic.  Envelope: 1 <= N <= LNB_MAX_N_ELL, 1 <= E1 <= LNB_MAX_E1
 * (LNB_ERR_UNSUPPORTED otherwise, nothing launched).
 * ------------------------------------------------------------------------------------- */
int lnb_mpnn_edge_aggregate(lnb_stream_t stream, const float* PQ, const float* ell_val, const uint8_t* ell_idx,
                            const int32_t* ell_max, int B, int N, int E1, int avg, float* S);
int lnb_mpnn_edge_aggregate_backward(lnb_stream_t stream, const float* PQ, const float* gS, const float* ell_val,
                                     const uint8_t* ell_idx, const int32_t* ell_max, const float* ellT_val,
                                     const uint8_t* ellT_idx, const int32_t* ellT_max, int B, int N, int E1,
                                     int avg, float* gPQ);

/* ---------------------------------------------------------------------------------------
 * Operator products over the ELL rows of lnb_graph_prepare / lnb_graph_prepare_sparse (the training
 * formulation's L_e X without the dense operators), for the channels c0 <= e < c0 + nc:
 *   out[b*N+n, col0 + (e-c0)*D + d] = sum_{t < ell_max[b,e]} (val[b,e,t,n] w[b,n,e]) X[b*N + idx[b,e,t,n], d]
 * and the adjoint over the ELL rows of the TRANSPOSED operators (ellT_*, gextT: lnb_graph_prepare of
 * L.transpose(1, 2), the contract of lnb_mpnn_edge_aggregate_backward), all channels summed in one thread:
 *   gX[b*N+m, d] = sum_e sum_t (valT[b,e,t,m] w[b,i,e]) G[b*N + i, (e-c0)*D + d],   i = idxT[b,e,t,m]
 * w [B,N,E1] is an optional row weight (NULL: 1), folded into every entry's coefficient (one rounding).
 * X, out, G and gX are row-strided (ldx, ldo, ldg, ldgx in floats, unit column stride) and must not
 * overlap; every channel writes straight into its column block of out.  Rows at or past gext[b,0] are 0.
 * Each sum is one fmaf chain in ascending column order (the row's diagonal, slot 0, taken in its place;
 * the adjoint: one chain per channel, added in channel order): lnb_batched_gemm's order on the dense
 * operator, so on 0/1 operators, weighted or not, both give the same bits.  One thread per output
 * element, no atomics: repeated launches are bit-identical.  A 4-wide path runs when D, the strides and
 * col0 are multiples of 4 and X / out (G / gX) are 16-byte aligned.
 * Envelope: 1 <= N <= LNB_MAX_N, 1 <= E1 <= LNB_MAX_E1, any D >= 1 (LNB_ERR_UNSUPPORTED otherwise, nothing launched).
 * ------------------------------------------------------------------------------------- */
int lnb_ell_messages(lnb_stream_t stream, const float* X, int64_t ldx, const float* ell_val, const uint8_t* ell_idx,
                     const int32_t* ell_max, const int32_t* gext, const float* w, int B, int N, int E1, int c0,
                     int nc, int D, float* out, int64_t ldo, int col0);
int lnb_ell_messages_adjoint(lnb_stream_t stream, const float* G, int64_t ldg, const float* ellT_val,
                             const uint8_t* ellT_idx, const int32_t* ellT_max, const int32_t* gextT, const float* w,
                             int B, int N, int E1, int c0, int nc, int D, float* gX, int64_t ldgx);

/* ---------------------------------------------------------------------------------------
 * Set2Vec readout + output_func of MPNN (model/set2set.py:60-100, model/mpnn.py:198-207), every graph
 * of the batch in one launch.  Per graph, over its set (nodes with mask != 0, or all N when mask is
 * NULL), hidden [2D] = 0, mem [D] = 0, and `steps` times:
 *   f, i, o = sigmoid, c = tanh of the gate rows of Wg hidden + bg (blocks forget, input, output, memory)
 *   mem = f * mem + i * c;  h = o * tanh(mem);  u = h W1;  e_n = tanh(u + x_n) . W2
 *   a = max-subtracted softmax of e over the set;  read = sum_n a_n x_n (0 for an empty set)
 *   hidden = [h | read]
 * then score[b] = W_out hidden + b_out.
 * X [B,N,D]; mask [B,N] uint8 or NULL; WgT [2D, 4D] = the four gate Linear weights stacked [4D, 2D] and
 * transposed; bg [4D]; W1 [D, D] used as [in, out]; W2 [D]; W_out [P, 2D]; b_out [P]; score [B,P].
 * fp32, every sum in a fixed order: repeated launches are bit-identical.
 * Envelope: 1 <= N <= LNB_MAX_N, D % 32 == 0, 32 <= D <= LNB_MAX_WIDTH, 1 <= P <= LNB_SET2VEC_MAX_P
 * (LNB_ERR_UNSUPPORTED otherwise, nothing launched).
 * ------------------------------------------------------------------------------------- */
int lnb_set2vec(lnb_stream_t stream, const float* X, const uint8_t* mask, const float* WgT, const float* bg,
                const float* W1, const float* W2, const float* W_out, const float* b_out, int B, int N, int D,
                int P, int steps, float* score);

/* ---------------------------------------------------------------------------------------
 * Operator chain on channel 0 of L [B,N,N,E1], per graph, starting from X [B,N,D]:
 *   chebyshev == 0: w_s = L_0 w_{s-1} (w_0 = X), s = 1..steps   (model/dcnn.py:88-92, the short
 *                   diffusion walk of model/lanczos_net.py:164-169);
 *   chebyshev != 0: s_0 = L_0 X, s_k = 2 L_0 s_{k-1} - s_{k-2} with s_{-1} = X, k < steps
 *                   (model/cheby_net.py:88-93).
 * Result number i (0-based) is written to out[b, n, (out_col0 + block_of_step[i]) * D + d] when
 * block_of_step[i] >= 0 (host array of `steps` ints); out strides in elements.  One launch for
 * the whole chain: operator and walk stay in shared memory / registers.  N <= LNB_CHAIN_MAX_N,
 * steps <= LNB_CHAIN_MAX_STEPS
 * (LNB_ERR_UNSUPPORTED otherwise: callers use lnb_batched_gemm per step).
 * ------------------------------------------------------------------------------------- */
int lnb_operator_chain(lnb_stream_t stream, const float* L, const float* X, int B, int N, int E1,
                       int D, int steps, int chebyshev, const int* block_of_step /* host */,
                       float* out, int64_t out_batch_stride, int64_t out_row_stride, int out_col0);

/* ---------------------------------------------------------------------------------------
 * The whole message matrix of a general-shape spectral convolution layer in one launch
 * (model/lanczos_net.py:157-180, model/ada_lanczos_net.py:321-345):
 *   out[b, n, :] = [ (L_0^k X)[n] : k selected ] ++ [ (Q G_s Q^T X)[n] : s < S ] ++ [ (L_e X)[n] : e < E1 ]
 * L [B,N,N,E1], X [B,N,D], Q [B,N,K]; filt = G [B,S,K,K] symmetric blocks when dense_filter != 0
 * (AdaLanczosNet's learned filter), else the diagonal coefficients [B,K,S] (LanczosNet).  Short walk:
 * step i (1-based) goes to column block block_of_step[i-1] (< 0: not stored; host array of
 * short_steps ints), the long scales to blocks n_short + s, the edge types to n_short + S + e; every
 * block is D columns wide; out strides in elements.  One CTA per graph, thread per feature column,
 * operators and filters in shared memory, every intermediate in registers.  N <= LNB_MESSAGES_MAX_N,
 * K <= LNB_MESSAGES_MAX_K, E1 <= LNB_MAX_E1, S <= LNB_MESSAGES_MAX_S, short_steps <= LNB_CHAIN_MAX_STEPS
 * (LNB_ERR_UNSUPPORTED otherwise: callers compose lnb_batched_gemm calls).
 * ------------------------------------------------------------------------------------- */
int lnb_graph_messages(lnb_stream_t stream, const float* L, const float* X, const float* Q,
                       const float* filt, int B, int N, int E1, int D, int K, int S, int dense_filter,
                       int short_steps, const int* block_of_step /* host */, int n_short, float* out,
                       int64_t out_batch_stride, int64_t out_row_stride);

/* ---------------------------------------------------------------------------------------
 * Gaussian-kernel graph Laplacian (model/ada_lanczos_net.py:101-137, adjacency from :310-311):
 *   adj = (L[b,i,j,0] != 0);  dist2 = |x_i - x_j|^2;  sigma2 = mean over all N^2 pairs;
 *   A = exp(-dist2/sigma2) * adj;  d = (rowsum + [rowsum==0])^-1/2;  out = d_i A_ij d_j
 * L has E1 channels innermost (dataset/qm8.py:262); only channel 0 is read.
 * ------------------------------------------------------------------------------------- */
int lnb_gaussian_laplacian(lnb_stream_t stream, const float* x, const float* L, int B, int N,
                           int Dx, int E1, float* out /* [B,N,N] */);

/* ---------------------------------------------------------------------------------------
 * Exact eigenpairs of every graph's simple-graph operator, in fp64: the reference's offline
 * preprocessing (utils/data_helper.py:169-226 dense eigh branch, dataset/get_qm8_data.py:63-83,
 * truncated / zero padded to K at collate, dataset/qm8.py:265-291) on the device.  Householder
 * tridiagonalisation, implicit-shift QL with the rotations accumulated, then the back-transform of the
 * kept columns only.  Graph b's operator is the leading n_b x n_b block, n_b = min(sizes[b], N);
 * its lower triangle is read (numpy's eigh default).
 * Outputs: D [B,K] = the eigenvalues by descending |lambda|, equal |lambda| by ascending lambda
 * (np.argsort(-|w|, kind='mergesort') over eigh's ascending order), the first min(n_b, K) of them,
 * then 0; the matching unit eigenvectors (columns >= min(n_b, K) and rows >= n_b are 0).  Every output
 * is one rounding of an fp64 value.  Eigenvectors are defined up to sign and, for a repeated
 * eigenvalue, up to a rotation inside its eigenspace.  status[b]: bit 0 = QL sweeps exhausted.
 * One warp per graph for N <= 32, one CTA per graph above; repeated launches are bit-identical.
 * Envelope: 1 <= N <= LNB_MAX_N, 1 <= K <= LNB_EIGS_MAX_K (LNB_ERR_UNSUPPORTED otherwise, nothing launched).
 *
 * lnb_graph_eigs_sparse: the operator is the fp64 L4 = D^-1/2 (A + I) D^-1/2 of the simple graph
 *   (A summed over bond types; a bond listed twice with one type counts once), built from the sparse
 *   records of lnb_graph_prepare_sparse (sizes, node_ptr, edge_ptr, edges with bond types < E,
 *   1 <= E <= LNB_EIGS_MAX_E, inv_sqrt_deg) with the same fp64 products in the same order, so the solver's input
 *   is bit for bit the matrix the reference hands eigh.  V_rows [node_ptr[B], K]: the rows of the real
 *   nodes, the layout lnb_graph_prepare_sparse reads (data.sparse_collate's).
 * lnb_sym_eigs: the operator is the fp32 A[((b*N + i)*N + j) * elem_stride] (elem_stride = E1 reads
 *   channel 0 of L [B,N,N,E1] in place), widened to fp64; V [B,N,K] padded.
 * ------------------------------------------------------------------------------------- */
int lnb_graph_eigs_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* node_ptr,
                          const int32_t* edge_ptr, const uint8_t* edges, const double* inv_sqrt_deg, int B,
                          int N, int E, int K, float* D /* [B,K] */, float* V_rows /* [node_ptr[B],K] */,
                          int32_t* status /* [B] */);
int lnb_sym_eigs(lnb_stream_t stream, const float* A, int64_t elem_stride, const int32_t* sizes, int B, int N,
                 int K, float* D /* [B,K] */, float* V /* [B,N,K] */, int32_t* status /* [B] */);

/* ---------------------------------------------------------------------------------------
 * GPNN's graph partition (utils/spectral_graph_partition.py:10-50 as the GPNN collate calls it per
 * padded graph, dataset/qm8.py:123-136) in one launch.  Per graph b:
 *   1. the operator: channel 0 of L read in place, L[((b*N + i)*N + j) * elem_stride].  The fp64 L4
 *      s_i s_j of its off-diagonal non-zero pattern is rebuilt with inv_sqrt_deg [LNB_INV_SQRT_DEG_LEN]
 *      (deg = 1 + the row's count; a node with a zero diagonal is padding and keeps a zero row); if its
 *      fp32 rounding is channel 0 bit for bit that fp64 matrix is decomposed (the matrix the reference hands eigsh),
 *      otherwise the widened fp32 values are and status bit 3 is set;
 *   2. the P eigenvectors of largest |lambda| of the whole padded N x N (the solver of lnb_sym_eigs);
 *      bit 1 when |lambda_P| and |lambda_P+1| are within 1e-9 (the reference's choice is then open);
 *   3. KMeans(n_clusters=P, random_state=seed) as scikit-learn >= 1.4 runs it, in fp64: centring,
 *      k-means++ with T = 2 + floor(ln P) local trials, Lloyd up to 300 iterations (bit 2 when they run
 *      out).  draws [lnb_spectral_partition_draws(P)] are the RandomState(seed) draws the seeding makes:
 *      draws[0] = choice(N, p=ones(N)/N), then uniform(size=T) per further centre;
 *   4. outputs: labels [B,N] int32 canonical (no edge: -1, the other clusters numbered by first
 *      appearance); L_cluster, L_cut [B,N,N] fp32 = the fp64 L4 of the within-cluster and of the cut
 *      part of the pattern (every node keeps its unit self-loop), bit for bit data.partition_operators.
 * status [B]: bit 0 = QL sweeps exhausted, bits 1-3 as above.  One warp per graph for N <= 32, one CTA
 * above; repeated launches are bit-identical; no allocation, no synchronisation (capturable).
 * Envelope: 1 <= N <= LNB_MAX_N, LNB_PARTITION_MIN_P <= P <= LNB_PARTITION_MAX_P, P < N
 * (LNB_ERR_UNSUPPORTED otherwise, nothing launched).
 * lnb_spectral_partition_draws: the draw count for P, 0 outside LNB_PARTITION_MIN_P..LNB_PARTITION_MAX_P.
 * ------------------------------------------------------------------------------------- */
int lnb_spectral_partition_draws(int P);
int lnb_spectral_partition(lnb_stream_t stream, const float* L, int64_t elem_stride, int B, int N, int P,
                           const double* inv_sqrt_deg /* [LNB_INV_SQRT_DEG_LEN] */, const double* draws, int32_t* labels /* [B,N] */,
                           float* L_cluster /* [B,N,N] */, float* L_cut /* [B,N,N] */, int32_t* status /* [B] */);

/* GPNN's graph partition from the sparse records of lnb_graph_prepare_sparse (sizes, edge_ptr, edges;
 * bond types >= E are ignored, E <= LNB_EIGS_MAX_E): steps 2-3 of lnb_spectral_partition on the fp64 L4 that
 * lnb_graph_eigs_sparse builds (padded rows zero, as the dense entry sees the collated channel 0), so
 * labels and status equal lnb_spectral_partition's on the collated L wherever no node pair carries two
 * bond types (status bit 3 is never set).  Outputs: labels, status, and the ELL rows of the two-channel
 * operator [L_cluster, L_cut] (ell_val / ell_idx [B,2,N,N], ell_max [B,2], gext [B,2] = {N, 0}) in the
 * layout and slot order of lnb_graph_prepare over stack([L_cluster, L_cut], 3) with a zero Q, so
 * lnb_gpnn_partition_update reads them as they are; L_cluster / L_cut [B,N,N] when not NULL (both or
 * neither).  Same envelope as lnb_spectral_partition (and 1 <= E <= LNB_EIGS_MAX_E); capturable, no
 * allocation. */
int lnb_spectral_partition_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* edge_ptr,
                                  const uint8_t* edges, const double* inv_sqrt_deg, int B, int N, int E, int P,
                                  const double* draws, int32_t* labels /* [B,N] */, int32_t* status /* [B] */,
                                  float* ell_val, uint8_t* ell_idx, int32_t* ell_max, int32_t* gext,
                                  float* L_cluster /* [B,N,N] or NULL */, float* L_cut /* [B,N,N] or NULL */);

/* GAT's additive attention bias [B,N,N,E1] fp32 from the sparse records (sizes, edge_ptr, edges of
 * lnb_graph_prepare_sparse): bit for bit data.gat_bias of the collated operators, i.e. -0.0 (sign
 * included) on the diagonal of every node (padded ones too) and on every bond of the channel (channel 0:
 * any bond type < E1 - 1, channel e: type e - 1), -1e9 elsewhere.  Envelope: 1 <= N <= LNB_MAX_N,
 * 2 <= E1 <= LNB_MAX_E1 (LNB_ERR_UNSUPPORTED otherwise, nothing launched). */
int lnb_gat_bias_sparse(lnb_stream_t stream, const int32_t* sizes, const int32_t* edge_ptr, const uint8_t* edges,
                        int B, int N, int E1, float* bias /* [B,N,N,E1] */);

/* ---------------------------------------------------------------------------------------
 * The north-star pipeline in ONE launch: operator -> K-step Lanczos with full double
 * re-orthogonalisation (rules of model/ada_lanczos_net.py:139-247) -> implicit-shift QL on (alpha, beta)
 * -> Ritz vectors V = Q S ordered by descending |theta| (utils/data_helper.py:217-223) -- the pair
 * (theta, V) is what utils/data_helper.py:169-226 + dataset/qm8.py:265-291 hand to
 * LanczosNet.forward as (D, V).  q1 is the raw start vector (the randn draw of :161); mask (uint8, may
 * be NULL) zeroes padded nodes.  One group of 32..512 threads per graph; the dense padded operator
 * A [B,N,N] is read from HBM exactly once (its non-zeros are packed into shared memory, exact zeros
 * contribute nothing to A q); the Krylov basis, (alpha, beta) and the QL rotations never leave the
 * SM.  Outputs: T [B,K,K] dense tridiagonal, Q [B,N,K], alpha [B,K], beta [B,K] (beta[b,K-1]=0),
 * idx [B] int32 = number of retained Krylov directions (:208-211).  T, Q may be NULL (not written).
 * theta / ritz_vec / status may be NULL together: then only the tridiagonalisation is produced
 * (AdaLanczosNet).  status[b]: bit 0 = QL sweeps exhausted, bit 1 = the graph's non-zeros did not fit
 * on chip and its rows were streamed per iteration.
 * flags: 0 = the reference's masking rules (idx = min(#valid betas, #real nodes) directions and node
 * rows kept; the alpha of the breakdown step dropped, ada_lanczos_net.py:207-237);
 * LNB_LANCZOS_PROPER = the textbook Krylov factorisation (m = #valid + 1 vectors, T_m with m alphas
 * and m-1 betas, no row masking; idx[b] = m) whose Ritz values are eigenvalues of A -- the mode of
 * the online (D, V) provider.
 * Limits: N <= LNB_LANCZOS_FUSED_MAX_N, K <= LNB_LANCZOS_MAX_K and a basis of K*(N+1) floats within shared memory
 * (LNB_ERR_UNSUPPORTED otherwise, nothing launched).
 * ------------------------------------------------------------------------------------- */
#define LNB_LANCZOS_PROPER 1
int lnb_lanczos_ritz(lnb_stream_t stream, const float* A, const uint8_t* mask, const float* q1,
                     int B, int N, int K, int flags, float* T, float* Q, float* alpha, float* beta,
                     int32_t* idx, float* theta /* [B,K] */, float* ritz_vec /* [B,N,K] */,
                     int32_t* status /* [B] */);

/* ---------------------------------------------------------------------------------------
 * Powers of the tridiagonal for the learned filter (model/ada_lanczos_net.py:262-274):
 *   out[b, r, s, c] = (T_b ** powers[s])[r, c]    (the MLP input layout r*S*K + s*K + c)
 * powers: host pointer to S strictly increasing positive ints, S <= LNB_TRIDIAG_POWERS_MAX_S.
 * ------------------------------------------------------------------------------------- */
int lnb_tridiag_powers(lnb_stream_t stream, const float* T, int B, int K, const int* powers, int S,
                       float* out /* [B,K,S,K] */);

/* ---------------------------------------------------------------------------------------
 * AdaLanczosNet's Lanczos layer for training (the formulation of train._lanczos_train): the K-step
 * recurrence with the reference's rules (cumulative validity from beta >= 1e-4, idx = min(#valid, #real
 * nodes), columns and node rows masked, zero padding to K when N < K) and two classical block Gram-Schmidt
 * passes with the 1/(q_j.q_j + EPS) scaling, in fp32 with a fixed reduction order.  One CTA per graph.
 * lnb_lanczos_tridiag_train writes T [B,K,K], Q [B,N,K], alpha, beta [B,K] and idx [B] (each may be NULL).
 * lnb_lanczos_tridiag_backward recomputes that forward with the same code (T, Q: its recomputed outputs,
 * optional, bit-equal to the training entry's) and writes gA [B,N,N] = d<gT,T> + <gQ,Q> / dA, the exact
 * adjoint of the recurrence with acceptance, idx and masks as data; no atomics (deterministic).
 * mask may be NULL (every node real).  Limits: 1 <= N <= LNB_LANCZOS_TRAIN_MAX_N, 1 <= K <= LNB_LANCZOS_MAX_K
 * (LNB_ERR_UNSUPPORTED otherwise, nothing launched).
 * ------------------------------------------------------------------------------------- */
int lnb_lanczos_tridiag_train(lnb_stream_t stream, const float* A /* [B,N,N] */, const uint8_t* mask,
                              const float* q1 /* [B,N] */, int B, int N, int K, float* T, float* Q,
                              float* alpha, float* beta, int32_t* idx);
int lnb_lanczos_tridiag_backward(lnb_stream_t stream, const float* A, const uint8_t* mask, const float* q1,
                                 int B, int N, int K, const float* gT /* [B,K,K] */,
                                 const float* gQ /* [B,N,K] */, float* gA /* [B,N,N] */, float* T,
                                 float* Q);

/* ---------------------------------------------------------------------------------------
 * Adjoint of lnb_tridiag_powers: gT[b] = d<gOut[b], out[b]>/dT[b] for the function the forward computes,
 * P_1 = T and P_{p+1} = P_p Tri(T) with Tri(T) the three diagonals of T (the forward reads only those).
 * One CTA per graph recomputes P_1 .. P_{pmax-1} in shared memory and runs the reverse sweep, no atomics
 * (deterministic).  Limit: (6 K + (powers[S-1] + 1) K^2) floats within 227 KB of shared memory
 * (LNB_ERR_UNSUPPORTED otherwise, nothing launched); S <= LNB_TRIDIAG_POWERS_MAX_S.
 * ------------------------------------------------------------------------------------- */
int lnb_tridiag_powers_backward(lnb_stream_t stream, const float* T /* [B,K,K] */,
                                const float* gOut /* [B,K,S,K] */, int B, int K, const int* powers, int S,
                                float* gT /* [B,K,K] */);

/* ---------------------------------------------------------------------------------------
 * AdaLanczosNet's Lanczos start vector drawn on the device (the reference draws torch.randn(B, N, 1)
 * on the CPU generator, model/ada_lanczos_net.py:161).  For graph b < B and node n < N (padded nodes
 * included; masking and normalisation stay in the Lanczos kernel):
 *   (x0, x1, x2, x3) = Philox4x32-10 (Random123's constants) at key (seed lo, seed hi) and counter
 *     (n >> 1, b, ctr lo, ctr hi), where (seed, ctr) = start_key[0..1] (int64, DEVICE memory: a captured
 *     graph draws anew when the key changes);
 *   u1 = (fp32(x0) + 1) * 2^-32 and u2 = fp32(x1) * 2^-32 in fp32 (round-to-nearest conversions), so
 *     u1 is in (0, 1];
 *   q1[b, n] = sqrtf(-2 logf(u1)) * (n even ? cos : sin)(2 pi u2), the sine and cosine from
 *     sincospif(2 u2); accurate logf / sincospif, not the fast-math intrinsics.
 * A standard normal per entry (Box-Muller); words x2, x3 are unused.
 * ------------------------------------------------------------------------------------- */
int lnb_ada_start_vector(lnb_stream_t stream, const int64_t* start_key, int B, int N, float* q1 /* [B,N] */);

/* Symmetrised filter blocks (model/ada_lanczos_net.py:275-278):
 *   G[b,s,r,c] = 0.5 * (Y[b, r*K*S + c*S + s] + Y[b, c*K*S + r*S + s])                     */
int lnb_symmetrize_filters(lnb_stream_t stream, const float* Y, int B, int K, int S,
                           float* G /* [B,S,K,K] */);

/* Profiling aid (not used by the product path): register a device buffer of (number of SMs) x 32 uint64 that
 * the wgmma kernels fill with per-CTA clock64 totals per phase; NULL disables. */
int lnb_debug_set_prof(unsigned long long* buf);

/* Testing aid (not used by the product path): n > 0 caps the grid of every persistent wgmma launch
 * (the dense layers, the GRU and LSTM steps, the filter-MLP chain and the convolution stacks) at n
 * CTAs, so that each CTA runs several work items; 0 (the default) removes the cap; n < 0 is
 * LNB_ERR_ARG.  An item's arithmetic does not depend on the CTA that runs it, so the outputs are
 * the same bits under any cap.  Read at launch: a captured graph keeps the grid it was captured
 * with. */
int lnb_debug_set_max_ctas(int n);

#ifdef __cplusplus
}
#endif
#endif /* LANCZOSNET_B200_H_ */
