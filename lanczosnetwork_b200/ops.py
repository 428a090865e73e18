"""torch-tensor front end of the C ABI (include/lanczosnet_b200.h).

PyTorch is plumbing here: device memory, streams, dtype/contiguity checks.  All arithmetic
runs in the hand-written CUDA kernels of liblanczosnet_b200.so.  Every function requires
CUDA tensors and raises otherwise -- there is no CPU path.
"""
import ctypes

import torch

from . import _lib
from ._lib import GemmDesc, SpectralStack

__all__ = [
    'bgemm', 'split_tf32', 'linear_tf32x3', 'linear_tf32x3_grouped', 'graph_prepare', 'tile_assign', 'spectral_conv_fused',
    'graph_prepare_sparse', 'graph_prepare_sparse_features', 'graph_prepare_sparse_packed', 'records_unpack',
    'graph_eigs_sparse', 'sym_eigs',
    'spectral_partition', 'spectral_partition_sparse', 'spectral_partition_supported', 'partition_draws', 'gat_bias_sparse',
    'fused_conv_supported', 'spectral_stack_forward', 'ritz_rowmap', 'ritz_filter_mlp', 'ritz_filter_mlp_supported', 'embedding_rows',
    'ritz_power_table', 'readout',
    'gat_attention', 'gat_attention_supported', 'gat_attention_backward', 'gat_attention_backward_supported',
    'check_dropout_key', 'gat_attention_dropout', 'gat_attention_dropout_backward', 'gat_dropout_project',
    'gat_dropout_project_backward', 'gat_dropout_project_supported',
    'sage_operators', 'sage_sample_sparse', 'neighbour_max', 'sage_lstm_step', 'sage_lstm_step_supported', 'sage_lstm_messages',
    'ggnn_update',
    'ggnn_update_supported', 'gpnn_partition_update', 'gpnn_partition_update_supported', 'mpnn_update', 'mpnn_update_supported', 'mpnn_edge_aggregate',
    'mpnn_edge_aggregate_backward', 'mpnn_edge_aggregate_supported', 'ell_messages', 'ell_messages_adjoint',
    'set2vec', 'set2vec_supported',
    'operator_chain', 'operator_chain_supported', 'graph_messages', 'graph_messages_supported', 'gaussian_laplacian', 'lanczos_ritz', 'tridiag_powers',
    'tridiag_powers_backward', 'tridiag_powers_backward_supported', 'ada_start_vector', 'check_start_key',
    'lanczos_tridiag_train', 'lanczos_tridiag_backward', 'lanczos_tridiag_train_supported', 'symmetrize_filters', 'segment_sum_forward', 'segment_sum_backward', 'launch_count',
]

# The kernels' shape limits: the LNB_* limits of include/lanczosnet_b200.h under the same names without the
# prefix, and SMEM_MAX of csrc/common.cuh.  The *_supported predicates and the argument checks read these.
MAX_N = 128
MAX_N_ELL = 255
MAX_E1 = 16
MAX_WIDTH = 128
PREPARE_MAX_F = 4096
CONV_MAX_K = 32
CONV_MAX_LAYERS = 8
FILTER_MLP_MAX_S = 32
GAT_MAX_WIDTH = 128
GAT_MAX_HEADS = 32
SET2VEC_MAX_P = 128
CHAIN_MAX_N = 32
CHAIN_MAX_STEPS = 64
MESSAGES_MAX_N = 32
MESSAGES_MAX_K = 32
MESSAGES_MAX_S = 8
LANCZOS_FUSED_MAX_N = 1024
LANCZOS_MAX_K = 64
LANCZOS_TRAIN_MAX_N = 128
TRIDIAG_POWERS_MAX_S = 32
EIGS_MAX_K = 128
EIGS_MAX_E = 32
PARTITION_MIN_P = 2
PARTITION_MAX_P = 16
SMEM_MAX = 227 * 1024


def _need_cuda(*tensors):
  for t in tensors:
    if t is None:
      continue
    if not t.is_cuda:
      raise RuntimeError('lanczosnetwork_b200 ops run on CUDA (sm_90a) only; got a %s tensor. '
                         'There is no CPU fallback.' % t.device)


def _f32c(t):
  if t.dtype != torch.float32:
    t = t.float()
  return t.contiguous()


def _ptr(t):
  return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream(t):
  return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _launch(name, on, *args):
  """Runs library entry `name` with `on`'s device current, on that device's current stream (the
  entry's first argument); tensors in `args` are passed as their data pointers, None as NULL, and
  everything else as given.  RuntimeError('<name> failed (status s): <text>') on a non-zero status."""
  with torch.cuda.device(on.device):
    _lib.check(getattr(_lib.load(), name)(
        _stream(on), *[_ptr(a) if a is None or isinstance(a, torch.Tensor) else a for a in args]), name)


def _ints(vals):
  arr = (ctypes.c_int * len(vals))(*[int(v) for v in vals])
  return arr


def launch_count():
  return _lib.launch_count()


# --------------------------------------------------------------------------------------------
def bgemm(A, a_str, Bm, b_str, C, c_str, batch, nz, M, N, K, kscale=None, s_str=(0, 0, 0),
          bias=None, bias_sz=0, relu=False, a_off=0, b_off=0, c_off=0, alpha=1.0, addend=None,
          add_str=(0, 0, 0, 0), add_off=0, beta=0.0):
  """C[b,z] = act(alpha * (A[b,z] * kscale[b,z]) @ B[b,z] + beta * addend[b,z] + bias); strides in
  elements, *_off element offsets into the (fp32, CUDA) storage of A / B / C / addend."""
  _need_cuda(A, Bm, C, kscale, bias)
  d = GemmDesc()
  d.A = A.data_ptr() + 4 * a_off
  d.a_sb, d.a_sz, d.a_sm, d.a_sk = [int(v) for v in a_str]
  d.B = Bm.data_ptr() + 4 * b_off
  d.b_sb, d.b_sz, d.b_sk, d.b_sn = [int(v) for v in b_str]
  d.C = C.data_ptr() + 4 * c_off
  d.c_sb, d.c_sz, d.c_sm, d.c_sn = [int(v) for v in c_str]
  d.kscale = kscale.data_ptr() if kscale is not None else None
  d.s_sb, d.s_sz, d.s_sk = [int(v) for v in s_str]
  d.bias = bias.data_ptr() if bias is not None else None
  d.bias_sz = int(bias_sz)
  d.batch, d.nz, d.M, d.N, d.K, d.relu = int(batch), int(nz), int(M), int(N), int(K), int(bool(relu))
  d.alpha, d.beta = float(alpha), float(beta)
  d.addend = addend.data_ptr() + 4 * add_off if addend is not None else None
  d.d_sb, d.d_sz, d.d_sm, d.d_sn = [int(v) for v in add_str]
  _launch('lnb_batched_gemm', C, ctypes.byref(d))
  return C


def split_tf32(x):
  """(hi, lo) tf32 split of an fp32 tensor: hi = rna_tf32(x), lo = rna_tf32(x - hi)."""
  _need_cuda(x)
  x = _f32c(x)
  hi = torch.empty_like(x)
  lo = torch.empty_like(x)
  _launch('lnb_split_tf32', x, x, x.numel(), hi, lo)
  return hi, lo


def linear_tf32x3(x, w_hi, w_lo, bias=None, relu=False, out=None):
  """act(x @ W^T + bias) on the tensor cores (wgmma, 3xTF32).  x [M,K], w_hi/w_lo [N,K]; ``out``, when
  given, must be a contiguous float32 [M,N] tensor on x's device."""
  _need_cuda(x, w_hi, w_lo, bias)
  x = _f32c(x)
  M, K = x.shape
  N = w_hi.shape[0]
  if out is None:
    out = torch.empty((M, N), device=x.device, dtype=torch.float32)
  elif (out.dtype != torch.float32 or tuple(out.shape) != (M, N) or not out.is_contiguous() or
        out.device != x.device):
    raise ValueError('linear_tf32x3: out must be a contiguous float32 [%d, %d] tensor on %s; got %s %s%s on %s'
                     % (M, N, x.device, out.dtype, tuple(out.shape),
                        '' if out.is_contiguous() else ' (not contiguous)', out.device))
  tiles = ((M + 127) // 128) * ((N + 127) // 128)
  nkb = (K + 31) // 32
  splits = 1
  if tiles * 2 <= _sm_count(x.device) and nkb >= 32:
    # few output tiles, deep K (the Ada filter MLP): split K so every SM streams weights
    splits = min(_sm_count(x.device) // tiles, 8, nkb // 16)
    while splits > 1 and ((nkb + splits - 1) // splits) * (splits - 1) >= nkb:
      splits -= 1
  if splits > 1:
    ws, counters = _splitk_workspace(x.device, tiles * splits * 128 * 128, tiles)
    _launch('lnb_linear_tf32x3_splitk', x, x, w_hi, w_lo, bias, M, N, K, int(bool(relu)), out, splits, ws,
            counters)
  else:
    _launch('lnb_linear_tf32x3', x, x, w_hi, w_lo, bias, M, N, K, int(bool(relu)), out)
  return out


_SPLITK_WS = {}
_SM_COUNT = {}


def _sm_count(device):
  idx = device.index if device.index is not None else torch.cuda.current_device()
  if idx not in _SM_COUNT:
    _SM_COUNT[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
  return _SM_COUNT[idx]


def _splitk_workspace(device, nfloats, ntiles):
  """Split-K scratch of the current stream on ``device``: partial tiles + per-tile arrival counters
  (zero between launches; launches on one stream are ordered, so one pair per device and stream is
  enough).  linear_tf32x3 never asks for more than tiles * splits <= SM count partial tiles, so the
  pair is allocated once at that size and never replaced: it lives as long as the process, because
  a captured CUDA graph binds its pointers.  Graphs captured on the same stream share it, so their
  replays must not run concurrently with each other or with launches on that stream."""
  key = (device.index, torch.cuda.current_stream(device).cuda_stream)
  pair = _SPLITK_WS.get(key)
  if pair is None:
    sms = _sm_count(device)
    pair = (torch.empty((sms * 128 * 128,), device=device, dtype=torch.float32),
            torch.zeros((max(sms, 256),), device=device, dtype=torch.int32))
    _SPLITK_WS[key] = pair
  ws, counters = pair
  assert nfloats <= ws.numel() and ntiles <= counters.numel(), (nfloats, ws.numel(), ntiles)
  return pair


def linear_tf32x3_grouped(x, w_hi, w_lo, bias, groups, relu=False):
  """Block-diagonal layer: out[:, g*N:(g+1)*N] = act(x[:, g*K:(g+1)*K] @ W_g^T + b_g) with
  x [M, groups*K], w_hi/w_lo [groups*N, K] (stacked), bias [groups*N]."""
  _need_cuda(x, w_hi, w_lo, bias)
  x = _f32c(x)
  M = x.shape[0]
  K = w_hi.shape[1]
  N = w_hi.shape[0] // groups
  assert x.shape[1] == groups * K and w_hi.shape[0] == groups * N
  out = torch.empty((M, groups * N), device=x.device, dtype=torch.float32)
  _launch('lnb_linear_tf32x3_grouped', x, x, w_hi, w_lo, bias, M, groups, N, K, int(bool(relu)), out)
  return out


class GraphPrep(tuple):
  """(ell_val, ell_idx, ell_max, gext, tiles) plus the compact Ritz row list of the same pass
  (attributes rowmap [B*K] int32, nrows [1] int32; see ritz_rowmap).  tiles_pending: built with
  defer_tiles, ``tiles`` is written by tile_assign."""
  rowmap = None
  nrows = None
  tiles_pending = False


def tile_assign(prep, K):
  """Writes the tile table and schedule of a GraphPrep built with defer_tiles (lnb_tile_assign) on
  the current stream; they equal what graph_prepare without defer_tiles writes."""
  gext, tiles = prep[3], prep[4]
  _launch('lnb_tile_assign', gext, gext, gext.shape[0], int(K), tiles)
  prep.tiles_pending = False


PREP_DEFER_TILES = 4    # LNB_PREP_DEFER_TILES
PACKED_HOST_TILES = 2   # LNB_PACKED_HOST_TILES


def graph_prepare(L, Q=None, binarize=False, defer_tiles=False):
  """Per-forward compression of the dense operators L [B,N,N,E1] (ELL rows), the real extents
  of every graph, the packed-tile assignment for the fused convolution kernel and the compact
  list of non-zero Ritz rows.  ``Q=None``: no Ritz vectors, an all-zero [B,N,4] block, so the
  extents come from L alone.  ``defer_tiles``: leave the tile assignment to tile_assign, which may
  run on another stream.  Returns GraphPrep(ell_val, ell_idx, ell_max, gext, tiles)."""
  if Q is None:
    Q = torch.zeros((L.shape[0], L.shape[1], 4), device=L.device, dtype=torch.float32)
  _need_cuda(L, Q)
  L, Q = _f32c(L), _f32c(Q)
  B, N, _, E1 = L.shape
  K = Q.shape[2]
  dev = L.device
  ell_val = torch.empty((B, E1, N, N), device=dev, dtype=torch.float32)
  ell_idx = torch.empty((B, E1, N, N), device=dev, dtype=torch.uint8)
  ell_max = torch.empty((B, E1), device=dev, dtype=torch.int32)
  gext = torch.empty((B, 2), device=dev, dtype=torch.int32)
  tiles = torch.empty((4 * B + 2,), device=dev, dtype=torch.int32)   # tile table + scratch
  rowmap = torch.empty((B * K,), device=dev, dtype=torch.int32)
  nrows = torch.empty((1,), device=dev, dtype=torch.int32)
  _launch('lnb_graph_prepare', L, L, Q, B, N, E1, K, ell_val, ell_idx, ell_max, gext, tiles, rowmap, nrows,
          (1 if binarize else 0) | (PREP_DEFER_TILES if defer_tiles else 0))
  prep = GraphPrep((ell_val, ell_idx, ell_max, gext, tiles))
  prep.rowmap, prep.nrows, prep.tiles_pending = rowmap, nrows, bool(defer_tiles) and B > 0
  return prep


_INV_SQRT_DEG = {}
# LNB_INV_SQRT_DEG_LEN: every simple-graph degree of the sparse producers' envelope, up to 1 + 32 * 128
INV_SQRT_DEG_LEN = 4098


def _inv_sqrt_deg_table(device):
  """deg^-1/2 in fp64 for deg = 0 .. INV_SQRT_DEG_LEN - 1 exactly as the reference's host code computes it
  (np.power(deg, -0.5) with inf -> 0, utils/data_helper.py:104-107), cached per device."""
  key = device.index if device.index is not None else torch.cuda.current_device()
  if key not in _INV_SQRT_DEG:
    import numpy as np
    deg = np.arange(INV_SQRT_DEG_LEN, dtype=np.float64)
    with np.errstate(divide='ignore'):
      t = np.power(deg, -0.5)
    t[np.isinf(t)] = 0.0
    _INV_SQRT_DEG[key] = torch.from_numpy(t).to(device)
  return _INV_SQRT_DEG[key]


def graph_prepare_sparse(sizes, node_ptr, node_feat, edge_ptr, edges, V_rows, N, E1, binarize=False,
                         want_dense=False, defer_tiles=False):
  """GPU-side batch construction from sparse records (see lnb_graph_prepare_sparse); defer_tiles
  as in graph_prepare.
  sizes [B] int32, node_ptr [B+1] int32, node_feat [>= node_ptr[B]] int32, edge_ptr [B+1] int32,
  edges [>= edge_ptr[B], 4] uint8, V_rows [>= node_ptr[B], K] fp32 -- all CUDA.
  Returns (GraphPrep, node_ids [B,N] int64, mask [B,N] uint8, V [B,N,K], L [B,N,N,E1] or None)."""
  _need_cuda(sizes, node_ptr, node_feat, edge_ptr, edges, V_rows)
  dev = sizes.device
  B = sizes.shape[0]
  K = V_rows.shape[1]
  assert sizes.dtype == torch.int32 and node_ptr.dtype == torch.int32 and node_feat.dtype == torch.int32
  assert edge_ptr.dtype == torch.int32 and edges.dtype == torch.uint8 and edges.shape[1] == 4
  assert V_rows.dtype == torch.float32 and V_rows.is_contiguous() and edges.is_contiguous()
  ell_val = torch.empty((B, E1, N, N), device=dev, dtype=torch.float32)
  ell_idx = torch.empty((B, E1, N, N), device=dev, dtype=torch.uint8)
  ell_max = torch.empty((B, E1), device=dev, dtype=torch.int32)
  gext = torch.empty((B, 2), device=dev, dtype=torch.int32)
  tiles = torch.empty((4 * B + 2,), device=dev, dtype=torch.int32)
  rowmap = torch.empty((B * K,), device=dev, dtype=torch.int32)
  nrows = torch.empty((1,), device=dev, dtype=torch.int32)
  node_ids = torch.empty((B, N), device=dev, dtype=torch.int64)
  mask = torch.empty((B, N), device=dev, dtype=torch.uint8)
  V = torch.empty((B, N, K), device=dev, dtype=torch.float32)
  L = torch.empty((B, N, N, E1), device=dev, dtype=torch.float32) if want_dense else None
  _launch('lnb_graph_prepare_sparse', sizes, sizes, node_ptr, node_feat, edge_ptr, edges, V_rows,
          _inv_sqrt_deg_table(dev), B, int(N), int(E1), int(K),
          (1 if binarize else 0) | (PREP_DEFER_TILES if defer_tiles else 0), ell_val, ell_idx, ell_max, gext, tiles,
          rowmap, nrows, node_ids, mask, V, L)
  prep = GraphPrep((ell_val, ell_idx, ell_max, gext, tiles))
  prep.rowmap, prep.nrows, prep.tiles_pending = rowmap, nrows, bool(defer_tiles) and B > 0
  return prep, node_ids, mask, V, L


def graph_prepare_sparse_features(sizes, node_ptr, node_x, edge_ptr, edges, V_rows, N, E1, binarize=False,
                                  want_dense=False, defer_tiles=False):
  """graph_prepare_sparse for records with float node features (lnb_graph_prepare_sparse_features):
  node_x [>= node_ptr[B], F] float32 holds the feature rows of the real nodes instead of atom ids, and the
  padded features X [B,N,F] (real rows bit for bit, padded rows 0) come back instead of node ids.
  1 <= F <= PREPARE_MAX_F.  Returns (GraphPrep, X [B,N,F], mask [B,N] uint8, V [B,N,K], L [B,N,N,E1] or None)."""
  for name, t in (('sizes', sizes), ('node_ptr', node_ptr), ('edge_ptr', edge_ptr)):
    if t.dtype != torch.int32:
      raise ValueError('graph_prepare_sparse_features: %s must be int32; got %s' % (name, t.dtype))
  if node_x.dtype != torch.float32 or node_x.dim() != 2 or not node_x.is_contiguous():
    raise ValueError('graph_prepare_sparse_features: node_x must be a contiguous float32 [rows, F] tensor; got '
                     '%s %s' % (node_x.dtype, tuple(node_x.shape)))
  if edges.dtype != torch.uint8 or edges.dim() != 2 or edges.shape[1] != 4 or not edges.is_contiguous():
    raise ValueError('graph_prepare_sparse_features: edges must be contiguous uint8 [E, 4]')
  if V_rows.dtype != torch.float32 or V_rows.dim() != 2 or not V_rows.is_contiguous():
    raise ValueError('graph_prepare_sparse_features: V_rows must be a contiguous float32 [rows, K] tensor')
  F = int(node_x.shape[1])
  if not (1 <= int(N) <= MAX_N and 2 <= int(E1) <= MAX_E1 and 1 <= F <= PREPARE_MAX_F):
    raise ValueError('graph_prepare_sparse_features: N=%d, E1=%d, F=%d outside 1 <= N <= %d, 2 <= E1 <= %d, '
                     '1 <= F <= %d' % (int(N), int(E1), F, MAX_N, MAX_E1, PREPARE_MAX_F))
  _need_cuda(sizes, node_ptr, node_x, edge_ptr, edges, V_rows)
  dev = sizes.device
  B = sizes.shape[0]
  K = V_rows.shape[1]
  ell_val = torch.empty((B, E1, N, N), device=dev, dtype=torch.float32)
  ell_idx = torch.empty((B, E1, N, N), device=dev, dtype=torch.uint8)
  ell_max = torch.empty((B, E1), device=dev, dtype=torch.int32)
  gext = torch.empty((B, 2), device=dev, dtype=torch.int32)
  tiles = torch.empty((4 * B + 2,), device=dev, dtype=torch.int32)
  rowmap = torch.empty((B * K,), device=dev, dtype=torch.int32)
  nrows = torch.empty((1,), device=dev, dtype=torch.int32)
  X = torch.empty((B, N, F), device=dev, dtype=torch.float32)
  mask = torch.empty((B, N), device=dev, dtype=torch.uint8)
  V = torch.empty((B, N, K), device=dev, dtype=torch.float32)
  L = torch.empty((B, N, N, E1), device=dev, dtype=torch.float32) if want_dense else None
  _launch('lnb_graph_prepare_sparse_features', sizes, sizes, node_ptr, node_x, edge_ptr, edges, V_rows,
          _inv_sqrt_deg_table(dev), B, int(N), int(E1), int(K), F,
          (1 if binarize else 0) | (PREP_DEFER_TILES if defer_tiles else 0), ell_val, ell_idx, ell_max, gext, tiles,
          rowmap, nrows, X, mask, V, L)
  prep = GraphPrep((ell_val, ell_idx, ell_max, gext, tiles))
  prep.rowmap, prep.nrows, prep.tiles_pending = rowmap, nrows, bool(defer_tiles) and B > 0
  return prep, X, mask, V, L


def graph_prepare_sparse_packed(blob, B, N, E1, K, binarize=False, want_dense=False, host_tiles=True,
                                feature_dim=0):
  """graph_prepare_sparse on a packed batch (data.pack_sparse: one contiguous uint8 buffer, see
  lnb_graph_prepare_sparse_packed).  host_tiles: the batch carries the tile table and the Ritz-row
  prefix sums (data.pack_sparse always writes them), so no tile-assignment kernel is launched and the
  stack kernel reads the table in place.  Returns (GraphPrep, node_ids, mask, V, L or None).

  ``feature_dim`` = F > 0: a batch of float feature rows (header slot F, lnb_graph_prepare_sparse_features_packed)
  whose padded features X [B,N,F] come back in place of node_ids; a batch of another F gives B empty graphs."""
  _need_cuda(blob)
  assert blob.dtype == torch.uint8 and blob.is_contiguous()
  F = int(feature_dim)
  if not 0 <= F <= PREPARE_MAX_F:
    raise ValueError('graph_prepare_sparse_packed: feature_dim=%d outside [0, %d]' % (F, PREPARE_MAX_F))
  dev = blob.device
  ell_val = torch.empty((B, E1, N, N), device=dev, dtype=torch.float32)
  ell_idx = torch.empty((B, E1, N, N), device=dev, dtype=torch.uint8)
  ell_max = torch.empty((B, E1), device=dev, dtype=torch.int32)
  gext = torch.empty((B, 2), device=dev, dtype=torch.int32)
  if host_tiles:
    from .data import packed_offsets, tile_segment_ints
    off_tiles = packed_offsets(B, K).tiles
    # the next-fit table and, behind it, the tile schedule the stack kernel runs
    tiles = blob[off_tiles:off_tiles + 4 * tile_segment_ints(B)].view(torch.int32)
  else:
    tiles = torch.empty((4 * B + 2,), device=dev, dtype=torch.int32)
  rowmap = torch.empty((B * K,), device=dev, dtype=torch.int32)
  nrows = torch.empty((1,), device=dev, dtype=torch.int32)
  mask = torch.empty((B, N), device=dev, dtype=torch.uint8)
  V = torch.empty((B, N, K), device=dev, dtype=torch.float32)
  L = torch.empty((B, N, N, E1), device=dev, dtype=torch.float32) if want_dense else None
  flags = (1 if binarize else 0) | (PACKED_HOST_TILES if host_tiles else 0)
  if F:
    x = torch.empty((B, N, F), device=dev, dtype=torch.float32)
    _launch('lnb_graph_prepare_sparse_features_packed', blob, blob, _inv_sqrt_deg_table(dev), int(B), int(N),
            int(E1), int(K), F, flags, ell_val, ell_idx, ell_max, gext, tiles, rowmap, nrows, x, mask, V, L)
  else:
    x = torch.empty((B, N), device=dev, dtype=torch.int64)
    _launch('lnb_graph_prepare_sparse_packed', blob, blob, _inv_sqrt_deg_table(dev), int(B), int(N), int(E1), int(K),
            flags, ell_val, ell_idx, ell_max, gext, tiles, rowmap, nrows, x, mask, V, L)
  prep = GraphPrep((ell_val, ell_idx, ell_max, gext, tiles))
  prep.rowmap, prep.nrows = rowmap, nrows
  return prep, x, mask, V, L


def records_unpack(blob, B, K, cap_rows, cap_edges, eigs=False, label_dim=0, feature_dim=0):
  """A packed batch (data.pack_sparse / data.PackedMolecules: a 16-byte aligned uint8 CUDA buffer) split
  into the records of data.sparse_collate by lnb_records_unpack, one launch whose segment offsets come from
  the header on the device.  cap_rows / cap_edges: rows of node_feat / edges (at least node_ptr[B] /
  edge_ptr[B]; rows past those stay unwritten).  eigs: also unpack D and V_rows (the batch must carry them).
  A malformed header or an overflow is reported in ``status`` (see the C header), with every graph empty.
  Returns (sizes [B], node_ptr [B+1], node_feat [cap_rows], edge_ptr [B+1], edges [cap_edges, 4], D [B, K]
  or None, V_rows [cap_rows, K] or None, status [1] int32).

  ``label_dim`` = P > 0: also unpack the batch's labels (data.pack_sparse(..., label=True)) through
  lnb_records_unpack_labels, in the same launch; a batch without them, or with another P, sets status bit 64.
  Returns (sizes, node_ptr, node_feat, edge_ptr, edges, D, V_rows, label [B, P] float32, status).

  ``feature_dim`` = F > 0: a batch of float feature rows (header slot F), through lnb_records_unpack_features;
  node_feat is then float32 [cap_rows, F], and labels come as above.  A header whose F differs from the
  caller's (F = 0 for atom ids) sets status bit 128, with every graph empty."""
  _need_cuda(blob)
  if blob.dtype != torch.uint8 or blob.dim() != 1 or not blob.is_contiguous() or blob.numel() < 64:
    raise ValueError('records_unpack: blob must be a contiguous 1-D uint8 tensor of >= 64 bytes')
  if blob.data_ptr() % 16:
    raise ValueError('records_unpack: blob must be 16-byte aligned')
  B, K, cap_rows, cap_edges, P, F = int(B), int(K), int(cap_rows), int(cap_edges), int(label_dim), int(feature_dim)
  if B < 1 or K < 1 or cap_rows < 0 or cap_edges < 0 or P < 0 or not 0 <= F <= PREPARE_MAX_F:
    raise ValueError('records_unpack: B=%d, K=%d, cap_rows=%d, cap_edges=%d, label_dim=%d, feature_dim=%d'
                     % (B, K, cap_rows, cap_edges, P, F))
  dev = blob.device
  i32 = dict(device=dev, dtype=torch.int32)
  sizes, node_ptr, edge_ptr = torch.empty((B,), **i32), torch.empty((B + 1,), **i32), torch.empty((B + 1,), **i32)
  node_feat = (torch.empty((cap_rows, F), device=dev, dtype=torch.float32) if F else
               torch.empty((cap_rows,), **i32))
  edges = torch.empty((cap_edges, 4), device=dev, dtype=torch.uint8)
  D = torch.empty((B, K), device=dev, dtype=torch.float32) if eigs else None
  V_rows = torch.empty((cap_rows, K), device=dev, dtype=torch.float32) if eigs else None
  status = torch.empty((1,), **i32)
  label = torch.empty((B, P), device=dev, dtype=torch.float32) if P else None
  if F:
    _launch('lnb_records_unpack_features', blob, blob, blob.numel(), B, K, F, cap_rows, cap_edges, sizes, node_ptr,
            node_feat, edge_ptr, edges, D, V_rows, status, P, label)
    out = (sizes, node_ptr, node_feat, edge_ptr, edges, D, V_rows)
    return out + ((label, status) if P else (status,))
  args = (blob, blob.numel(), B, K, cap_rows, cap_edges, sizes, node_ptr, node_feat, edge_ptr, edges, D, V_rows,
          status)
  if not P:
    _launch('lnb_records_unpack', blob, *args)
    return sizes, node_ptr, node_feat, edge_ptr, edges, D, V_rows, status
  _launch('lnb_records_unpack_labels', blob, *args, P, label)
  return sizes, node_ptr, node_feat, edge_ptr, edges, D, V_rows, label, status


def graph_eigs_sparse(sizes, node_ptr, edge_ptr, edges, N, K, num_edgetype=32, rows=None):
  """Exact eigenpairs of every molecule's simple-graph L4 from its bond list (lnb_graph_eigs_sparse):
  what the reference's preprocessing computes with fp64 eigh, truncated / zero padded to K.
  sizes [B], node_ptr [B+1], edge_ptr [B+1] int32, edges [>= edge_ptr[B], 4] uint8 -- all CUDA, the
  records of data.sparse_collate; bonds of type >= num_edgetype are ignored.  ``rows``: row count of
  V_rows, at least node_ptr[B] (default: node_ptr[B], read from the device; rows past it stay unwritten).
  Returns (D [B,K], V_rows [rows, K] in sparse_collate's layout, status [B] int32)."""
  _need_cuda(sizes, node_ptr, edge_ptr, edges)
  assert sizes.dtype == torch.int32 and node_ptr.dtype == torch.int32 and edge_ptr.dtype == torch.int32
  assert edges.dtype == torch.uint8 and edges.shape[1] == 4 and edges.is_contiguous()
  dev = sizes.device
  B = sizes.shape[0]
  if rows is None:
    rows = int(node_ptr[-1]) if B else 0
  D = torch.empty((B, int(K)), device=dev, dtype=torch.float32)
  V_rows = torch.empty((int(rows), int(K)), device=dev, dtype=torch.float32)
  status = torch.empty((B,), device=dev, dtype=torch.int32)
  _launch('lnb_graph_eigs_sparse', sizes, sizes, node_ptr, edge_ptr, edges, _inv_sqrt_deg_table(dev),
          B, int(N), int(num_edgetype), int(K), D, V_rows, status)
  return D, V_rows, status


def sym_eigs(A, sizes, K):
  """Exact eigenpairs of the leading sizes[b] x sizes[b] block of every symmetric operator (lnb_sym_eigs),
  ordered and padded like the reference's preprocessing.  A: [B,N,N] or [B,N,N,E1] (channel 0 is read
  in place); sizes [B] (any integer dtype).  Returns (D [B,K], V [B,N,K], status [B] int32)."""
  _need_cuda(A, sizes)
  if A.dim() == 4:
    A = A[..., 0]
  if A.dtype != torch.float32:
    A = A.float()
  B, N = A.shape[0], A.shape[1]
  es = A.stride(2)
  if es < 1 or tuple(A.stride()) != (N * N * es, N * es, es):
    A, es = A.contiguous(), 1
  sizes = sizes.to(torch.int32).contiguous()
  D = torch.empty((B, int(K)), device=A.device, dtype=torch.float32)
  V = torch.empty((B, N, int(K)), device=A.device, dtype=torch.float32)
  status = torch.empty((B,), device=A.device, dtype=torch.int32)
  _launch('lnb_sym_eigs', A, A, int(es), sizes, B, N, int(K), D, V, status)
  return D, V, status


def partition_draws(N, P, seed=1234):
  """The draws scikit-learn's k-means++ seeding takes from a fresh ``RandomState(seed)`` for N points and
  P clusters, as one fp64 numpy array: ``choice(N, p=ones(N)/N)``, then ``uniform(size=2 + int(log P))``
  per further centre.  They depend on (N, P, seed) only."""
  import numpy as np
  rs = np.random.RandomState(seed)
  T = 2 + int(np.log(P))
  out = [float(rs.choice(N, p=np.ones(N) / N))]
  for _ in range(P - 1):
    out.extend(rs.uniform(size=T).tolist())
  return np.asarray(out, dtype=np.float64)


_PARTITION_DRAWS = {}


def _partition_draws_table(device, N, P, seed):
  """partition_draws on ``device``, cached per (device, N, P, seed); the first call for a key copies the
  table from the host, so it has to happen outside a CUDA-graph capture (a model's warm-up run does)."""
  key = (device.index if device.index is not None else torch.cuda.current_device(), int(N), int(P), int(seed))
  if key not in _PARTITION_DRAWS:
    if torch.cuda.is_current_stream_capturing():
      raise RuntimeError('spectral_partition: the k-means++ draw table for N=%d, P=%d, seed=%d is built on '
                         'the host; call spectral_partition once outside the capture' % (N, P, seed))
    _PARTITION_DRAWS[key] = torch.from_numpy(partition_draws(N, P, seed)).to(device)
  return _PARTITION_DRAWS[key]


def spectral_partition(L, num_partition, seed=1234):
  """GPNN's graph partition of every padded graph on the device (lnb_spectral_partition): the reference's
  ``spectral_clustering(L, num_partition, seed)`` (the P eigenvectors of largest |lambda| of the whole padded
  simple-graph operator, then KMeans as scikit-learn >= 1.4 runs it) and ``get_L_cluster_cut``.
  L: [B,N,N,E1] (channel 0 is read in place) or [B,N,N], float32, CUDA.
  Returns (labels [B,N] int32 canonical: -1 for nodes without an edge, the other clusters numbered by
  first appearance; L_cluster [B,N,N]; L_cut [B,N,N]; status [B] int32: bit 0 QL sweeps exhausted, bit 1
  |lambda| tie at the cut, bit 2 Lloyd reached 300 iterations, bit 3 operator not an unweighted L4)."""
  if L.dim() not in (3, 4) or L.shape[1] != L.shape[2]:
    raise ValueError('spectral_partition: L must be [B,N,N] or [B,N,N,E1]; got %s' % (tuple(L.shape),))
  P, N = int(num_partition), int(L.shape[1])
  assert P < N - 1, 'spectral_partition: num_partition=%d needs more than %d nodes (N=%d)' % (P, P + 1, N)
  if not (PARTITION_MIN_P <= P <= PARTITION_MAX_P) or N > MAX_N:
    raise ValueError('spectral_partition: N=%d, num_partition=%d outside N <= %d, %d <= num_partition <= %d'
                     % (N, P, MAX_N, PARTITION_MIN_P, PARTITION_MAX_P))
  _need_cuda(L)
  A = L[..., 0] if L.dim() == 4 else L
  if A.dtype != torch.float32:
    A = A.float()
  B = A.shape[0]
  es = A.stride(2)
  if es < 1 or tuple(A.stride()) != (N * N * es, N * es, es):
    A, es = A.contiguous(), 1
  dev = A.device
  labels = torch.empty((B, N), device=dev, dtype=torch.int32)
  L_cluster = torch.empty((B, N, N), device=dev, dtype=torch.float32)
  L_cut = torch.empty((B, N, N), device=dev, dtype=torch.float32)
  status = torch.empty((B,), device=dev, dtype=torch.int32)
  draws = _partition_draws_table(dev, N, P, seed)
  _launch('lnb_spectral_partition', A, A, int(es), B, N, P, _inv_sqrt_deg_table(dev), draws, labels, L_cluster, L_cut,
          status)
  return labels, L_cluster, L_cut, status


def _check_records(who, sizes, edge_ptr, edges):
  _need_cuda(sizes, edge_ptr, edges)
  if sizes.dtype != torch.int32 or edge_ptr.dtype != torch.int32 or edge_ptr.shape[0] != sizes.shape[0] + 1:
    raise ValueError('%s: sizes [B] and edge_ptr [B+1] must be int32' % who)
  if edges.dtype != torch.uint8 or edges.dim() != 2 or edges.shape[1] != 4 or not edges.is_contiguous():
    raise ValueError('%s: edges must be a contiguous uint8 [E, 4] tensor' % who)


def spectral_partition_supported(N, num_partition):
  """The envelope of spectral_partition and spectral_partition_sparse: N <= MAX_N,
  PARTITION_MIN_P <= P <= PARTITION_MAX_P, P < N - 1."""
  P, N = int(num_partition), int(N)
  # the kernels take P < N; P < N - 1 is the reference's own assertion in spectral_clustering
  # (utils/spectral_graph_partition.py), so only partitions the reference can compute are accepted
  return PARTITION_MIN_P <= P <= PARTITION_MAX_P and 1 <= N <= MAX_N and P < N - 1


def spectral_partition_sparse(sizes, edge_ptr, edges, N, num_partition, num_edgetype, seed=1234,
                              want_dense=False):
  """spectral_partition from the sparse records of data.sparse_collate (lnb_spectral_partition_sparse):
  the same partition of every graph padded to N, without the padded operators.  Bond types >=
  num_edgetype are ignored.  Where no node pair carries two bond types, labels and status equal
  spectral_partition's on the collated L (status bit 3 is never set).
  Returns (labels [B,N] int32, status [B] int32, GraphPrep of the two-channel operator
  [L_cluster, L_cut] -- the ELL rows, ell_max and gext that graph_prepare(stack([L_cluster, L_cut], 3))
  writes, no tile table --, L_cluster, L_cut [B,N,N] when want_dense, else None)."""
  P, N, E = int(num_partition), int(N), int(num_edgetype)
  if not spectral_partition_supported(N, P):
    raise ValueError('spectral_partition_sparse: N=%d, num_partition=%d outside N <= %d, %d <= num_partition <= %d, '
                     'num_partition < N - 1' % (N, P, MAX_N, PARTITION_MIN_P, PARTITION_MAX_P))
  if not 1 <= E <= EIGS_MAX_E:
    raise ValueError('spectral_partition_sparse: num_edgetype=%d outside 1..%d' % (E, EIGS_MAX_E))
  _check_records('spectral_partition_sparse', sizes, edge_ptr, edges)
  dev = sizes.device
  B = sizes.shape[0]
  labels = torch.empty((B, N), device=dev, dtype=torch.int32)
  status = torch.empty((B,), device=dev, dtype=torch.int32)
  ell_val = torch.empty((B, 2, N, N), device=dev, dtype=torch.float32)
  ell_idx = torch.empty((B, 2, N, N), device=dev, dtype=torch.uint8)
  ell_max = torch.empty((B, 2), device=dev, dtype=torch.int32)
  gext = torch.empty((B, 2), device=dev, dtype=torch.int32)
  L_cluster = torch.empty((B, N, N), device=dev, dtype=torch.float32) if want_dense else None
  L_cut = torch.empty((B, N, N), device=dev, dtype=torch.float32) if want_dense else None
  draws = _partition_draws_table(dev, N, P, seed)
  _launch('lnb_spectral_partition_sparse', sizes, sizes, edge_ptr, edges, _inv_sqrt_deg_table(dev), B, N, E, P, draws,
          labels, status, ell_val, ell_idx, ell_max, gext, L_cluster, L_cut)
  return labels, status, GraphPrep((ell_val, ell_idx, ell_max, gext, None)), L_cluster, L_cut


def gat_bias_sparse(sizes, edge_ptr, edges, N, E1):
  """GAT's additive attention bias [B,N,N,E1] fp32 from the sparse records (lnb_gat_bias_sparse): bit for
  bit data.gat_bias of the collated operators (-0.0 on the diagonal and on the channel's bonds, -1e9
  elsewhere)."""
  N, E1 = int(N), int(E1)
  if not (1 <= N <= MAX_N and 2 <= E1 <= MAX_E1):
    raise ValueError('gat_bias_sparse: N=%d, E1=%d outside 1 <= N <= %d, 2 <= E1 <= %d' % (N, E1, MAX_N, MAX_E1))
  _check_records('gat_bias_sparse', sizes, edge_ptr, edges)
  B = sizes.shape[0]
  bias = torch.empty((B, N, N, E1), device=sizes.device, dtype=torch.float32)
  _launch('lnb_gat_bias_sparse', sizes, sizes, edge_ptr, edges, B, N, E1, bias)
  return bias


def fused_conv_supported(N, Din, K, H, n_short, dense_filter, S=8, E1=7):
  """Shapes the fused wgmma convolution kernel handles (others use the unfused ops);
  mirrors the checks of lnb_spectral_conv_fused."""
  if (n_short or dense_filter or N > MAX_N or Din % 32 or K > CONV_MAX_K or K % 4 or H % 4 or H > MAX_WIDTH or
      E1 > MAX_E1):
    return False
  smem = 4 * 32768 + 256 + 1024 + 128 * (max(Din, H) + 4) * 4 + 128 * K * 4 + 4096
  return smem <= SMEM_MAX


def spectral_conv_fused(X, Q, coeff, prep, w_hi, w_lo, bias, relu=True, write_pad=True):
  """One fused spectral convolution layer: X [B,N,Din], Q [B,N,K], coeff [B,K,S] diagonal
  filter coefficients (None when there are no long scales), prep = graph_prepare(L, Q),
  W [H, (S+E1)*Din] split -> [B,N,H].  write_pad=False leaves the rows of padded nodes
  unwritten (fine between layers: nothing reads them)."""
  _need_cuda(X, Q, coeff, w_hi, w_lo, bias)
  X, Q = _f32c(X), _f32c(Q)
  ell_val, ell_idx, ell_max, gext, tiles = prep
  B, N, Din = X.shape
  K = Q.shape[2]
  S = 0
  if coeff is not None:
    coeff = _f32c(coeff)
    S = coeff.shape[2]
  E1 = ell_val.shape[1]
  H = w_hi.shape[0]
  assert w_hi.shape[1] == (S + E1) * Din, (w_hi.shape, S, E1, Din)
  out = torch.empty((B, N, H), device=X.device, dtype=torch.float32)
  _launch('lnb_spectral_conv_fused', X, X, Q, coeff, ell_val, ell_idx, ell_max, gext, tiles, w_hi, w_lo, bias,
          B, N, Din, E1, K, S, H, int(bool(relu)), int(bool(write_pad)), out)
  return out


def sage_operators(nn_idx, nonempty):
  """GraphSAGE's count-weighted operators (lnb_sage_operators): nn_idx [B,N,K,E1] int64 neighbour
  samples, nonempty [B,N] or [B,N,1] -> M [B,N,N,E1] fp32 with M[b,n,m,e] = nonempty * count / K."""
  _need_cuda(nn_idx, nonempty)
  nn_idx = nn_idx.contiguous().long()
  nonempty = _f32c(nonempty)
  B, N, K, E1 = nn_idx.shape
  if nonempty.numel() != B * N:
    raise ValueError('sage_operators: nonempty %s does not match nn_idx %s'
                     % (tuple(nonempty.shape), tuple(nn_idx.shape)))
  out = torch.empty((B, N, N, E1), device=nn_idx.device, dtype=torch.float32)
  _launch('lnb_sage_operators', nn_idx, nn_idx, nonempty, B, N, K, E1, out)
  return out


def neighbour_max(X, prep):
  """Max messages of GraphSAGE (lnb_neighbour_max): X [B,N,D], prep = graph_prepare(M, ...) ->
  (msg [B,N,E1*D] channel-major, argmax [B,N,E1,D] int32 node index, -1 for empty rows)."""
  ell_val, ell_idx, ell_max = prep[0], prep[1], prep[2]
  _need_cuda(X, ell_val)
  X = _f32c(X)
  B, N, D = X.shape
  E1 = ell_val.shape[1]
  out = torch.empty((B, N, E1 * D), device=X.device, dtype=torch.float32)
  arg = torch.empty((B, N, E1, D), device=X.device, dtype=torch.int32)
  _launch('lnb_neighbour_max', X, X, ell_val, ell_idx, ell_max, B, N, E1, D, out, arg)
  return out, arg


SAGE_SAMPLE_NN_IDX, SAGE_SAMPLE_ELL, SAGE_SAMPLE_ELL_T = 1, 2, 4    # LNB_SAGE_SAMPLE_*


def sage_sample_sparse(sizes, node_ptr, node_feat, edge_ptr, edges, sample_key, N, E1, K, want_nn_idx=True,
                       want_ell=False, want_ell_t=False):
  """GraphSAGE's neighbour samples drawn on the device from the records of data.sparse_collate
  (lnb_sage_sample_sparse; the rule is in the C header): K samples per (graph, node, channel) from
  Philox4x32-10 keyed by ``sample_key``, an int64 [2] CUDA tensor (seed, counter) read on the device.
  ``want_nn_idx``: the samples [B,N,K,E1] int32.  ``want_ell``: a GraphPrep of the count-weighted operator
  M = sage_operators(samples, nonempty), the ELL rows, ell_max and gext that graph_prepare(M) writes, its
  tile table pending (tile_assign(prep, 4)).  ``want_ell_t``: the same for M.transpose(1, 2), no tiles.
  Returns (node_ids [B,N] int64, mask [B,N] uint8, nonempty [B,N,1] fp32, nn_idx or None, prep or None,
  prep_t or None)."""
  N, E1, K = int(N), int(E1), int(K)
  _check_records('sage_sample_sparse', sizes, edge_ptr, edges)
  _need_cuda(node_ptr, node_feat, sample_key)
  if node_ptr.dtype != torch.int32 or node_feat.dtype != torch.int32 or node_ptr.shape[0] != sizes.shape[0] + 1:
    raise ValueError('sage_sample_sparse: node_ptr [B+1] and node_feat must be int32')
  if sample_key.dtype != torch.int64 or tuple(sample_key.shape) != (2,) or not sample_key.is_contiguous():
    raise ValueError('sage_sample_sparse: sample_key must be a contiguous int64 tensor of shape (2,); got %s %s'
                     % (sample_key.dtype, tuple(sample_key.shape)))
  B = sizes.shape[0]
  if not (1 <= N <= MAX_N and 2 <= E1 <= MAX_E1 and K >= 1 and B * N * E1 < 2 ** 31):
    raise ValueError('sage_sample_sparse: B=%d N=%d E1=%d K=%d outside 1 <= N <= %d, 2 <= E1 <= %d, K >= 1, '
                     'B*N*E1 < 2^31' % (B, N, E1, K, MAX_N, MAX_E1))
  if want_ell_t and not want_ell:
    raise ValueError('sage_sample_sparse: want_ell_t needs want_ell')
  dev = sizes.device
  node_ids = torch.empty((B, N), device=dev, dtype=torch.int64)
  mask = torch.empty((B, N), device=dev, dtype=torch.uint8)
  nonempty = torch.empty((B, N, 1), device=dev, dtype=torch.float32)
  nn_idx = torch.empty((B, N, K, E1), device=dev, dtype=torch.int32) if want_nn_idx else None

  def ell():
    return (torch.empty((B, E1, N, N), device=dev, dtype=torch.float32),
            torch.empty((B, E1, N, N), device=dev, dtype=torch.uint8),
            torch.empty((B, E1), device=dev, dtype=torch.int32), torch.empty((B, 2), device=dev, dtype=torch.int32))
  rows = ell() if want_ell else (None,) * 4
  rows_t = ell() if want_ell_t else (None,) * 4
  flags = ((SAGE_SAMPLE_NN_IDX if want_nn_idx else 0) | (SAGE_SAMPLE_ELL if want_ell else 0) |
           (SAGE_SAMPLE_ELL_T if want_ell_t else 0))
  _launch('lnb_sage_sample_sparse', sizes, sizes, node_ptr, node_feat, edge_ptr, edges, sample_key, B, N, E1, K,
          flags, node_ids, mask, nonempty, nn_idx, *rows, *rows_t)
  prep = prep_t = None
  if want_ell:
    prep = GraphPrep(rows + (torch.empty((4 * B + 2,), device=dev, dtype=torch.int32),))
    prep.tiles_pending = B > 0
  if want_ell_t:
    prep_t = GraphPrep(rows_t + (None,))
  return node_ids, mask, nonempty, nn_idx, prep, prep_t


SAGE_MAX = 1        # LNB_SAGE_MAX


def spectral_stack_forward(prep, Q, w_hi, w_lo, bias, dins, H, S, coeff=None, coeff_stride=0,
                           X=None, node_ids=None, emb=None, want_state=False, write_pad=True,
                           readout=None, mask=None, relu=True, sage=None):
  """All convolution layers (+ optional embedding gather and readout) in one persistent kernel.

  prep = graph_prepare(L, Q); w_hi/w_lo [len(dins)*H, Kw] stacked split weights, bias
  [len(dins)*H]; dins = input width per layer; coeff = tensor whose layer l block starts at
  element l*coeff_stride (None when S == 0); X [B,N,dins[0]] or node_ids [B,N] + emb;
  readout = (W_out [P,H], b_out [P], w_att [H], b_att [1]) -> score [B,P].
  sage = None runs lnb_spectral_stack_forward; 'Mean' / 'Max' run the GraphSAGE variant
  (lnb_sage_stack_forward: rows L2-normalised after every layer, Max aggregation for 'Max').
  Returns (state or None, score or None)."""
  ell_val, ell_idx, ell_max, gext, tiles = prep
  _need_cuda(Q, w_hi, w_lo, bias, coeff, X, node_ids, emb, mask)
  Q = _f32c(Q)
  B, N, K = Q.shape
  E1 = ell_val.shape[1]
  dev = Q.device
  d = SpectralStack()
  if X is not None:
    X = _f32c(X)
    d.X = X.data_ptr()
  else:
    node_ids = node_ids.contiguous().long()
    emb = _f32c(emb)
    d.node_ids, d.emb_table, d.emb_rows = node_ids.data_ptr(), emb.data_ptr(), emb.shape[0]
  d.Q = Q.data_ptr()
  if coeff is not None:
    d.coeff, d.coeff_layer_stride = coeff.data_ptr(), int(coeff_stride)
  d.ell_val, d.ell_idx, d.ell_max = ell_val.data_ptr(), ell_idx.data_ptr(), ell_max.data_ptr()
  d.gext, d.tiles = gext.data_ptr(), tiles.data_ptr()
  d.W_hi, d.W_lo = w_hi.data_ptr(), w_lo.data_ptr()
  d.bias = bias.data_ptr() if bias is not None else None
  state = score = None
  if want_state or readout is None:
    state = torch.empty((B, N, H), device=dev, dtype=torch.float32)
    d.out_state = state.data_ptr()
  keep = []
  if readout is not None:
    W_out, b_out, w_att, b_att = [_f32c(t) for t in readout]
    keep += [W_out, b_out, w_att, b_att]
    score = torch.empty((B, W_out.shape[0]), device=dev, dtype=torch.float32)
    d.W_out, d.b_out, d.w_att, d.b_att = (W_out.data_ptr(), b_out.data_ptr(), w_att.data_ptr(),
                                          b_att.data_ptr())
    d.score, d.P = score.data_ptr(), W_out.shape[0]
    if mask is not None:
      if mask.dtype != torch.uint8:            # any non-zero byte counts as 'real node' in the kernel
        mask = (mask != 0).to(torch.uint8)
      mask = mask.contiguous()
      d.mask = mask.data_ptr()
  for i, v in enumerate(dins):
    d.Din[i] = int(v)
  d.num_layers, d.Kw, d.write_pad = len(dins), int(w_hi.shape[1]), int(bool(write_pad))
  d.B, d.N, d.E1, d.K, d.S, d.H, d.relu = B, N, E1, K, int(S), int(H), int(bool(relu))
  if sage is None:
    _launch('lnb_spectral_stack_forward', Q, ctypes.byref(d))
  elif sage not in ('Mean', 'Max'):
    raise ValueError('spectral_stack_forward: sage=%r (Mean or Max)' % (sage,))
  else:
    _launch('lnb_sage_stack_forward', Q, ctypes.byref(d), SAGE_MAX if sage == 'Max' else 0)
  return state, score


def ritz_rowmap(gext, K):
  """Compact list of the (graph, k) rows with k < k_eff(graph): (rowmap [B*K] int32, nrows [1])."""
  _need_cuda(gext)
  B = gext.shape[0]
  rowmap = torch.empty((B * K,), device=gext.device, dtype=torch.int32)
  nrows = torch.empty((1,), device=gext.device, dtype=torch.int32)
  _launch('lnb_ritz_rowmap', gext, gext, B, int(K), rowmap, nrows)
  return rowmap, nrows


def ritz_filter_mlp_supported(S, hidden):
  """Shapes lnb_ritz_filter_mlp accepts: S scales and a hidden width of ``hidden``."""
  return S <= FILTER_MLP_MAX_S and hidden % 32 == 0 and hidden <= MAX_WIDTH


def ritz_filter_mlp(table, w_hi, w_lo, bias_all, num_layers, rowmap=None, nrows=None, ctas=0):
  """coeff[l, r, :] = MLP_l(table[r, :]) for all layers in one persistent kernel.
  table [R, S]; w_hi/w_lo [L*(3*Hd+S), Hd] stacked split weights; returns coeff [L, R, S]
  (rows not listed in rowmap are left unwritten).  ctas > 0 caps the persistent grid (same bits)."""
  _need_cuda(table, w_hi, w_lo, bias_all, rowmap, nrows)
  table = _f32c(table)
  R, S = table.shape
  Hd = w_hi.shape[1]
  coeff = torch.empty((num_layers, R, S), device=table.device, dtype=torch.float32)
  _launch('lnb_ritz_filter_mlp_ctas', table, table, rowmap, nrows, w_hi, w_lo, bias_all, R, int(num_layers), S, Hd,
          coeff, int(ctas))
  return coeff


def embedding_rows(idx, table):
  _need_cuda(idx, table)
  idx = idx.contiguous().long()
  table = _f32c(table)
  rows = idx.numel()
  out = torch.empty(tuple(idx.shape) + (table.shape[1],), device=table.device, dtype=torch.float32)
  _launch('lnb_embedding_rows', table, idx, table, rows, table.shape[0], table.shape[1], out)
  return out


def ritz_power_table(D, powers):
  """table[..., s] = D ** powers[s]  (model/lanczos_net.py:146-149)."""
  _need_cuda(D)
  D = _f32c(D)
  S = len(powers)
  out = torch.empty(tuple(D.shape) + (S,), device=D.device, dtype=torch.float32)
  _launch('lnb_ritz_power_table', D, D, D.numel(), _ints(powers), S, out)
  return out


def readout(state, W_out, b_out, w_att, b_att, mask=None):
  _need_cuda(state, W_out, b_out, w_att, b_att, mask)
  state = _f32c(state)
  B, N, H = state.shape
  P = W_out.shape[0]
  if mask is not None:
    mask = (mask != 0).to(torch.uint8).contiguous()
  out = torch.empty((B, P), device=state.device, dtype=torch.float32)
  _launch('lnb_readout', state, state, _f32c(W_out), _f32c(b_out), _f32c(w_att), _f32c(b_att), mask, B, N, H, P,
          out)
  return out


def gat_attention_supported(N, F, E1, heads):
  """Shapes lnb_gat_attention accepts (mirrors its checks)."""
  return N <= MAX_N and F % 4 == 0 and F <= GAT_MAX_WIDTH and E1 <= MAX_E1 and heads <= GAT_MAX_HEADS


def gat_attention(Wh, bias, a1, a2, c1, c2, state_bias, last=False):
  """Graph attention of one GAT layer after the projection (see lnb_gat_attention).
  Wh [B,N,C*F], bias [B,N,N,E1], a1/a2/state_bias [C,F], c1/c2 [C] with C = E1*heads.
  Returns ELU(h_c) concatenated over c [B,N,C*F], or with ``last`` the mean over c [B,N,F]."""
  _need_cuda(Wh, bias, a1, a2, c1, c2, state_bias)
  Wh, bias = _f32c(Wh), _f32c(bias)
  a1, a2, c1, c2, state_bias = [_f32c(t) for t in (a1, a2, c1, c2, state_bias)]
  B, N, _, E1 = bias.shape
  C, F = a1.shape
  heads = C // E1
  if heads * E1 != C or tuple(Wh.shape) != (B, N, C * F) or tuple(state_bias.shape) != (C, F):
    raise ValueError('gat_attention: Wh %s, bias %s, a1 %s, state_bias %s do not agree'
                     % (tuple(Wh.shape), tuple(bias.shape), tuple(a1.shape), tuple(state_bias.shape)))
  out = torch.empty((B, N, F if last else C * F), device=Wh.device, dtype=torch.float32)
  _launch('lnb_gat_attention', Wh, Wh, bias, a1, a2, c1, c2, state_bias, B, N, E1, heads, F, int(bool(last)), out)
  return out


def gat_attention_backward_supported(N, F, E1, heads):
  """Shapes lnb_gat_attention_backward accepts (mirrors its checks): the forward's envelope."""
  return gat_attention_supported(N, F, E1, heads)


def gat_attention_backward(gout, Wh, bias, a1, a2, c1, c2, state_bias, out=None, last=False):
  """Adjoint of ``gat_attention`` (see lnb_gat_attention_backward); ``gout`` is the gradient of its
  output.  The kernel recomputes the attention and h from the inputs; ``out`` (the forward's output) is
  optional and only checked against the shapes.
  Returns (gWh [B,N,C*F], ga1 [C,F], ga2 [C,F], gc1 [C], gc2 [C], gsb [C,F]); the per-graph partials
  of the parameter gradients are summed over the batch here.  No gradient for the bias (data)."""
  _need_cuda(gout, Wh, bias, a1, a2, c1, c2, state_bias, out)
  Wh, bias, gout = _f32c(Wh), _f32c(bias), _f32c(gout)
  a1, a2, c1, c2, state_bias = [_f32c(t) for t in (a1, a2, c1, c2, state_bias)]
  B, N, _, E1 = bias.shape
  C, F = a1.shape
  heads = C // E1
  shape = (B, N, F if last else C * F)
  if (heads * E1 != C or tuple(Wh.shape) != (B, N, C * F) or tuple(state_bias.shape) != (C, F) or
      tuple(gout.shape) != shape or (out is not None and tuple(out.shape) != shape)):
    raise ValueError('gat_attention_backward: gout %s, Wh %s, bias %s, a1 %s, state_bias %s, out %s do not agree'
                     % (tuple(gout.shape), tuple(Wh.shape), tuple(bias.shape), tuple(a1.shape),
                        tuple(state_bias.shape), None if out is None else tuple(out.shape)))
  gWh = torch.empty((B, N, C * F), device=Wh.device, dtype=torch.float32)
  if B == 0:                                                # zero parameter gradients, nothing launched
    z = torch.zeros((C, F), device=Wh.device, dtype=torch.float32)
    return gWh, z, z.clone(), z[:, 0].clone(), z[:, 0].clone(), z.clone()
  gpar = torch.empty((B, C, 3 * F + 2), device=Wh.device, dtype=torch.float32)
  _launch('lnb_gat_attention_backward', Wh, gout, Wh, bias, a1, a2, c1, c2, state_bias, B, N, E1, heads, F,
          int(bool(last)), gWh, gpar)
  g = gpar.sum(dim=0)
  return (gWh, g[:, :F].contiguous(), g[:, F:2 * F].contiguous(), g[:, 3 * F].contiguous(),
          g[:, 3 * F + 1].contiguous(), g[:, 2 * F:3 * F].contiguous())


def check_dropout_key(who, key):
  """``dropout_key``: an int64 tensor of shape (2,), (seed, counter), as ``check_start_key`` asks of a start key."""
  if not torch.is_tensor(key) or key.dtype != torch.int64 or tuple(key.shape) != (2,):
    raise ValueError("%s: 'dropout_key' must be an int64 tensor of shape (2,) (seed, counter); got %r"
                     % (who, (key.dtype, tuple(key.shape)) if torch.is_tensor(key) else type(key)))


def _dropout_args(who, key, p, t):
  check_dropout_key(who, key)
  _need_cuda(key)
  p, t = float(p), int(t)
  if not 0.0 <= p <= 1.0:
    raise ValueError('%s: p=%g outside [0, 1]' % (who, p))
  if not 0 <= t < 1 << 16:
    raise ValueError('%s: layer %d outside 0 <= t < 2^16' % (who, t))
  return key.contiguous(), p, t


def gat_attention_dropout(Wh, bias, a1, a2, c1, c2, state_bias, dropout_key, p, t, last=False):
  """``gat_attention`` with the reference's attention and Wh dropout of layer ``t`` (lnb_gat_attention_dropout;
  the mask rule is in the C header): masks drawn on the device from ``dropout_key``, an int64 [2] CUDA
  tensor (seed, counter) read on the device."""
  key, p, t = _dropout_args('gat_attention_dropout', dropout_key, p, t)
  _need_cuda(Wh, bias, a1, a2, c1, c2, state_bias)
  Wh, bias = _f32c(Wh), _f32c(bias)
  a1, a2, c1, c2, state_bias = [_f32c(x) for x in (a1, a2, c1, c2, state_bias)]
  B, N, _, E1 = bias.shape
  C, F = a1.shape
  heads = C // E1
  if heads * E1 != C or tuple(Wh.shape) != (B, N, C * F) or tuple(state_bias.shape) != (C, F):
    raise ValueError('gat_attention_dropout: Wh %s, bias %s, a1 %s, state_bias %s do not agree'
                     % (tuple(Wh.shape), tuple(bias.shape), tuple(a1.shape), tuple(state_bias.shape)))
  out = torch.empty((B, N, F if last else C * F), device=Wh.device, dtype=torch.float32)
  _launch('lnb_gat_attention_dropout', Wh, Wh, bias, a1, a2, c1, c2, state_bias, B, N, E1, heads, F,
          int(bool(last)), key, p, t, out)
  return out


def gat_attention_dropout_backward(gout, Wh, bias, a1, a2, c1, c2, state_bias, dropout_key, p, t, last=False):
  """Adjoint of ``gat_attention_dropout`` with the same key, p and t (lnb_gat_attention_dropout_backward): the
  masks are drawn again.  Returns (gWh, ga1, ga2, gc1, gc2, gsb) as ``gat_attention_backward``."""
  key, p, t = _dropout_args('gat_attention_dropout_backward', dropout_key, p, t)
  _need_cuda(gout, Wh, bias, a1, a2, c1, c2, state_bias)
  Wh, bias, gout = _f32c(Wh), _f32c(bias), _f32c(gout)
  a1, a2, c1, c2, state_bias = [_f32c(x) for x in (a1, a2, c1, c2, state_bias)]
  B, N, _, E1 = bias.shape
  C, F = a1.shape
  heads = C // E1
  if (heads * E1 != C or tuple(Wh.shape) != (B, N, C * F) or tuple(state_bias.shape) != (C, F) or
      tuple(gout.shape) != (B, N, F if last else C * F)):
    raise ValueError('gat_attention_dropout_backward: gout %s, Wh %s, bias %s, a1 %s, state_bias %s do not agree'
                     % (tuple(gout.shape), tuple(Wh.shape), tuple(bias.shape), tuple(a1.shape),
                        tuple(state_bias.shape)))
  gWh = torch.empty((B, N, C * F), device=Wh.device, dtype=torch.float32)
  if B == 0:
    z = torch.zeros((C, F), device=Wh.device, dtype=torch.float32)
    return gWh, z, z.clone(), z[:, 0].clone(), z[:, 0].clone(), z.clone()
  gpar = torch.empty((B, C, 3 * F + 2), device=Wh.device, dtype=torch.float32)
  _launch('lnb_gat_attention_dropout_backward', Wh, gout, Wh, bias, a1, a2, c1, c2, state_bias, B, N, E1, heads, F,
          int(bool(last)), key, p, t, gWh, gpar)
  g = gpar.sum(dim=0)
  return (gWh, g[:, :F].contiguous(), g[:, F:2 * F].contiguous(), g[:, 3 * F].contiguous(),
          g[:, 3 * F + 1].contiguous(), g[:, 2 * F:3 * F].contiguous())


def gat_dropout_project_supported(Din, F):
  """Shapes lnb_gat_dropout_project(_backward) accept (mirrors their checks)."""
  return Din % 4 == 0 and F % 4 == 0 and F <= GAT_MAX_WIDTH


def _project_dims(who, X, W, C):
  M, Din = X.shape
  if C < 1 or W.dim() != 2 or W.shape[1] != Din or W.shape[0] % C:
    raise ValueError('%s: X %s, W %s do not agree with C=%d channels' % (who, tuple(X.shape), tuple(W.shape), C))
  return M, Din, W.shape[0] // C


def gat_dropout_project(X, W, C, dropout_key, p, t):
  """GAT's per-channel input dropout and projection of layer ``t`` (lnb_gat_dropout_project):
  Wh[:, c*F:(c+1)*F] = (X * M_c s) W_c^T for X [M, Din] and W [C*F, Din] (channel c's weight in rows
  c*F .. c*F+F-1).  Returns Wh [M, C*F]."""
  key, p, t = _dropout_args('gat_dropout_project', dropout_key, p, t)
  _need_cuda(X, W)
  X, W = _f32c(X), _f32c(W)
  M, Din, F = _project_dims('gat_dropout_project', X, W, int(C))
  Wh = torch.empty((M, W.shape[0]), device=X.device, dtype=torch.float32)
  _launch('lnb_gat_dropout_project', X, X, W, M, Din, int(C), F, key, p, t, Wh)
  return Wh


def gat_dropout_project_backward(X, W, gWh, C, dropout_key, p, t):
  """Adjoint of ``gat_dropout_project`` with the same key, p and t (lnb_gat_dropout_project_backward; the masks
  are drawn again).  Returns (gX [M, Din], gW [C*F, Din])."""
  key, p, t = _dropout_args('gat_dropout_project_backward', dropout_key, p, t)
  _need_cuda(X, W, gWh)
  X, W, gWh = _f32c(X), _f32c(W), _f32c(gWh)
  C = int(C)
  M, Din, F = _project_dims('gat_dropout_project_backward', X, W, C)
  if tuple(gWh.shape) != (M, C * F):
    raise ValueError('gat_dropout_project_backward: gWh %s, expected %s' % (tuple(gWh.shape), (M, C * F)))
  slabs = max(int(_lib.load().lnb_gat_dropout_project_slabs(M, Din, C, F)), 1)
  gX = torch.empty_like(X)
  gW = torch.empty_like(W)
  work = torch.empty((slabs, C * F, Din), device=X.device, dtype=torch.float32)
  _launch('lnb_gat_dropout_project_backward', X, X, W, gWh, M, Din, C, F, key, p, t, gX, gW, work)
  return gX, gW


def ggnn_update_supported(N, D, E1):
  """Shapes lnb_ggnn_update accepts (mirrors its checks)."""
  return 1 <= N <= MAX_N_ELL and D % 32 == 0 and 32 <= D <= MAX_WIDTH and 1 <= E1 <= MAX_E1


def ggnn_update(M, h, prep, w_hi, w_lo, bias, avg, out=None):
  """One GGNN propagation step after the message MLPs (see lnb_ggnn_update): the GRU cell of
  [A_0 M_0 | ... | A_{E1-1} M_{E1-1} | h] with A_e the 0/1 pattern of channel e (row-normalised when
  ``avg``), gathered through the ELL rows of ``prep`` (graph_prepare of the operators [B,N,N,E1]).
  M [B*N, E1*D], h [B*N, D]; w_hi / w_lo / bias: the re-laid-out gate matrix [4D, (E1+1)*D] and its
  bias [4D] (model.ggnn.gru_gate_matrix).  Returns h' [B*N, D] (written to ``out`` when given)."""
  _need_cuda(M, h, w_hi, w_lo, bias, out)
  M, h, bias = _f32c(M), _f32c(h), _f32c(bias)
  ell_val, ell_idx, ell_max = prep[0], prep[1], prep[2]
  B, E1, N = ell_val.shape[0], ell_val.shape[1], ell_val.shape[2]
  D = h.shape[1]
  if (tuple(h.shape) != (B * N, D) or tuple(M.shape) != (B * N, E1 * D) or
      tuple(w_hi.shape) != (4 * D, (E1 + 1) * D) or tuple(bias.shape) != (4 * D,)):
    raise ValueError('ggnn_update: M %s, h %s, W %s, bias %s do not agree with B=%d N=%d E1=%d'
                     % (tuple(M.shape), tuple(h.shape), tuple(w_hi.shape), tuple(bias.shape), B, N, E1))
  if out is None:
    out = torch.empty_like(h)
  _launch('lnb_ggnn_update', h, M, h, ell_val, ell_idx, ell_max, w_hi, w_lo, bias, B, N, D, E1, int(bool(avg)), out)
  return out


def sage_lstm_step_supported(D, E1, K):
  """Shapes lnb_sage_lstm_step accepts (mirrors its checks)."""
  return D % 32 == 0 and 32 <= D <= MAX_WIDTH and 1 <= E1 <= MAX_E1 and K >= 1


def sage_lstm_step(state, nn_idx, nonempty, h, c, w_hi, w_lo, bias, t, out):
  """Step t of GraphSAGE's LSTM aggregator for all B*N*E1 sequences of a layer (see lnb_sage_lstm_step).
  state [B*N, D]; nn_idx int32 [B, N, K, E1] (contiguous); nonempty float32 [B*N]; h (ignored at t = 0),
  c (updated in place) and out float32 [B*N*E1, D]; w_hi / w_lo / bias: lstm_gate_matrix of the cell,
  [4D, 2D] and [4D].  Returns out: h of step t, or on the last step the message matrix viewed [B*N, E1*D]."""
  _need_cuda(state, nn_idx, nonempty, h, c, w_hi, w_lo, bias, out)
  B, N, K, E1 = nn_idx.shape
  D = state.shape[1]
  R = B * N * E1
  ok = (nn_idx.dtype == torch.int32 and nn_idx.is_contiguous() and tuple(state.shape) == (B * N, D) and
        tuple(nonempty.shape) == (B * N,) and tuple(c.shape) == (R, D) and tuple(out.shape) == (R, D) and
        (h is None or tuple(h.shape) == (R, D)) and tuple(w_hi.shape) == (4 * D, 2 * D) and
        tuple(bias.shape) == (4 * D,))
  if not ok:
    raise ValueError('sage_lstm_step: state %s, nn_idx %s %s, nonempty %s, h %s, c %s, out %s, W %s, bias %s do '
                     'not agree' % (tuple(state.shape), tuple(nn_idx.shape), nn_idx.dtype, tuple(nonempty.shape),
                                    None if h is None else tuple(h.shape), tuple(c.shape), tuple(out.shape),
                                    tuple(w_hi.shape), tuple(bias.shape)))
  for name, x in (('state', state), ('nonempty', nonempty), ('h', h), ('c', c), ('out', out), ('bias', bias)):
    if x is not None and (x.dtype != torch.float32 or not x.is_contiguous()):
      raise ValueError('sage_lstm_step: %s must be a contiguous float32 tensor' % name)
  _launch('lnb_sage_lstm_step', state, state, nn_idx, nonempty, h, c, w_hi, w_lo, bias, B, N, K, E1, D, int(t), out)
  return out


def sage_lstm_messages(state, nn_idx, nonempty, w_hi, w_lo, bias):
  """The messages of one LSTM GraphSAGE layer: the K steps of ``sage_lstm_step`` over fresh h / c buffers.
  state [B*N, D], nn_idx int32 [B, N, K, E1], nonempty float32 [B*N].  Returns [B*N, E1*D], column block e
  = the final h of channel e times nonempty."""
  B, N, K, E1 = nn_idx.shape
  D = state.shape[1]
  R = B * N * E1
  state = _f32c(state)
  c = torch.empty((R, D), device=state.device, dtype=torch.float32)
  h = torch.empty_like(c)
  spare = torch.empty_like(c) if K > 1 else None
  for t in range(K):
    if t == K - 1:
      out = torch.empty((B * N, E1 * D), device=state.device, dtype=torch.float32)
      sage_lstm_step(state, nn_idx, nonempty, h if t else None, c, w_hi, w_lo, bias, t, out.view(R, D))
      return out
    sage_lstm_step(state, nn_idx, nonempty, h if t else None, c, w_hi, w_lo, bias, t, spare)
    h, spare = spare, h


def gpnn_partition_update_supported(N, H):
  """Shapes lnb_gpnn_partition_update accepts (mirrors its checks)."""
  return 1 <= N <= MAX_N_ELL and H % 32 == 0 and 32 <= H <= MAX_WIDTH


def _rows_view(who, t, rows, H):
  """(tensor, row stride) of a float32 CUDA [rows, H] view whose rows may be strided (a column block)."""
  if t.dtype != torch.float32 or t.dim() != 2 or tuple(t.shape) != (rows, H) or t.stride(1) != 1:
    raise ValueError('%s: expected a float32 [%d, %d] view with unit column stride, got %s %s stride %s'
                     % (who, rows, H, t.dtype, tuple(t.shape), t.stride()))
  return t, t.stride(0)


def gpnn_partition_update(parts, prep, w_hi, w_lo, bias, avg, h_copy=None):
  """GPNN propagation within clusters and across cuts (see lnb_gpnn_partition_update), both parts in one
  launch.  ``parts``: two entries, (M, h, out) for the cluster and the cut operator, or None to skip that
  part; M, h, out are float32 [B*N, H] views (rows may be strided, e.g. column blocks of the [B*N, 3H]
  input of state_func; one row stride each for all M, all h and all outputs).  M and h may be the same
  tensors for both parts; no output may overlap an h.  ``prep``: graph_prepare of
  stack([L_cluster, L_cut], 3), not binarised.  w_hi / w_lo / bias: gru_gate_matrix of the partition
  GRUCell [4H, 2H], [4H].  ``h_copy``: optional [B*N, H] view with the outputs' row stride that receives
  the h rows of the first active part.  Returns ``parts``' outputs."""
  ell_val, ell_idx, ell_max = prep[0], prep[1], prep[2]
  B, two, N = ell_val.shape[0], ell_val.shape[1], ell_val.shape[2]
  if two != 2 or len(parts) != 2:
    raise ValueError('gpnn_partition_update: needs the ELL rows of the two partition operators and two parts')
  live = [pt for pt in parts if pt is not None]
  if not live:
    raise ValueError('gpnn_partition_update: no active part')
  H = live[0][1].shape[1]
  rows = B * N
  _need_cuda(w_hi, w_lo, bias, h_copy, *[t for pt in live for t in pt])
  bias = _f32c(bias)
  if tuple(w_hi.shape) != (4 * H, 2 * H) or tuple(w_lo.shape) != (4 * H, 2 * H) or tuple(bias.shape) != (4 * H,):
    raise ValueError('gpnn_partition_update: W %s, bias %s do not agree with H=%d'
                     % (tuple(w_hi.shape), tuple(bias.shape), H))
  ptrs, strides = [], {'M': set(), 'h': set(), 'out': set()}
  for pt in parts:
    if pt is None:
      ptrs += [None, None, None]
      continue
    for key, t in zip(('M', 'h', 'out'), pt):
      _, ld = _rows_view('gpnn_partition_update: %s' % key, t, rows, H)
      strides[key].add(ld)
      ptrs.append(t)
  if h_copy is not None:
    strides['out'].add(_rows_view('gpnn_partition_update: h_copy', h_copy, rows, H)[1])
  if any(len(s) != 1 for s in strides.values()):
    raise ValueError('gpnn_partition_update: one row stride each for M, h and out, got %s' % strides)
  ldm, ldh, ldo = strides['M'].pop(), strides['h'].pop(), strides['out'].pop()
  _launch('lnb_gpnn_partition_update', live[0][1], *ptrs, ell_val, ell_idx, ell_max, w_hi, w_lo, bias, h_copy,
          B, N, H, ldm, ldh, ldo, int(bool(avg)))
  return [None if pt is None else pt[2] for pt in parts]


MPNN_EDGE_HIDDEN = 64      # width of the edge network's hidden layer, fixed in the reference (model/mpnn.py:60)


def mpnn_update_supported(N, D, E1):
  """Shapes lnb_mpnn_update accepts (mirrors its checks)."""
  return 1 <= N <= MAX_N_ELL and D % 32 == 0 and 32 <= D <= MAX_WIDTH and 1 <= E1 <= MAX_E1


def mpnn_update(PQ, h, prep, w_hi, w_lo, bias, avg, out=None):
  """One MPNN propagation step with the edge-network messages (see lnb_mpnn_update): the GRU cell of
  [S_0 | ... | S_{E1-1} | deg | h] against the folded gate matrix, S_e gathered through the ELL rows of
  ``prep`` (graph_prepare of the operators [B,N,N,E1]).  PQ [B*N, E1*128] (per channel 64 P columns, then
  64 Q columns), h [B*N, D]; w_hi / w_lo / bias: the gate matrix [4D, 64*E1 + 32 + D] and its bias [4D]
  (model.mpnn.MPNN._step_params).  Returns h' [B*N, D] (written to ``out`` when given)."""
  _need_cuda(PQ, h, w_hi, w_lo, bias, out)
  PQ, h, bias = _f32c(PQ), _f32c(h), _f32c(bias)
  ell_val, ell_idx, ell_max = prep[0], prep[1], prep[2]
  B, E1, N = ell_val.shape[0], ell_val.shape[1], ell_val.shape[2]
  D = h.shape[1]
  K = MPNN_EDGE_HIDDEN * E1 + 32 + D
  if (tuple(h.shape) != (B * N, D) or tuple(PQ.shape) != (B * N, E1 * 2 * MPNN_EDGE_HIDDEN) or
      tuple(w_hi.shape) != (4 * D, K) or tuple(bias.shape) != (4 * D,)):
    raise ValueError('mpnn_update: PQ %s, h %s, W %s, bias %s do not agree with B=%d N=%d E1=%d'
                     % (tuple(PQ.shape), tuple(h.shape), tuple(w_hi.shape), tuple(bias.shape), B, N, E1))
  if out is None:
    out = torch.empty_like(h)
  _launch('lnb_mpnn_update', h, PQ, h, ell_val, ell_idx, ell_max, w_hi, w_lo, bias, B, N, D, E1, int(bool(avg)), out)
  return out


def mpnn_edge_aggregate_supported(N, E1):
  """Shapes lnb_mpnn_edge_aggregate and its backward accept (mirrors their checks)."""
  return 1 <= N <= MAX_N_ELL and 1 <= E1 <= MAX_E1


def _check_pq(who, PQ, prep):
  B, E1, N = prep[0].shape[0], prep[0].shape[1], prep[0].shape[2]
  if tuple(PQ.shape) != (B * N, E1 * 2 * MPNN_EDGE_HIDDEN):
    raise ValueError('%s: PQ %s does not agree with B=%d N=%d E1=%d' % (who, tuple(PQ.shape), B, N, E1))
  return B, N, E1


def mpnn_edge_aggregate(PQ, prep, avg):
  """S [B*N, E1*64] of lnb_mpnn_edge_aggregate: S_e[i] = w_i sum_j A_e[i,j] relu(P_e[j] + Q_e[i])."""
  _need_cuda(PQ)
  PQ = _f32c(PQ)
  B, N, E1 = _check_pq('mpnn_edge_aggregate', PQ, prep)
  S = torch.empty((B * N, E1 * MPNN_EDGE_HIDDEN), device=PQ.device, dtype=torch.float32)
  _launch('lnb_mpnn_edge_aggregate', PQ, PQ, prep[0], prep[1], prep[2], B, N, E1, int(bool(avg)), S)
  return S


def mpnn_edge_aggregate_backward(PQ, gS, prep, prep_t, avg):
  """gPQ [B*N, E1*128] (lnb_mpnn_edge_aggregate_backward); prep_t = graph_prepare of the transposed
  operators."""
  _need_cuda(PQ, gS)
  PQ, gS = _f32c(PQ), _f32c(gS)
  B, N, E1 = _check_pq('mpnn_edge_aggregate_backward', PQ, prep)
  if tuple(gS.shape) != (B * N, E1 * MPNN_EDGE_HIDDEN) or tuple(prep_t[0].shape) != tuple(prep[0].shape):
    raise ValueError('mpnn_edge_aggregate_backward: gS %s / transposed ELL %s do not agree with B=%d N=%d E1=%d'
                     % (tuple(gS.shape), tuple(prep_t[0].shape), B, N, E1))
  gPQ = torch.empty_like(PQ)
  _launch('lnb_mpnn_edge_aggregate_backward', PQ, PQ, gS, prep[0], prep[1], prep[2], prep_t[0], prep_t[1], prep_t[2],
          B, N, E1, int(bool(avg)), gPQ)
  return gPQ


def _ell_operator(who, prep, c0, nc):
  """(B, N, E1, nc) of the ELL rows ``prep`` for the channels [c0, c0 + nc), or ValueError."""
  if len(prep) < 4:
    raise ValueError('%s: prep must be a GraphPrep (ell_val, ell_idx, ell_max, gext, ...)' % who)
  val, idx, emax, gext = prep[0], prep[1], prep[2], prep[3]
  if val.dim() != 4 or val.shape[2] != val.shape[3]:
    raise ValueError('%s: ell_val must be [B, E1, N, N]; got %s' % (who, tuple(val.shape)))
  B, E1, N = val.shape[0], val.shape[1], val.shape[2]
  if not (1 <= N <= MAX_N and 1 <= E1 <= MAX_E1):
    raise ValueError('%s: N=%d, E1=%d outside 1 <= N <= %d, 1 <= E1 <= %d' % (who, N, E1, MAX_N, MAX_E1))
  if (val.dtype != torch.float32 or idx.dtype != torch.uint8 or emax.dtype != torch.int32 or
      gext.dtype != torch.int32):
    raise ValueError('%s: ELL rows must be float32 / uint8 / int32 / int32 (ell_val, ell_idx, ell_max, gext)' % who)
  if (tuple(idx.shape) != tuple(val.shape) or tuple(emax.shape) != (B, E1) or tuple(gext.shape) != (B, 2) or
      not (val.is_contiguous() and idx.is_contiguous() and emax.is_contiguous() and gext.is_contiguous())):
    raise ValueError('%s: ell_idx / ell_max / gext do not agree with ell_val %s' % (who, tuple(val.shape)))
  nc = E1 - c0 if nc is None else int(nc)
  if not (0 <= c0 and nc >= 1 and c0 + nc <= E1):
    raise ValueError('%s: channels [%d, %d) outside [0, %d)' % (who, c0, c0 + nc, E1))
  return B, N, E1, nc


def _ell_rows(who, name, t, rows, width, dev):
  """A row-strided float32 [rows, >= width] view with unit column stride on ``dev``, or ValueError."""
  if t.dtype != torch.float32 or t.dim() != 2 or t.shape[0] != rows or t.shape[1] < width:
    raise ValueError('%s: %s must be float32 [%d, >= %d]; got %s %s' % (who, name, rows, width, t.dtype,
                                                                        tuple(t.shape)))
  if t.device != dev:
    raise ValueError('%s: %s is on %s, the operators on %s' % (who, name, t.device, dev))
  if rows > 1 and t.stride(0) < width or (width > 1 and t.stride(1) != 1):
    raise ValueError('%s: %s needs unit column stride and a row stride >= %d; got strides %s'
                     % (who, name, width, t.stride()))
  return max(int(t.stride(0)), width)


def _span(t, width):
  """[first, last) byte addresses a row-strided float32 view of ``width`` columns reads or writes."""
  rows = t.shape[0] if t.dim() == 2 else 1
  if rows == 0 or width == 0:
    return (t.data_ptr(), t.data_ptr())
  stride = t.stride(0) if t.dim() == 2 else 0
  return (t.data_ptr(), t.data_ptr() + 4 * ((rows - 1) * stride + width))


def _ell_no_overlap(who, out, out_width, inputs):
  """ValueError when ``out`` shares storage bytes with any of ``inputs`` ((name, tensor, width) triples):
  the kernels read their inputs while other threads write ``out``."""
  o0, o1 = _span(out, out_width)
  for name, t, width in inputs:
    if t is None:
      continue
    a0, a1 = _span(t, width)
    if a0 < o1 and o0 < a1:
      raise ValueError('%s: out overlaps %s' % (who, name))


def _ell_weight(who, w, B, N, E1, dev):
  if w is None:
    return None
  if w.dtype != torch.float32 or tuple(w.shape) != (B, N, E1) or not w.is_contiguous() or w.device != dev:
    raise ValueError('%s: w must be a contiguous float32 [%d, %d, %d] tensor on %s' % (who, B, N, E1, dev))
  return w


def ell_messages(X, prep, c0=0, nc=None, w=None, out=None, col0=0):
  """L_e X over the ELL rows ``prep`` (graph_prepare / graph_prepare_sparse) for the channels
  c0 <= e < c0 + nc (default: all from c0), without the dense operators (lnb_ell_messages):
  out[b*N+n, col0 + (e-c0)*D + d] = w[b,n,e] * sum_t val[b,e,t,n] X[b*N + idx[b,e,t,n], d].
  X [B*N, D] and ``out`` [B*N, >= col0 + nc*D] are float32 views with unit column stride (any row stride);
  w [B,N,E1] optional row weights.  Returns out (a new [B*N, nc*D] tensor when not given)."""
  B, N, E1, nc = _ell_operator('ell_messages', prep, int(c0), nc)
  dev = prep[0].device
  D = X.shape[1] if X.dim() == 2 else -1
  if D < 1:
    raise ValueError('ell_messages: X must be [B*N, D] with D >= 1; got %s' % (tuple(X.shape),))
  ldx = _ell_rows('ell_messages', 'X', X, B * N, D, dev)
  w = _ell_weight('ell_messages', w, B, N, E1, dev)
  col0 = int(col0)
  if col0 < 0:
    raise ValueError('ell_messages: negative column offset %d' % col0)
  if out is not None:
    _ell_rows('ell_messages', 'out', out, B * N, col0 + nc * D, dev)
    _ell_no_overlap('ell_messages', out, col0 + nc * D, (('X', X, D), ('w', w, None if w is None else w.numel())))
  _need_cuda(*prep[:4], X, w, out)
  if out is None:
    out = torch.empty((B * N, col0 + nc * D), device=dev, dtype=torch.float32)
  ldo = _ell_rows('ell_messages', 'out', out, B * N, col0 + nc * D, dev)
  _launch('lnb_ell_messages', X, X, ldx, prep[0], prep[1], prep[2], prep[3], w, B, N, E1, int(c0), nc, D, out, ldo,
          col0)
  return out


def ell_messages_adjoint(G, prep_t, D, c0=0, nc=None, w=None, out=None):
  """The adjoint of ell_messages (lnb_ell_messages_adjoint): gX[b*N+m, d] = sum_e L_e^T (w_e . G_e), read
  from the ELL rows ``prep_t`` of the TRANSPOSED operators, every channel summed in one thread without
  atomics.  G [B*N, >= nc*D] (column block e - c0 = G_e) and ``out`` [B*N, >= D] are float32 views with unit
  column stride; w [B,N,E1] the forward's row weights.  Returns out (a new [B*N, D] tensor when not given)."""
  B, N, E1, nc = _ell_operator('ell_messages_adjoint', prep_t, int(c0), nc)
  dev = prep_t[0].device
  D = int(D)
  if D < 1:
    raise ValueError('ell_messages_adjoint: D=%d must be >= 1' % D)
  ldg = _ell_rows('ell_messages_adjoint', 'G', G, B * N, nc * D, dev)
  w = _ell_weight('ell_messages_adjoint', w, B, N, E1, dev)
  if out is not None:
    _ell_rows('ell_messages_adjoint', 'out', out, B * N, D, dev)
    _ell_no_overlap('ell_messages_adjoint', out, D, (('G', G, nc * D), ('w', w, None if w is None else w.numel())))
  _need_cuda(*prep_t[:4], G, w, out)
  if out is None:
    out = torch.empty((B * N, D), device=dev, dtype=torch.float32)
  ldgx = _ell_rows('ell_messages_adjoint', 'out', out, B * N, D, dev)
  _launch('lnb_ell_messages_adjoint', G, G, ldg, prep_t[0], prep_t[1], prep_t[2], prep_t[3], w, B, N, E1, int(c0), nc,
          D, out, ldgx)
  return out


def set2vec_supported(N, D, P):
  """Shapes lnb_set2vec accepts (mirrors its checks)."""
  return 1 <= N <= MAX_N and D % 32 == 0 and 32 <= D <= MAX_WIDTH and 1 <= P <= SET2VEC_MAX_P


def set2vec(X, mask, WgT, bg, W1, W2, W_out, b_out, steps):
  """Set2Vec readout + output Linear of every graph (see lnb_set2vec).  X [B,N,D]; mask [B,N] (any dtype,
  non-zero = in the set) or None for all nodes; WgT [2D,4D] the stacked gate weights (forget, input,
  output, memory) transposed; bg [4D]; W1 [D,D] as [in, out]; W2 [D] (or [D,1]); W_out [P,2D]; b_out [P].
  Returns score [B,P]."""
  _need_cuda(X, mask, WgT, bg, W1, W2, W_out, b_out)
  X = _f32c(X)
  B, N, D = X.shape
  P = W_out.shape[0]
  WgT, bg, W1, W2, W_out, b_out = [_f32c(t) for t in (WgT, bg, W1, W2, W_out, b_out)]
  if (tuple(WgT.shape) != (2 * D, 4 * D) or tuple(bg.shape) != (4 * D,) or tuple(W1.shape) != (D, D) or
      W2.numel() != D or tuple(W_out.shape) != (P, 2 * D) or tuple(b_out.shape) != (P,)):
    raise ValueError('set2vec: WgT %s, bg %s, W1 %s, W2 %s, W_out %s, b_out %s do not agree with D=%d'
                     % (tuple(WgT.shape), tuple(bg.shape), tuple(W1.shape), tuple(W2.shape), tuple(W_out.shape),
                        tuple(b_out.shape), D))
  if mask is not None:
    mask = (mask != 0).to(torch.uint8).contiguous()
    if tuple(mask.shape) != (B, N):
      raise ValueError('set2vec: mask %s does not match X %s' % (tuple(mask.shape), tuple(X.shape)))
  out = torch.empty((B, P), device=X.device, dtype=torch.float32)
  _launch('lnb_set2vec', X, X, mask, WgT, bg, W1, W2, W_out, b_out, B, N, D, P, int(steps), out)
  return out


def operator_chain_supported(N, steps):
  return N <= CHAIN_MAX_N and steps <= CHAIN_MAX_STEPS


def operator_chain(L, X, steps, block_of_step, out, out_col0, chebyshev=False):
  """Power / Chebyshev chain of channel 0 of L [B,N,N,E1] applied to X [B,N,D]; result i goes to
  column block out_col0 + block_of_step[i] of out [B,N,C*D] (block < 0: not stored)."""
  _need_cuda(L, X, out)
  L, X = _f32c(L), _f32c(X)
  B, N, D = X.shape
  E1 = L.shape[3]
  assert out.dtype == torch.float32 and out.is_contiguous() and out.shape[:2] == (B, N)
  sel = (ctypes.c_int * steps)(*[int(v) for v in block_of_step])
  _launch('lnb_operator_chain', X, L, X, B, N, E1, D, int(steps), 1 if chebyshev else 0, sel, out, out.stride(0),
          out.stride(1), int(out_col0))
  return out


def graph_messages_supported(N, K, E1, S, max_short):
  return (N <= MESSAGES_MAX_N and (S == 0 or K <= MESSAGES_MAX_K) and E1 <= MAX_E1 and S <= MESSAGES_MAX_S and
          max_short <= CHAIN_MAX_STEPS)


def graph_messages(L, X, Q, filt, dense_filter, short_dist, out):
  """The whole message matrix [short walk | long scales | edge types] of a general-shape layer in one
  launch (see lnb_graph_messages).  filt: [B,S,K,K] dense blocks (dense_filter) or [B,K,S] diagonal
  coefficients, None when there are no long scales; out [B,N,>=C*D] contiguous."""
  _need_cuda(L, X, Q, filt, out)
  L, X = _f32c(L), _f32c(X)
  B, N, D = X.shape
  E1 = L.shape[3]
  S = K = 0
  if filt is not None:
    filt, Q = _f32c(filt), _f32c(Q)
    K = Q.shape[2]
    S = filt.shape[1] if dense_filter else filt.shape[2]
  steps = sorted(short_dist)
  max_short = max(steps) if steps else 0
  sel = [steps.index(s) if s in steps else -1 for s in range(1, max_short + 1)]
  arr = (ctypes.c_int * max(1, max_short))(*([int(v) for v in sel] or [0]))
  assert out.dtype == torch.float32 and out.is_contiguous()
  _launch('lnb_graph_messages', X, L, X, Q, filt, B, N, E1, D, K, S, 1 if dense_filter else 0, max_short, arr,
          len(steps), out, out.stride(0), out.stride(1))
  return out


def gaussian_laplacian(x, L):
  _need_cuda(x, L)
  x, L = _f32c(x), _f32c(L)
  B, N, Dx = x.shape
  E1 = L.shape[3]
  out = torch.empty((B, N, N), device=x.device, dtype=torch.float32)
  _launch('lnb_gaussian_laplacian', x, x, L, B, N, Dx, E1, out)
  return out


def lanczos_ritz(A, mask, q1, K, want_ritz=True, want_T=True, want_Q=True, proper=False):
  """adjacency operator -> Ritz pairs in ONE launch (Lanczos + QL + Ritz vectors fused).
  Returns dict(alpha, beta [B,K], idx [B] int32, T [B,K,K], Q [B,N,K] when asked for, and with
  want_ritz theta [B,K] by descending |theta|, V [B,N,K] = Q S, status [B] (bit 0: QL not
  converged, bit 1: operator streamed because its non-zeros did not fit on chip)).
  proper=False reproduces the reference's masking rules of _lanczos_layer; proper=True returns the
  textbook Krylov factorisation (LNB_LANCZOS_PROPER) whose Ritz values are eigenvalues of A."""
  _need_cuda(A, mask, q1)
  A = _f32c(A)
  B, N = A.shape[0], A.shape[1]
  q1 = _f32c(q1).reshape(B, N)
  if mask is not None:
    mask = (mask != 0).to(torch.uint8).contiguous()
  dev = A.device
  out = {'alpha': torch.empty((B, K), device=dev, dtype=torch.float32),
         'beta': torch.empty((B, K), device=dev, dtype=torch.float32),
         'idx': torch.empty((B,), device=dev, dtype=torch.int32)}
  if want_T:
    out['T'] = torch.empty((B, K, K), device=dev, dtype=torch.float32)
  if want_Q:
    out['Q'] = torch.empty((B, N, K), device=dev, dtype=torch.float32)
  if want_ritz:
    out['theta'] = torch.empty((B, K), device=dev, dtype=torch.float32)
    out['V'] = torch.empty((B, N, K), device=dev, dtype=torch.float32)
    out['status'] = torch.empty((B,), device=dev, dtype=torch.int32)
  _launch('lnb_lanczos_ritz', A, A, mask, q1, B, N, K, 1 if proper else 0, out.get('T'), out.get('Q'), out['alpha'],
          out['beta'], out['idx'], out.get('theta'), out.get('V'), out.get('status'))
  return out


def tridiag_powers(T, powers):
  """out[b, r, s, c] = (T_b ** powers[s])[r, c]  (MLP input layout of ada_lanczos_net.py:274)."""
  _need_cuda(T)
  T = _f32c(T)
  B, K = T.shape[0], T.shape[1]
  S = len(powers)
  out = torch.empty((B, K, S, K), device=T.device, dtype=torch.float32)
  _launch('lnb_tridiag_powers', T, T, B, K, _ints(powers), S, out)
  return out


def tridiag_powers_backward_supported(K, powers):
  """True when lnb_tridiag_powers_backward takes K and these powers: at most TRIDIAG_POWERS_MAX_S, positive
  and strictly increasing, (6 K + (max power + 1) K^2) floats within SMEM_MAX bytes of shared memory."""
  powers = [int(p) for p in powers]
  return (1 <= len(powers) <= TRIDIAG_POWERS_MAX_S and K >= 1 and powers[0] >= 1 and
          all(a < b for a, b in zip(powers, powers[1:])) and
          (6 * K + (powers[-1] + 1) * K * K) * 4 <= SMEM_MAX)


def tridiag_powers_backward(T, gOut, powers):
  """Adjoint of ``tridiag_powers``: gT [B,K,K] for gOut [B,K,S,K] (lnb_tridiag_powers_backward).  Raises
  ValueError before any launch outside ``tridiag_powers_backward_supported``."""
  B, K = T.shape[0], T.shape[1]
  S = len(powers)
  if not tridiag_powers_backward_supported(K, powers):
    raise ValueError('tridiag_powers_backward: K=%d with powers up to %d outside the shared-memory envelope '
                     '((6 K + (max power + 1) K^2) * 4 bytes <= %d KB, at most %d powers)'
                     % (K, max(powers) if powers else 0, SMEM_MAX // 1024, TRIDIAG_POWERS_MAX_S))
  if tuple(gOut.shape) != (B, K, S, K):
    raise ValueError('tridiag_powers_backward: gOut must be [B,K,S,K] = %s; got %s'
                     % ((B, K, S, K), tuple(gOut.shape)))
  _need_cuda(T, gOut)
  T, gOut = _f32c(T), _f32c(gOut)
  gT = torch.empty((B, K, K), device=T.device, dtype=torch.float32)
  _launch('lnb_tridiag_powers_backward', T, T, gOut, B, K, _ints(powers), S, gT)
  return gT


def lanczos_tridiag_train_supported(N, K):
  """True when lnb_lanczos_tridiag_train / _backward take N and K: 1 <= N <= LANCZOS_TRAIN_MAX_N,
  1 <= K <= LANCZOS_MAX_K."""
  return 1 <= int(N) <= LANCZOS_TRAIN_MAX_N and 1 <= int(K) <= LANCZOS_MAX_K


def _lanczos_train_args(who, A, mask, q1, K):
  B, N = A.shape[0], A.shape[1]
  if not lanczos_tridiag_train_supported(N, K):
    raise ValueError('%s: N=%d K=%d outside 1 <= N <= %d, 1 <= K <= %d' % (who, N, K, LANCZOS_TRAIN_MAX_N,
                                                                          LANCZOS_MAX_K))
  _need_cuda(A, mask, q1)
  A = _f32c(A)
  q1 = _f32c(q1).reshape(B, N)
  if mask is not None:
    mask = (mask != 0).to(torch.uint8).contiguous()
  return A, mask, q1, B, N


def lanczos_tridiag_train(A, mask, q1, K):
  """The Lanczos layer of the training path (lnb_lanczos_tridiag_train): returns dict(T [B,K,K], Q [B,N,K],
  alpha, beta [B,K], idx [B] int32).  ValueError before any launch outside lanczos_tridiag_train_supported."""
  A, mask, q1, B, N = _lanczos_train_args('lanczos_tridiag_train', A, mask, q1, K)
  dev = A.device
  out = {'T': torch.empty((B, K, K), device=dev, dtype=torch.float32),
         'Q': torch.empty((B, N, K), device=dev, dtype=torch.float32),
         'alpha': torch.empty((B, K), device=dev, dtype=torch.float32),
         'beta': torch.empty((B, K), device=dev, dtype=torch.float32),
         'idx': torch.empty((B,), device=dev, dtype=torch.int32)}
  _launch('lnb_lanczos_tridiag_train', A, A, mask, q1, B, N, int(K), out['T'], out['Q'], out['alpha'], out['beta'],
          out['idx'])
  return out


def lanczos_tridiag_backward(A, mask, q1, K, gT, gQ, want_tape=False):
  """gA [B,N,N], the adjoint of lanczos_tridiag_train for the gradients gT [B,K,K] and gQ [B,N,K]
  (lnb_lanczos_tridiag_backward).  ``want_tape``: also the (T, Q) its recompute produced.  ValueError before
  any launch outside lanczos_tridiag_train_supported."""
  A, mask, q1, B, N = _lanczos_train_args('lanczos_tridiag_backward', A, mask, q1, K)
  gT, gQ = _f32c(gT), _f32c(gQ)
  if tuple(gT.shape) != (B, K, K) or tuple(gQ.shape) != (B, N, K):
    raise ValueError('lanczos_tridiag_backward: gT must be %s and gQ %s; got %s, %s'
                     % ((B, K, K), (B, N, K), tuple(gT.shape), tuple(gQ.shape)))
  dev = A.device
  gA = torch.empty((B, N, N), device=dev, dtype=torch.float32)
  T = torch.empty((B, K, K), device=dev, dtype=torch.float32) if want_tape else None
  Q = torch.empty((B, N, K), device=dev, dtype=torch.float32) if want_tape else None
  _launch('lnb_lanczos_tridiag_backward', A, A, mask, q1, B, N, int(K), gT, gQ, gA, T, Q)
  return (gA, T, Q) if want_tape else gA


def check_start_key(who, key):
  if not torch.is_tensor(key) or key.dtype != torch.int64 or tuple(key.shape) != (2,):
    raise ValueError("%s: 'start_key' must be an int64 tensor of shape (2,) (seed, counter); got %r"
                     % (who, (key.dtype, tuple(key.shape)) if torch.is_tensor(key) else type(key)))


def ada_start_vector(start_key, B, N):
  """AdaLanczosNet's Lanczos start vector q1 [B,N] fp32 drawn on the device (lnb_ada_start_vector; the
  rule is in the C header): one standard normal per (graph, padded node) from Philox4x32-10 keyed by
  ``start_key``, an int64 [2] CUDA tensor (seed, counter) read on the device."""
  check_start_key('ada_start_vector', start_key)
  _need_cuda(start_key)
  B, N = int(B), int(N)
  if B < 0 or N < 1:
    raise ValueError('ada_start_vector: bad dims B=%d N=%d' % (B, N))
  key = start_key.contiguous()
  q1 = torch.empty((B, N), device=key.device, dtype=torch.float32)
  _launch('lnb_ada_start_vector', key, key, B, N, q1)
  return q1


def symmetrize_filters(Y, K, S):
  """G[b,s,r,c] = (Y[b,r,c,s] + Y[b,c,r,s]) / 2 for Y viewed as [B,K,K,S]."""
  _need_cuda(Y)
  Y = _f32c(Y)
  B = Y.shape[0]
  G = torch.empty((B, S, K, K), device=Y.device, dtype=torch.float32)
  _launch('lnb_symmetrize_filters', Y, Y, B, K, S, G)
  return G


def segment_sum_forward(data, segment_index, num_segments, output=None, exact=None):
  """output[b, ids[b, c], :] += data[b, c, :] for data [B, d1, d2] and ids [B, d1] in [0, num_segments)
  (other ids are skipped); output defaults to zeros [B, num_segments, d2].  ``exact=True`` sums in
  lnb_unsorted_segment_sum_exact, whose bits do not depend on row order or scheduling; ``exact=False`` in
  the fp32-atomic lnb_unsorted_segment_sum_forward.  ``exact=None`` follows
  torch.are_deterministic_algorithms_enabled(), read at each call (so at capture in a CUDA graph)."""
  _need_cuda(data, segment_index, output)
  data = _f32c(data)
  seg = segment_index.contiguous().long()
  B, d1, d2 = data.shape
  if output is None:
    output = torch.zeros((B, num_segments, d2), device=data.device, dtype=torch.float32)
  if exact is None:
    exact = torch.are_deterministic_algorithms_enabled()
  if exact:
    n = B * int(num_segments) * d2
    ws = torch.zeros((2, n), device=data.device, dtype=torch.int64)   # acc [n], then exp [n] and flags [n] int32
    words = ws[1].view(torch.int32)
    _launch('lnb_unsorted_segment_sum_exact', data, data, seg, _ints([B, d1, d2]), int(num_segments), ws[0],
            words[:n], words[n:], output)
  else:
    _launch('lnb_unsorted_segment_sum_forward', data, data, seg, _ints([B, d1, d2]), int(num_segments), output)
  return output


def segment_sum_backward(grad_output, segment_index, data_shape, grad_data=None):
  _need_cuda(grad_output, segment_index, grad_data)
  grad_output = _f32c(grad_output)
  seg = segment_index.contiguous().long()
  B, d1, d2 = [int(v) for v in data_shape]
  if grad_data is None:
    grad_data = torch.empty((B, d1, d2), device=grad_output.device, dtype=torch.float32)
  _launch('lnb_unsorted_segment_sum_backward', grad_output, grad_output, seg, _ints([B, d1, d2]),
          int(grad_output.shape[1]), grad_data)
  return grad_data
