"""Host-side graph preparation for the hot path (numpy; no torch, no CUDA).

Mirrors the parts of the reference that *feed* the spectral-convolution forward:

  * ``get_laplacian(adj, 'L4')``      utils/data_helper.py:119-166 (L4 branch :155-156,
                                      normalisation :92-116)
  * ``get_graph_laplacian_eigs``      utils/data_helper.py:169-226 (dense eigh branch,
                                      -|lambda| stable ordering :217-223)
  * ``prepare_graph``                 dataset/get_qm8_data.py:60-90 / get_graph_data.py:52-92
  * ``collate``                       dataset/qm8.py:57-90,220-291 (default branch)
  * synthetic generators              dataset/get_graph_data.py:15-49 (G(n,p) regression set)
                                      and a QM8-shaped molecule sampler (SURVEY.md 8d)

All arithmetic follows the reference's fp64-then-cast-to-fp32 convention so the padded
batch tensors are bit-identical to what the reference loader would hand the model.
"""
import collections

import numpy as np

__all__ = [
    'check_dist', 'get_laplacian', 'get_graph_laplacian_eigs', 'prepare_graph',
    'collate', 'gat_bias', 'partition_operators', 'random_partition_labels', 'sage_collate', 'sparse_collate', 'pack_sparse', 'packed_offsets', 'packed_layout', 'packed_capacity', 'read_packed_header', 'synthetic_molecule', 'synthetic_qm8_samples', 'synthetic_qm8_batch',
    'synthetic_regression_graphs',
]

EPS = float(np.finfo(np.float32).eps)


def check_dist(dist):
  """utils/data_helper.py:9-14: diffusion distances must be ints or the string 'inf'."""
  for dd in dist:
    if not isinstance(dd, int) and dd != 'inf':
      raise ValueError("Non-supported value of diffusion distance")
  return dist


def _normalize_sym(mat, exponent=0.5):
  deg = mat.sum(axis=1)
  with np.errstate(divide='ignore'):
    scale = np.power(deg, -exponent)
  scale[np.isinf(scale)] = 0.0
  # same rounding as diag(s) @ M @ diag(s): fl(fl(s_i * m_ij) * s_j)
  return (scale[:, None] * mat) * scale[None, :]


def get_laplacian(adj, graph_laplacian_type='L4', alpha=0.5):
  """Dense graph operators of utils/data_helper.py:119-166.  The hot path only consumes
  'L4' (GCN renormalisation); L1/L2/L6 are provided because the same file defines them."""
  adj = np.asarray(adj)
  if not np.issubdtype(adj.dtype, np.floating):
    adj = adj.astype(np.float64)
  # NB: like the reference, arithmetic stays in the adjacency's dtype (the shipped
  # preprocessors feed float64; eye() promotes the L4 / L2 sums to float64 either way)
  if adj.ndim != 2 or adj.shape[0] != adj.shape[1]:
    raise ValueError('adjacency must be square')
  eye = np.eye(adj.shape[0])
  if graph_laplacian_type == 'L1':
    return np.diag(adj.sum(axis=1)) - adj
  if graph_laplacian_type == 'L2':
    return eye - _normalize_sym(adj)
  if graph_laplacian_type == 'L4':
    return _normalize_sym(eye + adj)
  if graph_laplacian_type == 'L6':
    return _normalize_sym(adj, exponent=alpha)
  raise ValueError('Unsupported Graph Laplacian!')


def get_graph_laplacian_eigs(adj, k=100, graph_laplacian_type='L4'):
  """(eigs[:k], V[:, :k], L) with eigenpairs ordered by descending |lambda| (stable), the
  dense-eigh branch of utils/data_helper.py:169-226."""
  lap = get_laplacian(adj, graph_laplacian_type)
  vals, vecs = np.linalg.eigh(lap)
  order = np.argsort(-np.abs(vals), kind='mergesort')[:k]
  return vals[order], vecs[:, order], lap


def prepare_graph(adjs, node_feat, label=None, eigs=True):
  """Per-graph record with the keys the collate step reads.  ``eigs=False`` skips the host eigh: the
  record then has no ``D_simple`` / ``V_simple`` and the eigenpairs are computed on the device
  (``sparse_collate(..., eigs=False)`` -> ``LanczosNet.forward_sparse``, or ``ops.sym_eigs``)."""
  adjs = np.asarray(adjs, dtype=np.float64)
  if adjs.ndim == 2:
    adjs = adjs[:, :, None]
  if eigs:
    D, V, L4 = get_graph_laplacian_eigs(adjs.sum(axis=2))
  else:
    L4 = get_laplacian(adjs.sum(axis=2))
  L_multi = np.stack([get_laplacian(adjs[:, :, e]) for e in range(adjs.shape[2])], axis=2)
  # bond list {u, v, type}, u <= v, each undirected bond once: the sparse record sparse_collate ships
  edges = np.array([(u, v, c) for c in range(adjs.shape[2])
                    for u, v in zip(*np.nonzero(np.triu(adjs[:, :, c])))], dtype=np.uint8).reshape(-1, 3)
  rec = {'node_feat': np.asarray(node_feat), 'L_multi': L_multi, 'L_simple_4': L4, 'edges': edges}
  if eigs:
    rec['D_simple'], rec['V_simple'] = D, V
  if label is not None:
    rec['label'] = np.asarray(label)
  return rec


def collate(samples, num_eigs, num_nodes=None):
  """Zero-pad a list of ``prepare_graph`` records to the batch-max node count (or to ``num_nodes`` if
  that is larger: fixed shapes for a captured training step, train.GraphedStep).

  Returns numpy arrays: node_feat (B,N) int64 or (B,N,D) float32, node_mask (B,N) uint8,
  L (B,N,N,E+1) float32 with channel 0 the simple-graph operator, D (B,K), V (B,N,K)."""
  sizes = np.array([s['L_simple_4'].shape[0] for s in samples])
  B, N = len(samples), max(int(sizes.max()), int(num_nodes or 0))
  E = samples[0]['L_multi'].shape[2]
  nf0 = np.asarray(samples[0]['node_feat'])
  node_feat = (np.zeros((B, N), np.int64) if nf0.ndim == 1
               else np.zeros((B, N, nf0.shape[1]), np.float32))
  mask = (np.arange(N)[None, :] < sizes[:, None]).astype(np.uint8)
  L = np.zeros((B, N, N, E + 1), np.float32)
  D = np.zeros((B, num_eigs), np.float32)
  V = np.zeros((B, N, num_eigs), np.float32)
  for b, s in enumerate(samples):
    n = int(sizes[b])
    node_feat[b, :n] = s['node_feat']
    L[b, :n, :n, 0] = s['L_simple_4']
    L[b, :n, :n, 1:] = s['L_multi']
    kk = min(num_eigs, s['D_simple'].shape[0])
    D[b, :kk] = s['D_simple'][:kk]
    V[b, :n, :kk] = s['V_simple'][:, :kk]
  out = {'node_feat': node_feat, 'node_mask': mask, 'L': L, 'D': D, 'V': V}
  if 'label' in samples[0]:
    out['label'] = np.concatenate([np.asarray(s['label'], np.float32).reshape(1, -1)
                                   for s in samples], axis=0)
  return out


def gat_bias(L):
  """The additive attention bias the reference collate hands GAT (dataset/qm8.py:196-219), from the
  collated operators L [B,N,N,E1] of ``collate``, bit for bit: per channel m = I (adj + I) in fp64,
  every entry > 0 of the padded N x N block set to 1, bias = -1e9 * (1 - m) cast to fp32.  For the
  non-negative QM8 operators that is -0.0 (note the sign) on edges, on the diagonal and on every
  padded node's self-loop, and -1e9 elsewhere.  Returns float32 [B,N,N,E1]."""
  L = np.asarray(L)
  N = L.shape[1]
  mt = L.astype(np.float64) + np.eye(N)[None, :, :, None]      # I @ (adj + I) is exact
  mt[mt > 0.0] = 1.0
  return (-1e9 * (1.0 - mt)).astype(np.float32)


def partition_operators(L_simple, labels):
  """GPNN's partition operators (utils/spectral_graph_partition.py:get_L_cluster_cut, applied per graph
  by the GPNN collate, dataset/qm8.py:127-135), for a whole batch at once.

  L_simple [B, N, N] (or [N, N]): the padded simple-graph operators; labels [B, N] (or [N]): the cluster of
  every node, padded nodes included.  The adjacency is the off-diagonal non-zero pattern of L_simple;
  its within-cluster part (both ends in one cluster) and the rest (the cut) each get the L4
  renormalisation D^-1/2 (I + A) D^-1/2 in fp64, so every node, padded ones too, keeps a self-loop.
  Returns (L_cluster, L_cut) as float32, the dtype the collate hands the model."""
  L = np.asarray(L_simple)
  lab = np.asarray(labels)
  single = L.ndim == 2
  if single:
    L, lab = L[None], lab[None]
  B, N = L.shape[0], L.shape[1]
  if L.shape != (B, N, N) or lab.shape != (B, N):
    raise ValueError('partition_operators: L_simple %s and labels %s do not agree' % (L.shape, lab.shape))
  off = ~np.eye(N, dtype=bool)[None]
  adj = ((L != 0) & off).astype(np.float64)
  same = (lab[:, :, None] == lab[:, None, :]).astype(np.float64)
  cluster = adj * same
  cut = adj - cluster
  out = []
  for a in (cluster, cut):
    m = a + np.eye(N)[None]
    scale = np.power(m.sum(axis=2), -0.5)                  # every row has its self-loop: no zero degree
    out.append(((scale[:, :, None] * m) * scale[:, None, :]).astype(np.float32))
  if single:
    out = [o[0] for o in out]
  return out[0], out[1]


def random_partition_labels(rng, batch_size, num_nodes, num_partition=3):
  """Seeded stand-in for the spectral clustering of the GPNN collate: a uniformly drawn cluster label per
  node [B, N] (benchmarks and tests; partition_operators turns them into operators)."""
  return rng.randint(0, num_partition, size=(batch_size, num_nodes))


def sage_collate(samples, num_sample_neighbors, npr):
  """The GraphSAGE branch of the reference collate (dataset/qm8.py:57-90,137-166): the same
  ``npr.choice`` calls in the same order (graph, then channel -- simple graph first, then the bond
  types --, then node), so the same ``np.random.RandomState`` gives an identical batch.  A node with
  at least K neighbours draws K of them without replacement, one with fewer draws K with replacement,
  one without any keeps the zero fill (node 0); ``nonempty`` is 1 once any channel has a neighbour.

  Returns numpy arrays: node_feat (B,N) int64, node_mask (B,N) uint8, nn_idx (B,N,K,E+1) int64,
  nonempty_mask (B,N,1) float32, label (B,P) float32 if present."""
  K = int(num_sample_neighbors)
  sizes = np.array([s['L_simple_4'].shape[0] for s in samples])
  B, N = len(samples), int(sizes.max())
  E = samples[0]['L_multi'].shape[2]
  node_feat = np.zeros((B, N), np.int64)
  nonempty = np.zeros((B, N, 1))
  nn_idx = np.zeros((B, N, K, E + 1))
  for ii, s in enumerate(samples):
    node_feat[ii, :sizes[ii]] = s['node_feat']
    for jj in range(E + 1):
      tmp_L = s['L_simple_4'] if jj == 0 else s['L_multi'][:, :, jj - 1]
      for nn in range(tmp_L.shape[0]):
        nn_list = np.nonzero(tmp_L[nn, :])[0]
        if len(nn_list) >= K:
          nn_idx[ii, nn, :, jj] = npr.choice(nn_list, size=K, replace=False)
          nonempty[ii, nn] = 1
        elif len(nn_list) > 0:
          nn_idx[ii, nn, :, jj] = npr.choice(nn_list, size=K, replace=True)
          nonempty[ii, nn] = 1
  out = {'node_feat': node_feat, 'node_mask': (np.arange(N)[None, :] < sizes[:, None]).astype(np.uint8),
         'nn_idx': nn_idx.astype(np.int64), 'nonempty_mask': nonempty.astype(np.float32)}
  if 'label' in samples[0]:
    out['label'] = np.concatenate([np.asarray(s['label'], np.float32).reshape(1, -1)
                                   for s in samples], axis=0)
  return out


def sparse_collate(samples, num_eigs, eigs=True):
  """The same batch as ``collate`` in SPARSE form for the GPU-side batch construction
  (ops.graph_prepare_sparse / LanczosNet.forward_sparse): nothing is padded on the host and the
  dense operators are not shipped at all.

  Returns numpy arrays: sizes [B] int32, node_ptr [B+1] int32 (prefix sums), node_feat [sum n] int32
  atom ids, or [sum n, F] float32 feature rows when the records' node_feat is 2-D (the bits of collate's
  node_feat[b, :n]; SparseLanczosNetGeneral and ops.graph_prepare_sparse_features read them), edge_ptr [B+1] int32, edges [sum E, 4] uint8 = {u, v, bond type, 0}, D [B,K] float32 (truncated /
  zero padded like dataset/qm8.py:268-287), V_rows [sum n, K] float32 (rows of real nodes only),
  N = batch-max node count (the reference's padding target), num_edgetype, label if present.
  ``eigs=False`` (records of ``prepare_graph(..., eigs=False)`` do): no D and no V_rows, only K = num_eigs;
  forward_sparse then computes the eigenpairs on the device (ops.graph_eigs_sparse)."""
  sizes = np.array([s['L_simple_4'].shape[0] for s in samples], np.int32)
  B = len(samples)
  node_ptr = np.zeros(B + 1, np.int32)
  node_ptr[1:] = np.cumsum(sizes)
  edge_ptr = np.zeros(B + 1, np.int32)
  edge_ptr[1:] = np.cumsum([len(s['edges']) for s in samples])
  feats = [np.asarray(s['node_feat']) for s in samples]
  if feats[0].ndim == 2:               # float features: each fp64 value rounded once, as collate's float32 rows
    node_feat = np.concatenate([f.astype(np.float32) for f in feats]).reshape(-1, feats[0].shape[1])
  else:
    node_feat = np.concatenate([f.astype(np.int32) for f in feats])
  edges = np.zeros((int(edge_ptr[-1]), 4), np.uint8)
  for b, s in enumerate(samples):
    edges[edge_ptr[b]:edge_ptr[b + 1], :3] = s['edges']
  out = {'sizes': sizes, 'node_ptr': node_ptr, 'node_feat': node_feat, 'edge_ptr': edge_ptr, 'edges': edges}
  if eigs:
    D = np.zeros((B, num_eigs), np.float32)
    V_rows = np.zeros((int(node_ptr[-1]), num_eigs), np.float32)
    for b, s in enumerate(samples):
      kk = min(num_eigs, s['D_simple'].shape[0])
      D[b, :kk] = s['D_simple'][:kk]
      V_rows[node_ptr[b]:node_ptr[b + 1], :kk] = s['V_simple'][:, :kk]
    out['D'], out['V_rows'] = D, V_rows
  else:
    out['K'] = int(num_eigs)
  out['N'], out['num_edgetype'] = int(sizes.max()), int(samples[0]['L_multi'].shape[2])
  if 'label' in samples[0]:
    out['label'] = np.concatenate([np.asarray(s['label'], np.float32).reshape(1, -1)
                                   for s in samples], axis=0)
  return out


PACK_MAGIC = 0x4c4e4231          # "LNB1"

# the int32 slots of a packed batch's header in slot order: LNB_PACK_HDR_* of include/lanczosnet_b200.h
PackHeader = collections.namedtuple('PackHeader', 'magic B K sizes node_ptr edge_ptr D node_feat V_rows edges '
                                                  'total tiles krow label P F')
PackedOffsets = collections.namedtuple('PackedOffsets', 'sizes node_ptr edge_ptr D var tiles krow')


def _align16(x):
  return (int(x) + 15) & ~15


def packed_offsets(B, K):
  """Byte offsets of the segments of a packed batch that depend on B and K only (a PackedOffsets); ``var``
  is where the node ids of a batch with eigenpairs start."""
  off_sizes = 64
  off_node_ptr = off_sizes + _align16(4 * B)
  off_edge_ptr = off_node_ptr + _align16(4 * (B + 1))
  off_D = off_edge_ptr + _align16(4 * (B + 1))
  off_tiles = off_D + _align16(4 * B * K)
  off_krow = off_tiles + _align16(4 * tile_segment_ints(B))
  off_var = off_krow + _align16(4 * (B + 1))
  return PackedOffsets(off_sizes, off_node_ptr, off_edge_ptr, off_D, off_var, off_tiles, off_krow)


def packed_layout(B, K, rows, nedges, eigs, P=0, F=0):
  """The PackHeader of a packed batch of B graphs with ``rows`` nodes and ``nedges`` bonds in all.  Without
  ``eigs`` there is no D, V_rows, tiles or krow segment, and the node ids start where D would.  P > 0: a label
  segment [B, P] float32 behind the bonds.  F > 0: the node segment holds float32 feature rows [rows, F]
  instead of int32 atom ids; every other rule is the same."""
  o = packed_offsets(B, K)
  node_bytes = 4 * rows * (F if F else 1)
  if eigs:
    D, node_feat, tiles, krow = o.D, o.var, o.tiles, o.krow
    V_rows = node_feat + _align16(node_bytes)
    edges = V_rows + _align16(4 * rows * K)
  else:
    D, node_feat, V_rows, tiles, krow = 0, o.D, 0, 0, 0
    edges = node_feat + _align16(node_bytes)
  label = edges + _align16(4 * nedges)
  total = label + _align16(4 * B * P)
  return PackHeader(PACK_MAGIC, B, K, o.sizes, o.node_ptr, o.edge_ptr, D, node_feat, V_rows, edges, total, tiles,
                    krow, label if P else 0, P, F)


def packed_capacity(B, N, K, eigs, nbytes, label_dim=0, feature_dim=0, num_edgetype=1):
  """Static size of a packed batch's blob under graph replay, or the blob's own ``nbytes`` when that is
  larger.  ``label_dim`` = P > 0 counts a label segment [B, P] float32 (pack_sparse(..., label=True)).

  Atom ids (``feature_dim`` = 0): the blob of any B molecules of at most N nodes and 4 N bonds each.  Float
  feature rows (``feature_dim`` = F > 0, GraphData graphs such as G(n, 0.5), far denser than molecules): the
  blob of ANY B graphs of at most N nodes, whose bond lists hold each (u <= v, bond type) pair at most once,
  as prepare_graph writes them: ``num_edgetype`` * N (N + 1) / 2 bonds per graph."""
  F = int(feature_dim)
  bonds = int(num_edgetype) * N * (N + 1) // 2 if F else 4 * N
  return max(packed_layout(B, K, B * N, B * bonds, eigs, int(label_dim), F).total, int(nbytes))


def read_packed_header(blob):
  """The PackHeader of a packed batch's blob (numpy array or torch tensor): a host blob is read in place, a
  device blob with one 64-byte copy."""
  head = blob[:64].cpu().numpy() if hasattr(blob, 'cpu') else blob[:64]
  return PackHeader(*head.view(np.int32)[:len(PackHeader._fields)].tolist())


def host_tile_table(sizes, k_eff, rows_per_tile=128, graphs_per_tile=32):
  """Packed-tile table of the fused convolution kernel, computed on the host with the rule of
  lnb_graph_prepare (csrc/spectral_conv_fused.cu: next-fit over consecutive graphs, sum n_eff <= 128,
  sum ceil4(k_eff) <= 128, <= 32 graphs per tile; the first graph of a tile always fits).
  Returns int32 [B+2]: [T, first graph of tile 0..T-1, B, 0 ...]."""
  B = len(sizes)
  tiles = np.zeros(B + 2, np.int32)
  if B == 0:
    return tiles
  cn = np.concatenate([[0], np.cumsum(np.asarray(sizes, np.int64))])
  ck = np.concatenate([[0], np.cumsum((np.asarray(k_eff, np.int64) + 3) // 4 * 4)])
  # jump table for EVERY start i at once (largest j with prefix[j] - prefix[i] <= limit: graphs i .. j-1
  # share a tile), then the tiles are the orbit of graph 0 -- the pointer-jumping form of tile_assign_kernel
  first = np.arange(B, dtype=np.int64)
  jn = np.searchsorted(cn, cn[:-1] + rows_per_tile, side='right') - 1
  jk = np.searchsorted(ck, ck[:-1] + rows_per_tile, side='right') - 1
  nxt = np.maximum(first + 1, np.minimum(np.minimum(jn, jk), np.minimum(first + graphs_per_tile, B))).tolist()
  starts, i = [], 0
  while i < B:
    starts.append(i)
    i = nxt[i]
  T = len(starts)
  tiles[1:1 + T] = starts
  tiles[0] = T
  tiles[1 + T] = B
  return tiles


def tile_segment_ints(B):
  """Size in ints of the tile segment of a packed batch: the next-fit table [B + 2] followed by the
  tile schedule [2B + 2] (fixed size, so the segments behind it stay where (B, K) puts them)."""
  return 3 * B + 4


def host_tile_segment(sizes, k_eff):
  """The tile segment of a packed batch: next-fit table, then the tile schedule (int32 [3B + 4])."""
  return np.concatenate([host_tile_table(sizes, k_eff), host_tile_schedule(sizes, k_eff)])


def host_tile_schedule(sizes, k_eff, rows_per_tile=128, graphs_per_tile=32):
  """The tile schedule the fused convolution kernel runs (csrc/spectral_conv_fused.cu,
  tile_assign_kernel): first-fit decreasing.  Graphs are taken by n_eff descending, then k_eff
  descending, then index ascending; each goes into the lowest-numbered tile where sum n_eff <= 128,
  sum k_eff <= 128 (not rounded up to 4) and <= 32 graphs still hold, or opens a new tile (a lone graph
  always fits).  Inside a tile the graphs are listed in placement order.

  Vectorised over classes of identical (n_eff, k_eff): for identical graphs, giving every tile, lowest
  first, as many as still fit is what first-fit does one graph at a time.
  Returns int32 [2B+2]: [T', first slot of tile 0 .. T' (the last = B), graph ids in tile order, 0 ...]."""
  n = np.asarray(sizes, np.int64)
  k = np.asarray(k_eff, np.int64)
  B = len(n)
  out = np.zeros(2 * B + 2, np.int32)
  if B == 0:
    return out
  R, G = rows_per_tile, graphs_per_tile
  order = np.lexsort((np.arange(B), -k, -n))
  sn, sk = n[order], k[order]
  cut = np.flatnonzero((sn[1:] != sn[:-1]) | (sk[1:] != sk[:-1])) + 1
  bounds = np.concatenate([[0], cut, [B]])
  tn, tk, tc = (np.zeros(B, np.int64) for _ in range(3))      # per tile: sum n_eff, sum k_eff, graphs
  rec_t, rec_src, rec_slot, rec_m = [], [], [], []              # placements, in placement order
  T = 0
  for first, end in zip(bounds[:-1].tolist(), bounds[1:].tolist()):
    cn, ck, count = int(sn[first]), int(sk[first]), end - first
    done = 0
    if T:
      cap = G - tc[:T]
      if cn:
        cap = np.minimum(cap, (R - tn[:T]) // cn)
      if ck:
        cap = np.minimum(cap, (R - tk[:T]) // ck)
      cap = np.maximum(cap, 0)
      inc = np.cumsum(cap)
      m = np.clip(count - (inc - cap), 0, cap)
      t = np.flatnonzero(m)
      rec_t.append(t)
      rec_src.append(first + (inc - cap)[t])
      rec_slot.append(tc[t].copy())
      rec_m.append(m[t])
      tn[:T] += m * cn
      tk[:T] += m * ck
      tc[:T] += m
      done = min(count, int(inc[-1]))
    if done < count:                                            # new tiles, each as full as the limits allow
      ce = max(1, min(G, R // cn if cn else G, R // ck if ck else G))
      rem = count - done
      nt = -(-rem // ce)
      m = np.full(nt, ce, np.int64)
      m[-1] = rem - (nt - 1) * ce
      t = T + np.arange(nt)
      rec_t.append(t)
      rec_src.append(first + done + ce * np.arange(nt))
      rec_slot.append(np.zeros(nt, np.int64))
      rec_m.append(m)
      tn[t], tk[t], tc[t] = m * cn, m * ck, m
      T += nt
  rec_t, rec_src, rec_slot, rec_m = (np.concatenate(a) for a in (rec_t, rec_src, rec_slot, rec_m))
  starts = np.zeros(T + 1, np.int64)
  starts[1:] = np.cumsum(tc[:T])
  pos = np.zeros(B, np.int64)
  pos[PackedMolecules._ranges(rec_src, rec_m)] = PackedMolecules._ranges(starts[rec_t] + rec_slot, rec_m)
  out[0] = T
  out[1:T + 2] = starts
  out[T + 2 + pos] = order
  return out


def ritz_extents(V_rows, node_ptr):
  """k_eff per graph = last non-zero column of its Ritz rows + 1 (what the device measures in
  lnb_graph_prepare); vectorised over the batch (every graph has at least one node)."""
  B, K = len(node_ptr) - 1, V_rows.shape[1]
  if B == 0:
    return np.zeros(0, np.int64)
  any_col = np.logical_or.reduceat(V_rows != 0, np.asarray(node_ptr[:-1], np.int64), axis=0)   # [B, K]
  last = K - np.argmax(any_col[:, ::-1], axis=1)
  return np.where(any_col.any(axis=1), last, 0).astype(np.int64)


def pack_sparse(sp, label=False):
  """A ``sparse_collate`` batch as ONE contiguous uint8 buffer (layout: include/lanczosnet_b200.h,
  lnb_graph_prepare_sparse_packed): a 16-int header with the byte offsets of the segments, the
  fixed-size segments (sizes, node_ptr, edge_ptr, D), then node ids, Ritz rows and the bond list.
  One H2D copy per step ships the whole batch.  Records without eigenpairs (``sparse_collate(...,
  eigs=False)``) give a blob without D, Ritz rows, tiles and Ritz-row offsets (their header offsets are 0):
  the node ids start where D would.  ``label=True``: the records' labels [B, P] float32 follow the bonds as
  one more segment (slots label and P), for training from the blob (train.GraphedStep(..., packed=True));
  every other byte is that of the blob without them.  Records whose ``node_feat`` is 2-D (float feature rows
  [sum n, F], sparse_collate of GraphData samples) give a blob of feature rows: header slot F, 4 F bytes per node
  in the node segment, everything else as for atom ids.  Returns dict(blob, B, N, K, num_edgetype, eigs, F[, label])
  with F = 0 for atom ids."""
  eigs = 'D' in sp
  F = int(sp['node_feat'].shape[1]) if sp['node_feat'].ndim == 2 else 0
  if label and 'label' not in sp:
    raise ValueError('pack_sparse: label=True needs records with labels (samples with a label)')
  B, K = sp['D'].shape if eigs else (len(sp['sizes']), int(sp['K']))
  lab = np.ascontiguousarray(sp['label'], np.float32).reshape(B, -1) if label else None
  h = packed_layout(B, K, len(sp['node_feat']), len(sp['edges']), eigs, lab.shape[1] if label else 0, F)
  segs = [(h.sizes, sp['sizes']), (h.node_ptr, sp['node_ptr']), (h.edge_ptr, sp['edge_ptr']),
          (h.node_feat, sp['node_feat']), (h.edges, sp['edges'])]
  if eigs:
    # extents the device would measure: k_eff = last non-zero column of the graph's Ritz rows + 1
    k_eff = ritz_extents(sp['V_rows'], sp['node_ptr'])
    krow = np.zeros(B + 1, np.int32)
    krow[1:] = np.cumsum(np.minimum(k_eff, K))
    segs += [(h.tiles, host_tile_segment(sp['sizes'], k_eff)), (h.krow, krow), (h.D, sp['D']),
             (h.V_rows, sp['V_rows'])]
  if label:
    segs.append((h.label, lab))
  blob = np.zeros(h.total, np.uint8)
  blob[:64].view(np.int32)[:len(h)] = h
  for off, arr in segs:
    raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    blob[off:off + raw.size] = raw
  out = {'blob': blob, 'B': int(B), 'N': int(sp['N']), 'K': int(K), 'num_edgetype': int(sp['num_edgetype']),
         'eigs': eigs, 'F': F}
  if 'label' in sp:
    out['label'] = sp['label']
  return out


class PackedMolecules(object):
  """A whole split flattened ONCE into the segments of the packed batch format (node ids, bond lists,
  Ritz rows, Ritz values, extents): a batch over any index set is then a handful of vectorised gathers
  into one buffer -- the blob of ``pack_sparse(sparse_collate([samples[i] for i in idx], K))``, byte for
  byte -- instead of a Python loop over molecules per step (the reference pads and stacks per batch in
  DataLoader workers, dataset/qm8.py:220-291).  At 1024 molecules: ~1 ms per batch against 9 ms for
  sparse_collate + pack_sparse and 33 ms for the padded collate, i.e. one loader thread keeps up with
  a GPU step of 0.5 ms only with this path.

  ``eigs=False`` takes ``prepare_graph(..., eigs=False)`` samples (or ignores the eigenpairs of any
  others): the blobs are those of ``pack_sparse(sparse_collate(..., eigs=False))``, 4 bytes per node instead
  of 4 (K + 1), and the device computes the eigenpairs where a model reads them.

  ``labels=True`` writes each batch's labels into the blob, as ``pack_sparse(..., label=True)`` does: the
  batches train.GraphedStep(..., packed=True) trains from.

  Samples with float feature rows (GraphData records, ``node_feat`` [n, F]) give blobs of feature rows, those
  of ``pack_sparse`` for such records (header slot F = the feature width)."""

  def __init__(self, samples, num_eigs, eigs=True, labels=False):
    sp = sparse_collate(samples, num_eigs, eigs=eigs)
    if labels and 'label' not in sp:
      raise ValueError('PackedMolecules: labels=True needs samples with a label')
    self.K = int(num_eigs)
    self.eigs = bool(eigs)
    self.labels = bool(labels)
    self.num_edgetype = sp['num_edgetype']
    self.sizes, self.node_ptr, self.edge_ptr = sp['sizes'], sp['node_ptr'].astype(np.int64), sp['edge_ptr'].astype(np.int64)
    self.node_feat, self.edges, self.V_rows, self.D = sp['node_feat'], sp['edges'], sp.get('V_rows'), sp.get('D')
    self.k_eff = ritz_extents(self.V_rows, self.node_ptr) if eigs else None
    self.label = sp.get('label')
    self.F = int(self.node_feat.shape[1]) if self.node_feat.ndim == 2 else 0

  def __len__(self):
    return len(self.sizes)

  @staticmethod
  def _ranges(starts, lens):
    """Concatenation of arange(starts[i], starts[i] + lens[i]) without a Python loop."""
    total = int(lens.sum())
    if total == 0:
      return np.zeros(0, np.int64)
    ends = np.cumsum(lens)
    return np.repeat(starts - (ends - lens), lens) + np.arange(total, dtype=np.int64)

  def max_bytes(self, B):
    """Upper bound of the blob of any B molecules, repeats included (for a reusable pinned staging
    buffer): an index list may repeat the largest molecule B times."""
    P = self.label.shape[1] if self.labels else 0
    return packed_layout(B, self.K, B * int(self.sizes.max()), B * int(np.diff(self.edge_ptr).max()), self.eigs,
                         P, self.F).total

  def batch(self, idx, out=None):
    """Packed batch of the molecules ``idx`` (order kept).  ``out``: optional uint8 buffer (e.g. the numpy
    view of a pinned tensor) of at least the blob's size; the returned blob is a view of it."""
    idx = np.asarray(idx, np.int64)
    B, K = len(idx), self.K
    sizes = self.sizes[idx]
    n_len = sizes.astype(np.int64)
    e_len = self.edge_ptr[idx + 1] - self.edge_ptr[idx]
    node_ptr = np.zeros(B + 1, np.int32)
    node_ptr[1:] = np.cumsum(n_len)
    edge_ptr = np.zeros(B + 1, np.int32)
    edge_ptr[1:] = np.cumsum(e_len)
    rows = self._ranges(self.node_ptr[idx], n_len)
    erow = self._ranges(self.edge_ptr[idx], e_len)
    P = self.label.shape[1] if self.labels else 0
    F = self.F
    node_bytes = 4 * len(rows) * (F if F else 1)
    h = packed_layout(B, K, len(rows), len(erow), self.eigs, P, F)
    if out is None:
      blob = np.zeros(h.total, np.uint8)
    else:
      if out.dtype != np.uint8 or out.ndim != 1 or out.size < h.total:
        raise ValueError('PackedMolecules.batch: out must be a flat uint8 buffer of >= %d bytes' % h.total)
      blob = out[:h.total]
      blob[:h.node_feat] = 0                         # header + fixed segments (alignment gaps stay zero)
      body = [(off, n) for off, n in ((h.node_feat, node_bytes), (h.V_rows, 4 * len(rows) * K),
                                      (h.edges, 4 * len(erow)), (h.label, 4 * B * P)) if off]
      for (off, n), end in zip(body, [off for off, _ in body[1:]] + [h.total]):
        blob[off + n:end] = 0                        # the alignment gap behind each segment
    blob[:64].view(np.int32)[:len(h)] = h

    def put(off, arr):
      raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
      blob[off:off + raw.size] = raw

    if self.eigs:
      k_eff = self.k_eff[idx]
      krow = np.zeros(B + 1, np.int32)
      krow[1:] = np.cumsum(np.minimum(k_eff, K))
      put(h.tiles, host_tile_segment(sizes, k_eff))
      put(h.krow, krow)
      put(h.D, self.D[idx])
      np.take(self.V_rows, rows, axis=0,
              out=blob[h.V_rows:h.V_rows + 4 * len(rows) * K].view(np.float32).reshape(len(rows), K))
    put(h.sizes, sizes)
    put(h.node_ptr, node_ptr)
    put(h.edge_ptr, edge_ptr)
    if F:
      np.take(self.node_feat, rows, axis=0,
              out=blob[h.node_feat:h.node_feat + node_bytes].view(np.float32).reshape(len(rows), F))
    else:
      np.take(self.node_feat, rows, out=blob[h.node_feat:h.node_feat + node_bytes].view(np.int32))
    np.take(self.edges, erow, axis=0, out=blob[h.edges:h.edges + 4 * len(erow)].reshape(len(erow), 4))
    if self.labels:
      np.take(self.label, idx, axis=0, out=blob[h.label:h.label + 4 * B * P].view(np.float32).reshape(B, P))
    res = {'blob': blob, 'B': int(B), 'N': int(sizes.max()) if B else 0, 'K': K, 'num_edgetype': self.num_edgetype,
           'eigs': self.eigs, 'F': F}
    if self.label is not None:
      res['label'] = self.label[idx]
    return res


# ----------------------------------------------------------------------------
# synthetic inputs (no dataset can be downloaded; shapes follow the reference)
# ----------------------------------------------------------------------------
def synthetic_molecule(rng, num_nodes, num_bond_type=6, num_atom=70, max_degree=4,
                       extra_edge_frac=0.3):
  """Random connected, degree-capped, molecule-like multigraph.

  A random spanning tree (each new atom bonds to a random earlier atom with free valence)
  plus ~extra_edge_frac*n ring-closing bonds; every bond gets one of num_bond_type channels.
  Returns (node_feat (n,) int64 in [0,num_atom), adjs (n,n,num_bond_type) float64)."""
  n = int(num_nodes)
  adjs = np.zeros((n, n, num_bond_type), np.float64)
  deg = np.zeros(n, np.int64)
  for v in range(1, n):
    free = np.flatnonzero(deg[:v] < max_degree)
    u = int(free[rng.randint(len(free))]) if len(free) else int(rng.randint(v))
    c = int(rng.randint(num_bond_type))
    adjs[u, v, c] = adjs[v, u, c] = 1.0
    deg[u] += 1
    deg[v] += 1
  for _ in range(int(round(extra_edge_frac * n))):
    u, v = int(rng.randint(n)), int(rng.randint(n))
    if u == v or adjs[u, v].sum() > 0 or deg[u] >= max_degree or deg[v] >= max_degree:
      continue
    c = int(rng.randint(num_bond_type))
    adjs[u, v, c] = adjs[v, u, c] = 1.0
    deg[u] += 1
    deg[v] += 1
  node_feat = rng.randint(0, num_atom, size=n).astype(np.int64)
  return node_feat, adjs


def synthetic_qm8_sizes(rng, batch_size, min_nodes=3, max_nodes=26, mean_nodes=16.0):
  sizes = np.clip(np.rint(rng.normal(mean_nodes, 4.5, size=batch_size)), min_nodes,
                  max_nodes).astype(np.int64)
  sizes[rng.randint(batch_size)] = max_nodes      # batch-max padding target N = max_nodes
  return sizes


def synthetic_qm8_samples(batch_size, seed=1234, num_bond_type=6, num_atom=70, num_label=16,
                          max_nodes=26):
  """Per-molecule records of a QM8-shaped batch (SURVEY.md 8d config #2): n_b in [3,26], mean ~16."""
  rng = np.random.RandomState(seed)
  sizes = synthetic_qm8_sizes(rng, batch_size, max_nodes=max_nodes)
  samples = []
  for n in sizes:
    nf, adjs = synthetic_molecule(rng, n, num_bond_type, num_atom)
    samples.append(prepare_graph(adjs, nf, label=rng.randn(1, num_label)))
  return samples


def synthetic_qm8_batch(batch_size, seed=1234, num_eigs=20, num_bond_type=6, num_atom=70,
                        num_label=16, max_nodes=26):
  """QM8-shaped padded batch: ``collate`` of ``synthetic_qm8_samples``."""
  return collate(synthetic_qm8_samples(batch_size, seed, num_bond_type, num_atom, num_label,
                                       max_nodes), num_eigs)


def synthetic_regression_graphs(num_graphs=16, seed=123, min_num_nodes=20, max_num_nodes=100,
                                node_emb_dim=10, graph_emb_dim=2, edge_prob=0.5):
  """The reference's synthetic graph-regression set (dataset/get_graph_data.py:15-49):
  X ~ randn(n,10), A = G(n, 0.5) with one edge type, Y ~ randn(1,2).  Same RNG call order
  as the reference so identical seeds give identical graphs."""
  import networkx as nx
  rng = np.random.RandomState(seed)
  sizes = rng.randint(min_num_nodes, high=max_num_nodes + 1, size=num_graphs)
  out = []
  for n in sizes:
    X = rng.randn(n, node_emb_dim)
    g = nx.fast_gnp_random_graph(int(n), edge_prob, seed=int(rng.randint(1000)))
    A = np.asarray(nx.to_numpy_array(g), dtype=np.float64)[:, :, None]
    Y = rng.randn(1, graph_emb_dim)
    out.append(prepare_graph(A, X, label=Y))
  return out
