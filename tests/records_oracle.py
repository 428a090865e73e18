"""fp64 numpy reading of the sparse bond-list records that every device producer reads (sizes, node_ptr,
edge_ptr, edges = {u, v, bond type, 0}): ops.graph_prepare_sparse / _features / _packed,
ops.gat_bias_sparse, ops.graph_eigs_sparse, ops.spectral_partition_sparse and ops.sage_sample_sparse.
It does not go through data.prepare_graph, so it also reads records that prepare_graph never writes.

The rule, stated once, per graph b:
  * n = clamp(sizes[b], 0, N);
  * a record (u, v, c) counts only if u < n, v < n and c < E; every other record is ignored;
  * bond type c is a 0/1 adjacency A_c: a set, so a duplicate record, or (u, v) next to (v, u), counts
    once; a self-loop sets A_c[u, u];
  * the simple graph is sum_c A_c;
  * per channel (0 = the simple graph, 1 + c = bond type c) L4 = (s_i * m_ij) * s_j with m = I + A on the
    real nodes and s = np.power(deg, -0.5) (inf -> 0), in fp64, rounded once to fp32 -- the reference's
    order (utils/data_helper.py:92-116).

The second half is a seeded generator of adversarial record batches (multigraphs, ignored records, edge
sizes, degrees far above 255) that the GPU contract test runs every producer on.
"""
import numpy as np

from lanczosnetwork_b200 import data


# ---- reading ---------------------------------------------------------------------------------------
class Records(object):
  """The per-type adjacency sets of a record batch: n [B] int64, A [B, E, N, N] bool (symmetric)."""

  def __init__(self, sizes, edge_ptr, edges, N, E):
    sizes = np.asarray(sizes, np.int64)
    edge_ptr = np.asarray(edge_ptr, np.int64)
    edges = np.asarray(edges, np.uint8).reshape(-1, 4)
    B, N, E = len(sizes), int(N), int(E)
    self.N, self.E, self.B = N, E, B
    self.n = np.clip(sizes, 0, N)
    self.A = np.zeros((B, E, N, N), bool)
    if B and edge_ptr[-1] > edge_ptr[0]:
      rec = edges[edge_ptr[0]:edge_ptr[-1]].astype(np.int64)
      g = np.repeat(np.arange(B), np.diff(edge_ptr))
      u, v, c = rec[:, 0], rec[:, 1], rec[:, 2]
      keep = (u < self.n[g]) & (v < self.n[g]) & (c < E)
      g, u, v, c = g[keep], u[keep], v[keep], c[keep]
      self.A[g, c, u, v] = True
      self.A[g, c, v, u] = True

  def real(self):
    """[B, N] bool: the real nodes."""
    return np.arange(self.N)[None, :] < self.n[:, None]

  def mask(self):
    return self.real().astype(np.uint8)

  def multiplicity(self, channel):
    """m = I + A of one channel on the real nodes, fp64 [B, N, N] (channel 0: the simple graph)."""
    if channel == 0:
      a = self.A.sum(axis=1, dtype=np.float64)
    else:
      a = self.A[:, channel - 1].astype(np.float64)
    eye = np.eye(self.N, dtype=bool)[None] & self.real()[:, :, None]
    return a + eye

  def l4(self, channel=0):
    """The fp64 L4 of one channel [B, N, N], padded rows and columns 0."""
    m = self.multiplicity(channel)
    deg = m.sum(axis=2)
    with np.errstate(divide='ignore'):
      s = np.power(deg, -0.5)
    s[np.isinf(s)] = 0.0
    return (s[:, :, None] * m) * s[:, None, :]

  def degrees(self):
    """[B, N] int64: the simple-graph degree 1 + sum of multiplicities of every real node (0 on padding)."""
    return self.multiplicity(0).sum(axis=2).astype(np.int64)

  def operators(self):
    """L [B, N, N, E + 1] fp32: channel 0 the simple graph, channel 1 + c bond type c (collate's layout)."""
    return np.stack([self.l4(ch).astype(np.float32) for ch in range(self.E + 1)], axis=3)

  def pattern(self, channel):
    """[B, N, N] bool: the off-diagonal and self-loop entries of one channel (channel 0: any type)."""
    return self.A.any(axis=1) if channel == 0 else self.A[:, channel - 1]

  def gat_bias(self):
    """GAT's additive bias [B, N, N, E + 1] fp32: -0.0 on the diagonal of every node (padded ones too) and
    on the channel's bonds, -1e9 elsewhere (data.gat_bias's -1e9 * (1 - m))."""
    eye = np.eye(self.N, dtype=bool)[None]
    m = np.stack([(self.pattern(ch) | eye).astype(np.float64) for ch in range(self.E + 1)], axis=3)
    return (-1e9 * (1.0 - m)).astype(np.float32)

  def candidates(self):
    """The sampler's candidate columns, the non-zero columns of every L4 row (the pattern plus I), ascending,
    for the rows (b * N + n) * (E + 1) + e in that order; empty for padded nodes."""
    eye = np.eye(self.N, dtype=bool)[None]
    real = self.real()
    pats = np.stack([(self.pattern(ch) | eye) & real[:, :, None] for ch in range(self.E + 1)], axis=2)
    return [np.flatnonzero(row) for row in pats.reshape(-1, self.N)]


def pad_rows(rows, node_ptr, n, N):
  """Rows of real nodes [node_ptr[B], ...] -> padded [B, N, ...] (padded rows 0), as collate pads them."""
  rows = np.asarray(rows)
  out = np.zeros((len(n), N) + rows.shape[1:], rows.dtype)
  for b, nb in enumerate(n):
    out[b, :nb] = rows[node_ptr[b]:node_ptr[b] + nb]
  return out


def ell_rows(L, binarize=False):
  """lnb_graph_prepare's ELL rows of dense operators L [B, N, N, E1]: row n of channel ch lists the diagonal
  first (when non-zero), then the non-zero columns in ascending order.  Returns (val [B, E1, N(slot), N(row)]
  fp32, idx uint8 in the same layout, ell_max [B, E1] int32); slots >= a row's count are 0."""
  L = np.asarray(L, np.float32)
  B, N, _, E1 = L.shape
  Lc = L.transpose(0, 3, 1, 2)                                     # [B, E1, row, col]
  nz = Lc != 0
  col = np.arange(N)
  key = np.where(col[None, :] == col[:, None], -1, col[None, :])    # the diagonal sorts first
  key = np.where(nz, key[None, None], N + 1)
  order = np.argsort(key, axis=3, kind='stable')
  cnt = nz.sum(axis=3)
  live = col[None, None, None, :] < cnt[..., None]
  idx = np.where(live, order, 0)
  val = np.where(live, np.take_along_axis(Lc, order, axis=3), np.float32(0))
  if binarize:
    val = np.where(live, np.float32(1), np.float32(0))
  emax = cnt.max(axis=2).astype(np.int32) if N else np.zeros((B, E1), np.int32)
  return (np.ascontiguousarray(val.transpose(0, 1, 3, 2)).astype(np.float32),
          np.ascontiguousarray(idx.transpose(0, 1, 3, 2)).astype(np.uint8), emax)


# ---- adversarial record batches -------------------------------------------------------------------
BOUNDARY_NODES = (31, 32, 63, 64, 127)      # the 32-bit adjacency word edges


def _random_multigraph(rng, n, E, per_node=3, self_loops=True):
  """Records of a random multigraph: several types per pair, self-loops in some types, every boundary node
  bonded."""
  recs = []
  if n == 0:
    return recs
  for _ in range(per_node * n):
    u, v = int(rng.randint(n)), int(rng.randint(n))
    for c in rng.choice(E, size=int(rng.randint(1, min(E, 3) + 1)), replace=False):
      recs.append((u, v, int(c)))
  if self_loops:
    for u in rng.choice(n, size=max(1, n // 8), replace=True):
      recs.append((int(u), int(u), int(rng.randint(E))))
  for w in BOUNDARY_NODES:
    if w < n and n > 1:
      recs.append((w, int(rng.randint(n)), int(rng.randint(E))))
      recs.append((int(rng.randint(n)), w, int(rng.randint(E))))
  return recs


def _complete(n, types, self_loops=False):
  return [(u, v, c) for c in types for u in range(n) for v in range(u if self_loops else u + 1, n)]


def _noise(rng, recs, n, E, count):
  """Duplicates, reversed pairs, and records every producer must ignore: bond types >= E (up to 255) and
  endpoints >= n (up to 255, 128..255 included)."""
  out = list(recs)
  if recs:
    for i in rng.randint(len(recs), size=count):
      out.append(recs[i])                                       # duplicate
    for i in rng.randint(len(recs), size=count):
      u, v, c = recs[i]
      out.append((v, u, c))                                     # reversed
  for _ in range(count):
    u, v = int(rng.randint(max(n, 1))), int(rng.randint(max(n, 1)))
    out.append((u, v, int(rng.randint(E, 256))))                # type >= E
    out.append((int(rng.randint(n, 256)), v, int(rng.randint(E))))   # endpoint >= n
    out.append((u, int(rng.randint(max(n, 128), 256)), int(rng.randint(E))))
  return out


def _batch(name, N, E, graphs, rng, K=8):
  """A record batch from per-graph (n, records): records in shuffled order, random node ids and feature rows,
  Ritz rows with a graph-dependent number of trailing zero columns (so k_eff varies)."""
  B = len(graphs)
  sizes = np.array([n for n, _ in graphs], np.int32)
  node_ptr = np.zeros(B + 1, np.int32)
  node_ptr[1:] = np.cumsum(sizes)
  edge_ptr = np.zeros(B + 1, np.int32)
  edge_ptr[1:] = np.cumsum([len(r) for _, r in graphs])
  edges = np.zeros((int(edge_ptr[-1]), 4), np.uint8)
  for b, (_, recs) in enumerate(graphs):
    if recs:
      r = np.array(recs, np.int64)[rng.permutation(len(recs))]
      edges[edge_ptr[b]:edge_ptr[b + 1], :3] = r
  rows = int(node_ptr[-1])
  V_rows = rng.randn(rows, K).astype(np.float32)
  for b in range(B):
    V_rows[node_ptr[b]:node_ptr[b + 1], (b * 3) % (K + 1):] = 0.0
  return {'name': name, 'N': int(N), 'E': int(E), 'sizes': sizes, 'node_ptr': node_ptr, 'edge_ptr': edge_ptr,
          'edges': edges, 'node_feat': rng.randint(0, 70, size=rows).astype(np.int32),
          'node_x': rng.randn(rows, 5).astype(np.float32), 'V_rows': V_rows}


def _qm8(seed=11, B=37):
  sp = data.sparse_collate(data.synthetic_qm8_samples(B, seed=seed), 8)
  rng = np.random.RandomState(seed)
  out = {k: sp[k] for k in ('sizes', 'node_ptr', 'edge_ptr', 'edges', 'node_feat', 'V_rows')}
  out.update(name='qm8', N=sp['N'], E=sp['num_edgetype'],
             node_x=rng.randn(int(sp['node_ptr'][-1]), 5).astype(np.float32))
  return out


def _multigraphs(N, seed):
  """Sizes N, 0 (with records, all ignored), 1 (self-loops only), N without a record between non-empty
  ranges, then random sizes; B not a multiple of 4 at N <= 32."""
  rng = np.random.RandomState(seed)
  E = 5
  B = 11 if N <= 32 else 9
  graphs = []
  for b in range(B):
    n = [N, 0, 1, N][b] if b < 4 else int(rng.randint(1, N + 1))
    if b == 3:
      graphs.append((n, []))
      continue
    recs = _random_multigraph(rng, n, E) if n > 1 else [(0, 0, c) for c in range(E)][:n * E]
    graphs.append((n, _noise(rng, recs, n, E, 4)))
  return _batch('multigraph_N%d' % N, N, E, graphs, rng)


def _no_edges(seed=5):
  rng = np.random.RandomState(seed)
  return _batch('no_edges', 40, 4, [(n, []) for n in (40, 0, 1, 17, 40, 3)], rng)


def _complete_three_types(seed=6):
  """A complete 128-node graph whose pairs each carry 3 bond types: deg = 1 + 3 * 127 = 382 (E1 = 4)."""
  rng = np.random.RandomState(seed)
  graphs = [(128, _noise(rng, _complete(128, range(3)), 128, 3, 6)),
            (100, _noise(rng, _random_multigraph(rng, 100, 3, per_node=20), 100, 3, 4)),
            (128, _noise(rng, _random_multigraph(rng, 128, 3, per_node=40), 128, 3, 4))]
  return _batch('complete_3types_N128', 128, 3, graphs, rng)


def _fifteen_types(seed=7):
  """15 bond types on 40 nodes (E1 = 16): complete in every type, self-loops included (deg = 1 + 15 * 40)."""
  rng = np.random.RandomState(seed)
  graphs = [(40, _noise(rng, _complete(40, range(15), self_loops=True), 40, 15, 6)),
            (40, _noise(rng, _random_multigraph(rng, 40, 15, per_node=40), 40, 15, 4)),
            (33, _noise(rng, _complete(33, range(0, 15, 2)), 33, 15, 4)),
            (37, _noise(rng, _random_multigraph(rng, 37, 15, per_node=30), 37, 15, 4)),
            (40, _noise(rng, _random_multigraph(rng, 40, 15, per_node=60), 40, 15, 4))]
  return _batch('types15_N40', 40, 15, graphs, rng)


def _dense_32_types(N, seed):
  """E = 32 (the eigensolver's and the partition's limit): every pair carries a random half of the 32 types
  (degrees in the thousands at N = 128); graph 0 carries all 32 on every pair and every node, the largest
  degree the envelope allows, 1 + 32 * N."""
  rng = np.random.RandomState(seed)
  graphs = [(N, _complete(N, range(32), self_loops=True))]
  for b in range(1, 5 if N <= 32 else 3):
    n = N if b == 1 else int(rng.randint(N // 2, N + 1))
    up = np.triu(np.ones((n, n), bool), 1)
    us, vs = np.nonzero(up)
    recs = [(int(u), int(v), c) for u, v in zip(us, vs) for c in np.flatnonzero(rng.rand(32) < 0.5)]
    graphs.append((n, _noise(rng, recs, n, 32, 4)))
  return _batch('types32_N%d' % N, N, 32, graphs, rng)


MULTIGRAPH_N = (1, 31, 32, 33, 64, 96, 127, 128)
CASES = (['qm8', 'no_edges', 'complete_3types_N128', 'types15_N40', 'types32_N32', 'types32_N128'] +
         ['multigraph_N%d' % N for N in MULTIGRAPH_N])


def adversarial_batch(name):
  """The record batch of one case of CASES: dict(name, N, E, sizes, node_ptr, edge_ptr, edges, node_feat,
  node_x, V_rows), numpy, seeded."""
  if name == 'qm8':
    return _qm8()
  if name == 'no_edges':
    return _no_edges()
  if name == 'complete_3types_N128':
    return _complete_three_types()
  if name == 'types15_N40':
    return _fifteen_types()
  if name.startswith('types32_N'):
    N = int(name[len('types32_N'):])
    return _dense_32_types(N, seed=N)
  if name.startswith('multigraph_N'):
    N = int(name[len('multigraph_N'):])
    return _multigraphs(N, seed=100 + N)
  raise KeyError(name)


def read(batch, E=None):
  """Records of an adversarial batch read with E bond types (default: the batch's own E)."""
  return Records(batch['sizes'], batch['edge_ptr'], batch['edges'], batch['N'], batch['E'] if E is None else E)
