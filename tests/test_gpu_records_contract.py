"""Every device producer that reads bond-list records held to one contract: the fp64 reading of the records
in tests/records_oracle.py.  The batches are adversarial (multigraphs, self-loops, duplicated, reversed and
unsorted records, empty edge ranges, a batch without a single record, bond types >= E and endpoints >= n
that must be ignored, sizes 0, 1 and N across the 32-bit word boundaries, simple-graph degrees up to
1 + 32 * 128), plus a clean QM8-shaped batch.  Producers: graph_prepare_sparse / _features / _packed,
graph_eigs_sparse, spectral_partition_sparse, gat_bias_sparse and sage_sample_sparse.  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch

import partition_oracle
import records_oracle as ro
import sage_sample_oracle
from lanczosnetwork_b200 import data, ops
from test_gpu_graph_eigs import _check_eigenpairs
from test_gpu_sage_sampling import _ell_equal

pytestmark = pytest.mark.gpu

PARTITIONS = 3
SAGE_K = 6
SAGE_KEYS = [(1234, 0), (2 ** 40 + 17, 2 ** 35 + 3)]
_BATCHES = {}


def dev():
  return torch.device('cuda:0')


def _batch(name):
  if name not in _BATCHES:
    _BATCHES[name] = ro.adversarial_batch(name)
  return _BATCHES[name]


def _cuda(bt):
  return {k: torch.from_numpy(np.ascontiguousarray(bt[k])).to(dev())
          for k in ('sizes', 'node_ptr', 'edge_ptr', 'edges', 'node_feat', 'node_x', 'V_rows')}


def _prep_types(bt):
  """Bond types the E1 <= 16 producers read (types >= E1 - 1 are ignored)."""
  return min(bt['E'], 15)


def _bits(t):
  t = t.cpu() if torch.is_tensor(t) else torch.from_numpy(np.ascontiguousarray(t))
  return t.view(torch.int32) if t.dtype == torch.float32 else t


def _equal_bits(got, want, what):
  g, w = _bits(got), _bits(want)
  assert g.shape == w.shape, (what, tuple(g.shape), tuple(w.shape))
  bad = (g != w)
  assert not bool(bad.any()), (what, int(bad.sum()), [tuple(i) for i in bad.nonzero()[:5].tolist()])


def _k_eff(V_rows, node_ptr, n):
  """Last non-zero Ritz column + 1 of every graph's rows (0 for a graph without nodes)."""
  out = np.zeros(len(n), np.int32)
  for b, nb in enumerate(n):
    cols = np.flatnonzero((V_rows[node_ptr[b]:node_ptr[b] + nb] != 0).any(axis=0))
    out[b] = cols[-1] + 1 if len(cols) else 0
  return out


def _check_ell(prep, want, what):
  """ELL rows on every slot below ell_max (the slots a consumer reads), ell_max itself."""
  val, idx, emax = want
  _equal_bits(prep[2], emax, what + ' ell_max')
  N = val.shape[2]
  live = torch.from_numpy(np.arange(N)[None, None, :, None] < emax[:, :, None, None]).expand(val.shape)
  _equal_bits(prep[0].cpu()[live], torch.from_numpy(val)[live], what + ' ell_val')
  _equal_bits(prep[1].cpu()[live], torch.from_numpy(idx)[live], what + ' ell_idx')


@pytest.mark.parametrize('binarize', [False, True], ids=['l4', 'binarized'])
@pytest.mark.parametrize('name', ro.CASES)
def test_graph_prepare_sparse_entries_equal_the_oracle(name, binarize):
  bt = _batch(name)
  N, E = bt['N'], _prep_types(bt)
  rec = ro.read(bt, E)
  L = rec.operators()
  ell = ro.ell_rows(L, binarize)
  gext = np.stack([rec.n, _k_eff(bt['V_rows'], bt['node_ptr'], rec.n)], axis=1).astype(np.int32)
  V = ro.pad_rows(bt['V_rows'], bt['node_ptr'], rec.n, N)
  t = _cuda(bt)
  K = bt['V_rows'].shape[1]
  prep, ids, mask, Vd, Ld = ops.graph_prepare_sparse(t['sizes'], t['node_ptr'], t['node_feat'], t['edge_ptr'],
                                                     t['edges'], t['V_rows'], N, E + 1, binarize=binarize,
                                                     want_dense=True)
  prep_f, X, mask_f, V_f, L_f = ops.graph_prepare_sparse_features(
      t['sizes'], t['node_ptr'], t['node_x'], t['edge_ptr'], t['edges'], t['V_rows'], N, E + 1, binarize=binarize,
      want_dense=True)
  sp = {k: bt[k] for k in ('sizes', 'node_ptr', 'node_feat', 'edge_ptr', 'edges', 'V_rows')}
  sp.update(D=np.zeros((len(bt['sizes']), K), np.float32), N=N, num_edgetype=E)
  pk = data.pack_sparse(sp)
  prep_p, ids_p, mask_p, V_p, L_p = ops.graph_prepare_sparse_packed(
      torch.from_numpy(pk['blob']).to(dev()), len(bt['sizes']), N, E + 1, K, binarize=binarize, want_dense=True)
  _equal_bits(ids, ro.pad_rows(bt['node_feat'], bt['node_ptr'], rec.n, N).astype(np.int64), 'node ids')
  _equal_bits(X, ro.pad_rows(bt['node_x'], bt['node_ptr'], rec.n, N), 'X')
  for what, (p, m, v, l) in (('sparse', (prep, mask, Vd, Ld)), ('features', (prep_f, mask_f, V_f, L_f)),
                             ('packed', (prep_p, mask_p, V_p, L_p))):
    what = '%s %s' % (name, what)
    _equal_bits(l, L, what + ' L')
    _equal_bits(m, rec.mask(), what + ' mask')
    _equal_bits(v, V, what + ' V')
    _check_ell(p, ell, what)
    _equal_bits(p[3], gext, what + ' gext')
  _equal_bits(ids_p, ids, 'packed node ids')


@pytest.mark.parametrize('name', ro.CASES)
def test_graph_eigs_sparse_equals_eigh_of_the_oracle(name):
  bt = _batch(name)
  N, E = bt['N'], bt['E']
  rec = ro.read(bt)
  A64 = rec.l4(0)
  t = _cuda(bt)
  K = N
  D, V_rows, status = ops.graph_eigs_sparse(t['sizes'], t['node_ptr'], t['edge_ptr'], t['edges'], N, K,
                                            num_edgetype=E)
  assert not status.cpu().numpy().any(), (name, status.cpu().numpy())
  D, V_rows = D.cpu().numpy(), V_rows.cpu().numpy()
  ptr = bt['node_ptr']
  for b, n in enumerate(rec.n):
    if n == 0:
      assert not D[b].any(), (name, b)
      continue
    _check_eigenpairs(D[b], V_rows[ptr[b]:ptr[b] + n], A64[b, :n, :n], K, (name, b, int(rec.degrees()[b].max())))


@pytest.mark.parametrize('name', ro.CASES)
def test_spectral_partition_sparse_equals_the_oracle(name):
  bt = _batch(name)
  N, E, P = bt['N'], bt['E'], PARTITIONS
  if not ops.spectral_partition_supported(N, P):
    pytest.skip('N=%d outside the partition envelope at P=%d' % (N, P))
  rec = ro.read(bt)
  A64 = rec.l4(0)
  t = _cuda(bt)
  labels, status, prep, Lc, Lt = ops.spectral_partition_sparse(t['sizes'], t['edge_ptr'], t['edges'], N, P, E,
                                                               want_dense=True)
  lab, st = labels.cpu().numpy(), status.cpu().numpy()
  assert not (st & 0b1001).any(), (name, st)
  # the operators of the kernel's own labels
  want_c, want_t = data.partition_operators(A64, lab)
  _equal_bits(Lc, want_c, name + ' L_cluster')
  _equal_bits(Lt, want_t, name + ' L_cut')
  _check_ell(prep, ro.ell_rows(np.stack([want_c, want_t], axis=3)), name + ' partition')
  _equal_bits(prep[3], np.tile(np.array([[N, 0]], np.int32), (len(lab), 1)), name + ' partition gext')
  # the labels, wherever the reference's partition is determined
  if name == 'no_edges':
    assert (lab == -1).all()
    return
  qualified = 0
  for b in range(len(lab)):
    if st[b] & 0b110:
      continue
    orc = partition_oracle.spectral_clustering(A64[b], P)
    if orc['tie'] or orc['kmeans_tie']:
      continue
    assert np.array_equal(lab[b], orc['labels']), (name, b, lab[b], orc['labels'])
    qualified += 1
  assert 2 * qualified > len(lab), (name, qualified, len(lab))


@pytest.mark.parametrize('name', ro.CASES)
def test_gat_bias_sparse_equals_the_oracle(name):
  bt = _batch(name)
  E = _prep_types(bt)
  t = _cuda(bt)
  bias = ops.gat_bias_sparse(t['sizes'], t['edge_ptr'], t['edges'], bt['N'], E + 1)
  _equal_bits(bias, ro.read(bt, E).gat_bias(), name + ' gat bias')


@pytest.mark.parametrize('name', ro.CASES)
def test_sage_sample_sparse_equals_the_oracle(name):
  bt = _batch(name)
  N, E = bt['N'], _prep_types(bt)
  E1, B = E + 1, len(bt['sizes'])
  rec = ro.read(bt, E)
  cands = rec.candidates()
  t = _cuda(bt)
  for key in SAGE_KEYS:
    x = sage_sample_oracle.draws(key, np.arange(B * N * E1), SAGE_K)
    want = sage_sample_oracle.sample_rows(cands, x, SAGE_K).reshape(B, N, E1, SAGE_K).transpose(0, 1, 3, 2)
    ids, mask, nonempty, nn_idx, prep, prep_t = ops.sage_sample_sparse(
        t['sizes'], t['node_ptr'], t['node_feat'], t['edge_ptr'], t['edges'],
        torch.tensor(key, dtype=torch.int64, device=dev()), N, E1, SAGE_K, want_ell=True, want_ell_t=True)
    _equal_bits(nn_idx, np.ascontiguousarray(want), '%s %s nn_idx' % (name, key))
    _equal_bits(nonempty.view(B, N), rec.real().astype(np.float32), name + ' nonempty')
    _equal_bits(mask, rec.mask(), name + ' mask')
    _equal_bits(ids, ro.pad_rows(bt['node_feat'], bt['node_ptr'], rec.n, N).astype(np.int64), name + ' ids')
    M = ops.sage_operators(nn_idx.long(), nonempty)
    _ell_equal(prep, ops.graph_prepare(M))
    _ell_equal(prep_t, ops.graph_prepare(M.transpose(1, 2).contiguous()))


def test_empty_batch_launches_nothing():
  """B = 0: every producer returns empty outputs without a launch or an error."""
  z = lambda *shape, dtype=torch.int32: torch.zeros(shape, dtype=dtype, device=dev())
  sizes, ptr, edges = z(0), z(1), z(0, 4, dtype=torch.uint8)
  feat, x, V_rows = z(0), z(0, 5, dtype=torch.float32), z(0, 8, dtype=torch.float32)
  N, E1, K = 40, 7, 8
  key = torch.tensor(SAGE_KEYS[0], dtype=torch.int64, device=dev())
  ops._partition_draws_table(dev(), N, PARTITIONS, 1234)         # the host-built table, outside the count
  torch.cuda.synchronize()
  n0 = ops.launch_count()
  outs = [ops.graph_prepare_sparse(sizes, ptr, feat, ptr, edges, V_rows, N, E1, want_dense=True),
          ops.graph_prepare_sparse_features(sizes, ptr, x, ptr, edges, V_rows, N, E1, want_dense=True),
          ops.graph_eigs_sparse(sizes, ptr, ptr, edges, N, K, num_edgetype=32),
          ops.spectral_partition_sparse(sizes, ptr, edges, N, PARTITIONS, 32, want_dense=True),
          (ops.gat_bias_sparse(sizes, ptr, edges, N, E1),),
          ops.sage_sample_sparse(sizes, ptr, feat, ptr, edges, key, N, E1, SAGE_K, want_ell=True, want_ell_t=True)]
  sp = dict(sizes=np.zeros(0, np.int32), node_ptr=np.zeros(1, np.int32), node_feat=np.zeros(0, np.int32),
            edge_ptr=np.zeros(1, np.int32), edges=np.zeros((0, 4), np.uint8), V_rows=np.zeros((0, K), np.float32),
            D=np.zeros((0, K), np.float32), N=N, num_edgetype=E1 - 1)
  outs.append(ops.graph_prepare_sparse_packed(torch.from_numpy(data.pack_sparse(sp)['blob']).to(dev()), 0, N, E1,
                                              K, want_dense=True))
  torch.cuda.synchronize()
  assert ops.launch_count() == n0
  for out in outs:
    for o in out:
      for a in (o if isinstance(o, tuple) else (o,)):
        if torch.is_tensor(a) and a.dim() >= 2:
          assert a.shape[0] == 0, tuple(a.shape)


def test_degree_table_on_the_device():
  t = ops._inv_sqrt_deg_table(dev()).cpu().numpy()
  assert t.shape == (ops.INV_SQRT_DEG_LEN,) and t.dtype == np.float64 and t[0] == 0.0
  assert np.array_equal(t[1:], np.power(np.arange(1, ops.INV_SQRT_DEG_LEN, dtype=np.float64), -0.5))
