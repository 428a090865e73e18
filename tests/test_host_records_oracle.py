"""The fp64 reading of bond-list records (tests/records_oracle.py) pinned on the CPU: on the records of
clean ``prepare_graph`` samples it is ``data.collate`` and ``data.gat_bias`` bit for bit; duplicates,
reversed pairs and ignored records change nothing; the adversarial batches the GPU contract test runs
reach what they claim to (degrees above 255, ignored records, bonded word-boundary nodes); and the
deg^-1/2 table covers every degree the producers' envelope allows."""
import os
import re

import numpy as np
import pytest

import records_oracle as ro
from lanczosnetwork_b200 import data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('seed', [0, 3, 17, 2024])
def test_oracle_equals_collate_on_clean_records(seed):
  samples = data.synthetic_qm8_samples(24, seed=seed)
  dense = data.collate(samples, 12)
  sp = data.sparse_collate(samples, 12)
  rec = ro.Records(sp['sizes'], sp['edge_ptr'], sp['edges'], sp['N'], sp['num_edgetype'])
  L = rec.operators()
  assert L.dtype == np.float32 and np.array_equal(L.view(np.int32), dense['L'].view(np.int32))
  assert np.array_equal(rec.mask(), dense['node_mask'])
  V = ro.pad_rows(sp['V_rows'], sp['node_ptr'], rec.n, sp['N'])
  assert np.array_equal(V.view(np.int32), dense['V'].view(np.int32))
  assert np.array_equal(ro.pad_rows(sp['node_feat'], sp['node_ptr'], rec.n, sp['N']), dense['node_feat'])
  assert np.array_equal(rec.gat_bias().view(np.int32), data.gat_bias(dense['L']).view(np.int32))
  # the fp64 simple-graph operator is the one prepare_graph hands eigh
  L0 = rec.l4(0)
  for b, s in enumerate(samples):
    n = s['L_simple_4'].shape[0]
    assert np.array_equal(L0[b, :n, :n], s['L_simple_4']) and not L0[b, n:].any() and not L0[b, :, n:].any()


def test_candidates_are_the_nonzero_columns_of_the_collated_rows():
  samples = data.synthetic_qm8_samples(9, seed=4)
  sp = data.sparse_collate(samples, 4)
  rec = ro.Records(sp['sizes'], sp['edge_ptr'], sp['edges'], sp['N'], sp['num_edgetype'])
  L = data.collate(samples, 4)['L']
  B, N, _, E1 = L.shape
  cands = rec.candidates()
  assert len(cands) == B * N * E1
  for b in range(B):
    for n in range(N):
      for e in range(E1):
        assert np.array_equal(cands[(b * N + n) * E1 + e], np.flatnonzero(L[b, n, :, e]))


def _one_graph(recs, n=6, N=8, E=3):
  edges = np.zeros((len(recs), 4), np.uint8)
  if recs:
    edges[:, :3] = recs
  return ro.Records([n], [0, len(recs)], edges, N, E)


def test_duplicates_reversed_pairs_and_ignored_records_change_nothing():
  base = [(0, 1, 0), (1, 2, 0), (1, 2, 2), (3, 3, 1), (4, 5, 1), (0, 5, 2)]
  want = _one_graph(base)
  variants = [
      base + base,                                            # every record twice
      [(v, u, c) for u, v, c in base],                        # every pair reversed
      base[::-1] + [(v, u, c) for u, v, c in base[:3]],       # other order, some listed both ways
      base + [(0, 1, 3), (2, 4, 255), (6, 1, 0), (1, 7, 0), (128, 0, 0), (0, 200, 1), (255, 255, 2)],
  ]
  for recs in variants:
    got = _one_graph(recs)
    assert np.array_equal(got.A, want.A), recs
    assert np.array_equal(got.operators().view(np.int32), want.operators().view(np.int32))
    assert np.array_equal(got.gat_bias().view(np.int32), want.gat_bias().view(np.int32))
  # and the ignored records alone give the graph without bonds
  empty = _one_graph([(0, 1, 3), (2, 4, 255), (6, 1, 0), (128, 0, 0)])
  assert not empty.A.any()
  assert np.array_equal(empty.operators()[0, :6, :6, 0], np.eye(6, dtype=np.float32))


def test_hand_built_multigraph_values():
  """Two bond types on one pair and a self-loop: the simple graph sums the types, each type is a set."""
  rec = _one_graph([(0, 1, 0), (1, 0, 1), (0, 1, 0), (2, 2, 0)], n=3, N=4, E=2)
  m0 = rec.multiplicity(0)[0]
  assert np.array_equal(m0[:3, :3], [[1, 2, 0], [2, 1, 0], [0, 0, 2]]) and not m0[3].any()
  L0 = rec.l4(0)[0]
  s = np.power(np.array([3.0, 3.0, 2.0]), -0.5)
  assert L0[0, 1] == (s[0] * 2.0) * s[1] and L0[2, 2] == (s[2] * 2.0) * s[2]
  assert np.array_equal(rec.degrees()[0], [3, 3, 2, 0])
  bias = rec.gat_bias()[0]
  assert np.signbit(bias[0, 1, 2]) and bias[0, 1, 2] == 0 and bias[0, 2, 2] == np.float32(-1e9)
  assert bias[2, 2, 1] == 0 and bias[2, 2, 2] == 0 and bias[3, 3, 0] == 0 and bias[0, 3, 0] == np.float32(-1e9)


def test_ell_rows_list_the_diagonal_first_then_ascending_columns():
  rec = _one_graph([(0, 3, 0), (0, 1, 1), (2, 0, 0), (4, 4, 2)], n=5, N=6, E=3)
  L = rec.operators()
  val, idx, emax = ro.ell_rows(L)
  assert np.array_equal(idx[0, 0, :4, 0], [0, 1, 2, 3]) and emax[0, 0] == 4   # simple graph, row 0
  assert np.array_equal(idx[0, 1, :3, 0], [0, 2, 3]) and np.array_equal(idx[0, 2, :2, 0], [0, 1])
  assert idx[0, 3, 0, 4] == 4 and emax[0, 3] == 1 and not idx[0, 3, :, 0].any()   # a self-loop: one slot
  assert np.array_equal(val[0, 0, :4, 0], L[0, 0, [0, 1, 2, 3], 0])
  assert np.array_equal(val[0, 1, :3, 2], [L[0, 2, 2, 1], L[0, 2, 0, 1], 0])      # row 2: diagonal, then 0
  assert np.array_equal(idx[0, 1, :3, 2], [2, 0, 0])
  assert not val[0, 0, :, 5].any() and not idx[0, :, :, 5].any()           # a padded row is empty
  vb = ro.ell_rows(L, binarize=True)[0]
  assert np.array_equal(vb[0, 0, :4, 0], np.ones(4, np.float32)) and not vb[0, 0, 4:, 0].any()


@pytest.mark.parametrize('name', ro.CASES)
def test_adversarial_batches_cover_what_they_claim(name):
  bt = ro.adversarial_batch(name)
  B, N, E = len(bt['sizes']), bt['N'], bt['E']
  assert bt['edge_ptr'][0] == 0 and bt['edge_ptr'][-1] == len(bt['edges']) and np.all(np.diff(bt['edge_ptr']) >= 0)
  assert bt['node_ptr'][-1] == len(bt['node_feat']) == len(bt['V_rows']) == len(bt['node_x'])
  assert np.all(bt['sizes'] <= N) and int(bt['sizes'].max()) == N
  rec = ro.read(bt)
  deg = rec.degrees().max()
  if name == 'complete_3types_N128':
    assert deg == 382
  elif name == 'types15_N40':
    assert deg == 1 + 15 * 40
  elif name.startswith('types32_'):
    assert deg == 1 + 32 * N
  if name.startswith('multigraph_'):
    assert B % 4 != 0 or N > 32
    assert list(bt['sizes'][:4]) == [N, 0, 1, N]
    assert bt['edge_ptr'][4] == bt['edge_ptr'][3] < bt['edge_ptr'][5]     # an empty range between others
    e = bt['edges'][bt['edge_ptr'][0]:bt['edge_ptr'][1]].astype(int)
    assert (e[:, 2] >= E).any() and (e[:, :2] >= 128).any() and (e[:, 0] == e[:, 1]).any()
    A0 = rec.A[0].any(axis=0)
    for w in ro.BOUNDARY_NODES:
      if w < N and N > 1:
        assert A0[w].any(), w
    assert (rec.A[0].sum(axis=0) >= 2).any()               # a pair with several types
  if name == 'no_edges':
    assert len(bt['edges']) == 0 and 0 in bt['sizes']


def test_degree_table_covers_the_envelope():
  """The deg^-1/2 table the normalising producers index: long enough for the largest simple-graph degree
  of the envelope (1 + 32 * 128, E <= 32 bond types on N <= 128 nodes, self-loops included) and the same
  length as the C header declares."""
  from lanczosnetwork_b200 import ops
  with open(os.path.join(ROOT, 'include', 'lanczosnet_b200.h')) as fh:
    m = re.search(r'#define LNB_INV_SQRT_DEG_LEN (\d+)', fh.read())
  assert m and int(m.group(1)) == ops.INV_SQRT_DEG_LEN
  assert ops.INV_SQRT_DEG_LEN >= 1 + 32 * 128 + 1
  # the table is np.power over arange; the reference applies np.power to each graph's degree vector: the
  # same values at the degrees the adversarial batches reach
  deg = np.arange(ops.INV_SQRT_DEG_LEN, dtype=np.float64)
  with np.errstate(divide='ignore'):
    table = np.power(deg, -0.5)
  table[0] = 0.0
  d = ro.read(ro.adversarial_batch('types32_N128')).degrees()
  assert d.max() == ops.INV_SQRT_DEG_LEN - 1
  with np.errstate(divide='ignore'):
    s = np.power(d.astype(np.float64), -0.5)
  s[np.isinf(s)] = 0.0
  assert np.array_equal(s, table[d])
