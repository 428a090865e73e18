"""GPNN's device partition, host side: the fp64 oracle (tests/partition_oracle.py) against the reference's
partitions (tests/golden/gpnn_partitions.npz), the k-means++ draw table, the oracle's seeding against
scikit-learn's, ops.spectral_partition's argument checks, and the drop-in's ``--device-partition`` against
the reference's collate."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import partition_oracle
from helpers import ROOT
from lanczosnetwork_b200 import data, ops

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference'
GOLDEN = os.path.join(HERE, 'golden', 'gpnn_partitions.npz')
EQUAL_INERTIA = 1e-9


def golden_operators():
  """The fixture's padded fp64 operators, one [N, N] per graph in fixture order."""
  g = np.load(GOLDEN)
  out = []
  for count, seed, batch, max_nodes in g['sets']:
    samples = data.synthetic_qm8_samples(int(count), seed=int(seed), max_nodes=int(max_nodes))
    for s in range(0, int(count), int(batch)):
      grp = samples[s:s + int(batch)]
      N = max(r['L_simple_4'].shape[0] for r in grp)
      for r in grp:
        L = np.zeros((N, N))
        n = r['L_simple_4'].shape[0]
        L[:n, :n] = r['L_simple_4']
        out.append(L)
  return out


def test_oracle_matches_the_reference_partitions():
  """Identical canonical partitions on every graph without a tie at the cut, except graphs whose two
  partitions have the same inertia (a symmetric alternative); those are a handful."""
  g = np.load(GOLDEN)
  P = int(g['num_partition'])
  ops_ = golden_operators()
  assert len(ops_) == len(g['N']) == 1040
  equal = []
  for k, L in enumerate(ops_):
    N = L.shape[0]
    assert N == g['N'][k]
    if g['tie'][k]:
      continue
    r = partition_oracle.spectral_clustering(L, P)
    if np.array_equal(r['labels'], g['labels'][k, :N]):
      continue
    assert abs(r['inertia'] - g['inertia'][k]) <= EQUAL_INERTIA * abs(g['inertia'][k]), (k, r['inertia'], g['inertia'][k])
    equal.append(k)
  assert len(equal) <= 8, equal
  assert int(g['tie'].sum()) <= 8


def test_draw_table_is_randomstate():
  for N, P, seed in ((26, 3, 1234), (64, 16, 1234), (5, 2, 7), (128, 8, 1234)):
    rs = np.random.RandomState(seed)
    T = 2 + int(np.log(P))
    want = [rs.choice(N, p=np.ones(N) / N)] + [u for _ in range(P - 1) for u in rs.uniform(size=T)]
    got = ops.partition_draws(N, P, seed)
    assert got.dtype == np.float64 and np.array_equal(got, np.asarray(want, np.float64)), (N, P)


def test_oracle_seeding_equals_sklearn():
  cluster = pytest.importorskip('sklearn.cluster')
  rng = np.random.RandomState(3)
  for L in golden_operators()[::97] + [rng.rand(40, 40)]:
    L = (L + L.T) / 2 if L.shape[0] == 40 else L
    for P in (2, 3, 7):
      X, _, _ = partition_oracle.centred_embedding(L, P)
      C, idx = partition_oracle.kmeans_plusplus(X, P, np.random.RandomState(1234))
      C_sk, idx_sk = cluster.kmeans_plusplus(X, P, random_state=1234)
      assert np.array_equal(idx, idx_sk) and np.array_equal(C, C_sk), (P, idx, idx_sk)


def test_oracle_kmeans_equals_sklearn():
  cluster = pytest.importorskip('sklearn.cluster')
  for L in golden_operators()[::61]:
    X, _, _ = partition_oracle.centred_embedding(L, 3)
    km = cluster.KMeans(n_clusters=3, random_state=1234, n_init=1).fit(X)
    r = partition_oracle.spectral_clustering(L, 3)
    assert np.array_equal(r['raw'], km.labels_)


def test_ops_argument_checks():
  L = torch.zeros(2, 10, 10, 7)
  with pytest.raises(AssertionError):
    ops.spectral_partition(L, 9)                 # the reference's assert (K < num_nodes - 1)
  with pytest.raises(AssertionError):
    ops.spectral_partition(L[..., 0], 9)
  with pytest.raises(ValueError):
    ops.spectral_partition(torch.zeros(2, 10, 9), 3)
  with pytest.raises(ValueError):
    ops.spectral_partition(torch.zeros(10, 10), 3)
  with pytest.raises(ValueError):
    ops.spectral_partition(torch.zeros(1, 40, 40), 17)
  with pytest.raises(ValueError):
    ops.spectral_partition(torch.zeros(1, 129, 129), 3)
  with pytest.raises(ValueError):
    ops.spectral_partition(L, 1)
  with pytest.raises(RuntimeError, match='no CPU fallback'):
    ops.spectral_partition(L, 3)


SCRIPT = r'''
import sys, types
repo, ref = sys.argv[1], sys.argv[2]
sys.path.insert(0, repo)
import numpy as np
from lanczosnetwork_b200 import data, dropin
dropin.install(ref, runner_modules=(), compat=True, device_partition=True)
import utils.spectral_graph_partition as sgp
class Boom(object):
  def __init__(self, *a, **k):
    raise SystemExit('scikit-learn was called')
sgp.KMeans = Boom
from dataset.qm8 import QM8Data
ns = types.SimpleNamespace
cfg = ns(seed=1, dataset=ns(data_path='/nonexistent', num_bond_type=6), model=ns(name='GPNN', num_partition=3))
rng = np.random.RandomState(4)
recs = []
for n in (9, 14, 5):
  nf, adjs = data.synthetic_molecule(rng, n)
  rec = data.prepare_graph(adjs, nf, label=rng.randn(1, 16))
  recs.append(rec)
out = QM8Data(cfg, 'test').collate_fn(recs)
assert tuple(out['L_cluster'].shape) == (3, 0, 0) and tuple(out['L_cut'].shape) == (3, 0, 0), out['L_cluster'].shape
assert tuple(out['L'].shape) == (3, 14, 14, 7)
print('COLLATE_OK')
'''


@pytest.mark.skipif(not os.path.isdir(REF), reason='reference checkout not present')
def test_device_partition_dropin_skips_the_host_partition(tmp_path):
  script = tmp_path / 'collate.py'
  script.write_text(SCRIPT)
  proc = subprocess.run([sys.executable, str(script), ROOT, REF], capture_output=True, text=True, timeout=300)
  assert proc.returncode == 0 and 'COLLATE_OK' in proc.stdout, proc.stdout[-3000:] + proc.stderr[-3000:]
