"""Packed batches for every drop-in with a records entry, on the host: the blob without eigenpairs, the
PackedMolecules <-> pack_sparse byte contract for it, and the packed branch of forward_sparse -- its inputs
and graph-cache keys, and the refusals of malformed batches that come before any device work."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data
from lanczosnetwork_b200.model import (DCNN, GAT, GCN, GCNFP, GGNN, GPNN, MPNN, ChebyNet, KeyedAdaLanczosNet,
                                       KeyedGAT, LanczosNet, SampledGraphSAGE, SparseLanczosNetGeneral,
                                       TrainableGAT)
from lanczosnetwork_b200.data import packed_capacity
from lanczosnetwork_b200.model._common import Ragged

K = 20
DROPINS = {
    'GCN': lambda: GCN(configs.qm8_gcn()), 'GCNFP': lambda: GCNFP(configs.qm8_gcn()),
    'DCNN': lambda: DCNN(configs.qm8_dcnn()), 'ChebyNet': lambda: ChebyNet(configs.qm8_cheby_net()),
    'GAT': lambda: GAT(configs.qm8_gat()), 'TrainableGAT': lambda: TrainableGAT(configs.qm8_gat()),
    'KeyedGAT': lambda: KeyedGAT(configs.qm8_gat()), 'GGNN': lambda: GGNN(configs.qm8_ggnn()),
    'MPNN': lambda: MPNN(configs.qm8_mpnn()), 'GPNN': lambda: GPNN(configs.qm8_gpnn()),
    'SampledGraphSAGE': lambda: SampledGraphSAGE(configs.qm8_graphsage(agg_func='Mean')),
}
_SAMPLES = {}


def _samples(B=40, seed=3):
  if (B, seed) not in _SAMPLES:
    _SAMPLES[B, seed] = data.synthetic_qm8_samples(B, seed=seed)
  return _SAMPLES[B, seed]


def _packed(samples, eigs=False):
  pk = data.pack_sparse(data.sparse_collate(samples, K, eigs=eigs))
  pk['blob'] = torch.from_numpy(pk['blob'])
  pk['sample_key'] = torch.tensor([7, 0], dtype=torch.int64)
  return pk


def _hdr(blob):
  return np.asarray(blob[:64]).view(np.int32)


def test_blob_without_eigenpairs_layout():
  samples = _samples(12, seed=5)
  sp = data.sparse_collate(samples, K, eigs=False)
  blob = data.pack_sparse(sp)['blob']
  hdr = _hdr(blob)
  B = len(samples)
  off_sizes, off_node_ptr, off_edge_ptr, off_D = data.packed_offsets(B, K)[:4]
  assert hdr[0] == data.PACK_MAGIC and (hdr[1], hdr[2]) == (B, K)
  assert (hdr[3], hdr[4], hdr[5]) == (off_sizes, off_node_ptr, off_edge_ptr)
  assert hdr[6] == 0 and hdr[8] == 0 and hdr[11] == 0 and hdr[12] == 0      # D, V_rows, tiles, krow: absent
  assert hdr[7] == off_D                                                     # node ids start where D would
  assert hdr[10] == blob.size and blob.size % 16 == 0
  assert all(int(o) % 16 == 0 for o in (hdr[7], hdr[9]))
  rows, nedge = int(sp['node_ptr'][-1]), int(sp['edge_ptr'][-1])

  def seg(off, dtype, count):
    return blob[off:off + count * np.dtype(dtype).itemsize].view(dtype)

  assert np.array_equal(seg(hdr[3], np.int32, B), sp['sizes'])
  assert np.array_equal(seg(hdr[4], np.int32, B + 1), sp['node_ptr'])
  assert np.array_equal(seg(hdr[5], np.int32, B + 1), sp['edge_ptr'])
  assert np.array_equal(seg(hdr[7], np.int32, rows), sp['node_feat'])
  assert np.array_equal(seg(hdr[9], np.uint8, 4 * nedge).reshape(nedge, 4), sp['edges'])
  assert hdr[9] + 4 * nedge <= blob.size
  # the bytes outside the segments are zero
  used = np.zeros(blob.size, bool)
  used[:52] = True
  for off, n in ((hdr[3], 4 * B), (hdr[4], 4 * (B + 1)), (hdr[5], 4 * (B + 1)), (hdr[7], 4 * rows), (hdr[9], 4 * nedge)):
    used[off:off + n] = True
  assert not blob[~used].any()
  # at least 4 K bytes per node smaller than the blob with eigenpairs, whose layout is unchanged
  with_eigs = data.pack_sparse(data.sparse_collate(samples, K))
  assert with_eigs['eigs'] and not data.pack_sparse(sp)['eigs']
  assert with_eigs['blob'].size - blob.size >= 4 * rows * K
  assert all(_hdr(with_eigs['blob'])[i] != 0 for i in (6, 8, 11, 12))


def test_blob_without_eigenpairs_from_samples_without_them():
  rng = np.random.RandomState(2)
  samples = []
  for n in (5, 1, 26, 9):
    nf, adjs = data.synthetic_molecule(rng, n)
    samples.append(data.prepare_graph(adjs, nf, label=rng.randn(1, 16), eigs=False))
  pk = data.pack_sparse(data.sparse_collate(samples, K, eigs=False))
  assert pk['K'] == K and pk['N'] == 26 and not pk['eigs']
  assert np.array_equal(data.PackedMolecules(samples, K, eigs=False).batch([0, 1, 2, 3])['blob'], pk['blob'])
  with pytest.raises(KeyError):
    data.PackedMolecules(samples, K)                 # the eigenpair layout needs the host's eigenpairs


@pytest.mark.parametrize('seed', range(6))
def test_packed_molecules_without_eigenpairs_equal_pack_sparse(seed):
  samples = _samples(60, seed=seed % 3)
  pool = data.PackedMolecules(samples, K, eigs=False)
  rng = np.random.RandomState(seed)
  for _ in range(4):
    idx = rng.randint(0, len(samples), size=rng.randint(1, 50))
    if seed % 2:
      idx[:len(idx) // 2] = idx[0]                   # repeats
    ref = data.pack_sparse(data.sparse_collate([samples[i] for i in idx], K, eigs=False))
    got = pool.batch(idx)
    assert np.array_equal(got['blob'], ref['blob'])
    for k in ('B', 'N', 'K', 'num_edgetype', 'eigs'):
      assert got[k] == ref[k], k
    assert np.array_equal(got['label'], ref['label'])
    stale = np.full(pool.max_bytes(len(idx)) + 48, 0xAB, np.uint8)
    again = pool.batch(idx, out=stale)
    assert again['blob'].base is stale and np.array_equal(again['blob'], ref['blob'])


@pytest.mark.parametrize('eigs', [False, True])
def test_max_bytes_bounds_any_batch(eigs):
  samples = _samples(60, seed=1)
  pool = data.PackedMolecules(samples, K, eigs=eigs)
  big_n = int(np.argmax([len(s['node_feat']) for s in samples]))
  big_e = int(np.argmax([len(s['edges']) for s in samples]))
  rng = np.random.RandomState(4)
  for idx in ([big_n] * 33, [big_e] * 33, [big_n, big_e] * 9, list(rng.randint(0, 60, 50))):
    blob = pool.batch(idx)['blob']
    assert pool.max_bytes(len(idx)) >= blob.size
  assert data.PackedMolecules(samples, K, eigs=False).max_bytes(33) < data.PackedMolecules(samples, K).max_bytes(33)


@pytest.mark.parametrize('eigs', [False, True])
@pytest.mark.parametrize('name', sorted(DROPINS))
def test_packed_inputs_of_every_dropin(name, eigs):
  mod = DROPINS[name]().eval()
  pk = _packed(_samples(), eigs)
  B, N = pk['B'], pk['N']
  inputs, impl, key = mod._sparse_inputs(pk)
  assert key == ('packed_records', B, N, K) and callable(impl)
  assert len(inputs) == (2 if name == 'SampledGraphSAGE' else 1)
  assert isinstance(inputs[0], Ragged) and inputs[0].tensor is pk['blob']
  assert inputs[0].capacity == packed_capacity(B, N, K, eigs, pk['blob'].numel()) >= pk['blob'].numel()
  if name == 'SampledGraphSAGE':
    assert inputs[1] is pk['sample_key']
  # the capacity depends on (B, N, K) only: another batch of the same shape has the same static blob
  other = _packed(_samples(B, seed=9), eigs)
  assert other['N'] == N
  assert mod._sparse_inputs(other)[0][0].static_shape() == inputs[0].static_shape()


def test_keyed_gat_keeps_the_dropout_key_beside_a_packed_blob():
  pk = dict(_packed(_samples()), dropout_key=torch.tensor([1, 2], dtype=torch.int64))
  inputs, _, key = KeyedGAT(configs.qm8_gat()).eval()._sparse_inputs(pk)
  assert key == ('packed_records', pk['B'], pk['N'], K) and len(inputs) == 2 and inputs[1] is pk['dropout_key']


def test_lanczos_net_packed_entries():
  mod = LanczosNet(configs.qm8_lanczos_net()).eval()
  assert not hasattr(mod, '_forward_records')
  pk = _packed(_samples())
  B, N = pk['B'], pk['N']
  assert mod._sparse_inputs(pk)[2] == ('packed_eigs', B, N, K)
  with_eigs = _packed(_samples(), eigs=True)
  assert mod._sparse_inputs(with_eigs)[2] == ('packed', B, N, K)
  # without batch['eigs'] the header says which path runs
  assert mod._sparse_inputs({k: v for k, v in with_eigs.items() if k != 'eigs'})[2] == ('packed', B, N, K)
  assert mod._sparse_inputs({k: v for k, v in pk.items() if k != 'eigs'})[2] == ('packed_eigs', B, N, K)


def _bad(pk, **hdr_edits):
  blob = pk['blob'].clone()
  hdr = blob[:64].view(torch.int32)
  for i, v in hdr_edits.items():
    hdr[int(i[1:])] = v
  return dict(pk, blob=blob)


@pytest.mark.parametrize('name', ['GCN', 'GPNN', 'SampledGraphSAGE', 'LanczosNet'])
def test_malformed_packed_batches_are_refused_on_the_host(name):
  mod = (DROPINS[name] if name in DROPINS else lambda: LanczosNet(configs.qm8_lanczos_net()))().eval()
  pk = _packed(_samples())
  B = pk['B']
  size = pk['blob'].numel()
  for bad, match in ((_bad(pk, h0=0x12345678), 'magic'), (_bad(pk, h1=B + 1), 'B='), (_bad(pk, h2=K + 1), 'K='),
                     (dict(pk, B=B - 1), 'B='), (dict(pk, K=12), 'K='), (_bad(pk, h10=size + 16), 'total'),
                     (_bad(pk, h10=0), 'total'), (dict(pk, eigs=True), 'eigs'), (dict(pk, N=129), 'N=129'),
                     (dict(pk, blob=pk['blob'][:40]), 'blob'), (dict(pk, blob=pk['blob'].view(torch.int32)), 'blob')):
    with pytest.raises(ValueError, match=match):
      mod._sparse_inputs(bad)
  for drop in ('B', 'N', 'K'):                         # without 'blob' it is a records batch
    with pytest.raises(ValueError, match=drop):
      mod._sparse_inputs({k: v for k, v in pk.items() if k != drop})


def test_model_checks_come_before_the_packed_branch():
  pk = _packed(_samples())
  with pytest.raises(ValueError, match='num_partition=17'):
    GPNN(configs.qm8_gpnn(num_partition=17)).eval()._sparse_inputs(pk)
  with pytest.raises(TypeError):
    GGNN(configs.qm8_ggnn(update_func='MLP')).eval()._sparse_inputs(pk)
  with pytest.raises(ValueError, match='sample_key'):
    DROPINS['SampledGraphSAGE']().eval()._sparse_inputs({k: v for k, v in pk.items() if k != 'sample_key'})


def test_packed_training_stays_refused():
  for eigs in (False, True):
    pk = _packed(_samples(), eigs)
    for mod in (LanczosNet(configs.qm8_lanczos_net()), GCN(configs.qm8_gcn()),
                SampledGraphSAGE(configs.qm8_graphsage(agg_func='Mean'))):
      with pytest.raises(NotImplementedError, match='packed'):
        mod.train().forward_sparse_train(pk)
    with pytest.raises(NotImplementedError, match='packed'):
      KeyedAdaLanczosNet(configs.qm8_ada_lanczos_net())._sparse_inputs(
          dict(pk, start_key=torch.tensor([1, 0], dtype=torch.int64)))
    with pytest.raises(NotImplementedError, match='packed'):
      SparseLanczosNetGeneral(configs.graph_lanczos_net())._sparse_inputs(pk)
  from lanczosnetwork_b200.train import GraphedStep
  mod = GCN(configs.qm8_gcn())
  with pytest.raises(ValueError, match='records'):
    GraphedStep(mod, torch.optim.SGD(mod.parameters(), lr=0.1), (_packed(_samples()),),
                {'label': torch.zeros(1)}, sparse=True)


def test_host_blob_with_more_node_rows_than_the_padding_target_allows_is_refused():
  pk = _packed(_samples())
  off = int(_hdr(pk['blob'].numpy())[4])
  for mod in (GCN(configs.qm8_gcn()).eval(), LanczosNet(configs.qm8_lanczos_net()).eval()):
    with pytest.raises(ValueError, match='node_ptr'):
      mod._sparse_inputs(dict(pk, N=4))              # node_ptr[B] > B * 4
    with pytest.raises(ValueError, match='node_ptr offset'):
      mod._sparse_inputs(_bad(pk, h4=off + 4))
