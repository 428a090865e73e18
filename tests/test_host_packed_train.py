"""Packed training batches on the host: the label segment of the blob (pack_sparse / PackedMolecules byte
contract, the max_bytes and packed_capacity bounds) and GraphedStep(packed=True)'s refusals, which come before
any device work."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data
from lanczosnetwork_b200.model import (GAT, GCN, GGNN, KeyedAdaLanczosNet, KeyedGAT, LanczosNet, SampledGraphSAGE,
                                       SparseLanczosNetGeneral)
from lanczosnetwork_b200.data import packed_capacity
from lanczosnetwork_b200.train import GraphedStep

K = 20
_SAMPLES = {}


def _samples(B=40, seed=3):
  if (B, seed) not in _SAMPLES:
    _SAMPLES[B, seed] = data.synthetic_qm8_samples(B, seed=seed)
  return _SAMPLES[B, seed]


def _hdr(blob):
  return np.asarray(blob[:64]).view(np.int32)


@pytest.mark.parametrize('eigs', [False, True])
def test_labelled_blob_is_the_unlabelled_one_plus_a_label_tail(eigs):
  sp = data.sparse_collate(_samples(17, seed=5), K, eigs=eigs)
  plain = data.pack_sparse(sp)['blob']
  pk = data.pack_sparse(sp, label=True)
  blob, hdr, h0 = pk['blob'], _hdr(pk['blob']), _hdr(plain)
  B, P = sp['label'].shape
  assert h0[13] == 0 and h0[14] == 0                                 # no labels: today's zero-filled slots
  assert hdr[13] == plain.size and hdr[14] == P and hdr[13] % 16 == 0
  assert hdr[10] == blob.size == plain.size + -(-4 * B * P // 16) * 16
  same = np.ones(16, bool)
  same[[10, 13, 14]] = False
  assert np.array_equal(hdr[same], h0[same])
  assert np.array_equal(blob[64:plain.size], plain[64:])
  assert np.array_equal(blob[hdr[13]:hdr[13] + 4 * B * P].view(np.float32).reshape(B, P), sp['label'])
  assert not blob[hdr[13] + 4 * B * P:].any()
  assert np.array_equal(pk['label'], sp['label'])


def test_unlabelled_writers_are_unchanged_by_the_option():
  samples = _samples(12, seed=2)
  for eigs in (False, True):
    sp = data.sparse_collate(samples, K, eigs=eigs)
    assert np.array_equal(data.pack_sparse(sp)['blob'], data.pack_sparse(sp, label=False)['blob'])
    idx = [0, 3, 3, 7]
    assert np.array_equal(data.PackedMolecules(samples, K, eigs=eigs).batch(idx)['blob'],
                          data.PackedMolecules(samples, K, eigs=eigs, labels=False).batch(idx)['blob'])


def test_labels_are_required_to_write_them():
  rng = np.random.RandomState(2)
  nf, adjs = data.synthetic_molecule(rng, 6)
  samples = [data.prepare_graph(adjs, nf)]
  with pytest.raises(ValueError, match='label'):
    data.pack_sparse(data.sparse_collate(samples, K), label=True)
  with pytest.raises(ValueError, match='label'):
    data.PackedMolecules(samples, K, labels=True)


@pytest.mark.parametrize('eigs', [False, True])
@pytest.mark.parametrize('seed', range(4))
def test_packed_molecules_with_labels_equal_pack_sparse(seed, eigs):
  samples = _samples(60, seed=seed % 2)
  pool = data.PackedMolecules(samples, K, eigs=eigs, labels=True)
  rng = np.random.RandomState(seed)
  for _ in range(4):
    idx = rng.randint(0, len(samples), size=rng.randint(1, 50))
    if seed % 2:
      idx[:len(idx) // 2] = idx[0]                   # repeats
    ref = data.pack_sparse(data.sparse_collate([samples[i] for i in idx], K, eigs=eigs), label=True)
    got = pool.batch(idx)
    assert np.array_equal(got['blob'], ref['blob'])
    stale = np.full(pool.max_bytes(len(idx)) + 48, 0xAB, np.uint8)
    again = pool.batch(idx, out=stale)
    assert again['blob'].base is stale and np.array_equal(again['blob'], ref['blob'])


@pytest.mark.parametrize('eigs', [False, True])
def test_max_bytes_and_packed_capacity_bound_every_labelled_batch(eigs):
  samples = _samples(60, seed=1)
  pool = data.PackedMolecules(samples, K, eigs=eigs, labels=True)
  P = pool.label.shape[1]
  big_n = int(np.argmax([len(s['node_feat']) for s in samples]))
  big_e = int(np.argmax([len(s['edges']) for s in samples]))
  rng = np.random.RandomState(4)
  for idx in ([big_n] * 33, [big_e] * 33, [big_n, big_e] * 9, list(rng.randint(0, 60, 50)), [big_n]):
    b = pool.batch(idx)
    size = b['blob'].size
    assert pool.max_bytes(len(idx)) >= size
    assert packed_capacity(b['B'], b['N'], K, eigs, 0, label_dim=P) >= size
  # the label segment is counted, and without it nothing changes
  assert pool.max_bytes(33) >= data.PackedMolecules(samples, K, eigs=eigs).max_bytes(33) + 4 * 33 * P
  assert packed_capacity(33, 26, K, eigs, 0, label_dim=0) == packed_capacity(33, 26, K, eigs, 0)
  assert packed_capacity(33, 26, K, eigs, 0, label_dim=P) >= packed_capacity(33, 26, K, eigs, 0) + 4 * 33 * P


# ---- GraphedStep(packed=True) refusals on CPU modules --------------------------------------------------
def _packed(samples, label=True, eigs=False):
  pk = data.pack_sparse(data.sparse_collate(samples, K, eigs=eigs), label=label)
  pk['blob'] = torch.from_numpy(pk['blob'])
  pk['sample_key'] = torch.tensor([7, 0], dtype=torch.int64)
  return pk


def _step(mod, batch, **kw):
  return GraphedStep(mod, torch.optim.SGD(mod.parameters(), lr=0.1), (batch,), packed=True, **kw)


def test_models_outside_the_list_are_refused_by_name():
  pk = _packed(_samples())
  for mod in (GAT(configs.qm8_gat()), KeyedAdaLanczosNet(configs.qm8_ada_lanczos_net()),
              SparseLanczosNetGeneral(configs.graph_lanczos_net())):
    with pytest.raises(TypeError, match=type(mod).__name__):
      _step(mod, dict(pk, start_key=torch.tensor([1, 0], dtype=torch.int64)))


def test_unlabelled_blobs_and_label_arguments_are_refused():
  mod = GCN(configs.qm8_gcn())
  with pytest.raises(ValueError, match='labels'):
    _step(mod, _packed(_samples(), label=False))
  pk = _packed(_samples())
  with pytest.raises(ValueError, match='label='):
    _step(mod, pk, kwargs={'label': torch.from_numpy(pk['label'])})
  with pytest.raises(ValueError, match='packed batch'):
    _step(mod, {k: v for k, v in pk.items() if k != 'blob'})
  with pytest.raises(ValueError, match='exclude'):
    _step(mod, pk, sparse=True)


def _bad(pk, **edits):
  blob = pk['blob'].clone()
  hdr = blob[:64].view(torch.int32)
  for i, v in edits.items():
    hdr[int(i[1:])] = v
  return dict(pk, blob=blob)


@pytest.mark.parametrize('make', [lambda: GCN(configs.qm8_gcn()), lambda: LanczosNet(configs.qm8_lanczos_net()),
                                  lambda: SampledGraphSAGE(configs.qm8_graphsage(agg_func='Mean'))])
def test_malformed_labelled_headers_are_refused_on_the_host(make):
  mod = make()
  pk = _packed(_samples())
  h = _hdr(pk['blob'].numpy())
  B, size = pk['B'], pk['blob'].numel()
  for bad, match in ((_bad(pk, h0=0x12345678), 'magic'), (_bad(pk, h1=B + 1), 'B='), (_bad(pk, h10=size + 16), 'total'),
                     (_bad(pk, h13=0), 'labels'), (_bad(pk, h14=0), 'labels'), (_bad(pk, h13=int(h[13]) + 4), 'labels'),
                     (_bad(pk, h14=int(h[14]) + 1), 'labels'), (dict(pk, N=4), 'node_ptr'),
                     (dict(pk, eigs=True), 'eigs')):
    with pytest.raises(ValueError, match=match):
      _step(mod, bad)


def test_refused_calls_raise_before_any_copy():
  """A step's call checks the batch against the capture on the host first: another shape, another P, another
  key set, a label argument or a blob over the captured capacity raise and leave the static blob alone."""
  mod = SampledGraphSAGE(configs.qm8_graphsage(agg_func='Mean'))
  pk = _packed(_samples())
  B, N, P = pk['B'], pk['N'], pk['label'].shape[1]
  step = object.__new__(GraphedStep)                 # the captured state of a CPU step: nothing runs on a device
  step.model, step.packed, step.sparse = mod, True, False
  step._packed_shape = (B, N, K, False, P)
  static = torch.full((packed_capacity(B, N, K, False, pk['blob'].numel(), label_dim=P),), 0xAB, dtype=torch.uint8)
  step._args = [{'blob': static, 'B': B, 'N': N, 'K': K, 'eigs': False, 'sample_key': torch.zeros(2, dtype=torch.int64)}]
  over = torch.zeros(static.numel() + 64, dtype=torch.uint8)
  over[:pk['blob'].numel()] = pk['blob']
  over[:64].view(torch.int32)[10] = over.numel()
  other = data.pack_sparse(data.sparse_collate([_samples()[0]] * B, K, eigs=False), label=True)
  for bad, match in ((dict(pk, blob=over), 'capacity'),
                     ({k: v for k, v in pk.items() if k != 'sample_key'}, 'sample_key'),
                     (dict(pk, sample_key=torch.zeros(3, dtype=torch.int64)), 'sample_key'),
                     (dict(other, blob=torch.from_numpy(other['blob']), sample_key=pk['sample_key']), 'captured'),
                     (_bad(pk, h0=0), 'magic')):
    with pytest.raises(ValueError, match=match):
      step(bad)
  with pytest.raises(ValueError, match='label='):
    step(pk, label=torch.from_numpy(pk['label']))
  assert bool((static == 0xAB).all())
