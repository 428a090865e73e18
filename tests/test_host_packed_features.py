"""Packed batches of float feature rows on the host: header slot F, the PackedMolecules <-> pack_sparse byte
contract for GraphData samples, the segment offsets and zero gaps, the bond bound of their capacity, the
refusals that come before any device work, and the atom-id layout and bytes as they were."""
import hashlib
import os
import re

import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data
from lanczosnetwork_b200.model import GCN, LanczosNet, SparseLanczosNetGeneral
from lanczosnetwork_b200.model._common import Ragged
from lanczosnetwork_b200.train import GraphedStep

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = 20
F = 10
_SAMPLES = {}


def _samples(B=24, seed=5, max_nodes=60, eigs=True):
  if (B, seed, max_nodes, eigs) not in _SAMPLES:
    if eigs:
      s = data.synthetic_regression_graphs(B, seed=seed, max_num_nodes=max_nodes)
    else:
      rng = np.random.RandomState(seed)
      s = []
      for n in rng.randint(5, max_nodes + 1, size=B):
        A = np.triu((rng.rand(n, n) < 0.5).astype(np.float64), 1)
        s.append(data.prepare_graph((A + A.T)[:, :, None], rng.randn(n, F), label=rng.randn(1, 2), eigs=False))
    _SAMPLES[B, seed, max_nodes, eigs] = s
  return _SAMPLES[B, seed, max_nodes, eigs]


def _hdr(blob):
  return np.asarray(blob[:64]).view(np.int32)


def test_slot_15_is_the_feature_width():
  with open(os.path.join(ROOT, 'include', 'lanczosnet_b200.h')) as fh:
    src = fh.read()
  assert re.search(r'^#define LNB_PACK_HDR_F 15\b', src, re.M)
  assert data.PackHeader._fields.index('F') == 15 and len(data.PackHeader._fields) == 16
  assert int(re.search(r'^#define LNB_UNPACK_BAD_FEATURES (\d+)', src, re.M).group(1)) == 128


@pytest.mark.parametrize('label', [False, True])
@pytest.mark.parametrize('eigs', [False, True])
def test_feature_blob_segments(eigs, label):
  samples = _samples(eigs=eigs)
  sp = data.sparse_collate(samples, K, eigs=eigs)
  pk = data.pack_sparse(sp, label=label)
  blob, h = pk['blob'], data.read_packed_header(pk['blob'])
  B, rows, nedge = len(samples), int(sp['node_ptr'][-1]), int(sp['edge_ptr'][-1])
  P = sp['label'].shape[1] if label else 0
  assert pk['F'] == F == h.F and pk['eigs'] == eigs and (h.B, h.K, h.P) == (B, K, P)
  assert h == data.packed_layout(B, K, rows, nedge, eigs, P, F) and h.total == blob.size
  # every fixed segment sits where it sits in an atom-id blob; the node segment is 4 F bytes per node
  o = data.packed_offsets(B, K)
  assert (h.sizes, h.node_ptr, h.edge_ptr) == (o.sizes, o.node_ptr, o.edge_ptr)
  assert h.node_feat == (o.var if eigs else o.D)
  nxt = h.V_rows if eigs else h.edges
  assert nxt == h.node_feat + -(-4 * F * rows // 16) * 16
  segs = [(h.sizes, sp['sizes']), (h.node_ptr, sp['node_ptr']), (h.edge_ptr, sp['edge_ptr']),
          (h.node_feat, sp['node_feat']), (h.edges, sp['edges'])]
  if eigs:
    segs += [(h.D, sp['D']), (h.V_rows, sp['V_rows'])]
    k_eff = data.ritz_extents(sp['V_rows'], sp['node_ptr'])
    krow = np.concatenate([[0], np.cumsum(np.minimum(k_eff, K))]).astype(np.int32)
    segs += [(h.tiles, data.host_tile_segment(sp['sizes'], k_eff)), (h.krow, krow)]
  else:
    assert h.D == h.V_rows == h.tiles == h.krow == 0
  if label:
    segs.append((h.label, sp['label']))
  used = np.zeros(blob.size, bool)
  used[:64] = True
  for off, arr in segs:
    raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    assert off % 16 == 0 and np.array_equal(blob[off:off + raw.size], raw)
    used[off:off + raw.size] = True
  assert not blob[~used].any()                       # alignment gaps are zero


@pytest.mark.parametrize('seed', range(4))
@pytest.mark.parametrize('label', [False, True])
@pytest.mark.parametrize('eigs', [False, True])
def test_packed_molecules_equal_pack_sparse_for_feature_samples(eigs, label, seed):
  samples = _samples(eigs=eigs)
  pool = data.PackedMolecules(samples, K, eigs=eigs, labels=label)
  rng = np.random.RandomState(seed)
  stale = np.full(pool.max_bytes(40) + 48, 0xAB, np.uint8)
  for _ in range(3):
    idx = rng.randint(0, len(samples), size=rng.randint(1, 40))
    if seed % 2:
      idx[:len(idx) // 2] = idx[0]                   # repeats
    ref = data.pack_sparse(data.sparse_collate([samples[i] for i in idx], K, eigs=eigs), label=label)
    got = pool.batch(idx)
    assert np.array_equal(got['blob'], ref['blob'])
    for k in ('B', 'N', 'K', 'num_edgetype', 'eigs', 'F'):
      assert got[k] == ref[k], k
    assert got['F'] == F and np.array_equal(got['label'], ref['label'])
    assert pool.max_bytes(len(idx)) >= got['blob'].size
    again = pool.batch(idx, out=stale)                # a reused buffer holding an older, larger batch
    assert again['blob'].base is stale and np.array_equal(again['blob'], ref['blob'])


def test_capacity_of_feature_blobs_admits_the_densest_batch():
  B, N = 6, 40
  rng = np.random.RandomState(1)
  full = np.ones((N, N)) - np.eye(N)
  dense = [data.prepare_graph(full[:, :, None], rng.randn(N, F), label=rng.randn(1, 2)) for _ in range(B)]
  pk = data.pack_sparse(data.sparse_collate(dense, K), label=True)
  P = pk['label'].shape[1]
  cap = data.packed_capacity(B, N, K, True, 0, label_dim=P, feature_dim=F, num_edgetype=1)
  assert cap >= pk['blob'].size
  # self-loops kept by the upper-triangle bond list count too, and two bond types double the bound
  loops = np.ones((N, N))
  two = np.stack([loops, loops], axis=2)
  pk2 = data.pack_sparse(data.sparse_collate([data.prepare_graph(two, rng.randn(N, F)) for _ in range(B)], K))
  assert data.packed_capacity(B, N, K, True, 0, feature_dim=F, num_edgetype=2) >= pk2['blob'].size
  # the rule for atom ids is unchanged: 4 N bonds per graph
  assert data.packed_capacity(64, 26, 20, True, 0, 16) == 177536
  assert data.packed_capacity(1024, 26, 20, False, 0) == 544864


# ---- the atom-id layout and bytes as the previous layout wrote them --------------------------------------
def test_atom_id_layout_and_bytes_are_unchanged():
  assert tuple(data.packed_layout(9, 20, 140, 150, True, 16)) == (
      data.PACK_MAGIC, 9, 20, 64, 112, 160, 208, 1104, 1664, 12864, 14048, 928, 1056, 13472, 16, 0)
  assert tuple(data.packed_layout(9, 20, 140, 150, False)) == (
      data.PACK_MAGIC, 9, 20, 64, 112, 160, 0, 208, 0, 768, 1376, 0, 0, 0, 0, 0)
  samples = data.synthetic_qm8_samples(12, seed=4)
  # blobs without eigenpairs hold integer records and seeded labels only: their bytes are fixed
  digests = {False: '5d225d84f23e17a461380fbd983d6ad0', True: '75689b8db8efba320956c97e5b35c9c1'}
  sp = data.sparse_collate(samples, 20, eigs=False)
  for label, digest in digests.items():
    pk = data.pack_sparse(sp, label=label)
    assert pk['F'] == 0 and hashlib.sha256(pk['blob'].tobytes()).hexdigest()[:32] == digest
  got = data.PackedMolecules(samples, 20, eigs=False, labels=True).batch([3, 3, 0, 11, 7])
  assert got['F'] == 0 and hashlib.sha256(got['blob'].tobytes()).hexdigest()[:32] == 'bc5a0abcb77591459b2f9a5d69d3423b'
  # with eigenpairs: the header, and the Ritz bytes of the records, where they always were
  sp = data.sparse_collate(samples, 20)
  pk = data.pack_sparse(sp, label=True)
  assert tuple(data.read_packed_header(pk['blob'])) == (
      data.PACK_MAGIC, 12, 20, 64, 112, 176, 240, 1424, 2192, 17392, 19024, 1200, 1360, 18256, 16, 0)
  assert np.array_equal(pk['blob'][2192:2192 + sp['V_rows'].nbytes].view(np.float32).reshape(-1, 20), sp['V_rows'])


# ---- refusals before any device work (the modules sit on the CPU: device work would raise RuntimeError) ---
def _feature_packed(eigs=True, label=False):
  pk = data.pack_sparse(data.sparse_collate(_samples(8, eigs=eigs), K, eigs=eigs), label=label)
  pk['blob'] = torch.from_numpy(pk['blob'])
  return pk


def _atom_packed(eigs=True, label=False):
  pk = data.pack_sparse(data.sparse_collate(data.synthetic_qm8_samples(8, seed=3), K, eigs=eigs), label=label)
  pk['blob'] = torch.from_numpy(pk['blob'])
  return pk


def _set_slot(pk, slot, value):
  blob = pk['blob'].clone()
  blob[:64].view(torch.int32)[slot] = value
  return dict(pk, blob=blob)


@pytest.mark.parametrize('eigs', [False, True])
def test_feature_model_takes_feature_blobs(eigs):
  mod = SparseLanczosNetGeneral(configs.graph_lanczos_net()).eval()
  pk = _feature_packed(eigs)
  B, N = pk['B'], pk['N']
  inputs, impl, key = mod._sparse_inputs(pk)
  assert key == (('packed', B, N, K) if eigs else ('packed_eigs', B, N, K)) and callable(impl)
  assert len(inputs) == 1 and isinstance(inputs[0], Ragged) and inputs[0].tensor is pk['blob']
  assert inputs[0].capacity == data.packed_capacity(B, N, K, eigs, 0, feature_dim=F) >= pk['blob'].numel()
  # without batch['F'] the header says it
  assert mod._sparse_inputs({k: v for k, v in pk.items() if k != 'F'})[2] == key


def test_atom_id_blob_to_the_feature_model_is_not_implemented():
  mod = SparseLanczosNetGeneral(configs.graph_lanczos_net()).eval()
  for eigs in (False, True):
    pk = _atom_packed(eigs)
    for batch in (pk, {k: v for k, v in pk.items() if k != 'F'}):
      with pytest.raises(NotImplementedError, match='packed'):
        mod._sparse_inputs(batch)


@pytest.mark.parametrize('eigs', [False, True])
def test_feature_blob_to_atom_id_models_is_refused(eigs):
  pk = _feature_packed(eigs)
  for mod in (GCN(configs.qm8_gcn()).eval(), LanczosNet(configs.qm8_lanczos_net()).eval()):
    for batch in (pk, {k: v for k, v in pk.items() if k != 'F'}, dict(pk, N=26)):
      with pytest.raises(ValueError, match='feature rows'):
        mod._sparse_inputs(batch)


def test_other_feature_width_is_refused():
  pk = _feature_packed()
  cfg = configs.graph_lanczos_net(input_dim=12)
  cfg.dataset.node_emb_dim = 12
  mod = SparseLanczosNetGeneral(cfg).eval()
  for batch in (pk, {k: v for k, v in pk.items() if k != 'F'}):
    with pytest.raises(ValueError, match='F = 10'):
      mod._sparse_inputs(batch)
  ten = SparseLanczosNetGeneral(configs.graph_lanczos_net()).eval()
  with pytest.raises(ValueError, match="header says F=12"):
    ten._sparse_inputs(_set_slot(pk, 15, 12))         # batch['F'] = 10, header 12
  with pytest.raises(ValueError, match='F = 12'):
    ten._sparse_inputs({k: v for k, v in _set_slot(pk, 15, 12).items() if k != 'F'})


def test_graphed_packed_step_refusals():
  mod = SparseLanczosNetGeneral(configs.graph_lanczos_net())
  opt = torch.optim.SGD(mod.parameters(), lr=0.1)
  with pytest.raises(TypeError, match='SparseLanczosNetGeneral'):
    GraphedStep(mod, opt, (_atom_packed(label=True),), packed=True)
  with pytest.raises(ValueError, match='labels'):
    GraphedStep(mod, opt, (_feature_packed(label=False),), packed=True)
  gcn = GCN(configs.qm8_gcn())
  with pytest.raises(ValueError, match='feature rows'):
    GraphedStep(gcn, torch.optim.SGD(gcn.parameters(), lr=0.1), (_feature_packed(label=True),), packed=True)
  # a labelled feature blob passes every host check and reaches the device, which a CPU module does not have
  with pytest.raises(RuntimeError, match='CUDA'):
    GraphedStep(mod, opt, (_feature_packed(label=True),), packed=True)
