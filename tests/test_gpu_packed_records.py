"""Packed batches on the device: lnb_records_unpack against a numpy split of the blob (its status on
malformed headers included), and forward_sparse of every drop-in with a records entry on packed batches,
bit-equal to forward_sparse on the records they pack -- pinned-host and device-resident blobs, with and
without eigenpairs, several batches from one captured graph."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data, ops
from lanczosnetwork_b200.model import (DCNN, GAT, GCN, GCNFP, GGNN, GPNN, MPNN, ChebyNet, KeyedGAT, LanczosNet,
                                       SampledGraphSAGE, TrainableGAT)

from helpers import deterministic_state_dict

pytestmark = pytest.mark.gpu

K = 20
MODELS = {
    'GCN': lambda: GCN(configs.qm8_gcn()),
    'GCNFP': lambda: GCNFP(configs.qm8_gcn()),
    'DCNN': lambda: DCNN(configs.qm8_dcnn()),
    'ChebyNet': lambda: ChebyNet(configs.qm8_cheby_net()),
    'GAT': lambda: GAT(configs.qm8_gat()),
    'TrainableGAT': lambda: TrainableGAT(configs.qm8_gat()),
    'KeyedGAT': lambda: KeyedGAT(configs.qm8_gat()),
    'GGNN': lambda: GGNN(configs.qm8_ggnn()),
    'MPNN': lambda: MPNN(configs.qm8_mpnn()),
    'GPNN': lambda: GPNN(configs.qm8_gpnn()),
    'SampledGraphSAGE-Mean': lambda: SampledGraphSAGE(configs.qm8_graphsage(agg_func='Mean')),
    'SampledGraphSAGE-Max': lambda: SampledGraphSAGE(configs.qm8_graphsage(agg_func='Max')),
    'SampledGraphSAGE-LSTM': lambda: SampledGraphSAGE(configs.qm8_graphsage(agg_func='LSTM')),
    'LanczosNet': lambda: LanczosNet(configs.qm8_lanczos_net()),
}
SENTINEL = 0x5A


def dev():
  return torch.device('cuda:0')


def _build(name, seed=7):
  mod = MODELS[name]()
  mod.load_state_dict(deterministic_state_dict(mod, seed))
  return mod.to(dev()).eval()


def _tensors(d, where, key=(1234, 0)):
  out = {}
  for k, v in d.items():
    if isinstance(v, np.ndarray):
      t = torch.from_numpy(v)
      out[k] = t.pin_memory() if where == 'pinned' else t.to(dev())
    else:
      out[k] = v
  out['sample_key'] = torch.tensor(key, dtype=torch.int64, device=None if where == 'pinned' else dev())
  return out


def _records(samples, where, eigs=False, key=(1234, 0)):
  return _tensors(data.sparse_collate(samples, K, eigs=eigs), where, key)


def _packed(samples, where, eigs=False, key=(1234, 0)):
  return _tensors(data.pack_sparse(data.sparse_collate(samples, K, eigs=eigs)), where, key)


def _odd_samples():
  """An isolated node, a one-node graph and QM8-shaped molecules (N = 26)."""
  rng = np.random.RandomState(5)
  a = np.zeros((5, 5, 6))
  for u, v, c in ((0, 1, 0), (1, 2, 1), (2, 3, 0)):
    a[u, v, c] = a[v, u, c] = 1.0
  return ([data.prepare_graph(a, rng.randint(0, 70, 5), label=rng.randn(1, 16)),
           data.prepare_graph(np.zeros((1, 1, 6)), rng.randint(0, 70, 1), label=rng.randn(1, 16))] +
          data.synthetic_qm8_samples(14, seed=11))


# ------------------------------------------------------------------------------------------------------
# lnb_records_unpack
def _unpack_raw(blob, B, Kb, cap_rows, cap_edges, eigs, slack=64):
  """lnb_records_unpack into buffers ``slack`` elements longer than the capacities, filled with a sentinel,
  so writes past a capacity show.  Returns the buffers (full length) and the status."""
  fill = lambda shape, dtype: torch.full(shape, SENTINEL, device=dev(), dtype=torch.uint8).view(dtype)
  out = {
      'sizes': fill((4 * (B + slack),), torch.int32), 'node_ptr': fill((4 * (B + 1 + slack),), torch.int32),
      'edge_ptr': fill((4 * (B + 1 + slack),), torch.int32), 'node_feat': fill((4 * (cap_rows + slack),), torch.int32),
      'edges': fill((4 * (cap_edges + slack),), torch.uint8).view(-1, 4),
      'D': fill((4 * (B * Kb + slack),), torch.float32) if eigs else None,
      'V_rows': fill((4 * ((cap_rows + slack) * Kb),), torch.float32) if eigs else None,
  }
  status = torch.full((1,), -1, device=dev(), dtype=torch.int32)
  ops._launch('lnb_records_unpack', blob, blob, blob.numel(), B, Kb, cap_rows, cap_edges, out['sizes'],
              out['node_ptr'], out['node_feat'], out['edge_ptr'], out['edges'], out['D'], out['V_rows'], status)
  torch.cuda.synchronize()
  return {k: (v.cpu().numpy() if v is not None else None) for k, v in out.items()}, int(status.item())


def _sent(dtype):
  return np.full(1, SENTINEL, np.uint8).repeat(np.dtype(dtype).itemsize).view(dtype)[0]


@pytest.mark.parametrize('eigs', [False, True])
@pytest.mark.parametrize('B, seed', [(1, 2), (7, 3), (1024, 4)])
def test_records_unpack_is_the_numpy_split(B, seed, eigs):
  samples = data.synthetic_qm8_samples(B, seed=seed)
  sp = data.sparse_collate(samples, K, eigs=eigs)
  pk = data.pack_sparse(sp)
  rows, nedge = int(sp['node_ptr'][-1]), int(sp['edge_ptr'][-1])
  # the blob inside a larger buffer of stale bytes: nothing past hdr[10] matters
  buf = torch.full((pk['blob'].size + 4096,), 0xEE, dtype=torch.uint8)
  buf[:pk['blob'].size] = torch.from_numpy(pk['blob'])
  blob = buf.to(dev())
  cap_rows, cap_edges = rows + 37, nedge + 5
  out, status = _unpack_raw(blob, B, K, cap_rows, cap_edges, eigs)
  assert status == 0
  assert np.array_equal(out['sizes'][:B], sp['sizes']) and np.all(out['sizes'][B:] == _sent(np.int32))
  assert np.array_equal(out['node_ptr'][:B + 1], sp['node_ptr'])
  assert np.array_equal(out['edge_ptr'][:B + 1], sp['edge_ptr'])
  assert np.all(out['node_ptr'][B + 1:] == _sent(np.int32)) and np.all(out['edge_ptr'][B + 1:] == _sent(np.int32))
  assert np.array_equal(out['node_feat'][:rows], sp['node_feat']) and np.all(out['node_feat'][rows:] == _sent(np.int32))
  assert np.array_equal(out['edges'][:nedge], sp['edges']) and np.all(out['edges'][nedge:] == SENTINEL)
  if eigs:
    assert np.array_equal(out['D'][:B * K].view(np.int32), sp['D'].reshape(-1).view(np.int32))
    assert np.all(out['D'][B * K:].view(np.uint8) == SENTINEL)
    assert np.array_equal(out['V_rows'][:rows * K].view(np.int32), sp['V_rows'].reshape(-1).view(np.int32))
    assert np.all(out['V_rows'][rows * K:].view(np.uint8) == SENTINEL)
  # the op: the same records, at the capacities asked for
  got = ops.records_unpack(blob, B, K, cap_rows, cap_edges, eigs=eigs)
  assert int(got[7].item()) == 0
  for t, ref in zip(got[:5], (sp['sizes'], sp['node_ptr'], sp['node_feat'], sp['edge_ptr'], sp['edges'])):
    assert np.array_equal(t.cpu().numpy()[:len(ref)], ref)
  assert tuple(got[2].shape) == (cap_rows,) and tuple(got[4].shape) == (cap_edges, 4)


def _hdr_edit(pk, **edits):
  blob = pk['blob'].copy()
  hdr = blob[:64].view(np.int32)
  for i, v in edits.items():
    hdr[int(i[1:])] = v
  return torch.from_numpy(blob).to(dev())


def test_records_unpack_refuses_malformed_headers_and_overflows():
  samples = data.synthetic_qm8_samples(9, seed=1)
  sp = data.sparse_collate(samples, K, eigs=False)
  pk = data.pack_sparse(sp)
  B, size = 9, pk['blob'].size
  rows, nedge = int(sp['node_ptr'][-1]), int(sp['edge_ptr'][-1])
  good = torch.from_numpy(pk['blob']).to(dev())
  cases = [
      (_hdr_edit(pk, h0=0x12345678), B, K, rows, nedge, False, 1),
      (_hdr_edit(pk, h1=B + 1), B, K, rows, nedge, False, 2),
      (good, B, K + 1, rows, nedge, False, 2),
      (_hdr_edit(pk, h10=size + 16), B, K, rows, nedge, False, 4),
      (_hdr_edit(pk, h9=size), B, K, rows, nedge, False, 4),            # bonds past the total
      (_hdr_edit(pk, h7=pk['blob'][:64].view(np.int32)[7] + 4), B, K, rows, nedge, False, 4),   # unaligned
      (_hdr_edit(pk, h6=64), B, K, rows, nedge, False, 4),              # D without V_rows
      (good, B, K, rows - 1, nedge, False, 8),
      (good, B, K, rows, nedge - 1, False, 16),
      (good, B, K, rows, nedge, True, 32),
  ]
  for blob, b, k, cap_rows, cap_edges, eigs, want in cases:
    out, status = _unpack_raw(blob, b, k, cap_rows, cap_edges, eigs)
    assert status == want, (want, status)
    assert np.all(out['sizes'][:b] == 0) and np.all(out['sizes'][b:] == _sent(np.int32))
    assert np.all(out['node_ptr'][:b + 1] == 0) and np.all(out['edge_ptr'][:b + 1] == 0)
    assert np.all(out['node_ptr'][b + 1:] == _sent(np.int32)) and np.all(out['edge_ptr'][b + 1:] == _sent(np.int32))
    assert np.all(out['node_feat'] == _sent(np.int32)) and np.all(out['edges'] == SENTINEL)
    if eigs:
      assert np.all(out['D'].view(np.uint8) == SENTINEL) and np.all(out['V_rows'].view(np.uint8) == SENTINEL)
  # the same blob at the exact capacities is fine
  assert _unpack_raw(good, B, K, rows, nedge, False)[1] == 0


def test_records_unpack_host_refusals_launch_nothing():
  blob = torch.from_numpy(data.pack_sparse(data.sparse_collate(data.synthetic_qm8_samples(4, seed=1), K,
                                                               eigs=False))['blob']).to(dev())
  n0 = ops.launch_count()
  with pytest.raises(ValueError):
    ops.records_unpack(blob[1:], 4, K, 104, 100)                  # not 16-byte aligned
  with pytest.raises(ValueError):
    ops.records_unpack(blob[:32], 4, K, 104, 100)
  with pytest.raises(ValueError):
    ops.records_unpack(blob, 0, K, 104, 100)
  with pytest.raises(RuntimeError, match='CUDA'):
    ops.records_unpack(blob.cpu(), 4, K, 104, 100)
  assert ops.launch_count() == n0
  ops.records_unpack(blob, 4, K, 104, 100)
  assert ops.launch_count() == n0 + 1


# ------------------------------------------------------------------------------------------------------
# forward_sparse on packed batches
@pytest.mark.parametrize('B', [64, 1024])
@pytest.mark.parametrize('name', sorted(MODELS))
def test_packed_equals_records(name, B):
  samples = data.synthetic_qm8_samples(B, seed=B + 3)
  mod = _build(name)
  with torch.no_grad():
    ref = mod.forward_sparse(_records(samples, 'device'))
    res = _packed(samples, 'device')
    for _ in range(3):                 # copy-slot capture, then the resident capture and its replay
      assert torch.equal(mod.forward_sparse(res), ref), name
    host = _packed(samples, 'pinned')
    for _ in range(2):
      assert torch.equal(mod.forward_sparse(host), ref), name
    if B == 64:
      if name != 'LanczosNet':         # the drop-ins leave a blob's eigenpairs alone
        assert torch.equal(mod.forward_sparse(_packed(samples, 'pinned', eigs=True)), ref), name
      mod.use_cuda_graph = False
      assert torch.equal(mod.forward_sparse(res), ref), name
      assert torch.equal(mod.forward_sparse(host), ref), name


@pytest.mark.parametrize('name', sorted(MODELS))
def test_packed_odd_graphs_and_labels(name):
  samples = _odd_samples()
  mod = _build(name, seed=3)
  with torch.no_grad():
    ref = mod.forward_sparse(_records(samples, 'device'))
    assert torch.equal(mod.forward_sparse(_packed(samples, 'device')), ref)
    pool = data.PackedMolecules(samples, K, eigs=False)
    b = pool.batch(np.arange(len(samples)))
    host = _tensors(b, 'pinned')
    score, loss = mod.forward_sparse(host, label=host['label'].to(dev()))
    assert torch.equal(score, ref) and torch.isfinite(loss)


def test_lanczos_net_packed_without_eigenpairs_equals_both_records():
  """Without eigenpairs the blob runs records_unpack -> graph_eigs_sparse; the scores are those of the
  records without eigenpairs, which are (tests/test_gpu_graph_eigs.py) those of the host's eigenpairs."""
  samples = data.synthetic_qm8_samples(256, seed=8)
  mod = _build('LanczosNet')
  with torch.no_grad():
    ref = mod.forward_sparse(_records(samples, 'pinned'))
    assert torch.equal(mod.forward_sparse(_packed(samples, 'pinned')), ref)
    assert torch.equal(mod.forward_sparse(_packed(samples, 'device')), ref)
    # a device blob is told apart by batch['eigs']; the default is the blob with eigenpairs
    with_eigs = mod.forward_sparse(_packed(samples, 'device', eigs=True))
    assert torch.equal(with_eigs, mod.forward_sparse(_records(samples, 'device', eigs=True)))
    keys = {k[1] for k in mod._graphs}
    assert {'packed', 'packed_eigs', 'sparse_eigs', 'sparse'} <= keys, keys


@pytest.mark.parametrize('name', ['GCN', 'GGNN', 'GPNN', 'SampledGraphSAGE-Mean', 'LanczosNet'])
def test_one_capture_serves_batches_of_one_shape(name):
  """Batches of the same (B, N, K) with different node and bond totals replay ONE captured graph: the
  segment offsets are read on the device."""
  samples = data.synthetic_qm8_samples(400, seed=21)
  big = int(np.argmax([len(s['node_feat']) for s in samples]))
  pool = data.PackedMolecules(samples, K, eigs=False)
  rng = np.random.RandomState(0)
  idxs = []
  for _ in range(4):
    idx = rng.randint(0, len(samples), size=96)
    idx[rng.randint(96)] = big                       # N = 26 in every batch
    idxs.append(idx)
  mod = _build(name)
  with torch.no_grad():
    refs = [mod.forward_sparse(_records([samples[i] for i in idx], 'device')) for idx in idxs]
    mod.invalidate_caches()
    mod.__dict__.pop('_graph_stats', None)
    batches = [pool.batch(idx) for idx in idxs]
    assert len({(int(pool.sizes[idx].sum()), int(b['blob'].size)) for idx, b in zip(idxs, batches)}) == 4
    for b, ref in zip(batches, refs):
      assert torch.equal(mod.forward_sparse(_tensors(b, 'pinned')), ref)
    st = mod.graph_stats()
    assert st['captures'] == 1 and st['replays'] == 4, st


def test_sampled_graphsage_keys():
  samples = data.synthetic_qm8_samples(128, seed=4)
  mod = _build('SampledGraphSAGE-Mean')
  with torch.no_grad():
    scores = []
    for key in ((1234, 0), (1234, 1)):
      ref = mod.forward_sparse(_records(samples, 'device', key=key))
      assert torch.equal(mod.forward_sparse(_packed(samples, 'pinned', key=key)), ref)
      assert torch.equal(mod.forward_sparse(_packed(samples, 'device', key=key)), ref)
      scores.append(ref)
    assert not torch.equal(scores[0], scores[1])
    # a new key in the same device buffer: the captured graph reads it
    pk = _packed(samples, 'device', key=(1234, 0))
    for _ in range(3):
      assert torch.equal(mod.forward_sparse(pk), scores[0])
    pk['sample_key'].copy_(torch.tensor([1234, 1], dtype=torch.int64))
    assert torch.equal(mod.forward_sparse(pk), scores[1])


def test_host_refusal_of_a_malformed_pinned_blob_launches_nothing():
  samples = data.synthetic_qm8_samples(8, seed=1)
  pk = _packed(samples, 'pinned')
  pk['blob'][:4].view(torch.int32)[0] = 0
  mod = _build('GCN')
  n0 = ops.launch_count()
  with torch.no_grad(), pytest.raises(ValueError, match='magic'):
    mod.forward_sparse(pk)
  assert ops.launch_count() == n0


def test_keyed_gat_packed_with_a_dropout_key():
  samples = data.synthetic_qm8_samples(64, seed=13)
  mod = _build('KeyedGAT')
  dk = torch.tensor([5, 1], dtype=torch.int64, device=dev())
  with torch.no_grad():
    ref = mod.forward_sparse(dict(_records(samples, 'device'), dropout_key=dk))
    for where in ('pinned', 'device', 'device', 'device'):
      assert torch.equal(mod.forward_sparse(dict(_packed(samples, where), dropout_key=dk)), ref)


def _slices(batches):
  """Every batch's tensors copied into ONE reused device buffer per key, each call handed a slice of its
  own length (a loader that recycles device staging buffers)."""
  bufs = {}
  for b in batches:
    for k, v in b.items():
      if torch.is_tensor(v) and k != 'sample_key':
        n = max(bufs[k].shape[0] if k in bufs else 0, v.shape[0])
        bufs[k] = torch.zeros((n,) + tuple(v.shape[1:]), device=dev(), dtype=v.dtype)
  for b in batches:
    out = dict(b)
    for k, buf in bufs.items():
      view = buf[:b[k].shape[0]]
      view.copy_(b[k])
      out[k] = view
    yield out


@pytest.mark.parametrize('name', ['GCN', 'SampledGraphSAGE-Mean', 'LanczosNet'])
def test_growing_device_batches_from_reused_buffers(name):
  """Device batches of growing size, each a slice of the same reused buffer: every call reads its own batch,
  packed and records alike (the resident graphs are keyed by the slices' lengths, not only their addresses)."""
  samples = data.synthetic_qm8_samples(600, seed=17)
  big = int(np.argmax([len(s['node_feat']) for s in samples]))
  groups = []
  for n_small in (0, 40, 80, 120):                  # the same B and N, more and more node rows and bonds
    order = np.argsort([len(s['node_feat']) for s in samples])
    idx = np.concatenate([order[:96 - n_small - 1], order[-n_small - 1:-1] if n_small else [], [big]]).astype(int)
    groups.append([samples[i] for i in idx])
  mod = _build(name)
  with torch.no_grad():
    refs = [mod.forward_sparse(_records(g, 'device')) for g in groups]
    for fmt in (_packed, _records):
      mod.invalidate_caches()
      batches = [fmt(g, 'device') for g in groups]
      lens = [int(b['blob'].numel()) if 'blob' in b else int(b['edges'].shape[0]) for b in batches]
      assert lens == sorted(lens) and len(set(lens)) == 4, lens
      for b, ref in zip(_slices(batches), refs):
        for _ in range(3):            # copy-slot capture, resident capture, resident replay
          assert torch.equal(mod.forward_sparse(b), ref), (fmt.__name__, lens)


def test_device_blob_without_the_eigs_key_is_read_on_the_host():
  """A device blob whose batch does not say ``eigs`` has its header read with a small copy: LanczosNet
  picks the right path for both kinds of blob, and a malformed header is refused before any launch."""
  samples = data.synthetic_qm8_samples(128, seed=19)
  mod = _build('LanczosNet')
  with torch.no_grad():
    for eigs in (False, True):
      ref = mod.forward_sparse(_records(samples, 'device', eigs=eigs))
      pk = {k: v for k, v in _packed(samples, 'device', eigs=eigs).items() if k != 'eigs'}
      for _ in range(3):
        assert torch.equal(mod.forward_sparse(pk), ref), eigs
    bad = dict(pk, blob=pk['blob'].clone())
    bad['blob'][8:12] = 0                            # K = 0 in the header
    small = dict(pk, N=4)                            # node_ptr[B] > B * N
    n0 = ops.launch_count()
    for b, match in ((bad, 'K='), (small, 'node_ptr')):
      with pytest.raises(ValueError, match=match):
        mod.forward_sparse(b)
    assert ops.launch_count() == n0
