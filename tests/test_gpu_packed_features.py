"""Packed batches of float feature rows on the device: lnb_records_unpack_features against a numpy split of the
blob (its status on malformed headers and on blobs of the other kind, LNB_UNPACK_BAD_FEATURES both ways),
SparseLanczosNetGeneral.forward_sparse on feature blobs against the same records and against the padded
forward, one capture for every batch of a shape, and GraphedStep(packed=True) against GraphedStep(sparse=True).
``pytest -m gpu``."""
import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict
from lanczosnetwork_b200 import configs, data, ops, train
from lanczosnetwork_b200.model import SparseLanczosNetGeneral

pytestmark = pytest.mark.gpu

K = 20
F = 10
BAD_FEATURES = 128                                   # LNB_UNPACK_BAD_FEATURES
_SAMPLES = {}


def dev():
  return torch.device('cuda:0')


def _samples(B, seed):
  if (B, seed) not in _SAMPLES:
    _SAMPLES[B, seed] = data.synthetic_regression_graphs(B, seed=seed)     # G(n, 0.5), 20 <= n <= 100
  return _SAMPLES[B, seed]


def _build(seed=7):
  mod = SparseLanczosNetGeneral(configs.graph_lanczos_net())
  mod.load_state_dict(deterministic_state_dict(mod, seed))
  return mod.to(dev())


def _tensors(d, where):
  out = {}
  for k, v in d.items():
    if isinstance(v, np.ndarray):
      t = torch.from_numpy(v)
      out[k] = t.pin_memory() if where == 'pinned' else t.to(dev())
    else:
      out[k] = v
  return out


# ------------------------------------------------------------------------------------------------------
# lnb_records_unpack_features
@pytest.mark.parametrize('label', [False, True])
@pytest.mark.parametrize('eigs', [False, True])
@pytest.mark.parametrize('B, seed', [(1, 2), (13, 3)])
def test_records_unpack_features_is_the_numpy_split(B, seed, eigs, label):
  sp = data.sparse_collate(_samples(B, seed), K, eigs=eigs)
  pk = data.pack_sparse(sp, label=label)
  blob = torch.from_numpy(pk['blob']).to(dev())
  rows, nedge = int(sp['node_ptr'][-1]), int(sp['edge_ptr'][-1])
  P = sp['label'].shape[1] if label else 0
  out = ops.records_unpack(blob, B, K, rows + 5, nedge + 7, eigs=eigs, label_dim=P, feature_dim=F)
  status = out[-1]
  assert int(status.item()) == 0
  sizes, node_ptr, node_x, edge_ptr, edges, D, V_rows = out[:7]
  assert node_x.dtype == torch.float32 and tuple(node_x.shape) == (rows + 5, F)
  assert np.array_equal(sizes.cpu().numpy(), sp['sizes'])
  assert np.array_equal(node_ptr.cpu().numpy(), sp['node_ptr'])
  assert np.array_equal(edge_ptr.cpu().numpy(), sp['edge_ptr'])
  assert np.array_equal(node_x[:rows].cpu().numpy().view(np.uint32), sp['node_feat'].view(np.uint32))
  assert np.array_equal(edges[:nedge].cpu().numpy(), sp['edges'])
  if eigs:
    assert np.array_equal(D.cpu().numpy(), sp['D'])
    assert np.array_equal(V_rows[:rows].cpu().numpy(), sp['V_rows'])
  if label:
    assert np.array_equal(out[7].cpu().numpy(), sp['label'])


def _status(blob, B, feature_dim, eigs=False):
  out = ops.records_unpack(blob, B, K, B * 100, 200000, eigs=eigs, feature_dim=feature_dim)
  st = int(out[-1].item())
  if st:                                             # every graph empty
    assert not out[0].any() and not out[1].any() and not out[3].any()
  return st


def test_records_unpack_features_status_on_malformed_headers():
  B = 5
  feat = torch.from_numpy(data.pack_sparse(data.sparse_collate(_samples(B, 4), K))['blob']).to(dev())
  atom = torch.from_numpy(data.pack_sparse(data.sparse_collate(data.synthetic_qm8_samples(B, seed=4), K))['blob'])
  atom = atom.to(dev())
  assert _status(feat, B, F, eigs=True) == 0 and _status(atom, B, 0, eigs=True) == 0
  # the other kind of blob, both ways, and another width
  assert _status(atom, B, F) == BAD_FEATURES
  assert _status(feat, B, 0) == BAD_FEATURES
  assert _status(feat, B, F + 2) == BAD_FEATURES
  label_out = ops.records_unpack(feat, B, K, B * 100, 200000, label_dim=2)     # lnb_records_unpack_labels
  assert int(label_out[-1].item()) & BAD_FEATURES

  def edited(blob, slot, value):
    b = blob.clone()
    b[:64].view(torch.int32)[slot] = value
    return b

  assert _status(edited(feat, 0, 0x1234), B, F) == 1                          # magic
  assert _status(edited(feat, 1, B + 1), B, F) == 2                           # B
  assert _status(edited(feat, 15, 3), B, F) == BAD_FEATURES
  assert _status(edited(feat, 7, 40), B, F) == 4                              # node segment in the header
  assert _status(edited(feat, 10, feat.numel() + 16), B, F) == 4              # total past the allocation
  # a node segment with room for one atom id per node but not for F floats: the width sets its size
  h = data.read_packed_header(feat.cpu())
  rows = int(feat[h.node_ptr + 4 * B:h.node_ptr + 4 * B + 4].cpu().view(torch.int32).item())
  off = (h.total - 4 * rows) // 16 * 16
  assert off >= 64
  assert _status(edited(feat, 7, off), B, F) == 4
  small = ops.records_unpack(feat, B, K, 3, 200000, feature_dim=F)
  assert int(small[-1].item()) == 8                                           # rows over the capacity


# ------------------------------------------------------------------------------------------------------
# forward_sparse on feature blobs
def _packed(samples, eigs, where):
  pk = data.pack_sparse(data.sparse_collate(samples, K, eigs=eigs))
  return _tensors(pk, where)


@pytest.mark.parametrize('where', ['pinned', 'device'])
@pytest.mark.parametrize('eigs', [False, True])
@pytest.mark.parametrize('B, seed', [(16, 17), (1024, 5)])
def test_forward_sparse_on_feature_blobs_equals_the_records(B, seed, eigs, where):
  samples = _samples(B, seed)
  mod = _build().eval()
  rec = _tensors(data.sparse_collate(samples, K, eigs=eigs), where)
  pk = _packed(samples, eigs, where)
  assert pk['F'] == F and pk['N'] <= 100
  with torch.no_grad():
    want = mod.forward_sparse(rec)
    for _ in range(3):                 # capture, replay (and, from a device blob, the resident capture)
      assert torch.equal(mod.forward_sparse(pk), want)
    mod.use_cuda_graph = False
    assert torch.equal(mod.forward_sparse(pk), want)
    # without batch['F'] the header is read on the host first; the scores are the same
    assert torch.equal(mod.forward_sparse({k: v for k, v in pk.items() if k != 'F'}), want)


def test_feature_blob_with_eigenpairs_gives_the_padded_forward():
  samples = _samples(16, 17)
  mod = _build().eval()
  c = data.collate(samples, K)
  args = [torch.from_numpy(c[k]).to(dev()) for k in ('node_feat', 'L', 'D', 'V')]
  with torch.no_grad():
    want = mod(*args, mask=torch.from_numpy(c['node_mask']).to(dev()))
    assert torch.equal(mod.forward_sparse(_packed(samples, True, 'pinned')), want)


@pytest.mark.parametrize('eigs', [False, True])
def test_one_capture_serves_feature_blobs_of_one_shape(eigs):
  samples = _samples(96, 9)
  pool = data.PackedMolecules(samples, K, eigs=eigs)
  big = int(np.argmax(pool.sizes))
  rng = np.random.RandomState(2)
  mod = _build().eval()
  buf = torch.zeros(pool.max_bytes(32), dtype=torch.uint8).pin_memory()
  sizes = set()
  with torch.no_grad():
    for i in range(4):
      idx = rng.choice(len(samples), size=32, replace=False)
      if big not in idx:
        idx[0] = big
      want = mod.forward_sparse(_tensors(data.sparse_collate([samples[j] for j in idx], K, eigs=eigs), 'pinned'))
      torch.cuda.synchronize()                       # the previous replay has read the buffer
      b = pool.batch(idx, out=buf.numpy())
      sizes.add(b['blob'].size)
      got = mod.forward_sparse(dict(b, blob=buf[:b['blob'].size]))
      assert torch.equal(got, want), i
  assert len(sizes) == 4
  key = ('packed', 32, int(pool.sizes.max()), K) if eigs else ('packed_eigs', 32, int(pool.sizes.max()), K)
  assert sum(1 for k in mod._graphs if k[1:5] == key) == 1


# ------------------------------------------------------------------------------------------------------
# GraphedStep(packed=True) against GraphedStep(sparse=True)
def _batches(n, B, seed, eigs):
  samples = _samples(4 * B, seed)
  pool = data.PackedMolecules(samples, K, eigs=eigs, labels=True)
  big = int(np.argmax(pool.sizes))
  rng = np.random.RandomState(seed)
  out = []
  for _ in range(n):
    idx = rng.choice(len(samples), size=B, replace=False)
    if big not in idx:
      idx[rng.randint(B)] = big
    out.append((pool.batch(idx), data.sparse_collate([samples[i] for i in idx], K, eigs=eigs)))
  return out


def _run(batches, packed, optimizer):
  mod = _build()
  if packed:
    pks = [_tensors(pk, 'pinned') for pk, _ in batches]
    step = train.GraphedStep(mod, optimizer(mod), (pks[0],), packed=True)
    calls = [((pk,), {}) for pk in pks]
  else:
    recs = [_tensors(sp, 'pinned') for _, sp in batches]
    labels = [r.pop('label').to(dev()) for r in recs]
    step = train.GraphedStep(mod, optimizer(mod), (recs[0],), {'label': labels[0]}, sparse=True)
    calls = [((r,), {'label': lab}) for r, lab in zip(recs, labels)]
  out = []
  for args, kw in calls:
    score, loss = step(*args, **kw)
    if packed:
      assert int(step.status.item()) == 0
    out.append((score.clone(), loss.clone()))
  return mod, out


def _adam(mod):
  return torch.optim.Adam(mod.parameters(), lr=1e-3)


def _sgd(mod):
  return torch.optim.SGD(mod.parameters(), lr=1e-2, momentum=0.9)


@pytest.mark.parametrize('eigs', [False, True])
def test_packed_steps_follow_the_records_steps(eigs):
  batches = _batches(3, 64, seed=41, eigs=eigs)
  rec_a, out_a = _run(batches, False, _adam)
  rec_b, _ = _run(batches, False, _adam)
  pk, out_p = _run(batches, True, _adam)
  assert torch.equal(out_p[0][0], out_a[0][0]) and torch.equal(out_p[0][1], out_a[0][1])
  if all(torch.equal(p, q) for p, q in zip(rec_a.parameters(), rec_b.parameters())):
    for (sa, la), (sp_, lp) in zip(out_a, out_p):
      assert torch.equal(sp_, sa) and torch.equal(lp, la)
    for (n, p), (_, q) in zip(rec_a.named_parameters(), pk.named_parameters()):
      assert torch.equal(q, p), n
    return
  # a gradient summed with atomics: two records runs differ in the last bits too, so the packed run is held to
  # the records run within the tolerance, under momentum SGD, as tests/test_gpu_packed_train.py does
  for (sa, la), (sp_, lp) in zip(out_a, out_p):
    torch.testing.assert_close(lp, la, rtol=2e-4, atol=2e-6)
  rec_s, _ = _run(batches, False, _sgd)
  pk_s, _ = _run(batches, True, _sgd)
  for (n, p), (_, q) in zip(rec_s.named_parameters(), pk_s.named_parameters()):
    torch.testing.assert_close(q, p, rtol=2e-4, atol=2e-6, msg=lambda m: '%s: %s' % (n, m))
