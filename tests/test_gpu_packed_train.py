"""Training from packed batches on the device: lnb_records_unpack_labels against a numpy split of the blob (its
status without the label segment or with another P), inference unchanged by a label segment, and
GraphedStep(packed=True) against GraphedStep(sparse=True) on the same batches for every model it trains --
one capture for every batch of a shape, and refusals that leave the model untouched."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data, ops, train
from lanczosnetwork_b200.model import (DCNN, GCN, GCNFP, GGNN, GPNN, MPNN, ChebyNet, KeyedGAT, LanczosNet,
                                       SampledGraphSAGE, TrainableGAT)

from helpers import deterministic_state_dict

pytestmark = pytest.mark.gpu

K = 20
SENTINEL = 0x5A
MODELS = {
    'GCN': lambda: GCN(configs.qm8_gcn()),
    'GCNFP': lambda: GCNFP(configs.qm8_gcn()),
    'DCNN': lambda: DCNN(configs.qm8_dcnn()),
    'ChebyNet': lambda: ChebyNet(configs.qm8_cheby_net()),
    'TrainableGAT': lambda: TrainableGAT(configs.qm8_gat()),
    'KeyedGAT': lambda: KeyedGAT(configs.qm8_gat(dropout=0.1)),
    'GGNN': lambda: GGNN(configs.qm8_ggnn()),
    'MPNN': lambda: MPNN(configs.qm8_mpnn()),
    'GPNN': lambda: GPNN(configs.qm8_gpnn()),
    'SampledGraphSAGE-Mean': lambda: SampledGraphSAGE(configs.qm8_graphsage(agg_func='Mean')),
    'SampledGraphSAGE-Max': lambda: SampledGraphSAGE(configs.qm8_graphsage(agg_func='Max')),
    'SampledGraphSAGE-LSTM': lambda: SampledGraphSAGE(configs.qm8_graphsage(agg_func='LSTM')),
    'LanczosNet': lambda: LanczosNet(configs.qm8_lanczos_net()),
}


def dev():
  return torch.device('cuda:0')


def _build(name, seed=7):
  mod = MODELS[name]()
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
# lnb_records_unpack_labels
def _unpack_raw(blob, B, cap_rows, cap_edges, P, labels=True, slack=64):
  """The unpack into buffers ``slack`` elements longer than the capacities, filled with a sentinel (the old
  entry when ``labels`` is False).  Returns the buffers (full length) and the status."""
  fill = lambda n, dtype: torch.full((4 * n,), SENTINEL, device=dev(), dtype=torch.uint8).view(dtype)
  out = {'sizes': fill(B + slack, torch.int32), 'node_ptr': fill(B + 1 + slack, torch.int32),
         'edge_ptr': fill(B + 1 + slack, torch.int32), 'node_feat': fill(cap_rows + slack, torch.int32),
         'edges': fill(cap_edges + slack, torch.uint8).view(-1, 4), 'label': fill(B * P + slack, torch.float32)}
  status = torch.full((1,), -1, device=dev(), dtype=torch.int32)
  args = (blob, blob.numel(), B, K, cap_rows, cap_edges, out['sizes'], out['node_ptr'], out['node_feat'],
          out['edge_ptr'], out['edges'], None, None, status)
  if labels:
    ops._launch('lnb_records_unpack_labels', blob, *args, P, out['label'])
  else:
    ops._launch('lnb_records_unpack', blob, *args)
  torch.cuda.synchronize()
  return {k: v.cpu().numpy() for k, v in out.items()}, int(status.item())


def _sent(dtype):
  return np.full(1, SENTINEL, np.uint8).repeat(np.dtype(dtype).itemsize).view(dtype)[0]


@pytest.mark.parametrize('B, seed', [(1, 2), (7, 3), (1024, 4)])
def test_records_unpack_labels_is_the_numpy_split(B, seed):
  sp = data.sparse_collate(data.synthetic_qm8_samples(B, seed=seed), K, eigs=False)
  pk = data.pack_sparse(sp, label=True)
  P = sp['label'].shape[1]
  rows, nedge = int(sp['node_ptr'][-1]), int(sp['edge_ptr'][-1])
  buf = torch.full((pk['blob'].size + 4096,), 0xEE, dtype=torch.uint8)      # stale bytes past hdr[10]
  buf[:pk['blob'].size] = torch.from_numpy(pk['blob'])
  blob = buf.to(dev())
  cap_rows, cap_edges = rows + 37, nedge + 5
  out, status = _unpack_raw(blob, B, cap_rows, cap_edges, P)
  assert status == 0
  assert np.array_equal(out['sizes'][:B], sp['sizes']) and np.all(out['sizes'][B:] == _sent(np.int32))
  assert np.array_equal(out['node_ptr'][:B + 1], sp['node_ptr']) and np.all(out['node_ptr'][B + 1:] == _sent(np.int32))
  assert np.array_equal(out['edge_ptr'][:B + 1], sp['edge_ptr']) and np.all(out['edge_ptr'][B + 1:] == _sent(np.int32))
  assert np.array_equal(out['node_feat'][:rows], sp['node_feat']) and np.all(out['node_feat'][rows:] == _sent(np.int32))
  assert np.array_equal(out['edges'][:nedge], sp['edges']) and np.all(out['edges'][nedge:] == SENTINEL)
  assert np.array_equal(out['label'][:B * P].view(np.int32), sp['label'].reshape(-1).view(np.int32))
  assert np.all(out['label'][B * P:].view(np.uint8) == SENTINEL)
  # the old entry on the labelled blob: today's records, the label buffer untouched
  old, status = _unpack_raw(blob, B, cap_rows, cap_edges, P, labels=False)
  assert status == 0 and np.all(old['label'].view(np.uint8) == SENTINEL)
  for k in ('sizes', 'node_ptr', 'edge_ptr', 'node_feat', 'edges'):
    assert np.array_equal(old[k], out[k]), k
  # the op: the 9-tuple with label_dim, today's 8-tuple without
  got = ops.records_unpack(blob, B, K, cap_rows, cap_edges, label_dim=P)
  assert len(got) == 9 and int(got[8].item()) == 0 and got[5] is None and got[6] is None
  assert torch.equal(got[7].cpu(), torch.from_numpy(sp['label']))
  plain = ops.records_unpack(blob, B, K, cap_rows, cap_edges)
  assert len(plain) == 8 and int(plain[7].item()) == 0
  for a, b, n in zip(plain[:5], got[:5], (B, B + 1, rows, B + 1, nedge)):   # rows past the batch are unwritten
    assert torch.equal(a[:n], b[:n])


def test_records_unpack_labels_refuses_missing_and_other_label_segments():
  sp = data.sparse_collate(data.synthetic_qm8_samples(9, seed=1), K, eigs=False)
  B, P = sp['label'].shape
  rows, nedge = int(sp['node_ptr'][-1]), int(sp['edge_ptr'][-1])
  labelled = data.pack_sparse(sp, label=True)['blob']
  hdr = labelled[:64].view(np.int32)

  def edit(i, v):
    b = labelled.copy()
    b[:64].view(np.int32)[i] = v
    return torch.from_numpy(b).to(dev())

  cases = [(torch.from_numpy(data.pack_sparse(sp)['blob']).to(dev()), P),          # no label segment
           (torch.from_numpy(labelled).to(dev()), P - 1), (torch.from_numpy(labelled).to(dev()), P + 1),
           (edit(13, int(hdr[13]) + 4), P), (edit(13, int(hdr[10])), P)]             # unaligned, past the total
  for blob, want_p in cases:
    out, status = _unpack_raw(blob, B, rows, nedge, want_p)
    assert status == 64, status
    assert np.all(out['sizes'][:B] == 0) and np.all(out['node_ptr'][:B + 1] == 0) and np.all(out['edge_ptr'][:B + 1] == 0)
    assert np.all(out['node_feat'] == _sent(np.int32)) and np.all(out['edges'] == SENTINEL)
    assert np.all(out['label'].view(np.uint8) == SENTINEL)
  # other failures keep their own bits
  assert _unpack_raw(edit(0, 0), B, rows, nedge, P)[1] == 1
  assert _unpack_raw(torch.from_numpy(labelled).to(dev()), B, rows - 1, nedge, P)[1] == 8


@pytest.mark.parametrize('name', ['GCN', 'GGNN', 'SampledGraphSAGE-Mean', 'KeyedGAT', 'LanczosNet'])
def test_inference_is_unchanged_by_a_label_segment(name):
  samples = data.synthetic_qm8_samples(64, seed=31)
  mod = _build(name).eval()
  key = torch.tensor([1234, 0], dtype=torch.int64)
  with torch.no_grad():
    for eigs in (False, True):
      sp = data.sparse_collate(samples, K, eigs=eigs)
      for where in ('pinned', 'device'):
        plain = dict(_tensors(data.pack_sparse(sp), where), sample_key=key.to(dev()))
        lab = dict(_tensors(data.pack_sparse(sp, label=True), where), sample_key=key.to(dev()))
        ref = mod.forward_sparse(plain)
        for _ in range(3):
          assert torch.equal(mod.forward_sparse(lab), ref), (name, eigs, where)


# ------------------------------------------------------------------------------------------------------
# GraphedStep(packed=True) against GraphedStep(sparse=True)
def _pool_batches(n_batches, B, seed, eigs):
  """``n_batches`` index sets of B molecules with the largest molecule in each (one N): (pool, [(idx, packed
  batch with labels in the blob, records)])."""
  samples = data.synthetic_qm8_samples(4 * B, seed=seed)
  pool = data.PackedMolecules(samples, K, eigs=eigs, labels=True)
  big = int(np.argmax(pool.sizes))
  rng = np.random.RandomState(seed)
  out = []
  for _ in range(n_batches):
    idx = rng.choice(len(samples), size=B, replace=False)
    if big not in idx:
      idx[rng.randint(B)] = big
    out.append((idx, pool.batch(idx), data.sparse_collate([samples[i] for i in idx], K, eigs=eigs)))
  return pool, out


def _keys(name, i, key_seed):
  if name.startswith('SampledGraphSAGE'):
    return {'sample_key': torch.tensor([key_seed, i], dtype=torch.int64)}
  if name == 'KeyedGAT':
    return {'dropout_key': torch.tensor([key_seed, i], dtype=torch.int64)}
  return {}


def _adam(mod):
  return torch.optim.Adam(mod.parameters(), lr=1e-3)


def _sgd(mod):
  return torch.optim.SGD(mod.parameters(), lr=1e-2, momentum=0.9)


def _run_records(name, batches, key_seed, optimizer=_adam):
  mod = _build(name)
  recs = [dict(_tensors(sp, 'pinned'), **_keys(name, i, key_seed)) for i, (_, _, sp) in enumerate(batches)]
  labels = [r.pop('label').to(dev()) for r in recs]
  step = train.GraphedStep(mod, optimizer(mod), (recs[0],), {'label': labels[0]}, sparse=True)
  out = []
  for r, lab in zip(recs, labels):
    score, loss = step(r, label=lab)
    out.append((score.clone(), loss.clone()))
  return mod, out


def _run_packed(name, batches, key_seed, optimizer=_adam):
  mod = _build(name)
  pks = [dict(_tensors(pk, 'pinned'), **_keys(name, i, key_seed)) for i, (_, pk, _) in enumerate(batches)]
  step = train.GraphedStep(mod, optimizer(mod), (pks[0],), packed=True)
  out = []
  for pk in pks:
    score, loss = step(pk)
    assert int(step.status.item()) == 0
    out.append((score.clone(), loss.clone()))
  return mod, out


CASES = [(n, False, 1234) for n in sorted(MODELS) if n != 'LanczosNet'] + [
    ('SampledGraphSAGE-Mean', False, 77), ('LanczosNet', False, 0), ('LanczosNet', True, 0)]


@pytest.mark.parametrize('name, eigs, key_seed', CASES)
def test_packed_steps_follow_the_records_steps(name, eigs, key_seed):
  _, batches = _pool_batches(5, 64, seed=41, eigs=eigs)
  rec_a, out_a = _run_records(name, batches, key_seed)
  rec_b, out_b = _run_records(name, batches, key_seed)
  pk, out_p = _run_packed(name, batches, key_seed)
  assert torch.equal(out_p[0][0], out_a[0][0]) and torch.equal(out_p[0][1], out_a[0][1]), name
  for i, ((sa, la), (sp_, lp)) in enumerate(zip(out_a, out_p)):
    torch.testing.assert_close(lp, la, rtol=2e-4, atol=2e-6, msg=lambda m: '%s step %d: %s' % (name, i, m))
  # the weights: bit-equal wherever two records runs are.  Elsewhere (a gradient summed with atomics) Adam
  # turns last-bit differences into moves of about lr where a gradient is ~ 0 -- two records runs differ so
  # too -- and the weights are compared within the tolerance under momentum SGD, as tests/test_gpu_sparse_train.py does
  if all(torch.equal(p, q) for p, q in zip(rec_a.parameters(), rec_b.parameters())):
    for (n, p), (_, q) in zip(rec_a.named_parameters(), pk.named_parameters()):
      assert torch.equal(q, p), (name, n)
    return
  rec_s, _ = _run_records(name, batches, key_seed, optimizer=_sgd)
  pk_s, _ = _run_packed(name, batches, key_seed, optimizer=_sgd)
  for (n, p), (_, q) in zip(rec_s.named_parameters(), pk_s.named_parameters()):
    torch.testing.assert_close(q, p, rtol=2e-4, atol=2e-6, msg=lambda m: '%s %s: %s' % (name, n, m))


@pytest.mark.parametrize('name', ['GCN', 'SampledGraphSAGE-Mean', 'LanczosNet'])
@pytest.mark.parametrize('where', ['pinned', 'device'])
def test_one_capture_serves_batches_of_one_shape(name, where):
  """Four batches of one (B, N, K, P) with different node and bond totals: one capture (its warm-up rolled
  back), four replays, the records step's losses.  Pinned blobs are assembled into two reused buffers, each
  refilled once the ``input_consumed`` event of the call that read it has completed."""
  pool, batches = _pool_batches(4, 96, seed=53, eigs=False)
  assert len({int(pk['blob'].size) for _, pk, _ in batches}) == 4
  _, out_r = _run_records(name, batches, 1234)
  base, mod = _build(name), _build(name)
  if where == 'pinned':
    bufs = [torch.zeros(pool.max_bytes(96), dtype=torch.uint8).pin_memory() for _ in range(2)]
    events = [None, None]
  pks = [dict(_tensors(pk, where), **_keys(name, i, 1234)) for i, (_, pk, _) in enumerate(batches)]
  step = train.GraphedStep(mod, _adam(mod), (pks[0],), packed=True)
  for (n, p), (_, q) in zip(mod.named_parameters(), base.named_parameters()):
    assert torch.equal(p, q), n                                  # warm-up rolled back
  for i, (idx, _, _) in enumerate(batches):
    batch = pks[i]
    if where == 'pinned':
      slot = i % 2
      if events[slot] is not None:
        events[slot].synchronize()                               # the copy out of this buffer is done
      b = pool.batch(idx, out=bufs[slot].numpy())
      batch = dict(b, blob=bufs[slot][:b['blob'].size], **_keys(name, i, 1234))
    _, loss = step(batch)
    if where == 'pinned':
      events[slot] = step.input_consumed
    assert int(step.status.item()) == 0
    torch.testing.assert_close(loss, out_r[i][1], rtol=2e-4, atol=2e-6)
  assert step.replays == 4


@pytest.mark.parametrize('name', ['GCN', 'LanczosNet'])
def test_refused_batches_launch_nothing_and_leave_the_model_alone(name):
  pool, batches = _pool_batches(2, 64, seed=61, eigs=False)
  mod = _build(name)
  opt = _adam(mod)
  first = _tensors(batches[0][1], 'pinned')
  step = train.GraphedStep(mod, opt, (first,), packed=True)
  step(first)
  torch.cuda.synchronize()
  params = [p.detach().clone() for p in mod.parameters()]
  state = [{k: v.clone() for k, v in opt.state[p].items()} for p in mod.parameters()]
  static = step._args[0]['blob'].clone()
  cap = static.numel()
  over = torch.zeros(cap + 64, dtype=torch.uint8).pin_memory()
  over[:first['blob'].numel()] = first['blob']
  over[:64].view(torch.int32)[10] = cap + 64                     # hdr[10] past the captured capacity
  bad = first['blob'].clone().pin_memory()
  bad[:4].view(torch.int32)[0] = 0
  unlabelled = _tensors(data.pack_sparse(batches[1][2]), 'pinned')
  n0 = ops.launch_count()
  for b, match in ((dict(first, blob=over), 'capacity'), (dict(first, blob=bad), 'magic'), (unlabelled, 'labels')):
    with pytest.raises(ValueError, match=match):
      step(b)
  with pytest.raises(ValueError, match='label='):
    step(first, label=torch.zeros(64, 16, device=dev()))
  assert ops.launch_count() == n0
  torch.cuda.synchronize()
  assert torch.equal(step._args[0]['blob'], static)
  for p, q in zip(mod.parameters(), params):
    assert torch.equal(p, q)
  for p, st in zip(mod.parameters(), state):
    assert all(torch.equal(opt.state[p][k], v) for k, v in st.items())
