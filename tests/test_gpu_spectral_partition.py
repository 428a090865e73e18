"""GPNN's device partition (lnb_spectral_partition / ops.spectral_partition) on the GPU: the reference's
partitions (gpnn_qm8.npz, gpnn_partitions.npz), the fp64 oracle (tests/partition_oracle.py) on QM8-shaped
batches and G(n, 0.5) graphs up to N = 128, the operators bit for bit, status bits, determinism and
capture, envelope refusals, and GPNN with device partitioning (inference, training, GraphedStep).
``pytest -m gpu``."""
import ctypes

import numpy as np
import pytest
import torch

import partition_oracle
from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import _lib, configs, data, ops
from lanczosnetwork_b200.model import GPNN
from oracle import gpnn_oracle
from test_host_spectral_partition import golden_operators

pytestmark = pytest.mark.gpu

EQUAL_INERTIA = 1e-9


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _check_operators(L0, labels, Lc, Lt):
  want_c, want_t = data.partition_operators(L0.cpu().numpy(), labels.cpu().numpy())
  assert torch.equal(Lc.cpu(), _t(want_c)) and torch.equal(Lt.cpu(), _t(want_t))


def test_reference_golden_labels_and_operators():
  g, gp = load_golden('lanczosnet_qm8.npz'), load_golden('gpnn_qm8.npz')
  L = _t(g['L']).to(dev())
  labels, Lc, Lt, status = ops.spectral_partition(L, 3)
  assert np.array_equal(labels.cpu().numpy(), gp['partition_labels'])
  assert int((status & 0b1101).sum()) == 0
  assert torch.equal(Lc.cpu(), _t(gp['L_cluster'])) and torch.equal(Lt.cpu(), _t(gp['L_cut']))
  _check_operators(L[..., 0], labels, Lc, Lt)


def _batches_of(ops_list, sizes):
  """Group consecutive fixture graphs with equal N into [B, N, N] batches (the collate's batches)."""
  out, i = [], 0
  while i < len(ops_list):
    j = i
    while j < len(ops_list) and sizes[j] == sizes[i]:
      j += 1
    out.append((i, np.stack(ops_list[i:j])))
    i = j
  return out


def test_fixture_partitions_match_reference_and_oracle():
  """Every graph without a tie flag gets the reference's canonical partition, except where KMeans is
  undetermined (a tie in its seeding or assignment, or an alternative with the same inertia); those are a
  handful.  Includes the N = 64 batch (CTA eigen path)."""
  gp = load_golden('gpnn_partitions.npz')
  P = int(gp['num_partition'])
  Ls = golden_operators()
  alt, checked = [], 0
  for k0, L in _batches_of(Ls, gp['N']):
    L32 = _t(L.astype(np.float32)).to(dev())
    labels, Lc, Lt, status = ops.spectral_partition(L32, P)
    _check_operators(L32, labels, Lc, Lt)
    lab = labels.cpu().numpy()
    st = status.cpu().numpy()
    assert not (st & 0b1101).any(), st
    for i in range(L.shape[0]):
      k, N = k0 + i, L.shape[1]
      if gp['tie'][k]:
        assert st[i] & 2, k
        continue
      if np.array_equal(lab[i], gp['labels'][k, :N]):
        checked += 1
        continue
      # otherwise the reference is undetermined: a KMeans tie, or an alternative with the same inertia
      orc = partition_oracle.spectral_clustering(L[i], P)
      inertia = _best_inertia(L[i], P, lab[i])
      if orc['kmeans_tie']:
        continue
      assert abs(inertia - gp['inertia'][k]) <= EQUAL_INERTIA * gp['inertia'][k], (k, inertia, gp['inertia'][k])
      alt.append(k)
  assert checked >= 950 and len(alt) <= 8, (checked, alt)


def _best_inertia(L, P, lab):
  """Inertia of a canonical partition: the nodes without an edge (-1, the padding, one point of the
  embedding) joined to whichever cluster gives the least within-cluster sum of squares."""
  return min(partition_oracle.partition_inertia(L, P, np.where(lab < 0, c, lab)) for c in range(P))


@pytest.mark.parametrize('N,P', [(20, 3), (33, 4), (64, 7), (100, 16), (128, 5)])
def test_random_graphs_against_oracle(N, P):
  rng = np.random.RandomState(N * 31 + P)
  B = 6
  L = np.zeros((B, N, N))
  for b in range(B):
    n = int(rng.randint(max(P + 2, N - 12), N + 1))
    A = np.triu((rng.rand(n, n) < 0.5).astype(np.float64), 1)
    L[b, :n, :n] = data.get_laplacian(A + A.T, 'L4')
  L32 = _t(L.astype(np.float32)).to(dev())
  labels, Lc, Lt, status = ops.spectral_partition(L32, P)
  _check_operators(L32, labels, Lc, Lt)
  lab, st = labels.cpu().numpy(), status.cpu().numpy()
  assert not (st & 0b1101).any(), st
  for b in range(B):
    orc = partition_oracle.spectral_clustering(L[b], P)
    if orc['tie']:
      assert st[b] & 2
      continue
    if not np.array_equal(lab[b], orc['labels']):       # only where KMeans is undetermined
      inertia = _best_inertia(L[b], P, lab[b])
      assert orc['kmeans_tie'] or abs(inertia - orc['inertia']) <= EQUAL_INERTIA * orc['inertia'], \
          (b, inertia, orc['inertia'])


def test_status_bits_weighted_and_tie():
  rng = np.random.RandomState(2)
  L = np.zeros((2, 12, 12))
  A = np.triu((rng.rand(10, 10) < 0.4).astype(np.float64), 1)
  L[0, :10, :10] = data.get_laplacian(A + A.T, 'L4')
  L[0, 1, 2] = L[0, 2, 1] = 0.77                    # weighted: not the L4 of its pattern
  tri_ = np.ones((3, 3)) - np.eye(3)                # two identical triangles: every |lambda| is doubled
  two = np.zeros((6, 6))
  two[:3, :3] = tri_
  two[3:, 3:] = tri_
  L[1, :6, :6] = data.get_laplacian(two, 'L4')
  _, _, _, status = ops.spectral_partition(_t(L.astype(np.float32)).to(dev()), 3)
  st = status.cpu().numpy()
  assert st[0] & 8 and not st[1] & 8
  assert st[1] & 2


def test_repeatable_and_capturable():
  g = load_golden('lanczosnet_qm8.npz')
  L = _t(g['L']).to(dev())
  Lbig = _t(np.stack(golden_operators()[-16:]).astype(np.float32)).to(dev())
  for X in (L, Lbig):
    a = ops.spectral_partition(X, 3)
    b = ops.spectral_partition(X, 3)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
      with torch.cuda.graph(graph, stream=s):
        c = ops.spectral_partition(X, 3)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, c))


def test_envelope_refusals_launch_nothing():
  lib = _lib.load()
  L = torch.zeros((2, 129, 129), device=dev())
  out = [torch.zeros((2, 129), dtype=torch.int32, device=dev()), torch.zeros((2, 129, 129), device=dev()),
         torch.zeros((2, 129, 129), device=dev()), torch.zeros((2,), dtype=torch.int32, device=dev())]
  table = ops._inv_sqrt_deg_table(dev())
  draws = torch.zeros((64,), dtype=torch.float64, device=dev())
  ptr = lambda t: ctypes.c_void_p(t.data_ptr())
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  n0 = ops.launch_count()
  for N, P in ((129, 3), (40, 17), (40, 1), (5, 5), (1, 2)):
    rc = lib.lnb_spectral_partition(stream, ptr(L), 1, 2, N, P, ptr(table), ptr(draws), *[ptr(t) for t in out])
    assert rc == -2, (N, P, rc)
  torch.cuda.synchronize()
  assert ops.launch_count() == n0
  assert lib.lnb_spectral_partition_draws(17) == 0 and lib.lnb_spectral_partition_draws(3) == 1 + 2 * 3


def _build(cfg, seed):
  mod = GPNN(cfg)
  params = deterministic_state_dict(mod, seed)
  mod.load_state_dict(params)
  return mod.to(dev()).eval(), params


@pytest.mark.parametrize('prefix,over,dseed', [('config', {}, 0), ('small', dict(
    hidden_dim=32, num_prop=3, num_prop_cluster=2, num_prop_cut=1, aggregate_type='sum', update_func='RNN',
    output_dim=16), 1)], ids=['config', 'small'])
def test_model_device_partition_equals_golden_operators(prefix, over, dseed):
  g, gp = load_golden('lanczosnet_qm8.npz'), load_golden('gpnn_qm8.npz')
  nf, L, mask = _t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['node_mask']).to(dev())
  Lc, Lt = _t(gp['L_cluster']).to(dev()), _t(gp['L_cut']).to(dev())
  label = _t(g['label']).to(dev())
  mod, _ = _build(configs.qm8_gpnn(**over), int(gp['weight_seed']) + dseed)
  B = L.shape[0]
  empty = torch.zeros((B, 0, 0), device=dev())
  with torch.no_grad():
    want, want_loss = mod(nf, L, Lc, Lt, label=label, mask=mask)
    for _ in range(2):                       # eager-then-captured, then replays
      got, loss = mod(nf, L, label=label, mask=mask)
      assert torch.equal(got, want) and torch.equal(loss, want_loss)
      got = mod(nf, L, empty, empty.clone(), label=label, mask=mask)[0]
      assert torch.equal(got, want)
  np.testing.assert_allclose(want.cpu().numpy(), gp['%s_score' % prefix], rtol=1e-4, atol=2e-5)
  with pytest.raises(ValueError):
    mod(nf, L, Lc, None)


def test_training_gradients_equal_host_operators():
  """Partitioned on the device, the operators are the golden ones bit for bit, so the gradients agree up to
  the summation order of the backward's atomics."""
  g, gp = load_golden('lanczosnet_qm8.npz'), load_golden('gpnn_qm8.npz')
  nf, L, mask = _t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['node_mask']).to(dev())
  Lc, Lt = _t(gp['L_cluster']).to(dev()), _t(gp['L_cut']).to(dev())
  label = _t(g['label']).to(dev())
  grads = []
  for ops_ in ((Lc, Lt), (None, None)):
    mod, _ = _build(configs.qm8_gpnn(num_prop=3), 21)
    mod.train()
    _, loss = mod(nf, L, *ops_, label=label, mask=mask)
    loss.backward()
    grads.append({n: p.grad.clone() for n, p in mod.named_parameters()})
  for n in grads[0]:                          # the same operators: equal up to the order of atomic sums
    np.testing.assert_allclose(grads[1][n].cpu().numpy(), grads[0][n].cpu().numpy(), rtol=1e-5, atol=1e-10,
                               err_msg=n)


def test_graphed_step_with_device_partition_matches_eager():
  from lanczosnetwork_b200.train import GraphedStep
  cfg = configs.qm8_gpnn(num_prop=3)
  batches = []
  for i in range(3):
    bt = data.synthetic_qm8_batch(32, seed=60 + i)
    t = {k: _t(bt[k]).to(dev()) for k in ('node_feat', 'L', 'node_mask', 'label')}
    t['empty'] = torch.zeros((32, 0, 0), device=dev())
    batches.append(t)

  def make():
    m = GPNN(cfg)
    m.load_state_dict(deterministic_state_dict(m, 77))
    m = m.to(dev()).train()
    return m, torch.optim.SGD(m.parameters(), lr=1e-2, momentum=0.9)

  def call_args(bt):
    return (bt['node_feat'], bt['L'], bt['empty'], bt['empty']), {'label': bt['label'], 'mask': bt['node_mask']}

  eager, opt_e = make()
  losses_e = []
  for i in range(6):
    a, kw = call_args(batches[i % 3])
    opt_e.zero_grad()
    _, loss = eager(*a, **kw)
    loss.backward()
    opt_e.step()
    losses_e.append(float(loss.detach()))
  graphed, opt_g = make()
  step = GraphedStep(graphed, opt_g, *call_args(batches[0]))
  losses_g = []
  for i in range(6):
    a, kw = call_args(batches[i % 3])
    losses_g.append(float(step(*a, **kw)[1].detach()))
  np.testing.assert_allclose(losses_g, losses_e, rtol=1e-5)


def test_bench_batch_against_fp64_oracle_with_oracle_partitions():
  """B = 1024: the device-partition forward against the fp64 GPNN oracle fed the partition oracle's operators."""
  batch = data.synthetic_qm8_batch(1024, seed=5)
  cfg = configs.qm8_gpnn()
  mod, params = _build(cfg, 77)
  L0 = batch['L'][:, :, :, 0].astype(np.float64)
  labels, L_cluster, L_cut, status = ops.spectral_partition(_t(batch['L']).to(dev()), 3)
  st = status.cpu().numpy()
  keep = np.ones(len(st), bool)
  orc_labels = np.zeros(labels.shape, np.int64)
  lab = labels.cpu().numpy()
  for b in range(len(st)):
    r = partition_oracle.spectral_clustering(L0[b], 3)
    orc_labels[b] = r['labels']
    keep[b] = not r['tie'] and np.array_equal(r['labels'], lab[b])
  assert keep.sum() >= 1000, int(keep.sum())
  Lc, Lt = data.partition_operators(batch['L'][:, :, :, 0], orc_labels)
  t = {k: _t(batch[k]).to(dev()) for k in ('node_feat', 'L', 'node_mask')}
  with torch.no_grad():
    got = mod(t['node_feat'], t['L'], mask=t['node_mask'])
    s64 = gpnn_oracle.gpnn_forward(params, gpnn_oracle.make_spec(
        cfg.model.num_prop, cfg.model.num_prop_cluster, cfg.model.num_prop_cut, cfg.model.aggregate_type,
        cfg.model.update_func, cfg.dataset.num_bond_type), batch['node_feat'], t['L'], _t(Lc).to(dev()),
        _t(Lt).to(dev()), batch['node_mask'], dtype=torch.float64, device=dev())
  k = torch.from_numpy(keep).to(dev())
  np.testing.assert_allclose(got[k].cpu().numpy(), s64[k].cpu().numpy(), rtol=1e-4, atol=2e-5)


def test_data_parallel_scatters_empty_operators():
  """The collate's [B,0,0] operators under --device-partition pass nn.DataParallel's scatter as [b,0,0]."""
  g, gp = load_golden('lanczosnet_qm8.npz'), load_golden('gpnn_qm8.npz')
  nf, L, mask = _t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['node_mask']).to(dev())
  mod, _ = _build(configs.qm8_gpnn(), 3)
  empty = torch.zeros((L.shape[0], 0, 0), device=dev())
  with torch.no_grad():
    want = mod(nf, L, _t(gp['L_cluster']).to(dev()), _t(gp['L_cut']).to(dev()), mask=mask)
    dp = torch.nn.DataParallel(mod, device_ids=[0, 0])
    got = dp(nf, L, empty, empty, mask=mask)
  np.testing.assert_allclose(got.cpu().numpy(), want.cpu().numpy(), rtol=1e-5, atol=1e-6)
