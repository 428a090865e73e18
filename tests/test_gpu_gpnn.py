"""GPNN drop-in on the GPU: lnb_gpnn_partition_update across its envelope against fp64, the module against
the reference's outputs (tests/golden/gpnn_qm8.npz) and the fp64 oracle at the benchmark batch size,
unequal partition counts, CUDA-graph replay and its launch count, weight updates, the training path,
GraphedStep and nn.DataParallel.  ``pytest -m gpu``."""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, data, ops
from lanczosnetwork_b200.model import GPNN
from lanczosnetwork_b200.model.ggnn import gru_gate_matrix
from oracle import gpnn_oracle

pytestmark = pytest.mark.gpu

FWD_ATOL = 2e-5
FWD_RTOL = 1e-4
EPS = float(np.finfo(np.float32).eps)
SMALL = dict(hidden_dim=32, num_prop=3, num_prop_cluster=2, num_prop_cut=1, aggregate_type='sum',
             update_func='RNN', output_dim=16)
# floor of the kernel bound, in units of the output scale: 3xTF32 products over a fan-in of 2H <= 256
KERNEL_FLOOR = 8e-6


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _spec(cfg):
  m = cfg.model
  return gpnn_oracle.make_spec(m.num_prop, m.num_prop_cluster, m.num_prop_cut, m.aggregate_type, m.update_func,
                               cfg.dataset.num_bond_type)


def _build(cfg, seed):
  mod = GPNN(cfg)
  params = deterministic_state_dict(mod, seed)
  mod.load_state_dict(params)
  return mod.to(dev()).eval(), params


def _batch(B, seed):
  """A synthetic QM8 batch with partitions from seeded labels (numpy arrays)."""
  b = data.synthetic_qm8_batch(B, seed=seed)
  lab = data.random_partition_labels(np.random.RandomState(seed), B, b['L'].shape[1])
  b['L_cluster'], b['L_cut'] = data.partition_operators(b['L'][:, :, :, 0], lab)
  return b


# ------------------------------------------------------------------------------------------------
def partition_reference(M, h, P, w_ih, w_hh, b_ih, b_hh, avg, dtype):
  """The formula of one part of lnb_gpnn_partition_update in plain torch at ``dtype``: torch's GRUCell of
  P M with the valued operator P [B,N,N] (row-normalised by rowsum + eps for avg)."""
  B, N = P.shape[0], P.shape[1]
  H = h.shape[1]
  P = P.to(dtype)
  if avg:
    P = P / (P.sum(dim=2, keepdim=True) + EPS)
  agg = torch.bmm(P, M.to(dtype).view(B, N, H)).reshape(B * N, H)
  cell = torch.nn.GRUCell(H, H).to(device=M.device, dtype=dtype)
  with torch.no_grad():
    for dst, src in ((cell.weight_ih, w_ih), (cell.weight_hh, w_hh), (cell.bias_ih, b_ih), (cell.bias_hh, b_hh)):
      dst.copy_(src.to(dtype))
    return cell(agg, h.to(dtype))


def _operators(gen, B, N):
  """Positive-valued operators [B,N,N,2]: random sparse rows, a row without entries, and trailing
  'padded' rows that hold only a unit self-loop (as the L4 partition operators of padded nodes do)."""
  P = (torch.rand(B, N, N, 2, generator=gen) < 0.3).float() * (0.05 + torch.rand(B, N, N, 2, generator=gen))
  if N >= 4:
    P[:, N // 2] = 0.0                                    # an empty row in both operators
    pad = max(1, N // 5)
    P[:, N - pad:] = 0.0
    P[:, :, N - pad:] = 0.0
    idx = torch.arange(N - pad, N)
    P[:, idx, idx] = 1.0
  return P


def _weights(gen, H):
  r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
  w_ih = (r(3 * H, H) / np.sqrt(H)).float()
  w_hh = (r(3 * H, H) / np.sqrt(H)).float()
  b_ih, b_hh = (0.1 * r(3 * H)).float(), (0.1 * r(3 * H)).float()
  return [t.to(dev()) for t in (w_ih, w_hh, b_ih, b_hh)]


def _gates(w_ih, w_hh, b_ih, b_hh):
  W, b = gru_gate_matrix(w_ih, w_hh, b_ih, b_hh)
  w_hi, w_lo = ops.split_tf32(W)
  return w_hi, w_lo, b


SWEEP = list(itertools.product([1, 26, 128, 255], [32, 64, 96, 128]))


def _check(got, ref64, ref32, what):
  scale = max(1.0, float(ref64.abs().max()))
  e_ours = float((got.cpu().double() - ref64).abs().max())
  e_orc = float((ref32.double() - ref64).abs().max())
  bound = max(8 * e_orc, KERNEL_FLOOR * scale)
  assert e_ours <= bound, (what, e_ours, e_orc)
  return e_ours / bound


def test_partition_kernel_against_fp64_across_the_envelope():
  """Both parts in one launch with distinct M / h, written into column blocks 1 and 2 of a [B*N, 3H]
  buffer with the h copy in block 0; repeated launches are bit-identical."""
  gen = torch.Generator().manual_seed(0)
  worst = 0.0
  for N, H in SWEEP:
    B = 3                                                 # B*N not a multiple of 128 (except N = 128)
    P = _operators(gen, B, N).to(dev())
    prep = ops.graph_prepare(P, torch.zeros((B, N, 4), device=dev()))
    M = [torch.randn(B * N, H, generator=gen).to(dev()) for _ in range(2)]
    h = [(0.5 * torch.randn(B * N, H, generator=gen)).to(dev()) for _ in range(2)]
    wts = _weights(gen, H)
    gates = _gates(*wts)
    cpu_w = [t.cpu() for t in wts]
    for avg in (False, True):
      X = torch.full((B * N, 3 * H), float('nan'), device=dev())
      parts = [(M[p], h[p], X[:, (p + 1) * H:(p + 2) * H]) for p in (0, 1)]
      ops.gpnn_partition_update(parts, prep, *gates, avg, h_copy=X[:, :H])
      assert torch.equal(X[:, :H], h[0])                  # the h copy of the first part
      for p in (0, 1):
        args = (M[p].cpu(), h[p].cpu(), P[..., p].cpu(), *cpu_w, avg)
        worst = max(worst, _check(X[:, (p + 1) * H:(p + 2) * H], partition_reference(*args, torch.float64),
                                  partition_reference(*args, torch.float32), (N, H, avg, p)))
      X2 = torch.empty_like(X)
      parts2 = [(M[p], h[p], X2[:, (p + 1) * H:(p + 2) * H]) for p in (0, 1)]
      ops.gpnn_partition_update(parts2, prep, *gates, avg, h_copy=X2[:, :H])
      assert torch.equal(X, X2)                           # fixed order: bit-identical
  print('worst error / bound %.3g over %d cases' % (worst, 4 * len(SWEEP)))


@pytest.mark.parametrize('mode', ['shared', 'cluster-only', 'cut-only', 'contiguous'])
def test_partition_kernel_part_selection_and_aliasing(mode):
  """Aliased M / h between the parts (iteration 0 of the model), one-part launches (the extra iterations
  of the longer chain, strided h) and plain contiguous outputs without an h copy."""
  gen = torch.Generator().manual_seed(1)
  B, N, H = 5, 26, 128
  P = _operators(gen, B, N).to(dev())
  prep = ops.graph_prepare(P, torch.zeros((B, N, 4), device=dev()))
  wts = _weights(gen, H)
  gates = _gates(*wts)
  cpu_w = [t.cpu() for t in wts]
  M = torch.randn(B * N, H, generator=gen).to(dev())
  src = torch.randn(B * N, 3 * H, generator=gen).to(dev())
  h = src[:, :H].contiguous() if mode in ('shared', 'contiguous') else src[:, H:2 * H]   # strided h
  X = torch.full((B * N, 3 * H), float('nan'), device=dev())
  outs = [X[:, H:2 * H], X[:, 2 * H:]]
  if mode == 'contiguous':
    outs = [torch.empty(B * N, H, device=dev()) for _ in range(2)]
  active = {'shared': (0, 1), 'contiguous': (0, 1), 'cluster-only': (0,), 'cut-only': (1,)}[mode]
  parts = [(M, h, outs[p]) if p in active else None for p in (0, 1)]
  for avg in (True, False):
    ops.gpnn_partition_update(parts, prep, *gates, avg, h_copy=None)
    for p in (0, 1):
      if p in active:
        args = (M.cpu(), h.cpu(), P[..., p].cpu(), *cpu_w, avg)
        _check(outs[p], partition_reference(*args, torch.float64), partition_reference(*args, torch.float32),
               (mode, avg, p))
      elif mode != 'contiguous':
        assert torch.isnan(outs[p]).all()                 # a skipped part writes nothing
  assert torch.isnan(X[:, :H]).all()                      # no h copy asked for


def test_partition_kernel_refusals_launch_nothing():
  B, N, H = 2, 8, 32
  prep = tuple(t.to(dev()) for t in (torch.zeros((B, 2, N, N)), torch.zeros((B, 2, N, N), dtype=torch.uint8),
                                      torch.zeros((B, 2), dtype=torch.int32)))
  W = torch.zeros((4 * H, 2 * H), device=dev())
  b = torch.zeros((4 * H,), device=dev())
  buf = torch.zeros((B * N, 4 * H), device=dev())
  M, h = buf[:, :H], buf[:, H:2 * H]
  bad = [
      ('out aliases h', [(M, h, h), None], None),
      ('out overlaps the other part\'s h', [(M, h, buf[:, 2 * H:3 * H]), (M, buf[:, 2 * H:3 * H], buf[:, 3 * H:])], None),
      ('unaligned column offset', [(M, h, buf[:, 2 * H + 1:3 * H + 1]), None], None),
      ('h_copy over an output', [(M, h, buf[:, 2 * H:3 * H]), None], buf[:, 2 * H:3 * H]),
  ]
  for what, parts, h_copy in bad:
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match='status -2'):
      ops.gpnn_partition_update(parts, prep, W, W, b, True, h_copy=h_copy)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0, what
  for N2, H2 in ((256, 32), (8, 48), (8, 160), (8, 16)):
    prep2 = tuple(t.to(dev()) for t in (torch.zeros((B, 2, N2, N2)), torch.zeros((B, 2, N2, N2), dtype=torch.uint8),
                                         torch.zeros((B, 2), dtype=torch.int32)))
    W2 = torch.zeros((4 * H2, 2 * H2), device=dev())
    x = torch.zeros((B * N2, H2), device=dev())
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match='status -2'):
      ops.gpnn_partition_update([(x, x, torch.zeros_like(x)), None], prep2, W2, W2, torch.zeros(4 * H2, device=dev()), True)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
    assert not ops.gpnn_partition_update_supported(N2, H2)


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prefix,over,dseed', [('config', {}, 0), ('small', SMALL, 1)], ids=['config', 'small'])
def test_model_matches_reference_golden(prefix, over, dseed):
  g, gp = load_golden('lanczosnet_qm8.npz'), load_golden('gpnn_qm8.npz')
  nf, L, mask = _t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['node_mask']).to(dev())
  Lc, Lt = _t(gp['L_cluster']).to(dev()), _t(gp['L_cut']).to(dev())
  cfg = configs.qm8_gpnn(**over)
  mod, params = _build(cfg, int(gp['weight_seed']) + dseed)
  assert mod.fused_supported(26, 7) == (prefix == 'config')
  with torch.no_grad():
    score, loss = mod(nf, L, Lc, Lt, label=_t(g['label']).to(dev()), mask=mask)
    nomask = mod(nf, L, Lc, Lt)
  for got, key, m in ((score, '%s_score' % prefix, g['node_mask']), (nomask, '%s_score_nomask' % prefix, None)):
    np.testing.assert_allclose(got.cpu().numpy(), gp[key], rtol=FWD_RTOL, atol=FWD_ATOL, err_msg=key)
    s64 = gpnn_oracle.gpnn_forward(params, _spec(cfg), g['node_feat'], g['L'], gp['L_cluster'], gp['L_cut'], m,
                                   dtype=torch.float64).numpy()
    e_ref = np.abs(gp[key] - s64).max()
    e_ours = np.abs(got.cpu().numpy() - s64).max()
    assert e_ours <= max(4 * e_ref, 5e-6), (key, e_ours, e_ref)
  want = float(gp['%s_loss' % prefix])
  assert abs(float(loss) - want) <= 1e-4 * abs(want)


def _against_oracle(cfg, batch, seed):
  mod, params = _build(cfg, seed)
  t = {k: _t(batch[k]).to(dev()) for k in ('node_feat', 'L', 'L_cluster', 'L_cut', 'node_mask')}
  before = {k: v.clone() for k, v in t.items()}
  assert mod.fused_supported(t['L'].shape[1], t['L'].shape[3])
  with torch.no_grad():
    mod.use_cuda_graph = False
    eager = mod(t['node_feat'], t['L'], t['L_cluster'], t['L_cut'], mask=t['node_mask'])
    s64 = gpnn_oracle.gpnn_forward(params, _spec(cfg), batch['node_feat'], t['L'], t['L_cluster'], t['L_cut'],
                                   batch['node_mask'], dtype=torch.float64, device=dev())
    s32 = gpnn_oracle.gpnn_forward(params, _spec(cfg), batch['node_feat'], t['L'], t['L_cluster'], t['L_cut'],
                                   batch['node_mask'], device=dev())
  e_ours = float((eager.double() - s64).abs().max())
  e_orc = float((s32.double() - s64).abs().max())
  np.testing.assert_allclose(eager.cpu().numpy(), s64.cpu().numpy(), rtol=FWD_RTOL, atol=FWD_ATOL)
  assert e_ours <= max(4 * e_orc, 5e-6), (e_ours, e_orc)
  for k, v in t.items():
    assert torch.equal(v, before[k]), k                   # the caller's operators are not modified
  return mod, t, eager


@pytest.mark.parametrize('over', [dict(num_prop_cluster=2, num_prop_cut=0), dict(num_prop_cluster=0, num_prop_cut=3),
                                  dict(num_prop_cluster=2, num_prop_cut=3), dict(aggregate_type='sum'),
                                  dict(hidden_dim=64)],
                         ids=['2-0', '0-3', '2-3', 'sum', 'H64'])
def test_variants_against_fp64_oracle(over):
  cfg = configs.qm8_gpnn(**dict(dict(num_prop=3), **over))
  _against_oracle(cfg, _batch(1024, seed=6), 31)


def test_bench_batch_against_fp64_oracle_graph_replay_launches_and_updates():
  batch = _batch(1024, seed=5)
  cfg = configs.qm8_gpnn()
  mod, t, eager = _against_oracle(cfg, batch, 77)
  args = (t['node_feat'], t['L'], t['L_cluster'], t['L_cut'])
  with torch.no_grad():
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    mod(*args, mask=t['node_mask'])
    torch.cuda.synchronize()
    # 8 launches per step; the embedding, input_func, two graph_prepare (two kernels each) and the readout
    assert ops.launch_count() - n0 == 8 * cfg.model.num_prop + 7
    mod.use_cuda_graph = True
    replays = [mod(*args, mask=t['node_mask']) for _ in range(3)]
  assert all(torch.equal(eager, r) for r in replays)
  assert mod.graph_stats()['captures'] >= 1
  # an optimizer step updates the parameters in place: the captured graph and weight caches follow.  The
  # state_func MLP is unbounded, so the shift is kept small enough that the scores stay O(1).
  opt = torch.optim.SGD(mod.parameters(), lr=0.05)
  for p in mod.parameters():
    p.grad = torch.full_like(p, 0.01)
  with torch.no_grad():
    opt.step()
    updated = mod(*args, mask=t['node_mask'])
    mod.use_cuda_graph = False
    updated_eager = mod(*args, mask=t['node_mask'])
  assert not torch.equal(updated, eager) and torch.equal(updated, updated_eager)
  new_params = {k: v.detach() for k, v in mod.state_dict().items()}
  oargs = (new_params, _spec(cfg), batch['node_feat'], t['L'], t['L_cluster'], t['L_cut'], batch['node_mask'])
  with torch.no_grad():
    u64 = gpnn_oracle.gpnn_forward(*oargs, dtype=torch.float64, device=dev())
    u32 = gpnn_oracle.gpnn_forward(*oargs, device=dev())
  scale = max(1.0, float(u64.abs().max()))
  e_ours = float((updated.double() - u64).abs().max())
  e_orc = float((u32.double() - u64).abs().max())
  assert e_ours <= max(4 * e_orc, 5e-6 * scale), (e_ours, e_orc, scale)
  for k in ('L', 'L_cluster', 'L_cut'):
    assert torch.equal(t[k], _t(batch[k]).to(dev())), k


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prefix,over', [('config', dict(num_prop=4)), ('small', SMALL)], ids=['config', 'small'])
def test_gradients_match_fp64_oracle_autograd(prefix, over):
  g, gp = load_golden('lanczosnet_qm8.npz'), load_golden('gpnn_qm8.npz')
  cfg = configs.qm8_gpnn(**over)
  mod, params = _build(cfg, 21)
  nf, L = _t(g['node_feat']).to(dev()), _t(g['L']).to(dev())
  Lc, Lt = _t(gp['L_cluster']).to(dev()), _t(gp['L_cut']).to(dev())
  label, mask = _t(g['label']).to(dev()), _t(g['node_mask']).to(dev())
  with torch.no_grad():
    inference = mod(nf, L, Lc, Lt, mask=mask)
  mod.train()
  score, loss = mod(nf, L, Lc, Lt, label=label, mask=mask)
  loss.backward()
  np.testing.assert_allclose(score.detach().cpu().numpy(), inference.cpu().numpy(), rtol=FWD_RTOL, atol=FWD_ATOL)
  p64 = {k: v.double().requires_grad_(True) for k, v in params.items()}
  s64 = gpnn_oracle.gpnn_forward(p64, _spec(cfg), g['node_feat'], g['L'], gp['L_cluster'], gp['L_cut'],
                                 g['node_mask'], dtype=torch.float64, cast=False)
  l64 = F.mse_loss(s64, torch.from_numpy(g['label']).double())
  l64.backward()
  assert abs(float(loss.detach()) - float(l64.detach())) <= 1e-4 * float(l64.detach())
  for name, p in mod.named_parameters():
    ref = p64[name].grad
    err = float((p.grad.detach().cpu().double() - ref).abs().max())
    assert err <= 2e-3 * float(ref.abs().max()) + 1e-12, (name, err, float(ref.abs().max()))


def test_reference_training_loop_body_runs_and_learns():
  """The loop body of QM8Runner.train (runner/qm8_runner.py:226-259) through nn.DataParallel with Adam:
  the loss goes down and the inference forward picks up the trained weights."""
  batch = _batch(64, seed=4)
  model = GPNN(configs.qm8_gpnn())
  model.load_state_dict(deterministic_state_dict(model, 1234))
  model = torch.nn.DataParallel(model, device_ids=[0]).cuda()
  optimizer = torch.optim.Adam(filter(lambda p: p.requires_grad, model.parameters()), lr=1.0e-3)
  t = {k: _t(v).cuda() for k, v in batch.items() if k in ('node_feat', 'L', 'L_cluster', 'L_cut', 'label', 'node_mask')}
  args = (t['node_feat'], t['L'], t['L_cluster'], t['L_cut'])
  model.eval()
  with torch.no_grad():
    before = model(*args, label=t['label'], mask=t['node_mask'])[1]
  losses = []
  for _ in range(25):
    model.train()
    optimizer.zero_grad()
    _, train_loss = model(*args, label=t['label'], mask=t['node_mask'])
    train_loss.backward()
    optimizer.step()
    losses.append(float(train_loss))
  assert abs(losses[0] - float(before)) <= 1e-4 * max(1.0, float(before))
  assert max(losses[-3:]) < 0.985 * losses[0], losses
  model.eval()
  with torch.no_grad():
    after = model(*args, label=t['label'], mask=t['node_mask'])[1]
  assert float(after) < losses[0]


@pytest.mark.parametrize('over', [{}, SMALL], ids=['gru-avg', 'rnn-sum'])
def test_graphed_step_matches_eager_steps(over):
  from lanczosnetwork_b200.train import GraphedStep
  cfg = configs.qm8_gpnn(**dict(dict(num_prop=3), **over))
  batches = []
  for i in range(3):
    bt = _batch(32, seed=50 + i)
    batches.append({k: _t(bt[k]).to(dev()) for k in ('node_feat', 'L', 'L_cluster', 'L_cut', 'node_mask', 'label')})

  def make():
    m = GPNN(cfg)
    m.load_state_dict(deterministic_state_dict(m, 77))
    m = m.to(dev()).train()
    return m, torch.optim.SGD(m.parameters(), lr=1e-2, momentum=0.9)

  def call_args(bt):
    return (bt['node_feat'], bt['L'], bt['L_cluster'], bt['L_cut']), {'label': bt['label'], 'mask': bt['node_mask']}

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
  a, kw = call_args(batches[0])
  step = GraphedStep(graphed, opt_g, a, kw)
  for (n, p), (_, q) in zip(graphed.named_parameters(), make()[0].named_parameters()):
    assert torch.equal(p, q), n
  losses_g = []
  for i in range(6):
    a, kw = call_args(batches[i % 3])
    _, loss = step(*a, **kw)
    losses_g.append(float(loss.detach()))
  np.testing.assert_allclose(losses_g, losses_e, rtol=1e-5)
  for (n, p), (_, q) in zip(graphed.named_parameters(), eager.named_parameters()):
    np.testing.assert_allclose(p.detach().cpu().numpy(), q.detach().cpu().numpy(), rtol=2e-4, atol=2e-6, err_msg=n)
  assert step.replays == 6


def test_data_parallel_two_replicas_on_one_gpu():
  g, gp = load_golden('lanczosnet_qm8.npz'), load_golden('gpnn_qm8.npz')
  mod, _ = _build(configs.qm8_gpnn(), 3)
  nf, L, mask = _t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['node_mask']).to(dev())
  Lc, Lt = _t(gp['L_cluster']).to(dev()), _t(gp['L_cut']).to(dev())
  label = _t(g['label']).to(dev())
  with torch.no_grad():
    ref = mod(nf, L, Lc, Lt, mask=mask)
    dp = torch.nn.DataParallel(mod, device_ids=[0, 0]).eval()
    score, loss = dp(nf, L, Lc, Lt, label=label, mask=mask)
  assert loss.numel() == 2
  torch.testing.assert_close(score, ref, rtol=1e-5, atol=1e-6)
  dp.train()
  _, loss = dp(nf, L, Lc, Lt, label=label, mask=mask)
  loss.mean().backward()
  assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in mod.parameters())
  assert mod.update_func_partition.weight_ih.grad.abs().sum() > 0
