"""LSTM GraphSAGE on the GPU: lnb_sage_lstm_step one step at a time against torch's LSTMCell in fp64 on the
same gathered inputs, its refusals, the module against the executed reference
(tests/golden/graphsage_lstm_qm8.npz) and the fp64 oracle at a larger batch, CUDA-graph replay, the
fallback, gradients and GraphedStep.  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import sage_lstm_oracle as lo
from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, data, ops
from lanczosnetwork_b200.model import LSTMGraphSAGE
from lanczosnetwork_b200.model.graph_sage import lstm_gate_matrix

pytestmark = pytest.mark.gpu

FWD_ATOL = 2e-5
FWD_RTOL = 1e-4
SMALL = dict(num_layer=3, hidden_dim=[32, 32, 32], output_dim=5)
# Floor of the one-step tolerance relative to the output's scale.  The 3xTF32 products drop the lo x lo
# term (relative 2^-22 per product) and the epilogue's expf / tanhf are a few ulp off the correctly
# rounded values, so at fan-ins of 64-256 the kernel's h and c are expected within ~1e-6 of fp64 at unit
# scale; 1e-5 leaves an order of magnitude above that without admitting a wrong gate or unit (those are
# off by O(1e-2) and more).
STEP_FLOOR = 1e-5


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _spec(cfg):
  return lo.make_spec(cfg.model.num_layer, cfg.model.agg_func, cfg.dataset.num_bond_type)


def _build(cfg, seed):
  mod = LSTMGraphSAGE(cfg)
  params = deterministic_state_dict(mod, seed)
  mod.load_state_dict(params)
  return mod.to(dev()).eval(), params


def random_samples(rng, B, N, K, E1):
  """Samples with repeats, empty channels (all ids 0), live nodes without neighbours, padded rows
  (nonempty = 0) and a few ids outside [0, N)."""
  nn_idx = np.zeros((B, N, K, E1), np.int64)
  nonempty = np.zeros((B, N), np.float32)
  for b in range(B):
    n = rng.randint(1, N + 1) if b else N
    for i in range(n):
      if rng.rand() < 0.1:
        continue
      nonempty[b, i] = 1
      for e in range(E1):
        if rng.rand() < 0.2:
          continue                                       # empty channel: node 0, K times
        nn_idx[b, i, :, e] = rng.randint(0, n, size=K)
  hit = rng.rand(*nn_idx.shape) < 0.02
  nn_idx[hit] = rng.choice([-1, N, N + 3], size=int(hit.sum()))
  return nn_idx, nonempty


STEP_CASES = [  # B, N, D, E1, K
    (3, 9, 32, 1, 1), (3, 9, 32, 7, 2), (2, 26, 64, 7, 40), (2, 26, 96, 1, 2),
    (4, 26, 128, 7, 2), (1, 200, 128, 1, 40), (2, 150, 64, 7, 2), (5, 13, 96, 7, 40),
]


@pytest.mark.parametrize('case', STEP_CASES, ids=['B%d-N%d-D%d-E%d-K%d' % c for c in STEP_CASES])
def test_each_step_matches_fp64_lstm_cell(case):
  B, N, D, E1, K = case
  rng = np.random.RandomState(sum(case))
  nn_idx, ne = random_samples(rng, B, N, K, E1)
  state = _t((rng.randn(B * N, D) * 3 / np.sqrt(D)).astype(np.float32)).to(dev())
  cell = torch.nn.LSTMCell(D, D).to(dev())
  with torch.no_grad():
    for p in cell.parameters():
      p.uniform_(-0.3, 0.3)
  W, b = lstm_gate_matrix(cell.weight_ih.detach(), cell.weight_hh.detach(), cell.bias_ih.detach(),
                          cell.bias_hh.detach())
  w_hi, w_lo = ops.split_tf32(W)
  idx = _t(nn_idx).to(dev()).to(torch.int32)
  nev = _t(ne.reshape(-1)).to(dev())
  R = B * N * E1
  live = nev.view(B * N, 1).expand(B * N, E1).reshape(R) != 0
  # the gathered inputs of every step, sequence s = (b*N + n)*E1 + e
  gid = _t(nn_idx).to(dev())
  ok = (gid >= 0) & (gid < N)
  gid = torch.where(ok, gid + N * torch.arange(B, device=dev()).view(B, 1, 1, 1), torch.zeros_like(gid))
  c = torch.empty((R, D), device=dev())
  h = torch.empty_like(c)
  spare = torch.empty_like(c)
  h_prev = c_prev = torch.zeros((R, D), device=dev(), dtype=torch.float64)
  for t in range(K):
    out = spare
    ops.sage_lstm_step(state, idx, nev, h if t else None, c, w_hi, w_lo, b, t, out)
    x = state[gid[:, :, t, :].reshape(-1)] * ok[:, :, t, :].reshape(-1, 1)
    want = {}
    for dt in (torch.float64, torch.float32):
      ref = torch.nn.LSTMCell(D, D).to(dev(), dt)
      ref.load_state_dict(cell.state_dict())
      with torch.no_grad():
        want[dt] = ref(x.to(dt), (h_prev.to(dt), c_prev.to(dt)))
    for got, k, what in ((out, 0, 'h'), (c, 1, 'c')):
      r64, r32 = want[torch.float64][k][live], want[torch.float32][k][live]
      g = got[live].double()
      scale = float(r64.abs().max())
      err, e32 = float((g - r64).abs().max()), float((r32.double() - r64).abs().max())
      assert torch.isfinite(g).all()
      assert err <= max(4 * e32, STEP_FLOOR * scale), (case, t, what, err, e32, scale)
    if t == K - 1:                                           # dead rows: a zero message
      assert torch.equal(out[~live], torch.zeros_like(out[~live]))
    # the next step starts from the kernel's own state: each step is checked on its own
    h_prev =torch.zeros((R, D), device=dev(), dtype=torch.float64).index_put_((live,), out[live].double())
    c_prev = torch.zeros((R, D), device=dev(), dtype=torch.float64).index_put_((live,), c[live].double())
    h, spare = spare, h


def test_step_refuses_shapes_outside_the_kernel_without_launching():
  B, N, K = 2, 5, 3

  def attempt(D, E1):
    state = torch.zeros((B * N, D), device=dev())
    idx = torch.zeros((B, N, K, E1), dtype=torch.int32, device=dev())
    ne = torch.ones(B * N, device=dev())
    c = torch.zeros((B * N * E1, D), device=dev())
    w = torch.zeros((4 * D, 2 * D), device=dev())
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match='status -2'):
      ops.sage_lstm_step(state, idx, ne, None, c, w, w, torch.zeros(4 * D, device=dev()), 0, torch.empty_like(c))
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
    assert not ops.sage_lstm_step_supported(D, E1, K)

  attempt(48, 7)
  attempt(160, 7)
  attempt(64, 17)
  assert ops.sage_lstm_step_supported(64, 7, 40) and ops.sage_lstm_step_supported(32, 1, 1)


# ------------------------------------------------------------------------------------------------
def test_model_matches_reference_golden():
  gg = load_golden('graphsage_lstm_qm8.npz')
  args = [_t(gg[k]).to(dev()) for k in ('node_feat', 'nn_idx', 'nonempty_mask')]
  mask = _t(gg['node_mask']).to(dev())
  seed = int(gg['weight_seed'])
  cases = [(configs.qm8_graphsage(agg_func='LSTM'), seed, 'score'),
           (configs.qm8_graphsage(agg_func='LSTM', **SMALL), seed + 1, 'small')]
  for cfg, s, key in cases:
    mod, params = _build(cfg, s)
    assert mod.lstm_supported(7)
    with torch.no_grad():
      if key == 'score':
        score, loss = mod(*args, label=_t(gg['label']).to(dev()), mask=mask)
        assert abs(float(loss) - float(gg['loss'])) <= 1e-4 * abs(float(gg['loss']))
      else:
        score = mod(*args, mask=mask)
      nomask = mod(*args)
    for got, k, m in ((score, key, gg['node_mask']), (nomask, key + '_nomask', None)):
      np.testing.assert_allclose(got.cpu().numpy(), gg[k], rtol=FWD_RTOL, atol=FWD_ATOL, err_msg=k)
      s64 = lo.sage_lstm_forward(params, _spec(cfg), *[gg[x] for x in ('node_feat', 'nn_idx', 'nonempty_mask')],
                                 m, dtype=torch.float64).numpy()
      e_ref = np.abs(gg[k] - s64).max()
      e_ours = np.abs(got.cpu().numpy() - s64).max()
      print('%s: reference %.3g, kernel %.3g from fp64' % (k, e_ref, e_ours))
      assert e_ours <= max(4 * e_ref, 5e-6), (k, e_ours, e_ref)


def test_bench_batch_against_fp64_oracle_and_graph_replay():
  bt = data.sage_collate(data.synthetic_qm8_samples(256, seed=5), 40, np.random.RandomState(0))
  cfg = configs.qm8_graphsage(agg_func='LSTM')
  mod, params = _build(cfg, 77)
  args = [_t(bt[k]).to(dev()) for k in ('node_feat', 'nn_idx', 'nonempty_mask')]
  mask = _t(bt['node_mask']).to(dev())
  with torch.no_grad():
    mod.use_cuda_graph = False
    eager = mod(*args, mask=mask)
    mod.use_cuda_graph = True
    replays = [mod(*args, mask=mask) for _ in range(3)]
  assert all(torch.equal(eager, r) for r in replays)
  assert mod.graph_stats()['captures'] >= 1
  inputs = [bt[k] for k in ('node_feat', 'nn_idx', 'nonempty_mask', 'node_mask')]
  with torch.no_grad():
    s64 = lo.sage_lstm_forward(params, _spec(cfg), *inputs, dtype=torch.float64, device=dev())
    s32 = lo.sage_lstm_forward(params, _spec(cfg), *inputs, device=dev())
  e_ours = float((eager.double() - s64).abs().max())
  e_orc = float((s32.double() - s64).abs().max())
  print('B=256: kernel %.3g, fp32 oracle %.3g from fp64 (scale %.3g)' % (e_ours, e_orc, float(s64.abs().max())))
  np.testing.assert_allclose(eager.cpu().numpy(), s64.cpu().numpy(), rtol=FWD_RTOL, atol=FWD_ATOL)
  assert e_ours <= max(4 * e_orc, 5e-6), (e_ours, e_orc)


def test_off_kernel_width_runs_the_fallback_and_matches_the_oracle():
  gg = load_golden('graphsage_lstm_qm8.npz')
  cfg = configs.qm8_graphsage(agg_func='LSTM', num_layer=3, hidden_dim=[48, 48, 48], output_dim=5)
  mod, params = _build(cfg, 11)
  assert not mod.lstm_supported(7)
  args = [_t(gg[k]).to(dev()) for k in ('node_feat', 'nn_idx', 'nonempty_mask')]
  n0 = ops.launch_count()
  for m in (gg['node_mask'], None):
    with torch.no_grad():
      got = mod(*args, mask=None if m is None else _t(m).to(dev()))
    s64 = lo.sage_lstm_forward(params, _spec(cfg), gg['node_feat'], gg['nn_idx'], gg['nonempty_mask'], m,
                               dtype=torch.float64)
    np.testing.assert_allclose(got.cpu().numpy(), s64.numpy(), rtol=FWD_RTOL, atol=FWD_ATOL)
  assert ops.launch_count() > n0                         # the library's kernels ran


def test_gradients_match_the_reference_digests_and_fp64_autograd():
  gg = load_golden('graphsage_lstm_qm8.npz')
  cfg = configs.qm8_graphsage(agg_func='LSTM')
  mod, params = _build(cfg, int(gg['weight_seed']))
  mod.train()
  args = [_t(gg[k]).to(dev()) for k in ('node_feat', 'nn_idx', 'nonempty_mask')]
  label, mask = _t(gg['label']).to(dev()), _t(gg['node_mask']).to(dev())
  _, loss = mod(*args, label=label, mask=mask)
  loss.backward()
  assert abs(float(loss.detach()) - float(gg['grad_loss'])) <= 1e-4 * float(gg['grad_loss'])
  p64 = {k: v.double().requires_grad_(True) for k, v in params.items()}
  s64 = lo.sage_lstm_forward(p64, _spec(cfg), gg['node_feat'], gg['nn_idx'], gg['nonempty_mask'], gg['node_mask'],
                             dtype=torch.float64, cast=False)
  F.mse_loss(s64, torch.from_numpy(gg['label']).double()).backward()
  for name, p in mod.named_parameters():
    ref = p64[name].grad
    if ref is None:                                     # filter[num_layer - 1]: never read
      assert p.grad is None or not p.grad.any(), name
      assert 'grad|' + name not in gg
      continue
    err = float((p.grad.detach().cpu().double() - ref).abs().max())
    assert err <= 2e-3 * float(ref.abs().max()) + 1e-12, (name, err, float(ref.abs().max()))
    want, got = gg['grad|' + name], lo.grad_digest({name: p.grad.cpu()})[name]
    scale = max(np.sqrt(want[1]), 1e-12)
    assert abs(got[1] - want[1]) <= 2e-3 * want[1] + 1e-12, (name, got[1], want[1])
    assert abs(got[0] - want[0]) <= 2e-3 * scale * np.sqrt(p.numel()), (name, got[0], want[0])
    np.testing.assert_allclose(got[2:], want[2:], rtol=1e-2, atol=2e-3 * scale, err_msg=name)


def test_graphed_step_matches_eager_steps():
  from lanczosnetwork_b200.train import GraphedStep
  cfg = configs.qm8_graphsage(agg_func='LSTM', **SMALL)
  batches = []
  for i in range(2):
    bt = data.sage_collate(data.synthetic_qm8_samples(16, seed=60 + i), 40, np.random.RandomState(i))
    bt['label'] = np.random.RandomState(i).randn(16, 5).astype(np.float32)
    batches.append({k: _t(v).to(dev()) for k, v in bt.items()})

  def make():
    m = LSTMGraphSAGE(cfg)
    m.load_state_dict(deterministic_state_dict(m, 77))
    m = m.to(dev()).train()
    return m, torch.optim.Adam(m.parameters(), lr=1e-3)

  def call_args(bt):
    return (bt['node_feat'], bt['nn_idx'], bt['nonempty_mask']), {'label': bt['label'], 'mask': bt['node_mask']}

  eager, opt_e = make()
  losses_e = []
  for i in range(4):                                    # the reference runner's loop
    a, kw = call_args(batches[i % 2])
    opt_e.zero_grad()
    _, loss = eager(*a, **kw)
    loss.backward()
    opt_e.step()
    losses_e.append(float(loss.detach()))
  graphed, opt_g = make()
  a, kw = call_args(batches[0])
  step = GraphedStep(graphed, opt_g, a, kw)
  losses_g = []
  for i in range(4):
    a, kw = call_args(batches[i % 2])
    _, loss = step(*a, **kw)
    losses_g.append(float(loss.detach()))
  np.testing.assert_allclose(losses_g, losses_e, rtol=1e-5)
  for (n, p), (_, q) in zip(graphed.named_parameters(), eager.named_parameters()):
    np.testing.assert_allclose(p.detach().cpu().numpy(), q.detach().cpu().numpy(), rtol=2e-4, atol=2e-6, err_msg=n)
  assert step.replays == 4
