"""GraphSAGE drop-in on the GPU: lnb_sage_operators against a host construction, the GraphSAGE variant of
the stack kernel across its shapes against an fp64 torch restatement, refusals, neighbour_max, the module
against the reference's outputs (tests/golden/graphsage_qm8.npz) and the fp64 oracle at the benchmark
batch size, gradients, CUDA-graph replay, GraphedStep and nn.DataParallel.  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, data, ops
from lanczosnetwork_b200.model import GraphSAGE
from oracle import sage_oracle

pytestmark = pytest.mark.gpu

FWD_ATOL = 2e-5
FWD_RTOL = 1e-4
EPS = sage_oracle.EPS
SMALL = dict(num_layer=3, hidden_dim=[32, 32, 32], output_dim=5)


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _spec(cfg):
  return sage_oracle.make_spec(cfg.model.num_layer, cfg.model.agg_func, cfg.dataset.num_bond_type)


def _build(cfg, seed):
  mod = GraphSAGE(cfg)
  params = deterministic_state_dict(mod, seed)
  mod.load_state_dict(params)
  return mod.to(dev()).eval(), params


def host_operators(nn_idx, nonempty):
  """M[b, n, m, e] = nonempty * count / K in fp32 (one rounding of count / K), ids outside [0, N) dropped."""
  B, N, K, E1 = nn_idx.shape
  cnt = np.zeros((B, N, N, E1), np.int64)
  b, n, k, e = np.meshgrid(np.arange(B), np.arange(N), np.arange(K), np.arange(E1), indexing='ij')
  m = nn_idx
  ok = (m >= 0) & (m < N) & (nonempty.reshape(B, N, 1, 1) != 0)
  np.add.at(cnt, (b[ok], n[ok], m[ok], e[ok]), 1)
  return cnt.astype(np.float32) / np.float32(K)


def random_samples(rng, B, N, K, E1, oob=True):
  """Neighbour samples with repeats, empty channels (nn_idx 0: the node-0 quirk), nonempty = 0 real
  rows, padded rows and (optionally) ids outside [0, N)."""
  sizes = rng.randint(1, N + 1, size=B)
  sizes[0] = N
  nn_idx = np.zeros((B, N, K, E1), np.int64)
  nonempty = np.zeros((B, N, 1), np.float32)
  for b in range(B):
    n = sizes[b]
    for i in range(n):
      if rng.rand() < 0.1:
        continue                                       # real node without any neighbour
      nonempty[b, i] = 1
      for e in range(E1):
        if rng.rand() < 0.2:
          continue                                     # empty channel: aggregates node 0
        pool = rng.choice(n, size=min(n, rng.randint(1, 5)), replace=False)
        nn_idx[b, i, :, e] = rng.choice(pool, size=K, replace=True)
  if oob:
    hit = rng.rand(*nn_idx.shape) < 0.03
    nn_idx[hit] = rng.choice([-1, N, N + 7, -5], size=int(hit.sum()))
  return sizes, nn_idx, nonempty


# ------------------------------------------------------------------------------------------------
def test_sage_operators_are_bit_identical_to_the_host_construction():
  rng = np.random.RandomState(0)
  for (B, N, K, E1) in ((3, 1, 1, 1), (5, 7, 40, 7), (4, 26, 40, 7), (2, 128, 13, 16), (2, 200, 5, 3)):
    sizes, nn_idx, ne = random_samples(rng, B, N, K, E1)
    got = ops.sage_operators(_t(nn_idx).to(dev()), _t(ne).to(dev())).cpu().numpy()
    want = host_operators(nn_idx, ne)
    assert got.shape == (B, N, N, E1)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (B, N, K, E1)
  # the node-0 quirk: a live node whose channel list is empty takes node 0 with weight 1
  nn_idx = np.zeros((1, 3, 4, 2), np.int64)
  nn_idx[0, 1, :, 0] = [2, 2, 1, 2]
  ne = np.array([[[1], [1], [0]]], np.float32)
  got = ops.sage_operators(_t(nn_idx).to(dev()), _t(ne).to(dev())).cpu().numpy()
  assert got[0, 1, :, 0].tolist() == [0.0, 0.25, 0.75] and got[0, 1, :, 1].tolist() == [1.0, 0.0, 0.0]
  assert got[0, 0, :, 1].tolist() == [1.0, 0.0, 0.0] and not got[0, 2].any()


# ------------------------------------------------------------------------------------------------
def restate(M, ids, emb, Ws, bs, head, att, mask, agg, dtype):
  """The GraphSAGE stack in operator form, plain torch: per layer messages of every channel (M_e X, or
  the max over the entries of row n with M_e != 0, 0 for an empty row), Linear + ReLU, row / (norm + eps);
  then the gated masked-mean readout.  Returns (state, score)."""
  M = M.to(dtype)
  X = emb.to(dtype)[ids]
  B, N, _, E1 = M.shape
  for W, b in zip(Ws, bs):
    if agg == 'Max':
      msgs = []
      for e in range(E1):
        live = (M[:, :, :, e] != 0).unsqueeze(3)                                 # [B, n, m, 1]
        v = torch.where(live, X.unsqueeze(1), torch.tensor(float('-inf'), dtype=dtype, device=X.device))
        mx = v.max(dim=2).values
        msgs.append(torch.where(live.any(dim=2), mx, torch.zeros_like(mx)))
      msg = torch.cat(msgs, dim=2)
    else:
      msg = torch.cat([torch.bmm(M[:, :, :, e], X) for e in range(E1)], dim=2)
    y = F.relu(F.linear(msg, W.to(dtype), b.to(dtype)))
    X = y / (torch.norm(y, 2, dim=2, keepdim=True) + EPS)
  Wo, bo, wa, ba = [t.to(dtype) for t in (head.weight, head.bias, att.weight, att.bias)]
  yv = F.linear(X, Wo, bo) * torch.sigmoid(F.linear(X, wa, ba))
  if mask is None:
    return X, yv.mean(dim=1)
  m = (mask != 0).to(dtype).unsqueeze(2)
  return X, (yv * m).sum(dim=1) / m.sum(dim=1)


CASES = [  # N, Din0, H, layers, E1, agg, mask
    (1, 32, 32, 1, 1, 'Mean', False),
    (2, 64, 32, 2, 7, 'Max', True),
    (7, 128, 128, 3, 16, 'Mean', True),
    (7, 32, 32, 5, 16, 'Max', False),
    (26, 64, 128, 6, 7, 'Mean', True),
    (26, 64, 128, 6, 7, 'Max', False),
    (64, 32, 128, 8, 7, 'Max', True),
    (64, 128, 32, 7, 1, 'Mean', False),
    (128, 128, 32, 4, 16, 'Mean', False),
    (128, 64, 128, 2, 1, 'Max', True),
]


def _stack_case(N, Din0, H, layers, E1, agg, use_mask, seed, bias0=None):
  rng = np.random.RandomState(seed)
  B, K, P = (3 if N >= 64 else 6), 8, 5
  sizes, nn_idx, ne = random_samples(rng, B, N, K, E1)
  ids = _t(rng.randint(0, 70, size=(B, N))).to(dev())
  emb = _t(rng.randn(70, Din0).astype(np.float32)).to(dev())
  dins = [Din0] + [H] * (layers - 1)
  Ws = [_t(rng.uniform(-1, 1, size=(H, E1 * d)).astype(np.float32) * np.sqrt(6.0 / (H + E1 * d))).to(dev())
        for d in dins]
  bs = [_t(rng.uniform(-0.1, 0.1, size=H).astype(np.float32)).to(dev()) for _ in dins]
  if bias0 is not None:
    bs[0] = torch.full_like(bs[0], bias0)
  head, att = torch.nn.Linear(H, P).to(dev()), torch.nn.Linear(H, 1).to(dev())
  mask = _t((np.arange(N)[None, :] < sizes[:, None]).astype(np.uint8)).to(dev()) if use_mask else None
  M = ops.sage_operators(_t(nn_idx).to(dev()), _t(ne).to(dev()))
  V = torch.zeros((B, N, 4), device=dev())
  prep = ops.graph_prepare(M, V)
  kw = E1 * max(dins)
  w_hi, w_lo = ops.split_tf32(torch.cat([F.pad(W, (0, kw - W.shape[1])) for W in Ws]).contiguous())
  with torch.no_grad():
    state, score = ops.spectral_stack_forward(
        prep, V, w_hi, w_lo, torch.cat(bs), dins, H, 0, node_ids=ids, emb=emb, want_state=True,
        write_pad=True, readout=(head.weight, head.bias, att.weight.reshape(-1), att.bias), mask=mask, sage=agg)
    s64, c64 = restate(M, ids, emb, Ws, bs, head, att, mask, agg, torch.float64)
    s32, c32 = restate(M, ids, emb, Ws, bs, head, att, mask, agg, torch.float32)
  return state, score, (s64, c64), (s32, c32)


# Floor of the tolerance relative to the output's scale, per layer: the stack's 3xTF32 products drop the
# lo x lo term, so at fan-ins of 1-2 k the kernel lands further from fp64 than a plain fp32 restatement
# does; the same floor as the plain stack's envelope (tests/test_gpu_conv_envelope.py).
STACK_FLOOR_PER_LAYER = 8e-6


@pytest.mark.parametrize('case', CASES, ids=['N%d-D%d-H%d-L%d-E%d-%s-%s' % (c[:6] + ('mask' if c[6] else 'nomask',))
                                             for c in CASES])
def test_sage_stack_matches_fp64_restatement(case):
  state, score, (s64, c64), (s32, c32) = _stack_case(*case, seed=sum(case[:5]))
  assert torch.isfinite(state).all() and torch.isfinite(score).all()
  for got, ref, r32, what in ((state, s64, s32, 'state'), (score, c64, c32, 'score')):
    scale = float(ref.abs().max())
    err = float((got.double() - ref).abs().max())
    e32 = float((r32.double() - ref).abs().max())
    print('%s %s: max err %.3g (fp32 %.3g) at scale %.3g' % (case, what, err, e32, scale))
    assert err <= max(4 * e32, STACK_FLOOR_PER_LAYER * case[3] * scale), (case, what, err, e32, scale)


def test_sage_stack_all_zero_relu_rows_stay_zero():
  # one layer, bias far below every pre-activation: every row's ReLU output is 0, its norm is 0
  state, score, (s64, c64), _ = _stack_case(26, 64, 128, 1, 7, 'Mean', False, seed=3, bias0=-1e3)
  assert torch.equal(state, torch.zeros_like(state))
  torch.testing.assert_close(score.double(), c64, rtol=1e-6, atol=1e-7)
  # two layers (Max): layer 1 sees zero messages everywhere, so every row, real or padded, is the padded
  # constant relu(b) / (||relu(b)|| + eps) -- the same bits
  state, _, (s64, _), _ = _stack_case(26, 64, 128, 2, 7, 'Max', True, seed=4, bias0=-1e3)
  flat = state.reshape(-1, state.shape[2])
  assert torch.equal(flat, flat[:1].expand_as(flat))
  torch.testing.assert_close(state.double(), s64, rtol=1e-6, atol=1e-7)


def test_sage_stack_refuses_shapes_outside_the_kernel_without_launching():
  rng = np.random.RandomState(1)

  def attempt(N, Din0, H, S=0, E1=7, B=2):
    _, nn_idx, ne = random_samples(rng, B, N, 4, E1)
    M = ops.sage_operators(_t(nn_idx).to(dev()), _t(ne).to(dev()))
    V = torch.zeros((B, N, 4), device=dev())
    prep = ops.graph_prepare(M, V)
    w = torch.zeros((H, (E1 + S) * Din0), device=dev())
    coeff = torch.zeros((B, 4, S), device=dev()) if S else None
    ids = torch.zeros((B, N), dtype=torch.long, device=dev())
    emb = torch.zeros((70, Din0), device=dev())
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match='status -2'):
      ops.spectral_stack_forward(prep, V, w, w, torch.zeros(H, device=dev()), [Din0], H, S, coeff=coeff,
                                 node_ids=ids, emb=emb, want_state=True, sage='Max')
    torch.cuda.synchronize()
    assert ops.launch_count() == n0

  attempt(26, 64, 128, S=1)          # long scales
  attempt(130, 64, 128)              # N > 128
  attempt(26, 64, 132)               # H > 128
  attempt(26, 48, 128)               # Din % 32
  attempt(26, 4, 32)                 # Din < 32


# ------------------------------------------------------------------------------------------------
def test_neighbour_max_forward_argmax_and_backward():
  from lanczosnetwork_b200.train import neighbour_max
  rng = np.random.RandomState(2)
  B, N, K, E1, D = 4, 19, 6, 7, 24
  _, nn_idx, ne = random_samples(rng, B, N, K, E1)
  M = ops.sage_operators(_t(nn_idx).to(dev()), _t(ne).to(dev()))
  prep = ops.graph_prepare(M, torch.zeros((B, N, 4), device=dev()))
  X = _t(rng.randn(B, N, D).astype(np.float32)).to(dev())
  X[:, 3] = X[:, 5]                                      # exact ties between nodes 3 and 5
  msg, arg = ops.neighbour_max(X, prep)
  live = (M != 0).permute(0, 1, 3, 2)                    # [B, n, e, m]
  v = torch.where(live.unsqueeze(4), X.unsqueeze(1).unsqueeze(1), torch.tensor(float('-inf'), device=dev()))
  mx, _ = v.max(dim=3)                                   # [B, n, e, D]
  empty = ~live.any(dim=3)
  want = torch.where(empty.unsqueeze(3), torch.zeros_like(mx), mx)
  assert torch.equal(msg.view(B, N, E1, D), want)
  # argmax: lowest node index among the maxima, -1 for an empty row
  hits = (v == mx.unsqueeze(3)) & live.unsqueeze(4)
  idx = torch.arange(N, device=dev()).view(1, 1, 1, N, 1).expand_as(hits)
  lowest = torch.where(hits, idx, torch.full_like(idx, N)).min(dim=3).values
  want_arg = torch.where(empty.unsqueeze(3), torch.full_like(lowest, -1), lowest)
  assert torch.equal(arg.long(), want_arg)
  # backward: the gradient lands on the argmax node, per feature
  Xg = X.clone().requires_grad_(True)
  g = _t(rng.randn(B, N, E1 * D).astype(np.float32)).to(dev())
  neighbour_max(Xg, prep).backward(g)
  want_g = torch.zeros((B, N * D), dtype=torch.float64, device=dev())
  a = arg.long().view(B, -1)
  f = torch.arange(D, device=dev()).repeat(N * E1).view(1, -1).expand(B, -1)
  ok = a >= 0
  flat = torch.where(ok, a * D + f, torch.zeros_like(a))
  want_g.scatter_add_(1, flat, torch.where(ok, g.view(B, -1).double(), torch.zeros_like(g.view(B, -1).double())))
  torch.testing.assert_close(Xg.grad.double(), want_g.view(B, N, D), rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('agg', ['Mean', 'Max'])
def test_model_matches_reference_golden(agg):
  gg = load_golden('graphsage_qm8.npz')
  a = agg.lower()
  args = [_t(gg[k]).to(dev()) for k in ('node_feat', 'nn_idx', 'nonempty_mask')]
  mask = _t(gg['node_mask']).to(dev())
  cases = [(configs.qm8_graphsage(agg_func=agg), int(gg['weight_seed']), '%s_score' % a),
           (configs.qm8_graphsage(agg_func=agg, **SMALL), int(gg['weight_seed']) + 1, '%s_small' % a)]
  for cfg, seed, key in cases:
    mod, params = _build(cfg, seed)
    assert mod.stack_supported(26, 7)
    with torch.no_grad():
      if key.endswith('_score'):                        # the config shape: 16 outputs like the labels
        score, loss = mod(*args, label=_t(gg['label']).to(dev()), mask=mask)
      else:
        score = mod(*args, mask=mask)
      nomask = mod(*args)
    for got, k, m in ((score, key, gg['node_mask']), (nomask, key + '_nomask', None)):
      np.testing.assert_allclose(got.cpu().numpy(), gg[k], rtol=FWD_RTOL, atol=FWD_ATOL, err_msg=k)
      s64 = sage_oracle.sage_forward(params, _spec(cfg), gg['node_feat'], gg['nn_idx'], gg['nonempty_mask'], m,
                                     dtype=torch.float64).numpy()
      e_ref = np.abs(gg[k] - s64).max()
      e_ours = np.abs(got.cpu().numpy() - s64).max()
      assert e_ours <= max(4 * e_ref, 5e-6), (k, e_ours, e_ref)
    if key == 'mean_score':
      assert abs(float(loss) - float(gg['loss'])) <= 1e-4 * abs(float(gg['loss']))


@pytest.mark.parametrize('agg', ['Mean', 'Max'])
def test_bench_batch_against_fp64_oracle_and_graph_replay(agg):
  bt = data.sage_collate(data.synthetic_qm8_samples(1024, seed=5), 40, np.random.RandomState(0))
  cfg = configs.qm8_graphsage(agg_func=agg)
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
  with torch.no_grad():
    s64 = sage_oracle.sage_forward(params, _spec(cfg), bt['node_feat'], bt['nn_idx'], bt['nonempty_mask'],
                                   bt['node_mask'], dtype=torch.float64, device=dev())
    s32 = sage_oracle.sage_forward(params, _spec(cfg), bt['node_feat'], bt['nn_idx'], bt['nonempty_mask'],
                                   bt['node_mask'], device=dev())
  e_ours = float((eager.double() - s64).abs().max())
  e_orc = float((s32.double() - s64).abs().max())
  np.testing.assert_allclose(eager.cpu().numpy(), s64.cpu().numpy(), rtol=FWD_RTOL, atol=FWD_ATOL)
  assert e_ours <= max(4 * e_orc, 5e-6), (e_ours, e_orc)


@pytest.mark.parametrize('over', [dict(input_dim=4), dict(input_dim=10, agg_func='Max'),
                                  dict(num_layer=1, hidden_dim=[64], input_dim=64),
                                  dict(num_layer=3, hidden_dim=[64, 32, 32]),
                                  dict(num_layer=10, hidden_dim=[32] * 10, agg_func='Max'),
                                  dict(output_dim=50)],
                         ids=['din4', 'din10-max', 'one-layer', 'nonuniform', 'ten-layers', 'p50'])
def test_off_stack_shapes_run_and_match_the_oracle(over):
  gg = load_golden('graphsage_qm8.npz')
  cfg = configs.qm8_graphsage(**over)
  mod, params = _build(cfg, 11)
  assert not mod.stack_supported(26, 7)
  args = [_t(gg[k]).to(dev()) for k in ('node_feat', 'nn_idx', 'nonempty_mask')]
  for m in (gg['node_mask'], None):
    with torch.no_grad():
      got = mod(*args, mask=None if m is None else _t(m).to(dev()))
    s64 = sage_oracle.sage_forward(params, _spec(cfg), gg['node_feat'], gg['nn_idx'], gg['nonempty_mask'], m,
                                   dtype=torch.float64)
    np.testing.assert_allclose(got.cpu().numpy(), s64.numpy(), rtol=FWD_RTOL, atol=FWD_ATOL)


@pytest.mark.parametrize('agg', ['Mean', 'Max'])
def test_gradients_match_fp64_oracle_autograd(agg):
  gg = load_golden('graphsage_qm8.npz')
  cfg = configs.qm8_graphsage(agg_func=agg)
  mod, params = _build(cfg, 21)
  mod.train()
  args = [_t(gg[k]).to(dev()) for k in ('node_feat', 'nn_idx', 'nonempty_mask')]
  label, mask = _t(gg['label']).to(dev()), _t(gg['node_mask']).to(dev())
  _, loss = mod(*args, label=label, mask=mask)
  loss.backward()
  p64 = {k: v.double().requires_grad_(True) for k, v in params.items()}
  s64 = sage_oracle.sage_forward(p64, _spec(cfg), gg['node_feat'], gg['nn_idx'], gg['nonempty_mask'],
                                 gg['node_mask'], dtype=torch.float64, cast=False)
  l64 = F.mse_loss(s64, torch.from_numpy(gg['label']).double())
  l64.backward()
  assert abs(float(loss.detach()) - float(l64.detach())) <= 1e-4 * float(l64.detach())
  for name, p in mod.named_parameters():
    ref = p64[name].grad
    if ref is None:                                     # filter[num_layer - 1]: never read
      assert p.grad is None or not p.grad.any(), name
      continue
    err = float((p.grad.detach().cpu().double() - ref).abs().max())
    assert err <= 2e-3 * float(ref.abs().max()) + 1e-12, (name, err, float(ref.abs().max()))


@pytest.mark.parametrize('agg', ['Mean', 'Max'])
def test_graphed_step_matches_eager_steps(agg):
  from lanczosnetwork_b200.train import GraphedStep
  cfg = configs.qm8_graphsage(agg_func=agg, num_layer=3, hidden_dim=[64, 64, 64])
  batches = []
  for i in range(3):
    bt = data.sage_collate(data.synthetic_qm8_samples(32, seed=50 + i), 40, np.random.RandomState(i))
    bt['label'] = np.random.RandomState(i).randn(32, 16).astype(np.float32)
    batches.append({k: _t(v).to(dev()) for k, v in bt.items()})

  def make():
    m = GraphSAGE(cfg)
    m.load_state_dict(deterministic_state_dict(m, 77))
    m = m.to(dev()).train()
    return m, torch.optim.SGD(m.parameters(), lr=1e-2, momentum=0.9)

  def call_args(bt):
    return (bt['node_feat'], bt['nn_idx'], bt['nonempty_mask']), {'label': bt['label'], 'mask': bt['node_mask']}

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
  gg = load_golden('graphsage_qm8.npz')
  mod, _ = _build(configs.qm8_graphsage(), 3)
  args = [_t(gg[k]).to(dev()) for k in ('node_feat', 'nn_idx', 'nonempty_mask')]
  mask, label = _t(gg['node_mask']).to(dev()), _t(gg['label']).to(dev())
  with torch.no_grad():
    ref = mod(*args, mask=mask)
    dp = torch.nn.DataParallel(mod, device_ids=[0, 0]).eval()
    score, loss = dp(*args, label=label, mask=mask)
  assert loss.numel() == 2
  torch.testing.assert_close(score, ref, rtol=1e-5, atol=1e-6)
