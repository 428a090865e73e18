"""KeyedAdaLanczosNet on an H100: the device start vector against its numpy restatement, the module key's
advance (eager and under graph replay), forward_sparse bit-equal to the padded forward on the same start
vector, the powers adjoint against fp64 autograd, gradients against the fp64 oracle, training from records
against padded training, and captured steps (padded and from records) against eager steps."""
import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, load_golden, oracle_spec
from lanczosnetwork_b200 import configs, data, ops, train
from lanczosnetwork_b200.model import AdaLanczosNet, KeyedAdaLanczosNet
from oracle import lanczos_oracle as orc

import keyed_ada_oracle as oracle
from test_gpu_sparse_dropins import _odd_samples

pytestmark = pytest.mark.gpu

KEYS = [(1234, 0), (1234, 1), (2 ** 40 + 17, 2 ** 35 + 3), (-5, -1)]
SMALL = dict(num_layer=2, hidden_dim=[32, 32])


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _key(k):
  return torch.tensor(k, dtype=torch.int64, device=dev())


def _model(seed=11, **over):
  cfg = configs.qm8_ada_lanczos_net(**dict(SMALL, **over))
  mod = KeyedAdaLanczosNet(cfg)
  mod.load_state_dict(deterministic_state_dict(mod, seed))
  return mod.to(dev())


def _records(samples, key, where='device'):
  sp = data.sparse_collate(samples, 20, eigs=False)
  out = {}
  for k, v in sp.items():
    if isinstance(v, np.ndarray):
      t = torch.from_numpy(v)
      out[k] = t.pin_memory() if where == 'pinned' else t.to(dev())
    else:
      out[k] = v
  out['start_key'] = torch.tensor(key, dtype=torch.int64)
  out['start_key'] = out['start_key'].pin_memory() if where == 'pinned' else out['start_key'].to(dev())
  return out


def _padded(samples, N):
  b = data.collate(samples, 1, num_nodes=N)
  return _t(b['node_feat']).to(dev()), _t(b['L']).to(dev()), _t(b['node_mask']).to(dev())


# ---- start vector ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,N', [(1, 1), (3, 7), (64, 26), (1024, 26), (5, 128), (2, 1001)])
def test_start_vector_matches_the_restatement(B, N):
  for k in KEYS:
    q = ops.ada_start_vector(_key(k), B, N).cpu().numpy()
    ref = oracle.start_vector(k, B, N)
    # logf / sincospif are within ~1 ulp: a few ulps of max(|r|, 1), r the Box-Muller radius
    err = np.abs(q.astype(np.float64) - ref) / np.maximum(np.abs(ref), 1.0)
    assert err.max() <= 4 * 2.0 ** -23, (B, N, k, err.max())
    again = ops.ada_start_vector(_key(k), B, N)
    assert np.array_equal(again.cpu().numpy(), q)
  a = ops.ada_start_vector(_key((7, 9)), B, N)
  assert not torch.equal(a, ops.ada_start_vector(_key((8, 9)), B, N))
  assert not torch.equal(a, ops.ada_start_vector(_key((7, 10)), B, N))


def test_module_key_advances_once_per_forward_eager_and_replayed():
  samples = data.synthetic_qm8_samples(16, seed=3)
  mod = _model().eval()
  nf, L, mask = _padded(samples, 26)
  with torch.no_grad():
    outs = [mod(nf, L, mask=mask) for _ in range(4)]          # capture, then copy-slot / resident replays
  assert mod.start_key.tolist() == [1234, 4]
  with torch.no_grad():                                       # call i drew from (1234, i)
    for i in range(4):
      assert torch.equal(outs[i], mod._keyed_impl(nf, L, mask, _key((1234, i)))), i
  assert not torch.equal(outs[0], outs[1])
  with torch.no_grad():
    fixed = [mod(nf, L, mask=mask, start_key=_key((1234, 1))) for _ in range(2)]
  assert mod.start_key.tolist() == [1234, 4] and torch.equal(fixed[0], outs[1]) and torch.equal(fixed[1], outs[1])
  # a graph the user captures around forward advances the key on every replay
  graph = torch.cuda.CUDAGraph()
  with torch.no_grad():
    with torch.cuda.graph(graph):
      out = mod(nf, L, mask=mask)
  k0 = mod.start_key.tolist()
  graph.replay()
  first = out.clone()
  graph.replay()
  torch.cuda.synchronize()
  assert mod.start_key.tolist() == [k0[0], k0[1] + 2]
  assert not torch.equal(first, out)
  with torch.no_grad():
    assert torch.equal(first, mod._keyed_impl(nf, L, mask, _key((k0[0], k0[1]))))
  # the training forward advances it too
  mod.train()
  label = torch.zeros(nf.shape[0], 16, device=dev())
  mod(nf, L, label=label, mask=mask)[1].backward()
  assert mod.start_key.tolist() == [k0[0], k0[1] + 3]


# ---- forward_sparse ----------------------------------------------------------------------------------------
def _cases():
  return {'qm8_64': data.synthetic_qm8_samples(64, seed=67), 'qm8_1024': data.synthetic_qm8_samples(1024, seed=1027),
          'odd': _odd_samples(), 'n60': data.synthetic_qm8_samples(24, seed=5, max_nodes=60)}


@pytest.mark.parametrize('name', ['qm8_64', 'qm8_1024', 'odd', 'n60'])
def test_forward_sparse_equals_padded_forward_on_the_same_start_vector(name):
  samples = _cases()[name]
  mod = _model(seed=3).eval()
  for key in KEYS[:3]:
    rec = _records(samples, key)
    N, B = int(rec['N']), len(samples)
    if name == 'n60':
      assert N > 32
    nf, L, mask = _padded(samples, N)
    with torch.no_grad():
      ref = mod._forward_impl(nf, L, mask, ops.ada_start_vector(_key(key), B, N))
      for _ in range(3):
        assert torch.equal(mod.forward_sparse(rec), ref), (name, key)
      assert torch.equal(mod.forward_sparse(_records(samples, key, 'pinned')), ref), (name, key)
  assert mod.start_key.tolist() == [1234, 0]                 # an explicit key is not advanced


# ---- powers adjoint -------------------------------------------------------------------------------------
@pytest.mark.parametrize('K,powers', [(8, [2, 5]), (20, [5, 7, 10, 20, 30]), (20, [1, 2, 3, 5, 7, 10, 20, 30]),
                                      (33, [1, 4, 9]), (1, [1, 3])])
def test_tridiag_powers_backward_matches_fp64_autograd(K, powers):
  rng = np.random.RandomState(K)
  B = 37
  d = rng.uniform(-0.6, 0.6, (B, K))
  e = rng.uniform(-0.35, 0.35, (B, K - 1))
  T = np.stack([np.diag(d[b]) + np.diag(e[b], 1) + np.diag(e[b], -1) for b in range(B)])
  Tt = torch.from_numpy(T).requires_grad_(True)
  band = torch.from_numpy((np.abs(np.arange(K)[:, None] - np.arange(K)[None, :]) <= 1).astype(np.float64))
  outs, cur = [], Tt
  for p in range(1, max(powers) + 1):
    if p in powers:
      outs.append(cur)
    cur = cur @ (Tt * band)
  out = torch.stack(outs, dim=2)
  G = torch.from_numpy(rng.randn(B, K, len(powers), K))
  (out * G).sum().backward()
  ref = Tt.grad
  Tf = Tt.detach().float().to(dev()).requires_grad_(True)
  P = train.tridiag_powers(Tf, powers)
  np.testing.assert_allclose(P.detach().cpu().double().numpy(), out.detach().numpy(), rtol=1e-4, atol=1e-6)
  assert torch.equal(P.detach(), ops.tridiag_powers(Tf.detach(), powers))
  (P * G.float().to(dev())).sum().backward()
  err = float((Tf.grad.cpu().double() - ref).abs().max()) / float(ref.abs().max())
  assert err <= 1e-5, err
  again = ops.tridiag_powers_backward(Tf.detach(), G.float().to(dev()).contiguous(), powers)
  assert torch.equal(again, Tf.grad)                          # no atomics: repeatable bit for bit


# ---- gradients ----------------------------------------------------------------------------------------------
def _oracle_grads(forward, params, monkeypatch):
  p64 = {k: v.detach().double().requires_grad_(v.is_floating_point()) for k, v in params.items()}
  monkeypatch.setattr(orc, '_cast', lambda p, dtype: p)
  loss = forward(p64)
  loss.backward()
  return {k: v.grad for k, v in p64.items() if v.grad is not None}


def _worst(mod, grads_ref):
  worst = 0.0
  for name, p in mod.named_parameters():
    g, r = p.grad.detach().cpu().double(), grads_ref[name]
    worst = max(worst, float((g - r).abs().max()) / (float(r.abs().max()) + 1e-12))
  return worst


def test_gradients_match_the_fp64_oracle_as_closely_as_the_base_tape(monkeypatch):
  """The subclass's training formulation (powers of T on lnb_tridiag_powers and its adjoint) and
  AdaLanczosNet's (chain of GEMMs), same q1, against autograd over the fp64 oracle: both within the 2e-2
  bound of the base class's test, the subclass no further from the oracle (up to rounding: 1.5x) than the
  base tape."""
  g = load_golden('ada_forward_small.npz')
  cfg = configs.qm8_ada_lanczos_net(num_layer=2, hidden_dim=[32, 32], num_eig_vec=8,
                                    long_diffusion_dist=[2, 5], short_diffusion_dist=[1, 3])
  keyed, base = KeyedAdaLanczosNet(cfg), AdaLanczosNet(cfg)
  params = deterministic_state_dict(base, int(g['weight_seed']))
  keyed.load_state_dict(params)
  base.load_state_dict(params)
  keyed, base = keyed.to(dev()).train(), base.to(dev()).train()
  spec = oracle_spec(base, 'AdaLanczosNet')
  B, N = g['node_feat'].shape
  torch.manual_seed(int(g['torch_seed']))
  q1 = torch.randn(B, N, 1)
  label = torch.from_numpy(np.random.RandomState(0).randn(B, g['score'].shape[1]).astype(np.float32)).to(dev())

  def fwd(p64):
    s = orc.ada_lanczos_net_forward(p64, spec, g['node_feat'], g['L'], g['node_mask'], q1[:, :, 0].double(),
                                    dtype=torch.float64)
    return torch.nn.functional.mse_loss(s, label.cpu().double())

  grads_ref = _oracle_grads(fwd, params, monkeypatch)
  inputs = (_t(g['node_feat']).to(dev()), _t(g['L']).to(dev()), _t(g['node_mask']).to(dev()), q1.to(dev()))
  errs = {}
  for name, mod in (('keyed', keyed), ('base', base)):
    score = mod._train_impl(*inputs)
    mod.loss_func(score, label).backward()
    errs[name] = _worst(mod, grads_ref)
  print('max relative gradient error vs fp64 oracle: keyed %.3e, base %.3e' % (errs['keyed'], errs['base']))
  assert errs['keyed'] <= 2e-2 and errs['base'] <= 2e-2, errs
  assert errs['keyed'] <= 1.5 * errs['base'] + 1e-6, errs


def test_records_training_equals_padded_training():
  samples = data.synthetic_qm8_samples(64, seed=21)
  key = (99, 3)
  rec = _records(samples, key)
  N, B = int(rec['N']), len(samples)
  label = torch.from_numpy(data.sparse_collate(samples, 20, eigs=False)['label']).to(dev())
  a, b = _model(seed=5).train(), _model(seed=5).train()
  _, loss_r = a.forward_sparse_train(rec, label=label)
  loss_r.backward()
  nf, L, mask = _padded(samples, N)
  loss_p = b.loss_func(b._train_impl(nf, L, mask, ops.ada_start_vector(_key(key), B, N)), label)
  loss_p.backward()
  print('records loss %.9g, padded loss %.9g' % (float(loss_r), float(loss_p)))
  assert abs(float(loss_r) - float(loss_p)) <= 1e-6 * max(1.0, abs(float(loss_p)))
  for (name, p), q in zip(a.named_parameters(), b.parameters()):
    err = float((p.grad - q.grad).abs().max()) / (float(q.grad.abs().max()) + 1e-12)
    assert err <= 1e-4, (name, err)


# ---- captured steps ---------------------------------------------------------------------------------------
def _eager_losses(mod, batches, sparse):
  opt = torch.optim.SGD(mod.parameters(), lr=1e-2, momentum=0.9)
  out = []
  for args, kw in batches:
    opt.zero_grad()
    _, loss = mod.forward_sparse_train(*args, **kw) if sparse else mod(*args, **kw)
    loss.backward()
    opt.step()
    out.append(float(loss))
  return out


@pytest.mark.parametrize('sparse', [False, True])
def test_graphed_step_matches_eager_steps_with_explicit_keys(sparse):
  pool = [data.synthetic_qm8_samples(32, seed=s) for s in (1, 2, 3)]
  N = max(max(s['L_simple_4'].shape[0] for s in smp) for smp in pool)
  batches = []
  for i in range(6):
    smp = pool[i % 3]
    label = torch.from_numpy(data.sparse_collate(smp, 20, eigs=False)['label']).to(dev())
    key = (1000 + i, i)
    if sparse:
      rec = _records(smp, key)
      rec['N'] = N
      batches.append(((rec,), {'label': label}))
    else:
      nf, L, mask = _padded(smp, N)
      batches.append(((nf, L), {'label': label, 'mask': mask, 'start_key': _key(key)}))
  mod = _model(seed=8).train()
  ref = _eager_losses(_model(seed=8).train(), batches, sparse)
  opt = torch.optim.SGD(mod.parameters(), lr=1e-2, momentum=0.9)
  step = train.GraphedStep(mod, opt, batches[0][0], batches[0][1], sparse=sparse)
  got = [float(step(*args, **kw)[1]) for args, kw in batches]
  print('graphed', got, 'eager', ref)
  np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('sparse', [False, True])
def test_graphed_step_key_changes_the_loss(sparse):
  smp = data.synthetic_qm8_samples(32, seed=4)
  label = torch.from_numpy(data.sparse_collate(smp, 20, eigs=False)['label']).to(dev())
  mod = _model(seed=9).train()
  opt = torch.optim.SGD(mod.parameters(), lr=0.0)             # weights fixed: only the key moves the loss

  def call_args(key):
    if sparse:
      return (_records(smp, key),), {'label': label}
    nf, L, mask = _padded(smp, int(data.sparse_collate(smp, 20, eigs=False)['N']))
    return (nf, L), {'label': label, 'mask': mask, 'start_key': _key(key)}

  args, kw = call_args((5, 0))
  step = train.GraphedStep(mod, opt, args, kw, sparse=sparse)
  a = float(step(*args, **kw)[1])
  args2, kw2 = call_args((5, 1))
  b = float(step(*args2, **kw2)[1])
  c = float(step(*args, **kw)[1])
  assert a != b and a == c, (a, b, c)


def test_graphed_step_advances_the_module_key_per_replay():
  smp = data.synthetic_qm8_samples(32, seed=6)
  label = torch.from_numpy(data.sparse_collate(smp, 20, eigs=False)['label']).to(dev())
  nf, L, mask = _padded(smp, int(data.sparse_collate(smp, 20, eigs=False)['N']))
  mod = _model(seed=10).train()
  opt = torch.optim.SGD(mod.parameters(), lr=0.0)
  step = train.GraphedStep(mod, opt, (nf, L), {'label': label, 'mask': mask}, warmup=3)
  k = mod.start_key.tolist()
  assert k == [1234, 3]                                       # the warm-up steps drew from the module key
  losses = [float(step(nf, L, label=label, mask=mask)[1]) for _ in range(3)]
  assert mod.start_key.tolist() == [1234, 6]
  assert len(set(losses)) == 3, losses


# ---- Lanczos layer adjoint ----------------------------------------------------------------------------------
def _spd(B, N, seed):
  rng = np.random.RandomState(seed)
  X = rng.randn(B, N, N)
  A = X @ np.swapaxes(X, 1, 2) / N + np.eye(N)[None]
  return A / np.linalg.norm(A, axis=(1, 2), keepdims=True)


def _lanczos_case(A, mask, q1, K, seed):
  """(fp32 kernel gA, fp64 autograd gA of the restatement, kernel idx, restatement idx, kernel T/Q, tape T/Q)."""
  rng = np.random.RandomState(seed)
  B, N = A.shape[0], A.shape[1]
  gT, gQ = rng.randn(B, K, K), rng.randn(B, N, K)
  A64 = torch.from_numpy(A).requires_grad_(True)
  m64 = None if mask is None else torch.from_numpy(mask)
  T64, Q64, idx64 = oracle.lanczos_block_gs(A64, m64, torch.from_numpy(q1), K)
  ((T64 * torch.from_numpy(gT)).sum() + (Q64 * torch.from_numpy(gQ)).sum()).backward()
  Ad, qd = torch.from_numpy(A).float().to(dev()), torch.from_numpy(q1).float().to(dev())
  md = None if mask is None else torch.from_numpy(mask).to(dev())
  Ad.requires_grad_(True)
  T, Q = train.lanczos_tridiag(Ad, md, qd, K)
  ((T * torch.from_numpy(gT).float().to(dev())).sum() + (Q * torch.from_numpy(gQ).float().to(dev())).sum()).backward()
  fwd = ops.lanczos_tridiag_train(Ad.detach(), md, qd, K)
  gA2, T2, Q2 = ops.lanczos_tridiag_backward(Ad.detach(), md, qd, K, torch.from_numpy(gT).float().to(dev()),
                                             torch.from_numpy(gQ).float().to(dev()), want_tape=True)
  # the backward differentiates the tape the forward returned, bit for bit; repeated launches agree bit for bit
  assert torch.equal(T2, T.detach()) and torch.equal(Q2, Q.detach()) and torch.equal(gA2, Ad.grad)
  assert torch.equal(fwd['T'], T.detach())
  return Ad.grad.cpu().double(), A64.grad, fwd['idx'].cpu().long(), idx64, fwd


@pytest.mark.parametrize('N,K', [(26, 8), (40, 12), (128, 16), (64, 40), (9, 20)])
def test_lanczos_backward_matches_fp64_autograd_away_from_breakdown(N, K):
  """Random SPD operators, K below the number of real nodes (no breakdown), or N < K with the Krylov space
  exhausted at step N (zero padding): the adjoint within 1e-4 of max|ref| of fp64 autograd over the
  restatement, or within twice the error of the same restatement run in fp32 where the recurrence amplifies
  fp32 rounding past that (K = 12 of 40 and 40 of 48 real nodes: 1.3-1.6e-4).  Without a mask every node is real; with one, half of the graphs have padded nodes (zero
  operator rows and columns, as the collate builds them)."""
  B = 12
  rng = np.random.RandomState(N + K)
  q1 = rng.randn(B, N)
  mask = np.ones((B, N), np.uint8)
  mask[::2, N - N // 4:] = 0
  A = _spd(B, N, N * 7 + K)
  cases = ((A, None), (A * (mask[:, :, None] * mask[:, None, :]), mask))
  for Ac, msk in cases:
    got, ref, idx, idx64, _ = _lanczos_case(Ac, msk, q1, K, N)
    assert torch.equal(idx, idx64), (idx, idx64)
    err = float((got - ref).abs().max()) / float(ref.abs().max())
    # the same restatement in fp32 on the CPU: what fp32 arithmetic of this formula gives on this operator
    g = np.random.RandomState(N)
    gT, gQ = torch.from_numpy(g.randn(B, K, K)), torch.from_numpy(g.randn(B, N, K))
    A32 = torch.from_numpy(Ac).float().requires_grad_(True)
    T32, Q32, _ = oracle.lanczos_block_gs(A32, None if msk is None else torch.from_numpy(msk),
                                          torch.from_numpy(q1).float(), K)
    ((T32 * gT.float()).sum() + (Q32 * gQ.float()).sum()).backward()
    err32 = float((A32.grad.double() - ref).abs().max()) / float(ref.abs().max())
    print('lanczos adjoint N=%d K=%d mask=%s: %.3e of max|ref| (fp32 restatement %.3e)'
          % (N, K, msk is not None, err, err32))
    assert err <= max(1e-4, 2.0 * err32), (err, err32)


def test_lanczos_forward_agrees_with_lanczos_ritz():
  """The training layer's T and Q against lnb_lanczos_ritz(want_ritz=False) on QM8 Gaussian Laplacians: the
  same rules (idx equal), fp32 rounding apart (the two kernels reduce in different orders)."""
  samples = data.synthetic_qm8_samples(64, seed=31)
  mod = _model(seed=2)
  N = max(s['L_simple_4'].shape[0] for s in samples)
  nf, L, mask = _padded(samples, N)
  with torch.no_grad():
    Le = ops.gaussian_laplacian(ops.embedding_rows(nf, mod.embedding.weight), L)
  q1 = ops.ada_start_vector(_key((3, 4)), len(samples), N)
  ref = ops.lanczos_ritz(Le, mask, q1, 20, want_ritz=False)
  got = ops.lanczos_tridiag_train(Le, mask, q1, 20)
  same = got['idx'] == ref['idx']
  print('idx equal on %d of %d graphs' % (int(same.sum()), same.numel()))
  assert int(same.sum()) >= same.numel() - 2
  np.testing.assert_allclose(got['T'][same].cpu().numpy(), ref['T'][same].cpu().numpy(), atol=2e-4)


def test_lanczos_backward_on_qm8_laplacians_at_breakdown():
  """QM8 Gaussian Laplacians with K = 20 > n: the recurrence breaks down inside every graph.  Graphs whose
  acceptance (idx) fp32 and fp64 decide alike are compared; the measured bound is stated in DESIGN §8.6.5."""
  samples = data.synthetic_qm8_samples(64, seed=41)
  mod = _model(seed=4)
  N = max(s['L_simple_4'].shape[0] for s in samples)
  nf, L, mask = _padded(samples, N)
  with torch.no_grad():
    A = train._gaussian_laplacian_train(mod.embedding.weight[nf].double(), (L[:, :, :, 0] != 0).double())
  q1 = ops.ada_start_vector(_key((8, 1)), len(samples), N).double().cpu().numpy()
  got, ref, idx, idx64, _ = _lanczos_case(A.cpu().numpy(), mask.cpu().numpy(), q1, 20, 5)
  keep = idx == idx64
  assert int(keep.sum()) >= len(samples) - 4, (idx, idx64)
  g, r = got[keep], ref[keep]
  err = float((g - r).abs().max()) / float(r.abs().max())
  print('lanczos adjoint on QM8 Laplacians at breakdown: %.3e of max|ref| (%d of %d graphs with equal idx)'
        % (err, int(keep.sum()), len(samples)))
  assert err <= 1e-2, err
