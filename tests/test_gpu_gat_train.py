"""GAT training path on the GPU: lnb_gat_attention_backward across the forward's envelope against fp64
autograd, TrainableGAT's gradients against the fp64 oracle's autograd (golden batch and B = 1024), the
reference's training loop body, GraphedStep and nn.DataParallel.  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, data, ops
from lanczosnetwork_b200.model import TrainableGAT
from oracle import gat_oracle
import gat_train_oracle
from test_gpu_gat import FWD_ATOL, FWD_RTOL, SMALL, SWEEP, attention_reference, _attention_inputs

pytestmark = pytest.mark.gpu


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _spec(cfg):
  return gat_oracle.make_spec(cfg.model.num_layer, cfg.model.num_heads, cfg.dataset.num_bond_type)


def _build(cfg, seed):
  mod = TrainableGAT(cfg)
  params = deterministic_state_dict(mod, seed)
  mod.load_state_dict(params)
  return mod.to(dev()), params


# ------------------------------------------------------------------------------------------------
def _autograd_reference(args, gout, last, dtype):
  Wh, bias, a1, a2, c1, c2, sb = args
  leaves = [t.detach().to(dtype).requires_grad_(True) for t in (Wh, a1, a2, c1, c2, sb)]
  out = attention_reference(leaves[0], bias, *leaves[1:], last, dtype)
  out.backward(gout.to(dtype))
  return out.detach(), [t.grad for t in leaves]


def _gx_mass(args, gout, last):
  """max over the channels of sum_{b,i,k} |gX| in fp64: the size of the terms behind gc1 and gc2.  Their
  exact sums nearly cancel (sum_i gE[i,k] = 0 up to the leaky-ReLU kink), so the rounding of those terms,
  not the result, sets the attainable error."""
  Wh, bias, a1, a2, c1, c2, sb = [t.double() for t in args]
  B, N, _ = Wh.shape
  C, Fd = a1.shape
  E1 = bias.shape[3]
  W = Wh.view(B, N, C, Fd)
  s1 = torch.einsum('bncf,cf->bnc', W, a1) + c1
  s2 = torch.einsum('bncf,cf->bnc', W, a2) + c2
  x = (s1[:, :, None, :] + s2[:, None, :, :]).detach().requires_grad_(True)
  chan = torch.arange(C, device=Wh.device) // (C // E1)
  att = torch.softmax(F.leaky_relu(x, 0.2) + bias[..., chan], dim=1)
  h = torch.einsum('bikc,bkcf->bicf', att, W) + sb
  out = h.mean(dim=2) if last else F.elu(h).reshape(B, N, C * Fd)
  out.backward(gout.double())
  return float(x.grad.abs().sum(dim=(0, 1, 2)).max())


def _kernel_slopes(args):
  """The leaky-ReLU branch the kernel takes for every (b, i, k, c): s1 and s2 as fp32 fmaf chains in
  feature order plus a rounded bias add, x = s1[i] + s2[k] rounded to fp32 (gat_scores / gat_logit), each
  fmaf emulated exactly in fp64 (the fp32 product is exact there) and rounded back.  Where x is within
  fp32 rounding of the kink the kernel, the exact adjoint of its fp32 forward, and fp64 autograd take
  different slopes: a discrete 0.8 gE difference that no accumulation order removes, so the fp64
  reference takes the kernel's branch."""
  Wh, _, a1, a2, c1, c2, _ = args
  B, N, _ = Wh.shape
  C, Fd = a1.shape
  W = Wh.view(B, N, C, Fd).double()
  d1 = torch.zeros((B, N, C), dtype=torch.float32, device=Wh.device)
  d2 = torch.zeros_like(d1)
  for f in range(Fd):
    d1 = (W[..., f] * a1[:, f].double() + d1.double()).float()
    d2 = (W[..., f] * a2[:, f].double() + d2.double()).float()
  s1, s2 = d1 + c1, d2 + c2
  return (s1[:, :, None, :] + s2[:, None, :, :]) > 0


def _reference_on_kernel_slopes(args, gout, last):
  """fp64 autograd of attention_reference with the leaky-ReLU slopes of ``_kernel_slopes``."""
  Wh, bias, a1, a2, c1, c2, sb = args
  slope = torch.where(_kernel_slopes(args), 1.0, 0.2).double()
  leaves = [t.detach().double().requires_grad_(True) for t in (Wh, a1, a2, c1, c2, sb)]
  W, v1, v2, u1, u2, b = leaves
  B, N, _ = W.shape
  C, Fd = v1.shape
  E1 = bias.shape[3]
  W4 = W.view(B, N, C, Fd)
  s1 = torch.einsum('bncf,cf->bnc', W4, v1) + u1
  s2 = torch.einsum('bncf,cf->bnc', W4, v2) + u2
  chan = torch.arange(C, device=Wh.device) // (C // E1)
  att = torch.softmax((s1[:, :, None, :] + s2[:, None, :, :]) * slope + bias.double()[..., chan], dim=1)
  h = torch.einsum('bikc,bkcf->bicf', att, W4) + b
  out = h.mean(dim=2) if last else F.elu(h).reshape(B, N, C * Fd)
  out.backward(gout.double())
  return [t.grad for t in leaves]


def test_attention_backward_against_fp64_across_the_envelope():
  gen = torch.Generator().manual_seed(2)
  names = ('gWh', 'ga1', 'ga2', 'gc1', 'gc2', 'gsb')
  worst = 0.0
  for N, Fd, heads, E1 in SWEEP:
    for kind in ('mask', 'finite'):
      args = _attention_inputs(gen, 2, N, Fd, heads, E1, kind)
      for last in (False, True):
        out = ops.gat_attention(*args, last=last)
        gout = torch.randn(out.shape, generator=gen, dtype=torch.float64).float().to(dev())
        got = ops.gat_attention_backward(gout, *args, out, last=last)
        r64 = _reference_on_kernel_slopes(args, gout, last)
        _, r32 = _autograd_reference(args, gout, last, torch.float32)
        # ops returns (gWh, ga1, ga2, gc1, gc2, gsb); autograd of (Wh, a1, a2, c1, c2, sb)
        mass = _gx_mass(args, gout, last)
        for name, g, ref64, ref32 in zip(names, got, r64, r32):
          scale = max(1.0, float(ref64.abs().max()))
          e_ours = float((g.double() - ref64).abs().max())
          e_orc = float((ref32.double() - ref64).abs().max())
          # gc1 / gc2: a floor of 16 fp32 ulps of the summed terms' magnitude, see _gx_mass
          floor = 1e-6 * mass if name in ('gc1', 'gc2') else 0.0
          assert e_ours <= max(4 * e_orc, 2e-6 * scale, floor), '%s %s %.3g %.3g %.3g' % (
              name, (N, Fd, heads, E1, kind, last), e_ours, e_orc, scale)
          worst = max(worst, e_ours / scale)
        again = ops.gat_attention_backward(gout, *args, out, last=last)
        assert all(torch.equal(a, b) for a, b in zip(got, again))        # fixed order: bit-identical
  print('worst scaled error %.3g over %d shapes' % (worst, 4 * len(SWEEP)))


def test_attention_backward_refuses_shapes_outside_the_envelope():
  gen = torch.Generator().manual_seed(3)
  for N, Fd, heads, E1 in ((129, 4, 1, 1), (8, 6, 1, 1), (8, 132, 1, 1), (8, 4, 1, 17), (8, 4, 33, 1)):
    args = _attention_inputs(gen, 1, N, Fd, heads, E1, 'finite')
    C = E1 * heads
    out = torch.zeros((1, N, C * Fd), device=dev())
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match='status -2'):
      ops.gat_attention_backward(out, *args, out)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
    assert not ops.gat_attention_backward_supported(N, Fd, E1, heads)
  assert ops.gat_attention_backward_supported(128, 128, 16, 32)
  # an empty batch: zero parameter gradients, nothing launched
  args = _attention_inputs(gen, 1, 5, 8, 2, 3, 'finite')
  args = [args[0][:0], args[1][:0]] + args[2:]
  n0 = ops.launch_count()
  g = ops.gat_attention_backward(args[0], *args, args[0], last=False)
  assert ops.launch_count() == n0 and g[0].shape == (0, 5, 48)
  assert all(t.shape == s and not t.any() for t, s in zip(g[1:], [(6, 8), (6, 8), (6,), (6,), (6, 8)]))


def test_attention_backward_at_the_largest_shape():
  """N = F = 128 with one head per CTA: the shared-memory corner of the backward (195 KB)."""
  gen = torch.Generator().manual_seed(4)
  args = _attention_inputs(gen, 2, 128, 128, 2, 2, 'finite')
  out = ops.gat_attention(*args, last=False)
  gout = torch.randn(out.shape, generator=gen, dtype=torch.float64).float().to(dev())
  got = ops.gat_attention_backward(gout, *args, out, last=False)
  r64 = _reference_on_kernel_slopes(args, gout, False)
  _, r32 = _autograd_reference(args, gout, False, torch.float32)
  mass = _gx_mass(args, gout, False)
  for name, g, ref64, ref32 in zip(('gWh', 'ga1', 'ga2', 'gc1', 'gc2', 'gsb'), got, r64, r32):
    e_ours = float((g.double() - ref64).abs().max())
    e_orc = float((ref32.double() - ref64).abs().max())
    floor = 1e-6 * mass if name in ('gc1', 'gc2') else 0.0
    assert e_ours <= max(4 * e_orc, 2e-6 * max(1.0, float(ref64.abs().max())), floor), (name, e_ours, e_orc)


# ------------------------------------------------------------------------------------------------
def _grad_check(mod, p64, named_grads, p32=None, floor=1e-3):
  """Every parameter's gradient within 2e-3 of max|ref|, max|ref| floored at ``floor`` of the largest
  gradient entry of the model: the att_net bias gradients nearly cancel (see test_host_gat_train).
  With ``p32`` (the fp32 oracle's autograd) 4x its distance from fp64 is accepted too."""
  top = max(float(p.grad.abs().max()) for p in p64.values() if p.grad is not None)
  for name, g in named_grads:
    ref = p64[name].grad
    if ref is None:
      assert g is None, name
      continue
    err = float((g.detach().cpu().double() - ref.cpu()).abs().max())
    e_orc = 0.0 if p32 is None else float((p32[name].grad.double() - ref).abs().max())
    assert err <= max(2e-3 * max(float(ref.abs().max()), floor * top), 4 * e_orc) + 1e-12, (
        name, err, e_orc, float(ref.abs().max()), top)


@pytest.mark.parametrize('over,dseed', [({}, 0), (SMALL, 1)], ids=['config', 'small'])
def test_gradients_match_fp64_oracle_autograd(over, dseed):
  gg = load_golden('gat_qm8.npz')
  cfg = configs.qm8_gat(**over)
  mod, params = _build(cfg, int(gg['weight_seed']) + dseed)
  P = cfg.model.output_dim
  nf, L = _t(gg['node_feat']).to(dev()), _t(gg['L']).to(dev())
  label, mask = _t(gg['label'][:, :P]).to(dev()), _t(gg['node_mask']).to(dev())
  with torch.no_grad():
    inference = mod.eval()(nf, L, mask=mask)
  mod.train()
  score, loss = mod(nf, L, label=label, mask=mask)
  loss.backward()
  np.testing.assert_allclose(score.detach().cpu().numpy(), inference.cpu().numpy(), rtol=FWD_RTOL, atol=FWD_ATOL)
  p64 = {k: v.double().requires_grad_(True) for k, v in params.items()}
  s64 = gat_train_oracle.gat_forward(p64, _spec(cfg), gg['node_feat'], gg['L'], gg['node_mask'])
  l64 = F.mse_loss(s64, torch.from_numpy(gg['label'][:, :P]).double())
  l64.backward()
  assert abs(float(loss.detach()) - float(l64.detach())) <= 1e-4 * float(l64.detach())
  none = sorted(n for n, p in mod.named_parameters() if p.grad is None)
  assert none == sorted(load_golden('gat_train_grads.npz')['%s_none_grad' % ('small' if over else 'config')].tolist())
  _grad_check(mod, p64, [(n, p.grad) for n, p in mod.named_parameters()])


def test_bench_batch_gradients_match_fp64_oracle_autograd():
  batch = data.synthetic_qm8_batch(1024, seed=5)
  cfg = configs.qm8_gat()
  mod, params = _build(cfg, 77)
  mod.train()
  nf, mask = _t(batch['node_feat']).to(dev()), _t(batch['node_mask']).to(dev())
  L = _t(data.gat_bias(batch['L'])).to(dev())
  label = _t(batch['label']).to(dev())
  _, loss = mod(nf, L, label=label, mask=mask)
  loss.backward()
  p64 = {k: v.to(dev()).double().requires_grad_(True) for k, v in params.items()}
  s64 = gat_train_oracle.gat_forward(p64, _spec(cfg), batch['node_feat'], L, batch['node_mask'], device=dev())
  l64 = F.mse_loss(s64, label.double())
  l64.backward()
  p32 = {k: v.to(dev()).float().requires_grad_(True) for k, v in params.items()}
  s32 = gat_train_oracle.gat_forward(p32, _spec(cfg), batch['node_feat'], L, batch['node_mask'], device=dev())
  F.mse_loss(s32, label).backward()
  assert abs(float(loss.detach()) - float(l64.detach())) <= 1e-4 * float(l64.detach())
  # 2.7e8 (i, k) pairs per step: some sit within fp32 rounding of the leaky-ReLU kink (see _kernel_slopes),
  # and the att_net weights, whose gradients are 1e-3 of the largest here, feel those slope flips most
  _grad_check(mod, p64, [(n, p.grad) for n, p in mod.named_parameters()], p32, floor=1e-2)


def test_reference_training_loop_body_runs_and_learns():
  """The loop body of QM8Runner.train (runner/qm8_runner.py:226-259) through nn.DataParallel with Adam:
  the loss goes down over 25 steps and the inference forward picks up the trained weights."""
  batch = data.synthetic_qm8_batch(64, seed=4)
  model = TrainableGAT(configs.qm8_gat())
  model.load_state_dict(deterministic_state_dict(model, 1234))
  model = torch.nn.DataParallel(model, device_ids=[0]).cuda()
  optimizer = torch.optim.Adam(filter(lambda p: p.requires_grad, model.parameters()), lr=1.0e-3)
  t = {k: _t(v).cuda() for k, v in batch.items()}
  L = _t(data.gat_bias(batch['L'])).cuda()
  model.eval()
  with torch.no_grad():
    before = model(t['node_feat'], L, label=t['label'], mask=t['node_mask'])[1]
  losses = []
  for _ in range(25):
    model.train()
    optimizer.zero_grad()
    _, train_loss = model(t['node_feat'], L, label=t['label'], mask=t['node_mask'])
    train_loss.backward()
    optimizer.step()
    losses.append(float(train_loss))
  assert abs(losses[0] - float(before)) <= 1e-4 * max(1.0, float(before))
  # measured on an H100: 0.954 -> 1.047 after the first Adam step, then 0.9492 from step 3 on
  assert max(losses[-3:]) < 0.998 * losses[0], losses
  model.eval()
  with torch.no_grad():
    after = model(t['node_feat'], L, label=t['label'], mask=t['node_mask'])[1]
  assert float(after) < losses[0]


def test_graphed_step_matches_eager_steps():
  from lanczosnetwork_b200.train import GraphedStep
  cfg = configs.qm8_gat(num_layer=3, num_heads=[4, 4, 4], hidden_dim=[16, 16, 16])
  batches = []
  for i in range(3):
    bt = data.synthetic_qm8_batch(32, seed=50 + i)
    b = {k: _t(bt[k]).to(dev()) for k in ('node_feat', 'node_mask', 'label')}
    b['L'] = _t(data.gat_bias(bt['L'])).to(dev())
    batches.append(b)

  def make():
    m = TrainableGAT(cfg)
    m.load_state_dict(deterministic_state_dict(m, 77))
    m = m.to(dev()).train()
    return m, torch.optim.SGD(m.parameters(), lr=1e-2, momentum=0.9)

  def call_args(bt):
    return (bt['node_feat'], bt['L']), {'label': bt['label'], 'mask': bt['node_mask']}

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
  gg = load_golden('gat_qm8.npz')
  mod, _ = _build(configs.qm8_gat(), 3)
  nf, L, mask = _t(gg['node_feat']).to(dev()), _t(gg['L']).to(dev()), _t(gg['node_mask']).to(dev())
  label = _t(gg['label']).to(dev())
  with torch.no_grad():
    ref = mod.eval()(nf, L, mask=mask)
    dp = torch.nn.DataParallel(mod, device_ids=[0, 0]).eval()
    score, loss = dp(nf, L, label=label, mask=mask)
  torch.testing.assert_close(score, ref, rtol=1e-5, atol=1e-6)
  # training through the replicas: gradients reach the master's parameters that the forward reads
  dp.train()
  _, loss = dp(nf, L, label=label, mask=mask)
  assert loss.numel() == 2
  loss.mean().backward()
  read = [p for n, p in mod.named_parameters() if not (n.startswith('bias_') and int(n.split('_')[2]) < 6)]
  assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in read)
  assert mod.filter[0][0][0].weight.grad.abs().sum() > 0 and mod.att_net_1[6][6][7].weight.grad.abs().sum() > 0
  assert mod.bias_0_6_0.grad.abs().sum() > 0
