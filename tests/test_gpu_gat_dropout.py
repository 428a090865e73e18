"""KeyedGAT and its dropout kernels on the GPU: the masked projection and the attention dropout pair against
fp64 autograd on the masks of the rule (gat_dropout_oracle, run on the GPU), KeyedGAT's gradients against fp64
autograd of the masked oracle, the key semantics, GraphedStep (padded and sparse=True), the records entry
against the padded one, and the reference's training loop body with dropout.  ``pytest -m gpu``."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, data, dropin, ops
from lanczosnetwork_b200.model import GAT, KeyedGAT, TrainableGAT
from lanczosnetwork_b200.train import GraphedStep
from oracle import gat_oracle
import gat_dropout_oracle as oracle
from test_gpu_gat import SMALL, SWEEP, _attention_inputs
from test_gpu_gat_train import _grad_check, _kernel_slopes

pytestmark = pytest.mark.gpu
P_VALUES = (0.1, 0.5, 0.9, 1.0)
U = 2.0 ** -24                                          # fp32 unit roundoff


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _key(seed, ctr):
  return torch.tensor([seed, ctr], dtype=torch.int64, device=dev())


def _spec(cfg):
  return gat_oracle.make_spec(cfg.model.num_layer, cfg.model.num_heads, cfg.dataset.num_bond_type)


# ------------------------------------------------------------------------------------------------
# the masked projection
PROJECT = [(Din, Fd) for Din in (64, 896, 68) for Fd in (4, 16, 128)]


@pytest.mark.parametrize('Din,Fd', PROJECT)
def test_masked_projection_against_fp64_autograd(Din, Fd):
  """Every element within the fp32 summation bound (K + 2) u sum_k |a_k b_k| of fp64 autograd on the oracle's
  masks (K terms, one rounding of the scale): a wrong or shifted mask element misses by the element itself.
  Repeated backward launches are bit-identical."""
  gen = torch.Generator().manual_seed(Din * 1000 + Fd)
  cases = [(1, 3), (1024, 1 + (Din + Fd) % 5)]
  for i, (B, C) in enumerate(cases):
    p = P_VALUES[(PROJECT.index((Din, Fd)) + i) % 4]
    key = _key(B + Din, 3 * Fd + i)
    M = B * 26
    X = torch.randn(M, Din, generator=gen, dtype=torch.float64).float().to(dev())
    W = (torch.randn(C * Fd, Din, generator=gen, dtype=torch.float64) / np.sqrt(Din)).float().to(dev())
    g = torch.randn(M, C * Fd, generator=gen, dtype=torch.float64).float().to(dev())
    Wh = ops.gat_dropout_project(X, W, C, key, p, 4)
    gX, gW = ops.gat_dropout_project_backward(X, W, g, C, key, p, 4)
    gX2, gW2 = ops.gat_dropout_project_backward(X, W, g, C, key, p, 4)
    assert torch.equal(gX, gX2) and torch.equal(gW, gW2)
    x64 = X.double().requires_grad_(True)
    w64 = W.double().requires_grad_(True)
    outs, bound, gx_bound, gw_bound = [], [], torch.zeros_like(x64), []
    for c in range(C):
      m = oracle.mask(key.cpu(), p, 4, c, oracle.INPUT, (M, Din), dev())
      wc = w64[c * Fd:(c + 1) * Fd]
      outs.append((x64 * m) @ wc.t())
      xm = (X.double() * m).abs()
      gc = g.double()[:, c * Fd:(c + 1) * Fd].abs()
      bound.append((Din + 2) * U * (xm @ W.double()[c * Fd:(c + 1) * Fd].abs().t()))
      gx_bound += m.abs() * (gc @ W.double()[c * Fd:(c + 1) * Fd].abs())
      gw_bound.append((M + 2) * U * (gc.t() @ xm))
    ref = torch.cat(outs, dim=1)
    ref.backward(g.double())
    gx_bound = (Fd * C + 2) * U * gx_bound
    for name, got, want, bnd in (('Wh', Wh, ref.detach(), torch.cat(bound, dim=1)), ('gX', gX, x64.grad, gx_bound),
                                 ('gW', gW, w64.grad, torch.cat(gw_bound, dim=0))):
      err = (got.double() - want).abs()
      assert bool((err <= bnd + 1e-30).all()), (name, B, C, p, float(err.max()), float((err - bnd).max()))
    if p == 1.0:
      assert not Wh.any() and not gX.any() and not gW.any()


def test_masked_projection_at_the_reference_hidden_layer():
  """C = 56 channels of F = 16 over Din = 896 at B = 64, p = 0.1: the QM8 configuration's hidden layer."""
  gen = torch.Generator().manual_seed(11)
  M, Din, C, Fd, p = 64 * 26, 896, 56, 16, 0.1
  key = _key(5, 6)
  X = torch.randn(M, Din, generator=gen, dtype=torch.float64).float().to(dev())
  W = (torch.randn(C * Fd, Din, generator=gen, dtype=torch.float64) / 30).float().to(dev())
  Wh = ops.gat_dropout_project(X, W, C, key, p, 2)
  for c in (0, 17, 55):
    m = oracle.mask(key.cpu(), p, 2, c, oracle.INPUT, (M, Din), dev())
    ref = (X.double() * m) @ W.double()[c * Fd:(c + 1) * Fd].t()
    bnd = (Din + 2) * U * ((X.double() * m).abs() @ W.double()[c * Fd:(c + 1) * Fd].abs().t())
    assert bool(((Wh[:, c * Fd:(c + 1) * Fd].double() - ref).abs() <= bnd).all()), c


def test_masked_projection_refuses_shapes_outside_the_envelope():
  key = _key(1, 2)
  for Din, Fd in ((66, 4), (64, 6), (64, 132)):
    X, W = torch.zeros(8, Din, device=dev()), torch.zeros(2 * Fd, Din, device=dev())
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match='status -2'):
      ops.gat_dropout_project(X, W, 2, key, 0.1, 0)
    with pytest.raises(RuntimeError, match='status -2'):
      ops.gat_dropout_project_backward(X, W, torch.zeros(8, 2 * Fd, device=dev()), 2, key, 0.1, 0)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0 and not ops.gat_dropout_project_supported(Din, Fd)


# ------------------------------------------------------------------------------------------------
# the attention dropout pair
def _site_masks(key, p, t, B, N, C, Fd):
  """M_att s as [B, N, N, C] and M_wh s as [B, N, C, F] for the channels of a layer (fp64, on the GPU)."""
  Ma = oracle.channel_masks(key, p, t, C, oracle.ATT, (B, N, N), dev()).permute(1, 2, 3, 0)
  Mw = oracle.channel_masks(key, p, t, C, oracle.WH, (B, N, Fd), dev()).permute(1, 2, 0, 3)
  return Ma, Mw


def _dropout_reference(args, Ma, Mw, gout, last, dtype, slope=None):
  """lnb_gat_attention_dropout's formula at ``dtype`` and its autograd: (out, [gWh, ga1, ga2, gc1, gc2, gsb],
  mass), mass = max over channels of sum |d loss / d logit| (the terms behind gc1, gc2).  ``slope``: the
  kernel's leaky-ReLU branches (test_gpu_gat_train._kernel_slopes)."""
  Wh, bias, a1, a2, c1, c2, sb = args
  leaves = [t.detach().to(dtype).requires_grad_(True) for t in (Wh, a1, a2, c1, c2, sb)]
  W, v1, v2, u1, u2, b = leaves
  B, N, _ = W.shape
  C, Fd = v1.shape
  E1 = bias.shape[3]
  W4 = W.view(B, N, C, Fd)
  s1 = torch.einsum('bncf,cf->bnc', W4, v1) + u1
  s2 = torch.einsum('bncf,cf->bnc', W4, v2) + u2
  x = s1[:, :, None, :] + s2[:, None, :, :]
  x.retain_grad()
  chan = torch.arange(C, device=Wh.device) // (C // E1)
  lr = F.leaky_relu(x, 0.2) if slope is None else x * torch.where(slope, 1.0, 0.2).to(dtype)
  att = torch.softmax(lr + bias.to(dtype)[..., chan], dim=1) * Ma.to(dtype)
  h = torch.einsum('bikc,bkcf->bicf', att, W4 * Mw.to(dtype)) + b
  out = h.mean(dim=2) if last else F.elu(h).reshape(B, N, C * Fd)
  out.backward(gout.to(dtype))
  return out.detach(), [t.grad for t in leaves], float(x.grad.abs().sum(dim=(0, 1, 2)).max())


def test_attention_dropout_pair_against_fp64_across_the_envelope():
  """The bounds of the dropout-free pair (test_gpu_gat, test_gpu_gat_train): 4x the fp32 oracle's distance
  from fp64, floor 2e-6 of the scale, gc1 / gc2 floored at 1e-6 of the summed terms; p cycles over P_VALUES
  along the sweep.  Repeated backward launches are bit-identical."""
  gen = torch.Generator().manual_seed(21)
  names = ('gWh', 'ga1', 'ga2', 'gc1', 'gc2', 'gsb')
  for n, (N, Fd, heads, E1) in enumerate(SWEEP):
    p = P_VALUES[n % 4]
    C = E1 * heads
    for kind in ('mask', 'finite'):
      args = _attention_inputs(gen, 2, N, Fd, heads, E1, kind)
      key = _key(n, 7)
      Ma, Mw = _site_masks(key.cpu(), p, 3, 2, N, C, Fd)
      slope = _kernel_slopes(args)
      for last in (False, True):
        got = ops.gat_attention_dropout(*args, key, p, 3, last=last)
        gout = torch.randn(got.shape, generator=gen, dtype=torch.float64).float().to(dev())
        r64, g64, mass = _dropout_reference(args, Ma, Mw, gout, last, torch.float64, slope)
        r32, g32, _ = _dropout_reference(args, Ma, Mw, gout, last, torch.float32)
        scale = max(1.0, float(r64.abs().max()))
        e_ours, e_orc = float((got.double() - r64).abs().max()), float((r32.double() - r64).abs().max())
        assert e_ours <= max(4 * e_orc, 2e-6 * scale), ('out', N, Fd, heads, E1, kind, last, p, e_ours, e_orc)
        grads = ops.gat_attention_dropout_backward(gout, *args, key, p, 3, last=last)
        again = ops.gat_attention_dropout_backward(gout, *args, key, p, 3, last=last)
        assert all(torch.equal(a, b) for a, b in zip(grads, again))
        for name, g, ref64, ref32 in zip(names, grads, g64, g32):
          sc = max(1.0, float(ref64.abs().max()))
          e_ours, e_orc = float((g.double() - ref64).abs().max()), float((ref32.double() - ref64).abs().max())
          floor = 1e-6 * mass if name in ('gc1', 'gc2') else 0.0
          assert e_ours <= max(4 * e_orc, 2e-6 * sc, floor), (name, N, Fd, heads, E1, kind, last, p, e_ours, e_orc)


def test_attention_dropout_at_p0_is_the_dropout_free_pair():
  gen = torch.Generator().manual_seed(22)
  args = _attention_inputs(gen, 3, 26, 16, 8, 7, 'mask')
  key = _key(3, 4)
  for last in (False, True):
    out = ops.gat_attention(*args, last=last)
    assert torch.equal(ops.gat_attention_dropout(*args, key, 0.0, 0, last=last), out)
    gout = torch.randn(out.shape, generator=gen).to(dev())
    for a, b in zip(ops.gat_attention_backward(gout, *args, out, last=last),
                    ops.gat_attention_dropout_backward(gout, *args, key, 0.0, 0, last=last)):
      assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------
# KeyedGAT
def _build(cfg, seed, cls=KeyedGAT):
  mod = cls(cfg)
  params = deterministic_state_dict(mod, seed)
  mod.load_state_dict(params)
  return mod.to(dev()), params


def _model_slopes(mod, node_ids, L, key, p):
  """The leaky-ReLU branch the kernels take at every layer: the training forward's layers replayed through
  the same ops (same bits), and test_gpu_gat_train._kernel_slopes of each layer's Wh.  Where s1[i] + s2[k]
  lies within fp32 rounding of the kink the kernels and fp64 autograd take different slopes, a discrete
  0.8 gE difference that every upstream gradient inherits, so the fp64 oracle takes the kernels' branch."""
  state = ops.embedding_rows(node_ids, mod.embedding.weight)
  B, N = node_ids.shape
  E = mod.num_edgetype
  out = []
  with torch.no_grad():
    for t in range(mod.num_layer):
      mods = [(jj, ii) for jj in range(E + 1) for ii in range(mod.num_heads[t])]
      w = torch.cat([mod.filter[t][jj][ii].weight for jj, ii in mods], dim=0)
      a1 = torch.cat([mod.att_net_1[t][jj][ii].weight for jj, ii in mods], dim=0)
      a2 = torch.cat([mod.att_net_2[t][jj][ii].weight for jj, ii in mods], dim=0)
      c1 = torch.cat([mod.att_net_1[t][jj][ii].bias for jj, ii in mods], dim=0)
      c2 = torch.cat([mod.att_net_2[t][jj][ii].bias for jj, ii in mods], dim=0)
      sb = torch.stack([getattr(mod, 'bias_%d_%d_%d' % (ii, E, t)) for _, ii in mods], dim=0)
      Wh = ops.gat_dropout_project(state.reshape(B * N, -1), w, len(mods), key, p, t).view(B, N, -1)
      args = (Wh, L, a1, a2, c1, c2, sb)
      out.append(_kernel_slopes(args))
      state = ops.gat_attention_dropout(*args, key, p, t, last=(t == mod.num_layer - 1))
  return out


@pytest.mark.parametrize('p', [0.1, 0.5])
@pytest.mark.parametrize('which', ['golden', 'B256'])
def test_keyed_gat_gradients_match_fp64_masked_oracle(which, p):
  """Gradients against fp64 autograd of the masked oracle on the kernels' leaky-ReLU branches
  (_model_slopes), with test_gpu_gat_train's bounds (_grad_check); 4x the fp32 oracle's own distance from
  fp64 is accepted as there at B = 1024.  p = 0.5 runs three of the configuration's layers (same heads and
  widths): through all seven, the factor 2 at three sites per layer drives the loss from 1 to 2e3 and the
  fp32 oracle's own gradients 3e-3 of the largest away from fp64, which leaves no accuracy to check."""
  cfg = configs.qm8_gat(dropout=p) if p < 0.5 else configs.qm8_gat(dropout=p, num_layer=3, num_heads=[8] * 3,
                                                                     hidden_dim=[16] * 3)
  if which == 'golden':
    gg = load_golden('gat_qm8.npz')
    nf_np, L, mask_np, label_np, seed = gg['node_feat'], _t(gg['L']).to(dev()), gg['node_mask'], gg['label'], 3
  else:
    batch = data.synthetic_qm8_batch(256, seed=6)
    nf_np, mask_np, label_np, seed = batch['node_feat'], batch['node_mask'], batch['label'], 4
    L = _t(data.gat_bias(batch['L'])).to(dev())
  mod, params = _build(cfg, seed)
  mod.train()
  key = _key(1234, 9)
  label = _t(label_np[:, :cfg.model.output_dim]).to(dev())
  _, loss = mod(_t(nf_np).to(dev()), L, label=label, mask=_t(mask_np).to(dev()), dropout_key=key)
  loss.backward()
  slopes = _model_slopes(mod, _t(nf_np).to(dev()), L, key, p)
  grads = {}
  for dtype in (torch.float64, torch.float32):
    pd = {k: v.to(dev()).to(dtype).requires_grad_(True) for k, v in params.items()}
    s = oracle.gat_forward_dropout(pd, _spec(cfg), nf_np, L, mask_np, key.cpu(), p, device=dev(),
                                   slopes=slopes if dtype == torch.float64 else None)
    lo = F.mse_loss(s, label.to(dtype))
    lo.backward()
    grads[dtype] = (pd, float(lo.detach()))
  p64, l64 = grads[torch.float64]
  assert abs(float(loss.detach()) - l64) <= 1e-4 * l64
  _grad_check(mod, p64, [(n, q.grad) for n, q in mod.named_parameters()], grads[torch.float32][0],
              floor=1e-3 if which == 'golden' else 1e-2)


def test_key_semantics():
  gg = load_golden('gat_qm8.npz')
  cfg = configs.qm8_gat(dropout=0.3, **SMALL)
  nf, L, mask = _t(gg['node_feat']).to(dev()), _t(gg['L']).to(dev()), _t(gg['node_mask']).to(dev())
  mod, params = _build(cfg, 5)
  mod.train()
  k0 = mod.dropout_key.clone()
  a = mod(nf, L, mask=mask)
  b = mod(nf, L, mask=mask)
  assert not torch.equal(a, b)
  assert mod.dropout_key.tolist() == [k0[0].item(), k0[1].item() + 2]
  key = _key(8, 8)
  with torch.no_grad():                                   # the dropout formulation with or without autograd
    c = mod(nf, L, mask=mask, dropout_key=key)
  d = mod(nf, L, mask=mask, dropout_key=key)
  assert torch.equal(c, d.detach()) and key.tolist() == [8, 8]
  assert mod.dropout_key.tolist() == [k0[0].item(), k0[1].item() + 2]
  # eval: GAT's bits; p = 0 in training: TrainableGAT's bits
  ref_gat, _ = _build(cfg, 5, GAT)
  with torch.no_grad():
    assert torch.equal(mod.eval()(nf, L, mask=mask), ref_gat.eval()(nf, L, mask=mask))
  cfg0 = configs.qm8_gat(dropout=0.0, **SMALL)
  m0, _ = _build(cfg0, 5)
  t0, _ = _build(cfg0, 5, TrainableGAT)
  s0, s1 = m0.train()(nf, L, mask=mask), t0.train()(nf, L, mask=mask)
  assert torch.equal(s0, s1)
  s0.sum().backward()
  s1.sum().backward()
  _same_grads([x.grad for x in m0.parameters()], [y.grad for y in t0.parameters()], m0)
  assert m0.dropout_key.tolist() == [1234, 0]


def _same_grads(ga, gb, mod):
  """Equal gradients, bit for bit, except the embedding table's: its adjoint is the scatter-add of the
  reference's unsorted_segment_sum, whose atomics add a row's terms in no fixed order."""
  for (n, _), a, b in zip(mod.named_parameters(), ga, gb):
    if a is None or b is None:
      assert a is None and b is None, n
    elif n == 'embedding.weight':
      torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-7)
    else:
      assert torch.equal(a, b), n


def _samples_and_records(B, seed, N=26):
  samples = data.synthetic_qm8_samples(B, seed=seed)
  sp = data.sparse_collate(samples, 4, eigs=False)
  rec = {k: (torch.from_numpy(v).to(dev()) if isinstance(v, np.ndarray) else v) for k, v in sp.items()}
  c = data.collate(samples, 4, num_nodes=N)
  padded = {'node_feat': _t(c['node_feat']).to(dev()), 'L': _t(data.gat_bias(c['L'])).to(dev()),
            'node_mask': _t(c['node_mask']).to(dev()), 'label': _t(c['label']).to(dev())}
  return rec, padded


def test_records_train_equals_the_padded_training_forward():
  cfg = configs.qm8_gat(dropout=0.2, num_layer=3, num_heads=[4, 4, 4], hidden_dim=[16, 16, 16])
  mod, _ = _build(cfg, 9)
  mod.train()
  rec, pad = _samples_and_records(24, 31)
  key = _key(77, 3)
  rec['dropout_key'] = key
  s_rec, l_rec = mod.forward_sparse_train(rec, label=pad['label'])
  s_pad, l_pad = mod(pad['node_feat'], pad['L'], label=pad['label'], mask=pad['node_mask'], dropout_key=key)
  assert torch.equal(s_rec, s_pad) and torch.equal(l_rec, l_pad)
  g_rec = torch.autograd.grad(l_rec, list(mod.parameters()), allow_unused=True)
  g_pad = torch.autograd.grad(l_pad, list(mod.parameters()), allow_unused=True)
  _same_grads(g_rec, g_pad, mod)
  # without the entry the module's key is read and advanced
  del rec['dropout_key']
  k0 = mod.dropout_key.clone()
  mod.forward_sparse_train(rec, label=pad['label'])
  assert mod.dropout_key[1].item() == k0[1].item() + 1


@pytest.mark.parametrize('sparse', [False, True], ids=['padded', 'sparse'])
def test_graphed_step_replays_equal_eager_steps_with_the_same_keys(sparse):
  cfg = configs.qm8_gat(dropout=0.2, num_layer=3, num_heads=[4, 4, 4], hidden_dim=[16, 16, 16])
  batches = [_samples_and_records(32, 60 + i) for i in range(3)]
  keys = [_key(5, 100 + i) for i in range(6)]

  def make():
    m, _ = _build(cfg, 13)
    return m.train(), torch.optim.SGD(m.parameters(), lr=1e-2, momentum=0.9)

  def step_args(i):
    rec, pad = batches[i % 3]
    if sparse:
      r = dict(rec, dropout_key=keys[i])
      return (r,), {'label': pad['label']}
    return (pad['node_feat'], pad['L']), {'label': pad['label'], 'mask': pad['node_mask'], 'dropout_key': keys[i]}

  eager, opt_e = make()
  losses_e = []
  for i in range(6):
    a, kw = step_args(i)
    opt_e.zero_grad()
    _, loss = eager.forward_sparse_train(*a, **kw) if sparse else eager(*a, **kw)
    loss.backward()
    opt_e.step()
    losses_e.append(float(loss.detach()))
  graphed, opt_g = make()
  a, kw = step_args(0)
  step = GraphedStep(graphed, opt_g, a, kw, sparse=sparse)
  losses_g = []
  for i in range(6):
    a, kw = step_args(i)
    _, loss = step(*a, **kw)
    losses_g.append(float(loss.detach()))
  np.testing.assert_allclose(losses_g, losses_e, rtol=1e-5)
  for (n, p), (_, q) in zip(graphed.named_parameters(), eager.named_parameters()):
    np.testing.assert_allclose(p.detach().cpu().numpy(), q.detach().cpu().numpy(), rtol=2e-4, atol=2e-6, err_msg=n)
  # on the module's own key every replay draws new masks and advances the counter
  own, opt_o = make()
  a, kw = step_args(0)
  kw.pop('dropout_key', None)
  if sparse:
    a = ({k: v for k, v in a[0].items() if k != 'dropout_key'},)
  step = GraphedStep(own, opt_o, a, kw, sparse=sparse)
  c0 = own.dropout_key[1].item()
  with torch.no_grad():
    s1 = step(*a, **kw)[0].clone()
    s2 = step(*a, **kw)[0].clone()
  assert own.dropout_key[1].item() == c0 + 2 and not torch.equal(s1, s2)


def test_reference_training_loop_body_with_dropout_learns():
  """The loop body of QM8Runner.train (runner/qm8_runner.py:226-259) with dropout 0.1, on the class the
  drop-in binds under --opt-in GAT --keyed-dropout, through nn.DataParallel with Adam: the loss falls."""
  ns = types.ModuleType('fake_runner')
  ns.GAT = 'ref'
  dropin.patch_namespace(ns, training=True, opt_in=('GAT',), keyed_dropout=True)
  assert ns.GAT is KeyedGAT
  batch = data.synthetic_qm8_batch(64, seed=4)
  model = ns.GAT(configs.qm8_gat(dropout=0.1))
  model.load_state_dict(deterministic_state_dict(model, 1234))
  model = torch.nn.DataParallel(model, device_ids=[0]).cuda()
  optimizer = torch.optim.Adam(filter(lambda p: p.requires_grad, model.parameters()), lr=1.0e-3)
  t = {k: _t(v).cuda() for k, v in batch.items()}
  L = _t(data.gat_bias(batch['L'])).cuda()
  model.eval()
  with torch.no_grad():
    before = float(model(t['node_feat'], L, label=t['label'], mask=t['node_mask'])[1])
  losses = []
  for _ in range(40):
    model.train()
    optimizer.zero_grad()
    _, train_loss = model(t['node_feat'], L, label=t['label'], mask=t['node_mask'])
    train_loss.backward()
    optimizer.step()
    losses.append(float(train_loss))
  assert all(np.isfinite(losses))
  model.eval()
  with torch.no_grad():
    after = float(model(t['node_feat'], L, label=t['label'], mask=t['node_mask'])[1])
  assert after < before, (before, after, losses)
