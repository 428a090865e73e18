"""GAT training path, host side: the fp64 oracle's autograd against the reference's own backward
(tests/golden/gat_train_grads.npz, make_gat_train_golden.py), TrainableGAT's parameter surface, the
opt-in drop-in binding and the dropout refusal.  No GPU needed."""
import types

import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, dropin
from lanczosnetwork_b200.model import GAT, TrainableGAT
from oracle import gat_oracle
import gat_train_oracle

SMALL = dict(num_layer=2, num_heads=[3, 3], hidden_dim=[8, 8], output_dim=5)
CASES = (('config', {}, 0), ('small', SMALL, 1))


def _spec(cfg):
  return gat_oracle.make_spec(cfg.model.num_layer, cfg.model.num_heads, cfg.dataset.num_bond_type)


@pytest.mark.parametrize('prefix,over,dseed', CASES, ids=['config', 'small'])
def test_oracle_fp64_autograd_reproduces_the_reference_gradients(prefix, over, dseed):
  """The reference ran in fp32; the bounds are those of the GGNN oracle, with scale = sqrt(sum of
  squares) of the gradient floored at 1e-3 of the largest parameter's.  The floor is for the att_net
  biases: c1 (c2) shifts the logits of a whole row (column) of the attention, which the column softmax
  cancels everywhere but across the leaky-ReLU kink, so their gradients are 1e-6 of the largest and
  carry relative fp32 rounding up to 1.5e-3 in the reference (measured: 2e-8 of the largest scale)."""
  gg, gt = load_golden('gat_qm8.npz'), load_golden('gat_train_grads.npz')
  cfg = configs.qm8_gat(**over)
  params = {k: v.double().requires_grad_(True)
            for k, v in deterministic_state_dict(GAT(cfg), int(gg['weight_seed']) + dseed).items()}
  score = gat_train_oracle.gat_forward(params, _spec(cfg), gg['node_feat'], gg['L'], gg['node_mask'])
  label = torch.from_numpy(gg['label'][:, :cfg.model.output_dim]).double()
  loss = torch.nn.functional.mse_loss(score, label)
  loss.backward()
  want_loss = float(gt['%s_loss' % prefix])
  assert abs(float(loss.detach()) - want_loss) <= 1e-5 * want_loss
  # the same names have no gradient: the bias_{ii}_{jj}_{t} with jj < E, never read
  none = sorted(k for k, p in params.items() if p.grad is None)
  assert none == gt['%s_none_grad' % prefix].tolist()
  E = cfg.dataset.num_bond_type
  assert all(int(k.split('_')[2]) < E for k in none) and len(none) == E * sum(cfg.model.num_heads)
  names = gt['%s_names' % prefix].tolist()
  digests = gt['%s_digests' % prefix]
  assert sorted(names + none) == sorted(params)
  floor = 1e-3 * float(np.sqrt(digests[:, 1].max()))
  for name, want in zip(names, digests):
    got = gat_train_oracle.grad_digest({name: params[name].grad})[name]
    n = min(8, params[name].numel())
    scale = max(np.sqrt(want[1]), floor)
    assert abs(got[0] - want[0]) <= 1e-4 * scale * np.sqrt(params[name].numel()), (name, got[0], want[0])
    assert abs(got[1] - want[1]) <= 3e-4 * max(want[1], scale * scale), (name, got[1], want[1])
    np.testing.assert_allclose(got[2:2 + n], want[2:2 + n], rtol=0, atol=1e-4 * scale, err_msg=name)
    assert np.all(np.isnan(want[2 + n:]))


def test_differentiable_oracle_computes_what_the_oracle_computes():
  """gat_train_oracle.gat_forward is oracle.gat_oracle.gat_forward without the cast: same scores, bit for
  bit, at both precisions, with and without the mask; and autograd reaches the caller's tensors."""
  gg = load_golden('gat_qm8.npz')
  cfg = configs.qm8_gat(**SMALL)
  base = deterministic_state_dict(GAT(cfg), 3)
  for dtype in (torch.float32, torch.float64):
    for mask in (gg['node_mask'], None):
      want = gat_oracle.gat_forward(base, _spec(cfg), gg['node_feat'], gg['L'], mask, dtype=dtype)
      params = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in base.items()}
      got = gat_train_oracle.gat_forward(params, _spec(cfg), gg['node_feat'], gg['L'], mask)
      assert got.dtype == dtype and got.requires_grad and torch.equal(got.detach(), want)
  got.sum().backward()
  assert params['filter.0.0.0.weight'].grad is not None and params['bias_0_5_0'].grad is None


def test_trainable_gat_has_the_surface_and_initial_weights_of_gat():
  for over in ({}, SMALL):
    cfg = configs.qm8_gat(**over)
    torch.manual_seed(1234)
    a = GAT(cfg)
    torch.manual_seed(1234)
    b = TrainableGAT(cfg)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa.keys()) == list(sb.keys())
    assert all(sa[k].shape == sb[k].shape and torch.equal(sa[k], sb[k]) for k in sa)
    # checkpoints load both ways
    b.load_state_dict(deterministic_state_dict(a, 7))
    a.load_state_dict(b.state_dict())
    assert all(torch.equal(x, y) for x, y in zip(a.state_dict().values(), b.state_dict().values()))
  assert isinstance(b, GAT) and hasattr(TrainableGAT, '_train_impl') and not hasattr(GAT, '_train_impl')


def test_trainable_gat_refuses_dropout_in_training():
  m = TrainableGAT(configs.qm8_gat(dropout=0.1, **SMALL)).train()
  nf, L = torch.zeros(2, 4, dtype=torch.long), torch.zeros(2, 4, 4, 7)
  for grad in (False, True):
    with torch.set_grad_enabled(grad):
      with pytest.raises(NotImplementedError, match='input, the attention weights and Wh'):
        m(nf, L)
  m.eval()
  with pytest.raises(RuntimeError, match='no CPU'):       # eval: no dropout, but no CPU path either
    with torch.no_grad():
      m(nf, L)
  assert TrainableGAT(configs.qm8_gat(**SMALL))._check_mode() is True


def test_dropin_binds_trainable_gat_only_when_opted_in():
  for training in (False, True):
    ns = types.ModuleType('fake_runner')
    ns.GAT, ns.MPNN = 'ref', 'ref'
    dropin.patch_namespace(ns, training=training)
    assert ns.GAT == ('ref' if training else GAT) and ns.MPNN == 'ref'
    dropin.patch_namespace(ns, training=training, opt_in=('GAT',))
    assert ns.GAT is TrainableGAT and ns.MPNN == 'ref'
    ns = types.ModuleType('fake_runner')
    ns.GAT, ns.MPNN = 'ref', 'ref'
    dropin.patch_namespace(ns, training=training, opt_in=('GAT', 'MPNN'))
    assert ns.GAT is TrainableGAT and ns.MPNN is dropin._models.MPNN
  assert dropin.TRAINING_OPT_IN_CLASSES == ('GAT',) and dropin.OPT_IN_CLASSES == ('MPNN',)
  assert 'GAT' in dropin.DROPIN_CLASSES
  with pytest.raises(ValueError, match='OPT_IN_CLASSES'):
    dropin.patch_namespace(types.ModuleType('x'), opt_in=('GGNN',))


def test_dropin_main_passes_the_gat_opt_in(monkeypatch):
  seen = {}
  monkeypatch.setattr(dropin, 'install', lambda root, **kw: seen.update(kw, root=root) or [])
  monkeypatch.setattr(dropin.os, 'chdir', lambda path: None)
  fake = types.ModuleType('run_exp')
  fake.main = lambda: seen.update(argv=list(dropin.sys.argv))
  monkeypatch.setitem(dropin.sys.modules, 'run_exp', fake)
  monkeypatch.setattr(dropin.sys, 'argv', ['x'])
  dropin.main(['/ref', '-c', 'config/qm8_gat.yaml', '--opt-in', 'GAT'])
  assert seen['opt_in'] == ['GAT'] and seen['training'] is True
  assert seen['argv'] == ['run_exp.py', '-c', 'config/qm8_gat.yaml']
