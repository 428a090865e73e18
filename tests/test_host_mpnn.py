"""MPNN drop-in, host side: the oracle against the reference's own outputs and gradients
(tests/golden/mpnn_qm8.npz, make_mpnn_golden.py), the module's parameter surface, its refusals and the
opt-in drop-in rebinding.  No GPU needed."""
import hashlib
import types

import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, dropin
from lanczosnetwork_b200.model import MPNN
from oracle import mpnn_oracle

SMALL = dict(msg_func='embedding', aggregate_type='sum', hidden_dim=32, num_prop=3, num_step_set2vec=3)
CASES = (('config', {}, 0), ('small', SMALL, 1))


def _spec(cfg):
  m = cfg.model
  return mpnn_oracle.make_spec(m.num_prop, m.aggregate_type, m.msg_func, cfg.dataset.num_bond_type,
                               m.num_step_set2vec)


def _params(cfg, seed):
  return deterministic_state_dict(MPNN(cfg), seed)


@pytest.mark.parametrize('prefix,over,dseed', CASES, ids=['config', 'small'])
def test_oracle_reproduces_the_reference_scores_and_loss(prefix, over, dseed):
  g, gm = load_golden('lanczosnet_qm8.npz'), load_golden('mpnn_qm8.npz')
  cfg = configs.qm8_mpnn(**over)
  params = _params(cfg, int(gm['weight_seed']) + dseed)
  L = g['L'].copy()
  for mask, key in ((g['node_mask'], '%s_score' % prefix), (None, '%s_score_nomask' % prefix)):
    s32 = mpnn_oracle.mpnn_forward(params, _spec(cfg), g['node_feat'], L, mask)
    np.testing.assert_allclose(s32.numpy(), gm[key], rtol=1e-5, atol=1e-6, err_msg=key)
    s64 = mpnn_oracle.mpnn_forward(params, _spec(cfg), g['node_feat'], L, mask, dtype=torch.float64)
    np.testing.assert_allclose(s64.numpy(), gm[key], rtol=1e-4, atol=2e-5, err_msg=key)
    if mask is not None:
      loss = torch.nn.functional.mse_loss(s32, torch.from_numpy(g['label']))
      want = float(gm['%s_loss' % prefix])
      assert abs(float(loss) - want) <= 1e-5 * abs(want)
  assert np.array_equal(L, g['L'])                          # the oracle reads the pattern, L is untouched


@pytest.mark.parametrize('prefix,over,dseed', CASES, ids=['config', 'small'])
def test_oracle_fp64_autograd_reproduces_the_reference_gradients(prefix, over, dseed):
  """The reference ran in fp32, so its digests carry fp32 rounding; the bounds are those of the GGNN
  oracle (scale = sqrt(sum of squares) of the gradient)."""
  g, gm = load_golden('lanczosnet_qm8.npz'), load_golden('mpnn_qm8.npz')
  cfg = configs.qm8_mpnn(**over)
  params = {k: v.double().requires_grad_(True) for k, v in _params(cfg, int(gm['weight_seed']) + dseed).items()}
  score = mpnn_oracle.mpnn_forward(params, _spec(cfg), g['node_feat'], g['L'], g['node_mask'],
                                   dtype=torch.float64, cast=False)
  loss = torch.nn.functional.mse_loss(score, torch.from_numpy(g['label']).double())
  loss.backward()
  want_loss = float(gm['grad_%s_loss' % prefix])
  assert abs(float(loss.detach()) - want_loss) <= 1e-5 * want_loss
  names = [k for k in gm if k.startswith('grad_%s|' % prefix)]
  assert sorted(k.split('|', 1)[1] for k in names) == sorted(params)
  for k in names:
    name = k.split('|', 1)[1]
    want = gm[k]
    got = mpnn_oracle.grad_digest({name: params[name].grad})[name]
    scale = max(np.sqrt(want[1]), 1e-12)
    assert abs(got[0] - want[0]) <= 1e-4 * scale * np.sqrt(params[name].numel()), (k, got[0], want[0])
    assert abs(got[1] - want[1]) <= 3e-4 * want[1] + 1e-12, (k, got[1], want[1])
    np.testing.assert_allclose(got[2:], want[2:], rtol=0, atol=1e-4 * scale, err_msg=k)


def test_module_surface_matches_the_reference():
  gm = load_golden('mpnn_qm8.npz')
  cfg = configs.qm8_mpnn()
  m = MPNN(cfg)
  keys = list(m.state_dict().keys())
  assert keys == gm['keys'].tolist()
  assert sum(p.numel() for p in m.parameters()) == int(gm['num_params'])
  # Set2Vec's own parameters come before those of its LSTM
  assert keys.index('att_func.W_1') < keys.index('att_func.W_2') < keys.index('att_func.LSTM.forget_gate.0.weight')
  shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
  assert shapes['update_func.weight_ih'] == (384, 896) and shapes['update_func.weight_hh'] == (384, 128)
  assert shapes['edge_func.6.0.weight'] == (64, 256) and shapes['edge_func.6.2.weight'] == (128, 64)
  assert shapes['att_func.W_1'] == (128, 128) and shapes['att_func.W_2'] == (128, 1)
  assert shapes['att_func.LSTM.memory_gate.0.weight'] == (128, 256)
  assert shapes['output_func.0.weight'] == (16, 256) and shapes['node_embedding.weight'] == (70, 64)
  torch.manual_seed(int(gm['init_seed']))
  init = MPNN(cfg)
  h = hashlib.sha256()
  for name, t in init.state_dict().items():
    h.update(name.encode())
    h.update(t.detach().contiguous().numpy().tobytes())
  assert h.hexdigest() == str(gm['init_sha256'])
  # the edge network keeps PyTorch's default initialisation, the GRU and gate biases are zero
  assert init.edge_func[0][0].bias.abs().sum() > 0
  assert not init.update_func.bias_ih.any() and not init.att_func.LSTM.forget_gate[0].bias.any()
  small = {k: tuple(v.shape) for k, v in MPNN(configs.qm8_mpnn(**SMALL)).state_dict().items()}
  assert small['edge_embedding.weight'] == (7, 32 * 32) and not any(k.startswith('edge_func') for k in small)


def test_refusals():
  with pytest.raises(AssertionError):
    MPNN(configs.qm8_mpnn(num_layer=2))
  with pytest.raises(AssertionError):
    MPNN(configs.qm8_mpnn(aggregate_type='max'))
  with pytest.raises(ValueError, match='Non-supported message function'):
    MPNN(configs.qm8_mpnn(msg_func='GRU'))
  with pytest.raises(ValueError):
    MPNN(configs.qm8_mpnn(loss='hinge'))
  nf, L = torch.zeros(2, 4, dtype=torch.long), torch.zeros(2, 4, 4, 7)
  m = MPNN(configs.qm8_mpnn(**SMALL))
  for grad in (False, True):                      # CPU module: no fallback, in inference or training
    with pytest.raises(RuntimeError, match='no CPU'):
      with torch.set_grad_enabled(grad):
        m(nf, L)


def test_dropin_leaves_mpnn_alone_unless_opted_in():
  for training in (False, True):
    ns = types.ModuleType('fake_runner')
    ns.MPNN, ns.GGNN = 'ref', 'ref'
    dropin.patch_namespace(ns, training=training)
    assert ns.MPNN == 'ref' and ns.GGNN != 'ref'
    dropin.patch_namespace(ns, training=training, opt_in=('MPNN',))
    assert ns.MPNN is MPNN
  assert 'MPNN' not in dropin.DROPIN_CLASSES and dropin.OPT_IN_CLASSES == ('MPNN',)
  with pytest.raises(ValueError, match='OPT_IN_CLASSES'):
    dropin.patch_namespace(types.ModuleType('x'), opt_in=('GPNN',))
  with pytest.raises(ValueError, match='OPT_IN_CLASSES'):
    dropin.install(None, runner_modules=(), opt_in=('LanczosNet',))


def test_dropin_main_strips_the_opt_in_flag(monkeypatch):
  seen = {}
  monkeypatch.setattr(dropin, 'install', lambda root, **kw: seen.update(kw, root=root) or [])
  monkeypatch.setattr(dropin.os, 'chdir', lambda path: None)
  fake = types.ModuleType('run_exp')
  fake.main = lambda: seen.update(argv=list(dropin.sys.argv))
  monkeypatch.setitem(dropin.sys.modules, 'run_exp', fake)
  monkeypatch.setattr(dropin.sys, 'argv', ['x'])
  dropin.main(['/ref', '-c', 'config/qm8_mpnn.yaml', '--opt-in', 'MPNN', '-t'])
  assert seen['opt_in'] == ['MPNN'] and seen['training'] is False and seen['root'] == '/ref'
  assert seen['argv'] == ['run_exp.py', '-c', 'config/qm8_mpnn.yaml', '-t']
