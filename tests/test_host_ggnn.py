"""GGNN drop-in, host side: the oracle against the reference's own outputs and gradients
(tests/golden/ggnn_qm8.npz, make_ggnn_golden.py), the re-laid-out GRU gate matrix, the module's parameter
surface and its refusals.  No GPU needed."""
import hashlib
import types

import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, dropin
from lanczosnetwork_b200.model import GGNN
from lanczosnetwork_b200.model.ggnn import gru_gate_matrix
from oracle import ggnn_oracle

SMALL = dict(hidden_dim=32, num_prop=3, aggregate_type='sum', update_func='RNN', output_dim=16)
CASES = (('config', {}, 0), ('small', SMALL, 1))


def _spec(cfg):
  m = cfg.model
  return ggnn_oracle.make_spec(m.num_prop, m.aggregate_type, m.update_func, cfg.dataset.num_bond_type)


def _params(cfg, seed):
  return deterministic_state_dict(GGNN(cfg), seed)


@pytest.mark.parametrize('prefix,over,dseed', CASES, ids=['config', 'small'])
def test_oracle_reproduces_the_reference_scores_and_loss(prefix, over, dseed):
  g, gg = load_golden('lanczosnet_qm8.npz'), load_golden('ggnn_qm8.npz')
  cfg = configs.qm8_ggnn(**over)
  params = _params(cfg, int(gg['weight_seed']) + dseed)
  L = g['L'].copy()
  for mask, key in ((g['node_mask'], '%s_score' % prefix), (None, '%s_score_nomask' % prefix)):
    s32 = ggnn_oracle.ggnn_forward(params, _spec(cfg), g['node_feat'], L, mask)
    np.testing.assert_allclose(s32.numpy(), gg[key], rtol=1e-6, atol=1e-7, err_msg=key)
    s64 = ggnn_oracle.ggnn_forward(params, _spec(cfg), g['node_feat'], L, mask, dtype=torch.float64)
    np.testing.assert_allclose(s64.numpy(), gg[key], rtol=1e-4, atol=2e-5, err_msg=key)
    if mask is not None:
      loss = torch.nn.functional.mse_loss(s32, torch.from_numpy(g['label']))
      want = float(gg['%s_loss' % prefix])
      assert abs(float(loss) - want) <= 1e-6 * abs(want)
  assert np.array_equal(L, g['L'])                          # the oracle binarises a copy


@pytest.mark.parametrize('prefix,over,dseed', CASES, ids=['config', 'small'])
def test_oracle_fp64_autograd_reproduces_the_reference_gradients(prefix, over, dseed):
  """The reference ran in fp32, so its digests carry fp32 rounding through 15 (3) recurrent steps.
  Measured worst cases over every parameter, with scale = sqrt(sum of squares) of the gradient:
  config (15 steps) -- sum within 1.1e-5 of scale * sqrt(numel), sum of squares within 3.7e-5
  relative, leading entries within 1.7e-5 of scale; small (3 steps) -- 5.6e-8, 3.0e-7, 8.6e-8.  The
  bounds below leave 6-10x room over the config case."""
  g, gg = load_golden('lanczosnet_qm8.npz'), load_golden('ggnn_qm8.npz')
  cfg = configs.qm8_ggnn(**over)
  params = {k: v.double().requires_grad_(True) for k, v in _params(cfg, int(gg['weight_seed']) + dseed).items()}
  score = ggnn_oracle.ggnn_forward(params, _spec(cfg), g['node_feat'], g['L'], g['node_mask'],
                                   dtype=torch.float64, cast=False)
  loss = torch.nn.functional.mse_loss(score, torch.from_numpy(g['label']).double())
  loss.backward()
  want_loss = float(gg['grad_%s_loss' % prefix])
  assert abs(float(loss.detach()) - want_loss) <= 1e-5 * want_loss
  names = [k for k in gg if k.startswith('grad_%s|' % prefix)]
  assert sorted(k.split('|', 1)[1] for k in names) == sorted(params)
  for k in names:
    name = k.split('|', 1)[1]
    want = gg[k]
    got = ggnn_oracle.grad_digest({name: params[name].grad})[name]
    scale = max(np.sqrt(want[1]), 1e-12)
    assert abs(got[0] - want[0]) <= 1e-4 * scale * np.sqrt(params[name].numel()), (k, got[0], want[0])
    assert abs(got[1] - want[1]) <= 3e-4 * want[1] + 1e-12, (k, got[1], want[1])
    np.testing.assert_allclose(got[2:], want[2:], rtol=0, atol=1e-4 * scale, err_msg=k)


def test_module_surface_matches_the_reference():
  gg = load_golden('ggnn_qm8.npz')
  cfg = configs.qm8_ggnn()
  m = GGNN(cfg)
  assert sum(p.numel() for p in m.parameters()) == int(gg['num_params']) == 640145
  assert list(m.state_dict().keys()) == gg['keys'].tolist()
  shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
  assert shapes['update_func.weight_ih'] == (384, 896) and shapes['update_func.weight_hh'] == (384, 128)
  assert shapes['msg_func.6.0.weight'] == (128, 128) and shapes['msg_func.6.2.weight'] == (128, 128)
  assert shapes['input_func.0.weight'] == (128, 64) and shapes['output_func.0.weight'] == (16, 128)
  assert shapes['embedding.weight'] == (70, 64) and shapes['att_func.0.weight'] == (1, 128)
  torch.manual_seed(int(gg['init_seed']))
  init = GGNN(cfg)
  h = hashlib.sha256()
  for name, t in init.state_dict().items():
    h.update(name.encode())
    h.update(t.detach().contiguous().numpy().tobytes())
  assert h.hexdigest() == str(gg['init_sha256'])
  # the message MLPs keep PyTorch's default initialisation (non-zero biases), the GRU biases are zero
  assert init.msg_func[0][0].bias.abs().sum() > 0
  assert not init.update_func.bias_ih.any() and not init.update_func.bias_hh.any()


def test_gate_matrix_reproduces_the_gru_cell():
  """[x | h] @ W^T + b with the interleaved gate rows, evaluated in numpy, gives torch's GRUCell."""
  rng = np.random.RandomState(0)
  for D, Din in ((32, 32), (64, 7 * 64), (128, 2 * 128)):
    cell = torch.nn.GRUCell(Din, D).double()
    with torch.no_grad():
      for prm in cell.parameters():
        prm.copy_(torch.from_numpy(rng.uniform(-0.3, 0.3, size=tuple(prm.shape))))
    x, h = rng.randn(5, Din), rng.randn(5, D)
    W, b = [t.detach().numpy() for t in gru_gate_matrix(cell.weight_ih, cell.weight_hh, cell.bias_ih,
                                                          cell.bias_hh)]
    assert W.shape == (4 * D, Din + D) and b.shape == (4 * D,)
    G = np.concatenate([x, h], axis=1) @ W.T + b                     # [5, 4D]
    u = np.arange(D)
    row = lambda gate: (u // 4) * 16 + gate * 4 + u % 4
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    r, z = sig(G[:, row(0)]), sig(G[:, row(1)])
    n = np.tanh(G[:, row(2)] + r * G[:, row(3)])
    got = (1.0 - z) * n + z * h
    want = cell(torch.from_numpy(x), torch.from_numpy(h)).detach().numpy()
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
    # the n_in block is zero over the h columns, the n_h block over the message columns
    assert not W[row(2), Din:].any() and not W[row(3), :Din].any()


def test_refusals():
  with pytest.raises(AssertionError):
    GGNN(configs.qm8_ggnn(num_layer=2))
  with pytest.raises(AssertionError):
    GGNN(configs.qm8_ggnn(aggregate_type='max'))
  with pytest.raises(ValueError):
    GGNN(configs.qm8_ggnn(loss='hinge'))
  nf, L = torch.zeros(2, 4, dtype=torch.long), torch.zeros(2, 4, 4, 7)
  m = GGNN(configs.qm8_ggnn(**SMALL))
  with pytest.raises(RuntimeError):              # CPU module: no fallback
    with torch.no_grad():
      m(nf, L)
  # update_func 'MLP': the reference's parameters, and its TypeError before the device is looked at
  mlp = GGNN(configs.qm8_ggnn(update_func='MLP'))
  shapes = {k: tuple(v.shape) for k, v in mlp.state_dict().items()}
  assert shapes['update_func.0.weight'] == (128, 896) and 'update_func.weight_ih' not in shapes
  assert list(shapes)[:3] == ['embedding.weight', 'update_func.0.weight', 'update_func.0.bias']
  with pytest.raises(TypeError, match='2 positional arguments but 3'):
    with torch.no_grad():
      mlp(nf, L)


def test_dropin_rebinds_ggnn_for_test_and_training_runs():
  for training in (False, True):
    ns = types.ModuleType('fake_runner')
    ns.GGNN = 'ref'
    dropin.patch_namespace(ns, training=training)
    assert ns.GGNN is GGNN
  assert 'GGNN' in dropin.DROPIN_CLASSES
