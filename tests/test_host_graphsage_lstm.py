"""LSTM GraphSAGE, host side: the module's construction against the executed reference
(tests/golden/graphsage_lstm_qm8.npz, make_graphsage_lstm_golden.py), the fp64 oracle against the
reference's scores, loss and gradients, the gate re-layout, the opt-in binding and the refusals.  No GPU
needed."""
import hashlib
import os
import types

import numpy as np
import pytest
import torch

import sage_lstm_oracle as lo
from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, dropin
from lanczosnetwork_b200.model import GraphSAGE, LSTMGraphSAGE
from lanczosnetwork_b200.model.graph_sage import lstm_gate_matrix, lstm_gate_matrix_inverse

SMALL = dict(num_layer=3, hidden_dim=[32, 32, 32], output_dim=5)


def _spec(cfg):
  return lo.make_spec(cfg.model.num_layer, cfg.model.agg_func, cfg.dataset.num_bond_type)


def _params(cfg, seed):
  return deterministic_state_dict(LSTMGraphSAGE(cfg), seed)


def _inputs(gg):
  return gg['node_feat'], gg['nn_idx'], gg['nonempty_mask']


def test_construction_matches_the_reference():
  gg = load_golden('graphsage_lstm_qm8.npz')
  cfg = configs.qm8_graphsage(agg_func='LSTM')
  torch.manual_seed(int(gg['init_seed']))
  m = LSTMGraphSAGE(cfg)
  sd = m.state_dict()
  assert list(sd.keys()) == gg['keys'].tolist()
  assert [list(v.shape) + [0] * (2 - v.dim()) for v in sd.values()] == gg['shapes'].tolist()
  assert sum(p.numel() for p in m.parameters()) == int(gg['num_params'])
  assert sd['agg_func.0.weight_ih'].shape == (256, 64) and sd['agg_func.5.weight_hh'].shape == (512, 128)
  h = hashlib.sha256()
  for name, t in sd.items():
    h.update(name.encode())
    h.update(t.detach().contiguous().numpy().tobytes())
  assert h.hexdigest() == str(gg['init_sha256'])
  assert m.agg_func[0].bias_ih.abs().sum() == 0          # the reference zeroes the cell biases


def test_mean_and_max_construct_exactly_like_graphsage():
  for agg in ('Mean', 'Max'):
    cfg = configs.qm8_graphsage(agg_func=agg)
    torch.manual_seed(7)
    a = GraphSAGE(cfg).state_dict()
    torch.manual_seed(7)
    b = LSTMGraphSAGE(cfg).state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


def test_oracle_reproduces_the_reference_scores_and_loss():
  gg = load_golden('graphsage_lstm_qm8.npz')
  seed = int(gg['weight_seed'])
  cases = [(configs.qm8_graphsage(agg_func='LSTM'), seed, 'score'),
           (configs.qm8_graphsage(agg_func='LSTM', **SMALL), seed + 1, 'small')]
  for cfg, s, key in cases:
    params = _params(cfg, s)
    for mask, k in ((gg['node_mask'], key), (None, key + '_nomask')):
      s32 = lo.sage_lstm_forward(params, _spec(cfg), *_inputs(gg), mask).numpy()
      np.testing.assert_allclose(s32, gg[k], rtol=1e-5, atol=1e-7, err_msg=k)
      s64 = lo.sage_lstm_forward(params, _spec(cfg), *_inputs(gg), mask, dtype=torch.float64).numpy()
      np.testing.assert_allclose(s64, gg[k], rtol=1e-4, atol=2e-6, err_msg=k)
  cfg = configs.qm8_graphsage(agg_func='LSTM')
  s64 = lo.sage_lstm_forward(_params(cfg, seed), _spec(cfg), *_inputs(gg), gg['node_mask'], dtype=torch.float64)
  loss = torch.nn.functional.mse_loss(s64, torch.from_numpy(gg['label']).double())
  assert abs(float(loss) - float(gg['loss'])) <= 1e-5 * abs(float(gg['loss']))


def test_oracle_fp64_autograd_reproduces_the_reference_gradients():
  gg = load_golden('graphsage_lstm_qm8.npz')
  cfg = configs.qm8_graphsage(agg_func='LSTM')
  params = {k: v.double().requires_grad_(True) for k, v in _params(cfg, int(gg['weight_seed'])).items()}
  score = lo.sage_lstm_forward(params, _spec(cfg), *_inputs(gg), gg['node_mask'], dtype=torch.float64, cast=False)
  loss = torch.nn.functional.mse_loss(score, torch.from_numpy(gg['label']).double())
  loss.backward()
  assert abs(float(loss.detach()) - float(gg['grad_loss'])) <= 1e-5 * float(gg['grad_loss'])
  names = [k for k in gg if k.startswith('grad|')]
  assert len(names) == len(params) - 2                    # filter.6.{weight,bias} get no gradient
  assert params['filter.6.weight'].grad is None and params['filter.6.bias'].grad is None
  for k in names:
    name = k.split('|', 1)[1]
    want, got = gg[k], lo.grad_digest({name: params[name].grad})[name]
    scale = max(np.sqrt(want[1]), 1e-12)
    assert abs(got[0] - want[0]) <= 1e-4 * scale * np.sqrt(params[name].numel()), (k, got[0], want[0])
    assert abs(got[1] - want[1]) <= 1e-4 * want[1] + 1e-12, (k, got[1], want[1])
    np.testing.assert_allclose(got[2:], want[2:], rtol=1e-3, atol=1e-5 * scale, err_msg=k)


def test_quirks_of_the_reference():
  gg = load_golden('graphsage_lstm_qm8.npz')
  cfg = configs.qm8_graphsage(agg_func='LSTM', **SMALL)
  params = _params(cfg, 5)
  nf, nn_idx, ne = _inputs(gg)
  base = lo.sage_lstm_forward(params, _spec(cfg), nf, nn_idx, ne, gg['node_mask'])
  # filter[num_layer - 1] is registered but never read
  dead = dict(params, **{'filter.2.weight': params['filter.2.weight'] + 3.0})
  assert torch.equal(lo.sage_lstm_forward(dead, _spec(cfg), nf, nn_idx, ne, gg['node_mask']), base)
  # a padded row (nonempty = 0) gives a zero message whatever its samples are
  pad = np.argwhere(ne[:, :, 0] == 0)
  assert len(pad) > 0
  moved = nn_idx.copy()
  moved[pad[:, 0], pad[:, 1]] = 3
  assert torch.equal(lo.sage_lstm_forward(params, _spec(cfg), nf, moved, ne, gg['node_mask']), base)
  # a live node with an empty channel runs the LSTM over node 0 K times: its samples are all 0
  live = ne[:, :, 0] != 0
  empty = (nn_idx == 0).all(axis=2) & live[:, :, None]
  assert empty.any()


def test_gate_relayout_inverts_exactly():
  torch.manual_seed(3)
  for D in (32, 64, 96, 128):
    cell = torch.nn.LSTMCell(D, D)
    W, b = lstm_gate_matrix(cell.weight_ih.detach(), cell.weight_hh.detach(), cell.bias_ih.detach(),
                            cell.bias_hh.detach())
    assert W.shape == (4 * D, 2 * D) and b.shape == (4 * D,)
    wi, wh, bs = lstm_gate_matrix_inverse(W, b)
    assert torch.equal(wi, cell.weight_ih) and torch.equal(wh, cell.weight_hh)
    assert torch.equal(bs, cell.bias_ih + cell.bias_hh)
    # row (u // 4) * 16 + g * 4 + u % 4 is gate g of hidden unit u
    for u, g in ((0, 0), (5, 2), (D - 1, 3)):
      assert torch.equal(W[(u // 4) * 16 + g * 4 + u % 4, :D], cell.weight_ih[g * D + u])


def test_opt_in_binds_lstm_graphsage_and_graphsage_still_refuses():
  for training in (False, True):
    ns = types.ModuleType('fake_runner')
    ns.GraphSAGE = 'ref'
    dropin.patch_namespace(ns, training=training, opt_in=('GraphSAGE',))
    assert ns.GraphSAGE is LSTMGraphSAGE
    ns.GraphSAGE = 'ref'
    dropin.patch_namespace(ns, training=training)
    assert ns.GraphSAGE is GraphSAGE
  assert dropin.LSTM_OPT_IN_CLASSES == ('GraphSAGE',)
  assert dropin.OPT_IN_CLASSES == ('MPNN',) and dropin.TRAINING_OPT_IN_CLASSES == ('GAT',)
  with pytest.raises(ValueError, match='OPT_IN_CLASSES'):
    dropin.patch_namespace(types.ModuleType('x'), opt_in=('GGNN',))
  state = torch.random.get_rng_state()
  with pytest.raises(NotImplementedError, match='Mean, Max'):
    GraphSAGE(configs.qm8_graphsage(agg_func='LSTM'))
  assert torch.equal(torch.random.get_rng_state(), state)


def test_dropin_main_passes_the_graphsage_opt_in(monkeypatch):
  seen = {}
  monkeypatch.setattr(dropin, 'install', lambda root, **kw: seen.update(kw, root=root) or [])
  monkeypatch.setattr(dropin.os, 'chdir', lambda path: None)
  fake = types.ModuleType('run_exp')
  fake.main = lambda: seen.update(argv=list(dropin.sys.argv))
  monkeypatch.setitem(dropin.sys.modules, 'run_exp', fake)
  monkeypatch.setattr(dropin.sys, 'argv', ['x'])
  dropin.main(['/ref', '-c', 'config/qm8_graphsage.yaml', '--opt-in', 'GraphSAGE', '-t'])
  assert seen['opt_in'] == ['GraphSAGE'] and seen['training'] is False
  assert seen['argv'] == ['run_exp.py', '-c', 'config/qm8_graphsage.yaml', '-t']


def test_cpu_module_refuses_to_run():
  m = LSTMGraphSAGE(configs.qm8_graphsage(agg_func='LSTM', **SMALL))
  nf, nn_idx, ne = torch.zeros(2, 4, dtype=torch.long), torch.zeros(2, 4, 40, 7, dtype=torch.long), torch.ones(2, 4, 1)
  with pytest.raises(RuntimeError, match='CUDA'):
    with torch.no_grad():
      m(nf, nn_idx, ne)
  with pytest.raises(RuntimeError, match='CUDA'):
    m(nf, nn_idx, ne)


def test_step_kernel_sass_keeps_one_wgmma_group_queued():
  """sage_lstm_step_kernel is the skeleton's body under its own name: like every tc_gemm_kernel
  instantiation without acc_init() it issues its wgmma asynchronously (one WARPGROUP.ARRIVE per group of
  12 HGMMA) and keeps one group queued across k-blocks (wait_group 1)."""
  import re
  import shutil
  import subprocess
  from lanczosnetwork_b200 import build
  lib = build.build()
  tool = os.path.join(os.path.dirname(build.nvcc_path()), 'cuobjdump')
  tool = tool if os.path.exists(tool) else shutil.which('cuobjdump')
  assert tool is not None, 'cuobjdump not found next to nvcc or on PATH'
  text = subprocess.run([tool, '-sass', lib], check=True, capture_output=True, text=True).stdout
  parts = re.split(r'\n\s*Function : (\S+)\n', text)
  bodies = [body for name, body in zip(parts[1::2], parts[2::2]) if 'sage_lstm_step_kernel' in name]
  assert len(bodies) == 1
  n_mma = len(re.findall(r'\bHGMMA\.', bodies[0]))
  n_arrive = len(re.findall(r'\bWARPGROUP\.ARRIVE\b', bodies[0]))
  assert n_mma >= 12 and n_arrive * 12 <= n_mma, (n_mma, n_arrive)
  assert 'WARPGROUP.DEPBAR.LE gsb0, 0x1' in bodies[0]
