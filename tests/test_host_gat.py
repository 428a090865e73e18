"""GAT drop-in, host side: the GAT collate's attention bias, the oracle against the reference's own
outputs (tests/golden/gat_qm8.npz, make_gat_golden.py), the module's parameter surface and its
refusals.  No GPU needed."""
import hashlib
import types

import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, data, dropin
from lanczosnetwork_b200.model import GAT
from oracle import gat_oracle

SMALL = dict(num_layer=2, num_heads=[3, 3], hidden_dim=[8, 8], output_dim=5)


def _spec(cfg):
  return gat_oracle.make_spec(cfg.model.num_layer, cfg.model.num_heads, cfg.dataset.num_bond_type)


def _params(cfg, seed):
  mod = GAT(cfg)
  return deterministic_state_dict(mod, seed)


def test_gat_bias_is_bit_identical_to_the_reference_collate():
  g, gg = load_golden('lanczosnet_qm8.npz'), load_golden('gat_qm8.npz')
  # from the collated operators of the same molecules, and from data.collate of prepare_graph records
  got = data.gat_bias(g['L'])
  assert got.dtype == np.float32 and got.shape == gg['L'].shape
  assert np.array_equal(got.view(np.uint32), gg['L'].view(np.uint32))      # -0.0 included
  samples = [data.prepare_graph(g['adjs'][b, :n, :n], g['node_feat'][b, :n])
             for b, n in enumerate(g['sizes'])]
  assert np.array_equal(data.gat_bias(data.collate(samples, 20)['L']).view(np.uint32),
                        gg['L'].view(np.uint32))
  assert np.array_equal(gat_oracle.adj_to_bias(g['L']).view(np.uint32), gg['L'].view(np.uint32))
  # exactly two values; padded nodes attend only to themselves
  assert set(np.unique(gg['L'].view(np.uint32)).tolist()) == {0x80000000, 0xCE6E6B28}
  n = int(g['sizes'][1])
  pad = gg['L'][1, n:, :, :]
  assert np.all(pad[np.arange(26 - n), np.arange(n, 26)].view(np.uint32) == 0x80000000)
  assert np.count_nonzero(pad == -1e9) == pad.size - (26 - n) * 7


def test_oracle_reproduces_the_reference_gat():
  gg = load_golden('gat_qm8.npz')
  cfg = configs.qm8_gat()
  params = _params(cfg, int(gg['weight_seed']))
  spec = _spec(cfg)
  for mask, key in ((gg['node_mask'], 'score'), (None, 'score_nomask')):
    s32 = gat_oracle.gat_forward(params, spec, gg['node_feat'], gg['L'], mask).numpy()
    np.testing.assert_allclose(s32, gg[key], rtol=1e-6, atol=1e-7)
    s64 = gat_oracle.gat_forward(params, spec, gg['node_feat'], gg['L'], mask, dtype=torch.float64).numpy()
    np.testing.assert_allclose(s64, gg[key], rtol=1e-4, atol=2e-5)
  s32 = gat_oracle.gat_forward(params, spec, gg['node_feat'], gg['L'], gg['node_mask'])
  loss = torch.nn.functional.mse_loss(s32, torch.from_numpy(gg['label']))
  assert abs(float(loss) - float(gg['loss'])) <= 1e-6 * abs(float(gg['loss']))
  cfg_s = configs.qm8_gat(**SMALL)
  params_s = _params(cfg_s, int(gg['weight_seed']) + 1)
  for mask, key in ((gg['node_mask'], 'score_small'), (None, 'score_small_nomask')):
    s32 = gat_oracle.gat_forward(params_s, _spec(cfg_s), gg['node_feat'], gg['L'], mask).numpy()
    np.testing.assert_allclose(s32, gg[key], rtol=1e-6, atol=1e-7)


def test_module_surface_matches_the_reference():
  gg = load_golden('gat_qm8.npz')
  cfg = configs.qm8_gat()
  m = GAT(cfg)
  assert sum(p.numel() for p in m.parameters()) == int(gg['num_params']) == 4898609
  assert list(m.state_dict().keys()) == gg['keys'].tolist()
  shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
  assert shapes['filter.0.0.0.weight'] == (16, 64) and shapes['filter.1.6.7.weight'] == (16, 896)
  assert shapes['att_net_1.3.2.1.weight'] == (1, 16) and shapes['output_func.0.weight'] == (16, 16)
  # every channel's state_bias is the parameter registered for the last bond channel
  assert all(m.state_bias[t][jj][ii] is getattr(m, 'bias_%d_6_%d' % (ii, t))
             for t in range(7) for jj in range(7) for ii in range(8))
  # same construction + initialisation order as the reference: same initial parameters
  torch.manual_seed(int(gg['init_seed']))
  init = GAT(cfg)
  h = hashlib.sha256()
  for name, t in init.state_dict().items():
    h.update(name.encode())
    h.update(t.detach().contiguous().numpy().tobytes())
  assert h.hexdigest() == str(gg['init_sha256'])
  # layer input width uses num_heads of the layer itself (model/gat.py:34-38)
  odd = GAT(configs.qm8_gat(num_layer=2, num_heads=[2, 5], hidden_dim=[4, 4], output_dim=3))
  assert odd.filter[1][0][0].weight.shape == (4, 4 * 5 * 7)


def test_only_the_last_channel_bias_is_read():
  gg = load_golden('gat_qm8.npz')
  cfg = configs.qm8_gat(**SMALL)
  params = _params(cfg, 5)
  spec = _spec(cfg)
  args = (gg['node_feat'], gg['L'], gg['node_mask'])
  base = gat_oracle.gat_forward(params, spec, *args)
  dead = dict(params)
  for t in range(2):
    for jj in range(6):
      for ii in range(3):
        dead['bias_%d_%d_%d' % (ii, jj, t)] = params['bias_%d_%d_%d' % (ii, jj, t)] + 3.0
  assert torch.equal(gat_oracle.gat_forward(dead, spec, *args), base)
  live = dict(params)
  live['bias_1_6_0'] = params['bias_1_6_0'] + 3.0
  assert not torch.equal(gat_oracle.gat_forward(live, spec, *args), base)


def test_refusals():
  with pytest.raises(ValueError):
    GAT(configs.qm8_gat(loss='hinge'))
  m = GAT(configs.qm8_gat(**SMALL))
  nf, L = torch.zeros(2, 4, dtype=torch.long), torch.zeros(2, 4, 4, 7)
  with pytest.raises(RuntimeError):            # CPU module: no fallback
    with torch.no_grad():
      m(nf, L)
  # autograd on with trainable parameters: there is no training path, the forward refuses
  with pytest.raises(NotImplementedError):
    m._check_mode()
  with torch.no_grad():
    assert m._check_mode() is False
  for p in m.parameters():
    p.requires_grad_(False)
  assert m._check_mode() is False


def test_dropin_rebinds_gat_for_test_runs_only():
  test_ns = types.ModuleType('fake_test_runner')
  test_ns.GAT = 'ref'
  dropin.patch_namespace(test_ns)
  assert test_ns.GAT is GAT
  train_ns = types.ModuleType('fake_train_runner')
  train_ns.GAT = 'ref'
  dropin.patch_namespace(train_ns, training=True)
  assert train_ns.GAT == 'ref'
  assert 'GAT' in dropin.DROPIN_CLASSES
