"""GraphSAGE drop-in, host side: the collate's neighbour samples, the gather-form oracle against the
reference's own outputs and gradients (tests/golden/graphsage_qm8.npz, make_graphsage_golden.py), the
module's parameter surface and its refusals.  No GPU needed."""
import hashlib
import types

import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, load_golden
from lanczosnetwork_b200 import configs, data, dropin
from lanczosnetwork_b200.model import GraphSAGE
from oracle import sage_oracle

SMALL = dict(num_layer=3, hidden_dim=[32, 32, 32], output_dim=5)


def _spec(cfg):
  return sage_oracle.make_spec(cfg.model.num_layer, cfg.model.agg_func, cfg.dataset.num_bond_type)


def _params(cfg, seed):
  return deterministic_state_dict(GraphSAGE(cfg), seed)


def _inputs(gg):
  return gg['node_feat'], gg['nn_idx'], gg['nonempty_mask']


def test_sage_collate_is_bit_identical_to_the_reference_collate():
  g, gg = load_golden('lanczosnet_qm8.npz'), load_golden('graphsage_qm8.npz')
  samples = [data.prepare_graph(g['adjs'][b, :n, :n], g['node_feat'][b, :n], g['label'][b:b + 1])
             for b, n in enumerate(g['sizes'])]
  got = data.sage_collate(samples, 40, np.random.RandomState(int(gg['collate_seed'])))
  for key in ('nn_idx', 'nonempty_mask', 'node_feat', 'node_mask', 'label'):
    assert got[key].dtype == gg[key].dtype and got[key].shape == gg[key].shape, key
    assert np.array_equal(got[key], gg[key]), key
  # the batch exercises both sampling branches and the padded rows
  n0 = int(g['sizes'][0])
  assert np.all(gg['nonempty_mask'][0, :n0] == 1)
  assert np.all(gg['nonempty_mask'][1, int(g['sizes'][1]):] == 0)
  assert np.all(gg['nn_idx'][1, int(g['sizes'][1]):] == 0)


@pytest.mark.parametrize('agg', ['Mean', 'Max'])
def test_oracle_reproduces_the_reference_scores_and_loss(agg):
  gg = load_golden('graphsage_qm8.npz')
  a = agg.lower()
  cases = [(configs.qm8_graphsage(agg_func=agg), int(gg['weight_seed']), '%s_score' % a, '%s_score_nomask' % a),
           (configs.qm8_graphsage(agg_func=agg, **SMALL), int(gg['weight_seed']) + 1, '%s_small' % a,
            '%s_small_nomask' % a)]
  for cfg, seed, k_mask, k_nomask in cases:
    params = _params(cfg, seed)
    for mask, key in ((gg['node_mask'], k_mask), (None, k_nomask)):
      s32 = sage_oracle.sage_forward(params, _spec(cfg), *_inputs(gg), mask).numpy()
      np.testing.assert_allclose(s32, gg[key], rtol=1e-6, atol=1e-7, err_msg=key)
      s64 = sage_oracle.sage_forward(params, _spec(cfg), *_inputs(gg), mask, dtype=torch.float64).numpy()
      np.testing.assert_allclose(s64, gg[key], rtol=1e-4, atol=2e-5, err_msg=key)
  if agg == 'Mean':
    cfg = configs.qm8_graphsage()
    s32 = sage_oracle.sage_forward(_params(cfg, int(gg['weight_seed'])), _spec(cfg), *_inputs(gg), gg['node_mask'])
    loss = torch.nn.functional.mse_loss(s32, torch.from_numpy(gg['label']))
    assert abs(float(loss) - float(gg['loss'])) <= 1e-6 * abs(float(gg['loss']))


@pytest.mark.parametrize('agg', ['Mean', 'Max'])
def test_oracle_fp64_autograd_reproduces_the_reference_gradients(agg):
  gg = load_golden('graphsage_qm8.npz')
  cfg = configs.qm8_graphsage(agg_func=agg)
  params = {k: v.double().requires_grad_(True) for k, v in _params(cfg, int(gg['weight_seed'])).items()}
  score = sage_oracle.sage_forward(params, _spec(cfg), *_inputs(gg), gg['node_mask'], dtype=torch.float64,
                                   cast=False)
  loss = torch.nn.functional.mse_loss(score, torch.from_numpy(gg['label']).double())
  loss.backward()
  a = agg.lower()
  assert abs(float(loss.detach()) - float(gg['grad_%s_loss' % a])) <= 1e-5 * float(gg['grad_%s_loss' % a])
  names = [k for k in gg if k.startswith('grad_%s|' % a)]
  assert len(names) == len(params) - 2                    # filter.6.{weight,bias} get no gradient
  assert params['filter.6.weight'].grad is None and params['filter.6.bias'].grad is None
  for k in names:
    name = k.split('|', 1)[1]
    want = gg[k]
    got = sage_oracle.grad_digest({name: params[name].grad})[name]
    # sum / sum of squares / leading entries; the reference ran in fp32
    scale = max(np.sqrt(want[1]), 1e-12)
    assert abs(got[0] - want[0]) <= 1e-4 * scale * np.sqrt(params[name].numel()), (k, got[0], want[0])
    assert abs(got[1] - want[1]) <= 1e-4 * want[1] + 1e-12, (k, got[1], want[1])
    np.testing.assert_allclose(got[2:], want[2:], rtol=1e-3, atol=1e-5 * scale, err_msg=k)


def test_module_surface_matches_the_reference():
  gg = load_golden('graphsage_qm8.npz')
  cfg = configs.qm8_graphsage()
  m = GraphSAGE(cfg)
  assert sum(p.numel() for p in m.parameters()) == int(gg['num_params']) == 753041
  assert list(m.state_dict().keys()) == gg['keys'].tolist()
  shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
  assert shapes['filter.0.weight'] == (128, 448) and shapes['filter.5.weight'] == (128, 896)
  assert shapes['filter.6.weight'] == (128, 896) and shapes['filter.7.weight'] == (16, 128)
  assert shapes['att_func.0.weight'] == (1, 128) and shapes['embedding.weight'] == (70, 64)
  torch.manual_seed(int(gg['init_seed']))
  init = GraphSAGE(cfg)
  h = hashlib.sha256()
  for name, t in init.state_dict().items():
    h.update(name.encode())
    h.update(t.detach().contiguous().numpy().tobytes())
  assert h.hexdigest() == str(gg['init_sha256'])


def test_filter_of_the_last_hidden_layer_is_never_read():
  gg = load_golden('graphsage_qm8.npz')
  cfg = configs.qm8_graphsage(agg_func='Max', **SMALL)
  params = _params(cfg, 5)
  base = sage_oracle.sage_forward(params, _spec(cfg), *_inputs(gg), gg['node_mask'])
  dead = dict(params)
  dead['filter.2.weight'] = params['filter.2.weight'] + 3.0
  dead['filter.2.bias'] = params['filter.2.bias'] + 3.0
  assert torch.equal(sage_oracle.sage_forward(dead, _spec(cfg), *_inputs(gg), gg['node_mask']), base)
  live = dict(params)
  live['filter.3.bias'] = params['filter.3.bias'] + 3.0
  assert not torch.equal(sage_oracle.sage_forward(live, _spec(cfg), *_inputs(gg), gg['node_mask']), base)


def test_refusals():
  state = torch.random.get_rng_state()
  with pytest.raises(NotImplementedError, match='Mean, Max'):
    GraphSAGE(configs.qm8_graphsage(agg_func='LSTM'))
  assert torch.equal(torch.random.get_rng_state(), state)     # refused before any random draw
  with pytest.raises(ValueError):
    GraphSAGE(configs.qm8_graphsage(loss='hinge'))
  m = GraphSAGE(configs.qm8_graphsage(**SMALL))
  nf, nn_idx, ne = torch.zeros(2, 4, dtype=torch.long), torch.zeros(2, 4, 40, 7, dtype=torch.long), torch.ones(2, 4, 1)
  with pytest.raises(RuntimeError):            # CPU module: no fallback
    with torch.no_grad():
      m(nf, nn_idx, ne)
  # an unknown aggregator constructs (as in the reference) and has no aggregation function
  odd = GraphSAGE(configs.qm8_graphsage(agg_func='Sum', **SMALL))
  assert odd.agg_func is None


def test_dropin_rebinds_graphsage_for_test_and_training_runs():
  for training in (False, True):
    ns = types.ModuleType('fake_runner')
    ns.GraphSAGE = 'ref'
    dropin.patch_namespace(ns, training=training)
    assert ns.GraphSAGE is GraphSAGE
  assert 'GraphSAGE' in dropin.DROPIN_CLASSES
