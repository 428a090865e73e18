"""Reproducible training under torch.use_deterministic_algorithms(True), with torch's NaN fill of
uninitialised memory left on: two independently built copies of every trainable drop-in, loaded from the
same weights, end bit-equal after the same Adam steps -- eager, in a GraphedStep (padded, sparse=True and
packed=True wherever the model takes them), and across grid sizes of the persistent kernels."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import _lib, configs, data, train
from lanczosnetwork_b200.model import (DCNN, GCN, GCNFP, GGNN, GPNN, MPNN, AdaLanczosNet, ChebyNet, GraphSAGE,
                                       KeyedAdaLanczosNet, KeyedGAT, LanczosNet, LSTMGraphSAGE,
                                       SampledGraphSAGE, SparseLanczosNetGeneral, TrainableGAT)

from helpers import deterministic_state_dict

pytestmark = pytest.mark.gpu

K = 20
B = 32

# name -> (constructor, inputs): 'ids' data.collate of QM8 molecules, 'sage' data.sage_collate of them,
# 'feat' data.collate of float-feature graphs (SparseLanczosNetGeneral is LanczosNetGeneral with the records
# entries), 'records' data.sparse_collate records only
MODELS = {
    'LanczosNet': (lambda: LanczosNet(configs.qm8_lanczos_net()), 'ids'),
    'LanczosNetGeneral': (lambda: SparseLanczosNetGeneral(configs.graph_lanczos_net()), 'feat'),
    'AdaLanczosNet': (lambda: AdaLanczosNet(configs.qm8_ada_lanczos_net()), 'ids'),
    'KeyedAdaLanczosNet': (lambda: KeyedAdaLanczosNet(configs.qm8_ada_lanczos_net()), 'ids'),
    'GCN': (lambda: GCN(configs.qm8_gcn()), 'ids'),
    'GCNFP': (lambda: GCNFP(configs.qm8_gcn()), 'ids'),
    'DCNN': (lambda: DCNN(configs.qm8_dcnn()), 'ids'),
    'ChebyNet': (lambda: ChebyNet(configs.qm8_cheby_net()), 'ids'),
    'TrainableGAT': (lambda: TrainableGAT(configs.qm8_gat()), 'ids'),
    'KeyedGAT': (lambda: KeyedGAT(configs.qm8_gat(dropout=0.1)), 'ids'),
    'GraphSAGE-Mean': (lambda: GraphSAGE(configs.qm8_graphsage(agg_func='Mean')), 'sage'),
    'GraphSAGE-Max': (lambda: GraphSAGE(configs.qm8_graphsage(agg_func='Max')), 'sage'),
    'LSTMGraphSAGE': (lambda: LSTMGraphSAGE(configs.qm8_graphsage(agg_func='LSTM')), 'sage'),
    'SampledGraphSAGE': (lambda: SampledGraphSAGE(configs.qm8_graphsage(agg_func='Max')), 'records'),
    'GGNN': (lambda: GGNN(configs.qm8_ggnn()), 'ids'),
    'MPNN': (lambda: MPNN(configs.qm8_mpnn()), 'ids'),
    'GPNN': (lambda: GPNN(configs.qm8_gpnn()), 'ids'),
}


def dev():
  return torch.device('cuda:0')


@pytest.fixture(autouse=True)
def deterministic():
  prev = torch.are_deterministic_algorithms_enabled()
  fill = torch.utils.deterministic.fill_uninitialized_memory
  torch.use_deterministic_algorithms(True)
  torch.utils.deterministic.fill_uninitialized_memory = True
  try:
    yield
  finally:
    torch.use_deterministic_algorithms(prev)
    torch.utils.deterministic.fill_uninitialized_memory = fill


def _samples(name, seed):
  if MODELS[name][1] == 'feat':
    return data.synthetic_regression_graphs(B, seed=seed)
  return data.synthetic_qm8_samples(B, seed=seed)


def _build(name):
  mod = MODELS[name][0]()
  mod.load_state_dict(deterministic_state_dict(mod, 7))
  return mod.to(dev()).train()


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def _key(name, i):
  k = torch.tensor([1234, i], dtype=torch.int64, device=dev())
  return {'KeyedGAT': {'dropout_key': k}, 'KeyedAdaLanczosNet': {'start_key': k},
          'SampledGraphSAGE': {'sample_key': k}}.get(name, {})


def _padded(name, samples, i, num_nodes=None):
  """(args, kwargs) of the padded training call on ``samples``: label and mask in kwargs."""
  kind = MODELS[name][1]
  if kind == 'sage':
    c = data.sage_collate(samples, configs.qm8_graphsage().model.num_sample_neighbors, np.random.RandomState(i))
    args = (_t(c['node_feat']), _t(c['nn_idx']), _t(c['nonempty_mask']))
  else:
    c = data.collate(samples, K, num_nodes=num_nodes)
    L = _t(data.gat_bias(c['L']) if 'GAT' in name else c['L'])
    args = (_t(c['node_feat']), L)
    if name in ('LanczosNet', 'LanczosNetGeneral'):
      args += (_t(c['D']), _t(c['V']))
  kw = dict(label=_t(c['label']), mask=_t(c['node_mask']), **_key(name, i))
  return args, kw


def _records(name, samples, i):
  sp = data.sparse_collate(samples, K, eigs=(name == 'LanczosNet'))
  rec = {k: (_t(v) if isinstance(v, np.ndarray) else v) for k, v in sp.items()}
  label = rec.pop('label')
  rec.update(_key(name, i))
  return rec, label


def _eager_run(name, batches):
  """3 eager Adam steps on ``batches``: the model and the losses."""
  torch.manual_seed(1234)                # AdaLanczosNet draws its start vectors on the CPU generator
  mod = _build(name)
  opt = torch.optim.Adam(mod.parameters(), lr=1e-3)
  losses = []
  for i, samples in enumerate(batches):
    opt.zero_grad()
    if MODELS[name][1] == 'records':
      rec, label = _records(name, samples, i)
      _, loss = mod.forward_sparse_train(rec, label=label)
    else:
      args, kw = _padded(name, samples, i)
      _, loss = mod(*args, **kw)
    loss.backward()
    opt.step()
    losses.append(loss.detach().clone())
  return mod, losses


def _assert_equal_runs(name, a, b):
  (ma, la), (mb, lb) = a, b
  for i, (x, y) in enumerate(zip(la, lb)):
    assert torch.isfinite(x).all(), (name, i, float(x))
    assert torch.equal(x, y), (name, i, float(x), float(y))
  for (n, p), (_, q) in zip(ma.named_parameters(), mb.named_parameters()):
    assert torch.isfinite(p).all(), (name, n)
    assert torch.equal(p, q), (name, n, float((p - q).abs().max()))


@pytest.mark.parametrize('name', sorted(MODELS))
def test_eager_adam_steps_are_bit_reproducible(name):
  batches = [_samples(name, s) for s in (11, 12, 13)]
  _assert_equal_runs(name, _eager_run(name, batches), _eager_run(name, batches))


# ---- captured steps -----------------------------------------------------------------------------
def _graphed_run(name, mode, batches):
  mod = _build(name)
  opt = torch.optim.Adam(mod.parameters(), lr=1e-3)
  if mode == 'padded':
    N = max(max(s['L_simple_4'].shape[0] for s in b) for b in batches)
    calls = [_padded(name, b, i, num_nodes=N) for i, b in enumerate(batches)]
    if MODELS[name][1] == 'sage':      # sage_collate pads to the batch's own largest molecule: one batch
      calls = [_padded(name, batches[0], 0)] * len(batches)
    step = train.GraphedStep(mod, opt, calls[0][0], calls[0][1])
  elif mode == 'sparse':
    calls = [_records(name, batches[0], i) for i in range(len(batches))]
    calls = [((r,), {'label': lab}) for r, lab in calls]
    step = train.GraphedStep(mod, opt, calls[0][0], calls[0][1], sparse=True)
  else:
    sp = data.sparse_collate(batches[0], K, eigs=False)
    pk = {k: (_t(v) if isinstance(v, np.ndarray) else v) for k, v in data.pack_sparse(sp, label=True).items()}
    calls = [((dict(pk, **_key(name, i)),), {}) for i in range(len(batches))]
    step = train.GraphedStep(mod, opt, calls[0][0], packed=True)
  losses = []
  for args, kw in calls:
    _, loss = step(*args, **kw)
    losses.append(loss.detach().clone())
  assert step.replays == len(calls)
  return mod, losses


# the models GraphedStep(packed=True) trains (KeyedAdaLanczosNet refuses packed batches)
PACKED = {'LanczosNet', 'LanczosNetGeneral', 'GCN', 'GCNFP', 'DCNN', 'ChebyNet', 'TrainableGAT', 'KeyedGAT',
          'SampledGraphSAGE', 'GGNN', 'MPNN', 'GPNN'}


def _graphed_cases():
  cases = []
  for name in sorted(MODELS):
    if name == 'AdaLanczosNet':
      continue                         # draws its start vector on the host: not capturable
    if MODELS[name][1] != 'records':
      cases.append((name, 'padded'))
    if hasattr(MODELS[name][0](), '_train_records'):
      cases.append((name, 'sparse'))
    if name in PACKED:
      cases.append((name, 'packed'))
  return cases


@pytest.mark.parametrize('name, mode', _graphed_cases())
def test_graphed_steps_are_bit_reproducible(name, mode):
  batches = [_samples(name, s) for s in (21, 22, 23)]
  _assert_equal_runs(name, _graphed_run(name, mode, batches), _graphed_run(name, mode, batches))


def test_ggnn_five_adam_steps_from_records_repeat():
  samples = data.synthetic_qm8_samples(64, seed=71)
  runs = []
  for _ in range(2):
    mod = _build('GGNN')
    opt = torch.optim.Adam(mod.parameters(), lr=1e-3)
    rec, label = _records('GGNN', samples, 0)
    losses = []
    for _ in range(5):
      opt.zero_grad()
      _, loss = mod.forward_sparse_train(rec, label=label)
      loss.backward()
      opt.step()
      losses.append(loss.detach().clone())
    runs.append((mod, losses))
  _assert_equal_runs('GGNN', *runs)


def test_trainable_gat_records_gradients_equal_the_padded_ones():
  """Including embedding.weight, whose adjoint is the segment sum: exact, so the row order of the records
  path and of the padded path give the same bits."""
  samples = data.synthetic_qm8_samples(64, seed=5)
  mod = _build('TrainableGAT').eval()
  args, kw = _padded('TrainableGAT', samples, 0)
  mod.zero_grad(set_to_none=True)
  mod(*args, **kw)[1].backward()
  g_pad = {n: p.grad.clone() for n, p in mod.named_parameters() if p.grad is not None}
  rec, label = _records('TrainableGAT', samples, 0)
  mod.zero_grad(set_to_none=True)
  mod.forward_sparse_train(rec, label=label)[1].backward()
  g_rec = {n: p.grad.clone() for n, p in mod.named_parameters() if p.grad is not None}
  assert set(g_pad) == set(g_rec) and 'embedding.weight' in g_pad
  for n in g_pad:
    assert torch.equal(g_pad[n], g_rec[n]), (n, float((g_pad[n] - g_rec[n]).abs().max()))


def test_one_cta_grid_gives_the_full_grid_parameters():
  """LanczosNet's training step runs the persistent wgmma kernels: capped at one CTA they give the same
  parameters as on the full grid."""
  batches = [_samples('LanczosNet', s) for s in (31, 32, 33)]
  full = _eager_run('LanczosNet', batches)
  _lib.check(_lib.load().lnb_debug_set_max_ctas(1), 'lnb_debug_set_max_ctas')
  try:
    one = _eager_run('LanczosNet', batches)
  finally:
    _lib.check(_lib.load().lnb_debug_set_max_ctas(0), 'lnb_debug_set_max_ctas')
  _assert_equal_runs('LanczosNet', full, one)
