"""SparseLanczosNetGeneral and float-feature records without a GPU: sparse_collate's feature rows are
collate's bits, the subclass has LanczosNetGeneral's parameters and initial weights, every batch check
fires before any device work, and ops.graph_prepare_sparse_features checks its arguments first."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data, ops, train
from lanczosnetwork_b200.model import LanczosNetGeneral, SparseLanczosNetGeneral


def _config(F=10, **kw):
  cfg = configs.graph_lanczos_net(input_dim=F, **kw)
  cfg.dataset.node_emb_dim = F                 # the reference asserts input_dim == node_emb_dim
  return cfg


def _records(B=3, eigs=False, seed=5):
  sp = data.sparse_collate(data.synthetic_regression_graphs(B, seed=seed, max_num_nodes=40), 20, eigs=eigs)
  return {k: torch.from_numpy(v) if isinstance(v, np.ndarray) else v for k, v in sp.items()}


def test_float_feature_rows_are_the_bits_of_collate():
  samples = data.synthetic_regression_graphs(6, seed=123)
  sp = data.sparse_collate(samples, 20)
  c = data.collate(samples, 20)
  assert sp['node_feat'].dtype == np.float32 and sp['node_feat'].shape == (int(sp['node_ptr'][-1]), 10)
  for b, n in enumerate(sp['sizes']):
    rows = sp['node_feat'][sp['node_ptr'][b]:sp['node_ptr'][b + 1]]
    assert np.array_equal(rows.view(np.uint32), c['node_feat'][b, :n].view(np.uint32))
  # each fp64 feature is rounded once to fp32 (the truncation to int32 is gone)
  assert np.array_equal(sp['node_feat'], np.concatenate([s['node_feat'] for s in samples]).astype(np.float32))
  assert not np.array_equal(sp['node_feat'], np.trunc(sp['node_feat']))


def test_atom_id_records_are_unchanged():
  samples = data.synthetic_qm8_samples(8, seed=3)
  sp = data.sparse_collate(samples, 20)
  want = np.concatenate([np.asarray(s['node_feat']).astype(np.int32) for s in samples])
  assert sp['node_feat'].dtype == np.int32 and sp['node_feat'].tobytes() == want.tobytes()


def test_parameters_and_seeded_weights_equal_lanczos_net_general():
  cfg = configs.graph_lanczos_net()
  torch.manual_seed(11)
  base = LanczosNetGeneral(cfg)
  after_base = torch.randn(3)
  torch.manual_seed(11)
  sub = SparseLanczosNetGeneral(cfg)
  after_sub = torch.randn(3)
  assert isinstance(sub, LanczosNetGeneral)
  assert list(sub.state_dict()) == list(base.state_dict())
  for k, v in base.state_dict().items():
    assert torch.equal(v, sub.state_dict()[k]), k
  assert torch.equal(after_base, after_sub)               # the same CPU random numbers were consumed
  sub.load_state_dict(base.state_dict())                  # strict, both ways
  base.load_state_dict(sub.state_dict())
  assert SparseLanczosNetGeneral.forward is LanczosNetGeneral.forward


def test_the_base_class_keeps_refusing_records():
  base = LanczosNetGeneral(configs.graph_lanczos_net())
  assert not hasattr(base, '_train_records')
  with pytest.raises(NotImplementedError, match='LanczosNetGeneral'):
    base.train().forward_sparse_train(_records())
  with pytest.raises(NotImplementedError):
    base.eval()._sparse_inputs(_records())


def test_records_are_taken_with_and_without_eigenpairs():
  mod = SparseLanczosNetGeneral(configs.graph_lanczos_net()).eval()
  b = _records()
  inputs, impl, key = mod._sparse_inputs(b)
  assert key == ('sparse_eigs', b['N'], 20) and len(inputs) == 5 and callable(impl)
  assert inputs[2].static_shape() == (3 * b['N'], 10)      # feature rows: B * N rows of F floats
  assert mod._sparse_inputs(_records(eigs=True))[2] == ('sparse', b['N'])


# _sparse_inputs holds the batch checks of forward_sparse and GraphedStep(sparse=True)
@pytest.mark.parametrize('entry', ['_sparse_inputs', 'forward_sparse_train'])
def test_batch_checks_fire_before_device_work(entry):
  """The module sits on the CPU: any device work would raise RuntimeError instead."""
  mod = SparseLanczosNetGeneral(configs.graph_lanczos_net()).eval()
  call = getattr(mod, entry)
  b = _records()
  for drop in ('edges', 'N', 'node_ptr', 'node_feat'):
    with pytest.raises(ValueError, match=drop):
      call({k: v for k, v in b.items() if k != drop})
  bad = [(dict(b, node_feat=b['node_feat'].double()), 'node_feat'),
         (dict(b, node_feat=b['node_feat'][:, :9].contiguous()), 'node_feat'),
         (dict(b, node_feat=b['node_feat'].reshape(-1)), 'node_feat'),
         (dict(b, node_feat=b['node_feat'].to(torch.int32)), 'node_feat'),
         (dict(b, sizes=b['sizes'].long()), 'int32'), (dict(b, node_ptr=b['node_ptr'].long()), 'int32'),
         (dict(b, edge_ptr=b['edge_ptr'].long()), 'int32'),
         (dict(b, edges=b['edges'][:, :3].contiguous()), 'edges'), (dict(b, edges=b['edges'].int()), 'edges'),
         (dict(b, N=129), 'N=129'), ({k: v for k, v in b.items() if k != 'K'}, 'K')]
  e = _records(eigs=True)
  bad += [({k: v for k, v in e.items() if k != 'D'}, 'V_rows'), (dict(e, D=e['D'].double()), 'D'),
          (dict(e, V_rows=e['V_rows'].double()), 'V_rows'), (dict(e, D=e['D'][:, :5]), 'D')]
  for batch, what in bad:
    with pytest.raises(ValueError, match=what):
      call(batch)
  cfg = configs.graph_lanczos_net()
  cfg.dataset.num_edge_type = 16
  with pytest.raises(ValueError, match=r'E\+1=17'):
    getattr(SparseLanczosNetGeneral(cfg).eval(), entry)(b)
  packed = dict(b, blob=torch.zeros(64, dtype=torch.uint8))
  with pytest.raises(NotImplementedError, match='packed'):
    call(packed)


def test_input_width_other_than_ten():
  mod = SparseLanczosNetGeneral(_config(33))
  with pytest.raises(ValueError, match=r'\[rows, 33\]'):
    mod.eval()._sparse_inputs(_records())


def test_graphed_step_admits_the_subclass_and_checks_its_records():
  mod = SparseLanczosNetGeneral(configs.graph_lanczos_net())
  opt = torch.optim.Adam(mod.parameters())
  b = _records()
  label = torch.zeros((3, 2))
  with pytest.raises(ValueError, match='node_feat'):
    train.GraphedStep(mod, opt, (dict(b, node_feat=b['node_feat'].double()),), {'label': label}, sparse=True)
  with pytest.raises(RuntimeError, match='CUDA'):                     # a CPU module: refused after the checks
    train.GraphedStep(mod, opt, (b,), {'label': label}, sparse=True)
  with pytest.raises(TypeError):
    train.GraphedStep(LanczosNetGeneral(configs.graph_lanczos_net()), opt, (b,), {'label': label}, sparse=True)


def test_prepare_features_refuses_host_tensors_and_bad_arguments():
  b = _records(eigs=True)
  args = [b['sizes'], b['node_ptr'], b['node_feat'], b['edge_ptr'], b['edges'], b['V_rows'], b['N'], 2]
  with pytest.raises(RuntimeError, match='CUDA'):
    ops.graph_prepare_sparse_features(*args)

  def with_(i, v, what):
    a = list(args)
    a[i] = v
    with pytest.raises(ValueError, match=what):
      ops.graph_prepare_sparse_features(*a)

  with_(0, b['sizes'].long(), 'sizes')
  with_(1, b['node_ptr'].long(), 'node_ptr')
  with_(3, b['edge_ptr'].long(), 'edge_ptr')
  with_(2, b['node_feat'].double(), 'node_x')
  with_(2, b['node_feat'].reshape(-1), 'node_x')
  with_(2, b['node_feat'].t(), 'node_x')
  with_(4, b['edges'].int(), 'edges')
  with_(4, b['edges'][:, :3], 'edges')
  with_(5, b['V_rows'].double(), 'V_rows')
  with_(6, 129, 'N=129')
  with_(7, 17, 'E1=17')
  with_(7, 1, 'E1=1')
  with_(2, torch.zeros((10, 4097)), 'F=4097')
  with_(2, torch.zeros((10, 0)), 'F=0')
