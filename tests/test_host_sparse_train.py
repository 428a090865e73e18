"""Host-side checks of the training entry from sparse bond-list batches: which models take it, the refusals and
batch checks that come before any device work, and the argument checks of the ELL operator products and of
the captured step over records (no GPU needed)."""
import pytest
import torch

from lanczosnetwork_b200 import configs, data, ops, train
from lanczosnetwork_b200.model import (DCNN, GAT, GCN, GCNFP, GGNN, GPNN, MPNN, AdaLanczosNet, ChebyNet,
                                       GraphSAGE, LanczosNet, LanczosNetGeneral, LSTMGraphSAGE, TrainableGAT)

COVERED = [
    lambda: LanczosNet(configs.qm8_lanczos_net()), lambda: GCN(configs.qm8_gcn()), lambda: GCNFP(configs.qm8_gcn()),
    lambda: DCNN(configs.qm8_dcnn()), lambda: ChebyNet(configs.qm8_cheby_net()),
    lambda: GGNN(configs.qm8_ggnn()), lambda: GGNN(configs.qm8_ggnn(update_func='RNN', aggregate_type='sum')),
    lambda: MPNN(configs.qm8_mpnn()), lambda: MPNN(configs.qm8_mpnn(msg_func='embedding', aggregate_type='sum')),
    lambda: GPNN(configs.qm8_gpnn()), lambda: TrainableGAT(configs.qm8_gat()),
]
REFUSED = [
    lambda: GAT(configs.qm8_gat()), lambda: AdaLanczosNet(configs.qm8_ada_lanczos_net()),
    lambda: LanczosNetGeneral(configs.graph_lanczos_net()), lambda: GraphSAGE(configs.qm8_graphsage()),
    lambda: LSTMGraphSAGE(configs.qm8_graphsage(agg_func='LSTM')),
]


def _batch(B=4, seed=1, eigs=False):
  sp = data.sparse_collate(data.synthetic_qm8_samples(B, seed=seed), 20, eigs=eigs)
  return {k: torch.from_numpy(v) if hasattr(v, 'dtype') else v for k, v in sp.items()}


@pytest.mark.parametrize('make', COVERED)
def test_every_covered_model_has_the_records_hook(make):
  assert hasattr(make(), '_train_records')


@pytest.mark.parametrize('make', REFUSED)
def test_refusals_name_the_class_before_any_device_work(make):
  mod = make().train()
  assert not hasattr(mod, '_train_records')
  # a CPU module: any device work would raise RuntimeError instead
  with pytest.raises(NotImplementedError, match=type(mod).__name__):
    mod.forward_sparse_train(_batch())


def test_lanczos_net_refuses_packed_batches():
  sp = data.sparse_collate(data.synthetic_qm8_samples(4, seed=1), 20)
  packed = data.pack_sparse(sp)
  packed['blob'] = torch.from_numpy(packed['blob'])
  with pytest.raises(NotImplementedError, match='LanczosNet'):
    LanczosNet(configs.qm8_lanczos_net()).train().forward_sparse_train(packed)


def test_forward_sparse_still_refuses_autograd_and_points_to_the_new_entry():
  with pytest.raises(NotImplementedError, match='forward_sparse_train'):
    GCN(configs.qm8_gcn()).train().forward_sparse(_batch())


def test_malformed_batches_raise_the_errors_of_forward_sparse():
  mod = GCN(configs.qm8_gcn()).train()
  b = _batch()
  for drop in ('edges', 'N', 'node_ptr'):
    with pytest.raises(ValueError, match=drop):
      mod.forward_sparse_train({k: v for k, v in b.items() if k != drop})
  with pytest.raises(ValueError, match='N=129'):
    mod.forward_sparse_train(dict(b, N=129))
  with pytest.raises(ValueError, match='int32'):
    mod.forward_sparse_train(dict(b, sizes=b['sizes'].long()))
  with pytest.raises(ValueError, match='edges'):
    mod.forward_sparse_train(dict(b, edges=b['edges'][:, :3].contiguous()))
  with pytest.raises(ValueError, match='num_partition=17'):
    GPNN(configs.qm8_gpnn(num_partition=17)).train().forward_sparse_train(b)
  with pytest.raises(TypeError):
    GGNN(configs.qm8_ggnn(update_func='MLP')).train().forward_sparse_train(b)


def _prep(B=2, N=5, E1=3):
  """Host tensors in GraphPrep's layout (the checks run before any launch)."""
  return ops.GraphPrep((torch.zeros((B, E1, N, N)), torch.zeros((B, E1, N, N), dtype=torch.uint8),
                        torch.zeros((B, E1), dtype=torch.int32), torch.zeros((B, 2), dtype=torch.int32), None))


def test_ell_messages_refuse_host_tensors():
  prep = _prep()
  with pytest.raises(RuntimeError, match='CUDA'):
    ops.ell_messages(torch.zeros((10, 4)), prep)
  with pytest.raises(RuntimeError, match='CUDA'):
    ops.ell_messages_adjoint(torch.zeros((10, 12)), prep, 4)


@pytest.mark.parametrize('N, E1', [(129, 3), (5, 17)])
def test_ell_messages_envelope(N, E1):
  prep = _prep(1, N, E1)
  with pytest.raises(ValueError, match='N=%d, E1=%d' % (N, E1)):
    ops.ell_messages(torch.zeros((N, 4)), prep)
  with pytest.raises(ValueError, match='N=%d, E1=%d' % (N, E1)):
    ops.ell_messages_adjoint(torch.zeros((N, 4 * E1)), prep, 4)


def test_ell_messages_argument_checks():
  prep = _prep()
  X = torch.zeros((10, 4))
  for c0, nc in ((0, 4), (3, 1), (-1, 1), (1, 0)):
    with pytest.raises(ValueError, match='channels'):
      ops.ell_messages(X, prep, c0, nc)
    with pytest.raises(ValueError, match='channels'):
      ops.ell_messages_adjoint(torch.zeros((10, 12)), prep, 4, c0, nc)
  with pytest.raises(ValueError, match='X'):
    ops.ell_messages(X.double(), prep)
  with pytest.raises(ValueError, match='X'):
    ops.ell_messages(torch.zeros((9, 4)), prep)
  with pytest.raises(ValueError, match='stride'):
    ops.ell_messages(torch.zeros((4, 10)).t(), prep)
  with pytest.raises(ValueError, match='out'):
    ops.ell_messages(X, prep, out=torch.zeros((10, 11)))
  with pytest.raises(ValueError, match='out'):
    ops.ell_messages(X, prep, out=torch.zeros((10, 12)), col0=4)
  with pytest.raises(ValueError, match='w'):
    ops.ell_messages(X, prep, w=torch.zeros((2, 5, 2)))
  with pytest.raises(ValueError, match='ELL'):
    ops.ell_messages(X, ops.GraphPrep((prep[0], prep[1].float(), prep[2], prep[3], None)))
  with pytest.raises(ValueError, match='G'):
    ops.ell_messages_adjoint(torch.zeros((10, 11)), prep, 4)
  with pytest.raises(ValueError, match='D=0'):
    ops.ell_messages_adjoint(torch.zeros((10, 12)), prep, 0)


def test_ell_operator_defaults_to_its_own_transpose():
  prep = _prep()
  op = train.ell_operator(prep)
  assert op.prep_t is prep and op.weight is None and op.shape == (2, 5, 5, 3)


def test_graphed_step_sparse_argument_checks():
  b = _batch()
  label = torch.zeros((4, 16))
  with pytest.raises(TypeError, match='GAT'):
    train.GraphedStep(GAT(configs.qm8_gat()), None, (b,), {'label': label}, sparse=True)
  mod = GCN(configs.qm8_gcn())
  opt = torch.optim.Adam(mod.parameters())
  with pytest.raises(ValueError, match='label'):
    train.GraphedStep(mod, opt, (b,), {}, sparse=True)
  with pytest.raises(ValueError, match='records'):
    train.GraphedStep(mod, opt, (b, b), {'label': label}, sparse=True)
  with pytest.raises(ValueError, match='N=129'):
    train.GraphedStep(mod, opt, (dict(b, N=129),), {'label': label}, sparse=True)
  with pytest.raises(ValueError, match='capacity'):
    train.GraphedStep(mod, opt, (b,), {'label': label}, sparse=True, edge_capacity=int(b['edges'].shape[0]) - 1)
  with pytest.raises(RuntimeError, match='CUDA'):                     # a CPU module: refused after the checks
    train.GraphedStep(mod, opt, (b,), {'label': label}, sparse=True)


def test_ell_messages_refuse_overlapping_storage():
  prep = _prep()
  buf = torch.zeros((10, 16))
  with pytest.raises(ValueError, match='overlaps X'):
    ops.ell_messages(buf[:, :4], prep, 0, 1, out=buf[:, 4:8])
  with pytest.raises(ValueError, match='overlaps X'):
    ops.ell_messages(buf[:, :4], prep, 0, 1, out=buf[:, :4])
  w = torch.zeros((2, 5, 3))
  with pytest.raises(ValueError, match='overlaps w'):
    ops.ell_messages(torch.zeros((10, 1)), prep, 0, 1, w=w, out=w.view(10, 3))
  with pytest.raises(ValueError, match='overlaps G'):
    ops.ell_messages_adjoint(buf[:, :12], prep, 4, out=buf[:, 12:16])
