"""Host-side checks of the drop-ins' sparse entry: which models take bond-list batches, the refusals that
come before any device work, and the envelope of the two sparse producers (no GPU needed)."""
import pytest
import torch

from lanczosnetwork_b200 import configs, data, ops
from lanczosnetwork_b200.model import (DCNN, GAT, GCN, GCNFP, GGNN, GPNN, MPNN, AdaLanczosNet, ChebyNet,
                                       GraphSAGE, LanczosNet, TrainableGAT)

SPARSE_MODELS = [
    lambda: GCN(configs.qm8_gcn()), lambda: GCNFP(configs.qm8_gcn()), lambda: DCNN(configs.qm8_dcnn()),
    lambda: ChebyNet(configs.qm8_cheby_net()), lambda: GAT(configs.qm8_gat()),
    lambda: TrainableGAT(configs.qm8_gat()), lambda: GGNN(configs.qm8_ggnn()), lambda: MPNN(configs.qm8_mpnn()),
    lambda: GPNN(configs.qm8_gpnn()),
]


def _batch(B=4, seed=1):
  sp = data.sparse_collate(data.synthetic_qm8_samples(B, seed=seed), 20, eigs=False)
  return {k: torch.from_numpy(v) if hasattr(v, 'dtype') else v for k, v in sp.items()}


@pytest.mark.parametrize('make', SPARSE_MODELS)
def test_every_operator_dropin_has_the_records_hook(make):
  mod = make().eval()
  assert hasattr(mod, '_forward_records')
  inputs, impl, key = mod._sparse_inputs(_batch())
  assert key == ('records', 26) and len(inputs) == 5 and callable(impl)
  assert inputs[2].capacity == 4 * 26                     # node ids: B * N rows under graph replay


@pytest.mark.parametrize('make', SPARSE_MODELS)
def test_forward_sparse_refuses_autograd(make):
  mod = make().train()
  with pytest.raises(NotImplementedError):
    mod.forward_sparse(_batch())


def test_lanczos_net_keeps_its_own_entries():
  mod = LanczosNet(configs.qm8_lanczos_net()).eval()
  assert not hasattr(mod, '_forward_records')
  b = _batch()
  assert mod._sparse_inputs(b)[2] == ('sparse_eigs', 26, 20)
  sp = data.sparse_collate(data.synthetic_qm8_samples(4, seed=1), 20)
  with_eigs = {k: torch.from_numpy(v) if hasattr(v, 'dtype') else v for k, v in sp.items()}
  assert mod._sparse_inputs(with_eigs)[2] == ('sparse', 26)
  packed = data.pack_sparse(sp)
  packed['blob'] = torch.from_numpy(packed['blob'])
  assert mod._sparse_inputs(packed)[2] == ('packed', 4, 26, 20)


@pytest.mark.parametrize('make', [lambda: GraphSAGE(configs.qm8_graphsage()),
                                  lambda: AdaLanczosNet(configs.qm8_ada_lanczos_net())])
def test_models_without_a_sparse_entry_say_so(make):
  with pytest.raises(NotImplementedError, match='sparse'):
    make().eval()._sparse_inputs(_batch())


def test_malformed_batches_are_refused():
  mod = GCN(configs.qm8_gcn()).eval()
  b = _batch()
  for drop in ('edges', 'N', 'node_ptr'):
    with pytest.raises(ValueError, match=drop):
      mod._sparse_inputs({k: v for k, v in b.items() if k != drop})
  with pytest.raises(ValueError, match='N=129'):
    mod._sparse_inputs(dict(b, N=129))
  with pytest.raises(ValueError, match='int32'):
    mod._sparse_inputs(dict(b, sizes=b['sizes'].long()))
  with pytest.raises(ValueError, match='edges'):
    mod._sparse_inputs(dict(b, edges=b['edges'][:, :3].contiguous()))


def test_gpnn_checks_come_before_any_launch():
  b = _batch()
  with pytest.raises(ValueError, match='num_partition=17'):
    GPNN(configs.qm8_gpnn(num_partition=17)).eval()._sparse_inputs(b)
  with pytest.raises(ValueError):
    GPNN(configs.qm8_gpnn(num_partition=3)).eval()._sparse_inputs(dict(b, N=4))
  with pytest.raises(TypeError):
    GPNN(configs.qm8_gpnn(update_func='MLP')).eval()._sparse_inputs(b)
  with pytest.raises(TypeError):
    GGNN(configs.qm8_ggnn(update_func='MLP')).eval()._sparse_inputs(b)


@pytest.mark.parametrize('N, P', [(129, 3), (26, 1), (26, 17), (4, 3), (3, 2)])
def test_partition_envelope(N, P):
  assert not ops.spectral_partition_supported(N, P)
  b = _batch()
  with pytest.raises(ValueError):
    ops.spectral_partition_sparse(b['sizes'], b['edge_ptr'], b['edges'], N, P, 6)


def test_partition_envelope_accepts_the_dense_entrys_shapes():
  assert ops.spectral_partition_supported(26, 3) and ops.spectral_partition_supported(128, 16)
  assert ops.spectral_partition_supported(5, 3)


@pytest.mark.parametrize('N, E1', [(129, 7), (0, 7), (26, 1), (26, 17)])
def test_gat_bias_envelope(N, E1):
  b = _batch()
  with pytest.raises(ValueError):
    ops.gat_bias_sparse(b['sizes'], b['edge_ptr'], b['edges'], N, E1)


def test_sparse_producers_refuse_host_tensors():
  b = _batch()
  with pytest.raises(RuntimeError, match='CUDA'):
    ops.gat_bias_sparse(b['sizes'], b['edge_ptr'], b['edges'], 26, 7)
  with pytest.raises(RuntimeError, match='CUDA'):
    ops.spectral_partition_sparse(b['sizes'], b['edge_ptr'], b['edges'], 26, 3, 6)
