"""forward_sparse of the operator drop-ins (GCN, GCNFP, DCNN, ChebyNet, GAT, GGNN, MPNN, GPNN) against
their padded forward, and the two producers behind it: lnb_spectral_partition_sparse against
lnb_spectral_partition on the collated operators, lnb_gat_bias_sparse against data.gat_bias."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data, ops
from lanczosnetwork_b200.model import DCNN, GAT, GCN, GCNFP, GGNN, GPNN, MPNN, ChebyNet, TrainableGAT

from helpers import deterministic_state_dict

pytestmark = pytest.mark.gpu

K = 20
MODELS = {
    'GCN': lambda: GCN(configs.qm8_gcn()),
    'GCNFP': lambda: GCNFP(configs.qm8_gcn()),
    'GCN_unfused': lambda: GCN(configs.qm8_gcn(hidden_dim=[128, 64, 128], num_layer=3)),
    'DCNN': lambda: DCNN(configs.qm8_dcnn()),
    'ChebyNet': lambda: ChebyNet(configs.qm8_cheby_net()),
    'GAT': lambda: GAT(configs.qm8_gat()),
    'TrainableGAT': lambda: TrainableGAT(configs.qm8_gat()),
    'GGNN': lambda: GGNN(configs.qm8_ggnn()),
    'GGNN_sum': lambda: GGNN(configs.qm8_ggnn(aggregate_type='sum')),
    'GGNN_rnn': lambda: GGNN(configs.qm8_ggnn(update_func='RNN', num_prop=3)),
    'MPNN': lambda: MPNN(configs.qm8_mpnn()),
    'MPNN_sum': lambda: MPNN(configs.qm8_mpnn(aggregate_type='sum')),
    'MPNN_embedding': lambda: MPNN(configs.qm8_mpnn(msg_func='embedding')),
    'GPNN': lambda: GPNN(configs.qm8_gpnn()),
    'GPNN_unequal': lambda: GPNN(configs.qm8_gpnn(num_prop_cluster=2, num_prop_cut=3, num_partition=4,
                                                  aggregate_type='sum')),
}


def dev():
  return torch.device('cuda:0')


def _build(name, seed=7):
  mod = MODELS[name]()
  mod.load_state_dict(deterministic_state_dict(mod, seed))
  return mod.to(dev()).eval()


def _padded(name, mod, samples):
  """The padded forward on data.collate of the same samples (GAT: the collate's attention bias)."""
  c = data.collate(samples, K)
  nf = torch.from_numpy(c['node_feat']).to(dev())
  L = c['L'] if 'GAT' not in name else data.gat_bias(c['L'])
  mask = torch.from_numpy(c['node_mask']).to(dev())
  return mod(nf, torch.from_numpy(L).to(dev()), mask=mask)


def _records(samples, where, eigs=False):
  sp = data.sparse_collate(samples, K, eigs=eigs)
  out = {}
  for k, v in sp.items():
    if isinstance(v, np.ndarray):
      t = torch.from_numpy(v)
      out[k] = t.pin_memory() if where == 'pinned' else t.to(dev())
    else:
      out[k] = v
  return out


def _odd_samples():
  """An isolated node, a one-node graph, a node with no bond of most types, and QM8-shaped molecules."""
  rng = np.random.RandomState(5)
  a = np.zeros((5, 5, 6))
  for u, v, c in ((0, 1, 0), (1, 2, 1), (2, 3, 0)):             # node 4: no bond at all
    a[u, v, c] = a[v, u, c] = 1.0
  one = np.zeros((1, 1, 6))
  out = [data.prepare_graph(a, rng.randint(0, 70, 5), label=rng.randn(1, 16)),
         data.prepare_graph(one, rng.randint(0, 70, 1), label=rng.randn(1, 16))]
  return out + data.synthetic_qm8_samples(14, seed=11)


@pytest.mark.parametrize('B', [64, 1024])
@pytest.mark.parametrize('name', sorted(MODELS))
def test_forward_sparse_equals_padded_forward(name, B):
  samples = data.synthetic_qm8_samples(B, seed=B + 3)
  mod = _build(name)
  with torch.no_grad():
    ref = _padded(name, mod, samples)
    res = _records(samples, 'device')
    for _ in range(3):                 # copy-slot capture, then the resident capture and its replay
      assert torch.equal(mod.forward_sparse(res), ref), name
    host = _records(samples, 'pinned')
    for _ in range(2):
      assert torch.equal(mod.forward_sparse(host), ref), name
    if B == 64:
      assert torch.equal(mod.forward_sparse(_records(samples, 'device', eigs=True)), ref), name
      mod.use_cuda_graph = False
      assert torch.equal(mod.forward_sparse(res), ref), name


@pytest.mark.parametrize('name', ['GCN', 'GCNFP', 'DCNN', 'ChebyNet', 'GAT', 'GGNN', 'MPNN', 'GPNN'])
def test_forward_sparse_odd_graphs(name):
  samples = _odd_samples()
  mod = _build(name, seed=3)
  with torch.no_grad():
    ref = _padded(name, mod, samples)
    assert torch.equal(mod.forward_sparse(_records(samples, 'device')), ref)
    assert torch.equal(mod.forward_sparse(_records(samples, 'pinned')), ref)
    label = torch.from_numpy(data.sparse_collate(samples, K)['label']).to(dev())
    score, loss = mod.forward_sparse(_records(samples, 'device'), label=label)
    assert torch.equal(score, ref) and torch.isfinite(loss)


def test_one_capture_for_batches_of_one_padding_target():
  mod = _build('GPNN')
  batches = [data.synthetic_qm8_samples(64, seed=seed) for seed in (1, 2, 3)]
  assert len({sum(len(s['node_feat']) for s in b) for b in batches}) == 3      # different node totals, N = 26
  with torch.no_grad():
    scores = [mod.forward_sparse(_records(b, 'pinned')) for b in batches]
    st = mod.graph_stats()
    assert st['captures'] == 1 and st['replays'] == 3, st
    for b, score in zip(batches, scores):
      assert torch.equal(score, _padded('GPNN', mod, b))


def test_forward_sparse_under_autograd_raises():
  mod = _build('GCN').train()
  with pytest.raises(NotImplementedError):
    mod.forward_sparse(_records(data.synthetic_qm8_samples(4, seed=1), 'device'))


def _prepare_ell(L_cluster, L_cut):
  B, N = L_cluster.shape[0], L_cluster.shape[1]
  return ops.graph_prepare(torch.stack([L_cluster, L_cut], 3), torch.zeros((B, N, 4), device=dev()))


@pytest.mark.parametrize('P', [2, 3, 16])
@pytest.mark.parametrize('max_nodes', [26, 60, 128])
def test_spectral_partition_sparse_equals_dense_entry(max_nodes, P):
  samples = data.synthetic_qm8_samples(96, seed=max_nodes + P, max_nodes=max_nodes)
  if max_nodes == 26:
    samples = samples + _odd_samples()
  c = data.collate(samples, K)
  L = torch.from_numpy(c['L']).to(dev())
  N = L.shape[1]
  labels, Lc, Lt, status = ops.spectral_partition(L, P)
  rec = _records(samples, 'device')
  s_labels, s_status, prep, s_Lc, s_Lt = ops.spectral_partition_sparse(
      rec['sizes'], rec['edge_ptr'], rec['edges'], N, P, 6, want_dense=True)
  assert torch.equal(s_labels, labels) and torch.equal(s_status, status)
  assert int((s_status & 8).sum()) == 0
  assert torch.equal(s_Lc, Lc) and torch.equal(s_Lt, Lt)
  ref = _prepare_ell(Lc, Lt)
  _check_ell(prep, ref)
  # no dense outputs: the same labels and ELL rows; repeated launches are bit-identical
  s2 = ops.spectral_partition_sparse(rec['sizes'], rec['edge_ptr'], rec['edges'], N, P, 6)
  assert s2[3] is None and torch.equal(s2[0], s_labels)
  _check_ell(s2[2], ref)


def _check_ell(prep, ref):
  """ell_max, gext and every ELL slot graph_prepare writes (slots past ell_max are never written)."""
  assert torch.equal(prep[2], ref[2]) and torch.equal(prep[3], ref[3])
  N = ref[0].shape[2]
  slots = torch.arange(N, device=dev()).view(1, 1, N, 1) < ref[2].view(-1, 2, 1, 1)
  assert torch.equal(prep[0][slots.expand_as(prep[0])], ref[0][slots.expand_as(ref[0])])
  assert torch.equal(prep[1][slots.expand_as(prep[1])], ref[1][slots.expand_as(ref[1])])


@pytest.mark.parametrize('max_nodes', [26, 100])
def test_gat_bias_sparse_equals_collate_bias(max_nodes):
  samples = data.synthetic_qm8_samples(64, seed=max_nodes, max_nodes=max_nodes) + _odd_samples()
  c = data.collate(samples, K)
  ref = torch.from_numpy(data.gat_bias(c['L'])).to(dev())
  rec = _records(samples, 'device')
  got = ops.gat_bias_sparse(rec['sizes'], rec['edge_ptr'], rec['edges'], c['L'].shape[1], 7)
  assert torch.equal(got.view(torch.int32), ref.view(torch.int32))


def test_envelope_refusals_launch_nothing():
  rec = _records(data.synthetic_qm8_samples(8, seed=1), 'device')
  mod = _build('GPNN')
  mod.num_partition = 17
  n0 = ops.launch_count()
  for N, P in ((129, 3), (26, 1), (26, 17), (4, 3)):
    with pytest.raises(ValueError):
      ops.spectral_partition_sparse(rec['sizes'], rec['edge_ptr'], rec['edges'], N, P, 6)
  for N, E1 in ((129, 7), (26, 1), (26, 17)):
    with pytest.raises(ValueError):
      ops.gat_bias_sparse(rec['sizes'], rec['edge_ptr'], rec['edges'], N, E1)
  with torch.no_grad(), pytest.raises(ValueError):
    mod.forward_sparse(rec)
  assert ops.launch_count() == n0
