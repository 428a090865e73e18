"""KeyedAdaLanczosNet without a GPU: its parameters and initial weights are AdaLanczosNet's, its key and
records checks fire before any device work, GraphedStep admits it, and the restatements the GPU tests
compare the kernels against are right (the start vector's distribution, the reverse sweep of the powers
adjoint against fp64 autograd, the fp64 Lanczos restatement against train._lanczos_train)."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data, ops, train
from lanczosnetwork_b200.model import AdaLanczosNet, KeyedAdaLanczosNet

import keyed_ada_oracle as oracle

SMALL = dict(num_layer=2, hidden_dim=[16, 16], num_eig_vec=4, long_diffusion_dist=[1, 3],
             short_diffusion_dist=[1])


def _records(key=(1, 0)):
  sp = data.sparse_collate(data.synthetic_qm8_samples(3, seed=2), 4, eigs=False)
  out = {k: torch.from_numpy(v) if isinstance(v, np.ndarray) else v for k, v in sp.items()}
  if key is not None:
    out['start_key'] = torch.tensor(key, dtype=torch.int64)
  return out


def test_parameters_and_seeded_weights_equal_ada_lanczos_net():
  cfg = configs.qm8_ada_lanczos_net(**SMALL)
  torch.manual_seed(7)
  base = AdaLanczosNet(cfg)
  after_base = torch.randn(3)
  torch.manual_seed(7)
  keyed = KeyedAdaLanczosNet(cfg)
  after_keyed = torch.randn(3)
  assert list(keyed.state_dict()) == list(base.state_dict())
  for k, v in base.state_dict().items():
    assert torch.equal(v, keyed.state_dict()[k]), k
  assert torch.equal(after_base, after_keyed)            # the same CPU random numbers were consumed
  assert keyed.start_key.tolist() == [1234, 0]            # (config.seed, 0), not in the state_dict
  keyed.load_state_dict(base.state_dict())                # strict: no missing or extra keys


def test_key_defaults_to_zero_seed_without_config_seed():
  cfg = configs.qm8_ada_lanczos_net(**SMALL)
  cfg.seed = None
  assert KeyedAdaLanczosNet(cfg).start_key.tolist() == [0, 0]


@pytest.mark.parametrize('bad', [torch.zeros(2, dtype=torch.int32), torch.zeros(3, dtype=torch.int64),
                                 (1, 2), torch.zeros(1, 2, dtype=torch.int64)])
def test_start_key_checks_fire_before_device_work(bad):
  """The module sits on the CPU: any device work would raise RuntimeError instead of ValueError."""
  mod = KeyedAdaLanczosNet(configs.qm8_ada_lanczos_net(**SMALL))
  x, L = torch.zeros(2, 3, dtype=torch.long), torch.zeros(2, 3, 3, 7)
  with pytest.raises(ValueError, match='start_key'):
    mod(x, L, start_key=bad)
  with pytest.raises(ValueError, match='start_key'):
    ops.ada_start_vector(bad, 2, 3)
  rec = _records(None)
  rec['start_key'] = bad
  with pytest.raises(ValueError, match='start_key'):
    mod.forward_sparse_train(rec)


def test_records_need_a_key_and_refuse_packed_batches():
  mod = KeyedAdaLanczosNet(configs.qm8_ada_lanczos_net(**SMALL))
  with pytest.raises(ValueError, match="lacks 'start_key'"):
    mod.forward_sparse_train(_records(None))
  with pytest.raises(ValueError, match="lacks 'start_key'"):
    mod._sparse_inputs(_records(None))
  rec = _records()
  rec['blob'] = torch.zeros(4, dtype=torch.uint8)
  with pytest.raises(NotImplementedError, match='packed'):
    mod.forward_sparse_train(rec)
  with pytest.raises(NotImplementedError, match='packed'):
    mod._sparse_inputs(rec)
  # the base class keeps refusing records
  with pytest.raises(NotImplementedError):
    AdaLanczosNet(configs.qm8_ada_lanczos_net(**SMALL)).forward_sparse_train(_records())


def test_powers_adjoint_envelope():
  assert ops.tridiag_powers_backward_supported(20, [1, 2, 3, 5, 7, 10, 20, 30])
  assert ops.tridiag_powers_backward_supported(20, [5, 7, 10, 20, 30])
  assert not ops.tridiag_powers_backward_supported(64, [1, 30])
  assert not ops.tridiag_powers_backward_supported(20, list(range(1, 34)))
  T = torch.zeros(2, 64, 64)
  with pytest.raises(ValueError, match='envelope'):
    ops.tridiag_powers_backward(T, torch.zeros(2, 64, 2, 64), [1, 30])
  with pytest.raises(ValueError, match='outside'):
    train.tridiag_powers(T, [1, 30])
  with pytest.raises(ValueError, match='gOut'):
    ops.tridiag_powers_backward(torch.zeros(2, 8, 8), torch.zeros(2, 8, 3, 8), [1, 2])


def test_graphed_step_admits_the_keyed_class_only():
  from lanczosnetwork_b200.train import GraphedStep
  cfg = configs.qm8_ada_lanczos_net(**SMALL)
  x = (torch.zeros(2, 3, dtype=torch.long), torch.zeros(2, 3, 3, 7))
  ada = AdaLanczosNet(cfg)
  with pytest.raises(TypeError):
    GraphedStep(ada, torch.optim.SGD(ada.parameters(), lr=0.1), x, {'label': torch.zeros(2, 16)})
  keyed = KeyedAdaLanczosNet(cfg)
  opt = torch.optim.SGD(keyed.parameters(), lr=0.1)
  with pytest.raises(RuntimeError, match='CUDA'):        # past the class check: the CPU module is refused
    GraphedStep(keyed, opt, x, {'label': torch.zeros(2, 16)})
  with pytest.raises(ValueError, match="lacks 'start_key'"):
    GraphedStep(keyed, opt, (_records(None),), {'label': torch.zeros(3, 16)}, sparse=True)
  assert 'start_key' in GraphedStep._RECORD_KEYS


def test_start_vector_restatement_is_standard_normal():
  q = oracle.start_vector((1234, 5), 256, 257).astype(np.float64).ravel()
  assert q.shape == (256 * 257,) and np.all(np.isfinite(q))
  n = q.size
  assert abs(q.mean()) < 5 / np.sqrt(n)
  assert abs(q.var() - 1.0) < 5 * np.sqrt(2.0 / n)
  # even and odd entries are the two Box-Muller outputs of one draw: uncorrelated
  qq = oracle.start_vector((1234, 5), 256, 256)
  assert abs(float(np.mean(qq[:, 0::2] * qq[:, 1::2]))) < 5 / np.sqrt(qq.size / 2)
  assert not np.array_equal(qq, oracle.start_vector((1234, 6), 256, 256))
  assert not np.array_equal(qq, oracle.start_vector((1235, 5), 256, 256))
  assert np.array_equal(qq, oracle.start_vector((1234, 5), 256, 256))


@pytest.mark.parametrize('K,powers', [(6, [1]), (6, [2, 5]), (8, [1, 2, 3, 5, 7, 10]), (20, [5, 7, 10, 20, 30])])
def test_powers_reverse_sweep_equals_fp64_autograd(K, powers):
  """The reverse sweep the kernel runs against autograd of P_1 = T, P_{p+1} = P_p tri(T) in fp64, on a
  full (not only tridiagonal) T: the first power reads every entry, the later products only the band."""
  rng = np.random.RandomState(K + len(powers))
  T = rng.randn(3, K, K) / (3.0 * np.sqrt(K))
  G = rng.randn(3, K, len(powers), K)
  Tt = torch.from_numpy(T).requires_grad_(True)
  band = torch.from_numpy((np.abs(np.arange(K)[:, None] - np.arange(K)[None, :]) <= 1).astype(np.float64))
  outs, cur = [], Tt
  for p in range(1, max(powers) + 1):
    if p in powers:
      outs.append(cur)
    cur = cur @ (Tt * band)
  out = torch.stack(outs, dim=2)
  np.testing.assert_allclose(out.detach().numpy(), oracle.powers_forward(T, powers), rtol=1e-12, atol=1e-14)
  (out * torch.from_numpy(G)).sum().backward()
  ref = Tt.grad.numpy()
  got = oracle.powers_backward(T, G, powers)
  assert np.max(np.abs(got - ref)) <= 1e-12 * max(1.0, np.max(np.abs(ref)))


def _spd(B, N, seed):
  rng = np.random.RandomState(seed)
  X = rng.randn(B, N, N)
  A = X @ np.swapaxes(X, 1, 2) / N + np.eye(N)[None]
  return torch.from_numpy(A / np.linalg.norm(A, axis=(1, 2), keepdims=True))


@pytest.mark.parametrize('N,K,masked', [(12, 5, False), (9, 20, True), (30, 8, True)])
def test_lanczos_restatement_equals_the_training_formulation(monkeypatch, N, K, masked):
  """The fp64 restatement the GPU tests differentiate is train._lanczos_train's formulation (its batched
  products swapped for torch.bmm to run on the CPU): T, Q and their gradients agree in fp64, N < K included."""
  monkeypatch.setattr(train, 'bmm', torch.bmm)
  B = 3
  A = _spd(B, N, N + K)
  rng = np.random.RandomState(K)
  q1 = torch.from_numpy(rng.randn(B, N))
  mask = None
  if masked:
    mask = torch.ones(B, N, dtype=torch.uint8)
    mask[0, N - 2:] = 0
    mask[2, N - 4:] = 0
  gT, gQ = torch.from_numpy(rng.randn(B, K, K)), torch.from_numpy(rng.randn(B, N, K))
  A1, A2 = A.clone().requires_grad_(True), A.clone().requires_grad_(True)
  T1, Q1 = train._lanczos_train(A1, mask, q1, K)
  T2, Q2, _ = oracle.lanczos_block_gs(A2, mask, q1, K)
  assert torch.allclose(T1, T2, rtol=1e-12, atol=1e-12) and torch.allclose(Q1, Q2, rtol=1e-12, atol=1e-12)
  ((T1 * gT).sum() + (Q1 * gQ).sum()).backward()
  ((T2 * gT).sum() + (Q2 * gQ).sum()).backward()
  assert torch.allclose(A1.grad, A2.grad, rtol=1e-10, atol=1e-10)


def test_lanczos_layer_envelope():
  assert ops.lanczos_tridiag_train_supported(128, 64) and ops.lanczos_tridiag_train_supported(1, 1)
  assert not ops.lanczos_tridiag_train_supported(129, 20) and not ops.lanczos_tridiag_train_supported(26, 65)
  for N, K in ((129, 20), (26, 65)):
    A, q1 = torch.zeros(2, N, N), torch.zeros(2, N)
    with pytest.raises(ValueError, match='outside'):
      train.lanczos_tridiag(A, None, q1, K)
    with pytest.raises(ValueError, match='outside'):
      ops.lanczos_tridiag_train(A, None, q1, K)
    with pytest.raises(ValueError, match='outside'):
      ops.lanczos_tridiag_backward(A, None, q1, K, torch.zeros(2, K, K), torch.zeros(2, N, K))


def test_powers_envelope_needs_strictly_increasing_powers():
  assert not ops.tridiag_powers_backward_supported(20, [5, 3])
  assert not ops.tridiag_powers_backward_supported(20, [2, 2])
  assert not ops.tridiag_powers_backward_supported(20, [0, 2])
