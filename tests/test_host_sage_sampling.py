"""Host-side checks of GraphSAGE's device sampling: the numpy restatement of the sampler (Philox4x32-10
known answers, hand-built rows, the distributions of numpy's ``choice``), SampledGraphSAGE's hooks and
initial weights, and the refusals that come before any device work (no GPU needed)."""
import numpy as np
import pytest
import scipy.stats
import torch

from lanczosnetwork_b200 import configs, data, ops, train
from lanczosnetwork_b200.model import GraphSAGE, LSTMGraphSAGE, SampledGraphSAGE

import sage_sample_oracle as oracle


def _batch(B=4, seed=1, key=(7, 0)):
  sp = data.sparse_collate(data.synthetic_qm8_samples(B, seed=seed), 20, eigs=False)
  out = {k: torch.from_numpy(v) if hasattr(v, 'dtype') else v for k, v in sp.items()}
  if key is not None:
    out['sample_key'] = torch.tensor(key, dtype=torch.int64)
  return out


@pytest.mark.parametrize('ctr, key, want', [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
  assert tuple(int(v) for v in oracle.philox4x32_10(ctr, key)) == want


def test_draws_follow_the_counter_layout():
  # draw i of row r is word i % 4 of the block at counter (i / 4, r, ctr lo, ctr hi), key (seed lo, seed hi)
  seed, ctr = (5 << 32) | 9, (3 << 32) | 11
  x = oracle.draws((seed, ctr), [0, 17], 6)
  for r, row in zip((0, 17), x):
    for blk in range(2):
      want = oracle.philox4x32_10((blk, r, 11, 3), (9, 5))
      got = row[4 * blk:4 * blk + 4]
      assert [int(v) for v in got] == [int(v) for v in want[:len(got)]]


def test_hand_built_rows():
  K = 3
  cands = [np.array([2]), np.array([0, 4]), np.array([1, 3, 5, 6, 8]), np.zeros(0, np.int64),
           np.array([4, 5, 9])]
  x = oracle.draws((123, 4), np.arange(len(cands)), K)
  s = oracle.sample_rows(cands, x, K)
  assert (s[0] == 2).all()                                    # L = 1 < K: the one candidate K times
  assert set(s[1]) <= {0, 4}                                  # L < K: with replacement
  assert len(set(s[2])) == K and set(s[2]) <= {1, 3, 5, 6, 8}  # L >= K: K distinct candidates
  assert (s[3] == 0).all()                                    # L = 0: the zero fill
  assert sorted(s[4]) == [4, 5, 9]                            # L == K: a permutation
  # the rule spelled out for row 2
  c = [1, 3, 5, 6, 8]
  for i in range(K):
    j = i + int((int(x[2, i]) * (5 - i)) >> 32)
    c[i], c[j] = c[j], c[i]
  assert list(s[2]) == c[:K]
  assert list(s[1]) == [[0, 4][int((int(v) * 2) >> 32)] for v in x[1]]


def test_padded_rows_and_nonempty():
  samples = data.synthetic_qm8_samples(3, seed=2)
  sizes = [s['L_simple_4'].shape[0] for s in samples]
  nn_idx, nonempty = oracle.sample_batch(samples, 5, (1, 2), N=30)
  assert nn_idx.shape == (3, 30, 5, 7) and nn_idx.dtype == np.int32
  for b, n in enumerate(sizes):
    assert (nonempty[b, :n] == 1).all() and (nonempty[b, n:] == 0).all()
    assert (nn_idx[b, n:] == 0).all()
    # every sample is a candidate of its row: a non-zero of the channel's L4 row
    for e in range(7):
      op = samples[b]['L_simple_4'] if e == 0 else samples[b]['L_multi'][:, :, e - 1]
      rows = np.repeat(np.arange(n), 5)
      assert (op[rows, nn_idx[b, :n, :, e].reshape(-1)] != 0).all()


def _chi2_ok(counts, p_level=1e-6):
  counts = np.asarray(counts, np.float64)
  expected = counts.sum() / counts.size
  stat = ((counts - expected) ** 2 / expected).sum()
  return stat < scipy.stats.chi2.ppf(1 - p_level, counts.size - 1)


@pytest.mark.parametrize('key', [(0, 0), (1234, 1), (2 ** 40 + 3, 2 ** 33)])
def test_draws_with_replacement_are_uniform(key):
  R, K, L = 4000, 8, 5
  cand = np.array([1, 2, 6, 7, 11])
  s = oracle.sample_rows([cand] * R, oracle.draws(key, np.arange(R), K), K)
  assert _chi2_ok([(s == c).sum() for c in cand])
  for i in range(K):                                           # every draw on its own too
    assert _chi2_ok([(s[:, i] == c).sum() for c in cand])


@pytest.mark.parametrize('key', [(0, 0), (99, 5)])
def test_draws_without_replacement_are_uniform_ordered_subsets(key):
  R, K, L = 6000, 3, 6
  cand = np.arange(L) * 2
  s = oracle.sample_rows([cand] * R, oracle.draws(key, np.arange(R), K), K)
  assert all(len(set(row)) == K for row in s)
  for i in range(K):
    assert _chi2_ok([(s[:, i] == c).sum() for c in cand])
  # ordered pairs of the first two draws: uniform over the L * (L - 1) of them
  pair = s[:, 0] // 2 * L + s[:, 1] // 2
  counts = np.bincount(pair, minlength=L * L).reshape(L, L)
  assert (np.diag(counts) == 0).all()
  assert _chi2_ok(counts[~np.eye(L, dtype=bool)])


def test_only_the_sampled_class_has_the_records_hooks():
  mod = SampledGraphSAGE(configs.qm8_graphsage())
  assert hasattr(mod, '_forward_records') and hasattr(mod, '_train_records')
  for cls in (GraphSAGE, LSTMGraphSAGE):
    m = cls(configs.qm8_graphsage())
    assert not hasattr(m, '_forward_records') and not hasattr(m, '_train_records')
  inputs, impl, key = mod.eval()._sparse_inputs(_batch())
  assert key == ('sampled', 26) and len(inputs) == 6 and callable(impl)
  assert inputs[5].dtype == torch.int64 and tuple(inputs[5].shape) == (2,)


@pytest.mark.parametrize('agg', ['Mean', 'Max', 'LSTM'])
def test_initial_state_dict_is_the_same_across_the_classes(agg):
  classes = [SampledGraphSAGE, LSTMGraphSAGE] + ([GraphSAGE] if agg != 'LSTM' else [])
  dicts = []
  for cls in classes:
    torch.manual_seed(1234)
    dicts.append(cls(configs.qm8_graphsage(agg_func=agg)).state_dict())
  for d in dicts[1:]:
    assert list(d) == list(dicts[0])
    assert all(torch.equal(d[k], dicts[0][k]) for k in d)


# _sparse_inputs holds the batch checks of forward_sparse and GraphedStep(sparse=True)
@pytest.mark.parametrize('entry', ['_sparse_inputs', 'forward_sparse_train'])
def test_missing_or_malformed_sample_key_is_refused_before_device_work(entry):
  mod = SampledGraphSAGE(configs.qm8_graphsage()).eval()     # a CPU module: device work would raise RuntimeError
  for key in (None, (1, 2, 3), (1.0, 2.0)):
    b = _batch()
    if key is None:
      b.pop('sample_key')
    else:
      b['sample_key'] = torch.tensor(key)
    with pytest.raises(ValueError, match='sample_key'), torch.no_grad():
      getattr(mod, entry)(b)


def test_too_many_nodes_is_refused():
  mod = SampledGraphSAGE(configs.qm8_graphsage()).eval()
  b = _batch()
  b['N'] = 129
  with pytest.raises(ValueError, match='N=129'):
    mod._sparse_inputs(b)
  with pytest.raises(ValueError, match='N=129'):
    mod.forward_sparse_train(b)


def test_cpu_module_is_refused():
  with pytest.raises(RuntimeError, match='CUDA'), torch.no_grad():
    SampledGraphSAGE(configs.qm8_graphsage()).eval().forward_sparse(_batch())


def test_unknown_aggregator_is_refused_before_device_work():
  with pytest.raises(TypeError, match='agg_func'):
    SampledGraphSAGE(configs.qm8_graphsage(agg_func='Sum')).eval()._sparse_inputs(_batch())


def test_sampler_wrapper_checks_its_arguments():
  b = _batch()
  args = [b[k] for k in ('sizes', 'node_ptr', 'node_feat', 'edge_ptr', 'edges')]
  with pytest.raises(RuntimeError, match='CUDA'):
    ops.sage_sample_sparse(*args, b['sample_key'], 26, 7, 40)


def test_graphed_step_copies_the_sample_key():
  assert 'sample_key' in train.GraphedStep._RECORD_KEYS
  assert 'sample_key' not in train.GraphedStep._RAGGED
