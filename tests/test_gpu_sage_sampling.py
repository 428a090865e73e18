"""GraphSAGE's neighbour sampling on the device (lnb_sage_sample_sparse) and SampledGraphSAGE on an H100:
the samples against the numpy restatement of the rule, the ELL rows of the count-weighted operator and of
its transpose against graph_prepare of the dense operators, inference and training from records against the
padded path on the same samples, and captured graphs that draw new samples when the key changes."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data, ops
from lanczosnetwork_b200.model import SampledGraphSAGE

import sage_sample_oracle as oracle
from helpers import deterministic_state_dict
from test_gpu_sparse_dropins import _odd_samples

pytestmark = pytest.mark.gpu

KEYS = [(1234, 0), (1234, 1), (2 ** 40 + 17, 2 ** 35 + 3)]
SMALL = dict(hidden_dim=[64] * 3, num_layer=3)


def dev():
  return torch.device('cuda:0')


def _records(samples, key, where='device'):
  sp = data.sparse_collate(samples, 20, eigs=False)
  sp['sample_key'] = np.array(key, np.int64)
  out = {}
  for k, v in sp.items():
    if isinstance(v, np.ndarray):
      t = torch.from_numpy(v)
      out[k] = t.pin_memory() if where == 'pinned' else t.to(dev())
    else:
      out[k] = v
  return out


def _dense_graph(n=128, E=2, p=0.3, seed=3):
  """One graph of n nodes whose rows have many candidates (the no-replacement branch at K = 40)."""
  rng = np.random.RandomState(seed)
  a = np.zeros((n, n, E))
  for c in range(E):
    up = np.triu(rng.rand(n, n) < p, 1)
    a[:, :, c] = up + up.T
  return data.prepare_graph(a, rng.randint(0, 70, n), label=rng.randn(1, 16))


def _case(name):
  """(samples, K) of a named batch."""
  if name.startswith('qm8_'):
    B = int(name[4:])
    return data.synthetic_qm8_samples(B, seed=B + 5), 40
  if name.startswith('k'):
    return data.synthetic_qm8_samples(32, seed=9), int(name[1:])
  if name == 'odd':
    return _odd_samples(), 40
  return [_dense_graph(), _dense_graph(n=50, seed=4)], 40


def _sample(rec, E1, K, **want):
  return ops.sage_sample_sparse(rec['sizes'], rec['node_ptr'], rec['node_feat'], rec['edge_ptr'], rec['edges'],
                                rec['sample_key'], rec['N'], E1, K, **want)


CASES = ['qm8_64', 'qm8_1024', 'k2', 'k3', 'odd', 'n128']


@pytest.mark.parametrize('name', CASES)
def test_samples_equal_the_oracle(name):
  samples, K = _case(name)
  E1 = samples[0]['L_multi'].shape[2] + 1
  for key in KEYS:
    rec = _records(samples, key)
    node_ids, mask, nonempty, nn_idx, _, _ = _sample(rec, E1, K)
    want_idx, want_ne = oracle.sample_batch(samples, K, key, N=rec['N'])
    assert torch.equal(nn_idx.cpu(), torch.from_numpy(want_idx)), (name, key)
    assert torch.equal(nonempty.view(nonempty.shape[0], -1).cpu(), torch.from_numpy(want_ne)), (name, key)
    padded = data.collate(samples, 1) if 'D_simple' in samples[0] else None
    sizes = rec['sizes'].cpu()
    assert torch.equal(mask.cpu(), (torch.arange(rec['N'])[None, :] < sizes[:, None]).to(torch.uint8))
    if padded is not None:
      assert torch.equal(node_ids.cpu(), torch.from_numpy(padded['node_feat']))
    # the same key draws the same samples; another key draws others
    assert torch.equal(_sample(rec, E1, K)[3], nn_idx)
  if name != 'odd':
    other = _sample(_records(samples, (1, 1)), E1, K)[3]
    assert not torch.equal(other, nn_idx)


def _ell_equal(got, want):
  """ELL rows, ell_max and gext equal on every slot below ell_max (the slots a consumer reads)."""
  val, idx, emax, gext = got[:4]
  rval, ridx, rmax, rgext = want[:4]
  assert torch.equal(emax, rmax) and torch.equal(gext, rgext)
  N = val.shape[2]
  live = torch.arange(N, device=val.device).view(1, 1, N, 1) < emax[:, :, None, None]
  live = live.expand_as(val)
  assert torch.equal(val[live], rval[live]) and torch.equal(idx[live], ridx[live])


@pytest.mark.parametrize('name', CASES)
def test_ell_rows_equal_graph_prepare_of_the_dense_operators(name):
  samples, K = _case(name)
  E1 = samples[0]['L_multi'].shape[2] + 1
  rec = _records(samples, KEYS[2])
  _, _, nonempty, nn_idx, prep, prep_t = _sample(rec, E1, K, want_ell=True, want_ell_t=True)
  M = ops.sage_operators(nn_idx.long(), nonempty)
  ref = ops.graph_prepare(M)
  _ell_equal(prep, ref)
  _ell_equal(prep_t, ops.graph_prepare(M.transpose(1, 2).contiguous()))
  # the tile table lnb_tile_assign writes from the sampler's extents (the schedule behind it is checked by the
  # stack kernel's scores in the inference tests)
  assert prep.tiles_pending
  ops.tile_assign(prep, 4)
  B = nn_idx.shape[0]
  T = int(ref[4][0])                                  # [T, first graph of tiles 0..T-1, B]; scratch behind
  assert torch.equal(prep[4][:T + 2], ref[4][:T + 2])
  # the ELL-only launch writes the same rows as the one that also writes the samples
  _, _, ne2, none, prep2, none_t = _sample(rec, E1, K, want_nn_idx=False, want_ell=True)
  assert none is None and none_t is None and torch.equal(ne2, nonempty)
  _ell_equal(prep2, ref)


def _build(agg, **over):
  cfg = configs.qm8_graphsage(agg_func=agg, **over)
  mod = SampledGraphSAGE(cfg)
  mod.load_state_dict(deterministic_state_dict(mod, 21))
  return mod.to(dev())


def _padded(mod, rec, label=None):
  """forward on the padded batch built from the sampler's samples of ``rec``."""
  rec = {k: (v.to(dev()) if torch.is_tensor(v) else v) for k, v in rec.items()}
  node_ids, mask, nonempty, nn_idx, _, _ = _sample(rec, mod.num_edgetype + 1, mod.num_sample_neighbors)
  return mod(node_ids, nn_idx.long(), nonempty, label=label, mask=mask)


@pytest.mark.parametrize('agg', ['Mean', 'Max', 'LSTM'])
def test_forward_sparse_equals_padded_forward_on_the_same_samples(agg):
  samples = data.synthetic_qm8_samples(64, seed=31)
  mod = _build(agg).eval()
  with torch.no_grad():
    res = _records(samples, KEYS[0])
    ref = _padded(mod, res)
    for _ in range(3):                 # copy-slot capture, then the resident capture and its replay
      assert torch.equal(mod.forward_sparse(res), ref), agg
    host = _records(samples, KEYS[0], 'pinned')
    for _ in range(2):
      assert torch.equal(mod.forward_sparse(host), ref), agg
    mod.use_cuda_graph = False
    assert torch.equal(mod.forward_sparse(res), ref), agg


def test_forward_sparse_equals_padded_forward_at_1024():
  samples = data.synthetic_qm8_samples(1024, seed=32)
  mod = _build('Mean').eval()
  with torch.no_grad():
    res = _records(samples, KEYS[1])
    assert torch.equal(mod.forward_sparse(res), _padded(mod, res))


@pytest.mark.parametrize('agg', ['Mean', 'Max'])
def test_off_stack_shape_matches_the_padded_forward(agg):
  mod = _build(agg, hidden_dim=[128, 64, 128], num_layer=3).eval()
  assert not mod.stack_supported(26, 7)
  samples = data.synthetic_qm8_samples(64, seed=33)
  with torch.no_grad():
    res = _records(samples, KEYS[0])
    ref = _padded(mod, res)
    got = mod.forward_sparse(res)
  err = float((got - ref).abs().max())
  print('off-stack %s: max|diff| = %.3g, max|score| = %.3g, equal = %s'
        % (agg, err, float(ref.abs().max()), torch.equal(got, ref)))
  assert err <= 1e-6 * float(ref.abs().max())


@pytest.mark.parametrize('where', ['device', 'pinned'])
def test_captured_graph_draws_new_samples_for_a_new_key(where):
  samples = data.synthetic_qm8_samples(64, seed=34)
  mod = _build('Mean').eval()
  with torch.no_grad():
    rec = _records(samples, KEYS[0], where)
    for _ in range(3):
      mod.forward_sparse(rec)
    captures = mod.graph_stats()['captures']
    outs = []
    for key in (KEYS[1], KEYS[2], KEYS[1]):
      rec['sample_key'].copy_(torch.tensor(key, dtype=torch.int64))   # the same buffer, a new key
      outs.append(mod.forward_sparse(rec))
      mod.use_cuda_graph = False
      assert torch.equal(outs[-1], mod.forward_sparse(rec)), key
      assert torch.equal(outs[-1], _padded(mod, rec)), key
      mod.use_cuda_graph = True
    assert mod.graph_stats()['captures'] == captures
    assert not torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def _grads(mod):
  return {n: p.grad.detach().clone() for n, p in mod.named_parameters() if p.grad is not None}


def _padded_grads(mod, rec, label):
  mod.zero_grad(set_to_none=True)
  _, loss = _padded(mod, rec, label=label)
  loss.backward()
  return loss.detach(), _grads(mod)


@pytest.mark.parametrize('where', ['device', 'pinned'])
@pytest.mark.parametrize('agg', ['Mean', 'Max', 'LSTM'])
def test_forward_sparse_train_matches_padded_training(agg, where):
  samples = data.synthetic_qm8_samples(64, seed=35)
  mod = _build(agg, **SMALL).train()
  label = torch.from_numpy(np.random.RandomState(3).randn(64, 16).astype(np.float32)).to(dev())
  rec = _records(samples, KEYS[2], where)
  mod.zero_grad(set_to_none=True)
  _, loss = mod.forward_sparse_train(rec, label=label)
  loss.backward()
  got = _grads(mod)
  ref_loss, want = _padded_grads(mod, rec, label)
  _, again = _padded_grads(mod, rec, label)
  assert set(got) == set(want) and len(got) > 0
  # the backward's scatter-adds (embedding rows, the Max argmax, the LSTM gathers) use atomics, so two padded
  # runs need not agree bit for bit either: the records path is held to the padded path's tolerance
  worst = max(float((got[n] - want[n]).abs().max()) / max(float(want[n].abs().max()), 1e-30) for n in want)
  spread = max(float((again[n] - want[n]).abs().max()) / max(float(want[n].abs().max()), 1e-30) for n in want)
  print('%s: loss %.9g vs %.9g (equal %s); worst gradient diff / max|ref| = %.3g; padded run to run = %.3g'
        % (agg, float(loss), float(ref_loss), torch.equal(loss.detach(), ref_loss), worst, spread))
  assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
  if agg != 'Mean':
    assert torch.equal(loss.detach(), ref_loss), agg
  for n in want:
    err = float((got[n] - want[n]).abs().max())
    assert err <= 1e-5 * float(want[n].abs().max()) + 1e-12, (n, err)


@pytest.mark.parametrize('agg', ['Mean', 'Max', 'LSTM'])
def test_graphed_step_over_records_with_new_keys(agg):
  from lanczosnetwork_b200.train import GraphedStep
  samples = data.synthetic_qm8_samples(32, seed=36)
  label = torch.from_numpy(np.random.RandomState(4).randn(32, 16).astype(np.float32)).to(dev())
  recs = [_records(samples, key) for key in KEYS[:2]]

  def make():
    m = _build(agg, **SMALL).train()
    return m, torch.optim.Adam(m.parameters(), lr=1e-3)

  eager, opt_e = make()
  losses_e = []
  for i in range(4):
    opt_e.zero_grad()
    _, loss = eager.forward_sparse_train(recs[i % 2], label=label)
    loss.backward()
    opt_e.step()
    losses_e.append(float(loss.detach()))
  graphed, opt_g = make()
  step = GraphedStep(graphed, opt_g, (recs[0],), {'label': label}, sparse=True)
  losses_g = [float(step(recs[i % 2], label=label)[1].detach()) for i in range(4)]
  print('%s: eager %s, graphed %s' % (agg, losses_e, losses_g))
  assert losses_e[0] != losses_e[1]
  np.testing.assert_allclose(losses_g, losses_e, rtol=1e-5)
  for (n, p), (_, q) in zip(graphed.named_parameters(), eager.named_parameters()):
    np.testing.assert_allclose(p.detach().cpu().numpy(), q.detach().cpu().numpy(), rtol=2e-4, atol=2e-6, err_msg=n)
  assert step.replays == 4


def test_refusals_launch_nothing():
  samples = data.synthetic_qm8_samples(4, seed=1)
  rec = _records(samples, KEYS[0])
  mod = _build('Mean').eval()
  n0 = ops.launch_count()
  bad = dict(rec)
  bad.pop('sample_key')
  with torch.no_grad(), pytest.raises(ValueError, match='sample_key'):
    mod.forward_sparse(bad)
  bad = dict(rec, N=129)
  with torch.no_grad(), pytest.raises(ValueError, match='N=129'):
    mod.forward_sparse(bad)
  with pytest.raises(ValueError, match='sample_key'):
    _sample(dict(rec, sample_key=rec['sample_key'].int()), 7, 40)
  with pytest.raises(ValueError, match='want_ell_t'):
    _sample(rec, 7, 40, want_ell_t=True)
  with pytest.raises(ValueError):
    _sample(rec, 17, 40)
  assert ops.launch_count() == n0
