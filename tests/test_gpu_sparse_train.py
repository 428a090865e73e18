"""Training from sparse bond-list batches: lnb_ell_messages / lnb_ell_messages_adjoint against fp64 dense
products, the records' operators against their transposes, forward_sparse_train against the padded training
path (loss, every parameter gradient, five steps of momentum SGD and of Adam), and GraphedStep(sparse=True) over batches of
different node and edge totals."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import configs, data, ops, train
from lanczosnetwork_b200.model import DCNN, GCN, GCNFP, GGNN, GPNN, MPNN, ChebyNet, LanczosNet, TrainableGAT

from helpers import deterministic_state_dict
from oracle import ggnn_oracle, gpnn_oracle, mpnn_oracle
from test_gpu_sparse_dropins import _odd_samples

pytestmark = pytest.mark.gpu

K = 20


def dev():
  return torch.device('cuda:0')


# ---- kernels ------------------------------------------------------------------------------------
def _records_operators(samples):
  """(prep, L [B,N,N,E1]) of the records of ``samples`` (lnb_graph_prepare_sparse, dense L on request)."""
  sp = {k: torch.from_numpy(v).to(dev()) if isinstance(v, np.ndarray) else v
        for k, v in data.sparse_collate(samples, K, eigs=False).items()}
  V_rows = torch.zeros((sp['node_feat'].shape[0], 4), device=dev())
  prep, _, _, _, L = ops.graph_prepare_sparse(sp['sizes'], sp['node_ptr'], sp['node_feat'], sp['edge_ptr'],
                                              sp['edges'], V_rows, sp['N'], sp['num_edgetype'] + 1, want_dense=True)
  return prep, prep, L


def _random_operators(B, N, E1, seed):
  """Non-symmetric random operators of a few entries per row, zero past each graph's size, their ELL rows and
  those of their transposes."""
  g = torch.Generator().manual_seed(seed)
  sizes = torch.randint(1, N + 1, (B,), generator=g)
  sizes[0] = N
  live = (torch.arange(N)[None, :] < sizes[:, None]).float()
  keep = (torch.rand((B, N, N, E1), generator=g) < 3.0 / N).float() + torch.eye(N)[None, :, :, None]
  L = torch.randn((B, N, N, E1), generator=g) * (keep > 0).float() * live[:, :, None, None] * live[:, None, :, None]
  L = L.to(dev())
  return ops.graph_prepare(L), ops.graph_prepare(L.transpose(1, 2).contiguous()), L


def _operators(source, E1):
  if source == 'qm8':
    return _records_operators(data.synthetic_qm8_samples(16, seed=4))
  if source == 'odd':
    return _records_operators(_odd_samples())
  return _random_operators(3, int(source[1:]), E1, seed=int(source[1:]) + E1)


def _rows(R, D, strided, seed):
  """A float32 [R, D] operand: contiguous, or a view at column offset 4 of rows of D + 8 floats."""
  g = torch.Generator().manual_seed(seed)
  if not strided:
    return torch.randn((R, D), generator=g).to(dev())
  return torch.randn((R, D + 8), generator=g).to(dev())[:, 4:4 + D]


CASES = [('qm8', 7), ('odd', 7), ('n60', 2), ('n60', 7), ('n128', 16), ('n128', 7)]


@pytest.mark.parametrize('strided', [False, True])
@pytest.mark.parametrize('weighted', [False, True])
@pytest.mark.parametrize('D', [1, 3, 64, 128, 130])
@pytest.mark.parametrize('source, E1', CASES)
def test_ell_messages_match_fp64_dense_products(source, E1, D, weighted, strided):
  prep, prep_t, L = _operators(source, E1)
  B, N, _, E1 = L.shape
  tol = 1e-5 if N == 128 else 2e-6
  c0 = 1 if strided else 0
  nc = E1 - c0
  L64 = L.double()
  w = (torch.rand((B, N, E1), generator=torch.Generator().manual_seed(D)) + 0.5).to(dev()) if weighted else None
  w64 = w.double() if weighted else torch.ones((B, N, E1), dtype=torch.float64, device=dev())
  # forward, into column block col0 of a wider message matrix when strided
  X = _rows(B * N, D, strided, seed=D + 1)
  col0 = 4 if strided else 0
  out = torch.full((B * N, col0 + nc * D + (4 if strided else 0)), float('nan'), device=dev())
  res = ops.ell_messages(X, prep, c0, nc, w=w, out=out, col0=col0)[:, col0:col0 + nc * D]
  assert bool(out[:, :col0].isnan().all()) and bool(out[:, col0 + nc * D:].isnan().all())   # nothing outside the block
  X64 = X.double().reshape(B, N, D)
  ref = torch.cat([torch.bmm(L64[..., e], X64) * w64[:, :, e:e + 1] for e in range(c0, E1)], dim=2)
  ref = ref.reshape(B * N, nc * D)
  scale = max(float(ref.abs().max()), 1e-30)
  assert float((res.double() - ref).abs().max()) <= tol * scale
  again = torch.full_like(out, float('nan'))
  assert torch.equal(ops.ell_messages(X, prep, c0, nc, w=w, out=again, col0=col0)[:, col0:col0 + nc * D], res)
  n_eff = prep[3][:, 0].long()
  past = (torch.arange(N, device=dev())[None, :] >= n_eff[:, None]).reshape(B * N)
  assert bool((res[past] == 0).all())
  # adjoint: sum_e L_e^T (w_e . G_e)
  G = _rows(B * N, nc * D, strided, seed=D + 2)
  gX = ops.ell_messages_adjoint(G, prep_t, D, c0, nc, w=w)
  G64 = G.double().reshape(B, N, nc, D)
  ref_t = sum(torch.bmm(L64[..., e].transpose(1, 2), w64[:, :, e:e + 1] * G64[:, :, e - c0]) for e in range(c0, E1))
  ref_t = ref_t.reshape(B * N, D)
  scale = max(float(ref_t.abs().max()), 1e-30)
  assert float((gX.double() - ref_t).abs().max()) <= tol * scale
  assert torch.equal(ops.ell_messages_adjoint(G, prep_t, D, c0, nc, w=w), gX)
  past_t = (torch.arange(N, device=dev())[None, :] >= prep_t[3][:, 0].long()[:, None]).reshape(B * N)
  assert bool((gX[past_t] == 0).all())


@pytest.mark.parametrize('which', ['qm8', 'qm8_1024', 'odd'])
def test_records_operators_equal_their_transposes(which):
  """The records' adjoint reads prep itself as the transposed rows: every dense operator the records give
  (graph_prepare_sparse's L, the partition's L_cluster and L_cut) equals its transpose bit for bit."""
  samples = (_odd_samples() if which == 'odd' else
             data.synthetic_qm8_samples(1024 if which == 'qm8_1024' else 64, seed=9))
  _, _, L = _records_operators(samples)
  bad = int((L != L.transpose(1, 2)).sum())
  assert bad == 0, '%d of %d entries differ from their transposes' % (bad, L.numel())
  sp = {k: torch.from_numpy(v).to(dev()) if isinstance(v, np.ndarray) else v
        for k, v in data.sparse_collate(samples, K, eigs=False).items()}
  if not ops.spectral_partition_supported(sp['N'], 3):
    return
  _, _, _, Lc, Lt = ops.spectral_partition_sparse(sp['sizes'], sp['edge_ptr'], sp['edges'], sp['N'], 3,
                                                  sp['num_edgetype'], want_dense=True)
  for P in (Lc, Lt):
    bad = int((P != P.transpose(1, 2)).sum())
    assert bad == 0, '%d of %d partition entries differ from their transposes' % (bad, P.numel())


@pytest.mark.parametrize('binarize, avg', [(False, False), (True, False), (True, True)])
def test_ell_products_give_the_dense_training_paths_bits(binarize, avg):
  """train.operator_messages and its adjoint over the records' ELL rows equal the dense path's on the same
  operators bit for bit: every channel at once, one channel, and the 0/1 operators row-normalised for avg."""
  samples = data.synthetic_qm8_samples(64, seed=13)
  prep, _, L = _records_operators(samples)
  if binarize:
    prep = ops.graph_prepare(L, binarize=True)
    L = (L != 0).float()
  op = train.ell_operator(prep)
  if avg:
    L, op = train._row_normalised(L).contiguous(), train._row_normalised(op)
  B, N = L.shape[0], L.shape[1]
  X = torch.randn((B, N, 24), generator=torch.Generator().manual_seed(1)).to(dev()).requires_grad_(True)
  for c0, nc in ((0, None), (0, 1), (2, 1), (1, 6)):
    yd = train.operator_messages(L, X, c0, nc)
    ys = train.operator_messages(op, X, c0, nc)
    assert torch.equal(yd, ys), (c0, nc)
    g = torch.randn(yd.shape, generator=torch.Generator().manual_seed(2)).to(dev())
    assert torch.equal(torch.autograd.grad(yd, X, g)[0], torch.autograd.grad(ys, X, g)[0]), (c0, nc)


# ---- models -------------------------------------------------------------------------------------
MODELS = {
    'LanczosNet': lambda: LanczosNet(configs.qm8_lanczos_net()),
    'LanczosNet_device_eigs': lambda: LanczosNet(configs.qm8_lanczos_net()),
    'GCN': lambda: GCN(configs.qm8_gcn()),
    'GCNFP': lambda: GCNFP(configs.qm8_gcn()),
    'GCN_unfused': lambda: GCN(configs.qm8_gcn(hidden_dim=[128, 64, 128], num_layer=3)),
    'DCNN': lambda: DCNN(configs.qm8_dcnn()),
    'ChebyNet': lambda: ChebyNet(configs.qm8_cheby_net()),
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


def _build(name, seed=7):
  mod = MODELS[name]()
  mod.load_state_dict(deterministic_state_dict(mod, seed))
  return mod.to(dev()).eval()          # eval: no dropout; autograd on: the training formulation runs


def _records(name, samples, where):
  sp = data.sparse_collate(samples, K, eigs=(name == 'LanczosNet'))
  out = {}
  for k, v in sp.items():
    if isinstance(v, np.ndarray):
      t = torch.from_numpy(v)
      out[k] = t.pin_memory() if where == 'pinned' else t.to(dev())
    else:
      out[k] = v
  return out


def _padded_call(name, mod, samples, label):
  """The padded training path on data.collate of the same samples (device eigenpairs: those of
  graph_eigs_sparse on the records, padded)."""
  c = data.collate(samples, K)
  nf = torch.from_numpy(c['node_feat']).to(dev())
  mask = torch.from_numpy(c['node_mask']).to(dev())
  L = torch.from_numpy(data.gat_bias(c['L']) if 'GAT' in name else c['L']).to(dev())
  if name == 'LanczosNet':
    return mod(nf, L, torch.from_numpy(c['D']).to(dev()), torch.from_numpy(c['V']).to(dev()), label=label, mask=mask)
  if name == 'LanczosNet_device_eigs':
    r = _records(name, samples, 'device')
    D, V_rows, _ = ops.graph_eigs_sparse(r['sizes'], r['node_ptr'], r['edge_ptr'], r['edges'], r['N'], K,
                                         num_edgetype=mod.num_edgetype)
    V = ops.graph_prepare_sparse(r['sizes'], r['node_ptr'], r['node_feat'], r['edge_ptr'], r['edges'], V_rows,
                                 r['N'], mod.num_edgetype + 1)[3]
    return mod(nf, L, D, V, label=label, mask=mask)
  return mod(nf, L, label=label, mask=mask)


def _grads(mod, loss):
  mod.zero_grad(set_to_none=True)
  loss.backward()
  return {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in mod.named_parameters()}


def _oracle_grads(name, mod, samples, label):
  """d loss / d params by autograd over the model's fp64 oracle on the collated batch (GPNN: the partition
  operators of the device partition, as both paths use), or None for models without one here."""
  c = data.collate(samples, K)
  p64 = {k: v.detach().cpu().double().requires_grad_(True) for k, v in mod.named_parameters()}
  if name.startswith('GGNN'):
    spec = ggnn_oracle.make_spec(mod.num_prop, mod.aggregate_type, mod.update_func_name, mod.num_edgetype)
    score = ggnn_oracle.ggnn_forward(p64, spec, c['node_feat'], c['L'], c['node_mask'], dtype=torch.float64,
                                     cast=False)
  elif name.startswith('GPNN'):
    _, Lc, Lt, _ = ops.spectral_partition(torch.from_numpy(c['L']).to(dev()), mod.num_partition)
    spec = gpnn_oracle.make_spec(mod.num_prop, mod.num_prop_cluster, mod.num_prop_cut, mod.aggregate_type,
                                 mod.update_func_name, mod.num_edgetype)
    score = gpnn_oracle.gpnn_forward(p64, spec, c['node_feat'], c['L'], Lc.cpu().numpy(), Lt.cpu().numpy(),
                                     c['node_mask'], dtype=torch.float64, cast=False)
  elif name.startswith('MPNN'):
    spec = mpnn_oracle.make_spec(mod.num_prop, mod.aggregate_type, mod.msg_func_name, mod.num_edgetype,
                                 mod.num_step_set2vec)
    score = mpnn_oracle.mpnn_forward(p64, spec, c['node_feat'], c['L'], c['node_mask'], dtype=torch.float64,
                                     cast=False)
  else:
    return None
  torch.nn.functional.mse_loss(score, label.cpu().double()).backward()
  return {k: v.grad for k, v in p64.items()}


def _compare(name, mod, samples, where):
  """The loss within 1e-5 relative and every parameter gradient within 1e-4 of its largest entry.  A gradient
  that misses the bound is put to the model's fp64 oracle: the sparse path must be no farther from it than
  the padded path is."""
  label = torch.from_numpy(data.sparse_collate(samples, K, eigs=False)['label']).to(dev())
  _, loss_p = _padded_call(name, mod, samples, label)
  g_p = _grads(mod, loss_p)
  _, loss_s = mod.forward_sparse_train(_records(name, samples, where), label=label)
  g_s = _grads(mod, loss_s)
  assert abs(float(loss_s) - float(loss_p)) <= 1e-5 * abs(float(loss_p)), (name, float(loss_s), float(loss_p))
  oracle = None
  for n, gp in g_p.items():
    gs = g_s[n]
    assert (gp is None) == (gs is None), n
    if gp is None:
      continue
    scale = float(gp.abs().max())
    diff = float((gs - gp).abs().max())
    if diff <= 1e-4 * scale:
      continue
    if oracle is None:
      oracle = _oracle_grads(name, mod, samples, label)
    assert oracle is not None, (name, n, diff, scale)
    ref = oracle[n]
    err_s = float((gs.cpu().double() - ref).abs().max())
    err_p = float((gp.cpu().double() - ref).abs().max())
    assert err_s <= err_p, (name, n, 'sparse %g, padded %g from fp64; difference %g, scale %g'
                            % (err_s, err_p, diff, scale))


@pytest.mark.parametrize('where', ['device', 'pinned'])
@pytest.mark.parametrize('name', sorted(MODELS))
def test_forward_sparse_train_matches_the_padded_training_path(name, where):
  _compare(name, _build(name), data.synthetic_qm8_samples(64, seed=67), where)


@pytest.mark.parametrize('name', ['GCN', 'GGNN', 'MPNN', 'GPNN'])
def test_forward_sparse_train_at_b1024(name):
  _compare(name, _build(name), data.synthetic_qm8_samples(1024, seed=1027), 'device')


@pytest.mark.parametrize('name', sorted(MODELS))
def test_forward_sparse_train_odd_graphs(name):
  _compare(name, _build(name, seed=3), _odd_samples(), 'device')


def test_forward_sparse_train_without_autograd_returns_the_same_score():
  samples = data.synthetic_qm8_samples(64, seed=67)
  mod = _build('GGNN')
  rec = _records('GGNN', samples, 'device')
  score = mod.forward_sparse_train(rec)
  with torch.no_grad():
    assert torch.equal(mod.forward_sparse_train(rec), score.detach())


def _optimizer(mod):
  # momentum SGD, as test_graphed_training_step_matches_eager_steps compares weights: Adam's m / sqrt(v)
  # turns fp32 reorderings into +-lr moves where a gradient is ~ 0 (measured: a few elements per tensor)
  return torch.optim.SGD(mod.parameters(), lr=1e-2, momentum=0.9)


@pytest.mark.parametrize('name', sorted(MODELS))
def test_five_steps_match_the_padded_path(name):
  samples = data.synthetic_qm8_samples(64, seed=71)
  label = torch.from_numpy(data.sparse_collate(samples, K, eigs=False)['label']).to(dev())
  rec = _records(name, samples, 'device')
  pad, sp = _build(name), _build(name)
  opt_p, opt_s = _optimizer(pad), _optimizer(sp)
  for step in range(5):
    opt_p.zero_grad()
    _, lp = _padded_call(name, pad, samples, label)
    lp.backward()
    opt_p.step()
    opt_s.zero_grad()
    _, ls = sp.forward_sparse_train(rec, label=label)
    ls.backward()
    opt_s.step()
    assert abs(float(ls) - float(lp)) <= 1e-5 * abs(float(lp)), (name, step, float(ls), float(lp))
  for (n, p), (_, q) in zip(pad.named_parameters(), sp.named_parameters()):
    torch.testing.assert_close(q, p, rtol=2e-4, atol=2e-6, msg=lambda m: '%s %s: %s' % (name, n, m))


@pytest.mark.parametrize('name', sorted(MODELS))
def test_five_adam_steps_give_the_padded_losses(name):
  """Adam over records walks the padded path's loss trajectory (the weights are compared under momentum SGD
  above, as Adam moves a weight by about lr wherever its gradient is ~ 0 and changes sign in the last bit)."""
  samples = data.synthetic_qm8_samples(64, seed=71)
  label = torch.from_numpy(data.sparse_collate(samples, K, eigs=False)['label']).to(dev())
  rec = _records(name, samples, 'device')
  pad, sp = _build(name), _build(name)
  opt_p = torch.optim.Adam(pad.parameters(), lr=1e-3)
  opt_s = torch.optim.Adam(sp.parameters(), lr=1e-3)
  for step in range(5):
    opt_p.zero_grad()
    _, lp = _padded_call(name, pad, samples, label)
    lp.backward()
    opt_p.step()
    opt_s.zero_grad()
    _, ls = sp.forward_sparse_train(rec, label=label)
    ls.backward()
    opt_s.step()
    assert abs(float(ls) - float(lp)) <= 1e-5 * abs(float(lp)), (name, step, float(ls), float(lp))


# ---- captured step ------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['GCN', 'GGNN', 'MPNN', 'GPNN', 'LanczosNet_device_eigs'])
def test_graphed_sparse_step_replays_batches_of_different_totals(name):
  batches = [data.synthetic_qm8_samples(64, seed=s) for s in (1, 2, 3)]
  recs = [_records(name, b, 'pinned') for b in batches]
  assert len({r['N'] for r in recs}) == 1
  assert len({int(r['node_ptr'][-1]) for r in recs}) == 3 and len({int(r['edge_ptr'][-1]) for r in recs}) == 3
  labels = [torch.from_numpy(data.sparse_collate(b, K, eigs=False)['label']).to(dev()) for b in batches]
  base = _build(name)
  eager, graphed = _build(name).train(), _build(name)
  opt_e, opt_g = _optimizer(eager), _optimizer(graphed)
  step = train.GraphedStep(graphed, opt_g, (recs[0],), {'label': labels[0]}, sparse=True)
  for (n, p), (_, q) in zip(graphed.named_parameters(), base.named_parameters()):
    assert torch.equal(p, q), n                                # warm-up rolled back
  for r, lab in zip(recs, labels):
    opt_e.zero_grad()
    _, le = eager.forward_sparse_train(r, label=lab)
    le.backward()
    opt_e.step()
    _, lg = step(r, label=lab)
    assert abs(float(lg) - float(le)) <= 1e-5 * abs(float(le)), (name, float(lg), float(le))
  assert step.replays == 3
  for (n, p), (_, q) in zip(eager.named_parameters(), graphed.named_parameters()):
    torch.testing.assert_close(q, p, rtol=2e-4, atol=2e-6, msg=lambda m: '%s %s: %s' % (name, n, m))
  big = _records(name, data.synthetic_qm8_samples(64, seed=1), 'device')
  big['edges'] = torch.cat([big['edges']] * 80)                 # more rows than the captured buffer
  with pytest.raises(ValueError, match='edges'):
    step(big, label=labels[0])
  with pytest.raises(ValueError):
    step(_records(name, data.synthetic_qm8_samples(32, seed=1), 'device'), label=labels[0][:32])
  before = {k: v.clone() for k, v in step._args[0].items() if torch.is_tensor(v)}
  with pytest.raises(ValueError, match='label'):
    step(recs[1], label=labels[1][0])                            # [16] would broadcast into [64, 16]
  assert all(torch.equal(step._args[0][k], v) for k, v in before.items())   # refused before any copy
