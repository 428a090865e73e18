"""SparseLanczosNetGeneral from bond-list records with float feature rows: lnb_graph_prepare_sparse_features
against the golden GraphData batch and against lnb_graph_prepare_sparse, forward_sparse against forward
(records with eigenpairs: the same bits; without: the bits of forward fed the device eigenpairs),
forward_sparse_train against the padded training path, and GraphedStep(sparse=True).  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, load_golden, oracle_spec
from lanczosnetwork_b200 import _lib, configs, data, ops, train
from lanczosnetwork_b200.model import SparseLanczosNetGeneral
from oracle import lanczos_oracle as orc
from test_gpu_sage_sampling import _ell_equal

pytestmark = pytest.mark.gpu

K = 20
FWD_ATOL = 2e-5           # the forward tolerances of test_gpu_models / test_gpu_graph_eigs
FWD_RTOL = 1e-4


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _config(F=10, num_edge_type=1):
  cfg = configs.graph_lanczos_net(input_dim=F)
  cfg.dataset.node_emb_dim = F
  cfg.dataset.num_edge_type = num_edge_type
  return cfg


def _build(cfg=None, seed=7):
  mod = SparseLanczosNetGeneral(cfg or _config())
  mod.load_state_dict(deterministic_state_dict(mod, seed))
  return mod.to(dev()).eval()


def _to(sp, where):
  out = {}
  for k, v in sp.items():
    if isinstance(v, np.ndarray):
      t = torch.from_numpy(v)
      out[k] = t.pin_memory() if where == 'pinned' else t.to(dev())
    else:
      out[k] = v
  return out


def _records(samples, where, eigs):
  return _to(data.sparse_collate(samples, K, eigs=eigs), where)


def _prepare(r, E1, V_rows=None, **kw):
  if V_rows is None:
    V_rows = r['V_rows']
  return ops.graph_prepare_sparse_features(r['sizes'], r['node_ptr'], r['node_feat'], r['edge_ptr'], r['edges'],
                                           V_rows, r['N'], E1, **kw)


def _bits(t):
  return t.contiguous().view(torch.int32)


def _rowmap_equal(got, want):
  """The compact Ritz row lists: the same count and the same rows below it (the rest is never read)."""
  n = int(want.nrows[0])
  assert int(got.nrows[0]) == n and torch.equal(got.rowmap[:n], want.rowmap[:n])


# ---- the golden GraphData batch -----------------------------------------------------------------------
def _golden_records(g, eigs):
  """Records rebuilt from the golden batch: bonds = the upper-triangle non-zeros of L[..., 1], features =
  node_feat; the golden eigenpairs when ``eigs``."""
  samples = []
  for b, n in enumerate(g['sizes'].astype(int)):
    a = np.triu(g['L'][b, :n, :n, 1] != 0, 1).astype(np.float64)
    samples.append(data.prepare_graph((a + a.T)[:, :, None], g['node_feat'][b, :n], eigs=False))
  sp = data.sparse_collate(samples, K, eigs=False)
  if eigs:
    del sp['K']
    sp['D'] = g['D']
    sp['V_rows'] = np.concatenate([g['V'][b, :n] for b, n in enumerate(g['sizes'].astype(int))])
  return sp


def test_prepare_features_reproduces_the_golden_batch():
  g = load_golden('lanczosnet_general_synth.npz')
  r = _to(_golden_records(g, eigs=True), 'device')
  assert r['N'] == g['L'].shape[1]
  prep, X, mask, V, L = _prepare(r, 2, want_dense=True)
  assert torch.equal(_bits(L.cpu()), _bits(_t(g['L'])))
  assert torch.equal(_bits(X.cpu()), _bits(_t(g['node_feat'])))
  assert torch.equal(mask.cpu(), _t(g['node_mask']))
  assert torch.equal(_bits(V.cpu()), _bits(_t(g['V'])))
  _ell_equal(prep, ops.graph_prepare(_t(g['L']).to(dev()), _t(g['V']).to(dev())))
  again = _prepare(r, 2, want_dense=True)                      # repeated launches: the same bits
  _ell_equal(again[0], prep)
  _rowmap_equal(again[0], prep)
  for a, b in zip((X, mask, V, L), again[1:]):
    assert torch.equal(a, b)


def test_forward_sparse_meets_the_golden_scores():
  g = load_golden('lanczosnet_general_synth.npz')
  mod = _build(seed=int(g['weight_seed']))
  with torch.no_grad():
    score = mod.forward_sparse(_to(_golden_records(g, eigs=True), 'device'))
  np.testing.assert_allclose(score.cpu().numpy(), g['score'], rtol=FWD_RTOL, atol=FWD_ATOL)


# ---- the prepare op ------------------------------------------------------------------------------------
def _envelope_samples(F, seed=3, E=2):
  """N = 128, two edge types, a one-node graph, an edgeless graph and G(n, 0.5) graphs."""
  rng = np.random.RandomState(seed)
  sizes = [128, 1, 7] + list(rng.randint(20, 129, size=5))
  out = []
  for i, n in enumerate(sizes):
    a = np.triu(rng.rand(n, n) < 0.5, 1) if i != 2 else np.zeros((n, n), bool)
    kind = rng.randint(0, E, size=(n, n))
    adjs = np.zeros((n, n, E))
    for c in range(E):
      m = (a & (kind == c)).astype(np.float64)
      adjs[:, :, c] = m + m.T
    out.append(data.prepare_graph(adjs, rng.randn(n, F), label=rng.randn(1, 2)))
  return out


@pytest.mark.parametrize('F, misaligned', [(1, False), (4, False), (4, True), (10, False), (33, False),
                                           (64, False), (64, True), (4096, False)])
def test_prepare_features_writes_what_the_atom_id_entry_writes(F, misaligned):
  """Every output of lnb_graph_prepare_sparse on the same bonds, plus X: the feature rows bit for bit, padded
  rows zero, through the 16-byte copy (F % 4 == 0, aligned) and the scalar copy."""
  samples = _envelope_samples(F, seed=F)[:4] if F == 4096 else _envelope_samples(F, seed=F)
  sp = data.sparse_collate(samples, K)
  r = _to(sp, 'device')
  if misaligned:                      # node_x one float past a 16-byte boundary: the scalar path
    buf = torch.empty(r['node_feat'].numel() + 1, device=dev())
    buf[1:].copy_(r['node_feat'].reshape(-1))
    r['node_feat'] = buf[1:].view(r['node_feat'].shape)
  prep, X, mask, V, L = _prepare(r, 3, want_dense=True)
  ids = torch.zeros(r['node_feat'].shape[0], dtype=torch.int32, device=dev())
  prep_i, _, mask_i, V_i, L_i = ops.graph_prepare_sparse(r['sizes'], r['node_ptr'], ids, r['edge_ptr'], r['edges'],
                                                         r['V_rows'], r['N'], 3, want_dense=True)
  _ell_equal(prep, prep_i)
  _rowmap_equal(prep, prep_i)
  assert torch.equal(mask, mask_i) and torch.equal(_bits(V), _bits(V_i)) and torch.equal(_bits(L), _bits(L_i))
  want = torch.zeros((len(samples), r['N'], F))
  for b, s in enumerate(samples):
    want[b, :len(s['node_feat'])] = torch.from_numpy(s['node_feat'].astype(np.float32))
  assert torch.equal(_bits(X.cpu()), _bits(want))
  assert torch.equal(_prepare(r, 3)[1], X)


def test_prepare_features_refusals_launch_nothing():
  r = _records(_envelope_samples(4)[:3], 'device', eigs=True)
  lib = _lib.load()
  out = [torch.empty(1 << 16, device=dev()) for _ in range(11)]
  for N, E1, F in ((129, 3, 4), (128, 17, 4), (128, 1, 4), (128, 3, 0), (128, 3, 4097)):
    n0 = ops.launch_count()
    st = lib.lnb_graph_prepare_sparse_features(
        ops._stream(r['sizes']), ops._ptr(r['sizes']), ops._ptr(r['node_ptr']), ops._ptr(r['node_feat']),
        ops._ptr(r['edge_ptr']), ops._ptr(r['edges']), ops._ptr(r['V_rows']),
        ops._ptr(ops._inv_sqrt_deg_table(dev())), 3, N, E1, K, F, 0, *[ops._ptr(o) for o in out])
    assert st == -2 and ops.launch_count() == n0, (N, E1, F, st)
  torch.cuda.synchronize()


# ---- contracts 1-3 -------------------------------------------------------------------------------------
def _padded(samples, mod, D=None, V=None):
  """forward's arguments on data.collate of the samples (X, L, D, V, mask), D / V replaced when given."""
  c = data.collate(samples, K)
  return (_t(c['node_feat']).to(dev()), _t(c['L']).to(dev()), D if D is not None else _t(c['D']).to(dev()),
          V if V is not None else _t(c['V']).to(dev()), _t(c['node_mask']).to(dev()))


def _device_eigs(samples, E1):
  """D and padded V of ops.graph_eigs_sparse on the records of the samples."""
  r = _records(samples, 'device', eigs=False)
  D, V_rows, st = ops.graph_eigs_sparse(r['sizes'], r['node_ptr'], r['edge_ptr'], r['edges'], r['N'], K,
                                        num_edgetype=E1 - 1)
  assert int(st.abs().sum()) == 0
  return D, _prepare(r, E1, V_rows=V_rows)[3]


def _cases():
  return [('B16', lambda: (data.synthetic_regression_graphs(16, seed=17), _config())),
          ('B64', lambda: (data.synthetic_regression_graphs(64, seed=123), _config())),
          ('envelope_F1', lambda: (_envelope_samples(1), _config(1, 2))),
          ('envelope_F33', lambda: (_envelope_samples(33), _config(33, 2)))]


CASES = dict(_cases())


@pytest.mark.parametrize('where', ['device', 'pinned'])
@pytest.mark.parametrize('case', sorted(CASES))
def test_records_with_eigenpairs_give_the_bits_of_forward(case, where):
  samples, cfg = CASES[case]()
  mod = _build(cfg)
  with torch.no_grad():
    X, L, D, V, mask = _padded(samples, mod)
    want = mod(X, L, D, V, mask=mask)
    rec = _records(samples, where, eigs=True)
    mod.use_cuda_graph = False
    assert torch.equal(mod.forward_sparse(rec), want)
    mod.use_cuda_graph = True
    for _ in range(3):                 # capture, replay (and, from device records, the resident capture)
      assert torch.equal(mod.forward_sparse(rec), want)


@pytest.mark.parametrize('where', ['device', 'pinned'])
@pytest.mark.parametrize('case', sorted(CASES))
def test_records_without_eigenpairs_give_the_bits_of_forward_on_device_eigenpairs(case, where):
  samples, cfg = CASES[case]()
  mod = _build(cfg)
  with torch.no_grad():
    D, V = _device_eigs(samples, mod.num_edgetype + 1)
    X, L, _, _, mask = _padded(samples, mod)
    want = mod(X, L, D, V, mask=mask)
    rec = _records(samples, where, eigs=False)
    mod.use_cuda_graph = False
    got = mod.forward_sparse(rec)
    assert torch.equal(got, want)
    mod.use_cuda_graph = True
    for _ in range(3):
      assert torch.equal(mod.forward_sparse(rec), want)
    host = mod(*_padded(samples, mod)[:4], mask=mask)          # forward with the host's eigenpairs
  keep = np.array([s['D_simple'].shape[0] <= K or abs(s['D_simple'][K - 1]) - abs(s['D_simple'][K]) > 1e-6
                   for s in samples])
  print('%s: excluded %d of %d graphs (|lambda| gap at the K cut <= 1e-6)' % (case, int((~keep).sum()), len(keep)))
  assert keep.sum() >= len(keep) // 2
  np.testing.assert_allclose(got.cpu().numpy()[keep], host.cpu().numpy()[keep], rtol=FWD_RTOL, atol=FWD_ATOL)


def _grads(mod, loss):
  mod.zero_grad(set_to_none=True)
  loss.backward()
  return {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in mod.named_parameters()}


def _oracle_grads(mod, args, label):
  """d loss / d params by autograd over the fp64 oracle on the padded batch."""
  X, L, D, V, mask = [a.cpu().numpy() for a in args]
  p64 = {k: v.detach().cpu().double().requires_grad_(True) for k, v in mod.named_parameters()}
  score = orc.lanczos_net_forward(p64, oracle_spec(mod, 'LanczosNetGeneral'), X, L, D, V, mask, dtype=torch.float64)
  torch.nn.functional.mse_loss(score, label.cpu().double()).backward()
  return {k: v.grad for k, v in p64.items()}


@pytest.mark.parametrize('eigs', [True, False])
@pytest.mark.parametrize('where', ['device', 'pinned'])
@pytest.mark.parametrize('case', sorted(CASES))
def test_forward_sparse_train_matches_the_padded_training_path(case, where, eigs):
  """The loss within 1e-5 relative and every gradient within 1e-4 of its largest entry; a gradient that
  misses the bound is no farther from the fp64 oracle's than the padded path's is."""
  samples, cfg = CASES[case]()
  mod = _build(cfg)
  label = _t(data.sparse_collate(samples, K, eigs=False)['label']).to(dev())
  if eigs:
    args = _padded(samples, mod)
  else:
    args = _padded(samples, mod, *_device_eigs(samples, mod.num_edgetype + 1))
  _, loss_p = mod(*args[:4], label=label, mask=args[4])
  g_p = _grads(mod, loss_p)
  _, loss_s = mod.forward_sparse_train(_records(samples, where, eigs), label=label)
  g_s = _grads(mod, loss_s)
  loss_s, loss_p = float(loss_s.detach()), float(loss_p.detach())
  assert abs(loss_s - loss_p) <= 1e-5 * abs(loss_p), (loss_s, loss_p)
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
      oracle = _oracle_grads(mod, args, label)
    err_s = float((gs.cpu().double() - oracle[n]).abs().max())
    err_p = float((gp.cpu().double() - oracle[n]).abs().max())
    assert err_s <= err_p, (n, 'sparse %g, padded %g from fp64; difference %g, scale %g' % (err_s, err_p, diff, scale))


# ---- captured step -------------------------------------------------------------------------------------
@pytest.mark.parametrize('eigs', [False, True])
def test_graphed_sparse_step_gives_the_eager_losses(eigs):
  """Five Adam steps replayed over three batches of different node and bond totals (one padding target N)
  walk the eager forward_sparse_train losses; the warm-up is rolled back."""
  batches = [data.synthetic_regression_graphs(16, seed=s) for s in (1, 2, 3)]
  recs = [_records(b, 'pinned', eigs) for b in batches]
  N = max(r['N'] for r in recs)
  for r in recs:
    r['N'] = N
  assert len({int(r['node_ptr'][-1]) for r in recs}) == 3 and len({int(r['edge_ptr'][-1]) for r in recs}) == 3
  labels = [_t(data.sparse_collate(b, K, eigs=False)['label']).to(dev()) for b in batches]
  base, eager, graphed = _build(), _build().train(), _build()
  opt_e = torch.optim.Adam(eager.parameters(), lr=1e-3)
  opt_g = torch.optim.Adam(graphed.parameters(), lr=1e-3)
  step = train.GraphedStep(graphed, opt_g, (recs[0],), {'label': labels[0]}, sparse=True,
                           edge_capacity=max(int(r['edges'].shape[0]) for r in recs))
  for (n, p), (_, q) in zip(graphed.named_parameters(), base.named_parameters()):
    assert torch.equal(p, q), n                                # warm-up rolled back
  for i in (0, 1, 2, 0, 1):
    opt_e.zero_grad()
    _, le = eager.forward_sparse_train(recs[i], label=labels[i])
    le.backward()
    opt_e.step()
    _, lg = step(recs[i], label=labels[i])
    np.testing.assert_allclose(float(lg), float(le), rtol=2e-4)
  assert step.replays == 5
