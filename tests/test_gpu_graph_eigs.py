"""The device eigensolver (lnb_graph_eigs_sparse / lnb_sym_eigs) against the reference's preprocessing
(fp64 eigh, descending |lambda|, truncated / zero padded to K) and numpy fp64 across its envelope, and
LanczosNet / LanczosNetGeneral fed with device eigenpairs.  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, load_golden, oracle_spec
from lanczosnetwork_b200 import configs, data, ops, provider
from lanczosnetwork_b200.model import LanczosNet, LanczosNetGeneral
from oracle import lanczos_oracle as orc

pytestmark = pytest.mark.gpu

FWD_ATOL = 2e-5
FWD_RTOL = 1e-4
ORDER_GAP = 1e-9      # adjacent |lambda| further apart than this must keep the reference's order
CLUSTER = 1e-6        # eigenvalues closer than this form one eigenspace (compared as a projector)


def dev():
  return torch.device('cuda:0')


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


def _cuda(sp):
  return {k: (_t(v).to(dev()) if isinstance(v, np.ndarray) else v) for k, v in sp.items()}


def _ref_order(w):
  """The reference's order of an ascending eigh spectrum: np.argsort(-|w|, kind='mergesort')."""
  return np.argsort(-np.abs(w), kind='mergesort')


def _full_spectrum(A):
  w, v = np.linalg.eigh(A)
  o = _ref_order(w)
  return w[o], v[:, o]


def _sparse_records(adjs_list, feats):
  samples = [data.prepare_graph(a, f, eigs=False) for a, f in zip(adjs_list, feats)]
  return samples, data.sparse_collate(samples, 1, eigs=False)


def _check_against_reference(D, V, D_ref, V_ref, A64, K, tol_d, tol_p):
  """One graph: values, order and the projector of every eigenspace kept whole."""
  n = A64.shape[0]
  kk = min(n, K)
  w, _ = _full_spectrum(A64)
  assert np.abs(D[:kk] - D_ref[:kk]).max() <= tol_d, (np.abs(D[:kk] - D_ref[:kk]).max(), n)
  assert not D[kk:].any() and not V[:, kk:].any()
  a = np.abs(D_ref[:kk].astype(np.float64))
  for r in range(kk - 1):
    if a[r] - a[r + 1] > ORDER_GAP:
      assert abs(D[r]) > abs(D[r + 1]), (n, r, D[r], D[r + 1])
  r = 0
  while r < kk:
    e = r + 1
    while e < n and abs(w[e] - w[r]) <= CLUSTER:
      e += 1
    if e <= kk:                                   # the whole eigenspace is kept
      P = V[:, r:e].astype(np.float64) @ V[:, r:e].T.astype(np.float64)
      P_ref = V_ref[:, r:e].astype(np.float64) @ V_ref[:, r:e].T.astype(np.float64)
      assert np.abs(P - P_ref).max() <= tol_p, (n, r, e, np.abs(P - P_ref).max())
    r = e


def test_graph_eigs_sparse_reproduces_the_reference_on_the_golden_molecules():
  g = load_golden('lanczosnet_qm8.npz')
  K = g['D'].shape[1]
  sizes = g['sizes'].astype(int)
  adjs = [g['adjs'][b, :n, :n].astype(np.float64) for b, n in enumerate(sizes)]
  samples, sp = _sparse_records(adjs, [g['node_feat'][b, :n] for b, n in enumerate(sizes)])
  t = _cuda(sp)
  D, V_rows, status = ops.graph_eigs_sparse(t['sizes'], t['node_ptr'], t['edge_ptr'], t['edges'], sp['N'], K)
  assert int(status.abs().sum()) == 0
  D, V_rows = D.cpu().numpy(), V_rows.cpu().numpy()
  repeated = 0
  for b, n in enumerate(sizes):
    A64 = samples[b]['L_simple_4']
    w, _ = _full_spectrum(A64)
    if n > K:                                    # the cut is reproducible only across a gap
      assert abs(w[K - 1]) - abs(w[K]) > 1e-6, (n, abs(w[K - 1]) - abs(w[K]))
    repeated += int((np.diff(np.abs(w[:min(n, K)])) > -1e-12).any())
    V = V_rows[sp['node_ptr'][b]:sp['node_ptr'][b + 1]]
    _check_against_reference(D[b], V, g['D'][b], g['V'][b, :n], A64, K, 2.4e-7, 1e-6)
  assert repeated >= 2          # the fixture exercises the eigenspace check
  assert sorted(int(n) for n in sizes if n > K) == [21, 25, 26]


def test_sym_eigs_reproduces_the_reference_on_the_golden_synthetic_graphs():
  g = load_golden('lanczosnet_general_synth.npz')
  K = g['D'].shape[1]
  L = _t(g['L']).to(dev())
  D, V, status = ops.sym_eigs(L, _t(g['sizes']).to(dev()), K)           # channel 0 read in place
  assert int(status.abs().sum()) == 0
  D, V = D.cpu().numpy(), V.cpu().numpy()
  for b, n in enumerate(g['sizes'].astype(int)):
    A64 = g['L'][b, :n, :n, 0].astype(np.float64)
    w, _ = _full_spectrum(A64)
    if n > K:
      assert abs(w[K - 1]) - abs(w[K]) > 1e-6
    assert not V[b, n:].any()
    _check_against_reference(D[b], V[b, :n], g['D'][b], g['V'][b, :n], A64, K, 1e-6, 1e-6)


# ---- envelope sweep against numpy fp64 -----------------------------------------------------------
def _graphs(n, rng):
  """Adjacency stacks [n, n, E] of the sweep's graph kinds at n nodes."""
  out = []
  out.append(data.synthetic_molecule(rng, n)[1])
  for p in (0.1, 0.5, 0.9):
    a = np.triu(rng.rand(n, n) < p, 1).astype(np.float64)
    out.append((a + a.T)[:, :, None])
  if n >= 2:                                      # the last atom has no bonds
    a = np.zeros((n, n, 6))
    a[:n - 1, :n - 1] = data.synthetic_molecule(rng, n - 1)[1]
    out.append(a)
  out.append((np.ones((n, n)) - np.eye(n))[:, :, None])          # complete graph: eigenvalue 0, n-1 times
  star = np.zeros((n, n))
  star[0, 1:] = star[1:, 0] = 1
  out.append(star[:, :, None])
  if n >= 8:                                      # disjoint copies of one molecule
    m = n // 4
    mol = data.synthetic_molecule(rng, m)[1]
    a = np.zeros((n, n, 6))
    for c in range(4):
      a[c * m:(c + 1) * m, c * m:(c + 1) * m] = mol
    out.append(a)
  E = max(x.shape[2] for x in out)
  return [np.concatenate([x, np.zeros(x.shape[:2] + (E - x.shape[2],))], axis=2) for x in out]


def _check_eigenpairs(D, V, A64, K, what):
  n = A64.shape[0]
  kk = min(n, K)
  w, _ = _full_spectrum(A64)
  assert np.abs(D[:kk] - w[:kk]).max() <= 2.4e-7, (what, np.abs(D[:kk] - w[:kk]).max())
  for r in range(kk - 1):                         # the reference's rule on the values returned
    assert abs(D[r]) > abs(D[r + 1]) or (abs(D[r]) == abs(D[r + 1]) and D[r] <= D[r + 1]), (what, r)
  assert not D[kk:].any() and not V[:, kk:].any(), what
  Vk = V[:, :kk].astype(np.float64)
  res = A64 @ Vk - Vk * D[:kk].astype(np.float64)[None, :]
  assert np.abs(res).max() <= 1e-6, (what, np.abs(res).max())
  assert np.abs(Vk.T @ Vk - np.eye(kk)).max() <= 1e-6, (what, np.abs(Vk.T @ Vk - np.eye(kk)).max())


@pytest.mark.parametrize('n', [1, 2, 3, 17, 26, 32, 33, 64, 100, 128])
def test_envelope_sweep_against_numpy_fp64(n):
  rng = np.random.RandomState(1000 + n)
  adjs = _graphs(n, rng)
  samples, sp = _sparse_records(adjs, [np.zeros(n, np.int64)] * len(adjs))
  t = _cuda(sp)
  ops_A = np.stack([s['L_simple_4'] for s in samples]).astype(np.float32)       # [B, n, n]
  A_dev = _t(np.stack([ops_A, 2 * ops_A], axis=3)).to(dev())                    # channel 0 at stride 2
  sizes_dev = t['sizes']
  for K in (1, 8, 20, 64, 128):
    D, V_rows, st = ops.graph_eigs_sparse(t['sizes'], t['node_ptr'], t['edge_ptr'], t['edges'], n, K,
                                          num_edgetype=sp['num_edgetype'])
    D2, V_rows2, st2 = ops.graph_eigs_sparse(t['sizes'], t['node_ptr'], t['edge_ptr'], t['edges'], n, K,
                                             num_edgetype=sp['num_edgetype'])
    assert torch.equal(D, D2) and torch.equal(V_rows, V_rows2) and torch.equal(st, st2)
    assert int(st.abs().sum()) == 0
    assert tuple(V_rows.shape) == (int(sp['node_ptr'][-1]), K)                # sparse_collate's layout
    Dd, Vd, std = ops.sym_eigs(A_dev, sizes_dev, K)
    Dd2, Vd2, _ = ops.sym_eigs(A_dev, sizes_dev, K)
    assert torch.equal(Dd, Dd2) and torch.equal(Vd, Vd2) and int(std.abs().sum()) == 0
    Dn, Vn, Dp, Vp = D.cpu().numpy(), V_rows.cpu().numpy(), Dd.cpu().numpy(), Vd.cpu().numpy()
    for b, s in enumerate(samples):
      A64 = s['L_simple_4']
      _check_eigenpairs(Dn[b], Vn[sp['node_ptr'][b]:sp['node_ptr'][b + 1]], A64, K, ('sparse', n, K, b))
      _check_eigenpairs(Dp[b], Vp[b], ops_A[b].astype(np.float64), K, ('dense', n, K, b))   # the operator it read
  # the host records of the same graphs: same node_ptr, same V_rows shape
  host = data.sparse_collate([data.prepare_graph(a, np.zeros(n, np.int64)) for a in adjs], 128)
  assert np.array_equal(host['node_ptr'], sp['node_ptr']) and host['V_rows'].shape == tuple(V_rows.shape)


def test_sym_eigs_padding_rows_and_partial_sizes():
  """Rows and columns past sizes[b] are ignored on input and zero on output."""
  rng = np.random.RandomState(7)
  n, N, K = 20, 40, 24
  a = np.triu(rng.rand(n, n) < 0.3, 1).astype(np.float64)
  A64 = data.get_laplacian(a + a.T)
  A = np.full((2, N, N), 7.0, np.float32)
  A[:, :n, :n] = A64
  D, V, st = ops.sym_eigs(_t(A).to(dev()), torch.tensor([n, 0], dtype=torch.int32, device=dev()), K)
  D, V = D.cpu().numpy(), V.cpu().numpy()
  assert int(st.abs().sum()) == 0
  assert not V[0, n:].any() and not D[1].any() and not V[1].any()
  _check_eigenpairs(D[0], V[0, :n], A64, K, 'padded')


def test_refusals_launch_nothing():
  sp = _cuda(_sparse_records([np.ones((3, 3, 1)) - np.eye(3)[:, :, None]], [np.zeros(3, np.int64)])[1])
  A = torch.zeros((1, 129, 129), device=dev())
  for N, K in ((129, 4), (26, 0), (26, 129)):
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match='status -2'):
      ops.graph_eigs_sparse(sp['sizes'], sp['node_ptr'], sp['edge_ptr'], sp['edges'], N, K)
    with pytest.raises(RuntimeError, match='status -2'):
      ops.sym_eigs(A if N == 129 else A[:, :N, :N], torch.tensor([3], dtype=torch.int32, device=dev()), K)
    assert ops.launch_count() == n0


# ---- models --------------------------------------------------------------------------------------
def _build(cls, cfg, seed):
  mod = cls(cfg)
  params = deterministic_state_dict(mod, seed)
  mod.load_state_dict(params)
  return mod.to(dev()).eval(), params


def _no_eigs_batch(sp):
  out = {k: v for k, v in sp.items() if k not in ('D', 'V_rows')}
  out['K'] = sp['D'].shape[1]
  return out


def test_forward_sparse_with_device_eigenpairs_matches_the_reference_golden():
  g = load_golden('lanczosnet_qm8.npz')
  sizes = g['sizes'].astype(int)
  samples = [data.prepare_graph(g['adjs'][b, :n, :n], g['node_feat'][b, :n], eigs=False) for b, n in enumerate(sizes)]
  sp = data.sparse_collate(samples, g['D'].shape[1], eigs=False)
  mod, params = _build(LanczosNet, configs.qm8_lanczos_net(), int(g['weight_seed']))
  with torch.no_grad():
    mod.use_cuda_graph = False
    eager = mod.forward_sparse(_cuda(sp))
    mod.use_cuda_graph = True
    host = {k: (_t(v).pin_memory() if isinstance(v, np.ndarray) else v) for k, v in sp.items()}
    for _ in range(3):
      assert torch.equal(mod.forward_sparse(host), eager)      # graph replay: the bits of eager
    res = _cuda(sp)
    for _ in range(3):
      assert torch.equal(mod.forward_sparse(res), eager)
  score = eager.cpu().numpy()
  np.testing.assert_allclose(score, g['score'], rtol=FWD_RTOL, atol=FWD_ATOL)
  spec = oracle_spec(mod, 'LanczosNet')
  s64 = orc.lanczos_net_forward(params, spec, g['node_feat'], g['L'], g['D'], g['V'], g['node_mask'],
                                dtype=torch.float64).numpy()
  e_ref = np.abs(g['score'] - s64).max()
  e_ours = np.abs(score - s64).max()
  assert e_ours <= max(4 * e_ref, 5e-6), (e_ours, e_ref)


def test_forward_sparse_device_eigenpairs_against_host_eigenpairs_at_qm8_scale():
  samples = data.synthetic_qm8_samples(1024, seed=5)
  K = 20
  sp = data.sparse_collate(samples, K)
  mod, _ = _build(LanczosNet, configs.qm8_lanczos_net(), 1234)
  with torch.no_grad():
    mod.use_cuda_graph = False
    host_eigs = mod.forward_sparse(_cuda(sp))
    dense = data.collate(samples, K)
    want = mod(*[_t(dense[k]).to(dev()) for k in ('node_feat', 'L', 'D', 'V')], mask=_t(dense['node_mask']).to(dev()))
    assert torch.equal(host_eigs, want)           # an eigs=True batch: the bits of forward, as before
    dev_eigs = mod.forward_sparse(_cuda(_no_eigs_batch(sp)))
    mod.use_cuda_graph = True
    assert torch.equal(mod.forward_sparse(_cuda(_no_eigs_batch(sp))), dev_eigs)
  keep = np.array([s['D_simple'].shape[0] <= K or abs(s['D_simple'][K - 1]) - abs(s['D_simple'][K]) > 1e-6
                   for s in samples])
  print('excluded %d of %d molecules (|lambda| gap at the K cut <= 1e-6)' % (int((~keep).sum()), len(keep)))
  assert keep.sum() >= 1000
  np.testing.assert_allclose(dev_eigs.cpu().numpy()[keep], host_eigs.cpu().numpy()[keep], rtol=FWD_RTOL,
                             atol=FWD_ATOL)


def test_exact_eigenpairs_feed_lanczosnet_general_to_the_golden_scores():
  g = load_golden('lanczosnet_general_synth.npz')
  L = _t(g['L']).to(dev())
  mask = _t(g['node_mask']).to(dev())
  D, V, info = provider.exact_eigenpairs(L, mask, g['D'].shape[1])
  assert int(info['status'].abs().sum()) == 0
  D2, V2, _ = provider.exact_eigenpairs(L, _t(g['sizes']).to(dev()), g['D'].shape[1])
  assert torch.equal(D, D2) and torch.equal(V, V2)
  mod, _ = _build(LanczosNetGeneral, configs.graph_lanczos_net(), int(g['weight_seed']))
  with torch.no_grad():
    score = mod(_t(g['node_feat']).to(dev()), L, D, V, mask=mask)
  np.testing.assert_allclose(score.cpu().numpy(), g['score'], rtol=FWD_RTOL, atol=FWD_ATOL)
