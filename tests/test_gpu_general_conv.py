"""The general-shape spectral convolution path (``spectral_conv.graph_conv_layer_unfused``, the layer of
every shape the fused kernel does not take), the kernels on that path at the edges of their envelopes,
and the models that run it off the QM8 shape, against fp64 restatements of the same math.

Every result is bounded by max(c |fp32 restatement - fp64|, floor * scale): c = 4 for FFMA-only kernels,
c = 8 where the 3xTF32 dense layer is involved; scale is the largest |fp64| value of the result
compared.  Each sweep prints its worst error divided by its bound.

The layer is routed through each of its three branches the inputs are eligible for -- one
``graph_messages`` launch, ``operator_chain`` plus batched GEMMs, the per-step batched GEMM chain -- by
monkeypatching the dispatch predicates, and the branches are checked against fp64 and each other.
Operators are non-symmetric and valued (channel 0 is D A D^-1 with A symmetric, scaled to spectral
radius 1, so 65-step power walks and 64-step Chebyshev chains stay bounded), graphs are ragged
with operators and Ritz / Lanczos rows zero past each graph's n, and dense filters include
non-symmetric G, so a transposed G in any branch fails.  ``pytest -m gpu``.

Floors calibrated on an H100 80GB HBM3 (700 W); the worst err / bound measured there per sweep:
  layer on every branch         0.24   (c = 8, KERNEL_FLOOR)
  operator_chain                0.25   (c = 4, FFMA_FLOOR per step; with a flat floor a 63-step
                                        Chebyshev chain reached 0.97: its rounding compounds per step)
  graph_messages corner         0.20   (c = 4, FFMA_FLOOR)
  gaussian_laplacian            0.10   (c = 4, FFMA_FLOOR)
  readout                       0.26   (c = 4, FFMA_FLOOR)
  tridiag_powers                0.11   (c = 4, FFMA_FLOOR)
  models: Le 0.09 (the 2e-6 floor of the full-QM8 test), Lanczos T 0.14 (floor 5e-5), scores 0.27
  (c = 8, KERNEL_FLOOR per layer)."""
import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, oracle_spec
from lanczosnetwork_b200 import configs, data
from oracle import lanczos_oracle as orc

pytestmark = pytest.mark.gpu

# Floor of a layer's error relative to its output's scale: the bound of the fused-layer suite (~K/8
# truncating accumulation steps of the 3xTF32 dense layer); models compound it per layer.
KERNEL_FLOOR = 8e-6
# Floor of the FFMA-only kernels (operator chain, messages, Laplacian, readout, powers of T).
FFMA_FLOOR = 2e-6

_WORST = {}


def dev():
  return torch.device('cuda:0')


def ops():
  from lanczosnetwork_b200 import ops as _ops
  return _ops


@pytest.fixture(scope='module', autouse=True)
def _report_worst():
  yield
  for k in sorted(_WORST):
    print('worst err/bound %-20s %.3g' % (k, _WORST[k]))


def _check(out, ref64, ref32, c, floor, sweep, what, scale=None):
  """|out - ref64| <= max(c |ref32 - ref64|, floor * scale); NaNs must sit where the reference has them."""
  out = out.detach().double().cpu()
  ref64, ref32 = ref64.double(), ref32.double()
  nan = torch.isnan(ref64)
  assert torch.equal(torch.isnan(out), nan), (what, 'NaN pattern')
  if bool(nan.all()):
    return
  keep = ~nan
  err = (out[keep] - ref64[keep]).abs().max().item()
  err32 = (ref32[keep] - ref64[keep]).abs().max().item()
  if scale is None:
    scale = ref64[keep].abs().max().item()
  bound = max(c * err32, floor * scale)
  ratio = err / bound if bound > 0 else (0.0 if err == 0 else float('inf'))
  _WORST[sweep] = max(_WORST.get(sweep, 0.0), ratio)
  print('%s: err/bound %.3g (err %.3g, fp32 %.3g, scale %.3g)' % (what, ratio, err, err32, scale))
  assert err <= bound, (what, err, err32, scale)


def _refused(fn):
  """The call raises RuntimeError before launching anything."""
  o = ops()
  n0 = o.launch_count()
  with pytest.raises(RuntimeError):
    fn()
  assert o.launch_count() == n0


def _spy(fn, name, calls):
  def wrapped(*a, **k):
    calls.append(name)
    return fn(*a, **k)
  return wrapped


# ------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------
def _sizes(rng, B, N):
  sizes = rng.randint(1, N + 1, size=B)
  sizes[0] = N
  return sizes


def _walk_operator(rng, n):
  """D A D^-1, A symmetric, sparse and valued, scaled to spectral radius 1: non-symmetric with a real
  spectrum in [-1, 1], so power walks and Chebyshev chains stay within max(D) / min(D) = 4."""
  A = rng.randn(n, n) * (rng.rand(n, n) < min(1.0, 4.0 / n))
  A = (A + A.T) / 2
  r = np.abs(np.linalg.eigvalsh(A)).max()
  if r > 0:
    A /= r
  d = rng.uniform(0.5, 2.0, size=n)
  return d[:, None] * A / d[None, :]


def _operators(rng, B, N, E1, sizes):
  """L [B,N,N,E1]: channel 0 a walk operator, the others sparse random values; zero past each n."""
  L = np.zeros((B, N, N, E1))
  for b, n in enumerate(sizes):
    n = int(n)
    L[b, :n, :n, 0] = _walk_operator(rng, n)
    for e in range(1, E1):
      L[b, :n, :n, e] = rng.randn(n, n) * (rng.rand(n, n) < min(1.0, 4.0 / n))
  return torch.from_numpy(L.astype(np.float32))


def _basis(rng, B, N, K, sizes):
  """Orthonormal columns on each graph's leading n rows (min(K, n) of them), zero elsewhere."""
  Q = np.zeros((B, N, K))
  for b, n in enumerate(sizes):
    n = int(n)
    kk = min(K, n)
    Q[b, :n, :kk] = np.linalg.qr(rng.randn(n, kk))[0]
  return torch.from_numpy(Q.astype(np.float32))


def _filters(rng, B, K, S, kind):
  if kind == 'diag':
    return torch.from_numpy(rng.randn(B, K, S).astype(np.float32))
  G = rng.randn(B, S, K, K) / np.sqrt(K)
  if kind == 'dense':
    G = (G + G.transpose(0, 1, 3, 2)) / 2
  return torch.from_numpy(G.astype(np.float32))


def _messages_ref(X, L, Q, filt, dense, short):
  """The message blocks [L_0^k X (k in short, ascending)] ++ [Q G_s Q^T X] ++ [L_e X] in X's dtype."""
  L = L.to(X.dtype)
  blocks = []
  walk = X
  for step in range(1, (max(short) if short else 0) + 1):
    walk = torch.bmm(L[..., 0], walk)
    if step in short:
      blocks.append(walk)
  if filt is not None:
    Q, filt = Q.to(X.dtype), filt.to(X.dtype)
    U = Q.transpose(1, 2) @ X
    S = filt.shape[1] if dense else filt.shape[2]
    for s in range(S):
      W = filt[:, s] @ U if dense else filt[:, :, s:s + 1] * U
      blocks.append(Q @ W)
  for e in range(L.shape[3]):
    blocks.append(torch.bmm(L[..., e], X))
  return blocks


def _molecules(sizes, K, num_bond_type=6, seed=0, feat_dim=None):
  """data.collate of synthetic molecules with the given node counts (float features when feat_dim)."""
  rng = np.random.RandomState(seed)
  samples = []
  for n in sizes:
    nf, adjs = data.synthetic_molecule(rng, int(n), num_bond_type)
    if feat_dim:
      nf = rng.randn(int(n), feat_dim).astype(np.float32)
    samples.append(data.prepare_graph(adjs, nf))
  return data.collate(samples, K)


def _build(cls, cfg, seed):
  mod = cls(cfg)
  params = deterministic_state_dict(mod, seed)
  mod.load_state_dict(params)
  return mod.to(dev()).eval(), params


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(a))


# ------------------------------------------------------------------------------------------
# 1. the layer, on every branch
# ------------------------------------------------------------------------------------------
LAYER_CASES = [
    # N, K, S, E1, short, Din, H
    (1, 1, 1, 1, [1], 3, 16),
    (1, 4, 9, 16, [65], 64, 36),
    (7, 4, 8, 7, [3, 1, 2], 10, 36),
    (7, 20, 9, 16, [1], 1, 16),
    (7, 1, 1, 17, [], 130, 128),
    (31, 20, 1, 17, [64], 1, 36),
    (31, 1, 0, 7, [], 10, 16),
    (31, 32, 8, 16, [64], 64, 128),
    (32, 32, 8, 16, [3, 1, 2], 130, 36),
    (32, 33, 1, 7, [1], 10, 128),
    (32, 40, 8, 1, [], 3, 16),
    (32, 4, 0, 17, [65], 3, 36),
    (33, 20, 8, 7, [3, 1, 2], 64, 128),
    (33, 40, 9, 1, [], 3, 36),
    (64, 40, 1, 7, [1], 10, 128),
    (64, 40, 8, 16, [65], 1, 36),
    (64, 32, 9, 17, [1], 64, 16),
    (130, 40, 1, 7, [3, 1, 2], 3, 128),
    (130, 33, 0, 1, [64], 130, 36),
    (130, 20, 8, 16, [1], 64, 128),
]


def _layer_params():
  out = []
  for i, (N, K, S, E1, short, Din, H) in enumerate(LAYER_CASES):
    for kind in (('diag', 'dense', 'dense_nonsym') if S else ('diag',)):
      out.append(pytest.param(i, N, K, S, E1, short, Din, H, kind,
                              id='N%d-K%d-S%d-E%d-short%s-Din%d-H%d-%s' % (
                                  N, K, S, E1, '.'.join(map(str, short)) or 'none', Din, H, kind)))
  return out


def _layer_ref(X, L, Q, filt, dense, short, W, bias):
  """oracle.conv_layer with Lf[..., s] = Q G_s Q^T (dense) or Q diag(f_s) Q^T, in X's dtype."""
  dt = X.dtype
  S = 0 if filt is None else (filt.shape[1] if dense else filt.shape[2])
  Lf = None
  if S:
    Q, filt = Q.to(dt), filt.to(dt)
    Qt = Q.transpose(1, 2)
    Lf = torch.stack([(Q @ filt[:, s] if dense else Q * filt[:, :, s].unsqueeze(1)) @ Qt
                      for s in range(S)], dim=3)
  spec = {'short': list(short), 'long': list(range(1, S + 1)), 'num_edgetype': L.shape[3] - 1}
  params = {'filter.0.weight': W.to(dt), 'filter.0.bias': bias.to(dt)}
  return orc.conv_layer(params, spec, 0, X, L.to(dt), Lf)


@pytest.mark.parametrize('case,N,K,S,E1,short,Din,H,kind', _layer_params())
def test_unfused_layer_every_branch_vs_fp64(case, N, K, S, E1, short, Din, H, kind, monkeypatch):
  from lanczosnetwork_b200 import spectral_conv as sc
  o = ops()
  rng = np.random.RandomState(1000 + 10 * case + ('diag', 'dense', 'dense_nonsym').index(kind))
  B = 4
  sizes = _sizes(rng, B, N)
  L = _operators(rng, B, N, E1, sizes)
  dense = kind != 'diag'
  Q = _basis(rng, B, N, K, sizes) if S else None
  filt = _filters(rng, B, K, S, kind) if S else None
  X = torch.from_numpy(rng.randn(B, N, Din).astype(np.float32))
  C = len(short) + S + E1
  W = torch.from_numpy((rng.randn(H, C * Din) / np.sqrt(C * Din)).astype(np.float32))
  bias = torch.from_numpy((rng.randn(H) * 0.1).astype(np.float32))
  d = dev()
  Xg, Lg, Wg, bg = X.to(d), L.to(d), W.to(d), bias.to(d)
  Qg = Q.to(d) if S else None
  fg = filt.to(d) if S else None

  max_short = max(short) if short else 0
  branches = []
  if o.graph_messages_supported(N, K if S else 0, E1, S, max_short):
    branches.append('messages')
  if short and o.operator_chain_supported(N, max_short):
    branches.append('chain')
  branches.append('bgemm')
  expected_calls = {'messages': ['graph_messages'], 'chain': ['operator_chain'], 'bgemm': []}
  outs = {}
  for br in branches:
    calls = []
    with monkeypatch.context() as m:
      if br != 'messages':
        m.setattr(o, 'graph_messages_supported', lambda *a: False)
      if br == 'bgemm':
        m.setattr(o, 'operator_chain_supported', lambda *a: False)
      for name in ('graph_messages', 'operator_chain'):
        m.setattr(o, name, _spy(getattr(o, name), name, calls))
      outs[br] = sc.graph_conv_layer_unfused(Xg, Lg, Qg, fg, dense, short, S, Wg, bg, sc.WeightCache(),
                                             'filter.0')
    assert calls == expected_calls[br], (br, calls)
    assert outs[br].shape == (B, N, H)

  ref64 = _layer_ref(X.double(), L, Q, filt, dense, short, W, bias)
  ref32 = _layer_ref(X, L, Q, filt, dense, short, W, bias)
  tag = 'layer N=%d K=%d S=%d E1=%d short=%s Din=%d H=%d %s' % (N, K, S, E1, short, Din, H, kind)
  for br in branches:
    _check(outs[br], ref64, ref32, 8, KERNEL_FLOOR, 'layer', '%s [%s]' % (tag, br))
  # the branches agree with each other within one layer bound
  first = outs[branches[0]].double().cpu()
  bound = max(8 * (ref32.double() - ref64).abs().max().item(), KERNEL_FLOOR * ref64.abs().max().item())
  for br in branches[1:]:
    diff = (outs[br].double().cpu() - first).abs().max().item()
    assert diff <= bound, (tag, branches[0], br, diff, bound)


# ------------------------------------------------------------------------------------------
# 2. kernel sweeps at the edges of their envelopes
# ------------------------------------------------------------------------------------------
def _chain_ref(L0, X, steps, cheby):
  """Every step of the power walk w_s = L_0 w_{s-1} or of the Chebyshev chain s_0 = L_0 X,
  s_k = 2 L_0 s_{k-1} - s_{k-2}, s_{-1} = X, in X's dtype."""
  L0 = L0.to(X.dtype)
  prev2, cur, out = X, X, []
  for s in range(steps):
    nxt = torch.bmm(L0, cur)
    if cheby and s > 0:
      nxt = 2.0 * nxt - prev2
    prev2, cur = cur, nxt
    out.append(nxt)
  return out


def _chain_cases():
  cases = []
  for i, (N, steps) in enumerate((n, s) for n in (1, 2, 17, 32) for s in (1, 2, 63, 64)):
    D = (1, 127, 128, 129, 300)[i % 5]
    E1 = (1, 17)[(i // 2) % 2]
    cases.append(pytest.param(N, steps, D, E1, id='N%d-steps%d-D%d-E%d' % (N, steps, D, E1)))
  return cases


@pytest.mark.parametrize('cheby', [False, True], ids=['power', 'chebyshev'])
@pytest.mark.parametrize('N,steps,D,E1', _chain_cases())
def test_operator_chain_envelope(N, steps, D, E1, cheby):
  """Selected steps land in their column block after out_col0, in any block order; unselected steps,
  the blocks in front of out_col0 and the columns past the last block stay untouched."""
  rng = np.random.RandomState(N * 1000 + steps * 10 + E1 + int(cheby))
  B = 3
  sizes = _sizes(rng, B, N)
  L = _operators(rng, B, N, E1, sizes)
  X = torch.from_numpy(rng.randn(B, N, D).astype(np.float32))
  chosen = [s for s in range(steps) if s % 3 != 1]
  sel = [-1] * steps
  for j, s in enumerate(reversed(chosen)):          # later steps to lower blocks
    sel[s] = j
  col0 = 2
  width = (col0 + len(chosen) + 1) * D
  out = torch.full((B, N, width), 7.0, device=dev())
  ops().operator_chain(L.to(dev()), X.to(dev()), steps, sel, out, col0, chebyshev=cheby)
  got = out.cpu()
  ref64 = _chain_ref(L[..., 0].double(), X.double(), steps, cheby)
  ref32 = _chain_ref(L[..., 0], X, steps, cheby)
  written = torch.zeros(width, dtype=torch.bool)
  for s in range(steps):
    if sel[s] < 0:
      continue
    c0 = (col0 + sel[s]) * D
    written[c0:c0 + D] = True
    # rounding compounds over the steps: the floor is per step, as in test_gpu_kernels
    _check(got[:, :, c0:c0 + D], ref64[s], ref32[s], 4, FFMA_FLOOR * (s + 1), 'operator_chain',
           'chain N=%d steps=%d D=%d E1=%d cheby=%d step %d' % (N, steps, D, E1, cheby, s + 1))
  assert torch.all(got[:, :, ~written] == 7.0)


def test_operator_chain_refuses_outside_envelope():
  d = dev()
  assert not ops().operator_chain_supported(33, 1) and not ops().operator_chain_supported(32, 65)
  for N, steps in ((33, 1), (32, 65)):
    L = torch.zeros(2, N, N, 2, device=d)
    X = torch.zeros(2, N, 8, device=d)
    out = torch.zeros(2, N, 8 * (steps + 1), device=d)
    _refused(lambda: ops().operator_chain(L, X, steps, list(range(steps)), out, 0))


@pytest.mark.parametrize('kind', ['diag', 'dense_nonsym'])
@pytest.mark.parametrize('D', [1, 129])
def test_graph_messages_envelope_corner(D, kind):
  """N = K = 32, E1 = 16, S = 8, a 64-step walk (shared memory above 48 KB), selected steps with gaps
  in an unsorted list, rows wider than the message matrix."""
  N = K = 32
  E1, S = 16, 8
  short = [64, 1, 5, 33]
  rng = np.random.RandomState(D + (kind == 'diag'))
  B = 3
  sizes = _sizes(rng, B, N)
  L = _operators(rng, B, N, E1, sizes)
  Q = _basis(rng, B, N, K, sizes)
  filt = _filters(rng, B, K, S, kind)
  X = torch.from_numpy(rng.randn(B, N, D).astype(np.float32))
  dense = kind != 'diag'
  C = len(short) + S + E1
  assert ops().graph_messages_supported(N, K, E1, S, max(short))
  out = torch.full((B, N, C * D + 5), 7.0, device=dev())
  d = dev()
  ops().graph_messages(L.to(d), X.to(d), Q.to(d), filt.to(d), dense, short, out)
  got = out.cpu()
  ref64 = _messages_ref(X.double(), L, Q, filt, dense, short)
  ref32 = _messages_ref(X, L, Q, filt, dense, short)
  assert len(ref64) == C
  for c in range(C):
    _check(got[:, :, c * D:(c + 1) * D], ref64[c], ref32[c], 4, FFMA_FLOOR, 'graph_messages',
           'messages D=%d %s block %d' % (D, kind, c))
  assert torch.all(got[:, :, C * D:] == 7.0)


@pytest.mark.parametrize('N,K,E1,S,short', [(33, 4, 2, 0, []), (8, 33, 2, 1, []), (8, 4, 17, 1, []),
                                            (8, 4, 2, 9, []), (8, 4, 2, 1, [65])],
                         ids=['N33', 'K33', 'E17', 'S9', 'short65'])
def test_graph_messages_refuses_each_limit(N, K, E1, S, short):
  assert not ops().graph_messages_supported(N, K, E1, S, max(short) if short else 0)
  d = dev()
  B, D = 2, 4
  L = torch.zeros(B, N, N, E1, device=d)
  X = torch.zeros(B, N, D, device=d)
  Q = torch.zeros(B, N, K, device=d) if S else None
  filt = torch.zeros(B, K, S, device=d) if S else None
  out = torch.zeros(B, N, (len(short) + S + E1) * D, device=d)
  _refused(lambda: ops().graph_messages(L, X, Q, filt, False, short, out))


def _gl_fits(N, Dx):
  """lnb_gaussian_laplacian's shared-memory condition: features, degrees and the reduction scratch."""
  return (N * (Dx | 1) + N + 32) * 4 <= 227 * 1024


GL_NMAX64 = max(n for n in range(1, 4096) if _gl_fits(n, 64))


@pytest.mark.parametrize('N,Dx,E1', [(1, 3, 1), (2, 1, 7), (2, 128, 1), (26, 64, 7), (26, 128, 1),
                                     (33, 3, 7), (33, 64, 1), (255, 1, 1), (255, 128, 7),
                                     (GL_NMAX64, 64, 1)])
def test_gaussian_laplacian_envelope(N, Dx, E1):
  """Isolated real nodes and padded rows take the pad term; N = 1 has sigma^2 = 0 and gives NaN where
  the reference does."""
  rng = np.random.RandomState(N + Dx + E1)
  B = 1 if N > 300 else 3
  sizes = rng.randint(1, N + 1, size=B)
  sizes[0] = max(1, N - N // 5)
  L = _operators(rng, B, N, E1, sizes).numpy()
  for b, n in enumerate(sizes):
    if n >= 3:                                         # an isolated real node
      iso = int(rng.randint(n))
      L[b, iso, :, 0] = 0.0
      L[b, :, iso, 0] = 0.0
  L = torch.from_numpy(L)
  x = torch.from_numpy(rng.randn(B, N, Dx).astype(np.float32))
  out = ops().gaussian_laplacian(x.to(dev()), L.to(dev()))
  adj = orc.adjacency_from_laplacian(L[..., 0].double())
  ref64 = orc.gaussian_kernel_laplacian(x.double(), adj)
  ref32 = orc.gaussian_kernel_laplacian(x, adj.float())
  if N == 1:
    assert bool(torch.isnan(ref64).all())
  _check(out, ref64, ref32, 4, FFMA_FLOOR, 'gaussian_laplacian', 'Le N=%d Dx=%d E1=%d' % (N, Dx, E1))


def test_gaussian_laplacian_refuses_features_beyond_shared_memory():
  N = GL_NMAX64 + 1
  assert _gl_fits(GL_NMAX64, 64) and not _gl_fits(N, 64)
  d = dev()
  x = torch.zeros(1, N, 64, device=d)
  L = torch.zeros(1, N, N, 1, device=d)
  _refused(lambda: ops().gaussian_laplacian(x, L))


def _ro_fits(H, P):
  HP = H | 1
  return P < 256 and ((P + 1) * HP + 32 * HP + 32 * (P + 1)) * 4 <= 227 * 1024


RO_CASES = [
    # N, H, P, mask
    (1, 1, 1, 'none'), (1, 3, 255, 'ragged'), (1, 36, 16, 'allmasked'), (31, 36, 49, 'ragged'),
    (31, 128, 49, 'allmasked'), (32, 128, 16, 'allmasked'), (32, 1000, 1, 'none'),
    (33, 1000, 16, 'ragged'), (33, 36, 255, 'none'), (100, 128, 255, 'ragged'), (100, 3, 1, 'allmasked'),
    (100, 1000, 16, 'none'),
]


@pytest.mark.parametrize('N,H,P,mask_kind', RO_CASES)
def test_readout_envelope(N, H, P, mask_kind):
  """Gated masked mean over 32-node chunks and their tails; a graph with no unmasked node gives a NaN
  row, like torch.mean of an empty set."""
  assert _ro_fits(H, P)
  rng = np.random.RandomState(N * 7 + H + P)
  B = 5
  state = torch.from_numpy(rng.randn(B, N, H).astype(np.float32))
  params = {'filter.0.weight': torch.from_numpy((rng.randn(P, H) / np.sqrt(H)).astype(np.float32)),
            'filter.0.bias': torch.from_numpy(rng.randn(P).astype(np.float32)),
            'att_func.0.weight': torch.from_numpy((rng.randn(1, H) / np.sqrt(H)).astype(np.float32)),
            'att_func.0.bias': torch.from_numpy(rng.randn(1).astype(np.float32))}
  mask = None
  if mask_kind != 'none':
    sizes = [N, min(N, 32), min(N, 33), 1, int(rng.randint(1, N + 1))]
    if mask_kind == 'allmasked':
      sizes[1] = 0
    mask = (torch.arange(N)[None, :] < torch.tensor(sizes)[:, None]).to(torch.uint8)
  d = dev()
  out = ops().readout(state.to(d), params['filter.0.weight'].to(d), params['filter.0.bias'].to(d),
                      params['att_func.0.weight'].reshape(-1).to(d), params['att_func.0.bias'].to(d),
                      None if mask is None else mask.to(d))
  spec = {'num_layer': 0}
  ref64 = orc.readout({k: v.double() for k, v in params.items()}, spec, state.double(), mask)
  ref32 = orc.readout(params, spec, state, mask)
  if mask_kind == 'allmasked':
    assert bool(torch.isnan(ref64[1]).all())
  _check(out, ref64, ref32, 4, FFMA_FLOOR, 'readout', 'readout N=%d H=%d P=%d %s' % (N, H, P, mask_kind))


@pytest.mark.parametrize('H,P', [(16, 256), (1000, 49), (128, 300)])
def test_readout_refuses_outside_envelope(H, P):
  assert not _ro_fits(H, P)
  d = dev()
  N, B = 8, 2
  _refused(lambda: ops().readout(torch.zeros(B, N, H, device=d), torch.zeros(P, H, device=d),
                                 torch.zeros(P, device=d), torch.zeros(H, device=d), torch.zeros(1, device=d)))


@pytest.mark.parametrize('K', [1, 33, 64])
def test_tridiag_powers_envelope(K):
  """Powers of symmetric tridiagonal T (spectral radius <= 1, one with a zero trailing block as a
  Lanczos run that stopped early leaves it, one all zero) against repeated fp64 products."""
  powers = [1, 2, 3, 5, 7, 10, 20, 30]
  rng = np.random.RandomState(K)
  B = 4
  T = np.zeros((B, K, K))
  for b in range(B - 1):
    k = K if b != 1 else max(1, K // 2)
    t = np.diag(rng.randn(k)) + np.diag(rng.randn(k - 1), 1)
    t = np.triu(t) + np.triu(t, 1).T
    T[b, :k, :k] = t / np.abs(np.linalg.eigvalsh(t)).max()
  T = torch.from_numpy(T.astype(np.float32))
  out = ops().tridiag_powers(T.to(dev()), powers).cpu()          # [B,K,S,K]
  ref64 = orc.tridiag_power_stack(T.double(), powers)
  ref32 = orc.tridiag_power_stack(T, powers)
  for s, p in enumerate(powers):
    _check(out[:, :, s], ref64[s], ref32[s], 4, FFMA_FLOOR, 'tridiag_powers', 'T^%d K=%d' % (p, K))
  assert torch.equal(out[B - 1], torch.zeros(K, len(powers), K))


@pytest.mark.parametrize('powers', [[5, 3], [2, 2], [0, 1], [1, 7, 5], list(range(1, 34))],
                         ids=['decreasing', 'repeated', 'zero', 'unsorted', 'S33'])
def test_tridiag_powers_refuses_non_increasing_powers(powers):
  """AdaLanczosNet sorts its long distances before calling the kernel; the kernel keeps refusing
  anything but at most 32 positive, strictly increasing powers."""
  T = torch.eye(4, device=dev()).expand(2, 4, 4).contiguous()
  _refused(lambda: ops().tridiag_powers(T, powers))


# ------------------------------------------------------------------------------------------
# 3. models off the QM8 shape against the fp64 oracle
# ------------------------------------------------------------------------------------------
def _ada_compose(params, spec, T, Q, node_feat, L, mask, dtype):
  """AdaLanczosNet's layers and readout on given (T, Q): oracle filters, conv_layer and readout."""
  p = {k: v.to(dtype) for k, v in params.items()}
  T, Q, L = T.cpu().to(dtype), Q.cpu().to(dtype), L.to(dtype)
  state = p['embedding.weight'][node_feat.long()]
  for layer in range(spec['num_layer']):
    Lf = orc.spectral_filters_from_tridiag(p, spec, T, Q, layer)
    state = orc.conv_layer(p, spec, layer, state, L, Lf)
  return orc.readout(p, spec, state, mask)


def _check_ada(mod, params, nf, L, mask, q1, out, tag):
  """Le against fp64 (rule of the full-QM8 test), T against the oracle's Lanczos on the same Le, the
  score against the fp64 composition on the module's own T and Q."""
  lz = mod.last_lanczos
  spec = oracle_spec(mod, 'AdaLanczosNet')
  K = spec['K']
  d = dev()
  state = ops().embedding_rows(nf.to(d).long(), mod.embedding.weight)
  Le = ops().gaussian_laplacian(state, L.to(d).float().contiguous()).cpu()
  adj = orc.adjacency_from_laplacian(L[..., 0].double())
  emb = params['embedding.weight']
  Le64 = orc.gaussian_kernel_laplacian(emb.double()[nf.long()], adj)
  e_ref = float((orc.gaussian_kernel_laplacian(emb[nf.long()], adj.float()).double() - Le64).abs().max())
  e_ours = float((Le.double() - Le64).abs().max())
  _WORST['model Le'] = max(_WORST.get('model Le', 0.0), e_ours / max(4 * e_ref, 2e-6))
  print('%s Le: err %.3g (fp32 %.3g)' % (tag, e_ours, e_ref))
  assert e_ours <= max(4 * e_ref, 2e-6) and e_ours <= 2e-5, (tag, e_ours, e_ref)
  q = q1.reshape(q1.shape[0], -1)
  lz64 = orc.lanczos_tridiagonalise(Le.double(), mask, q.double(), K)
  lz32 = orc.lanczos_tridiagonalise(Le, mask, q.float(), K)
  assert np.array_equal(lz['idx'].cpu().numpy(), lz64['idx'].numpy()), tag
  _check(lz['T'], lz64['T'], lz32['T'], 4, 5e-5, 'model T', tag + ' T', scale=1.0)
  nl = spec['num_layer']
  s64 = _ada_compose(params, spec, lz['T'], lz['Q'], nf, L, mask, torch.float64)
  s32 = _ada_compose(params, spec, lz['T'], lz['Q'], nf, L, mask, torch.float32)
  _check(out, s64, s32, 8, KERNEL_FLOOR * nl, 'model scores', tag + ' score')


ADA_CASES = [(33, 20, 'MLP'), (33, 20, 'power'), (64, 40, 'MLP'), (64, 40, 'power'), (130, 40, 'MLP'),
             (130, 40, 'power'), (26, 40, 'MLP'), (26, 40, 'power')]


@pytest.mark.parametrize('N,K,filter_kind', ADA_CASES)
def test_ada_lanczos_net_off_qm8_shape_vs_fp64(N, K, filter_kind):
  from lanczosnetwork_b200.model import AdaLanczosNet
  if K > 32:       # the filter MLP's input is K*K*S wide: one layer, two long scales
    over = dict(num_layer=1, hidden_dim=[36], long_diffusion_dist=[3, 7], short_diffusion_dist=[1, 2])
  else:
    over = dict(num_layer=2, hidden_dim=[36, 36], long_diffusion_dist=[2, 5, 7], short_diffusion_dist=[1, 3])
  cfg = configs.qm8_ada_lanczos_net(num_eig_vec=K, spectral_filter_kind=filter_kind, **over)
  mod, params = _build(AdaLanczosNet, cfg, N + K)
  rng = np.random.RandomState(N)
  sizes = [N, max(3, N // 3), int(rng.randint(3, N + 1)), 3]
  batch = _molecules(sizes, K, seed=N + K)
  nf, L, mask = _t(batch['node_feat']), _t(batch['L']), _t(batch['node_mask'])
  torch.manual_seed(N)
  q1 = torch.randn(len(sizes), N, 1)
  torch.manual_seed(N)                 # the module draws the same q1 (CPU generator)
  mod.use_cuda_graph = False
  with torch.no_grad():
    out = mod(nf.to(dev()), L.to(dev()), mask=mask.to(dev()))
  _check_ada(mod, params, nf, L, mask, q1, out, 'ada N=%d K=%d %s' % (N, K, filter_kind))


def test_lanczosnet_general_first_layer_on_the_bgemm_branch(monkeypatch):
  """N = 40: the 10-wide first layer runs the per-step batched GEMMs, the others the fused stack."""
  from lanczosnetwork_b200.model import LanczosNetGeneral
  cfg = configs.graph_lanczos_net(num_layer=2, hidden_dim=[128, 128])
  mod, params = _build(LanczosNetGeneral, cfg, 40)
  batch = _molecules([40, 17, 33, 5], 20, num_bond_type=1, seed=40, feat_dim=10)
  args = [batch[k] for k in ('node_feat', 'L', 'D', 'V')]
  o = ops()
  calls = []
  for name in ('graph_messages', 'operator_chain'):
    monkeypatch.setattr(o, name, _spy(getattr(o, name), name, calls))
  mod.use_cuda_graph = False
  with torch.no_grad():
    out = mod(*[_t(a).to(dev()) for a in args], mask=_t(batch['node_mask']).to(dev()))
  assert calls == []
  spec = oracle_spec(mod, 'LanczosNetGeneral')
  ref64 = orc.lanczos_net_forward(params, spec, *args, batch['node_mask'], dtype=torch.float64)
  ref32 = orc.lanczos_net_forward(params, spec, *args, batch['node_mask'], dtype=torch.float32)
  _check(out, ref64, ref32, 8, KERNEL_FLOOR * 2, 'model scores', 'LanczosNetGeneral N=40')


@pytest.mark.parametrize('long', [[1, 2, 3, 5, 7, 10, 20, 30], [10, 2, 30, 5]], ids=['sorted', 'unsorted'])
def test_lanczosnet_unfused_kscale_above_32_nodes(long, monkeypatch):
  """hidden_dim=[36, 36], K = 40, N = 64: both layers unfused, the long scales through the batched GEMM's
  kscale; an unsorted long list keeps the config order (reference lanczos_net.py:148)."""
  from lanczosnetwork_b200.model import LanczosNet
  cfg = configs.qm8_lanczos_net(num_layer=2, hidden_dim=[36, 36], num_eig_vec=40, long_diffusion_dist=long)
  mod, params = _build(LanczosNet, cfg, 64)
  batch = _molecules([64, 40, 31, 7], 40, seed=64)
  args = [batch[k] for k in ('node_feat', 'L', 'D', 'V')]
  o = ops()
  kscaled = []
  bgemm = o.bgemm

  def spy_bgemm(*a, **k):
    if k.get('kscale') is not None:
      kscaled.append(a[8])                             # M = N rows
    return bgemm(*a, **k)
  monkeypatch.setattr(o, 'bgemm', spy_bgemm)
  mod.use_cuda_graph = False
  with torch.no_grad():
    out = mod(*[_t(a).to(dev()) for a in args], mask=_t(batch['node_mask']).to(dev()))
  assert kscaled == [64, 64]
  spec = oracle_spec(mod, 'LanczosNet')
  ref64 = orc.lanczos_net_forward(params, spec, *args, batch['node_mask'], dtype=torch.float64)
  ref32 = orc.lanczos_net_forward(params, spec, *args, batch['node_mask'], dtype=torch.float32)
  _check(out, ref64, ref32, 8, KERNEL_FLOOR * 2, 'model scores', 'LanczosNet N=64 K=40 long=%s' % long)


def test_dcnn_seventeen_channels_runs_the_operator_chain_branch(monkeypatch):
  """num_bond_type = 16 (E1 = 17 > the one-launch messages kernel's 16): DCNN's chain-only branch."""
  from lanczosnetwork_b200.model import DCNN
  cfg = configs.qm8_dcnn(num_layer=2, hidden_dim=[36, 36], diffusion_dist=[5, 2, 30])
  cfg.dataset.num_bond_type = 16
  mod, params = _build(DCNN, cfg, 17)
  batch = _molecules([26, 12, 20, 3], 4, num_bond_type=16, seed=17)
  nf, L, mask = batch['node_feat'], batch['L'], batch['node_mask']
  assert L.shape[3] == 17
  o = ops()
  calls = []
  for name in ('graph_messages', 'operator_chain'):
    monkeypatch.setattr(o, name, _spy(getattr(o, name), name, calls))
  mod.use_cuda_graph = False
  with torch.no_grad():
    out = mod(_t(nf).to(dev()), _t(L).to(dev()), mask=_t(mask).to(dev()))
  assert calls == ['operator_chain'] * 2
  ref64 = orc.dcnn_forward(params, [5, 2, 30], 16, 2, nf, L, mask, dtype=torch.float64)
  ref32 = orc.dcnn_forward(params, [5, 2, 30], 16, 2, nf, L, mask, dtype=torch.float32)
  _check(out, ref64, ref32, 8, KERNEL_FLOOR * 2, 'model scores', 'DCNN E1=17')


@pytest.mark.parametrize('order', [64, 65])
def test_cheby_net_longest_chain_and_its_fallback(order, monkeypatch):
  """polynomial_order 64: the Chebyshev operator chain in one launch; 65: the alpha / addend batched GEMMs."""
  from lanczosnetwork_b200.model import ChebyNet
  cfg = configs.qm8_cheby_net(num_layer=2, hidden_dim=[36, 36], polynomial_order=order)
  mod, params = _build(ChebyNet, cfg, order)
  batch = _molecules([32, 9, 25, 3], 4, seed=order)
  nf, L, mask = batch['node_feat'], batch['L'], batch['node_mask']
  o = ops()
  calls = []
  monkeypatch.setattr(o, 'operator_chain', _spy(o.operator_chain, 'operator_chain', calls))
  mod.use_cuda_graph = False
  with torch.no_grad():
    out = mod(_t(nf).to(dev()), _t(L).to(dev()), mask=_t(mask).to(dev()))
  assert calls == (['operator_chain'] * 2 if order == 64 else [])
  ref64 = orc.cheby_net_forward(params, order, 6, 2, nf, L, mask, dtype=torch.float64)
  ref32 = orc.cheby_net_forward(params, order, 6, 2, nf, L, mask, dtype=torch.float32)
  _check(out, ref64, ref32, 8, KERNEL_FLOOR * 2, 'model scores', 'ChebyNet order=%d' % order)


@pytest.mark.parametrize('keyed', [False, True], ids=['AdaLanczosNet', 'KeyedAdaLanczosNet'])
def test_ada_unsorted_diffusion_distances(keyed):
  """long_diffusion_dist=[10, 5, 7], short_diffusion_dist=[3, 1]: the powers of T go in ascending order
  like the reference's T_list (ada_lanczos_net.py:266-268); eager forward and CUDA-graph replay agree
  with each other and with the oracle."""
  from lanczosnetwork_b200.model import AdaLanczosNet, KeyedAdaLanczosNet
  cfg = configs.qm8_ada_lanczos_net(num_layer=2, hidden_dim=[32, 32], num_eig_vec=8,
                                    long_diffusion_dist=[10, 5, 7], short_diffusion_dist=[3, 1])
  mod, params = _build(KeyedAdaLanczosNet if keyed else AdaLanczosNet, cfg, 310)
  batch = data.synthetic_qm8_batch(6, seed=31, num_eigs=8)
  nf, L, mask = _t(batch['node_feat']), _t(batch['L']), _t(batch['node_mask'])
  B, N = nf.shape
  d = dev()
  key = torch.tensor([7, 3], dtype=torch.int64, device=d)

  def run():
    with torch.no_grad():
      if keyed:
        return mod(nf.to(d), L.to(d), mask=mask.to(d), start_key=key)
      torch.manual_seed(31)
      return mod(nf.to(d), L.to(d), mask=mask.to(d))
  if keyed:
    q1 = ops().ada_start_vector(key, B, N).cpu()
  else:
    torch.manual_seed(31)
    q1 = torch.randn(B, N, 1)
  mod.use_cuda_graph = False
  eager = run()
  _check_ada(mod, params, nf, L, mask, q1, eager, 'ada unsorted keyed=%d' % keyed)
  mod.use_cuda_graph = True
  replays = [run() for _ in range(2)]
  mod.use_cuda_graph = False
  assert all(torch.equal(r, eager) for r in replays)
  spec = oracle_spec(mod, 'AdaLanczosNet')
  ref = orc.ada_lanczos_net_forward(params, spec, batch['node_feat'], batch['L'], batch['node_mask'],
                                    q1.reshape(B, N))
  np.testing.assert_allclose(eager.cpu().numpy(), ref.numpy(), rtol=5e-4, atol=5e-5)


def test_keyed_ada_unsorted_distances_train_on_the_powers_kernel(monkeypatch):
  """The training path sorts the long distances too, so an unsorted config takes the powers kernel and
  its adjoint, with the scores of the inference forward and the gradients of the GEMM chain."""
  from lanczosnetwork_b200 import train
  from lanczosnetwork_b200.model import KeyedAdaLanczosNet
  cfg = configs.qm8_ada_lanczos_net(num_layer=2, hidden_dim=[32, 32], num_eig_vec=8,
                                    long_diffusion_dist=[10, 5, 7], short_diffusion_dist=[3, 1])
  mod, _ = _build(KeyedAdaLanczosNet, cfg, 311)
  batch = data.synthetic_qm8_batch(6, seed=32, num_eigs=8)
  d = dev()
  nf, L, mask = [_t(batch[k]).to(d) for k in ('node_feat', 'L', 'node_mask')]
  key = torch.tensor([5, 1], dtype=torch.int64, device=d)
  mod.use_cuda_graph = False
  with torch.no_grad():
    ref = mod(nf, L, mask=mask, start_key=key)
  params = [p for p in mod.parameters() if p.requires_grad]

  def grads():
    score = mod(nf, L, mask=mask, start_key=key)
    return score.detach(), torch.autograd.grad(score.square().sum(), params, allow_unused=True)
  calls = []
  monkeypatch.setattr(train, 'tridiag_powers', _spy(train.tridiag_powers, 'tridiag_powers', calls))
  score_k, g_k = grads()
  assert calls == ['tridiag_powers']
  monkeypatch.setattr(ops(), 'tridiag_powers_backward_supported', lambda *a: False)
  score_c, g_c = grads()
  assert calls == ['tridiag_powers']                   # the GEMM chain this time
  # the training formulation runs its own Lanczos kernel: scores agree to its rounding, gradients to the
  # conditioning of the Lanczos adjoint (2e-2 against fp64 in test_gpu_keyed_ada); a power in the wrong
  # place moves both by O(1)
  scale = ref.abs().max().item()
  print('train vs inference scores: powers kernel %.3g, GEMM chain %.3g (scale %.3g)'
        % ((score_k - ref).abs().max().item(), (score_c - ref).abs().max().item(), scale))
  assert (score_k - ref).abs().max().item() <= 1e-3 * scale
  assert (score_c - ref).abs().max().item() <= 1e-3 * scale
  for gk, gc in zip(g_k, g_c):
    assert (gk is None) == (gc is None)
    if gk is not None:
      assert (gk - gc).abs().max().item() <= 1e-2 * max(gc.abs().max().item(), 1e-6)
