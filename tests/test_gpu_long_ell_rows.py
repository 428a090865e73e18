"""The ELL (sparse row list) kernels on long and uneven operator rows, against fp64.

The other sweeps feed these kernels molecule-like operators of about four entries per row.  Here the rows
are long (dense graphs: every pair of real nodes), uneven (hub nodes next to short rows), past the
convolution stack's staging budget (E1 = 16 with every channel's longest row 17 or 19 entries: 272 / 304
ELL lines, more than the 255 a tile stages, so the stack's producers gather the remaining lines from global
memory, and a budget splits a channel between the two), or mixed in one tile (a dense graph, short rows
and a graph without nodes, whose short rows are zero-filled up to the dense graph's row length).  The
generators and a numpy restatement of graph_prepare's layout are in tests/test_host_long_ell_rows.py.

Every output is judged graph by graph against its own scale: a dense graph's outputs are about sqrt(n)
larger than a short-row neighbour's in the same tile, and a batch-wide scale would hide the small graph's
errors.  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import ops, train
from lanczosnetwork_b200 import spectral_conv as sc
from test_gpu_conv_envelope import STACK_FLOOR_PER_LAYER, _check, _graphs, conv_ref, stack_ref
from test_gpu_graphsage import restate
from test_gpu_persistent_grid import _assert_same, max_ctas
from test_gpu_sparse_train import _rows
from test_host_long_ell_rows import ell_rows, mixed_tile, operators

pytestmark = pytest.mark.gpu

# Floors of the tolerance relative to a graph's own output scale.  Long rows lengthen the edge producers'
# fp32 sums (up to 128 terms per row and channel), and the fp32 restatement's error grows with them.  The
# stack, its single layer and the GraphSAGE stack keep the short-row floors (STACK_FLOOR_PER_LAYER per
# layer, CONV_FLOOR for one layer).  Measured on an H100 80GB HBM3 (700 W), the worst graph of these sweeps
# reached, as a share of its floor: the stack 0.60 (1 layer, budget17, 4.8e-6 of the scale) and 0.57
# (3 layers, mixed tile, 1.4e-5), the single layer 0.56 (budget17, 4.5e-6), GraphSAGE Max 0.41 and Mean
# 0.28.  The ELL products are plain fp32 sums: within 1.6x of the fp32 restatement's error, and at most
# 4.7e-7 of the scale against ELL_FLOOR.
CONV_FLOOR = 8e-6
ELL_FLOOR = 1e-6


def dev():
  return torch.device('cuda:0')


def _per_graph(out, ref64, ref32, floor, what):
  """_check on every graph b = out[b] alone: its own error against its own scale."""
  for b in range(out.shape[0]):
    _check(out[b], ref64[b], ref32[b], floor, '%s graph %d' % (what, b))


def _batch(profile, N, E1, K, seed):
  """(L, V, sizes) on the device for a stack case.  profile: 'mixed' (mixed_tile), 'control' (E1 = 1,
  at most four entries per row), or a PROFILES name for every graph.  One graph has no node (not in
  the control)."""
  rng = np.random.RandomState(seed)
  if profile == 'mixed':
    profiles, sizes = mixed_tile(N)
  else:
    lo = max(19, N // 4) if profile.startswith('budget') else N // 4
    sizes = rng.randint(lo, N + 1, size=8)
    sizes[0] = N
    if profile != 'control':
      sizes[3] = 0
    profiles = 'sparse' if profile == 'control' else profile
  sizes = [int(s) for s in sizes]
  L = torch.from_numpy(operators(profiles, sizes, N, E1, seed))
  _, V, _ = _graphs(len(sizes), N, K, 1, seed, sizes=sizes, empty=[b for b, s in enumerate(sizes) if s == 0])
  return L.to(dev()), V.to(dev()), sizes


# ------------------------------------------------------------------------------------------
# graph_prepare: the ELL rows, bit for bit
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('binarize', [False, True])
@pytest.mark.parametrize('E1', [1, 7, 16])
@pytest.mark.parametrize('N', [26, 128, 255])
def test_graph_prepare_long_rows_bit_for_bit(N, E1, binarize):
  """Rows of up to N entries (N = 255: the largest uint8 column), hub rows, budget-crossing rows, short
  rows and an empty graph in one batch; graphs of N = 26 and N = 128 at E1 = 1 have their operators staged
  in shared memory, the others read from global memory."""
  profiles = ['dense', 'hub', 'budget19', 'sparse', 'empty', 'dense']
  sizes = [N, N - 3, N, N // 2, 0, N // 3 + 1]
  K = 8
  L = operators(profiles, sizes, N, E1, seed=N + E1)
  rng = np.random.RandomState(N * E1)
  Q = np.zeros((len(sizes), N, K), np.float32)
  for b, n in enumerate(sizes):
    k = min(K, n, 1 + b)
    Q[b, :n, :k] = rng.uniform(0.5, 1.0, size=(n, k))
  val, idx, emax, n_eff = ell_rows(L, binarize)
  prep = ops.graph_prepare(torch.from_numpy(L).to(dev()), torch.from_numpy(Q).to(dev()), binarize=binarize)
  got_val, got_idx, got_max, gext = [t.cpu().numpy() for t in prep[:4]]
  assert np.array_equal(got_max, emax), (got_max, emax)
  assert emax[0].min() == sizes[0] and emax[2].min() == 19    # rows of N entries; 19 in every channel
  want_ext = np.stack([np.maximum(n_eff, sizes), [min(K, n, 1 + b) for b, n in enumerate(sizes)]], axis=1)
  assert np.array_equal(gext, want_ext), (gext, want_ext)
  live = np.arange(N)[None, None, :, None] < emax[:, :, None, None]          # slots up to the longest row
  live = np.broadcast_to(live, val.shape)
  bad = (got_val.view(np.uint32) != val.view(np.uint32)) & live
  assert not bad.any(), 'ell_val: %d slots differ, first at %s' % (bad.sum(), np.argwhere(bad)[0])
  bad = (got_idx != idx) & live
  assert not bad.any(), 'ell_idx: %d slots differ, first at %s' % (bad.sum(), np.argwhere(bad)[0])


# ------------------------------------------------------------------------------------------
# the LanczosNet convolution stack and its single layer
# ------------------------------------------------------------------------------------------
STACK_CASES = [
    # profile, layers, S, K, E1, N, Din0, H, readout
    ('dense', 1, 0, 8, 1, 128, 64, 128, False),
    ('dense', 3, 5, 32, 7, 64, 128, 128, True),
    ('dense', 1, 5, 8, 16, 64, 64, 64, False),
    ('dense', 3, 0, 32, 16, 128, 32, 128, False),
    ('hub', 1, 5, 32, 7, 128, 128, 128, False),
    ('hub', 3, 0, 8, 16, 64, 64, 64, True),
    ('hub', 1, 0, 8, 1, 64, 32, 32, False),
    ('budget17', 1, 0, 8, 16, 64, 128, 128, False),
    ('budget17', 3, 5, 32, 16, 128, 128, 128, True),
    ('budget19', 1, 5, 32, 16, 64, 64, 128, False),
    ('budget19', 3, 0, 8, 16, 128, 64, 64, False),
    ('mixed', 1, 5, 8, 7, 64, 64, 128, False),
    ('mixed', 3, 0, 32, 16, 128, 128, 128, True),
    ('mixed', 3, 5, 32, 1, 128, 32, 64, False),
    ('control', 1, 0, 8, 1, 64, 64, 128, False),
    ('control', 3, 5, 32, 1, 128, 128, 32, True),
]


def _stack_id(c):
  return '%s-L%d-S%d-K%d-E%d-N%d-Din%d-H%d%s' % (c[:8] + ('-readout' if c[8] else '',))


def _stack_model(layers, S, K, E1, Din0, H, B, seed):
  g = torch.Generator().manual_seed(seed)
  dins = [Din0] + [H] * (layers - 1)
  Ws = [(torch.randn(H, (S + E1) * d, generator=g) / np.sqrt((S + E1) * d)).to(dev()) for d in dins]
  bs = [torch.randn(H, generator=g).to(dev()) for _ in dins]
  coeffs = torch.randn(layers, B, K, S, generator=g).to(dev()) if S else None
  ro = [t.to(dev()) for t in (torch.randn(16, H, generator=g) / np.sqrt(H), torch.randn(16, generator=g),
                              torch.randn(H, generator=g) / np.sqrt(H), torch.randn(1, generator=g))]
  return dins, Ws, bs, coeffs, ro


def _run_stack(prep, V, X, dins, H, S, coeffs, split, ro):
  w_hi, w_lo, ball = split
  return ops.spectral_stack_forward(prep, V, w_hi, w_lo, ball, dins, H, S, coeff=coeffs,
                                    coeff_stride=coeffs.stride(0) if S else 0, X=X, want_state=True,
                                    readout=ro)


@pytest.mark.parametrize('profile,layers,S,K,E1,N,Din0,H,readout', STACK_CASES,
                         ids=[_stack_id(c) for c in STACK_CASES])
def test_spectral_stack_long_rows(profile, layers, S, K, E1, N, Din0, H, readout):
  seed = layers * 1000 + S * 100 + K + E1 * 7 + N
  L, V, sizes = _batch(profile, N, E1, K, seed)
  B = len(sizes)
  dins, Ws, bs, coeffs, ro = _stack_model(layers, S, K, E1, Din0, H, B, seed)
  for d in dins:
    assert ops.fused_conv_supported(N, d, K, H, 0, False, S, E1)
  X = torch.randn(B, N, Din0, generator=torch.Generator().manual_seed(seed + 1)).to(dev())
  prep = ops.graph_prepare(L, V)
  if profile == 'mixed':
    # the first-fit schedule puts every graph in one tile, the dense graph (largest n_eff) first
    tiles, gext = prep[4].cpu(), prep[3].cpu()
    assert int(tiles[B + 2]) == 1 and int(tiles[B + 4]) == B, tiles[B + 2:B + 5]
    assert sorted(tiles[B + 5:2 * B + 5].tolist()) == list(range(B))
    assert int(tiles[B + 5]) == int(gext[:, 0].argmax()) and gext[:, 0].tolist() == sizes
  split = sc.WeightCache().split_conv_stack('long', Ws, bs, (S + E1) * max(dins))
  st, score = _run_stack(prep, V, X, dins, H, S, coeffs, split, ro if readout else None)
  c64 = coeffs.double() if S else None
  st64, sc64 = stack_ref(X.double(), L.double(), V.double(), c64, [w.double() for w in Ws],
                         [b.double() for b in bs], [t.double() for t in ro] if readout else None)
  torch.backends.cuda.matmul.allow_tf32 = False
  st32, sc32 = stack_ref(X, L, V, coeffs, Ws, bs, ro if readout else None)
  tag = 'stack ' + _stack_id((profile, layers, S, K, E1, N, Din0, H, readout))
  floor = STACK_FLOOR_PER_LAYER * layers
  _per_graph(st, st64, st32, floor, tag + ' state')
  if readout:
    _per_graph(score, sc64, sc32, floor, tag + ' score')


CONV_CASES = [
    # profile, S, K, E1, N, Din, H
    ('dense', 5, 32, 7, 128, 128, 128),
    ('dense', 0, 8, 16, 64, 64, 100),
    ('budget17', 5, 8, 16, 64, 128, 128),
    ('budget19', 0, 32, 16, 128, 64, 36),
    ('budget19', 9, 4, 16, 64, 32, 64),
]


@pytest.mark.parametrize('profile,S,K,E1,N,Din,H', CONV_CASES, ids=['%s-S%d-K%d-E%d-N%d-Din%d-H%d' % c
                                                                       for c in CONV_CASES])
def test_conv_layer_long_rows(profile, S, K, E1, N, Din, H):
  """spectral_conv_fused, one layer of the stack kernel."""
  seed = S * 100 + K + E1 * 7 + N + H
  L, V, sizes = _batch(profile, N, E1, K, seed)
  B = len(sizes)
  assert ops.fused_conv_supported(N, Din, K, H, 0, False, S, E1)
  g = torch.Generator().manual_seed(seed)
  X = torch.randn(B, N, Din, generator=g).to(dev())
  coeff = torch.randn(B, K, S, generator=g).to(dev()) if S else None
  W = (torch.randn(H, (S + E1) * Din, generator=g) / np.sqrt((S + E1) * Din)).to(dev())
  bias = torch.randn(H, generator=g).to(dev())
  w_hi, w_lo = ops.split_tf32(W)
  out = ops.spectral_conv_fused(X, V, coeff, ops.graph_prepare(L, V), w_hi, w_lo, bias, True)
  ref = conv_ref(X.double(), L.double(), V.double(), coeff.double() if S else None, W.double(), bias.double())
  torch.backends.cuda.matmul.allow_tf32 = False
  _per_graph(out, ref, conv_ref(X, L, V, coeff, W, bias), CONV_FLOOR, 'conv %s S=%d K=%d E1=%d N=%d' % (
      profile, S, K, E1, N))


def test_stack_budget_crossing_one_cta_is_bit_identical_to_the_full_grid():
  """One CTA runs every tile of the budget-crossing batch in turn, its staged and unstaged lines included."""
  N, E1, K, S, H = 64, 16, 32, 5, 128
  L, V, sizes = _batch('budget17', N, E1, K, 17)
  L, V = torch.cat([L] * 4), torch.cat([V] * 4)
  B = L.shape[0]
  dins, Ws, bs, coeffs, ro = _stack_model(2, S, K, E1, 64, H, B, 17)
  X = torch.randn(B, N, 64, generator=torch.Generator().manual_seed(18)).to(dev())
  prep = ops.graph_prepare(L, V)
  assert int(prep[4][B + 2]) >= 4
  split = sc.WeightCache().split_conv_stack('long', Ws, bs, (S + E1) * max(dins))
  full = [t.clone() for t in _run_stack(prep, V, X, dins, H, S, coeffs, split, ro)]
  with max_ctas(1):
    one = _run_stack(prep, V, X, dins, H, S, coeffs, split, ro)
  torch.cuda.synchronize()
  _assert_same(one[0], full[0], 'budget-crossing state at one CTA')
  _assert_same(one[1], full[1], 'budget-crossing score at one CTA')


# ------------------------------------------------------------------------------------------
# GraphSAGE stack, Mean and Max
# ------------------------------------------------------------------------------------------
SAGE_CASES = [
    # agg, profile, N, Din0, H, layers, E1, mask
    ('Max', 'dense', 128, 64, 128, 2, 7, True),
    ('Max', 'hub', 128, 128, 64, 1, 16, False),
    ('Max', 'budget17', 64, 64, 128, 2, 16, False),
    ('Mean', 'dense', 64, 64, 128, 2, 16, False),
    ('Mean', 'hub', 128, 32, 128, 1, 7, True),
    ('Mean', 'budget19', 64, 128, 32, 2, 16, True),
]

NEG_ROWS = 10      # embedding rows 0 .. NEG_ROWS - 1 are strictly negative


@pytest.mark.parametrize('agg,profile,N,Din0,H,layers,E1,use_mask', SAGE_CASES,
                         ids=['%s-%s-N%d-Din%d-H%d-L%d-E%d-%s' % (c[:7] + ('mask' if c[7] else 'nomask',))
                              for c in SAGE_CASES])
def test_sage_stack_long_rows(agg, profile, N, Din0, H, layers, E1, use_mask):
  """Graphs 0 and 2 take their input rows from a strictly negative block of the embedding, so the Max
  of every one of their rows is negative in the first layer."""
  seed = N + Din0 + H + layers + E1
  M, _, sizes = _batch(profile, N, E1, 4, seed)
  B = len(sizes)
  if use_mask:                 # the masked mean of a graph without nodes is 0 / 0
    sizes[3] = N // 2
    M = torch.from_numpy(operators(profile, sizes, N, E1, seed)).to(dev())
  rng = np.random.RandomState(seed)
  emb = rng.randn(70, Din0).astype(np.float32)
  emb[:NEG_ROWS] = -rng.uniform(0.25, 1.0, size=(NEG_ROWS, Din0))
  ids = rng.randint(NEG_ROWS, 70, size=(B, N))
  ids[[0, 2]] = rng.randint(0, NEG_ROWS, size=(2, N))
  ids, emb = torch.from_numpy(ids).to(dev()), torch.from_numpy(emb).to(dev())
  dins = [Din0] + [H] * (layers - 1)
  Ws = [torch.from_numpy(rng.uniform(-1, 1, size=(H, E1 * d)).astype(np.float32) * np.sqrt(6.0 / (H + E1 * d))).to(dev())
        for d in dins]
  bs = [torch.from_numpy(rng.uniform(-0.1, 0.1, size=H).astype(np.float32)).to(dev()) for _ in dins]
  g = torch.Generator().manual_seed(seed)
  head, att = torch.nn.Linear(H, 5), torch.nn.Linear(H, 1)
  with torch.no_grad():
    for p in list(head.parameters()) + list(att.parameters()):
      p.copy_(torch.rand(p.shape, generator=g) - 0.5)
  head, att = head.to(dev()), att.to(dev())
  mask = (torch.arange(N)[None, :] < torch.tensor(sizes)[:, None]).to(torch.uint8).to(dev()) if use_mask else None
  V = torch.zeros((B, N, 4), device=dev())
  prep = ops.graph_prepare(M, V)
  kw = E1 * max(dins)
  w_hi, w_lo = ops.split_tf32(torch.cat([torch.nn.functional.pad(W, (0, kw - W.shape[1])) for W in Ws]).contiguous())
  readout = (head.weight.detach(), head.bias.detach(), att.weight.detach().reshape(-1), att.bias.detach())
  with torch.no_grad():
    state, score = ops.spectral_stack_forward(prep, V, w_hi, w_lo, torch.cat(bs), dins, H, 0, node_ids=ids, emb=emb,
                                              want_state=True, readout=readout, mask=mask, sage=agg)
    s64, c64 = restate(M, ids, emb, Ws, bs, head, att, mask, agg, torch.float64)
    s32, c32 = restate(M, ids, emb, Ws, bs, head, att, mask, agg, torch.float32)
  tag = 'GraphSAGE %s %s N=%d E1=%d L=%d' % (agg, profile, N, E1, layers)
  _per_graph(state, s64, s32, STACK_FLOOR_PER_LAYER * layers, tag + ' state')
  _per_graph(score, c64, c32, STACK_FLOOR_PER_LAYER * layers, tag + ' score')


# ------------------------------------------------------------------------------------------
# ELL operator products and their adjoints
# ------------------------------------------------------------------------------------------
def _ell_batch(E1, seed):
  """Dense and hub rows at N = 128: the diagonal of rows 0, 64 and 127 is the first, a middle and the last
  column of a full row; a graph of 77 nodes and one without nodes."""
  N = 128
  sizes = [N, N, 77, 0]
  L = torch.from_numpy(operators(['dense', 'hub', 'dense', 'empty'], sizes, N, E1, seed)).to(dev())
  return L, ops.graph_prepare(L), ops.graph_prepare(L.transpose(1, 2).contiguous())


@pytest.mark.parametrize('strided', [False, True])
@pytest.mark.parametrize('weighted', [False, True])
@pytest.mark.parametrize('D', [3, 64])
def test_ell_messages_long_rows(D, weighted, strided):
  E1 = 7
  L, prep, prep_t = _ell_batch(E1, seed=D)
  B, N = L.shape[0], L.shape[1]
  assert int(prep[2][0].min()) == N and int(prep_t[2][0].min()) == N
  c0 = 1 if strided else 0
  nc = E1 - c0
  w = (torch.rand((B, N, E1), generator=torch.Generator().manual_seed(D)) + 0.5).to(dev()) if weighted else None
  wf = w if weighted else torch.ones((B, N, E1), device=dev())
  X = _rows(B * N, D, strided, seed=D + 1)
  G = _rows(B * N, nc * D, strided, seed=D + 2)

  def fwd(Lx, Xx, wx):
    Xb = Xx.reshape(B, N, D)
    return torch.cat([torch.bmm(Lx[..., e], Xb) * wx[:, :, e:e + 1] for e in range(c0, E1)], dim=2).reshape(B, N, -1)

  def adj(Lx, Gx, wx):
    Gb = Gx.reshape(B, N, nc, D)
    return sum(torch.bmm(Lx[..., e].transpose(1, 2), wx[:, :, e:e + 1] * Gb[:, :, e - c0]) for e in range(c0, E1))

  torch.backends.cuda.matmul.allow_tf32 = False
  got = ops.ell_messages(X, prep, c0, nc, w=w).reshape(B, N, -1)
  _per_graph(got, fwd(L.double(), X.double(), wf.double()), fwd(L, X, wf), ELL_FLOOR,
             'ell_messages D=%d w=%d' % (D, weighted))
  got_t = ops.ell_messages_adjoint(G, prep_t, D, c0, nc, w=w).reshape(B, N, D)
  _per_graph(got_t, adj(L.double(), G.double(), wf.double()), adj(L, G, wf), ELL_FLOOR,
             'ell_messages_adjoint D=%d w=%d' % (D, weighted))
  assert bool((got[3] == 0).all()) and bool((got_t[3] == 0).all()) and bool((got[2, 77:] == 0).all())


@pytest.mark.parametrize('E1', [1, 7])
def test_ell_products_give_the_dense_paths_bits_on_full_rows(E1):
  """Unweighted, the ELL products sum each row in ascending column order with the diagonal between its
  neighbours, as the dense path's batched GEMM does: the same bits, forward and adjoint, on rows of 128."""
  L, prep, prep_t = _ell_batch(E1, seed=E1)
  B, N = L.shape[0], L.shape[1]
  op = train.ell_operator(prep, prep_t)
  X = torch.randn((B, N, 40), generator=torch.Generator().manual_seed(E1)).to(dev()).requires_grad_(True)
  yd, ys = train.operator_messages(L, X), train.operator_messages(op, X)
  _assert_same(ys, yd, 'ELL forward vs dense')
  g = torch.randn(yd.shape, generator=torch.Generator().manual_seed(E1 + 1)).to(dev())
  _assert_same(torch.autograd.grad(ys, X, g)[0], torch.autograd.grad(yd, X, g)[0], 'ELL adjoint vs dense')


# ------------------------------------------------------------------------------------------
# neighbour_max
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N', [128, 255])
def test_neighbour_max_long_rows_and_ties(N):
  """Rows of up to N entries, features from a handful of integers (ties everywhere, broken toward the
  lowest node index) and a graph whose features are all negative (the max is negative, not 0)."""
  E1, D = 3, 8
  sizes = [N, N - 1, N // 2, 0, 40]
  L = torch.from_numpy(operators(['dense', 'hub', 'dense', 'empty', 'sparse'], sizes, N, E1, seed=N)).to(dev())
  B = len(sizes)
  rng = np.random.RandomState(N)
  X = rng.randint(-3, 4, size=(B, N, D)).astype(np.float32)
  X[2] = -rng.randint(1, 4, size=(N, D))
  X = torch.from_numpy(X).to(dev())
  prep = ops.graph_prepare(L)
  msg, arg = ops.neighbour_max(X, prep)
  live = (L != 0).permute(0, 1, 3, 2)                    # [B, n, e, m]
  v = torch.where(live.unsqueeze(4), X.unsqueeze(1).unsqueeze(1), torch.tensor(float('-inf'), device=dev()))
  mx = v.max(dim=3).values                               # [B, n, e, D]
  empty = ~live.any(dim=3)
  want = torch.where(empty.unsqueeze(3), torch.zeros_like(mx), mx)
  _assert_same(msg.view(B, N, E1, D), want, 'neighbour_max value')
  assert bool((want[2, :sizes[2]] < 0).all())
  hits = (v == mx.unsqueeze(3)) & live.unsqueeze(4)
  idx = torch.arange(N, device=dev()).view(1, 1, 1, N, 1).expand_as(hits)
  lowest = torch.where(hits, idx, torch.full_like(idx, N)).min(dim=3).values
  want_arg = torch.where(empty.unsqueeze(3), torch.full_like(lowest, -1), lowest)
  assert int((hits.sum(dim=3) > 1).sum()) > B * N       # ties are common
  assert torch.equal(arg.long(), want_arg)
