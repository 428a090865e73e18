"""The fused spectral convolution (one layer and the whole stack) and the Ritz filter-MLP chain
across the shapes their entry points accept, against fp64 references of the same math.

The sweeps cover the paths the QM8 shape never takes: H % 16 != 0 (a 16-column epilogue chunk
that ends past the row), S == 0 and S > 8 (filter coefficients read from global memory), K up
to 32 with Z filling a whole tile, E1 from 1 to 16, N = 127 / 128, empty graphs, several tiles
per CTA, up to 8 layers and readouts of up to 48 outputs; for the MLP chain S > 8 (first stage
on the tensor cores), Hd < 128, row lists and enough items that a CTA moves between layers.
``pytest -m gpu``."""
import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, oracle_spec
from lanczosnetwork_b200 import configs, data
from oracle import lanczos_oracle as orc
from test_gpu_models import FWD_ATOL, FWD_RTOL

pytestmark = pytest.mark.gpu

# Floor of the stack tolerance relative to the output's scale, per layer: the single-layer bound
# (8e-6, ~K/8 truncating accumulation steps) compounding over the layers.  The 3xTF32 kernel
# is often more than 8x further from fp64 than true fp32 (cuBLAS, no TF32) is, so the floor
# decides.  Calibrated on an H100 80GB HBM3 (700 W): the worst case, 8 layers with E1 = 16 and
# H = 128, was 2.7e-5 of the scale against a floor of 6.4e-5.
STACK_FLOOR_PER_LAYER = 8e-6


def dev():
  return torch.device('cuda:0')


def ops():
  from lanczosnetwork_b200 import ops as _ops
  return _ops


def _act(y, relu):
  return torch.relu(y) if relu else y


# ------------------------------------------------------------------------------------------
# references (plain torch, any dtype)
# ------------------------------------------------------------------------------------------
def conv_ref(X, L, V, coeff, W, bias, relu=True):
  """One layer: act(cat([V diag(f_s) V^T X]_s ++ [L_e X]_e) W^T + b); coeff [B,K,S] or None."""
  msgs = []
  if coeff is not None:
    U = V.transpose(1, 2) @ X
    msgs += [V @ (coeff[:, :, s:s + 1] * U) for s in range(coeff.shape[2])]
  msgs += [L[..., e] @ X for e in range(L.shape[3])]
  y = torch.cat(msgs, dim=2) @ W.t()
  if bias is not None:
    y = y + bias
  return _act(y, relu)


def stack_ref(X, L, V, coeffs, Ws, bs, readout=None, mask=None):
  """Layers 0..len(Ws)-1 (model/lanczos_net.py:157-182), then the gated, masked-mean readout
  (:185-194).  coeffs: per-layer [B,K,S] or None.  Returns (state, score or None)."""
  for l in range(len(Ws)):
    X = conv_ref(X, L, V, None if coeffs is None else coeffs[l], Ws[l], bs[l])
  if readout is None:
    return X, None
  W_out, b_out, w_att, b_att = readout
  y = (X @ W_out.t() + b_out) * torch.sigmoid(X @ w_att + b_att).unsqueeze(2)
  if mask is None:
    return X, y.mean(dim=1)
  m = mask.to(y.dtype).unsqueeze(2)
  return X, (y * m).sum(dim=1) / m.sum(dim=1)


def mlp_ref(table, layers):
  out = []
  for ps in layers:
    h = table.double()
    for i, (_, w, b) in enumerate(ps):
      h = h @ w.double().t() + b.double()
      if i < 3:
        h = torch.relu(h)
    out.append(h)
  return torch.stack(out)


# ------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------
def _graphs(B, N, K, E1, seed, sizes=None, empty=(1,)):
  """Random sparse operators L [B,N,N,E1] and orthonormal Ritz vectors V [B,N,K] on the leading
  sizes[b] nodes of every graph; graphs listed in `empty` have no real node at all."""
  rng = np.random.RandomState(seed)
  if sizes is None:
    sizes = rng.randint(max(2, N // 4), N + 1, size=B)
    sizes[0] = N
  sizes = np.array(sizes)
  L = np.zeros((B, N, N, E1), np.float32)
  V = np.zeros((B, N, K), np.float32)
  for b in range(B):
    if b in empty:
      sizes[b] = 0
      continue
    n = int(sizes[b])
    L[b, :n, :n] = rng.randn(n, n, E1) * (rng.rand(n, n, E1) < min(1.0, 4.0 / n))
    kk = min(K, n)
    V[b, :n, :kk] = np.linalg.qr(rng.randn(n, n))[0][:, :kk]
  return torch.from_numpy(L), torch.from_numpy(V), sizes


def _weights(g, H, kin, n=1):
  Ws = [torch.randn(H, kin, generator=g) / np.sqrt(kin) for _ in range(n)]
  bs = [torch.randn(H, generator=g) for _ in range(n)]
  return Ws, bs


def _check(out, ref64, ref32, floor, what):
  """|out - ref64| <= max(8 |ref32 - ref64|, floor * scale): the kernel is no worse than 8x the
  same math in fp32, or within `floor` of the output's scale."""
  err = (out.double() - ref64).abs().max().item()
  err32 = (ref32.double() - ref64).abs().max().item()
  scale = ref64.abs().max().item()
  print('%s: max err %.3g (fp32 %.3g) at scale %.3g' % (what, err, err32, scale))
  assert err <= max(8 * err32, floor * scale), (what, err, err32, scale)


def _conv_raw(X, Q, coeff, prep, w_hi, w_lo, bias, relu, write_pad, out):
  """lnb_spectral_conv_fused into a caller-provided output (ops.spectral_conv_fused allocates its
  own), so rows the kernel must not write can be checked against a sentinel."""
  ell_val, ell_idx, ell_max, gext, tiles = prep
  B, N, Din = X.shape
  S = 0 if coeff is None else coeff.shape[2]
  ops()._launch('lnb_spectral_conv_fused', X, X, Q, coeff, ell_val, ell_idx, ell_max, gext, tiles, w_hi, w_lo, bias,
                B, N, Din, ell_val.shape[1], Q.shape[2], S, w_hi.shape[0], int(relu), int(write_pad), out)
  torch.cuda.synchronize()
  return out


# ------------------------------------------------------------------------------------------
# one fused layer
# ------------------------------------------------------------------------------------------
HS = [4, 36, 40, 100, 120, 124, 128]
DINS = [32, 64, 96]
SS = [0, 1, 5, 9, 16]
# (Din, H) pairs whose last 16-column epilogue chunk ends past the row pitch max(Din, H) + 4
OVERRUN = {(32, h) for h in (36, 40, 52, 56, 68, 72, 84, 88, 100, 104, 116, 120)} | \
          {(64, h) for h in (68, 72, 84, 88, 100, 104, 116, 120)} | {(96, h) for h in (100, 104, 116, 120)}


def _layer_cases():
  cases = []
  for i, (din, h, s) in enumerate((d, h, s) for d in DINS for h in HS for s in SS):
    K = (4, 8, 32)[i % 3]
    E1 = (1, 2, 16)[(i // 3) % 3]
    N = (26, 40, 127, 128, 64)[(i // 2) % 5]
    cases.append(pytest.param(din, h, s, K, E1, N, i % 4 != 3, i % 5 != 4,
                              id='Din%d-H%d-S%d-K%d-E%d-N%d' % (din, h, s, K, E1, N)))
  for i, (din, h) in enumerate(sorted(OVERRUN - {(d, h) for d in DINS for h in HS})):
    K, E1, N = (4, 8, 32)[i % 3], (2, 7)[i % 2], 40
    cases.append(pytest.param(din, h, 5, K, E1, N, True, True,
                              id='Din%d-H%d-S5-K%d-E%d-N%d' % (din, h, K, E1, N)))
  return cases


@pytest.mark.parametrize('Din,H,S,K,E1,N,relu,with_bias', _layer_cases())
def test_conv_layer_envelope(Din, H, S, K, E1, N, relu, with_bias):
  assert ops().fused_conv_supported(N, Din, K, H, 0, False, S, E1)
  seed = Din * 10007 + H * 101 + S * 7 + K
  B = 6
  L, V, sizes = _graphs(B, N, K, E1, seed)
  g = torch.Generator().manual_seed(seed)
  X = torch.randn(B, N, Din, generator=g)
  coeff = torch.randn(B, K, S, generator=g) if S else None
  (W,), (b,) = _weights(g, H, (S + E1) * Din)
  bias = b if with_bias else None
  d = dev()
  Xg, Lg, Vg, Wg = X.to(d), L.to(d), V.to(d), W.to(d)
  cg = coeff.to(d) if S else None
  bg = bias.to(d) if with_bias else None
  prep = ops().graph_prepare(Lg, Vg)
  w_hi, w_lo = ops().split_tf32(Wg)
  out = ops().spectral_conv_fused(Xg, Vg, cg, prep, w_hi, w_lo, bg, relu)
  ref = conv_ref(Xg.double(), Lg.double(), Vg.double(), None if cg is None else cg.double(),
                 Wg.double(), None if bg is None else bg.double(), relu)
  torch.backends.cuda.matmul.allow_tf32 = False
  ref32 = conv_ref(Xg, Lg, Vg, cg, Wg, bg, relu)
  # a graph without real nodes: every row is the constant act(b), exactly
  const = _act(bg if with_bias else torch.zeros(H, device=d), relu)
  assert torch.equal(out[1], const.expand(N, H)), 'empty graph'
  # single layer: the bound of test_spectral_conv_fused_matches_fp64_and_unfused, or 8x fp32
  err = (out.double() - ref).abs().max().item()
  err32 = (ref32.double() - ref).abs().max().item()
  scale = ref.abs().max().item()
  print('conv Din=%d H=%d S=%d K=%d E1=%d N=%d: max err %.3g (fp32 %.3g) at scale %.3g'
        % (Din, H, S, K, E1, N, err, err32, scale))
  assert err <= max(8e-6 * scale + 1e-6, 8 * err32), (err, err32, scale)


def test_conv_layer_full_tiles_many_per_cta():
  """Z and the node rows both fill 128-row tiles (four 32-node graphs, K = 32), and the batch
  needs more than two tiles per SM, so every CTA stages several tiles in turn."""
  d = dev()
  sms = torch.cuda.get_device_properties(d).multi_processor_count
  B, N, K, S, E1, Din, H = 8 * sms + 8, 32, 32, 9, 3, 64, 100
  L, V, _ = _graphs(B, N, K, E1, 77, sizes=[N] * B, empty=(5,))
  g = torch.Generator().manual_seed(77)
  X = torch.randn(B, N, Din, generator=g)
  coeff = torch.randn(B, K, S, generator=g)
  (W,), (b,) = _weights(g, H, (S + E1) * Din)
  Xg, Lg, Vg, cg, Wg, bg = [t.to(d) for t in (X, L, V, coeff, W, b)]
  prep = ops().graph_prepare(Lg, Vg)
  gext, tiles = prep[3].cpu(), prep[4].cpu()
  T = int(tiles[0])
  assert T >= 2 * sms, T
  assert int(tiles[2]) == 4                    # tile 0 = graphs 0..3: 128 node rows, 128 Ritz rows
  assert int(gext[:4, 1].sum()) == 128 and int(gext[:4, 0].sum()) == 128
  w_hi, w_lo = ops().split_tf32(Wg)
  out = ops().spectral_conv_fused(Xg, Vg, cg, prep, w_hi, w_lo, bg, True)
  ref = conv_ref(Xg.double(), Lg.double(), Vg.double(), cg.double(), Wg.double(), bg.double())
  torch.backends.cuda.matmul.allow_tf32 = False
  _check(out, ref, conv_ref(Xg, Lg, Vg, cg, Wg, bg), 8e-6, 'full tiles')


@pytest.mark.parametrize('Din,H,S', [(64, 100, 5), (32, 128, 0), (96, 36, 16)])
def test_conv_layer_write_pad_false_leaves_padded_rows(Din, H, S):
  K, E1, N, B = 20, 7, 26, 9
  L, V, sizes = _graphs(B, N, K, E1, H + S)
  g = torch.Generator().manual_seed(H + S)
  X = torch.randn(B, N, Din, generator=g)
  coeff = torch.randn(B, K, S, generator=g) if S else None
  (W,), (b,) = _weights(g, H, (S + E1) * Din)
  d = dev()
  Xg, Lg, Vg, Wg, bg = [t.to(d) for t in (X, L, V, W, b)]
  cg = coeff.to(d) if S else None
  prep = ops().graph_prepare(Lg, Vg)
  w_hi, w_lo = ops().split_tf32(Wg)
  sentinel = torch.full((B, N, H), 12345.0, device=d)
  out = _conv_raw(Xg, Vg, cg, prep, w_hi, w_lo, bg, True, False, sentinel.clone())
  ref = conv_ref(Xg.double(), Lg.double(), Vg.double(), None if S == 0 else cg.double(), Wg.double(),
                 bg.double())
  real = (torch.arange(N)[None, :] < torch.from_numpy(sizes)[:, None]).to(d)
  assert torch.equal(out[~real], sentinel[~real])
  err = (out[real].double() - ref[real]).abs().max().item()
  assert err <= 8e-6 * ref.abs().max().item() + 1e-6, err
  # write_pad=True fills the same rows with act(b) and leaves the real rows bit-identical
  full = _conv_raw(Xg, Vg, cg, prep, w_hi, w_lo, bg, True, True, sentinel.clone())
  assert torch.equal(full[real], out[real])
  assert torch.equal(full[~real], torch.relu(bg).expand(B, N, H)[~real])


def test_conv_layer_binarized_operators():
  """graph_prepare(..., binarize=True): the operators enter as their non-zero pattern."""
  K, S, E1, N, B, Din, H = 8, 5, 16, 40, 7, 64, 120
  L, V, _ = _graphs(B, N, K, E1, 5)
  g = torch.Generator().manual_seed(5)
  X = torch.randn(B, N, Din, generator=g)
  coeff = torch.randn(B, K, S, generator=g)
  (W,), (b,) = _weights(g, H, (S + E1) * Din)
  d = dev()
  Xg, Lg, Vg, cg, Wg, bg = [t.to(d) for t in (X, L, V, coeff, W, b)]
  prep = ops().graph_prepare(Lg, Vg, binarize=True)
  w_hi, w_lo = ops().split_tf32(Wg)
  out = ops().spectral_conv_fused(Xg, Vg, cg, prep, w_hi, w_lo, bg, True)
  Lb = (Lg != 0).to(torch.float32)
  ref = conv_ref(Xg.double(), Lb.double(), Vg.double(), cg.double(), Wg.double(), bg.double())
  torch.backends.cuda.matmul.allow_tf32 = False
  _check(out, ref, conv_ref(Xg, Lb, Vg, cg, Wg, bg), 8e-6, 'binarized')


@pytest.mark.parametrize('N,Din,K,H', [(129, 64, 20, 128), (26, 64, 36, 128), (26, 64, 20, 132),
                                       (26, 48, 20, 128)])
def test_conv_layer_refuses_unsupported_shapes(N, Din, K, H):
  """Shapes fused_conv_supported rejects are rejected by the C entry point too, before launch."""
  S, E1, B = 8, 7, 2
  assert not ops().fused_conv_supported(N, Din, K, H, 0, False, S, E1)
  d = dev()
  L, V, _ = _graphs(B, N, K, E1, 1)
  X = torch.randn(B, N, Din, device=d)
  coeff = torch.randn(B, K, S, device=d)
  w_hi, w_lo = ops().split_tf32(torch.randn(H, (S + E1) * Din, device=d))
  prep = ops().graph_prepare(L.to(d), V.to(d))
  with pytest.raises(RuntimeError, match='unsupported shape'):
    ops().spectral_conv_fused(X, V.to(d), coeff, prep, w_hi, w_lo, torch.randn(H, device=d), True)


# ------------------------------------------------------------------------------------------
# the one-launch stack: embedding gather, layers, fused readout
# ------------------------------------------------------------------------------------------
STACK_CASES = [
    # dins, H, S, K, E1, P, masked, embedding input
    ([64], 100, 5, 20, 7, 16, True, True),
    ([64, 128], 128, 8, 20, 7, 16, False, False),
    ([96] + [64] * 7, 64, 16, 32, 2, 1, True, True),
    ([32] + [128] * 7, 128, 0, 8, 16, 48, False, False),
    ([128, 64], 64, 9, 32, 16, 1, False, True),
    # the fused readout's scratch is largest next to the smallest tile state: H = Din = 32 / 64
    ([32, 32], 32, 9, 4, 3, 48, True, False),
    ([32, 32, 32], 32, 5, 20, 7, 48, True, True),
    ([32, 32], 32, 1, 28, 1, 48, False, False),
    ([64, 64], 64, 5, 4, 7, 48, False, True),
    ([32], 32, 8, 4, 7, 28, True, False),
]


@pytest.mark.parametrize('dins,H,S,K,E1,P,masked,emb_in', STACK_CASES,
                         ids=['L%d-Din%d-H%d-S%d-K%d-P%d' % (len(c[0]), c[0][0], c[1], c[2], c[3], c[5])
                              for c in STACK_CASES])
def test_spectral_stack_vs_fp64(dins, H, S, K, E1, P, masked, emb_in):
  nl, B, N = len(dins), 40, 26
  d = dev()
  seed = nl * 1000 + H * 10 + P + S
  L, V, sizes = _graphs(B, N, K, E1, seed)
  g = torch.Generator().manual_seed(seed)
  ids = torch.randint(0, 70, (B, N), generator=g)
  emb = torch.randn(70, dins[0], generator=g)
  Ws, bs = [], []
  for din in dins:
    (w,), (b,) = _weights(g, H, (S + E1) * din)
    Ws.append(w)
    bs.append(b)
  coeffs = torch.randn(nl, B, K, S, generator=g) if S else None
  W_out, b_out = torch.randn(P, H, generator=g) / np.sqrt(H), torch.randn(P, generator=g)
  w_att, b_att = torch.randn(H, generator=g) / np.sqrt(H), torch.randn(1, generator=g)
  mask = None
  if masked:
    mask = (torch.arange(N)[None, :] < torch.randint(1, N + 1, (B, 1), generator=g)).to(torch.uint8)
  from lanczosnetwork_b200 import spectral_conv as sc
  kw = (S + E1) * max(dins)
  Wg, bg = [w.to(d) for w in Ws], [b.to(d) for b in bs]
  w_hi, w_lo, ball = sc.WeightCache().split_conv_stack('t', Wg, bg, kw)
  Lg, Vg, idg, embg = L.to(d), V.to(d), ids.to(d), emb.to(d)
  cg = coeffs.to(d) if S else None
  ro = [t.to(d) for t in (W_out, b_out, w_att, b_att)]
  mg = mask.to(d) if masked else None
  for l in range(nl):
    assert ops().fused_conv_supported(N, dins[l], K, H, 0, False, S, E1)
  prep = ops().graph_prepare(Lg, Vg)
  X0 = embg[idg]
  kwargs = dict(node_ids=idg, emb=embg) if emb_in else dict(X=X0)
  st, score = ops().spectral_stack_forward(prep, Vg, w_hi, w_lo, ball, dins, H, S, coeff=cg,
                                           coeff_stride=cg.stride(0) if S else 0, want_state=True,
                                           readout=ro, mask=mg, **kwargs)
  # the readout alone (no state requested) gives the same scores
  st2, score2 = ops().spectral_stack_forward(prep, Vg, w_hi, w_lo, ball, dins, H, S, coeff=cg,
                                             coeff_stride=cg.stride(0) if S else 0, readout=ro,
                                             mask=mg, **kwargs)
  assert st2 is None and torch.equal(score2, score)
  c64 = None if cg is None else cg.double()
  st64, sc64 = stack_ref(X0.double(), Lg.double(), Vg.double(), c64, [w.double() for w in Wg],
                         [b.double() for b in bg], [t.double() for t in ro], mg)
  torch.backends.cuda.matmul.allow_tf32 = False
  st32, sc32 = stack_ref(X0, Lg, Vg, cg, Wg, bg, ro, mg)
  tag = 'stack L=%d Din0=%d H=%d S=%d K=%d P=%d' % (nl, dins[0], H, S, K, P)
  _check(st, st64, st32, STACK_FLOOR_PER_LAYER * nl, tag + ' state')
  _check(score, sc64, sc32, STACK_FLOOR_PER_LAYER * nl, tag + ' score')


# ------------------------------------------------------------------------------------------
# Ritz filter-MLP chain
# ------------------------------------------------------------------------------------------
def _mlp_layers(g, nl, S, Hd):
  layers = []
  for l in range(nl):
    ps = []
    for i, (o, k) in enumerate([(Hd, S), (Hd, Hd), (Hd, Hd), (S, Hd)]):
      w = (torch.randn(o, k, generator=g) / np.sqrt(k)).to(dev())
      b = (torch.randn(o, generator=g) * 0.1).to(dev())
      ps.append(('l%d.%d' % (l, i), w, b))
    layers.append(ps)
  return layers


def _mlp_raw(table, w_hi, w_lo, bias_all, nl, rowmap, nrows, coeff):
  R, S = table.shape
  ops()._launch('lnb_ritz_filter_mlp', table, table, rowmap, nrows, w_hi, w_lo, bias_all, R, nl, S, w_hi.shape[1],
                coeff)
  torch.cuda.synchronize()
  return coeff


def _assert_mlp(out, ref, what):
  for l in range(ref.shape[0]):
    err = (out[l].double() - ref[l]).abs().max().item()
    assert err <= 5e-6 * ref[l].abs().max().item() + 1e-6, (what, l, err)


def _mlp_cases():
  cases = []
  for i, (S, Hd) in enumerate((s, h) for s in (1, 4, 8, 9, 16, 32) for h in (32, 64, 96, 128)):
    nl = (1, 2, 7)[i % 3]
    R = (1, 128, 129)[(i // 3) % 3] if i % 5 else 300
    cases.append(pytest.param(S, Hd, nl, R, id='S%d-Hd%d-L%d-R%d' % (S, Hd, nl, R)))
  # the benchmark shape (1024 graphs x 20 Ritz values, 7 layers): 1120 items, CTAs change layer
  cases += [pytest.param(8, 128, 7, 20480, id='S8-Hd128-L7-R20480'),
            pytest.param(16, 64, 7, 20480, id='S16-Hd64-L7-R20480')]
  return cases


@pytest.mark.parametrize('S,Hd,nl,R', _mlp_cases())
def test_filter_mlp_chain_envelope(S, Hd, nl, R):
  from lanczosnetwork_b200 import spectral_conv as sc
  g = torch.Generator().manual_seed(S * 1000 + Hd + nl)
  layers = _mlp_layers(g, nl, S, Hd)
  table = (torch.rand(R, S, generator=g) * 2 - 1).to(dev())
  w_hi, w_lo, bias_all = sc.WeightCache().split_mlp_chain('chain', layers)
  out = ops().ritz_filter_mlp(table, w_hi, w_lo, bias_all, nl)
  _assert_mlp(out, mlp_ref(table, layers), 'S=%d Hd=%d L=%d R=%d' % (S, Hd, nl, R))


@pytest.mark.parametrize('S', [8, 16])
def test_filter_mlp_chain_row_list(S):
  """Only the rows in the list are evaluated (in list order, any order); the others are left
  as they were."""
  R, nl, Hd = 300, 3, 64
  g = torch.Generator().manual_seed(S)
  layers = _mlp_layers(g, nl, S, Hd)
  table = (torch.rand(R, S, generator=g) * 2 - 1).to(dev())
  from lanczosnetwork_b200 import spectral_conv as sc
  w_hi, w_lo, bias_all = sc.WeightCache().split_mlp_chain('chain', layers)
  ref = mlp_ref(table, layers)
  perm = torch.randperm(R, generator=g).int().to(dev())
  for n in (0, 137, R):
    rowmap = torch.full((R,), -7, dtype=torch.int32, device=dev())
    rowmap[:n] = perm[:n]
    nrows = torch.tensor([n], dtype=torch.int32, device=dev())
    sentinel = torch.full((nl, R, S), -12345.0, device=dev())
    out = _mlp_raw(table, w_hi, w_lo, bias_all, nl, rowmap, nrows, sentinel.clone())
    listed = torch.zeros(R, dtype=torch.bool, device=dev())
    listed[perm[:n].long()] = True
    assert torch.equal(out[:, ~listed], sentinel[:, ~listed]), n
    if n:
      _assert_mlp(out[:, listed], ref[:, listed], 'rows=%d' % n)


@pytest.mark.parametrize('S,Hd', [(8, 100), (6, 100), (12, 128)])
def test_ritz_filter_coefficients_paths(S, Hd):
  """ritz_filter_coefficients: the chain kernel (Hd % 32 == 0), the grouped dense layers
  (Hd = 100, S % 4 == 0) and the per-layer dense fallback (S = 6), all against fp64."""
  from lanczosnetwork_b200 import spectral_conv as sc
  g = torch.Generator().manual_seed(S + Hd)
  B, K, nl = 37, 20, 3
  D = (torch.rand(B, K, generator=g) * 2 - 1).to(dev())
  powers = [1, 2, 3, 5, 7, 10, 20, 30, 4, 6, 8, 9][:S]
  layers = _mlp_layers(g, nl, S, Hd)
  out, table = sc.ritz_filter_coefficients(D, powers, layers, sc.WeightCache())
  ref = mlp_ref(table.reshape(B * K, S), layers).reshape(nl, B, K, S)
  _assert_mlp(out, ref, 'S=%d Hd=%d' % (S, Hd))


# ------------------------------------------------------------------------------------------
# models routed through these kernels, against the fp64 oracle
# ------------------------------------------------------------------------------------------
MODEL_CASES = {
    'H100-1layer': (dict(input_dim=64, hidden_dim=[100], num_layer=1), 20),
    'H100-2layers': (dict(input_dim=64, hidden_dim=[100, 100], num_layer=2), 20),
    'S12': (dict(long_diffusion_dist=[1, 2, 3, 4, 5, 7, 10, 15, 20, 25, 30, 40], num_layer=2,
                 hidden_dim=[128, 128]), 20),
    'K32': (dict(num_eig_vec=32, num_layer=2, hidden_dim=[128, 128]), 32),
    'H32-P48': (dict(input_dim=32, hidden_dim=[32, 32], num_layer=2, output_dim=48), 20),
}


@pytest.mark.parametrize('case', sorted(MODEL_CASES))
def test_lanczosnet_envelope_vs_fp64_oracle(case):
  from lanczosnetwork_b200.model import LanczosNet
  over, K = MODEL_CASES[case]
  batch = data.synthetic_qm8_batch(64, seed=7, num_eigs=K)
  mod = LanczosNet(configs.qm8_lanczos_net(**over))
  params = deterministic_state_dict(mod, 99)
  mod.load_state_dict(params)
  mod = mod.to(dev()).eval()
  args = [batch[k] for k in ('node_feat', 'L', 'D', 'V')]
  with torch.no_grad():
    out = mod(*[torch.from_numpy(a).to(dev()) for a in args],
              mask=torch.from_numpy(batch['node_mask']).to(dev()))
  ref = orc.lanczos_net_forward(params, oracle_spec(mod, 'LanczosNet'), *args, batch['node_mask'],
                                dtype=torch.float64).numpy()
  np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=FWD_RTOL, atol=FWD_ATOL)
