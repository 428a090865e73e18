"""The training path's autograd Functions (lanczosnetwork_b200.train) across the shapes they accept,
each forward and every input gradient against torch.autograd over the same operation written as
plain fp64 torch on the CPU.

Tolerances are stated against a yardstick: the error of the same computation done in fp32 by CPU
torch.  A result may be a few times further from fp64 than that, with a floor relative to the
result's scale for the 3xTF32 tensor-core products (their accumulation truncates).  The operators
are random and non-symmetric, so an adjoint that applied L_e where it needs L_e^T fails here; the
dense layer runs each case through both of its paths (strided fp32 GEMM and wgmma 3xTF32, split-K
included) and the two have to agree.  The whole-model gradients run off the QM8 grid (N = 33 / 128,
hidden widths that need K padding, 40 Ritz pairs) at batch sizes that put every convolution Linear
on the tensor cores; there the oracle takes the library's ReLU pattern, which may differ from its
own only on pre-activations within rounding of zero.  The captured training step is compared with
the eager one for the models that have a host-free training forward.  ``pytest -m gpu``."""
import math

import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict, oracle_spec
from lanczosnetwork_b200 import configs, data, ops, train
from lanczosnetwork_b200.model import ChebyNet, DCNN, GCN, LanczosNet, LanczosNetGeneral
from oracle import lanczos_oracle as orc

pytestmark = pytest.mark.gpu

# max|got - fp64| <= max(MULT * max|fp32 CPU - fp64|, FLOOR * max|fp64|)
MULT = 8.0
FLOOR_FP32 = 2e-6          # the strided fp32 GEMM at contractions of <= 200
# Whole-model parameter gradients: each weight gradient is a 3xTF32 contraction over all B*N rows
# (4k - 10k deep) whose result cancels well below the magnitude of its terms.  Worst measured on
# an H100 80GB HBM3 (700 W): 7e-6 of the gradient's scale (att_func.0.weight of LanczosNet).
FLOOR_MODEL = 2e-5


def _deep_floor(depth):
  """Floor of a dense-layer product contracting over ``depth`` terms: 6e-6 of the scale up to 4096
  (test_linear_tf32x3_fp32_grade), growing like the rounding error of a long sum, sqrt(depth),
  beyond.  The FFMA path sums sequentially in fp32 (K = 4096: 2.8e-6 measured), the weight gradient
  of either path runs on the tensor cores (depth 26624, split-K: 9.2e-6 measured)."""
  return 6e-6 * max(1.0, math.sqrt(depth / 4096.0))


def dev():
  return torch.device('cuda:0')


def _run(fn, inputs, needs, gout, device, dtype=None):
  """(output, [input gradient or None]) of fn by torch.autograd: floating inputs are cast to dtype
  (when given) on device, and only the inputs flagged in ``needs`` require a gradient."""
  xs = []
  for t, n in zip(inputs, needs):
    t = t.detach().to(device)
    if t.is_floating_point():
      t = t.to(dtype or t.dtype).requires_grad_(bool(n))
    xs.append(t)
  y = fn(*xs)
  wrt = [x for x, n in zip(xs, needs) if n]
  gs = iter(torch.autograd.grad(y, wrt, gout.to(device=device, dtype=y.dtype)))
  return y.detach(), [next(gs) if n else None for n in needs]


def _err(a, b):
  return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max()) if a.numel() else 0.0


def _bound(r64, r32, floor):
  scale = float(r64.abs().max()) if r64.numel() else 0.0
  return max(MULT * _err(r32, r64), floor * scale), scale


def _check(what, got, r64, r32, floor):
  """got within max(MULT x the fp32 CPU error, floor x scale) of fp64; returns the bound."""
  bound, scale = _bound(r64, r32, floor)
  err = _err(got, r64)
  print('%s: err %.3g  fp32 CPU %.3g  bound %.3g  scale %.3g  err/bound %.3f' % (
      what, err, _err(r32, r64), bound, scale, err / bound if bound else 0.0))
  assert err <= bound, (what, err, bound, scale)
  return bound


# ------------------------------------------------------------------------------------------
# 1. dense: act(x W^T + b) on the FFMA path and on the wgmma 3xTF32 path
# ------------------------------------------------------------------------------------------
def _dense_ref(relu, has_bias):
  def f(x, w, b):
    y = x @ w.t()
    if has_bias:
      y = y + b
    return torch.relu(y) if relu else y
  return f


# M, N, K, relu, bias, x needs grad, W needs grad, weight gradient runs split-K on the tensor path
DENSE = [
    (1, 1, 1, False, True, True, True, False),
    (1, 520, 1920, True, False, True, True, False),       # forward split-K
    (127, 3, 5, True, True, False, True, False),
    (127, 129, 1, False, False, True, False, False),
    (128, 16, 8, True, True, True, True, False),
    (128, 1, 4096, False, True, False, True, False),      # forward split-K, N = 1
    (129, 129, 130, True, True, True, True, False),
    (129, 520, 4096, True, False, True, True, False),
    (1664, 128, 1920, False, True, True, True, True),
    (1664, 520, 64, True, True, False, True, True),
    (26624, 16, 130, True, True, True, True, True),
    (26624, 3, 5, False, False, True, True, True),
]


@pytest.mark.parametrize('M,N,K,relu,has_bias,gx,gw,split_w', DENSE)
def test_dense_both_paths_vs_fp64(M, N, K, relu, has_bias, gx, gw, split_w, monkeypatch):
  g = torch.Generator().manual_seed(M * 31 + N * 7 + K)
  x = torch.randn(M, K, generator=g)
  w = torch.randn(N, K, generator=g) / math.sqrt(K)
  b = torch.randn(N, generator=g) if has_bias else torch.zeros(N)
  gy = torch.randn(M, N, generator=g)
  needs = (gx, gw, has_bias)
  ref = _dense_ref(relu, has_bias)
  y64, g64 = _run(ref, (x, w, b), needs, gy, 'cpu', torch.float64)
  y32, g32 = _run(ref, (x, w, b), needs, gy, 'cpu', torch.float32)
  splits = []
  real_ws = ops._splitk_workspace
  monkeypatch.setattr(ops, '_splitk_workspace', lambda *a: splits.append(a) or real_ws(*a))

  def lib(xx, ww, bb):
    return train.dense(xx, ww, bb if has_bias else None, relu)

  out = {}
  for path, threshold in (('ffma', float('inf')), ('wgmma', 0.0)):
    monkeypatch.setattr(train, '_SMALL_DENSE_FLOPS', threshold)
    xs = [t.detach().to(dev()).requires_grad_(n) for t, n in zip((x, w, b), needs)]
    y = lib(*xs)
    del splits[:]
    y.backward(gy.to(dev()))
    if path == 'wgmma' and split_w:
      tiles = -(-N // 128) * -(-K // 128)             # output tiles of g^T x [N, K]
      assert 2 * tiles <= ops._sm_count(dev()) and splits, 'weight gradient did not run split-K'
    grads = [t.grad if n else None for t, n in zip(xs, needs)]
    if not gx:
      assert xs[0].grad is None
    tag = 'dense %s M=%d N=%d K=%d relu=%d' % (path, M, N, K, relu)
    bounds = [_check(tag + ' y', y, y64, y32, _deep_floor(K))]
    for name, depth, got, r64, r32 in zip(('gx', 'gW', 'gb'), (N, M, M), grads, g64, g32):
      if r64 is not None:
        bounds.append(_check('%s %s' % (tag, name), got, r64, r32, _deep_floor(depth)))
    out[path] = ([y] + [t for t in grads if t is not None], bounds)
  # the two paths agree with each other as closely as each agrees with fp64
  for a, b_, bound in zip(out['ffma'][0], out['wgmma'][0], out['wgmma'][1]):
    assert _err(a, b_) <= bound, (_err(a, b_), bound)


@pytest.mark.parametrize('path', ['ffma', 'wgmma'])
def test_dense_relu_mask_at_exact_zero(path, monkeypatch):
  """Integer data keep every product and sum exact, so many pre-activations are exactly 0: the
  gradient there is 0, as torch's ReLU has it (result > 0), and every output is bit-exact."""
  monkeypatch.setattr(train, '_SMALL_DENSE_FLOPS', float('inf') if path == 'ffma' else 0.0)
  g = torch.Generator().manual_seed(5)
  M, N, K = 129, 19, 10
  x = torch.randint(-2, 3, (M, K), generator=g).float()
  w = torch.randint(-1, 2, (N, K), generator=g).float()
  b = torch.randint(-1, 2, (N,), generator=g).float()
  gy = torch.randint(-3, 4, (M, N), generator=g).float()
  assert int(((x @ w.t() + b) == 0).sum()) > M            # plenty of exact zeros
  y64, g64 = _run(_dense_ref(True, True), (x, w, b), (True,) * 3, gy, 'cpu', torch.float64)
  y, gs = _run(lambda xx, ww, bb: train.dense(xx, ww, bb, True), (x, w, b), (True,) * 3, gy, dev())
  assert torch.equal(y.cpu().double(), y64)
  for got, ref in zip(gs, g64):
    assert torch.equal(got.cpu().double(), ref)


# ------------------------------------------------------------------------------------------
# 2. operator_messages: msg_e = L_e X for the channels c0 .. c0+nc-1; gX = sum_e L_e^T g_e
# ------------------------------------------------------------------------------------------
def _opmsg_ref(c0, nc):
  def f(L, X):
    B, N, D = X.shape
    return torch.einsum('bnme,bmd->bned', L[..., c0:c0 + nc], X).reshape(B, N, nc * D)
  return f


# B, N, E1, c0, nc, D
OPMSG = [
    (3, 1, 1, 0, 1, 1),
    (4, 26, 7, 0, 7, 64),
    (4, 26, 7, 1, 6, 3),
    (3, 32, 2, 0, 1, 130),
    (2, 33, 16, 1, 15, 64),
    (3, 33, 1, 0, 1, 130),
    (2, 100, 7, 0, 1, 3),
    (2, 200, 2, 1, 1, 130),
    (2, 200, 16, 0, 16, 1),
]


@pytest.mark.parametrize('B,N,E1,c0,nc,D', OPMSG)
def test_operator_messages_non_symmetric_vs_fp64(B, N, E1, c0, nc, D):
  g = torch.Generator().manual_seed(B * 1000 + N * 17 + E1 * 3 + c0 + D)
  L = torch.randn(B, N, N, E1, generator=g) / math.sqrt(N)
  X = torch.randn(B, N, D, generator=g)
  gout = torch.randn(B, N, nc * D, generator=g)
  ref = _opmsg_ref(c0, nc)
  y64, (_, gx64) = _run(ref, (L, X), (False, True), gout, 'cpu', torch.float64)
  y32, (_, gx32) = _run(ref, (L, X), (False, True), gout, 'cpu', torch.float32)
  y, (_, gx) = _run(lambda LL, XX: train.operator_messages(LL, XX, c0, nc), (L, X), (False, True), gout, dev())
  tag = 'operator_messages B=%d N=%d E1=%d c0=%d nc=%d D=%d' % (B, N, E1, c0, nc, D)
  _check(tag + ' msg', y, y64, y32, FLOOR_FP32)
  bound = _check(tag + ' gX', gx, gx64, gx32, FLOOR_FP32)
  if N > 1:
    # the check can tell L^T from L: the adjoint of the transposed operator is far outside the bound
    _, (_, gx_t) = _run(ref, (L.transpose(1, 2), X), (False, True), gout, 'cpu', torch.float64)
    assert _err(gx, gx_t) > 100 * bound


# ------------------------------------------------------------------------------------------
# 3. spectral_messages: msg_s = V diag(F_s) V^T X with V non-orthogonal; gX and gF
# ------------------------------------------------------------------------------------------
def _specmsg_ref(V, X, F):
  B, N, D = X.shape
  U = torch.einsum('bnk,bnd->bkd', V, X)
  return torch.einsum('bnk,bks,bkd->bnsd', V, F, U).reshape(B, N, -1)


# B, N, K, S, D
SPECMSG = [
    (2, 1, 1, 1, 3),
    (3, 26, 20, 8, 64),
    (3, 20, 33, 5, 16),        # K > N: zero columns past N
    (2, 33, 64, 16, 3),        # K > N
    (2, 100, 64, 16, 130),
    (2, 200, 4, 1, 1),
    (2, 200, 33, 8, 64),
]


@pytest.mark.parametrize('B,N,K,S,D', SPECMSG)
def test_spectral_messages_vs_fp64(B, N, K, S, D):
  g = torch.Generator().manual_seed(B * 1000 + N * 13 + K * 5 + S + D)
  V = torch.randn(B, N, K, generator=g) / math.sqrt(N)
  if K > N:
    V[:, :, N:] = 0.0
  X = torch.randn(B, N, D, generator=g)
  F = torch.randn(B, K, S, generator=g)
  gout = torch.randn(B, N, S * D, generator=g)
  needs = (False, True, True)
  y64, (_, gx64, gf64) = _run(_specmsg_ref, (V, X, F), needs, gout, 'cpu', torch.float64)
  y32, (_, gx32, gf32) = _run(_specmsg_ref, (V, X, F), needs, gout, 'cpu', torch.float32)
  y, (_, gx, gf) = _run(train.spectral_messages, (V, X, F), needs, gout, dev())
  tag = 'spectral_messages B=%d N=%d K=%d S=%d D=%d' % (B, N, K, S, D)
  _check(tag + ' msg', y, y64, y32, FLOOR_FP32)
  _check(tag + ' gX', gx, gx64, gx32, FLOOR_FP32)
  _check(tag + ' gF', gf, gf64, gf32, FLOOR_FP32)


# ------------------------------------------------------------------------------------------
# 4. embedding: rows of the table, zero rows for out-of-range ids; the gradient is the adjoint
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('rows,D,kind', [(70, 64, 'same'), (70, 3, 'same'), (70, 1, 'edges'),
                                         (70, 4, 'edges'), (70, 130, 'edges'), (2, 3, 'edges'),
                                         (5000, 64, 'edges')])
def test_embedding_gradient_is_the_adjoint(rows, D, kind):
  """Every id equal (all atomics on one row), ids 0 and rows-1, and ids < 0 or >= rows: those
  read a zero row and add nothing to any row of the table gradient.  A row that k ids hit is a
  sum of k terms in whatever order the atomics land: its error is bounded by (k-1) 2^-24 sum|g|."""
  g = torch.Generator().manual_seed(rows + D)
  table = torch.randn(rows, D, generator=g)
  if kind == 'same':
    ids = torch.full((1024, 26), rows // 2, dtype=torch.long)
  else:
    ids = torch.randint(0, rows, (8, 26), generator=g)
    ids[0, :6] = torch.tensor([0, rows - 1, -1, -rows, rows, rows + 1000])
    ids[1, :3] = torch.tensor([-(2 ** 40), 2 ** 40, rows - 1])
  gout = torch.randn(ids.shape + (D,), generator=g)
  out, (_, gt) = _run(train.embedding, (ids, table), (False, True), gout, dev())
  valid = (ids >= 0) & (ids < rows)
  want = torch.where(valid.unsqueeze(-1), table[ids.clamp(0, rows - 1)], torch.zeros(()))
  assert torch.equal(out.cpu(), want)
  flat_ids, flat_g = ids[valid], gout[valid].double()
  ref = torch.zeros(rows, D, dtype=torch.float64).index_add_(0, flat_ids, flat_g)
  absum = torch.zeros(rows, D, dtype=torch.float64).index_add_(0, flat_ids, flat_g.abs())
  count = torch.zeros(rows, dtype=torch.float64).index_add_(0, flat_ids, torch.ones(len(flat_ids), dtype=torch.float64))
  bound = (count.clamp(min=1) - 1).unsqueeze(1) * 2.0 ** -24 * absum + 2.0 ** -24 * ref.abs()
  err = (gt.cpu().double() - ref).abs()
  print('embedding rows=%d D=%d %s: err %.3g  max count %d' % (rows, D, kind, float(err.max()), int(count.max())))
  assert bool((err <= bound).all()), float((err - bound).max())
  assert bool((gt.cpu()[count == 0] == 0).all())


# ------------------------------------------------------------------------------------------
# 5. bmm: non-contiguous operands (transposed and expanded views)
# ------------------------------------------------------------------------------------------
# nb, M, N, K, A layout, B layout, A needs grad
BMM = [
    (1, 1, 1, 1, 'plain', 'plain', True),
    (3, 65, 1, 70, 'transposed', 'plain', True),
    (2, 1, 65, 1, 'plain', 'expanded', True),
    (4, 65, 66, 67, 'expanded', 'transposed', True),
    (2, 100, 3, 130, 'transposed', 'expanded', False),
    (5, 1, 2, 200, 'plain', 'transposed', True),
    (3, 70, 80, 2, 'transposed', 'transposed', True),
]


def _operand(kind, nb, rows, cols, g):
  """[nb, rows, cols] as a contiguous tensor, a transposed view or a batch-expanded view."""
  if kind == 'transposed':
    return torch.randn(nb, cols, rows, generator=g).transpose(1, 2)
  if kind == 'expanded':
    return torch.randn(1, rows, cols, generator=g).expand(nb, rows, cols)
  return torch.randn(nb, rows, cols, generator=g)


@pytest.mark.parametrize('nb,M,N,K,ka,kb,ga', BMM)
def test_bmm_strided_operands_vs_fp64(nb, M, N, K, ka, kb, ga):
  g = torch.Generator().manual_seed(nb + M * 3 + N * 5 + K * 7)
  A, Bm = _operand(ka, nb, M, K, g), _operand(kb, nb, K, N, g)
  gout = torch.randn(nb, M, N, generator=g)

  def leaves(dtype, device, fn):
    # the views are taken after the leaves, so the gradient flows back through them
    def run(a0, b0):
      a = a0.expand(nb, M, K) if ka == 'expanded' else (a0.transpose(1, 2) if ka == 'transposed' else a0)
      b = b0.expand(nb, K, N) if kb == 'expanded' else (b0.transpose(1, 2) if kb == 'transposed' else b0)
      assert (ka == 'plain') == a.is_contiguous() and (kb == 'plain') == b.is_contiguous()
      return fn(a, b)
    a0 = A[:1] if ka == 'expanded' else (A.transpose(1, 2) if ka == 'transposed' else A)
    b0 = Bm[:1] if kb == 'expanded' else (Bm.transpose(1, 2) if kb == 'transposed' else Bm)
    return _run(run, (a0.contiguous(), b0.contiguous()), (ga, True), gout, device, dtype)

  y64, g64 = leaves(torch.float64, 'cpu', torch.bmm)
  y32, g32 = leaves(torch.float32, 'cpu', torch.bmm)
  y, gs = leaves(None, dev(), train.bmm)
  tag = 'bmm nb=%d M=%d N=%d K=%d A %s B %s' % (nb, M, N, K, ka, kb)
  _check(tag + ' C', y, y64, y32, FLOOR_FP32)
  for name, got, r64, r32 in zip(('gA', 'gB'), gs, g64, g32):
    if r64 is not None:
      _check('%s %s' % (tag, name), got, r64, r32, FLOOR_FP32)


# ------------------------------------------------------------------------------------------
# 6. whole-model gradients off the QM8 grid: random non-symmetric operators, N = 33 / 128
# ------------------------------------------------------------------------------------------
def _random_batch(B, N, E1, K, P, seed, feat_dim=None):
  """Padded batch of B graphs with 3N/4 .. N real nodes: E1 random sparse non-symmetric operator
  channels (rows scaled to an l1 norm <= 1 so powers stay bounded, zero on padded nodes), random
  Ritz values in (-1, 1), non-orthogonal Ritz vectors with zero columns past a graph's size."""
  rng = np.random.RandomState(seed)
  n = rng.randint(3 * N // 4, N + 1, size=B)
  n[0] = N
  mask = (np.arange(N)[None, :] < n[:, None]).astype(np.uint8)
  m = mask.astype(np.float64)
  A = (rng.rand(B, N, N, E1) < 4.0 / N) * rng.rand(B, N, N, E1)
  A[..., 0] += np.eye(N)
  A *= m[:, :, None, None] * m[:, None, :, None]
  L = (A / np.maximum(A.sum(axis=2, keepdims=True), 1.0)).astype(np.float32)
  assert N == 1 or np.abs(L - L.transpose(0, 2, 1, 3)).max() > 0.1
  V = rng.randn(B, N, K) / np.sqrt(N) * m[:, :, None] * (np.arange(K)[None, None, :] < n[:, None, None])
  if feat_dim is None:
    feat = rng.randint(0, 70, size=(B, N)) * mask
  else:
    feat = (rng.randn(B, N, feat_dim) * m[:, :, None]).astype(np.float32)
  return {'node_feat': feat, 'L': L, 'D': rng.uniform(-1, 1, (B, K)).astype(np.float32),
          'V': V.astype(np.float32), 'node_mask': mask, 'label': rng.randn(B, P).astype(np.float32)}


def _model_case(name, N):
  """(module class, config, oracle forward(params, batch, dtype), uses Ritz pairs, feature width)."""
  if name == 'LanczosNet':
    cfg = configs.qm8_lanczos_net(num_layer=2, hidden_dim=[30, 36], num_eig_vec=40, short_diffusion_dist=[1, 3])
    return LanczosNet, cfg, None, True, None
  if name == 'LanczosNetGeneral':
    cfg = configs.graph_lanczos_net(num_layer=2, hidden_dim=[130, 30], num_eig_vec=40)
    cfg.dataset.num_edge_type = 2
    return LanczosNetGeneral, cfg, None, True, 10
  if name == 'GCN':
    return GCN, configs.qm8_gcn(num_layer=2, hidden_dim=[30, 36]), None, False, None
  if name == 'DCNN':
    cfg = configs.qm8_dcnn(num_layer=2, hidden_dim=[30, 36], diffusion_dist=[2, 5])
    return DCNN, cfg, (lambda p, b, dt: orc.dcnn_forward(p, [2, 5], 6, 2, b['node_feat'], b['L'],
                                                           b['node_mask'], dtype=dt)), False, None
  cfg = configs.qm8_cheby_net(num_layer=2, hidden_dim=[30, 36], polynomial_order=4)
  return ChebyNet, cfg, (lambda p, b, dt: orc.cheby_net_forward(p, 4, 6, 2, b['node_feat'], b['L'],
                                                                 b['node_mask'], dtype=dt)), False, None


def _oracle_loss_grads(forward, params, label, dtype, masks, monkeypatch):
  """d loss / d params by autograd over the oracle in ``dtype`` (its _cast detaches: bypassed), with
  the oracle's ReLUs taking the library's activation pattern ``masks`` (in call order).  ReLU's
  derivative jumps at 0, so a pre-activation within rounding of 0 may fall on either side; away
  from 0 the patterns have to agree.  Returns (loss, grads, worst |pre| / scale where they differ)."""
  p = {k: v.detach().to(dtype).requires_grad_() if v.is_floating_point() else v for k, v in params.items()}
  calls, flips = iter(masks), [0.0]

  def relu(x):
    m = next(calls)
    assert m.shape == x.shape
    pre = x.detach()
    differ = m != (pre > 0)
    if bool(differ.any()):
      flips[0] = max(flips[0], float(pre[differ].abs().max()) / float(pre.abs().max()))
    return x * m.to(x.dtype)

  with monkeypatch.context() as mp:
    mp.setattr(orc, '_cast', lambda p_, dtype_: p_)
    mp.setattr(torch, 'relu', relu)
    loss = torch.nn.functional.mse_loss(forward(p, dtype), torch.from_numpy(label).to(dtype))
  assert next(calls, None) is None
  loss.backward()
  return float(loss.detach()), {k: v.grad for k, v in p.items() if v.is_floating_point()}, flips[0]


@pytest.mark.parametrize('name,N', [('LanczosNet', 33), ('LanczosNet', 128), ('LanczosNetGeneral', 33),
                                    ('GCN', 128), ('DCNN', 33), ('ChebyNet', 128)])
def test_model_gradients_off_grid_vs_fp64(name, N, monkeypatch):
  cls, cfg, forward, ritz, feat_dim = _model_case(name, N)
  mod = cls(cfg)
  params = deterministic_state_dict(mod, 17)
  mod.load_state_dict(params)
  spec = oracle_spec(mod, name) if forward is None else None
  # the smallest batch that puts every convolution Linear on the tensor cores
  per_row = min(2 * f.weight.shape[0] * f.weight.shape[1] for f in mod.filter[:mod.num_layer])
  B = -(-int(train._SMALL_DENSE_FLOPS) // (per_row * N)) + 1
  assert all(2.0 * B * N * f.weight.numel() >= train._SMALL_DENSE_FLOPS for f in mod.filter[:mod.num_layer])
  assert any(f.weight.shape[1] % 4 for f in mod.filter[:mod.num_layer])       # the K padding path
  E1 = mod.num_edgetype + 1
  b = _random_batch(B, N, E1, 40, cfg.model.output_dim, seed=N + E1, feat_dim=feat_dim)
  if forward is None:
    if ritz:
      forward = lambda p, dt: orc.lanczos_net_forward(p, spec, b['node_feat'], b['L'], b['D'], b['V'],
                                                      b['node_mask'], dtype=dt)
    else:
      forward = lambda p, dt: orc.gcn_forward(p, spec, b['node_feat'], b['L'], b['node_mask'], dtype=dt)
  else:
    forward = (lambda f: lambda p, dt: f(p, b, dt))(forward)
  # the library's forward, recording the activation pattern of every ReLU dense layer
  masks = []
  real_dense = train.dense

  def recording_dense(x, weight, bias, relu=False):
    y = real_dense(x, weight, bias, relu)
    if relu:
      masks.append((y.detach() > 0).cpu())
    return y

  monkeypatch.setattr(train, 'dense', recording_dense)
  mod = mod.to(dev()).train()
  args = [torch.from_numpy(b[k]).to(dev()) for k in (('node_feat', 'L', 'D', 'V') if ritz else ('node_feat', 'L'))]
  _, loss = mod(*args, label=torch.from_numpy(b['label']).to(dev()),
                mask=torch.from_numpy(b['node_mask']).to(dev()))
  loss.backward()
  loss64, g64, flip = _oracle_loss_grads(forward, params, b['label'], torch.float64, masks, monkeypatch)
  _, g32, _ = _oracle_loss_grads(forward, params, b['label'], torch.float32, masks, monkeypatch)
  print('%s N=%d: largest |pre-activation| / scale on which the ReLU patterns differ: %.3g' % (name, N, flip))
  assert flip <= 1e-4
  assert abs(float(loss.detach()) - loss64) <= 1e-5 * max(1.0, abs(loss64))
  for pname, p in mod.named_parameters():
    assert p.grad is not None, pname
    _check('%s N=%d B=%d %s' % (name, N, B, pname), p.grad, g64[pname], g32[pname], FLOOR_MODEL)


# ------------------------------------------------------------------------------------------
# 7. the captured training step beyond LanczosNet
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['GCN', 'DCNN', 'ChebyNet', 'LanczosNetGeneral'])
def test_graphed_step_matches_eager_steps(name):
  """Momentum SGD over 6 steps / 3 rotating batches: the captured step (forward + loss + backward
  + optimizer in one CUDA graph) walks the eager trajectory, and building it does not train."""
  from lanczosnetwork_b200.train import GraphedStep
  if name == 'GCN':
    cls, cfg = GCN, configs.qm8_gcn(num_layer=3, hidden_dim=[64, 64, 64])
  elif name == 'DCNN':
    cls, cfg = DCNN, configs.qm8_dcnn(num_layer=3, hidden_dim=[64, 64, 64], diffusion_dist=[1, 3])
  elif name == 'ChebyNet':
    cls, cfg = ChebyNet, configs.qm8_cheby_net(num_layer=3, hidden_dim=[64, 64, 64], polynomial_order=4)
  else:
    cls, cfg = LanczosNetGeneral, configs.graph_lanczos_net(num_layer=3, hidden_dim=[64, 64, 64])
  general = name == 'LanczosNetGeneral'
  batches = []
  for i in range(3):
    bt = data.collate(data.synthetic_qm8_samples(32, seed=50 + i), 20, num_nodes=27)
    rng = np.random.RandomState(i)
    if general:
      bt['node_feat'] = (rng.randn(32, 27, 10) * bt['node_mask'][:, :, None]).astype(np.float32)
      bt['L'] = np.ascontiguousarray(bt['L'][..., :2])
    bt['label'] = rng.randn(32, cfg.model.output_dim).astype(np.float32)
    batches.append({k: torch.from_numpy(v).to(dev()) for k, v in bt.items() if isinstance(v, np.ndarray)})

  def make():
    m = cls(cfg)
    m.load_state_dict(deterministic_state_dict(m, 77))
    m = m.to(dev()).train()
    return m, torch.optim.SGD(m.parameters(), lr=1e-2, momentum=0.9)

  def call_args(bt):
    keys = ('node_feat', 'L', 'D', 'V') if general else ('node_feat', 'L')
    return tuple(bt[k] for k in keys), {'label': bt['label'], 'mask': bt['node_mask']}

  eager, opt_e = make()
  losses_e = []
  for i in range(6):
    a, kw = call_args(batches[i % 3])
    opt_e.zero_grad()
    _, loss = eager(*a, **kw)
    loss.backward()
    opt_e.step()
    losses_e.append(float(loss.detach()))

  graphed, opt_g = make()
  a, kw = call_args(batches[0])
  step = GraphedStep(graphed, opt_g, a, kw)
  for (n, p), (_, q) in zip(graphed.named_parameters(), make()[0].named_parameters()):
    assert torch.equal(p, q), n                              # warm-up rolled back
  losses_g = []
  for i in range(6):
    a, kw = call_args(batches[i % 3])
    _, loss = step(*a, **kw)
    losses_g.append(float(loss.detach()))
  np.testing.assert_allclose(losses_g, losses_e, rtol=1e-5)
  for (n, p), (_, q) in zip(graphed.named_parameters(), eager.named_parameters()):
    np.testing.assert_allclose(p.detach().cpu().numpy(), q.detach().cpu().numpy(), rtol=2e-4, atol=2e-6, err_msg=n)
  assert step.replays == 6
