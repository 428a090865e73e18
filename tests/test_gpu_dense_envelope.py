"""The three forms of the wgmma 3xTF32 dense layer -- plain (lnb_linear_tf32x3), block-diagonal
(lnb_linear_tf32x3_grouped) and split-K (lnb_linear_tf32x3_splitk) -- across the shapes they accept,
against the same product in fp64 on the CPU, and the lifetime of the split-K workspace that
ops.linear_tf32x3 keeps per stream.

Tolerance, as in test_gpu_train_envelope.py: max|got - fp64| <= max(8 x max|fp32 CPU - fp64|,
_deep_floor(K) x scale).  For a grouped layer the scale is taken per group's column block, so a
large group cannot hide an error in a small one.  Where two forms run the same arithmetic they are
also compared bit for bit: a group of the grouped layer is the plain layer on that group's operands
(same k-block order; the W rows a 128-row TMA box reads past the end of a group feed only columns
the epilogue discards), split-K with one split is the plain layer, and the split sums are added in a
fixed order, so a second launch repeats the first.  ``pytest -m gpu``."""
import gc
import math
import random
import weakref

import numpy as np
import pytest
import torch

from helpers import deterministic_state_dict
from lanczosnetwork_b200 import configs, data, ops
from lanczosnetwork_b200.model import LanczosNet
from lanczosnetwork_b200.train import GraphedStep
from test_gpu_train_envelope import MULT, _deep_floor

pytestmark = pytest.mark.gpu

BM = BN = 128          # output tile of the kernel
BK = 32                # k-block
SENTINEL = -1234.5


def dev():
  return torch.device('cuda:0')


def _err(a, b):
  return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max()) if a.numel() else 0.0


def _check(what, got, r64, r32, depth):
  """got within max(MULT x the fp32 CPU error, _deep_floor(depth) x scale) of fp64."""
  scale = float(r64.abs().max()) if r64.numel() else 0.0
  bound = max(MULT * _err(r32, r64), _deep_floor(depth) * scale)
  err = _err(got, r64)
  print('%s: err %.3g  fp32 CPU %.3g  bound %.3g  scale %.3g  err/bound %.3f' % (
      what, err, _err(r32, r64), bound, scale, err / bound if bound else 0.0))
  assert err <= bound, (what, err, bound, scale)


def _ref(x, w, b, relu, dtype):
  y = x.to(dtype) @ w.to(dtype).t()
  if b is not None:
    y = y + b.to(dtype)
  return torch.relu(y) if relu else y


def _operands(M, N, K, has_bias, seed):
  """CPU fp32 x [M,K], w [N,K] (rows of unit norm on average), b [N] or None."""
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(M, K, generator=g)
  w = torch.randn(N, K, generator=g) / math.sqrt(K)
  b = torch.randn(N, generator=g) if has_bias else None
  return x, w, b


def _grouped_operands(M, groups, N, K, has_bias, seed):
  """x [M, groups*K], stacked w [groups*N, K], b [groups*N] or None."""
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(M, groups * K, generator=g)
  w = torch.randn(groups * N, K, generator=g) / math.sqrt(K)
  b = torch.randn(groups * N, generator=g) if has_bias else None
  return x, w, b


def _to_dev(x, w, b):
  w_hi, w_lo = ops.split_tf32(w.to(dev()))
  return x.to(dev()), w_hi, w_lo, (b.to(dev()) if b is not None else None)


def _bits(t):
  return t.contiguous().view(torch.int32)


def _same_bits(a, b):
  return torch.equal(_bits(a), _bits(b))


def _plain_c(x, w_hi, w_lo, b, relu, out, M=None, K=None):
  """lnb_linear_tf32x3 through the C ABI (never split-K, whatever the shape)."""
  M = x.shape[0] if M is None else M
  K = x.shape[1] if K is None else K
  ops._launch('lnb_linear_tf32x3', out, x, w_hi, w_lo, b, M, w_hi.shape[0], K, int(relu), out)


def _splitk_c(x, w_hi, w_lo, b, relu, out, splits, ws, counters, M=None, K=None):
  M = x.shape[0] if M is None else M
  K = x.shape[1] if K is None else K
  ops._launch('lnb_linear_tf32x3_splitk', out, x, w_hi, w_lo, b, M, w_hi.shape[0], K, int(relu), out, splits, ws,
              counters)


def _grouped_c(x, w_hi, w_lo, b, groups, relu, out, M=None):
  M = x.shape[0] if M is None else M
  ops._launch('lnb_linear_tf32x3_grouped', out, x, w_hi, w_lo, b, M, groups, w_hi.shape[0] // groups, w_hi.shape[1],
              int(relu), out)


def _tiles(M, N):
  return -(-M // BM) * -(-N // BN)


# ------------------------------------------------------------------------------------------
# 1. grouped (block-diagonal) layer
# ------------------------------------------------------------------------------------------
G_GROUPS, G_N, G_K, G_M = (1, 2, 7, 16), (1, 8, 32, 100, 128, 200, 256), (4, 32, 36, 128, 132), (1, 127, 129, 700)


def _grouped_cases():
  """Every value of every axis at least once, then a seeded sample of the rest of the grid.
  groups, N per group, K, M, relu, bias."""
  cases = [(1, 1, 4, 1, False, False),
           (2, 8, 32, 127, True, True),
           (7, 32, 36, 129, False, True),
           (16, 100, 128, 700, True, False),
           (7, 128, 132, 129, True, True),
           (16, 200, 36, 700, False, True),    # second column tile of a group: its box reads 56 rows of the next
           (16, 256, 132, 700, True, True)]
  rng = random.Random(90)
  while len(cases) < 48:
    c = (rng.choice(G_GROUPS), rng.choice(G_N), rng.choice(G_K), rng.choice(G_M), rng.random() < 0.5,
         rng.random() < 0.5)
    if c not in cases:
      cases.append(c)
  return cases


@pytest.mark.parametrize('groups,N,K,M,relu,has_bias', _grouped_cases())
def test_grouped_vs_fp64_and_plain_layer(groups, N, K, M, relu, has_bias):
  x, w, b = _grouped_operands(M, groups, N, K, has_bias, groups * 1000 + N * 31 + K * 7 + M)
  xd, w_hi, w_lo, bd = _to_dev(x, w, b)
  out = ops.linear_tf32x3_grouped(xd, w_hi, w_lo, bd, groups, relu)
  assert out.shape == (M, groups * N)
  assert -(-K // BK) < 32                                      # ops.linear_tf32x3 below runs without split-K
  for g in range(groups):
    cols, rows = slice(g * K, (g + 1) * K), slice(g * N, (g + 1) * N)
    bg = b[rows] if has_bias else None
    tag = 'grouped groups=%d N=%d K=%d M=%d relu=%d bias=%d group %d' % (groups, N, K, M, relu, has_bias, g)
    _check(tag, out[:, rows], _ref(x[:, cols], w[rows], bg, relu, torch.float64),
           _ref(x[:, cols], w[rows], bg, relu, torch.float32), K)
    alone = ops.linear_tf32x3(xd[:, cols].contiguous(), w_hi[rows], w_lo[rows],
                              bd[rows] if has_bias else None, relu)
    assert _same_bits(out[:, rows], alone), tag


@pytest.mark.parametrize('groups,N,K', [(7, 200, 36), (16, 8, 132)])
@pytest.mark.parametrize('poisoned', ['middle', 'last'])
def test_grouped_groups_do_not_see_each_other(groups, N, K, poisoned):
  """NaN in one group's A columns and W rows reaches that group's block only.  N = 200 puts the
  second column tile's TMA box across the next group's rows; N = 8 puts 16 groups in one box;
  K = 36 leaves a partial k-block whose load must stop at the group's own columns."""
  M = 129
  x, w, b = _grouped_operands(M, groups, N, K, True, groups + N + K)
  xd, w_hi, w_lo, bd = _to_dev(x, w, b)
  clean = ops.linear_tf32x3_grouped(xd, w_hi, w_lo, bd, groups, False)
  p = groups // 2 if poisoned == 'middle' else groups - 1
  xp, wp = x.clone(), w.clone()
  xp[:, p * K:(p + 1) * K] = float('nan')
  wp[p * N:(p + 1) * N] = float('nan')
  xpd, wp_hi, wp_lo, _ = _to_dev(xp, wp, None)
  out = ops.linear_tf32x3_grouped(xpd, wp_hi, wp_lo, bd, groups, False)
  assert bool(torch.isnan(out[:, p * N:(p + 1) * N]).all())        # the poison did reach the kernel
  for g in range(groups):
    if g == p:
      continue
    blk = out[:, g * N:(g + 1) * N]
    assert bool(torch.isfinite(blk).all()), (g, p)
    assert _same_bits(blk, clean[:, g * N:(g + 1) * N]), (g, p)


# ------------------------------------------------------------------------------------------
# 2. split-K through the C ABI, with the test's own workspace and counters
# ------------------------------------------------------------------------------------------
# M, N, K, splits, relu, bias; the k-block ranges of the splits in the comments
SPLITK = [
    (1, 1, 64, 2, False, True),              # nkb 2: 1, 1
    (127, 3, 68, 3, True, True),             # nkb 3: 1, 1, 1 (the last k-block 4 columns wide)
    (128, 128, 544, 5, False, True),         # nkb 17: 4, 4, 4, 4, 1
    (129, 129, 540, 3, True, False),         # nkb 17: 6, 6, 5
    (1000, 1, 520, 2, False, True),          # nkb 17: 9, 8
    (127, 1, 2016, 16, True, True),          # nkb 63: 15 x 4, 3
    (129, 3, 2000, 5, False, False),         # nkb 63: 4 x 13, 11
    (128, 520, 2016, 8, True, True),         # nkb 63: 7 x 8, 7
    (1000, 3, 2016, 16, False, True),        # nkb 63: 15 x 4, 3
    (1, 128, 4096, 3, False, True),          # nkb 128: 43, 43, 42
    (129, 520, 4096, 5, True, True),         # nkb 128: 4 x 26, 24
    (1000, 520, 4096, 16, True, False),      # nkb 128: 16 x 8; 640 work items, several per CTA
    (1, 520, 4100, 8, False, True),          # nkb 129: 7 x 17, 10
    (1000, 129, 4128, 2, True, True),        # nkb 129: 65, 64
    (127, 129, 96, 1, False, True),          # nkb 3, one split
    (1000, 520, 40, 1, True, True),          # nkb 2, one split
]


@pytest.mark.parametrize('M,N,K,splits,relu,has_bias', SPLITK)
def test_splitk_c_entry_vs_fp64(M, N, K, splits, relu, has_bias):
  nkb = -(-K // BK)
  per = -(-nkb // splits)
  assert per * (splits - 1) < nkb                              # a shape the entry accepts
  tiles = _tiles(M, N)
  x, w, b = _operands(M, N, K, has_bias, M * 7 + N * 3 + K + splits)
  xd, w_hi, w_lo, bd = _to_dev(x, w, b)
  need, guard = tiles * splits * BM * BN, 4096
  ws = torch.full((need + guard,), SENTINEL, device=dev())
  counters = torch.zeros(tiles + 64, device=dev(), dtype=torch.int32)
  outs = [torch.empty(M, N, device=dev()) for _ in range(2)]
  for o in outs:
    _splitk_c(xd, w_hi, w_lo, bd, relu, o, splits, ws, counters)
  tag = 'splitk M=%d N=%d K=%d splits=%d (ranges %d x %d, last %d; %d items on %d SMs) relu=%d bias=%d' % (
      M, N, K, splits, splits - 1, per, nkb - per * (splits - 1), tiles * splits, ops._sm_count(dev()),
      relu, has_bias)
  _check(tag, outs[0], _ref(x, w, b, relu, torch.float64), _ref(x, w, b, relu, torch.float32), K)
  assert _same_bits(outs[0], outs[1]), tag                     # the split sums have a fixed order
  assert int(counters.abs().sum()) == 0, counters.nonzero()    # every counter back at zero
  assert bool((ws[need:] == SENTINEL).all())                   # nothing written past the workspace
  if splits == 1:
    plain = torch.empty(M, N, device=dev())
    _plain_c(xd, w_hi, w_lo, bd, relu, plain)
    assert _same_bits(outs[0], plain)
    nows = torch.empty(M, N, device=dev())
    _splitk_c(xd, w_hi, w_lo, bd, relu, nows, 1, None, None)   # one split needs no workspace
    assert _same_bits(nows, plain)


# ------------------------------------------------------------------------------------------
# 3. writes stay inside the output
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M', [1, 129])
def test_writes_stay_inside_the_output(M):
  """The output is the first M rows of an (M+1)-row buffer filled with a sentinel: all of those M
  rows are written, row M keeps the sentinel."""
  def run(what, width, fn, ref64, ref32, depth):
    buf = torch.full((M + 1, width), SENTINEL, device=dev())
    fn(buf)
    torch.cuda.synchronize()
    assert bool((buf[M] == SENTINEL).all()), what + ': wrote past row M'
    assert not bool((buf[:M] == SENTINEL).any()), what + ': left output entries unwritten'
    _check('%s M=%d' % (what, M), buf[:M], ref64, ref32, depth)

  N = 129
  for K in (36, 2016):                                         # K = 2016: ops.linear_tf32x3 runs split-K
    x, w, b = _operands(M, N, K, True, M + K)
    xd, w_hi, w_lo, bd = _to_dev(x, w, b)
    r64, r32 = _ref(x, w, b, True, torch.float64), _ref(x, w, b, True, torch.float32)

    def plain(buf):
      y = ops.linear_tf32x3(xd, w_hi, w_lo, bd, True, out=buf[:M])
      assert y.data_ptr() == buf.data_ptr()
    run('plain out= K=%d' % K, N, plain, r64, r32, K)
    if K == 2016:
      splits, tiles = 5, _tiles(M, N)
      ws = torch.empty(tiles * splits * BM * BN, device=dev())
      counters = torch.zeros(tiles, device=dev(), dtype=torch.int32)
      run('splitk C entry K=%d' % K, N, lambda buf: _splitk_c(xd, w_hi, w_lo, bd, True, buf, splits, ws, counters, M=M),
          r64, r32, K)
  groups, N, K = 3, 200, 36
  x, w, b = _grouped_operands(M, groups, N, K, True, M + 7)
  xd, w_hi, w_lo, bd = _to_dev(x, w, b)
  r = [torch.cat([_ref(x[:, g * K:(g + 1) * K], w[g * N:(g + 1) * N], b[g * N:(g + 1) * N], False, dt)
                  for g in range(groups)], dim=1) for dt in (torch.float64, torch.float32)]
  run('grouped C entry', groups * N, lambda buf: _grouped_c(xd, w_hi, w_lo, bd, groups, False, buf, M=M),
      r[0], r[1], K)


# ------------------------------------------------------------------------------------------
# 4. refusals, before any launch
# ------------------------------------------------------------------------------------------
def test_refusals_happen_before_launch():
  M, N, K = 129, 129, 160                                      # nkb = 5
  x, w, b = _operands(M, N, K, True, 3)
  xd, w_hi, w_lo, bd = _to_dev(x, w, b)
  tiles = _tiles(M, N)
  ws = torch.zeros(tiles * 17 * BM * BN, device=dev())
  counters = torch.zeros(tiles, device=dev(), dtype=torch.int32)
  out = torch.full((M, N), SENTINEL, device=dev())
  x_odd = torch.zeros(M * K + 4, device=dev())[1:1 + M * K].view(M, K)   # 4 bytes off 16-byte alignment
  x_odd.copy_(xd)
  assert x_odd.data_ptr() % 16 == 4
  x12, w12 = torch.zeros(M, 12, device=dev()), torch.zeros(N, 12, device=dev())   # read as K = 10

  def refused(what, exc, fn):
    n0 = ops.launch_count()
    with pytest.raises(exc) as info:
      fn()
    torch.cuda.synchronize()
    assert ops.launch_count() == n0, what
    assert bool((out == SENTINEL).all()), what
    print('%s: %s' % (what, info.value))

  refused('splits = 0', RuntimeError, lambda: _splitk_c(xd, w_hi, w_lo, bd, False, out, 0, ws, counters))
  refused('splits = 17', RuntimeError, lambda: _splitk_c(xd, w_hi, w_lo, bd, False, out, 17, ws, counters))
  refused('nkb = 5, splits = 4: empty last range', RuntimeError,
          lambda: _splitk_c(xd, w_hi, w_lo, bd, False, out, 4, ws, counters))
  refused('null workspace', RuntimeError, lambda: _splitk_c(xd, w_hi, w_lo, bd, False, out, 2, None, counters))
  refused('null counters', RuntimeError, lambda: _splitk_c(xd, w_hi, w_lo, bd, False, out, 2, ws, None))
  for name, fn in (('plain', _plain_c), ('splitk', lambda *a, **k: _splitk_c(*a, 2, ws, counters, **k))):
    refused('%s K %% 4 != 0' % name, RuntimeError, lambda: fn(x12, w12, w12, None, False, out, K=10))
    refused('%s A not 16-byte aligned' % name, RuntimeError, lambda: fn(x_odd, w_hi, w_lo, bd, False, out))
  refused('grouped A not 16-byte aligned', RuntimeError,
          lambda: _grouped_c(x_odd, w_hi, w_lo, bd, 1, False, out))
  # ops.linear_tf32x3(out=...) takes a contiguous float32 [M, N] tensor on the input's device only
  for what, bad in (('float64', torch.empty(M, N, device=dev(), dtype=torch.float64)),
                    ('[M, N+1]', torch.empty(M, N + 1, device=dev())),
                    ('[M+1, N]', torch.empty(M + 1, N, device=dev())),
                    ('transposed view', torch.empty(N, M, device=dev()).t()),
                    ('cpu', torch.empty(M, N))):
    refused('out= ' + what, ValueError, lambda: ops.linear_tf32x3(xd, w_hi, w_lo, bd, False, out=bad))


# ------------------------------------------------------------------------------------------
# 5. the split-K workspace of ops.linear_tf32x3 outlives the graphs that captured it
# ------------------------------------------------------------------------------------------
def _record_workspaces(monkeypatch):
  """Start from no split-K workspaces and record (stream handle, request, weakrefs to the pair) of
  every workspace ops.linear_tf32x3 asks for."""
  monkeypatch.setattr(ops, '_SPLITK_WS', {})
  calls = []
  real = ops._splitk_workspace

  def recording(device, nfloats, ntiles):
    ws, counters = real(device, nfloats, ntiles)
    calls.append({'stream': torch.cuda.current_stream(device).cuda_stream, 'nfloats': nfloats,
                  'numel': ws.numel(), 'ws': weakref.ref(ws), 'counters': weakref.ref(counters)})
    return ws, counters

  monkeypatch.setattr(ops, '_splitk_workspace', recording)
  return calls


def _larger_request_on(calls):
  """Another user of each recorded stream handle (torch hands pooled handles out again) runs a
  split-K GEMM that needs more partial tiles than any request so far; afterwards every recorded
  workspace must still be alive.  Returns the recorded entries."""
  held = list(calls)
  assert held, 'nothing ran split-K'
  x, w, _ = _operands(1, 4096, 4096, False, 11)
  xd, w_hi, w_lo, _ = _to_dev(x, w, None)
  cur = torch.cuda.current_stream(dev())
  for handle in sorted({c['stream'] for c in held}):
    ext = torch.cuda.ExternalStream(handle, device=dev())
    ext.wait_stream(cur)
    n = len(calls)
    with torch.cuda.stream(ext):
      ops.linear_tf32x3(xd, w_hi, w_lo)
    assert len(calls) == n + 1 and calls[-1]['nfloats'] > max(c['nfloats'] for c in held)
    cur.wait_stream(ext)
  torch.cuda.synchronize()
  gc.collect()
  dead = [c['nfloats'] for c in held if c['ws']() is None or c['counters']() is None]
  assert not dead, ('%d of %d split-K workspaces (requests of %s floats) freed while a captured graph '
                    'still uses them' % (len(dead), len(held), sorted(set(dead))))
  return held


def _victim(held):
  """A patterned tensor the size of the largest recorded workspace, allocated on its stream."""
  c = max(held, key=lambda c: c['numel'])
  ext = torch.cuda.ExternalStream(c['stream'], device=dev())
  with torch.cuda.stream(ext):
    v = torch.arange(c['numel'], device=dev(), dtype=torch.float32).remainder_(1021.0)
  torch.cuda.synchronize()
  return v, v.clone()


def test_graphed_step_keeps_its_splitk_workspace(monkeypatch):
  """The default QM8 LanczosNet at B = 64, N = 27: every convolution Linear's weight gradient g^T x
  contracts over 1728 rows and runs split-K.  GraphedStep warms up and captures on a fresh stream;
  a later, larger split-K request on the same stream handle must not free the workspace the graph
  holds, and the replays walk the eager trajectory."""
  cfg = configs.qm8_lanczos_net()
  batches = []
  for i in range(3):
    bt = data.collate(data.synthetic_qm8_samples(64, seed=60 + i), cfg.model.num_eig_vec, num_nodes=27)
    bt['label'] = np.random.RandomState(i).randn(64, cfg.model.output_dim).astype(np.float32)
    batches.append({k: torch.from_numpy(v).to(dev()) for k, v in bt.items() if isinstance(v, np.ndarray)})

  def make():
    m = LanczosNet(cfg)
    m.load_state_dict(deterministic_state_dict(m, 78))
    m = m.to(dev()).train()
    return m, torch.optim.SGD(m.parameters(), lr=1e-2, momentum=0.9)

  def call_args(bt):
    return (bt['node_feat'], bt['L'], bt['D'], bt['V']), {'label': bt['label'], 'mask': bt['node_mask']}

  eager, opt_e = make()
  losses_e = []
  for i in range(6):
    a, kw = call_args(batches[i % 3])
    opt_e.zero_grad()
    _, loss = eager(*a, **kw)
    loss.backward()
    opt_e.step()
    losses_e.append(float(loss.detach()))

  calls = _record_workspaces(monkeypatch)
  graphed, opt_g = make()
  a, kw = call_args(batches[0])
  step = GraphedStep(graphed, opt_g, a, kw)
  held = _larger_request_on(calls)
  victim, pattern = _victim(held)
  losses_g = []
  for i in range(6):
    a, kw = call_args(batches[i % 3])
    _, loss = step(*a, **kw)
    losses_g.append(float(loss.detach()))
  torch.cuda.synchronize()
  assert torch.equal(victim, pattern)
  np.testing.assert_allclose(losses_g, losses_e, rtol=1e-5)
  for (n, p), (_, q) in zip(graphed.named_parameters(), eager.named_parameters()):
    np.testing.assert_allclose(p.detach().cpu().numpy(), q.detach().cpu().numpy(), rtol=2e-4, atol=2e-6, err_msg=n)


def test_captured_linear_keeps_its_splitk_workspace(monkeypatch):
  """The same warm-up-then-capture pattern on ops.linear_tf32x3 alone: warm-up and capture on a fresh
  stream, a larger request on that stream handle, then replays on new inputs."""
  calls = _record_workspaces(monkeypatch)
  M, N, K = 128, 256, 2048                                     # 2 tiles, 4 splits
  _, w, b = _operands(M, N, K, True, 5)
  xs = [torch.randn(M, K, generator=torch.Generator().manual_seed(100 + i)) for i in range(4)]
  x_static, w_hi, w_lo, bd = _to_dev(xs[0], w, b)
  cur = torch.cuda.current_stream(dev())
  side = torch.cuda.Stream(device=dev())
  side.wait_stream(cur)
  with torch.cuda.stream(side):
    for _ in range(3):
      ops.linear_tf32x3(x_static, w_hi, w_lo, bd, True)
  cur.wait_stream(side)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, stream=side):
    y_static = ops.linear_tf32x3(x_static, w_hi, w_lo, bd, True)
  assert {c['stream'] for c in calls} == {side.cuda_stream}
  held = _larger_request_on(calls)
  victim, pattern = _victim(held)
  for i in (1, 2, 3):
    x_static.copy_(xs[i].to(dev()))
    graph.replay()
    eager = ops.linear_tf32x3(x_static, w_hi, w_lo, bd, True)
    assert _same_bits(y_static, eager), i
    _check('captured split-K replay %d' % i, y_static, _ref(xs[i], w, b, True, torch.float64),
           _ref(xs[i], w, b, True, torch.float32), K)
  torch.cuda.synchronize()
  assert torch.equal(victim, pattern)


# ------------------------------------------------------------------------------------------
# 6. two streams, two split-K GEMMs in flight together
# ------------------------------------------------------------------------------------------
def test_two_streams_keep_separate_splitk_workspaces(monkeypatch):
  """Two different split-K GEMMs interleaved on two streams with no synchronisation between them,
  8 launches each: every result within the bound and equal to the others of its stream."""
  calls = _record_workspaces(monkeypatch)
  shapes = [(256, 128, 4096, False), (64, 384, 2048, True)]    # 2 tiles x 8 splits, 3 tiles x 4 splits
  cur = torch.cuda.current_stream(dev())
  streams = [torch.cuda.Stream(device=dev()) for _ in shapes]
  assert streams[0].cuda_stream != streams[1].cuda_stream
  ops_in, refs, outs = [], [], []
  for i, (M, N, K, relu) in enumerate(shapes):
    x, w, b = _operands(M, N, K, True, 40 + i)
    ops_in.append(_to_dev(x, w, b) + (relu,))
    refs.append((_ref(x, w, b, relu, torch.float64), _ref(x, w, b, relu, torch.float32), K))
    outs.append([torch.empty(M, N, device=dev()) for _ in range(8)])
  for s in streams:
    s.wait_stream(cur)
  for it in range(8):
    for s, args, o in zip(streams, ops_in, outs):
      with torch.cuda.stream(s):
        xd, w_hi, w_lo, bd, relu = args
        ops.linear_tf32x3(xd, w_hi, w_lo, bd, relu, out=o[it])
  for s in streams:
    cur.wait_stream(s)
  torch.cuda.synchronize()
  pairs = {c['stream']: c['ws']() for c in calls}
  assert set(pairs) == {s.cuda_stream for s in streams}, 'both GEMMs run split-K, one workspace per stream'
  assert pairs[streams[0].cuda_stream].data_ptr() != pairs[streams[1].cuda_stream].data_ptr()
  for (M, N, K, _), o, (r64, r32, depth) in zip(shapes, outs, refs):
    for it in range(8):
      _check('two streams M=%d N=%d K=%d launch %d' % (M, N, K, it), o[it], r64, r32, depth)
      assert _same_bits(o[it], o[0]), it
