"""The persistent wgmma kernels with several work items per CTA.  Every tensor-core kernel is one
launch of the skeleton in csrc/tc_gemm.cuh on min(items, SMs) CTAs, each striding over the items;
the ring counters and their mbarrier parities, the W cursor, the producer group that owns a k-block,
kept drains and the policies' per-item members all carry over from one item to the next, and at the
envelope tests' batch sizes no CTA ever takes a second item.  lnb_debug_set_max_ctas caps the grid,
and no kernel waits on another CTA or adds floats in an order that depends on the grid, so under
every cap each output must be bit-identical to the full grid's.  At one CTA, where a single CTA
runs every item, the output is also checked against fp64 with the envelope tests' bounds.  Every
float32 output starts as NaN, so a row a cap leaves unwritten shows.  ``pytest -m gpu``."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import deterministic_state_dict
from lanczosnetwork_b200 import _lib, configs, data, ops
from lanczosnetwork_b200 import spectral_conv as sc
from lanczosnetwork_b200.model import GGNN, LanczosNet, LSTMGraphSAGE
from lanczosnetwork_b200.model.ggnn import gru_gate_matrix
from lanczosnetwork_b200.model.graph_sage import lstm_gate_matrix
from test_gpu_conv_envelope import STACK_FLOOR_PER_LAYER, _assert_mlp, _check, _mlp_cases, _mlp_layers, conv_ref, \
    mlp_ref, stack_ref
from test_gpu_dense_envelope import _check as dense_check
from test_gpu_dense_envelope import _grouped_c, _grouped_operands, _operands, _plain_c, _splitk_c, _to_dev
from test_gpu_dense_envelope import _ref as dense_ref
from test_gpu_ggnn import KERNEL_FLOOR as GGNN_FLOOR
from test_gpu_ggnn import _update_inputs as ggnn_inputs
from test_gpu_ggnn import update_reference as ggnn_reference
from test_gpu_gpnn import _check as gpnn_check
from test_gpu_gpnn import _gates as gpnn_gates
from test_gpu_gpnn import _operators as gpnn_operators
from test_gpu_gpnn import _weights as gpnn_weights
from test_gpu_gpnn import partition_reference
from test_gpu_graphsage import CASES as SAGE_CASES
from test_gpu_graphsage import random_samples as sage_samples
from test_gpu_graphsage import restate
from test_gpu_graphsage_lstm import STEP_CASES, STEP_FLOOR
from test_gpu_graphsage_lstm import random_samples as lstm_samples
from test_gpu_mpnn import H as MPNN_H
from test_gpu_mpnn import _bound_check as mpnn_check
from test_gpu_mpnn import _prep as mpnn_prep
from test_gpu_mpnn import _update_inputs as mpnn_inputs
from test_gpu_mpnn import update_reference as mpnn_reference
from test_gpu_stack_vz import _batch as stack_batch
from test_gpu_stack_vz import _model as stack_model

pytestmark = pytest.mark.gpu

CAPS = (1, 2, 3, 7)
BM = 128


def dev():
  return torch.device('cuda:0')


def _sms():
  return torch.cuda.get_device_properties(dev()).multi_processor_count


# ------------------------------------------------------------------------------------------
# the cap, NaN outputs, bit-identity
# ------------------------------------------------------------------------------------------
def _set_cap(n):
  _lib.check(_lib.load().lnb_debug_set_max_ctas(int(n)), 'lnb_debug_set_max_ctas')


@contextlib.contextmanager
def max_ctas(n):
  """Every persistent wgmma launch inside runs on at most n CTAs; the cap is removed on the way out,
  whatever happens inside."""
  _set_cap(n)
  try:
    yield
  finally:
    _set_cap(0)


_PROF = []


def _prof_buffer():
  """The phase-timer buffer of this module, allocated once and never freed: a kernel's copy of the
  buffer pointer is only cleared at that kernel's next launch, so it must stay valid until then."""
  if not _PROF:
    _PROF.append(torch.zeros(_sms() * 32, dtype=torch.int64, device=dev()))
  return _PROF[0]


def _ctas_of(run):
  """CTAs of the one persistent launch run() makes: slot 13 of the phase timers (the CTA's start
  time) is written by every CTA of the grid."""
  buf = _prof_buffer()
  buf.zero_()
  lib = _lib.load()
  _lib.check(lib.lnb_debug_set_prof(ctypes.c_void_p(buf.data_ptr())), 'lnb_debug_set_prof')
  try:
    run()
    torch.cuda.synchronize()
  finally:
    _lib.check(lib.lnb_debug_set_prof(None), 'lnb_debug_set_prof')
  return int((buf.view(-1, 32)[:, 13] != 0).sum())


def _probe_grid():
  """The grid of a dense-layer launch over more items than SMs (two launches: the second clears the
  dense kernel's copy of the phase-timer pointer)."""
  n = _sms() + 5
  x = torch.zeros(BM, 4, device=dev())
  w = torch.zeros(n * 128, 4, device=dev())
  out = torch.empty(BM, n * 128, device=dev())
  run = lambda: _plain_c(x, w, w, None, False, out)
  ctas = _ctas_of(run)
  run()
  torch.cuda.synchronize()
  return ctas


@pytest.fixture(autouse=True)
def _cap_is_not_left_set():
  """A cap that leaked out of a test would make every later test run something else."""
  yield
  ctas = _probe_grid()
  if ctas != _sms():
    _set_cap(0)
    pytest.fail('the grid cap was left set: a dense launch ran on %d of %d SMs' % (ctas, _sms()))


class _NaNEmpty:
  """torch as ops.py sees it, except that torch.empty fills float32 tensors with NaN."""

  def __getattr__(self, name):
    return getattr(torch, name)

  @staticmethod
  def empty(*args, **kwargs):
    t = torch.empty(*args, **kwargs)
    return t.fill_(float('nan')) if t.dtype == torch.float32 else t


@contextlib.contextmanager
def _nan_outputs():
  """Every float32 buffer the ops allocate inside starts as NaN."""
  real = ops.torch
  ops.torch = _NaNEmpty()
  try:
    yield
  finally:
    ops.torch = real


def _nan(*shape):
  return torch.full(shape, float('nan'), device=dev())


def _bits(t):
  return t.contiguous().view(torch.int32)


def _assert_same(got, want, what):
  assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
  diff = _bits(got) != _bits(want)
  if bool(diff.any()):
    first = diff.nonzero()[0].tolist()
    raise AssertionError('%s: %d elements differ from the full grid, first at %s: %r vs %r' % (
        what, int(diff.sum()), first, float(got[tuple(first)]), float(want[tuple(first)])))


def _caps_for(items, caps=CAPS):
  """The caps under which every CTA takes at least three items (cap 1 whenever there are two)."""
  assert items >= 2, items
  return [c for c in caps if c == 1 or items >= 3 * c]


def _sweep(run, items, what, caps=CAPS):
  """run() -> float32 outputs.  Runs at the full grid and under each cap, with NaN outputs, and
  asserts bit-identity.  Returns the outputs at one CTA."""
  caps = _caps_for(items, caps)
  with _nan_outputs():
    full = [t.clone() for t in run()]
  at_one = None
  for cap in caps:
    with max_ctas(cap), _nan_outputs():
      got = run()
    torch.cuda.synchronize()
    for i, (g, f) in enumerate(zip(got, full)):
      _assert_same(g, f, '%s cap=%d output %d' % (what, cap, i))
    if cap == 1:
      at_one = got
  print('%s: %d items, caps %s: bit-identical' % (what, items, caps))
  return at_one


def _graphs_for_tiles(rows_per_graph, tiles):
  """Graphs whose rows fill `tiles` 128-row tiles, the last one only partly."""
  return ((tiles - 1) * BM) // rows_per_graph + 1


def _stack_tiles(prep, B):
  return int(prep[4][B + 2] if B >= 2 else prep[4][0])


# ------------------------------------------------------------------------------------------
# the cap reaches every launch site
# ------------------------------------------------------------------------------------------
def _launch_sites():
  """(name, run, items as the launch counts them, ctas argument) of every persistent wgmma entry."""
  d = dev()
  g = torch.Generator().manual_seed(13)
  rnd = lambda *s: torch.randn(*s, generator=g).to(d)
  sites = []
  # dense: plain, grouped, split-K
  x, w = rnd(1000, 36), rnd(257, 36) / 6
  w_hi, w_lo = ops.split_tf32(w)
  out = torch.empty(1000, 257, device=d)
  sites.append(('dense', lambda: _plain_c(x, w_hi, w_lo, None, True, out), 8 * 3, 0))
  xg, wg = rnd(129, 7 * 36), rnd(7 * 200, 36) / 6
  wg_hi, wg_lo = ops.split_tf32(wg)
  outg = torch.empty(129, 7 * 200, device=d)
  sites.append(('grouped', lambda: _grouped_c(xg, wg_hi, wg_lo, None, 7, False, outg), 2 * 2 * 7, 0))
  xs, ws_ = rnd(129, 4096), rnd(129, 4096) / 64
  ws_hi, ws_lo = ops.split_tf32(ws_)
  outs = torch.empty(129, 129, device=d)
  work = torch.empty(4 * 5 * BM * BM, device=d)
  counters = torch.zeros(4, dtype=torch.int32, device=d)
  sites.append(('split-K', lambda: _splitk_c(xs, ws_hi, ws_lo, None, False, outs, 5, work, counters), 4 * 5, 0))
  # GRU updates
  B, N, D, E1 = 40, 26, 128, 7
  M, h, L, w_ih, w_hh, b_ih, b_hh = ggnn_inputs(g, B, N, D, E1, d)
  gprep = ops.graph_prepare(L, torch.zeros((B, N, 4), device=d), binarize=True)
  Wgg, bgg = gru_gate_matrix(w_ih, w_hh, b_ih, b_hh)
  gg_hi, gg_lo = ops.split_tf32(Wgg)
  outgg = torch.empty(B * N, D, device=d)
  items = -(-B * N // BM) * D // 32
  sites.append(('GGNN', lambda: ops.ggnn_update(M, h, gprep, gg_hi, gg_lo, bgg, True, out=outgg), items, 0))
  PQ, hm, Lm, Fm, whm, bim, bhm = mpnn_inputs(g, B, N, D, E1)
  Wm, bm = gru_gate_matrix(F.pad(Fm, (0, E1 * MPNN_H + 32 - Fm.shape[1])), whm, bim, bhm)
  m_hi, m_lo = ops.split_tf32(Wm)
  mprep = mpnn_prep(Lm)
  outm = torch.empty(B * N, D, device=d)
  sites.append(('MPNN', lambda: ops.mpnn_update(PQ, hm, mprep, m_hi, m_lo, bm, False, out=outm), items, 0))
  Bp, H = 10, 128
  P = gpnn_operators(g, Bp, N).to(d)
  pprep = ops.graph_prepare(P, torch.zeros((Bp, N, 4), device=d))
  gates = gpnn_gates(*gpnn_weights(g, H))
  Mp, hp = rnd(Bp * N, H), rnd(Bp * N, H)
  outp = [torch.empty(Bp * N, H, device=d) for _ in range(2)]
  sites.append(('GPNN partition', lambda: ops.gpnn_partition_update([(Mp, hp, outp[0]), (Mp, hp, outp[1])], pprep,
                                                                    *gates, True),
                -(-Bp * N // BM) * 2 * 4, 0))
  # LSTM step
  Bl, Nl, Dl, El, Kl = 4, 26, 64, 7, 3
  nn_idx, ne = lstm_samples(np.random.RandomState(3), Bl, Nl, Kl, El)
  R = Bl * Nl * El
  state, idx, nev = rnd(Bl * Nl, Dl), torch.from_numpy(nn_idx).to(d).int(), torch.from_numpy(ne.reshape(-1)).to(d)
  Wl, bl = lstm_gate_matrix(rnd(4 * Dl, Dl) / 8, rnd(4 * Dl, Dl) / 8, rnd(4 * Dl), rnd(4 * Dl))
  l_hi, l_lo = ops.split_tf32(Wl)
  hl, cl, outl = rnd(R, Dl), rnd(R, Dl), torch.empty(R, Dl, device=d)
  sites.append(('LSTM step', lambda: ops.sage_lstm_step(state, idx, nev, hl, cl, l_hi, l_lo, bl, 1, outl),
                -(-R // BM) * 2, 0))
  # filter-MLP chain, also with its ctas argument
  layers = _mlp_layers(g, 3, 8, 128)
  table = (torch.rand(1000, 8, generator=g) * 2 - 1).to(d)
  c_hi, c_lo, c_b = sc.WeightCache().split_mlp_chain('chain', layers)
  for ctas in (0, 5):
    sites.append(('chain ctas=%d' % ctas, lambda ctas=ctas: ops.ritz_filter_mlp(table, c_hi, c_lo, c_b, 3, ctas=ctas),
                  8 * 3, ctas))
  # convolution stacks: one layer, the plain stack, GraphSAGE Mean and Max
  Bs, Ns, Ks, Es, S = 40, 26, 20, 7, 8
  sizes = np.random.RandomState(5).randint(3, Ns + 1, size=Bs)
  Ls, Vs = stack_batch(Bs, Ns, Ks, Es, sizes, [min(Ks, int(s)) for s in sizes], 5)
  Ls, Vs = Ls.to(d), Vs.to(d)
  sprep = ops.graph_prepare(Ls, Vs)
  dins, Hs = [64, 128], 128
  Wgs, bgs, coeffs, ro, (s_hi, s_lo, s_b) = stack_model(dins, Hs, S, Ks, Es, 16, Bs, 5)
  Xs = rnd(Bs, Ns, 64)
  cv_hi, cv_lo = ops.split_tf32(Wgs[0][:, :(S + Es) * 64].contiguous())
  sites.append(('conv layer', lambda: ops.spectral_conv_fused(Xs, Vs, coeffs[0], sprep, cv_hi, cv_lo, bgs[0], True),
                Bs, 0))
  sites.append(('stack', lambda: ops.spectral_stack_forward(sprep, Vs, s_hi, s_lo, s_b, dins, Hs, S, coeff=coeffs,
                                                            coeff_stride=coeffs.stride(0), X=Xs, readout=ro), Bs, 0))
  Msg = ops.sage_operators(torch.from_numpy(nn_idx).to(d), nev.view(Bl, Nl))
  gsprep = ops.graph_prepare(torch.cat([Msg] * 10), torch.zeros((10 * Bl, Nl, 4), device=d))
  sw_hi, sw_lo = ops.split_tf32(rnd(2 * Hs, El * Hs) / 30)
  sb = rnd(2 * Hs)
  Xg, Vg = rnd(10 * Bl, Nl, 64), torch.zeros((10 * Bl, Nl, 4), device=d)
  for agg in ('Mean', 'Max'):
    sites.append(('GraphSAGE %s stack' % agg,
                  lambda agg=agg: ops.spectral_stack_forward(gsprep, Vg, sw_hi, sw_lo, sb, [64, Hs], Hs, 0, X=Xg,
                                                             want_state=True, sage=agg), 10 * Bl, 0))
  return sites


def test_cap_reaches_every_launch_site():
  """Each entry runs on min(items, cap) CTAs under a cap and min(items, SMs) without one (the chain:
  also at most its ctas argument), and still counts one launch per op."""
  sms = _sms()
  sites = _launch_sites()
  assert len(sites) == 13
  try:
    for name, run, items, ctas in sites:
      for cap in (0, 3, 7):
        bounds = [b for b in (items, sms, ctas, cap) if b > 0]
        n0 = ops.launch_count()
        with max_ctas(cap):
          got = _ctas_of(run)
        assert ops.launch_count() == n0 + 1, (name, cap)
        print('%s: %d items, cap %d: %d CTAs' % (name, items, cap, got))
        assert got == min(bounds), (name, items, cap, got, min(bounds))
  finally:
    for _, run, _, _ in sites:         # each kernel's copy of the phase-timer pointer is cleared at its next launch
      run()
    torch.cuda.synchronize()


def test_cap_refuses_a_negative_count():
  with pytest.raises(RuntimeError, match='status -1'):
    _set_cap(-1)
  assert _probe_grid() == _sms()


# ------------------------------------------------------------------------------------------
# dense layer: plain, grouped, split-K
# ------------------------------------------------------------------------------------------
def _dense_cases():
  cases = []
  for i, (M, N, K) in enumerate((m, n, k) for m in (129, 1000) for n in (1, 100, 130, 257) for k in (4, 36, 100, 1920)):
    cases.append(pytest.param(M, N, K, i % 2 == 0, i % 3 != 2, id='M%d-N%d-K%d' % (M, N, K)))
  return cases


@pytest.mark.parametrize('M,N,K,relu,has_bias', _dense_cases())
def test_dense_layer(M, N, K, relu, has_bias):
  """Several n-tiles: a CTA's consecutive items switch W rows as well as A rows."""
  x, w, b = _operands(M, N, K, has_bias, M + N * 7 + K * 31)
  xd, w_hi, w_lo, bd = _to_dev(x, w, b)

  def run():
    out = _nan(M, N)
    _plain_c(xd, w_hi, w_lo, bd, relu, out)
    return (out,)
  items = -(-M // BM) * -(-N // BM)
  got, = _sweep(run, items, 'dense M=%d N=%d K=%d' % (M, N, K))
  dense_check('dense M=%d N=%d K=%d at one CTA' % (M, N, K), got, dense_ref(x, w, b, relu, torch.float64),
              dense_ref(x, w, b, relu, torch.float32), K)


@pytest.mark.parametrize('M', [129, 1000])
def test_grouped_layer(M):
  groups, N, K = 7, 200, 36
  x, w, b = _grouped_operands(M, groups, N, K, True, M)
  xd, w_hi, w_lo, bd = _to_dev(x, w, b)

  def run():
    out = _nan(M, groups * N)
    _grouped_c(xd, w_hi, w_lo, bd, groups, True, out)
    return (out,)
  got, = _sweep(run, -(-M // BM) * 2 * groups, 'grouped M=%d' % M)
  for g in range(groups):
    cols, rows = slice(g * K, (g + 1) * K), slice(g * N, (g + 1) * N)
    dense_check('grouped M=%d group %d at one CTA' % (M, g), got[:, rows],
                dense_ref(x[:, cols], w[rows], b[rows], True, torch.float64),
                dense_ref(x[:, cols], w[rows], b[rows], True, torch.float32), K)


# M, N, splits at K = 4096 (128 k-blocks: ranges 64 x 2; 43, 43, 42; 4 x 26, 24; 16 x 8)
SPLITK = [(129, 129, 2), (129, 129, 3), (1, 520, 5), (129, 257, 16)]


@pytest.mark.parametrize('M,N,splits', SPLITK)
def test_splitk_layer(M, N, splits):
  """A cap below `splits` makes one CTA run several splits of a tile and reduce the tile itself.
  Every capped launch runs twice: the per-tile counters must be back at zero in between."""
  K = 4096
  x, w, b = _operands(M, N, K, True, M + N + splits)
  xd, w_hi, w_lo, bd = _to_dev(x, w, b)
  tiles = -(-M // BM) * -(-N // BM)
  ws = _nan(tiles * splits * BM * BM)
  counters = torch.zeros(tiles, dtype=torch.int32, device=dev())

  def run():
    outs = [_nan(M, N), _nan(M, N)]
    for o in outs:
      _splitk_c(xd, w_hi, w_lo, bd, False, o, splits, ws, counters)
    torch.cuda.synchronize()
    _assert_same(outs[1], outs[0], 'split-K second launch')
    assert int(counters.abs().sum()) == 0, counters
    return outs[:1]
  got, = _sweep(run, tiles * splits, 'split-K M=%d N=%d splits=%d' % (M, N, splits))
  dense_check('split-K M=%d N=%d splits=%d at one CTA' % (M, N, splits), got,
              dense_ref(x, w, b, False, torch.float64), dense_ref(x, w, b, False, torch.float32), K)


# ------------------------------------------------------------------------------------------
# GRU updates
# ------------------------------------------------------------------------------------------
GRU_TILES = {32: 25, 64: 13, 96: 9, 128: 8}      # row tiles: 25, 26, 27, 32 items


def _gru_case_id(c):
  return 'N%d-D%d-E%d' % c


GGNN_SWEEP = [(n, d, e) for n in (1, 2, 7, 26, 64, 128) for d in (32, 64, 128) for e in (1, 7)]


@pytest.mark.parametrize('N,D,E1', GGNN_SWEEP, ids=[_gru_case_id(c) for c in GGNN_SWEEP])
def test_ggnn_update(N, D, E1):
  B = _graphs_for_tiles(N, GRU_TILES[D])
  gen = torch.Generator().manual_seed(N * 1000 + D * 10 + E1)
  args = ggnn_inputs(gen, B, N, D, E1, dev())
  M, h, L, w_ih, w_hh, b_ih, b_hh = args
  prep = ops.graph_prepare(L, torch.zeros((B, N, 4), device=dev()), binarize=True)
  W, b = gru_gate_matrix(w_ih, w_hh, b_ih, b_hh)
  w_hi, w_lo = ops.split_tf32(W)
  cpu = [t.cpu() for t in args]
  for avg in (False, True):
    def run():
      out = _nan(B * N, D)
      ops.ggnn_update(M, h, prep, w_hi, w_lo, b, avg, out=out)
      return (out,)
    got, = _sweep(run, -(-B * N // BM) * D // 32, 'GGNN B=%d N=%d D=%d E1=%d avg=%d' % (B, N, D, E1, avg))
    r64 = ggnn_reference(*cpu, avg, torch.float64)
    r32 = ggnn_reference(*cpu, avg, torch.float32)
    scale = max(1.0, float(r64.abs().max()))
    e_ours = float((got.cpu().double() - r64).abs().max())
    e_orc = float((r32.double() - r64).abs().max())
    assert e_ours <= max(8 * e_orc, GGNN_FLOOR * scale), (N, D, E1, avg, e_ours, e_orc)


MPNN_SWEEP = [(n, d, e) for n in (1, 7, 26, 100, 255) for d in (32, 64, 128) for e in (1, 7, 16)]


@pytest.mark.parametrize('N,D,E1', MPNN_SWEEP, ids=[_gru_case_id(c) for c in MPNN_SWEEP])
def test_mpnn_update(N, D, E1):
  B = _graphs_for_tiles(N, GRU_TILES[D])
  gen = torch.Generator().manual_seed(N * 1000 + D * 10 + E1)
  PQ, h, L, Fm, w_hh, b_ih, b_hh = args = mpnn_inputs(gen, B, N, D, E1)
  W, b = gru_gate_matrix(F.pad(Fm, (0, E1 * MPNN_H + 32 - Fm.shape[1])), w_hh, b_ih, b_hh)
  w_hi, w_lo = ops.split_tf32(W)
  prep = mpnn_prep(L)
  for avg in (False, True):
    def run():
      out = _nan(B * N, D)
      ops.mpnn_update(PQ, h, prep, w_hi, w_lo, b, avg, out=out)
      return (out,)
    got, = _sweep(run, -(-B * N // BM) * D // 32, 'MPNN B=%d N=%d D=%d E1=%d avg=%d' % (B, N, D, E1, avg))
    r64, gates = mpnn_reference(*args, avg, torch.float64)
    r32, _ = mpnn_reference(*args, avg, torch.float32)
    mpnn_check(got, r64, r32, (N, D, E1, avg), scale=gates)


@pytest.mark.parametrize('H', [32, 96, 128])
@pytest.mark.parametrize('mode', ['shared', 'cluster-only', 'cut-only'])
def test_gpnn_partition_update(mode, H):
  """A CTA's consecutive items change part as well as row and column tile; a skipped part writes
  nothing."""
  gen = torch.Generator().manual_seed(H + len(mode))
  N = 26
  active = {'shared': (0, 1), 'cluster-only': (0,), 'cut-only': (1,)}[mode]
  B = _graphs_for_tiles(N, GRU_TILES[H])
  P = gpnn_operators(gen, B, N).to(dev())
  prep = ops.graph_prepare(P, torch.zeros((B, N, 4), device=dev()))
  wts = gpnn_weights(gen, H)
  gates = gpnn_gates(*wts)
  cpu_w = [t.cpu() for t in wts]
  M = torch.randn(B * N, H, generator=gen).to(dev())
  h = (0.5 * torch.randn(B * N, H, generator=gen)).to(dev())
  for avg in (False, True):
    def run():
      X = _nan(B * N, 3 * H)
      parts = [(M, h, X[:, (p + 1) * H:(p + 2) * H]) if p in active else None for p in (0, 1)]
      ops.gpnn_partition_update(parts, prep, *gates, avg, h_copy=X[:, :H])
      return (X,)
    items = -(-B * N // BM) * len(active) * H // 32
    X, = _sweep(run, items, 'GPNN %s B=%d H=%d avg=%d' % (mode, B, H, avg))
    assert torch.equal(X[:, :H], h)
    for p in (0, 1):
      blk = X[:, (p + 1) * H:(p + 2) * H]
      if p in active:
        args = (M.cpu(), h.cpu(), P[..., p].cpu(), *cpu_w, avg)
        gpnn_check(blk, partition_reference(*args, torch.float64), partition_reference(*args, torch.float32),
                   (mode, H, avg, p))
      else:
        assert bool(torch.isnan(blk).all())


# ------------------------------------------------------------------------------------------
# LSTM step
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', STEP_CASES, ids=['B%d-N%d-D%d-E%d-K%d' % c for c in STEP_CASES])
def test_lstm_steps(case):
  """Every step t = 0 .. K-1 under each cap; out and the in-place c after each step are compared with
  the full grid's, and at one CTA each step against torch's LSTMCell in fp64 from the kernel's own
  previous state."""
  _, N, D, E1, K = case
  B = _graphs_for_tiles(N * E1, GRU_TILES[D])
  rng = np.random.RandomState(sum(case))
  nn_idx, ne = lstm_samples(rng, B, N, K, E1)
  d = dev()
  state = torch.from_numpy((rng.randn(B * N, D) * 3 / np.sqrt(D)).astype(np.float32)).to(d)
  g = torch.Generator().manual_seed(sum(case))
  cell = torch.nn.LSTMCell(D, D)
  with torch.no_grad():
    for p in cell.parameters():
      p.copy_(torch.rand(p.shape, generator=g) * 0.6 - 0.3)
  cell = cell.to(d)
  W, b = lstm_gate_matrix(cell.weight_ih.detach(), cell.weight_hh.detach(), cell.bias_ih.detach(),
                          cell.bias_hh.detach())
  w_hi, w_lo = ops.split_tf32(W)
  idx = torch.from_numpy(nn_idx).to(d).to(torch.int32)
  nev = torch.from_numpy(ne.reshape(-1)).to(d)
  R = B * N * E1

  def run():
    c, h, outs, cs = _nan(R, D), None, [], []
    for t in range(K):
      out = _nan(R, D)
      ops.sage_lstm_step(state, idx, nev, h, c, w_hi, w_lo, b, t, out)
      outs.append(out)
      cs.append(c.clone())
      h = out
    return outs + cs
  got = _sweep(run, -(-R // BM) * D // 32, 'LSTM B=%d N=%d D=%d E1=%d K=%d' % (B, N, D, E1, K))
  outs, cs = got[:K], got[K:]
  live = nev.view(B * N, 1).expand(B * N, E1).reshape(R) != 0
  gid = torch.from_numpy(nn_idx).to(d)
  ok = (gid >= 0) & (gid < N)
  gid = torch.where(ok, gid + N * torch.arange(B, device=d).view(B, 1, 1, 1), torch.zeros_like(gid))
  h_prev = c_prev = torch.zeros((R, D), device=d, dtype=torch.float64)
  for t in range(K):
    x = state[gid[:, :, t, :].reshape(-1)] * ok[:, :, t, :].reshape(-1, 1)
    want = {}
    for dt in (torch.float64, torch.float32):
      ref = torch.nn.LSTMCell(D, D).to(d, dt)
      ref.load_state_dict(cell.state_dict())
      with torch.no_grad():
        want[dt] = ref(x.to(dt), (h_prev.to(dt), c_prev.to(dt)))
    for got_t, k, what in ((outs[t], 0, 'h'), (cs[t], 1, 'c')):
      r64, r32 = want[torch.float64][k][live], want[torch.float32][k][live]
      gl = got_t[live].double()
      scale = float(r64.abs().max())
      err, e32 = float((gl - r64).abs().max()), float((r32.double() - r64).abs().max())
      assert err <= max(4 * e32, STEP_FLOOR * scale), (case, t, what, err, e32, scale)
    if t == K - 1:
      assert torch.equal(outs[t][~live], torch.zeros_like(outs[t][~live]))
    h_prev = torch.zeros((R, D), device=d, dtype=torch.float64).index_put_((live,), outs[t][live].double())
    c_prev = torch.zeros((R, D), device=d, dtype=torch.float64).index_put_((live,), cs[t][live].double())


# ------------------------------------------------------------------------------------------
# filter-MLP chain
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('S,Hd,nl,R', _mlp_cases())
def test_filter_mlp_chain(S, Hd, nl, R):
  """All rows and a row list, under the global cap and under the chain's own ctas argument.  Items
  that take their operand from the accumulators follow one another inside a CTA.  R grows by whole
  tiles until there are enough items for the largest cap (R mod 128 stays)."""
  tiles = -(-R // BM)
  R += (max(tiles, -(-3 * max(CAPS) // nl)) - tiles) * BM
  g = torch.Generator().manual_seed(S * 1000 + Hd + nl + R)
  layers = _mlp_layers(g, nl, S, Hd)
  table = (torch.rand(R, S, generator=g) * 2 - 1).to(dev())
  w_hi, w_lo, bias_all = sc.WeightCache().split_mlp_chain('chain', layers)
  ref = mlp_ref(table, layers)
  n = max(1, (3 * R) // 5)
  perm = torch.randperm(R, generator=g)[:n]
  rowmap = perm.int().to(dev())
  nrows = torch.tensor([n], dtype=torch.int32, device=dev())
  listed = torch.zeros(R, dtype=torch.bool, device=dev())
  listed[perm.to(dev())] = True
  items = -(-R // BM) * nl
  for rows, what in (((None, None), 'all rows'), ((rowmap, nrows), '%d listed rows' % n)):
    run = lambda ctas=0: (ops.ritz_filter_mlp(table, w_hi, w_lo, bias_all, nl, *rows, ctas=ctas),)
    tag = 'chain S=%d Hd=%d L=%d R=%d %s' % (S, Hd, nl, R, what)
    out, = _sweep(run, items, tag)
    with _nan_outputs():
      full, = run()
    for ctas in _caps_for(items):
      with _nan_outputs():
        got, = run(ctas)
      _assert_same(got, full, '%s ctas=%d' % (tag, ctas))
    if rows[0] is None:
      _assert_mlp(out, ref, tag)
    else:
      assert bool(torch.isnan(out[:, ~listed]).all()), tag
      _assert_mlp(out[:, listed], ref[:, listed], tag)


# ------------------------------------------------------------------------------------------
# convolution stack
# ------------------------------------------------------------------------------------------
def _mixed_batch(B, N, K, E1, seed):
  """Graphs that make a CTA's consecutive tiles differ: graphs of N nodes with k_eff = K (N = 128:
  one graph fills a tile), graphs of N / 4 nodes (four fill a tile), small graphs, graphs with
  k_eff = 0 and graphs without nodes."""
  rng = np.random.RandomState(seed)
  sizes, keffs = [], []
  for kind in rng.randint(0, 5, size=B):
    n = [N, max(1, N // 4), int(rng.randint(1, 9)), int(rng.randint(2, N + 1)), 0][kind]
    k = [min(K, n), min(K, n), int(rng.randint(0, min(K, n) + 1)), 0, 0][kind]
    sizes.append(n)
    keffs.append(k)
  sizes[0], keffs[0] = N, min(K, N)
  L, V = stack_batch(B, N, K, E1, sizes, keffs, seed)
  return L.to(dev()), V.to(dev()), np.array(sizes)


STACK_CASES = {
    # dins, H, S, K, E1, N, B, write_pad, readout
    'S4-Din64-H64-N128': ([64, 64], 64, 4, 32, 3, 128, 60, True, True),
    'S4-Din128-H64-N128-nopad': ([128, 64], 64, 4, 32, 3, 128, 60, False, True),
    'S0-Din64-H128-N32': ([64, 128], 128, 0, 32, 3, 32, 150, True, False),
    'S5-E7-Din32-H32-odd-kblocks-nopad': ([32, 32], 32, 5, 20, 7, 64, 100, False, False),
    'S8-QM8-3layers': ([64, 128, 128], 128, 8, 20, 7, 26, 200, True, True),
}


@pytest.mark.parametrize('case', sorted(STACK_CASES))
def test_stack(case):
  """Kept drains and step 0 (S > 0) and the plain S = 0 path across tiles of different shapes;
  with write_pad off the padded rows keep the NaN."""
  dins, H, S, K, E1, N, B, write_pad, readout = STACK_CASES[case]
  L, V, sizes = _mixed_batch(B, N, K, E1, len(case))
  prep = ops.graph_prepare(L, V)
  T = _stack_tiles(prep, B)
  X = torch.randn(B, N, dins[0], generator=torch.Generator().manual_seed(B)).to(dev())
  model = stack_model(dins, H, S if S else 1, K, E1, 16, B, seed=len(case))
  Wg, bg, coeffs, ro, _ = model
  if S == 0:                                   # the same layers without long scales
    Wg = [w[:, din:].contiguous() for w, din in zip(Wg, dins)]
    w_hi, w_lo, ball = sc.WeightCache().split_conv_stack('s0', Wg, bg, E1 * max(dins))
  else:
    w_hi, w_lo, ball = model[4]

  def run():
    return [t for t in ops.spectral_stack_forward(prep, V, w_hi, w_lo, ball, dins, H, S,
                                                  coeff=coeffs if S else None,
                                                  coeff_stride=coeffs.stride(0) if S else 0, X=X, want_state=True,
                                                  write_pad=write_pad, readout=ro if readout else None)
            if t is not None]
  got = _sweep(run, T, 'stack %s (%d tiles)' % (case, T))
  c64 = coeffs.double() if S else None
  st64, sc64 = stack_ref(X.double(), L.double(), V.double(), c64, [w.double() for w in Wg],
                         [b.double() for b in bg], [t.double() for t in ro])
  torch.backends.cuda.matmul.allow_tf32 = False
  st32, sc32 = stack_ref(X, L, V, coeffs if S else None, Wg, bg, ro)
  floor = STACK_FLOOR_PER_LAYER * len(dins)
  real = torch.arange(N, device=dev())[None, :] < torch.as_tensor(sizes, device=dev())[:, None]
  if write_pad:
    _check(got[0], st64, st32, floor, case + ' state')
  else:
    assert bool(torch.isnan(got[0][~real]).all()), case
    _check(got[0][real], st64[real], st32[real], floor, case + ' state (real rows)')
  if readout:
    _check(got[1], sc64, sc32, floor, case + ' score')


@pytest.mark.parametrize('S,write_pad', [(5, True), (0, True), (9, False)])
def test_conv_layer(S, write_pad):
  """spectral_conv_fused: one layer through the stack kernel."""
  B, N, K, E1, Din, H = 120, 40, 20, 7, 64, 100
  L, V, sizes = _mixed_batch(B, N, K, E1, S + 3)
  prep = ops.graph_prepare(L, V)
  T = _stack_tiles(prep, B)
  g = torch.Generator().manual_seed(S)
  X = torch.randn(B, N, Din, generator=g).to(dev())
  coeff = torch.randn(B, K, S, generator=g).to(dev()) if S else None
  W = (torch.randn(H, (S + E1) * Din, generator=g) / np.sqrt((S + E1) * Din)).to(dev())
  bias = torch.randn(H, generator=g).to(dev())
  w_hi, w_lo = ops.split_tf32(W)
  out, = _sweep(lambda: (ops.spectral_conv_fused(X, V, coeff, prep, w_hi, w_lo, bias, True, write_pad),), T,
                'conv layer S=%d write_pad=%d (%d tiles)' % (S, write_pad, T))
  ref = conv_ref(X.double(), L.double(), V.double(), coeff.double() if S else None, W.double(), bias.double())
  torch.backends.cuda.matmul.allow_tf32 = False
  ref32 = conv_ref(X, L, V, coeff, W, bias)
  if not write_pad:
    real = torch.arange(N, device=dev())[None, :] < torch.as_tensor(sizes, device=dev())[:, None]
    assert bool(torch.isnan(out[~real]).all())
    out, ref, ref32 = out[real], ref[real], ref32[real]
  _check(out, ref, ref32, 8e-6, 'conv layer S=%d' % S)


@pytest.mark.parametrize('case', SAGE_CASES, ids=['N%d-D%d-H%d-L%d-E%d-%s-%s' % (c[:6] + ('mask' if c[6] else 'nomask',))
                                                  for c in SAGE_CASES])
def test_sage_stack(case):
  N, Din0, H, layers, E1, agg, use_mask = case
  rng = np.random.RandomState(sum(case[:5]))
  B, K, P = _graphs_for_tiles(N, 24), 8, 5
  sizes, nn_idx, ne = sage_samples(rng, B, N, K, E1)
  d = dev()
  ids = torch.from_numpy(rng.randint(0, 70, size=(B, N))).to(d)
  emb = torch.from_numpy(rng.randn(70, Din0).astype(np.float32)).to(d)
  dins = [Din0] + [H] * (layers - 1)
  Ws = [torch.from_numpy(rng.uniform(-1, 1, size=(H, E1 * dd)).astype(np.float32) * np.sqrt(6.0 / (H + E1 * dd))).to(d)
        for dd in dins]
  bs = [torch.from_numpy(rng.uniform(-0.1, 0.1, size=H).astype(np.float32)).to(d) for _ in dins]
  g = torch.Generator().manual_seed(N)
  head, att = torch.nn.Linear(H, P), torch.nn.Linear(H, 1)
  with torch.no_grad():
    for p in list(head.parameters()) + list(att.parameters()):
      p.copy_(torch.rand(p.shape, generator=g) - 0.5)
  head, att = head.to(d), att.to(d)
  mask = torch.from_numpy((np.arange(N)[None, :] < sizes[:, None]).astype(np.uint8)).to(d) if use_mask else None
  M = ops.sage_operators(torch.from_numpy(nn_idx).to(d), torch.from_numpy(ne).to(d))
  V = torch.zeros((B, N, 4), device=d)
  prep = ops.graph_prepare(M, V)
  T = _stack_tiles(prep, B)
  kw = E1 * max(dins)
  w_hi, w_lo = ops.split_tf32(torch.cat([F.pad(W, (0, kw - W.shape[1])) for W in Ws]).contiguous())
  readout = (head.weight.detach(), head.bias.detach(), att.weight.detach().reshape(-1), att.bias.detach())
  run = lambda: list(ops.spectral_stack_forward(prep, V, w_hi, w_lo, torch.cat(bs), dins, H, 0, node_ids=ids, emb=emb,
                                                want_state=True, write_pad=True, readout=readout, mask=mask, sage=agg))
  state, score = _sweep(run, T, 'GraphSAGE %s B=%d (%d tiles)' % (case, B, T))
  with torch.no_grad():
    s64, c64 = restate(M, ids, emb, Ws, bs, head, att, mask, agg, torch.float64)
    s32, c32 = restate(M, ids, emb, Ws, bs, head, att, mask, agg, torch.float32)
  for got, ref, r32, what in ((state, s64, s32, 'state'), (score, c64, c32, 'score')):
    scale = float(ref.abs().max())
    err = float((got.double() - ref).abs().max())
    e32 = float((r32.double() - ref).abs().max())
    assert err <= max(4 * e32, STACK_FLOOR_PER_LAYER * layers * scale), (case, what, err, e32, scale)


# ------------------------------------------------------------------------------------------
# models at their benchmark batches
# ------------------------------------------------------------------------------------------
def _lanczosnet():
  cfg = configs.qm8_lanczos_net()
  bt = data.collate(data.synthetic_qm8_samples(1024, seed=11), cfg.model.num_eig_vec)
  args = [torch.from_numpy(bt[k]).to(dev()) for k in ('node_feat', 'L', 'D', 'V')]
  mask = torch.from_numpy(bt['node_mask']).to(dev())
  return LanczosNet, cfg, lambda mod: mod(*args, mask=mask)


def _ggnn():
  cfg = configs.qm8_ggnn()
  bt = data.synthetic_qm8_batch(1024, seed=5)
  nf, L, mask = [torch.from_numpy(bt[k]).to(dev()) for k in ('node_feat', 'L', 'node_mask')]
  return GGNN, cfg, lambda mod: mod(nf, L, mask=mask)


def _graphsage_lstm():
  cfg = configs.qm8_graphsage(agg_func='LSTM')
  bt = data.sage_collate(data.synthetic_qm8_samples(256, seed=5), 40, np.random.RandomState(0))
  args = [torch.from_numpy(np.ascontiguousarray(bt[k])).to(dev()) for k in ('node_feat', 'nn_idx', 'nonempty_mask')]
  mask = torch.from_numpy(bt['node_mask']).to(dev())
  return LSTMGraphSAGE, cfg, lambda mod: mod(*args, mask=mask)


@pytest.mark.parametrize('model', ['LanczosNet', 'GGNN', 'GraphSAGE-LSTM'])
def test_model_scores_do_not_depend_on_the_grid(model):
  """A fresh module per cap: the forward captures CUDA graphs, whose launch configuration is fixed
  at capture."""
  cls, cfg, forward = {'LanczosNet': _lanczosnet, 'GGNN': _ggnn, 'GraphSAGE-LSTM': _graphsage_lstm}[model]()

  def score():
    mod = cls(cfg)
    mod.load_state_dict(deterministic_state_dict(mod, 77))
    mod = mod.to(dev()).eval()
    with torch.no_grad():
      out = forward(mod)
    torch.cuda.synchronize()
    return out
  full = score()
  assert bool(torch.isfinite(full).all())
  for cap in (1, 7, 64):
    with max_ctas(cap):
      got = score()
    _assert_same(got, full, '%s cap=%d' % (model, cap))
