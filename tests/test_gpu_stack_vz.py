"""The convolution stack's V Z term against fp64.  The edge step of a layer with long scales starts
from V Z: every consumer thread sums Q_g[n, k] Z[kbase_g + k, :] over the graph's k_eff Ritz rows of
the tile (Z of step 0, kept in the A ring).  The cases move the tile's Ritz-row count Ztot across the
32-row boundaries of the Z rows (1, 31, 33, 97, 128), take graphs with k_eff < K and k_eff = 0, both
widths and an input wider than the state, write_pad and the fused readout on and off, a batch with
more tiles than SMs (CTAs run several tiles), and two captured CUDA graphs replayed alternately on
one stream.  ``pytest -m gpu``."""
import numpy as np
import pytest
import torch

from test_gpu_conv_envelope import STACK_FLOOR_PER_LAYER, _check, dev, ops, stack_ref

pytestmark = pytest.mark.gpu


def _batch(B, N, K, E1, sizes, keffs, seed):
  """Sparse operators on the leading sizes[b] nodes and orthonormal Ritz vectors in the leading
  keffs[b] columns of V (k_eff = keffs[b]; zero columns elsewhere)."""
  rng = np.random.RandomState(seed)
  L = np.zeros((B, N, N, E1), np.float32)
  V = np.zeros((B, N, K), np.float32)
  for b in range(B):
    n, k = int(sizes[b]), int(keffs[b])
    if n == 0:
      continue
    L[b, :n, :n] = rng.randn(n, n, E1) * (rng.rand(n, n, E1) < min(1.0, 4.0 / n))
    L[b, 0, 0, 0] = 1.0                           # n_eff = n for every graph with nodes
    L[b, n - 1, n - 1, 0] = 1.0
    if k:
      V[b, :n, :k] = np.linalg.qr(rng.randn(n, n))[0][:, :k]
  return torch.from_numpy(L), torch.from_numpy(V)


def _model(dins, H, S, K, E1, P, B, seed):
  from lanczosnetwork_b200 import spectral_conv as sc
  g = torch.Generator().manual_seed(seed)
  d = dev()
  Ws = [torch.randn(H, (S + E1) * din, generator=g) / np.sqrt((S + E1) * din) for din in dins]
  bs = [torch.randn(H, generator=g) for _ in dins]
  coeffs = torch.randn(len(dins), B, K, S, generator=g).to(d)
  ro = [t.to(d) for t in (torch.randn(P, H, generator=g) / np.sqrt(H), torch.randn(P, generator=g),
                          torch.randn(H, generator=g) / np.sqrt(H), torch.randn(1, generator=g))]
  Wg, bg = [w.to(d) for w in Ws], [b.to(d) for b in bs]
  w_hi, w_lo, ball = sc.WeightCache().split_conv_stack('vz', Wg, bg, (S + E1) * max(dins))
  return Wg, bg, coeffs, ro, (w_hi, w_lo, ball)


def _run(L, V, X, dins, H, S, model, readout, write_pad, mask=None):
  Wg, bg, coeffs, ro, (w_hi, w_lo, ball) = model
  prep = ops().graph_prepare(L, V)
  return ops().spectral_stack_forward(prep, V, w_hi, w_lo, ball, dins, H, S, coeff=coeffs,
                                      coeff_stride=coeffs.stride(0), X=X, want_state=True,
                                      write_pad=write_pad, readout=ro if readout else None, mask=mask)


def _assert_close(L, V, X, dins, H, S, model, readout, write_pad, sizes, tag):
  Wg, bg, coeffs, ro, _ = model
  N = X.shape[1]
  st, score = _run(L, V, X, dins, H, S, model, readout, write_pad)
  torch.cuda.synchronize()
  st64, sc64 = stack_ref(X.double(), L.double(), V.double(), coeffs.double(), [w.double() for w in Wg],
                         [b.double() for b in bg], [t.double() for t in ro])
  torch.backends.cuda.matmul.allow_tf32 = False
  st32, sc32 = stack_ref(X, L, V, coeffs, Wg, bg, ro)
  floor = STACK_FLOOR_PER_LAYER * len(dins)
  if write_pad:
    _check(st, st64, st32, floor, tag + ' state')
  else:                                           # padded rows are not written: real rows only
    real = (torch.arange(N, device=X.device)[None, :] < torch.as_tensor(sizes, device=X.device)[:, None])
    _check(st[real], st64[real], st32[real], floor, tag + ' state (real rows)')
  if readout:
    _check(score, sc64, sc32, floor, tag + ' score')


# keffs of the graphs of one tile (N = 32: every graph's rows fit the tile with the Ritz rows)
ZTOT_CASES = {
    'Ztot1': [1],
    'Ztot31': [31],
    'Ztot33': [32, 1],
    'Ztot97': [32, 32, 32, 1],
    'Ztot128': [32, 32, 32, 32],
    'keff_lt_K_and_0': [20, 0, 7, 32, 0],
}


@pytest.mark.parametrize('case', sorted(ZTOT_CASES))
@pytest.mark.parametrize('H,dins', [(64, [64, 64]), (128, [64, 128]), (64, [128, 64])],
                         ids=['H64', 'H128', 'Din0gtH'])
def test_stack_vz_ritz_rows(case, H, dins):
  keffs = ZTOT_CASES[case]
  B, N, K, E1, S = len(keffs), 32, 32, 3, 4
  sizes = [max(k, 4) if i % 2 == 0 else 32 for i, k in enumerate(keffs)]
  sizes = [min(32, max(s, k)) for s, k in zip(sizes, keffs)]
  L, V = _batch(B, N, K, E1, sizes, keffs, seed=len(keffs) * 7 + H)
  d = dev()
  X = torch.randn(B, N, dins[0], generator=torch.Generator().manual_seed(H)).to(d)
  model = _model(dins, H, S, K, E1, 8, B, seed=H + len(dins))
  _assert_close(L.to(d), V.to(d), X, dins, H, S, model, True, True, sizes, 'vz %s H=%d' % (case, H))


@pytest.mark.parametrize('readout,write_pad', [(True, False), (False, True), (False, False)])
def test_stack_vz_write_pad_and_readout(readout, write_pad):
  B, N, K, E1, S, H, dins = 24, 26, 20, 7, 8, 128, [64, 128, 128]
  rng = np.random.RandomState(5)
  sizes = rng.randint(3, N + 1, size=B)
  keffs = [min(K, int(s)) - (b % 3) for b, s in enumerate(sizes)]
  L, V = _batch(B, N, K, E1, sizes, keffs, seed=11)
  d = dev()
  X = torch.randn(B, N, dins[0], generator=torch.Generator().manual_seed(3)).to(d)
  model = _model(dins, H, S, K, E1, 16, B, seed=21)
  _assert_close(L.to(d), V.to(d), X, dins, H, S, model, readout, write_pad, sizes,
                'vz readout=%d write_pad=%d' % (readout, write_pad))


def _qm8_like(B, seed):
  rng = np.random.RandomState(seed)
  N, K, E1 = 26, 20, 7
  sizes = rng.randint(9, N + 1, size=B)
  keffs = [min(K, int(s)) for s in sizes]
  return _batch(B, N, K, E1, sizes, keffs, seed), sizes


def test_stack_vz_more_tiles_than_sms():
  """Enough graphs for about two tiles per SM: CTAs run Z and V Z of several tiles."""
  d = dev()
  sms = torch.cuda.get_device_properties(d).multi_processor_count
  B = 20 * sms
  (L, V), sizes = _qm8_like(B, 7)
  K, E1, S, H, dins = 20, 7, 8, 128, [64, 128, 128]
  Lg, Vg = L.to(d), V.to(d)
  prep = ops().graph_prepare(Lg, Vg)
  T = int(prep[4][B + 2].item())                  # tiles the stack kernel runs
  assert T > sms, (T, sms)
  X = torch.randn(B, 26, dins[0], generator=torch.Generator().manual_seed(1)).to(d)
  model = _model(dins, H, S, K, E1, 16, B, seed=9)
  _assert_close(Lg, Vg, X, dins, H, S, model, True, True, sizes, 'vz B=%d (%d tiles)' % (B, T))


def test_stack_vz_two_graphs_alternate_on_one_stream():
  """Two captured CUDA graphs of the stack (different batches) replayed alternately on one stream
  reproduce their eager results bit for bit."""
  d = dev()
  K, E1, S, H, dins = 20, 7, 8, 128, [64, 128]
  model = _model(dins, H, S, K, E1, 16, 300, seed=4)
  runs = []
  for seed, B in ((1, 300), (2, 200)):
    (L, V), _ = _qm8_like(B, seed)
    X = torch.randn(B, 26, dins[0], generator=torch.Generator().manual_seed(seed)).to(d)
    runs.append((L.to(d), V.to(d), X))
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  graphs, outs, eager = [], [], []
  with torch.cuda.stream(s):
    for L, V, X in runs:
      st, score = _run(L, V, X, dins, H, S, model, True, True)
      eager.append((st.clone(), score.clone()))
    torch.cuda.synchronize()
    for L, V, X in runs:
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g, stream=s):
        outs.append(_run(L, V, X, dins, H, S, model, True, True))
      graphs.append(g)
    for _ in range(3):
      for g in graphs:
        g.replay()
  torch.cuda.synchronize()
  for (st, score), (st_e, score_e) in zip(outs, eager):
    assert torch.equal(st, st_e) and torch.equal(score, score_e)
