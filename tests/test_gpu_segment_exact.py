"""lnb_unsorted_segment_sum_exact against its numpy statement (segment_exact_oracle), bit for bit, and the
switch in ops.segment_sum_forward: the exact sum under torch.use_deterministic_algorithms(True), the atomic
sum without it."""
import numpy as np
import pytest
import torch

from lanczosnetwork_b200 import _lib, ops

import segment_exact_oracle as seo

pytestmark = pytest.mark.gpu


def dev():
  return torch.device('cuda:0')


def _same(got, want):
  """Equal bits, except that any NaN equals any NaN."""
  got = got.cpu().numpy() if torch.is_tensor(got) else np.asarray(got)
  want = np.asarray(want, np.float32)
  assert got.shape == want.shape
  nan = np.isnan(got)
  assert np.array_equal(nan, np.isnan(want))
  g, w = got.view(np.uint32)[~nan], want.view(np.uint32)[~nan]
  bad = np.flatnonzero(g != w)
  assert bad.size == 0, '%d of %d differ, first %r vs %r' % (
      bad.size, g.size, got[~nan][bad[:4]], want[~nan][bad[:4]])


def _wide(rng, shape, lo, hi):
  m = rng.uniform(1, 2, shape) * rng.choice([-1, 1], shape)
  return np.ldexp(m, rng.randint(lo, hi + 1, shape)).astype(np.float32)


def _exact(data, ids, S, out=None):
  return ops.segment_sum_forward(torch.from_numpy(data).to(dev()), torch.from_numpy(ids).to(dev()), S,
                                 output=None if out is None else torch.from_numpy(out).to(dev()), exact=True)


CASES = [  # B, d1, d2, S, exponent range
    (2, 37, 8, 5, (-20, 20)), (3, 50, 7, 9, (-20, 20)), (1, 300, 4, 3, (-149, 127)), (4, 64, 1, 16, (-60, 60)),
    (2, 129, 12, 70, (-126, -100)), (1, 1000, 5, 2, (100, 120)),
]


@pytest.mark.parametrize('B, d1, d2, S, exps', CASES)
def test_exact_sum_is_the_oracle(B, d1, d2, S, exps):
  rng = np.random.RandomState(B * 1000 + d1)
  data = _wide(rng, (B, d1, d2), *exps)
  data[rng.rand(B, d1, d2) < 0.1] = 0
  ids = rng.randint(-1, S + 2, (B, d1)).astype(np.int64)       # -1 and ids >= S are skipped
  _same(_exact(data, ids, S), seo.segment_sum_exact(data, ids, S))
  out_in = _wide(rng, (B, S, d2), -10, 10)
  _same(_exact(data, ids, S, out_in), seo.segment_sum_exact(data, ids, S, out_in))


def test_unaligned_data_and_output_take_the_scalar_path():
  rng = np.random.RandomState(5)
  B, d1, d2, S = 2, 40, 8, 6
  raw = torch.from_numpy(_wide(rng, (B * d1 * d2 + 1,), -30, 30)).to(dev())
  data = raw[1:].view(B, d1, d2)                               # 4-byte offset: not 16-byte aligned
  ids = torch.from_numpy(rng.randint(0, S, (B, d1))).to(dev())
  out_raw = torch.zeros(B * S * d2 + 1, device=dev())
  out = out_raw[1:].view(B, S, d2)
  ops.segment_sum_forward(data, ids, S, output=out, exact=True)
  _same(out, seo.segment_sum_exact(data.cpu().numpy(), ids.cpu().numpy(), S))


def test_nan_inf_zero_segments_and_extreme_exponents():
  nan, inf, tiny, huge = np.nan, np.inf, np.float32(2.0 ** -149), np.float32(3.0 * 2.0 ** 126)
  segs = [[1.0, nan], [inf, -inf], [inf, 2.0, inf], [-inf, 1.0], [0.0, -0.0], [], [tiny, tiny, -tiny],
          [huge, huge], [-huge, -huge], [huge, -huge, tiny], [1e30, 1e-30, -1e30], [tiny, 1.0]]
  d1 = sum(len(s) for s in segs)
  data = np.zeros((1, d1, 1), np.float32)
  ids = np.zeros((1, d1), np.int64)
  r = 0
  for i, s in enumerate(segs):
    data[0, r:r + len(s), 0] = s
    ids[0, r:r + len(s)] = i
    r += len(s)
  got = _exact(data, ids, len(segs))
  want = seo.segment_sum_exact(data, ids, len(segs))
  _same(got, want)
  w = want[0, :, 0]
  assert np.isnan(w[0]) and np.isnan(w[1]) and w[2] == inf and w[3] == -inf and w[4] == 0 and w[5] == 0
  assert w[6] == tiny and w[7] == inf and w[8] == -inf and w[11] == 1.0
  # terms below 2^(e_max - 61 + H) vanish beside a huge one: within the error bound, not summed
  assert w[9] == 0 and w[10] == 0
  # an out_in of -0 stays -0 only where nothing was added; with no finite nonzero term it becomes -0 + 0
  out_in = np.full((1, len(segs), 1), -0.0, np.float32)
  _same(_exact(data, ids, len(segs), out_in), seo.segment_sum_exact(data, ids, len(segs), out_in))


def test_empty_batches_launch_nothing():
  for shape in [(0, 5, 4), (3, 0, 4), (3, 5, 0)]:
    data = torch.zeros(shape, device=dev())
    ids = torch.zeros(shape[:2], dtype=torch.int64, device=dev())
    out = torch.full((shape[0], 3, shape[2]), -0.0, device=dev())
    n0 = ops.launch_count()
    ops.segment_sum_forward(data, ids, 3, output=out, exact=True)
    assert ops.launch_count() == n0
    assert torch.equal(out.view(torch.int32), torch.full_like(out, -0.0).view(torch.int32))


def test_neighbour_max_shape_at_b1024_and_any_row_order():
  """GraphSAGE Max's adjoint at B = 1024: B N E1 D = 3.4 M scalars into B N D segments (-1: an empty row)."""
  rng = np.random.RandomState(11)
  B, N, E1, D = 1024, 26, 2, 64
  d1, S = B * N * E1 * D, B * N * D
  g = (rng.randn(d1) * np.exp(rng.randn(d1) * 3)).astype(np.float32).reshape(1, d1, 1)
  seg = rng.randint(-1, S, (1, d1)).astype(np.int64)
  got = _exact(g, seg, S)
  _same(got, seo.segment_sum_exact(g, seg, S))
  p = torch.randperm(d1, generator=torch.Generator().manual_seed(3)).to(dev())
  gd, sd = torch.from_numpy(g).to(dev()), torch.from_numpy(seg).to(dev())
  again = ops.segment_sum_forward(gd[:, p], sd[:, p], S, exact=True)
  assert torch.equal(again, got)


@pytest.mark.parametrize('d2', [64, 5])
def test_row_permutation_gives_equal_output(d2):
  rng = np.random.RandomState(d2)
  B, d1, S = 3, 4096, 40
  data = torch.from_numpy(_wide(rng, (B, d1, d2), -30, 30)).to(dev())
  ids = torch.from_numpy(rng.randint(0, S, (B, d1))).to(dev())
  ref = ops.segment_sum_forward(data, ids, S, exact=True)
  for s in range(3):
    p = torch.randperm(d1, generator=torch.Generator().manual_seed(s)).to(dev())
    assert torch.equal(ops.segment_sum_forward(data[:, p], ids[:, p], S, exact=True), ref)


def _entries(fn):
  """The library entries fn launches through ops._launch."""
  names = []
  real = ops._launch

  def spy(name, on, *args):
    names.append(name)
    return real(name, on, *args)
  ops._launch = spy
  try:
    fn()
  finally:
    ops._launch = real
  return names


def test_the_flag_selects_the_entry():
  data = torch.randn(2, 30, 8, device=dev())
  ids = torch.randint(0, 5, (2, 30), device=dev())
  prev = torch.are_deterministic_algorithms_enabled()
  try:
    torch.use_deterministic_algorithms(False)
    assert _entries(lambda: ops.segment_sum_forward(data, ids, 5)) == ['lnb_unsorted_segment_sum_forward']
    n0 = _lib.launch_count()
    ops.segment_sum_forward(data, ids, 5)
    assert _lib.launch_count() - n0 == 1
    torch.use_deterministic_algorithms(True)
    assert _entries(lambda: ops.segment_sum_forward(data, ids, 5)) == ['lnb_unsorted_segment_sum_exact']
    assert _entries(lambda: ops.segment_sum_forward(data, ids, 5, exact=False)) == \
        ['lnb_unsorted_segment_sum_forward']
    exact = ops.segment_sum_forward(data, ids, 5)
  finally:
    torch.use_deterministic_algorithms(prev)
  _same(exact, seo.segment_sum_exact(data.cpu().numpy(), ids.cpu().numpy(), 5))
  atomic = ops.segment_sum_forward(data, ids, 5)
  torch.testing.assert_close(atomic, exact, rtol=1e-6, atol=1e-6)
