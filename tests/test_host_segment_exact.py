"""The exact segment sum's numpy statement (segment_exact_oracle) on the CPU: the same bits for any row
order, the NaN / Inf rules, and the error bound against sums in exact rational arithmetic."""
import math
from fractions import Fraction

import numpy as np
import pytest

import segment_exact_oracle as seo


def _bits(a):
  return np.asarray(a, np.float32).view(np.uint32)


def _same(a, b):
  """Equal bits, except that any NaN equals any NaN."""
  a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
  return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and \
      np.array_equal(_bits(np.where(np.isnan(a), 0, a)), _bits(np.where(np.isnan(b), 0, b)))


def _wide(rng, shape, lo=-40, hi=40):
  """float32 values with exponents spread over [lo, hi] and both signs."""
  m = rng.uniform(1, 2, shape) * rng.choice([-1, 1], shape)
  return np.ldexp(m, rng.randint(lo, hi + 1, shape)).astype(np.float32)


def _scalar(xs, d1):
  """One output element's s from its terms, in Python integers and Fractions (no numpy tricks)."""
  xs = [float(v) for v in xs]
  if any(math.isnan(v) for v in xs) or (math.inf in xs and -math.inf in xs):
    return math.nan
  if math.inf in xs or -math.inf in xs:
    return math.inf if math.inf in xs else -math.inf
  live = [v for v in xs if v != 0]
  if not live:
    return 0.0
  e_max = max(math.frexp(v)[1] - 1 for v in live)
  k = 61 - d1.bit_length() - e_max
  acc = sum(round(Fraction(v) * Fraction(2) ** k) for v in live)     # round(): ties to even
  assert abs(acc) < 2 ** 62
  m, sh = abs(acc), max(abs(acc).bit_length() - 24, 0)
  r, rem = m >> sh, m & ((1 << sh) - 1)
  if sh and (2 * rem > (1 << sh) or (2 * rem == (1 << sh) and r & 1)):
    r += 1
  with np.errstate(over='ignore'):
    return float(np.float32(math.copysign(math.ldexp(float(r), sh - k), acc)))


def _scalar_sum(data, ids, S, out=None):
  B, d1, d2 = data.shape
  res = np.zeros((B, S, d2), np.float32) if out is None else out.astype(np.float32).copy()
  for b in range(B):
    for s in range(S):
      for c in range(d2):
        terms = [data[b, r, c] for r in range(d1) if ids[b, r] == s]
        with np.errstate(invalid='ignore', over='ignore'):
          res[b, s, c] = res[b, s, c] + np.float32(_scalar(terms, d1))
  return res


def test_matches_a_scalar_statement_in_python_integers():
  rng = np.random.RandomState(0)
  for B, d1, d2, S in [(2, 7, 3, 4), (1, 33, 5, 6), (3, 5, 4, 2)]:
    data = _wide(rng, (B, d1, d2), -149, 127)
    data[rng.rand(B, d1, d2) < 0.15] = 0
    ids = rng.randint(-1, S + 1, (B, d1))
    out_in = _wide(rng, (B, S, d2), -20, 20)
    assert _same(seo.segment_sum_exact(data, ids, S, out_in), _scalar_sum(data, ids, S, out_in))


def test_any_row_order_gives_the_same_bits():
  rng = np.random.RandomState(1)
  B, d1, d2, S = 3, 200, 5, 7
  data = _wide(rng, (B, d1, d2), -149, 127)
  ids = rng.randint(-1, S, (B, d1))
  ref = seo.segment_sum_exact(data, ids, S)
  for _ in range(5):
    p = rng.permutation(d1)
    assert _same(seo.segment_sum_exact(data[:, p], ids[:, p], S), ref)


def test_nan_and_inf_rules():
  nan, inf = np.nan, np.inf
  cases = [
      ([1.0, nan, 2.0], nan), ([inf, -inf], nan), ([inf, 1.0, inf], inf), ([-inf, 5.0], -inf),
      ([nan, inf], nan), ([0.0, -0.0], 0.0), ([], 0.0), ([3.0, -3.0], 0.0), ([inf, 0.0], inf),
  ]
  d1 = max(len(t) for t, _ in cases)
  data = np.zeros((1, len(cases) * d1, 1), np.float32)
  ids = np.full((1, len(cases) * d1), -1, np.int64)
  for s, (terms, _) in enumerate(cases):
    data[0, s * d1:s * d1 + len(terms), 0] = terms
    ids[0, s * d1:s * d1 + len(terms)] = s
  out_in = np.full((1, len(cases), 1), -0.0, np.float32)
  got = seo.segment_sum_exact(data, ids, len(cases), out_in)[0, :, 0]
  for s, (_, want) in enumerate(cases):
    assert _same(got[s], np.float32(want + 0.0)), (s, got[s], want)
  # out_in + s: -0 + 0 is +0, and an infinite out_in meets an infinite s of the other sign as NaN
  assert _bits(got[5]) == 0 and _bits(got[6]) == 0
  out_in = np.array([[[-inf], [1.0]]], np.float32)
  got = seo.segment_sum_exact(np.array([[[inf], [0.0]]], np.float32), np.array([[0, 1]]), 2, out_in)
  assert np.isnan(got[0, 0, 0]) and got[0, 1, 0] == 1.0


@pytest.mark.parametrize('case', ['mixed_1e30_1e-30', 'tiny_beside_huge', 'subnormals', 'cancellation', 'many'])
def test_error_bound_against_exact_sums(case):
  rng = np.random.RandomState(sum(map(ord, case)))
  S = 4
  if case == 'mixed_1e30_1e-30':
    data = np.array([1e30, 1e-30, -1e30, 1e-30, 3e-30, 1e30, -1e-30, 2.5] * 8, np.float32)
    ids = np.array([0, 0, 0, 0, 1, 1, 1, 2] * 8)
  elif case == 'tiny_beside_huge':
    data = np.concatenate([_wide(rng, 60, 100, 120), _wide(rng, 60, -149, -120)]).astype(np.float32)
    ids = np.concatenate([rng.randint(0, 2, 60), rng.randint(2, 4, 60)])
  elif case == 'subnormals':
    data = _wide(rng, 90, -149, -126)
    ids = rng.randint(0, S, 90)
  elif case == 'cancellation':
    big = _wide(rng, 40, 20, 30)
    data = np.concatenate([big, -big, _wide(rng, 40, -10, 0)]).astype(np.float32)
    ids = np.tile(rng.randint(0, S, 40), 3)
  else:
    data = _wide(rng, 5000, -30, 30)
    ids = rng.randint(0, S, 5000)
  d1 = len(data)
  got = seo.segment_sum_exact(data.reshape(1, d1, 1), ids.reshape(1, d1), S)[0, :, 0]
  for s in range(S):
    terms = [float(v) for v, i in zip(data, ids) if i == s]
    live = [v for v in terms if v != 0]
    exact = sum(Fraction(v) for v in terms)
    if not live:
      assert got[s] == 0
      continue
    e_max = max(math.frexp(v)[1] - 1 for v in live)
    bound = Fraction(seo.error_bound(len(terms), e_max, d1))
    half_ulp = Fraction(float(np.spacing(np.abs(got[s])))) / 2
    err = abs(Fraction(float(got[s])) - exact)
    assert err <= bound + half_ulp, (case, s, float(err), float(bound), float(half_ulp))
    # below half an ulp of the largest term: never worse than one fp32 rounding of that size
    assert bound <= Fraction(float(np.spacing(np.float32(max(abs(v) for v in live))))) / 2


def test_integer_to_float_rounding_ties_to_even():
  a = np.array([0, 1, -1, 2 ** 24 + 1, 2 ** 24 + 3, 2 ** 25 + 2, 2 ** 25 + 6, -(2 ** 25 + 6), 2 ** 53 + 1,
                2 ** 62 - 1, 2 ** 61 + 2 ** 37, 2 ** 61 + 2 ** 37 + 1, 2 ** 61 + 3 * 2 ** 37], np.int64)
  got = seo._round_to_24_bits(a)
  assert list(got[:5]) == [0.0, 1.0, -1.0, 2.0 ** 24, 2.0 ** 24 + 4]
  for v, g in zip(a, got):
    v = int(v)
    m, sh = abs(v), max(abs(v).bit_length() - 24, 0)
    r, rem = m >> sh, m & ((1 << sh) - 1)
    if sh and (2 * rem > (1 << sh) or (2 * rem == (1 << sh) and r & 1)):
      r += 1
    assert g == math.copysign(math.ldexp(r, sh), v), (v, g)
