"""numpy statement of lnb_unsorted_segment_sum_exact (include/lanczosnet_b200.h), bit for bit.

data [B, d1, d2] float32, ids [B, d1] int64, output [B, S, d2] accumulated into; ids outside [0, S) are
skipped.  Per output element with terms x_i:
  * e_max = max ilogb|x_i| over the finite nonzero terms; flags for NaN, +Inf, -Inf;
  * H = bit length of d1, k = 61 - H - e_max, acc = sum of rint(x_i 2^k) (ties to even), an exact integer
    sum: x_i 2^k is exact in float64 and |acc| < 2^62;
  * s = NaN if a NaN or both infinities occurred, +-Inf if one sign of infinity did, 0 with no finite
    nonzero term, else float32(acc) * 2^-k: acc rounded once to 24 bits (ties to even, the device's
    __ll2float_rn), then scaled and rounded once more only where the result is subnormal or overflows
    (ldexpf);
  * out = out_in + s in float32.
Integer arithmetic throughout, so the result does not depend on the order of the terms.
"""
import numpy as np

_NONE = np.iinfo(np.int64).min


def _ilogb(x):
  """floor(log2 |x|) of finite nonzero float32 values, subnormals included."""
  return np.frexp(np.abs(x.astype(np.float64)))[1].astype(np.int64) - 1


def _round_to_24_bits(a):
  """int64 -> float64 holding a rounded to 24 significant bits, ties to even (a float32 value)."""
  m = np.abs(a)
  L = np.frexp(m.astype(np.float64))[1].astype(np.int64)          # bit length, or one more if it rounded up
  L = np.where((L > 0) & ((m >> np.maximum(L - 1, 0)) == 0), L - 1, L)
  sh = np.maximum(L - 24, 0)
  r = m >> sh
  rem = m - (r << sh)
  half = np.where(sh > 0, np.int64(1) << np.maximum(sh - 1, 0), 0)
  r = r + ((sh > 0) & ((rem > half) | ((rem == half) & (r % 2 == 1))))
  return np.sign(a) * np.ldexp(r.astype(np.float64), sh)


def segment_sum_exact(data, ids, num_segments, out=None):
  data = np.asarray(data, dtype=np.float32)
  ids = np.asarray(ids, dtype=np.int64)
  B, d1, d2 = data.shape
  S = int(num_segments)
  out = np.zeros((B, S, d2), np.float32) if out is None else np.array(out, dtype=np.float32, copy=True)
  if B * d1 * d2 == 0:
    return out
  H = int(d1).bit_length()
  b = np.repeat(np.arange(B, dtype=np.int64), d1)
  seg = ids.reshape(-1)
  ok = (seg >= 0) & (seg < S)
  rows = (b * S + seg)[ok]
  x = data.reshape(B * d1, d2)[ok]
  o = (rows[:, None] * d2 + np.arange(d2, dtype=np.int64)[None, :]).reshape(-1)
  x = x.reshape(-1)
  n = B * S * d2

  flags = np.zeros(n, np.int64)
  np.bitwise_or.at(flags, o[np.isnan(x)], 1)
  np.bitwise_or.at(flags, o[x == np.inf], 2)
  np.bitwise_or.at(flags, o[x == -np.inf], 4)
  live = np.isfinite(x) & (x != 0)
  e_max = np.full(n, _NONE, np.int64)
  np.maximum.at(e_max, o[live], _ilogb(x[live]))
  have = e_max != _NONE
  k = np.where(have, 61 - H - e_max, 0)

  acc = np.zeros(n, np.int64)
  q = np.rint(np.ldexp(x[live].astype(np.float64), k[o[live]])).astype(np.int64)
  np.add.at(acc, o[live], q)

  with np.errstate(over='ignore'):
    s = np.ldexp(_round_to_24_bits(acc), -k).astype(np.float32)
  s[~have] = 0
  s[(flags & 2) != 0] = np.inf
  s[(flags & 4) != 0] = -np.inf
  s[((flags & 1) != 0) | ((flags & 6) == 6)] = np.nan
  with np.errstate(invalid='ignore', over='ignore'):
    return (out.reshape(-1) + s).reshape(B, S, d2)


def error_bound(count, e_max, d1):
  """The bound on |s - exact sum| before the final rounding: count * 2^(e_max - 62 + H)."""
  return count * 2.0 ** (e_max - 62 + int(d1).bit_length())
