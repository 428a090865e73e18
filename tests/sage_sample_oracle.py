"""numpy restatement of GraphSAGE's device sampler (lnb_sage_sample_sparse; the rule is in the C header):
Philox4x32-10 and the per-row draws, from the collate's view of the records (the non-zero columns of the
padded L4 rows, as ``np.nonzero`` gives them to the reference's collate)."""
import numpy as np

_MASK = np.uint64(0xffffffff)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)


def philox4x32_10(ctr, key):
  """Philox4x32-10 of counters ctr [..., 4] and keys key [..., 2] (uint32 values, broadcast) -> [..., 4]
  uint32."""
  ctr = np.asarray(ctr, np.uint64) & _MASK
  key = np.asarray(key, np.uint64) & _MASK
  c0, c1, c2, c3 = (ctr[..., i] for i in range(4))
  k0, k1 = key[..., 0], key[..., 1]
  for r in range(10):
    if r:
      k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
    p0, p1 = _M0 * c0, _M1 * c2                      # < 2^64: exact in uint64
    c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK
  return np.stack(np.broadcast_arrays(c0, c1, c2, c3), axis=-1).astype(np.uint32)


def _split(v):
  v = int(v) & 0xffffffffffffffff
  return v & 0xffffffff, v >> 32


def draws(sample_key, rows, K):
  """x[r, i] for the row ids ``rows`` [R] and i < K: word i % 4 of Philox at key (seed lo, seed hi) and
  counter (i / 4, r, ctr lo, ctr hi).  Returns uint64 [R, K]."""
  seed, ctr = (int(v) for v in np.asarray(sample_key).reshape(2))
  k = np.array(_split(seed), np.uint64)
  clo, chi = _split(ctr)
  rows = np.asarray(rows, np.uint64)
  blocks = (K + 3) // 4
  c = np.zeros((rows.shape[0], blocks, 4), np.uint64)
  c[..., 0] = np.arange(blocks, dtype=np.uint64)[None, :]
  c[..., 1] = rows[:, None]
  c[..., 2], c[..., 3] = clo, chi
  return philox4x32_10(c, k).reshape(rows.shape[0], blocks * 4)[:, :K].astype(np.uint64)


def sample_rows(cands, x, K):
  """The samples of rows with candidate lists ``cands`` (ascending int arrays) and draws x [R, K] (uint64):
  a partial Fisher-Yates when L >= K, draws with replacement when 1 <= L < K, zeros when L = 0.
  Returns int32 [R, K]."""
  R = len(cands)
  out = np.zeros((R, K), np.int32)
  L = np.array([len(c) for c in cands], np.int64)
  width = max(int(L.max()) if R else 0, 1)
  table = np.zeros((R, width), np.int64)
  for r, c in enumerate(cands):
    table[r, :len(c)] = c
  ar = np.arange(R)
  rep = (L >= 1) & (L < K)
  if rep.any():
    j = ((x[rep] * L[rep, None].astype(np.uint64)) >> np.uint64(32)).astype(np.int64)
    out[rep] = np.take_along_axis(table[rep], j, axis=1)
  fy = L >= K
  if fy.any():
    t, xf, Lf, rr = table[fy].copy(), x[fy], L[fy], ar[:int(fy.sum())]
    for i in range(K):
      j = i + ((xf[:, i] * (Lf - i).astype(np.uint64)) >> np.uint64(32)).astype(np.int64)
      ci, cj = t[rr, i].copy(), t[rr, j].copy()
      t[rr, i], t[rr, j] = cj, ci
    out[fy] = t[:, :K]
  return out


def sample_batch(samples, K, sample_key, N=None):
  """The sampler on a list of ``data.prepare_graph`` records padded to N (default: the batch maximum).
  Returns (nn_idx [B,N,K,E1] int32, nonempty [B,N] float32)."""
  sizes = [s['L_simple_4'].shape[0] for s in samples]
  B, N = len(samples), int(N or max(sizes))
  E1 = samples[0]['L_multi'].shape[2] + 1
  cands, rows = [], []
  for b, s in enumerate(samples):
    for n in range(N):
      for e in range(E1):
        if n < sizes[b]:
          op = s['L_simple_4'] if e == 0 else s['L_multi'][:, :, e - 1]
          cands.append(np.nonzero(op[n, :])[0])
        else:
          cands.append(np.zeros(0, np.int64))
        rows.append((b * N + n) * E1 + e)
  x = draws(sample_key, rows, K)
  nn_idx = sample_rows(cands, x, K).reshape(B, N, E1, K).transpose(0, 1, 3, 2)
  L = np.array([len(c) for c in cands]).reshape(B, N, E1)
  nonempty = (L >= 1).any(axis=2).astype(np.float32)
  return np.ascontiguousarray(nn_idx), nonempty
