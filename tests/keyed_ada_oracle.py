"""Restatements for KeyedAdaLanczosNet's kernels: the start vector of lnb_ada_start_vector (Philox4x32-10 +
Box-Muller, the rule in the C header) in numpy, and the reverse sweep of lnb_tridiag_powers_backward in
fp64 numpy."""
import numpy as np

from sage_sample_oracle import philox4x32_10


def _split(v):
  v = int(v) & 0xffffffffffffffff
  return v & 0xffffffff, v >> 32


def start_vector(start_key, B, N):
  """q1 [B, N]: u1 = (fp32(x0) + 1) 2^-32 and u2 = fp32(x1) 2^-32 in fp32, then sqrt(-2 log u1) times
  cos (even n) or sin (odd n) of 2 pi u2, the transcendental functions in fp64 and rounded once to fp32
  (the kernel's logf / sincospif are within an ulp or two of that)."""
  seed, ctr = (int(v) for v in np.asarray(start_key).reshape(2))
  half = (N + 1) // 2
  c = np.zeros((B, half, 4), np.uint64)
  c[..., 0] = np.arange(half, dtype=np.uint64)[None, :]
  c[..., 1] = np.arange(B, dtype=np.uint64)[:, None]
  c[..., 2], c[..., 3] = _split(ctr)
  x = philox4x32_10(c, np.array(_split(seed), np.uint64))
  scale = np.float32(2.0 ** -32)
  u1 = (x[..., 0].astype(np.float32) + np.float32(1.0)) * scale
  u2 = x[..., 1].astype(np.float32) * scale
  r = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
  ang = 2.0 * np.pi * u2.astype(np.float64)
  q = np.stack([r * np.cos(ang), r * np.sin(ang)], axis=-1).reshape(B, 2 * half)[:, :N]
  return q.astype(np.float32)


def tri(T):
  """The three diagonals of T [..., K, K] (what lnb_tridiag_powers reads after the first power)."""
  K = T.shape[-1]
  band = np.abs(np.arange(K)[:, None] - np.arange(K)[None, :]) <= 1
  return T * band


def powers_forward(T, powers):
  """out [B, K, S, K]: P_1 = T, P_{p+1} = P_p tri(T)."""
  out, cur, s = [], T, 0
  for p in range(1, max(powers) + 1):
    if p == powers[s]:
      out.append(cur)
      s += 1
      if s == len(powers):
        break
    cur = cur @ tri(T)
  return np.stack(out, axis=2)


def powers_backward(T, gOut, powers):
  """The reverse sweep lnb_tridiag_powers_backward runs: H_pmax = G_pmax; for p = pmax-1 .. 1,
  gTri += tri(P_p^T H_{p+1}), H_p = G_p + H_{p+1} tri(T)^T; gT = H_1 + gTri."""
  pmax = max(powers)
  P = [T]
  for _ in range(pmax - 2):
    P.append(P[-1] @ tri(T))
  G = {p: gOut[:, :, s, :] for s, p in enumerate(powers)}
  H = G[pmax]
  gtri = np.zeros_like(T)
  for p in range(pmax - 1, 0, -1):
    gtri += tri(np.swapaxes(P[p - 1], -1, -2) @ H)
    H = G.get(p, 0) + H @ np.swapaxes(tri(T), -1, -2)
  return H + gtri


def lanczos_block_gs(A, mask, q1, K):
  """fp64 torch restatement of the training Lanczos layer (lnb_lanczos_tridiag_train, train._lanczos_train):
  A [B,N,N] (may require grad), mask [B,N] or None, q1 [B,N].  Two classical block Gram-Schmidt passes with
  c_j = (q_j . z) / (q_j . q_j + EPS); acceptance, idx and the masks as data.  Returns (T [B,K,K], Q [B,N,K],
  idx [B])."""
  import torch
  eps = 1.1920928955078125e-07
  B, N = A.shape[0], A.shape[1]
  iters = min(N, K)
  m = torch.ones(B, N, dtype=A.dtype) if mask is None else (mask != 0).to(A.dtype)
  q = q1.reshape(B, N).to(A.dtype) * m
  q = q / q.norm(dim=1, keepdim=True)
  basis, alphas, betas, oks = [q], [], [], []
  ok = torch.ones(B, dtype=A.dtype)
  bprev = torch.zeros(B, dtype=A.dtype)
  for i in range(iters):
    qi = basis[i]
    z = torch.einsum('bnm,bm->bn', A, qi)
    a = (qi * z).sum(1)
    z = z - a[:, None] * qi
    if i > 0:
      z = z - bprev[:, None] * basis[i - 1]
      Qb = torch.stack(basis[:i], dim=2)                           # [B,N,i]
      s = 1.0 / ((Qb * Qb).sum(1) + eps)                            # [B,i]
      for _ in range(2):
        c = torch.einsum('bni,bn->bi', Qb, z) * s
        z = z - torch.einsum('bni,bi->bn', Qb, c)
    b = z.norm(dim=1)
    ok = ok * (b.detach() >= 1.0e-4).to(A.dtype)
    alphas.append(a)
    betas.append(b)
    oks.append(ok)
    basis.append(z * ok[:, None] / (b[:, None] + eps))
    bprev = b
  valid = torch.stack(oks, 1)
  idx = torch.minimum(valid.sum(1).long(), m.sum(1).long())
  valid = valid * (torch.arange(iters)[None, :] < idx[:, None]).to(A.dtype)
  T = torch.diag_embed(torch.stack(alphas, 1) * valid)
  if iters > 1:
    be = torch.stack(betas[:-1], 1) * valid[:, :-1]
    T = T + torch.diag_embed(be, 1) + torch.diag_embed(be, -1)
  Q = torch.stack(basis[:iters], 2) * (valid[:, None, :] * (torch.arange(N)[None, :, None] < idx[:, None, None]).to(A.dtype))
  if iters < K:
    T = torch.nn.functional.pad(T, (0, K - iters, 0, K - iters))
    Q = torch.nn.functional.pad(Q, (0, K - iters))
  return T, Q, idx
