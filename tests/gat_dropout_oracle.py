"""The GAT dropout mask rule of include/lanczosnet_b200.h over torch int64 tensors, and a masked form of
gat_train_oracle.gat_forward.  TEST INFRASTRUCTURE.

Element i of site (t, c, sigma) is kept iff word (i & 3) of Philox4x32-10 at counter
(i >> 2, (t << 16) | (c << 2) | sigma, ctr lo, ctr hi) and key (seed lo, seed hi) is >= floor(p * 2^32);
a kept value is scaled by s = fp32(1 / (1 - p)).  The arithmetic stays in int64 with every product below
2^63 (16-bit splits of the 32x32 multiplies), so the rule runs on the GPU as well as on the CPU.
"""
import torch
import torch.nn.functional as F

from gat_train_oracle import _linear

_MASK = 0xffffffff
_M0, _M1 = 0xD2511F53, 0xCD9E8D57
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
INPUT, ATT, WH = 0, 1, 2


def _mul32(m, c):
  """(hi, lo) words of the 64-bit product of the constant m and c < 2^32 (int64 tensors)."""
  a = m * (c & 0xffff)                                  # < 2^48
  b = m * (c >> 16)                                     # < 2^48
  t = a + ((b & 0xffff) << 16)                          # < 2^49
  return ((t >> 32) + (b >> 16)) & _MASK, t & _MASK


def philox4x32_10(c0, c1, c2, c3, k0, k1):
  """Philox4x32-10 (Random123's constants) of int64 tensors / ints holding uint32 values -> (x, y, z, w)."""
  c0, c1, c2, c3 = (torch.as_tensor(v, dtype=torch.int64) for v in (c0, c1, c2, c3))
  for r in range(10):
    if r:
      k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
    hi0, lo0 = _mul32(_M0, c0)
    hi1, lo1 = _mul32(_M1, c2)
    c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
  return c0, c1, c2, c3


def site(t, c, sigma):
  return (int(t) << 16) | (int(c) << 2) | int(sigma)


def words(key, site_word, idx):
  """The uint32 decision words (as int64) of elements ``idx`` (int64 tensor) of one site, or of several:
  ``site_word`` an int or an int64 tensor that broadcasts against ``idx``."""
  seed, ctr = (int(v) & 0xffffffffffffffff for v in torch.as_tensor(key).reshape(2).tolist())
  st = torch.as_tensor(site_word, dtype=torch.int64, device=idx.device).expand_as(idx)
  x, y, z, w = philox4x32_10(idx >> 2, st, ctr & _MASK, ctr >> 32, seed & _MASK, seed >> 32)
  j = idx & 3
  return torch.where(j == 0, x, torch.where(j == 1, y, torch.where(j == 2, z, w)))


def threshold(p):
  return int(float(p) * 4294967296.0)                   # floor of a non-negative fp64 value


def scale(p):
  return float(torch.tensor(1.0 / (1.0 - p) if p < 1.0 else float('inf'), dtype=torch.float32))


def mask(key, p, t, c, sigma, shape, device='cpu', dtype=torch.float64):
  """M * s over a tensor of ``shape`` (elements in row-major order are the site's element indices)."""
  n = 1
  for d in shape:
    n *= int(d)
  idx = torch.arange(n, device=device, dtype=torch.int64)
  keep = words(key, site(t, c, sigma), idx) >= threshold(p)
  s = scale(p)
  out = torch.zeros(n, device=device, dtype=dtype)
  if p < 1.0:
    out[keep] = s
  return out.reshape(tuple(shape))


def channel_masks(key, p, t, C, sigma, shape, device='cpu', dtype=torch.float64):
  """``mask`` of channels 0 .. C-1 stacked: [C, *shape]."""
  n = 1
  for d in shape:
    n *= int(d)
  idx = torch.arange(n, device=device, dtype=torch.int64)[None, :].expand(C, n)
  sites = torch.tensor([site(t, c, sigma) for c in range(C)], device=device, dtype=torch.int64)[:, None]
  keep = words(key, sites, idx) >= threshold(p)
  out = torch.zeros((C, n), device=device, dtype=dtype)
  if p < 1.0:
    out[keep] = scale(p)
  return out.reshape((C,) + tuple(shape))


def gat_forward_dropout(params, spec, node_feat, L, mask_, key, p, device='cpu', slopes=None):
  """gat_train_oracle.gat_forward with the reference's three dropout sites (model/gat.py:149-163) drawn by
  the rule above (input, attention, Wh), on ``params`` as given.  ``slopes``: per layer a bool [B,N,N,C], the
  leaky-ReLU branch (s1[i] + s2[k] > 0) to take instead of the one of this arithmetic."""
  dtype = params['embedding.weight'].dtype
  L = torch.as_tensor(L).to(device=device, dtype=dtype)
  node_feat = torch.as_tensor(node_feat).to(device).long()
  B, N = node_feat.shape
  E = spec['num_edgetype']
  nl = spec['num_layer']
  state = params['embedding.weight'][node_feat]
  for t in range(nl):
    h = []
    heads = spec['num_heads'][t]
    for jj in range(E + 1):
      for ii in range(heads):
        c = jj * heads + ii
        k = '%d.%d.%d' % (t, jj, ii)
        x = state * mask(key, p, t, c, INPUT, state.shape, device, dtype)
        Wh = _linear(params, 'filter.' + k, x.reshape(B * N, -1)).reshape(B, N, -1)
        s1 = _linear(params, 'att_net_1.' + k, Wh)
        s2 = _linear(params, 'att_net_2.' + k, Wh)
        x = s1 + s2.transpose(1, 2)
        if slopes is None:
          x = F.leaky_relu(x, negative_slope=0.2)
        else:
          x = x * torch.where(slopes[t][..., c], 1.0, 0.2).to(dtype)
        att = F.softmax(x + L[:, :, :, jj], dim=1)
        att = att * mask(key, p, t, c, ATT, att.shape, device, dtype)
        Whd = Wh * mask(key, p, t, c, WH, Wh.shape, device, dtype)
        out = torch.bmm(att, Whd) + params['bias_%d_%d_%d' % (ii, E, t)].view(1, 1, -1)
        h.append(out if t == nl - 1 else F.elu(out))
    state = torch.mean(torch.stack(h, dim=0), dim=0) if t == nl - 1 else torch.cat(h, dim=2)
  flat = state.reshape(B * N, -1)
  y = _linear(params, 'output_func.0', flat)
  gate = torch.sigmoid(_linear(params, 'att_func.0', flat))
  y = (gate * y).reshape(B, N, -1)
  if mask_ is None:
    return torch.stack([y[b].mean(dim=0) for b in range(B)])
  m = torch.as_tensor(mask_).to(device=device, dtype=torch.bool)
  return torch.stack([y[b, m[b], :].mean(dim=0) for b in range(B)])
