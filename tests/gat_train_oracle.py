"""Differentiable form of the GAT oracle, for gradient checks.  TEST INFRASTRUCTURE.

``oracle.gat_oracle.gat_forward`` casts (and so detaches) the parameters it is given.  ``gat_forward``
here is the same computation (model/gat.py:125-201 of the reference, dropout 0) on the caller's tensors as
they are, so autograd reaches them: pass fp64 leaves for the rounding budget, fp32 leaves for the
reference's own arithmetic.  tests/test_host_gat_train.py checks that both give the same scores.
"""
import numpy as np
import torch
import torch.nn.functional as F


def _linear(params, prefix, x):
  return F.linear(x, params[prefix + '.weight'], params.get(prefix + '.bias'))


def gat_forward(params, spec, node_feat, L, mask, device='cpu'):
  """GAT.forward without the loss, on ``params`` as given (no cast, no detach).  ``L`` (the attention
  bias, adj_to_bias) is converted to the parameters' dtype; mask=None averages over all N rows."""
  dtype = params['embedding.weight'].dtype
  L = torch.as_tensor(L).to(device=device, dtype=dtype)
  node_feat = torch.as_tensor(node_feat).to(device).long()
  B, N = node_feat.shape
  E = spec['num_edgetype']
  nl = spec['num_layer']
  state = params['embedding.weight'][node_feat]                                    # gat.py:142
  for t in range(nl):
    h = []
    for jj in range(E + 1):
      for ii in range(spec['num_heads'][t]):
        key = '%d.%d.%d' % (t, jj, ii)
        Wh = _linear(params, 'filter.' + key, state.reshape(B * N, -1)).reshape(B, N, -1)   # :150-152
        s1 = _linear(params, 'att_net_1.' + key, Wh)                              # :153
        s2 = _linear(params, 'att_net_2.' + key, Wh)                              # :154
        att = F.softmax(F.leaky_relu(s1 + s2.transpose(1, 2), negative_slope=0.2) + L[:, :, :, jj],
                        dim=1)                                                    # :155-160, dim=1
        # every channel reads bias_{ii}_{E}_{t}: the shared state_bias list (:62-70)
        out = torch.bmm(att, Wh) + params['bias_%d_%d_%d' % (ii, E, t)].view(1, 1, -1)
        h.append(out if t == nl - 1 else F.elu(out))                             # :165-175
    state = torch.mean(torch.stack(h, dim=0), dim=0) if t == nl - 1 else torch.cat(h, dim=2)
  flat = state.reshape(B * N, -1)                                                 # :183-186
  y = _linear(params, 'output_func.0', flat)
  gate = torch.sigmoid(_linear(params, 'att_func.0', flat))
  y = (gate * y).reshape(B, N, -1)
  if mask is None:
    return torch.stack([y[b].mean(dim=0) for b in range(B)])                      # :193-194
  m = torch.as_tensor(mask).to(device=device, dtype=torch.bool)
  return torch.stack([y[b, m[b], :].mean(dim=0) for b in range(B)])               # :189-191


def grad_digest(grads):
  """Per-parameter digest of the gradient goldens: sum, sum of squares, first 8 entries."""
  out = {}
  for name, g in grads.items():
    g = g.detach().double().cpu().numpy().reshape(-1)
    out[name] = np.concatenate([[g.sum(), (g * g).sum()], g[:8]])
  return out
