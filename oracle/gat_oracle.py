"""Functional torch-CPU oracle of the reference GAT forward.  TEST INFRASTRUCTURE -- see
oracle/__init__.py.

``params`` is a flat dict keyed like the reference ``state_dict`` (``filter.{t}.{jj}.{ii}.weight``,
``att_net_{1,2}.{t}.{jj}.{ii}.{weight,bias}``, ``bias_{ii}_{jj}_{t}``, ``embedding.weight``,
``att_func.0.*``, ``output_func.0.*``); ``dtype`` selects fp32 (parity with the reference) or fp64
(rounding budget).

Reference lines followed (relative to the reference checkout):
  dataset/qm8.py:196-219     adj_to_bias: the additive attention mask the GAT collate builds
  model/gat.py:62-70         state_bias: one inner list per layer, shared by every bond channel
  model/gat.py:125-201       GAT.forward
"""
import numpy as np
import torch
import torch.nn.functional as F


def adj_to_bias(L):
  """dataset/qm8.py:196-219 on a collated [B,N,N,E1] operator batch: per graph and channel
  mt = I @ (adj + I) in fp64, entries > 0 of the whole padded block set to 1, -1e9 * (1 - mt);
  returned as float32 like ``torch.from_numpy(...).float()``."""
  L = np.asarray(L, dtype=np.float64)
  B, N, _, E1 = L.shape
  out = np.empty(L.shape, np.float64)
  eye = np.eye(N)
  for b in range(B):
    for e in range(E1):
      mt = np.matmul(eye, L[b, :, :, e] + eye)
      mt[mt > 0.0] = 1.0
      out[b, :, :, e] = -1e9 * (1.0 - mt)
  return out.astype(np.float32)


def make_spec(num_layer, num_heads, num_edgetype):
  return {'num_layer': int(num_layer), 'num_heads': [int(h) for h in num_heads],
          'num_edgetype': int(num_edgetype)}


def _cast(params, dtype, device='cpu'):
  return {k: (v.detach().to(device).to(dtype) if v.is_floating_point() else v.detach().to(device))
          for k, v in params.items()}


def _linear(params, prefix, x):
  b = params.get(prefix + '.bias')
  return F.linear(x, params[prefix + '.weight'], b)


def gat_forward(params, spec, node_feat, L, mask, dtype=torch.float32, return_states=False,
                device='cpu'):
  """GAT.forward without the loss (model/gat.py:125-201).  L is the attention bias (adj_to_bias);
  mask=None averages over all N rows (:193-194).  ``device`` only places the computation (an fp64
  run of a benchmark-sized batch is slow on the CPU); results come back on that device."""
  params = _cast(params, dtype, device)
  L = torch.as_tensor(L).to(device=device, dtype=dtype)
  node_feat = torch.as_tensor(node_feat).to(device).long()
  B, N = node_feat.shape
  E = spec['num_edgetype']
  nl = spec['num_layer']
  state = params['embedding.weight'][node_feat]                                    # gat.py:142
  states = []
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
    states.append(state)
  flat = state.reshape(B * N, -1)                                                 # :183-186
  y = _linear(params, 'output_func.0', flat)
  gate = torch.sigmoid(_linear(params, 'att_func.0', flat))
  y = (gate * y).reshape(B, N, -1)
  if mask is None:
    score = torch.stack([y[b].mean(dim=0) for b in range(B)])                     # :193-194
  else:
    m = torch.as_tensor(mask).to(device=device, dtype=torch.bool)
    score = torch.stack([y[b, m[b], :].mean(dim=0) for b in range(B)])           # :189-191
  return (score, states) if return_states else score
