"""Functional torch-CPU oracle of the reference GraphSAGE forward, in the reference's GATHER formulation
(not the count-weighted operator form the library runs, so it checks that construction independently).
TEST INFRASTRUCTURE -- see oracle/__init__.py.

``params`` is a flat dict keyed like the reference ``state_dict`` (``embedding.weight``,
``att_func.0.{weight,bias}``, ``filter.{t}.{weight,bias}``); ``dtype`` selects fp32 (parity with the
reference) or fp64 (rounding budget); the forward is differentiable in ``params``.

Reference lines followed (relative to the reference checkout):
  dataset/qm8.py:137-166        the neighbour samples nn_idx and the per-node nonempty flag
  model/graph_sage.py:98-175    GraphSAGE.forward (Mean / Max aggregators)
"""
import numpy as np
import torch
import torch.nn.functional as F

EPS = float(np.finfo(np.float32).eps)          # model/graph_sage.py:6


def make_spec(num_layer, agg_func, num_edgetype):
  return {'num_layer': int(num_layer), 'agg_func': str(agg_func), 'num_edgetype': int(num_edgetype)}


def cast_params(params, dtype, device='cpu'):
  return {k: (v.detach().to(device).to(dtype) if v.is_floating_point() else v.detach().to(device))
          for k, v in params.items()}


def sage_forward(params, spec, node_feat, nn_idx, nonempty_mask, mask, dtype=torch.float32, device='cpu',
                 cast=True):
  """GraphSAGE.forward without the loss.  mask=None averages over all N rows (:166-168).  With
  ``cast=False`` the params are used as given (autograd leaves of the caller)."""
  p = cast_params(params, dtype, device) if cast else params
  node_feat = torch.as_tensor(node_feat).to(device).long()
  nn_idx = torch.as_tensor(nn_idx).to(device).long()
  nonempty = torch.as_tensor(nonempty_mask).to(device=device, dtype=dtype).reshape(node_feat.shape + (1,))
  B, N = node_feat.shape
  E = spec['num_edgetype']
  state = p['embedding.weight'][node_feat]                                      # :117
  rows = torch.arange(B, device=device).view(B, 1, 1)
  for ii in range(spec['num_layer'] - 1):                                       # :120
    msg = []
    for jj in range(E + 1):
      nn_state = state[rows, nn_idx[:, :, :, jj], :]                            # :124-128, B x N x K x D
      if spec['agg_func'] == 'Max':
        agg, _ = torch.max(nn_state, dim=2)                                     # :141-142
      else:
        agg = torch.mean(nn_state, dim=2)                                       # :143-144
      msg.append(agg * nonempty)                                                # :146
    y = F.relu(F.linear(torch.cat(msg, dim=2).view(B * N, -1), p['filter.%d.weight' % ii],
                        p['filter.%d.bias' % ii]))                              # :150-151
    state = (y / (torch.norm(y, 2, dim=1, keepdim=True) + EPS)).view(B, N, -1)  # :152-153
  flat = state.reshape(B * N, -1)
  head = spec['num_layer']                                                      # filter[-1]
  y = F.linear(flat, p['filter.%d.weight' % head], p['filter.%d.bias' % head])  # :158
  gate = torch.sigmoid(F.linear(flat, p['att_func.0.weight'], p['att_func.0.bias']))
  y = (gate * y).view(B, N, -1)
  if mask is None:
    return torch.stack([y[b].mean(dim=0) for b in range(B)])                    # :166-168
  m = torch.as_tensor(mask).to(device=device, dtype=torch.bool)
  return torch.stack([y[b, m[b], :].mean(dim=0) for b in range(B)])             # :163-165


def grad_digest(grads):
  """Per-parameter digest of make_golden.golden_train_grads: sum, sum of squares, first 8 entries."""
  out = {}
  for name, g in grads.items():
    g = g.detach().double().numpy().reshape(-1)
    out[name] = np.concatenate([[g.sum(), (g * g).sum()], g[:8]])
  return out
