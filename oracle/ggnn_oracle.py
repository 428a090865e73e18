"""Functional torch-CPU oracle of the reference GGNN forward (not the fused kernels' formulation: dense
bmm's against the operators, torch's own GRUCell / RNNCell math, so it checks the gate re-layout and
the gathered aggregation independently).  TEST INFRASTRUCTURE -- see oracle/__init__.py.

``params`` is a flat dict keyed like the reference ``state_dict`` (``embedding.weight``,
``update_func.{weight_ih,weight_hh,bias_ih,bias_hh}``, ``msg_func.{e}.{0,2}.{weight,bias}``,
``att_func.0.*``, ``input_func.0.*``, ``output_func.0.*``); ``dtype`` selects fp32 (parity with the
reference) or fp64 (rounding budget); the forward is differentiable in ``params``.

Reference lines followed (relative to the reference checkout):
  model/ggnn.py:6         EPS = float32 machine epsilon
  model/ggnn.py:137       L[L != 0] = 1 (here on a copy)
  model/ggnn.py:140-141   state = input_func(embedding(node_feat))
  model/ggnn.py:143-171   _prop: msg_func[e], A_e m_e ('sum' / 'avg'), update_func(cat(msgs), state)
  model/ggnn.py:174-176   num_prop steps (dropout is the identity in eval mode)
  model/ggnn.py:179-192   output_func * att_func gate, per-graph (masked) mean
"""
import numpy as np
import torch
import torch.nn.functional as F

EPS = float(np.finfo(np.float32).eps)


def make_spec(num_prop, aggregate_type, update_func, num_edgetype):
  return {'num_prop': int(num_prop), 'aggregate_type': str(aggregate_type), 'update_func': str(update_func),
          'num_edgetype': int(num_edgetype)}


def cast_params(params, dtype, device='cpu'):
  return {k: (v.detach().to(device).to(dtype) if v.is_floating_point() else v.detach().to(device))
          for k, v in params.items()}


def ggnn_forward(params, spec, node_feat, L, mask, dtype=torch.float32, device='cpu', cast=True):
  """GGNN.forward without the loss, in eval mode.  mask=None averages over all N rows (:189-190).
  ``L`` is not modified.  With ``cast=False`` the params are used as given (autograd leaves)."""
  p = cast_params(params, dtype, device) if cast else params
  node_feat = torch.as_tensor(node_feat).to(device).long()
  L = torch.as_tensor(L).to(device=device)
  A = (L != 0).to(dtype)                                                        # :137
  B, N = node_feat.shape
  E1 = spec['num_edgetype'] + 1
  state = F.linear(p['embedding.weight'][node_feat], p['input_func.0.weight'], p['input_func.0.bias'])
  for _ in range(spec['num_prop']):
    flat = state.reshape(B * N, -1)
    msg = []
    for e in range(E1):
      hid = F.relu(F.linear(flat, p['msg_func.%d.0.weight' % e], p['msg_func.%d.0.bias' % e]))
      m = F.linear(hid, p['msg_func.%d.2.weight' % e], p['msg_func.%d.2.bias' % e]).view(B, N, -1)
      Ae = A[:, :, :, e]
      if spec['aggregate_type'] == 'avg':
        Ae = Ae / (torch.sum(Ae, dim=2, keepdim=True) + EPS)                    # :155-157
      msg.append(torch.bmm(Ae, m))                                              # :153-154
    x = torch.cat(msg, dim=2).view(B * N, -1)
    gi = F.linear(x, p['update_func.weight_ih'], p['update_func.bias_ih'])
    gh = F.linear(flat, p['update_func.weight_hh'], p['update_func.bias_hh'])
    if spec['update_func'] == 'GRU':                                            # nn.GRUCell
      i_r, i_z, i_n = gi.chunk(3, dim=1)
      h_r, h_z, h_n = gh.chunk(3, dim=1)
      r = torch.sigmoid(i_r + h_r)
      z = torch.sigmoid(i_z + h_z)
      n = torch.tanh(i_n + r * h_n)
      flat = (flat - n) * z + n                                                 # h' = (1 - z) n + z h
    else:                                                                       # nn.RNNCell, relu
      flat = F.relu(gi + gh)
    state = flat.view(B, N, -1)
  flat = state.reshape(B * N, -1)
  y = F.linear(flat, p['output_func.0.weight'], p['output_func.0.bias'])        # :180
  gate = torch.sigmoid(F.linear(flat, p['att_func.0.weight'], p['att_func.0.bias']))
  y = (gate * y).view(B, N, -1)
  if mask is None:
    return torch.stack([y[b].mean(dim=0) for b in range(B)])                    # :189-190
  m = torch.as_tensor(mask).to(device=device, dtype=torch.bool)
  return torch.stack([y[b, m[b], :].mean(dim=0) for b in range(B)])             # :186-187


def grad_digest(grads):
  """Per-parameter digest of make_golden.golden_train_grads: sum, sum of squares, first 8 entries."""
  out = {}
  for name, g in grads.items():
    g = g.detach().double().numpy().reshape(-1)
    out[name] = np.concatenate([[g.sum(), (g * g).sum()], g[:8]])
  return out
