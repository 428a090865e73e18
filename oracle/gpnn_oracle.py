"""Functional torch-CPU oracle of the reference GPNN forward (not the kernels' formulation: dense bmm's
against the operators, torch's own GRUCell / RNNCell math, so it checks the gate re-layout, the valued
partition aggregation and the concatenation independently).  TEST INFRASTRUCTURE -- see oracle/__init__.py.

``params`` is a flat dict keyed like the reference ``state_dict`` (``embedding.weight``,
``update_func.*``, ``update_func_partition.{weight_ih,weight_hh,bias_ih,bias_hh}``,
``state_func.{0,2}.*``, ``msg_func.{e}.{0,2}.*``, ``att_func.0.*``, ``input_func.0.*``,
``output_func.0.*``); ``dtype`` selects fp32 (parity with the reference) or fp64 (rounding budget); the
forward is differentiable in ``params``.

Reference lines followed (relative to the reference checkout):
  model/gpnn.py:7         EPS = float32 machine epsilon
  model/gpnn.py:158       L[L != 0] = 1 (here on a copy); L_cluster / L_cut keep their values
  model/gpnn.py:161-162   state = input_func(embedding(node_feat))
  model/gpnn.py:164-190   _prop: msg_func[e], A_e m_e ('sum' / 'avg'), update_func(cat(msgs), state)
  model/gpnn.py:192-213   _prop_partition: msg_func[0], L_step m ('sum' / 'avg'), update_func_partition
  model/gpnn.py:216-230   num_prop steps: cluster / cut chains from the same state, state_func on the
                          concatenation, _prop (dropout is the identity in eval mode)
  model/gpnn.py:233-246   output_func * att_func gate, per-graph (masked) mean
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.ggnn_oracle import cast_params, grad_digest  # noqa: F401  (same conventions as GGNN)

EPS = float(np.finfo(np.float32).eps)


def make_spec(num_prop, num_prop_cluster, num_prop_cut, aggregate_type, update_func, num_edgetype):
  return {'num_prop': int(num_prop), 'num_prop_cluster': int(num_prop_cluster), 'num_prop_cut': int(num_prop_cut),
          'aggregate_type': str(aggregate_type), 'update_func': str(update_func), 'num_edgetype': int(num_edgetype)}


def _cell(p, name, kind, x, h):
  gi = F.linear(x, p[name + '.weight_ih'], p[name + '.bias_ih'])
  gh = F.linear(h, p[name + '.weight_hh'], p[name + '.bias_hh'])
  if kind == 'GRU':                                                             # nn.GRUCell
    i_r, i_z, i_n = gi.chunk(3, dim=1)
    h_r, h_z, h_n = gh.chunk(3, dim=1)
    r = torch.sigmoid(i_r + h_r)
    z = torch.sigmoid(i_z + h_z)
    n = torch.tanh(i_n + r * h_n)
    return (h - n) * z + n                                                      # h' = (1 - z) n + z h
  return F.relu(gi + gh)                                                        # nn.RNNCell, relu


def _aggregate(op, m, kind):
  if kind == 'avg':
    op = op / (torch.sum(op, dim=2, keepdim=True) + EPS)
  return torch.bmm(op, m)


def _msg(p, e, flat):
  hid = F.relu(F.linear(flat, p['msg_func.%d.0.weight' % e], p['msg_func.%d.0.bias' % e]))
  return F.linear(hid, p['msg_func.%d.2.weight' % e], p['msg_func.%d.2.bias' % e])


def gpnn_forward(params, spec, node_feat, L, L_cluster, L_cut, mask, dtype=torch.float32, device='cpu', cast=True):
  """GPNN.forward without the loss, in eval mode.  mask=None averages over all N rows (:243-244).
  ``L`` is not modified.  With ``cast=False`` the params are used as given (autograd leaves)."""
  p = cast_params(params, dtype, device) if cast else params
  node_feat = torch.as_tensor(node_feat).to(device).long()
  A = (torch.as_tensor(L).to(device=device) != 0).to(dtype)                    # :158
  parts = [torch.as_tensor(t).to(device=device, dtype=dtype) for t in (L_cluster, L_cut)]
  B, N = node_feat.shape
  E1 = spec['num_edgetype'] + 1
  kind, agg = spec['update_func'], spec['aggregate_type']
  state = F.linear(p['embedding.weight'][node_feat], p['input_func.0.weight'], p['input_func.0.bias'])
  state = state.reshape(B * N, -1)
  for _ in range(spec['num_prop']):
    chains = []
    for op, count in zip(parts, (spec['num_prop_cluster'], spec['num_prop_cut'])):
      s = state
      for _ in range(count):                                                    # :192-213
        m = _msg(p, 0, s).view(B, N, -1)
        s = _cell(p, 'update_func_partition', kind, _aggregate(op, m, agg).reshape(B * N, -1), s)
      chains.append(s)
    x = torch.cat([state] + chains, dim=1)                                      # :227-228
    s = F.linear(F.relu(F.linear(x, p['state_func.0.weight'], p['state_func.0.bias'])),
                 p['state_func.2.weight'], p['state_func.2.bias'])
    msg = [_aggregate(A[:, :, :, e], _msg(p, e, s).view(B, N, -1), agg) for e in range(E1)]   # :164-190
    state = _cell(p, 'update_func', kind, torch.cat(msg, dim=2).view(B * N, -1), s)
  y = F.linear(state, p['output_func.0.weight'], p['output_func.0.bias'])      # :234
  gate = torch.sigmoid(F.linear(state, p['att_func.0.weight'], p['att_func.0.bias']))
  y = (gate * y).view(B, N, -1)
  if mask is None:
    return torch.stack([y[b].mean(dim=0) for b in range(B)])                    # :243-244
  m = torch.as_tensor(mask).to(device=device, dtype=torch.bool)
  return torch.stack([y[b, m[b], :].mean(dim=0) for b in range(B)])             # :240-241
