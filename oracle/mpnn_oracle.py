"""Functional torch oracle of the reference MPNN forward (model/mpnn.py, model/set2set.py).  TEST
INFRASTRUCTURE -- see oracle/__init__.py.

Independent of the kernels' algebra on purpose: the edge network runs in full (both layers, input
[h_j | h_i]) on every non-zero pair (b, i, j) of every channel, listed edge by edge, and the messages are
summed per receiver afterwards -- no split of the first layer, no W2 moved out of the sum, no fold into
the GRU weights.  The GRU is torch's GRUCell math, and Set2Vec runs graph by graph over the selected
nodes as in the reference.

``params`` is a flat dict keyed like the reference ``state_dict`` (``node_embedding.weight``,
``input_func.0.*``, ``update_func.*``, ``edge_func.{e}.{0,2}.*`` or ``edge_embedding.weight``,
``att_func.W_1``, ``att_func.W_2``, ``att_func.LSTM.{forget,input,output,memory}_gate.0.*``,
``output_func.0.*``); ``dtype`` selects fp32 (parity with the reference) or fp64 (rounding budget); the
forward is differentiable in ``params``.

Reference lines followed (relative to the reference checkout):
  model/mpnn.py:8         EPS = float32 machine epsilon
  model/mpnn.py:125       L[L != 0] = 1 (here the pattern of L; L is not modified)
  model/mpnn.py:128-129   state = input_func(node_embedding(node_feat))
  model/mpnn.py:132-134   edge-MLP input [h_j | h_i]: neighbour j first, receiver i second
  model/mpnn.py:141-179   messages: h E_e (embedding) or edge_func[e] (MLP), summed over A_e (sum), or
                          divided by (rowsum(A_e) + EPS) (avg)
  model/mpnn.py:184-196   GRUCell(cat(messages), state); dropout is the identity in eval mode
  model/mpnn.py:199-207   Set2Vec per graph over state[b, mask[b]] (all N rows without a mask), output_func
  model/set2set.py:39-57  LSTM gates forget, input, output (sigmoid), memory (tanh)
  model/set2set.py:79-100 energy = tanh(h W_1 + X) W_2, softmax over the set, read = sum a x
"""
import numpy as np
import torch
import torch.nn.functional as F

from .ggnn_oracle import cast_params, grad_digest  # noqa: F401  (grad_digest: same digest format)

EPS = float(np.finfo(np.float32).eps)
GATES = ('forget', 'input', 'output', 'memory')


def make_spec(num_prop, aggregate_type, msg_func, num_edgetype, num_step_set2vec):
  return {'num_prop': int(num_prop), 'aggregate_type': str(aggregate_type), 'msg_func': str(msg_func),
          'num_edgetype': int(num_edgetype), 'num_step_set2vec': int(num_step_set2vec)}


def set2vec(p, X):
  """model/set2set.py:79-100 for one set X [n, D]; returns hidden [1, 2D]."""
  D = X.shape[1]
  hidden = X.new_zeros((1, 2 * D))
  memory = X.new_zeros((1, D))
  steps = p['_num_step_set2vec']
  for _ in range(steps):
    g = {k: F.linear(hidden, p['att_func.LSTM.%s_gate.0.weight' % k], p['att_func.LSTM.%s_gate.0.bias' % k])
         for k in GATES}
    memory = torch.sigmoid(g['forget']) * memory + torch.sigmoid(g['input']) * torch.tanh(g['memory'])
    h = torch.sigmoid(g['output']) * torch.tanh(memory)
    energy = torch.tanh(h.mm(p['att_func.W_1']) + X).mm(p['att_func.W_2'])       # [n, 1]
    att = F.softmax(energy, dim=0)
    read = (X * att).sum(dim=0, keepdim=True)                                    # 0 for an empty set
    hidden = torch.cat([h, read], dim=1)
  return hidden


def mpnn_forward(params, spec, node_feat, L, mask, dtype=torch.float32, device='cpu', cast=True):
  """MPNN.forward without the loss, in eval mode.  ``L`` is not modified.  With ``cast=False`` the params
  are used as given (autograd leaves)."""
  p = dict(cast_params(params, dtype, device) if cast else params)
  p['_num_step_set2vec'] = spec['num_step_set2vec']
  node_feat = torch.as_tensor(node_feat).to(device).long()
  L = torch.as_tensor(L).to(device=device)
  A = L != 0
  B, N = node_feat.shape
  E1 = spec['num_edgetype'] + 1
  flat = F.linear(p['node_embedding.weight'][node_feat], p['input_func.0.weight'],
                  p['input_func.0.bias']).reshape(B * N, -1)
  D = flat.shape[1]
  edges = []
  for e in range(E1):                                     # (receiver, neighbour) row indices per channel
    b, i, j = A[:, :, :, e].nonzero(as_tuple=True)
    edges.append((b * N + i, b * N + j))
  nnz = A.to(dtype).sum(dim=2).reshape(B * N, E1)
  for _ in range(spec['num_prop']):
    msgs = []
    for e, (recv, nbr) in enumerate(edges):
      if spec['msg_func'] == 'MLP':
        x = torch.cat([flat[nbr], flat[recv]], dim=1)                             # [h_j | h_i]
        hid = F.relu(F.linear(x, p['edge_func.%d.0.weight' % e], p['edge_func.%d.0.bias' % e]))
        m = F.linear(hid, p['edge_func.%d.2.weight' % e], p['edge_func.%d.2.bias' % e])
      else:
        m = flat[nbr].mm(p['edge_embedding.weight'][e].view(D, D))
      agg = flat.new_zeros((B * N, D)).index_add(0, recv, m)
      if spec['aggregate_type'] == 'avg':
        agg = agg / (nnz[:, e:e + 1] + EPS)
      msgs.append(agg)
    gi = F.linear(torch.cat(msgs, dim=1), p['update_func.weight_ih'], p['update_func.bias_ih'])
    gh = F.linear(flat, p['update_func.weight_hh'], p['update_func.bias_hh'])
    i_r, i_z, i_n = gi.chunk(3, dim=1)
    h_r, h_z, h_n = gh.chunk(3, dim=1)
    r = torch.sigmoid(i_r + h_r)
    z = torch.sigmoid(i_z + h_z)
    n = torch.tanh(i_n + r * h_n)
    flat = (flat - n) * z + n
  state = flat.view(B, N, D)
  if mask is None:
    y = [set2vec(p, state[b]) for b in range(B)]
  else:
    m = torch.as_tensor(mask).to(device=device) != 0
    y = [set2vec(p, state[b, m[b], :]) for b in range(B)]
  return F.linear(torch.cat(y, dim=0), p['output_func.0.weight'], p['output_func.0.bias'])
