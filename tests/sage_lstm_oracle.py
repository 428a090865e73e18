"""Functional torch-CPU oracle of the reference GraphSAGE forward with the LSTM aggregator, restated from
the formula as a gather plus a loop of LSTM cells (model/graph_sage.py:98-175, the LSTM branch :131-140).
It complements oracle/sage_oracle.py (Mean / Max) and uses that module's spec, parameter casting and
gradient digest.

``params`` is a flat dict keyed like the reference ``state_dict`` (``embedding.weight``,
``agg_func.{ii}.{weight_ih,weight_hh,bias_ih,bias_hh}``, ``att_func.0.*``, ``filter.{t}.*``); ``dtype``
selects fp32 or fp64; the forward is differentiable in ``params``.  An id outside [0, N) reads a zero input
row (the reference raises an IndexError there); ``K`` defaults to nn_idx's sample count."""
import torch
import torch.nn.functional as F

from oracle.sage_oracle import EPS, cast_params, grad_digest, make_spec  # noqa: F401  (re-exported)


def lstm_cell(x, h, c, w_ih, w_hh, b_ih, b_hh):
  """torch.nn.LSTMCell: gates i, f, g, o in that order."""
  i, f, g, o = (F.linear(x, w_ih, b_ih) + F.linear(h, w_hh, b_hh)).chunk(4, dim=1)
  c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
  return torch.sigmoid(o) * torch.tanh(c), c


def sage_lstm_forward(params, spec, node_feat, nn_idx, nonempty_mask, mask, dtype=torch.float32, device='cpu',
                      cast=True, K=None):
  p = cast_params(params, dtype, device) if cast else params
  node_feat = torch.as_tensor(node_feat).to(device).long()
  nn_idx = torch.as_tensor(nn_idx).to(device).long()
  B, N = node_feat.shape
  K = nn_idx.shape[2] if K is None else K
  nonempty = torch.as_tensor(nonempty_mask).to(device=device, dtype=dtype).reshape(B, N, 1)
  state = p['embedding.weight'][node_feat]                                       # [B, N, D]
  rows = torch.arange(B, device=device).view(B, 1)
  for ii in range(spec['num_layer'] - 1):
    cell = [p['agg_func.%d.%s' % (ii, k)] for k in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')]
    D = state.shape[2]
    padded = torch.cat([state, state.new_zeros(B, 1, D)], dim=1)                 # row N: the zero row
    msg = []
    for jj in range(spec['num_edgetype'] + 1):
      h = c = state.new_zeros(B * N, D)
      for tt in range(K):
        m = nn_idx[:, :, tt, jj]
        m = torch.where((m >= 0) & (m < N), m, torch.full_like(m, N))
        x = padded[rows, m].reshape(B * N, D)
        h, c = lstm_cell(x, h, c, *cell)
      msg.append(h.view(B, N, D) * nonempty)
    y = F.relu(F.linear(torch.cat(msg, dim=2).view(B * N, -1), p['filter.%d.weight' % ii],
                        p['filter.%d.bias' % ii]))
    state = (y / (torch.norm(y, 2, dim=1, keepdim=True) + EPS)).view(B, N, -1)
  flat = state.reshape(B * N, -1)
  head = spec['num_layer']
  y = F.linear(flat, p['filter.%d.weight' % head], p['filter.%d.bias' % head])
  gate = torch.sigmoid(F.linear(flat, p['att_func.0.weight'], p['att_func.0.bias']))
  y = (gate * y).view(B, N, -1)
  if mask is None:
    return y.mean(dim=1)
  m = torch.as_tensor(mask).to(device=device, dtype=torch.bool)
  return torch.stack([y[b, m[b], :].mean(dim=0) for b in range(B)])
