"""Drop-in for the reference ``model.GraphSAGE`` (model/graph_sage.py:10-175) with the ``Mean`` and ``Max``
aggregators.  Same constructor fields, parameter names, registration and initialisation order (so
``torch.manual_seed(s)`` gives the reference's initial weights and its checkpoints load by name), and the
same ``forward(node_feat, nn_idx, nonempty_mask, label=None, mask=None)`` the runner calls
(runner/qm8_runner.py:134-140).

The reference gathers ``state[b, nn_idx[b, :, :, jj]]`` in a Python loop over the batch for every channel
of every layer (graph_sage.py:120-146).  Here the K neighbour samples of each node become the
count-weighted operator M_e[n, m] = nonempty[n] * count_e(n, m) / K (``ops.sage_operators``): the Mean
message is M_e X, and the non-zeros of row n of M_e are the neighbours the Max takes.  M does not depend
on the layer, so inference is ``sage_operators -> graph_prepare -> sage_stack_forward`` -- 4 launches
with the embedding gather and the readout fused, replayed as one CUDA graph.

Semantics kept from the reference:
  * ``num_layer - 1`` propagation layers use filter[0 .. num_layer-2]; filter[num_layer-1] is registered
    and initialised but never read; the head is filter[num_layer] (graph_sage.py:53-56,120,158);
  * a node with nonempty = 1 and no neighbour in channel jj has nn_idx[..., jj] = 0 and aggregates node
    0 (the collate's zero fill, dataset/qm8.py:143-163): the operator built from nn_idx does the same;
  * each layer is relu(Linear(msg)) / (||.||_2 + float32 eps), then dropout; padded nodes (nonempty = 0)
    get the constant row relu(b) / (||relu(b)|| + eps), which enters the mean when mask is None.
``GraphSAGE`` does not take ``agg_func: LSTM``: the constructor raises NotImplementedError before drawing
any random number.  ``LSTMGraphSAGE`` (below; ``--opt-in GraphSAGE`` of lanczosnetwork_b200.dropin) takes
it.  An unknown aggregator fails in the forward, as in the reference.  Ids outside [0, N) contribute
nothing (the reference raises an IndexError); under the LSTM aggregator such an id is a zero input row."""
import torch
import torch.nn as nn

from ._common import SpectralNetBase, init_cell, init_linears, loss_function
from .. import ops

__all__ = ['GraphSAGE', 'LSTMGraphSAGE', 'lstm_gate_matrix', 'lstm_gate_matrix_inverse']

SUPPORTED_AGGREGATORS = ('Mean', 'Max')
EPS = 1.1920928955078125e-07       # np.finfo(np.float32).eps (graph_sage.py:6)


class GraphSAGE(SpectralNetBase):
  _takes_lstm = False

  def __init__(self, config):
    m = config.model
    if m.agg_func == 'LSTM' and not self._takes_lstm:
      raise NotImplementedError(
          "GraphSAGE drop-in: agg_func 'LSTM' is not implemented; supported aggregators: %s"
          % ', '.join(SUPPORTED_AGGREGATORS))
    super(GraphSAGE, self).__init__()
    self._setup_fields(config, config.dataset.num_bond_type)
    self.num_sample_neighbors = m.num_sample_neighbors
    assert self.num_layer == len(self.hidden_dim)
    dims = [self.input_dim] + list(self.hidden_dim) + [self.output_dim]

    self.embedding = nn.Embedding(self.num_atom, self.input_dim)
    self.agg_func_name = m.agg_func
    if self.agg_func_name == 'LSTM':            # LSTMGraphSAGE only; each cell draws its default init here
      self.agg_func = nn.ModuleList([nn.LSTMCell(dims[t], dims[t]) for t in range(self.num_layer - 1)])
    else:
      self.agg_func = {'Mean': torch.mean, 'Max': torch.max}.get(self.agg_func_name)
    self.att_func = nn.Sequential(nn.Linear(dims[-2], 1), nn.Sigmoid())
    self.filter = nn.ModuleList(
        [nn.Linear(dims[t] * (self.num_edgetype + 1), dims[t + 1]) for t in range(self.num_layer)] +
        [nn.Linear(dims[-2], dims[-1])])
    self.loss_func = loss_function(m.loss)
    self._init_param()

  def _init_param(self):
    """Xavier-uniform weights and zero biases, att_func first, then (LSTM) Xavier on weight_hh, weight_ih
    and zero biases of every cell, then filter (graph_sage.py:69-96); the embedding keeps nn.Embedding's
    default N(0, 1)."""
    init_linears(self.att_func)
    if self.agg_func_name == 'LSTM':
      for cell in self.agg_func:
        init_cell(cell)
    init_linears(self.filter)

  def forward(self, node_feat, nn_idx, nonempty_mask, label=None, mask=None):
    """
      node_feat: long B x N (atom ids); nn_idx: long B x N x K x (E+1) neighbour samples;
      nonempty_mask: float B x N x 1; label: B x P; mask: B x N (uint8 / bool / float).
      Returns score (B x P) or (score, loss).
    """
    self._device()                        # a CPU module refuses before the aggregator is checked
    if self.agg_func is None:
      raise TypeError("GraphSAGE: unknown agg_func %r ('NoneType' object is not callable, as in the "
                      "reference); supported: %s" % (self.agg_func_name, ', '.join(SUPPORTED_AGGREGATORS)))
    return self._forward((node_feat, nn_idx, nonempty_mask, mask), label)

  def _train_impl(self, node_feat, nn_idx, nonempty_mask, mask):
    from ..train import sage_train
    M = ops.sage_operators(nn_idx, nonempty_mask)
    return sage_train(self, node_feat, M, mask)

  def stack_supported(self, N, E1):
    """True when the whole model runs in the one-launch stack kernel: 1..8 propagation layers of one
    hidden width, every layer within the kernel's shapes (N <= 128, widths % 32, H <= 128) and at most
    48 outputs."""
    layers = self.num_layer - 1
    if layers < 1 or layers > 8 or self.filter[self.num_layer].weight.shape[0] > 48:
      return False
    dims = [self.embedding.weight.shape[1]] + list(self.hidden_dim[:layers])
    H = dims[1]
    if any(d != H for d in dims[1:]):
      return False
    return all(ops.fused_conv_supported(N, dims[t], 4, H, 0, False, 0, E1) for t in range(layers))

  def _forward_impl(self, node_feat, nn_idx, nonempty_mask, mask):
    B, N = node_feat.shape
    M = ops.sage_operators(nn_idx, nonempty_mask)
    E1 = M.shape[3]
    if not self.stack_supported(N, E1):
      from ..train import sage_train                # off the stack: the training formulation (no_grad)
      return sage_train(self, node_feat, M, mask)
    # no Ritz vectors: an all-zero block makes lnb_graph_prepare take the extents from M alone
    V = torch.zeros((B, N, 4), device=M.device, dtype=torch.float32)
    prep = ops.graph_prepare(M, V)
    layers = list(range(self.num_layer - 1))
    dims = [self.embedding.weight.shape[1]] + list(self.hidden_dim[:len(layers)])
    H = dims[1]
    w_hi, w_lo, bias = self._wcache.split_conv_stack(
        'filter.sage', [self.filter[t].weight for t in layers], [self.filter[t].bias for t in layers],
        E1 * max(dims[:len(layers)]))
    head, att = self.filter[self.num_layer], self.att_func[0]
    _, score = ops.spectral_stack_forward(
        prep, V, w_hi, w_lo, bias, dims[:len(layers)], H, 0, node_ids=node_feat.long(),
        emb=self.embedding.weight, readout=(head.weight, head.bias, att.weight.reshape(-1), att.bias),
        mask=mask, sage=self.agg_func_name)
    return score


def lstm_gate_matrix(weight_ih, weight_hh, bias_ih, bias_hh):
  """An nn.LSTMCell as one GEMM over [x | h] (layout of lnb_sage_lstm_step): returns W [4D, 2D] and b [4D]
  whose row (u // 4) * 16 + g * 4 + u % 4 is gate g (i, f, g, o) of hidden unit u: [W_ih | W_hh] rows
  g*D + u, and b_ih + b_hh in the same order.  Works on any device."""
  D = weight_hh.shape[1]
  W = torch.cat([weight_ih, weight_hh], dim=1)
  b = bias_ih + bias_hh
  W = W.reshape(4, D // 4, 4, 2 * D).permute(1, 0, 2, 3).reshape(4 * D, 2 * D).contiguous()
  b = b.reshape(4, D // 4, 4).permute(1, 0, 2).reshape(4 * D).contiguous()
  return W, b


def lstm_gate_matrix_inverse(W, b):
  """(weight_ih, weight_hh, b_ih + b_hh) of a matrix from lstm_gate_matrix."""
  D = W.shape[1] // 2
  W = W.reshape(D // 4, 4, 4, 2 * D).permute(1, 0, 2, 3).reshape(4 * D, 2 * D)
  b = b.reshape(D // 4, 4, 4).permute(1, 0, 2).reshape(4 * D)
  return W[:, :D].contiguous(), W[:, D:].contiguous(), b.contiguous()


class LSTMGraphSAGE(GraphSAGE):
  """GraphSAGE with the reference's three aggregators.  ``Mean`` and ``Max`` behave exactly as in
  GraphSAGE.  ``LSTM`` builds the reference's ``agg_func`` (one nn.LSTMCell per propagation layer, shared
  by the E+1 channels) in the reference's construction and initialisation order, so a seed gives its
  initial weights and its checkpoints load by name.

  LSTM inference per layer ii: K = num_sample_neighbors launches of ``lnb_sage_lstm_step`` (all
  B*N*(E+1) sequences per launch, the neighbour rows gathered in the producer warps, the cell in the
  epilogue, the last step writing the message matrix), then ``linear_tf32x3`` + ReLU for filter[ii] and
  the row normalisation in torch; the embedding gather in front and ``ops.readout`` behind, all replayed
  as one CUDA graph.  Widths outside the kernel (D % 32 != 0, D > 128) or more than 16 channels run the
  training formulation (``train.sage_train``) under no_grad.  Training: ``train.lstm_messages``."""
  _takes_lstm = True

  def _samples(self, nn_idx):
    K = self.num_sample_neighbors
    if nn_idx.shape[2] < K:
      raise ValueError('LSTMGraphSAGE: nn_idx holds %d samples per node, num_sample_neighbors is %d'
                       % (nn_idx.shape[2], K))
    return nn_idx[:, :, :K]

  def _train_impl(self, node_feat, nn_idx, nonempty_mask, mask):
    if self.agg_func_name != 'LSTM':
      return super(LSTMGraphSAGE, self)._train_impl(node_feat, nn_idx, nonempty_mask, mask)
    from ..train import sage_train
    return sage_train(self, node_feat, None, mask, samples=(self._samples(nn_idx), nonempty_mask))

  def lstm_supported(self, E1):
    """True when every propagation layer runs on lnb_sage_lstm_step (and its filter on the dense kernel)."""
    dims = [self.embedding.weight.shape[1]] + list(self.hidden_dim[:self.num_layer - 1])
    return all(ops.sage_lstm_step_supported(dims[t], E1, self.num_sample_neighbors)
               for t in range(self.num_layer - 1))

  def _gates(self, t):
    cell = self.agg_func[t]

    def build():
      W, b = lstm_gate_matrix(cell.weight_ih.detach(), cell.weight_hh.detach(), cell.bias_ih.detach(),
                              cell.bias_hh.detach())
      return ops.split_tf32(W) + (b,)
    return self._wcache.derived('agg_func.%d.gates' % t,
                                [cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh], build)

  def _forward_impl(self, node_feat, nn_idx, nonempty_mask, mask):
    if self.agg_func_name != 'LSTM':
      return super(LSTMGraphSAGE, self)._forward_impl(node_feat, nn_idx, nonempty_mask, mask)
    B, N = node_feat.shape
    E1 = nn_idx.shape[3]
    nn_idx = self._samples(nn_idx)
    if not self.lstm_supported(E1):
      from ..train import sage_train                # off the kernel: the training formulation (no_grad)
      return sage_train(self, node_feat, None, mask, samples=(nn_idx, nonempty_mask))
    idx = nn_idx.to(torch.int32).contiguous()        # converted once per forward
    ne = nonempty_mask.reshape(B * N).float().contiguous()
    state = ops.embedding_rows(node_feat.long().reshape(-1), self.embedding.weight)
    for t in range(self.num_layer - 1):
      g_hi, g_lo, g_b = self._gates(t)
      msg = ops.sage_lstm_messages(state, idx, ne, g_hi, g_lo, g_b)
      lin = self.filter[t]
      w_hi, w_lo = self._wcache.split('filter.%d' % t, lin.weight)
      y = ops.linear_tf32x3(msg, w_hi, w_lo, lin.bias, relu=True)
      state = y / (torch.norm(y, 2, dim=1, keepdim=True) + EPS)
    return self._readout(state.view(B, N, -1), mask)
