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

from ._common import SparseRecords, SpectralNetBase, init_cell, init_linears, loss_function
from .. import ops

__all__ = ['GraphSAGE', 'LSTMGraphSAGE', 'SampledGraphSAGE', 'lstm_gate_matrix', 'lstm_gate_matrix_inverse']

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
    if layers < 1 or layers > ops.CONV_MAX_LAYERS or self.filter[self.num_layer].weight.shape[0] > 48:
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
    return self._stack_score(ops.graph_prepare(M, V), V, node_feat, mask)

  def _stack_score(self, prep, V, node_feat, mask):
    """The whole model in lnb_sage_stack_forward on the ELL rows ``prep`` of M (V: the zero [B, N, 4])."""
    E1 = prep[0].shape[1]
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
    return self._lstm_score(node_feat, nn_idx.to(torch.int32).contiguous(),   # converted once per forward
                            nonempty_mask.reshape(B * N).float().contiguous(), mask)

  def _lstm_score(self, node_feat, idx, ne, mask):
    """LSTM inference on lnb_sage_lstm_step: idx int32 [B, N, K, E1], ne float32 [B*N]."""
    B, N = node_feat.shape
    state = ops.embedding_rows(node_feat.long().reshape(-1), self.embedding.weight)
    for t in range(self.num_layer - 1):
      g_hi, g_lo, g_b = self._gates(t)
      msg = ops.sage_lstm_messages(state, idx, ne, g_hi, g_lo, g_b)
      lin = self.filter[t]
      w_hi, w_lo = self._wcache.split('filter.%d' % t, lin.weight)
      y = ops.linear_tf32x3(msg, w_hi, w_lo, lin.bias, relu=True)
      state = y / (torch.norm(y, 2, dim=1, keepdim=True) + EPS)
    return self._readout(state.view(B, N, -1), mask)


class SampledGraphSAGE(LSTMGraphSAGE):
  """``LSTMGraphSAGE`` (same constructor, parameters, initialisation and ``state_dict``; the same padded
  ``forward``) that also runs and trains from the bond-list records of data.sparse_collate:
  ``forward_sparse``, ``forward_sparse_train`` and ``train.GraphedStep(..., sparse=True)``.  ``forward_sparse``
  also takes packed batches (data.pack_sparse / data.PackedMolecules, with the same ``sample_key``): the same
  scores as the records they pack.

  The records carry no neighbour samples: they are drawn on the device (``ops.sage_sample_sparse``) from
  the distributions of the reference's collate -- K distinct neighbours, or K with replacement when a node
  has fewer -- with a counter-based generator keyed by ``batch['sample_key']``, an int64 tensor (seed,
  counter) that the caller changes to get new samples (inside a captured graph too).  numpy's draws are not
  reproduced, so this class does not make ``forward_sparse``'s usual promise of the collate's scores.  Its
  contract instead: the scores are, bit for bit, those of ``forward`` on the padded batch built from
  ``ops.sage_sample_sparse``'s samples (node_ids, nn_idx, nonempty, mask=mask), and the training entry
  computes ``forward``'s training formulation on the same samples.

  Mean / Max from records: sampler -> tile_assign -> lnb_sage_stack_forward (the count-weighted operator
  M exists only as ELL rows); off the stack kernel they run ``train.sage_train`` under no_grad on those
  rows.  LSTM reads the int32 samples directly.  Training: ``train.sage_train`` on the ELL rows of M and
  M^T (Mean), of M (Max), or on the samples (LSTM)."""

  def _check_runnable(self, N=None, E1=None):
    if self.agg_func is None:
      raise TypeError("SampledGraphSAGE: unknown agg_func %r; supported: Mean, Max, LSTM" % (self.agg_func_name,))

  def _sparse_inputs(self, batch):
    key = batch.get('sample_key') if isinstance(batch, dict) else None
    if key is None:
      raise ValueError("SampledGraphSAGE: the batch lacks 'sample_key', the int64 (seed, counter) tensor of "
                       "the neighbour sampler")
    if not torch.is_tensor(key) or key.dtype != torch.int64 or tuple(key.shape) != (2,):
      raise ValueError("SampledGraphSAGE: 'sample_key' must be an int64 tensor of shape (2,); got %r"
                       % ((key.dtype, tuple(key.shape)) if torch.is_tensor(key) else type(key),))
    if 'blob' in batch:
      blob, unpack, pkey = self._packed_records(batch)
      return (blob, key), lambda b_, k_: self._forward_records(unpack(b_), k_), pkey
    inputs, _, _ = super(SampledGraphSAGE, self)._sparse_inputs(batch)
    N = int(batch['N'])
    return (inputs + (key,), lambda *a: self._forward_records(SparseRecords(*a[:5], N=N), a[5]),
            ('sampled', N))

  def _sample(self, recs, key, **want):
    return ops.sage_sample_sparse(recs.sizes, recs.node_ptr, recs.node_feat, recs.edge_ptr, recs.edges,
                                  key.contiguous(), recs.N, self.num_edgetype + 1, self.num_sample_neighbors,
                                  **want)

  def _forward_records(self, recs, key):
    from ..train import EllOperator, sage_train
    E1 = self.num_edgetype + 1
    if self.agg_func_name == 'LSTM':
      node_ids, mask, nonempty, nn_idx, _, _ = self._sample(recs, key)
      if not self.lstm_supported(E1):
        return sage_train(self, node_ids, None, mask, samples=(nn_idx, nonempty))
      return self._lstm_score(node_ids, nn_idx, nonempty.view(-1), mask)
    node_ids, mask, _, _, prep, _ = self._sample(recs, key, want_nn_idx=False, want_ell=True)
    if not self.stack_supported(recs.N, E1):
      return sage_train(self, node_ids, EllOperator(prep, None, None), mask, prep=prep)   # no adjoint under no_grad
    ops.tile_assign(prep, 4)
    V = torch.zeros((node_ids.shape[0], recs.N, 4), device=node_ids.device, dtype=torch.float32)
    return self._stack_score(prep, V, node_ids, mask)

  def _train_records(self, recs, key):
    from ..train import EllOperator, sage_train
    if self.agg_func_name == 'LSTM':
      node_ids, mask, nonempty, nn_idx, _, _ = self._sample(recs, key)
      return sage_train(self, node_ids, None, mask, samples=(nn_idx, nonempty))
    mean = self.agg_func_name == 'Mean'
    node_ids, mask, _, _, prep, prep_t = self._sample(recs, key, want_nn_idx=False, want_ell=True, want_ell_t=mean)
    # Max routes its gradient through the argmax and never reads the transposed rows
    return sage_train(self, node_ids, EllOperator(prep, prep_t, None), mask, prep=prep)
