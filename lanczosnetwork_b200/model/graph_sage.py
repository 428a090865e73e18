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
``agg_func: LSTM`` is not implemented: the constructor raises NotImplementedError before drawing any
random number.  An unknown aggregator fails in the forward, as in the reference.  Ids outside [0, N)
contribute nothing (the reference raises an IndexError)."""
import torch
import torch.nn as nn

from ._common import SpectralNetBase, init_linears, loss_function
from .. import ops

__all__ = ['GraphSAGE']

SUPPORTED_AGGREGATORS = ('Mean', 'Max')


class GraphSAGE(SpectralNetBase):

  def __init__(self, config):
    m = config.model
    if m.agg_func == 'LSTM':
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
    self.agg_func = {'Mean': torch.mean, 'Max': torch.max}.get(self.agg_func_name)
    self.att_func = nn.Sequential(nn.Linear(dims[-2], 1), nn.Sigmoid())
    self.filter = nn.ModuleList(
        [nn.Linear(dims[t] * (self.num_edgetype + 1), dims[t + 1]) for t in range(self.num_layer)] +
        [nn.Linear(dims[-2], dims[-1])])
    self.loss_func = loss_function(m.loss)
    self._init_param()

  def _init_param(self):
    """Xavier-uniform weights and zero biases, att_func first, then filter (graph_sage.py:69-96); the
    embedding keeps nn.Embedding's default N(0, 1)."""
    init_linears([*self.att_func, *self.filter])

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
