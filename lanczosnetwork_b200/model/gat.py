"""Drop-in for the reference ``model.GAT`` (model/gat.py:8-201): graph attention over the bond channels,
inference only.  Same constructor fields, parameter names, registration and initialisation order (so
``torch.manual_seed(s)`` gives the reference's initial weights and its checkpoints load by name), and
the same ``forward(node_feat, L, label=None, mask=None)``, where ``L`` is the additive attention bias
the reference collate builds for GAT (``data.gat_bias``).

Per layer the reference runs one Linear / two scorers / softmax / bmm sequence for each of the
(E+1) * heads channels (model/gat.py:145-180).  Here a layer is two launches: the per-head weights,
stacked in concat order into one [C*F, Din] matrix, go through the 3xTF32 wgmma dense layer once for
all B*N rows, and ``lnb_gat_attention`` does the scorers, the column softmax, the aggregation and the
ELU (or, in the last layer, the mean over channels).  With the embedding gather and the readout that is
2 + 2 * num_layer launches, captured as one CUDA graph.

Quirk kept on purpose: the reference's ``state_bias`` repeats one inner list for every bond channel
(model/gat.py:62-70), so every channel of layer t uses ``bias_{ii}_{E}_{t}``; the other
``bias_{ii}_{jj}_{t}`` are registered and saved but never read.  ``GAT`` has no training path: under
autograd with trainable parameters the forward raises, and ``dropin.patch_namespace(training=True)``
keeps the reference class for training runs.  ``TrainableGAT`` (same constructor, parameters and
checkpoints) adds one: under autograd its forward is ``train.gat_train``, whose attention adjoint is
``lnb_gat_attention_backward``; the drop-in binds it under the name ``GAT`` by opt-in only
(``dropin.TRAINING_OPT_IN_CLASSES``, ``--opt-in GAT``).  ``KeyedGAT`` (same again) also trains with
``dropout > 0``, its masks drawn on the device from a key (``--opt-in GAT --keyed-dropout``)."""
import torch
import torch.nn as nn

from ._common import SpectralNetBase, init_linears, loss_function
from .. import ops

__all__ = ['GAT', 'TrainableGAT', 'KeyedGAT']


def _linear_grid(num_layer, num_channel, num_heads, make):
  return nn.ModuleList([
      nn.ModuleList([nn.ModuleList([make(t) for _ in range(num_heads[t])]) for _ in range(num_channel)])
      for t in range(num_layer)])


class GAT(SpectralNetBase):

  def __init__(self, config):
    super(GAT, self).__init__()
    m = config.model
    self._setup_fields(config, config.dataset.num_bond_type)
    self.num_heads = m.num_heads
    E1 = self.num_edgetype + 1
    dims = [self.input_dim] + list(self.hidden_dim) + [self.output_dim]

    self.embedding = nn.Embedding(self.num_atom, self.input_dim)
    # input width of layer t > 0 is dims[t] * num_heads[t] * (E+1): num_heads of layer t itself,
    # as the reference constructor has it (model/gat.py:34-38)
    din = [dims[t] if t == 0 else dims[t] * self.num_heads[t] * E1 for t in range(self.num_layer)]
    self.filter = _linear_grid(self.num_layer, E1, self.num_heads,
                               lambda t: nn.Linear(din[t], dims[t + 1], bias=False))
    self.att_net_1 = _linear_grid(self.num_layer, E1, self.num_heads, lambda t: nn.Linear(dims[t + 1], 1))
    self.att_net_2 = _linear_grid(self.num_layer, E1, self.num_heads, lambda t: nn.Linear(dims[t + 1], 1))
    # bias_{ii}_{jj}_{t}, registered on the module itself (first in the state_dict); state_bias[t][jj]
    # is ONE list shared by every jj, so it ends up holding the jj = E parameters
    self.state_bias = []
    for t in range(self.num_layer):
      shared = [None] * self.num_heads[t]
      self.state_bias.append([shared] * E1)
      for jj in range(E1):
        for ii in range(self.num_heads[t]):
          shared[ii] = nn.Parameter(torch.zeros(dims[t + 1]))
          self.register_parameter('bias_%d_%d_%d' % (ii, jj, t), shared[ii])
    self.att_func = nn.Sequential(nn.Linear(dims[-2], 1), nn.Sigmoid())
    self.output_func = nn.Sequential(nn.Linear(dims[-2], dims[-1]))
    self.loss_func = loss_function(m.loss)
    self._init_param()

  def _init_param(self):
    """Xavier-uniform weights and zero biases, in the reference's order (model/gat.py:88-123):
    att_func, output_func, filter, att_net_1, att_net_2."""
    linears = list(self.att_func) + list(self.output_func)
    for grid in (self.filter, self.att_net_1, self.att_net_2):
      linears += [mod for per_layer in grid for per_channel in per_layer for mod in per_channel]
    init_linears(linears)

  def _param_device(self):
    return self.embedding.weight.device

  def forward(self, node_feat, L, label=None, mask=None):
    """
      node_feat: long B x N (atom ids); L: float B x N x N x (E+1), the attention bias of the GAT
      collate (data.gat_bias); label: B x P; mask: B x N (uint8 / bool / float).
      Returns score (B x P) or (score, loss).
    """
    return self._forward((node_feat, L, mask), label)          # no training path: raises under autograd

  def _layer_params(self, t):
    """Per-layer tensors in concat order c = jj * heads + ii, stacked once per parameter version."""
    E = self.num_edgetype
    mods = [(jj, ii) for jj in range(E + 1) for ii in range(self.num_heads[t])]
    cache = self._wcache
    w = [self.filter[t][jj][ii].weight for jj, ii in mods]
    a1, = cache.stacked('att_net_1.%d.weight' % t, [self.att_net_1[t][jj][ii].weight for jj, ii in mods])
    a2, = cache.stacked('att_net_2.%d.weight' % t, [self.att_net_2[t][jj][ii].weight for jj, ii in mods])
    c1, = cache.stacked('att_net_1.%d.bias' % t, [self.att_net_1[t][jj][ii].bias for jj, ii in mods])
    c2, = cache.stacked('att_net_2.%d.bias' % t, [self.att_net_2[t][jj][ii].bias for jj, ii in mods])
    # every channel reads the bias registered for jj = E (the shared state_bias list)
    sb, = cache.stacked('state_bias.%d' % t, [getattr(self, 'bias_%d_%d_%d' % (ii, E, t)) for _, ii in mods])
    return w, a1, a2, c1, c2, sb.view(len(mods), -1)

  def _project(self, x2d, weights, t):
    """x2d @ [W_0; W_1; ...]^T: every head of every channel in one dense launch."""
    M, K = x2d.shape
    if K % 4 == 0:
      w_hi, w_lo = self._wcache.stacked('filter.%d' % t, weights, split=True)
      return ops.linear_tf32x3(x2d, w_hi, w_lo)
    w, = self._wcache.stacked('filter.%d' % t, weights)       # rows not 16-byte multiples: FFMA GEMM
    out = torch.empty((M, w.shape[0]), device=x2d.device, dtype=torch.float32)
    ops.bgemm(x2d, (0, 0, K, 1), w, (0, 0, 1, K), out, (0, 0, w.shape[0], 1), 1, 1, M, w.shape[0], K)
    return out

  def _forward_impl(self, node_feat, L, mask):
    bias = L.float().contiguous()
    B, N = node_feat.shape
    state = ops.embedding_rows(node_feat.long(), self.embedding.weight)
    for t in range(self.num_layer):
      w, a1, a2, c1, c2, sb = self._layer_params(t)
      Wh = self._project(state.reshape(B * N, -1), w, t).view(B, N, -1)
      state = ops.gat_attention(Wh, bias, a1, a2, c1, c2, sb, last=(t == self.num_layer - 1))
    head, att = self.output_func[0], self.att_func[0]
    return ops.readout(state, head.weight, head.bias, att.weight.reshape(-1), att.bias, mask)

  def _forward_records(self, recs):
    _, node_ids, mask, _, _ = self._prepare_records(recs)
    bias = ops.gat_bias_sparse(recs.sizes, recs.edge_ptr, recs.edges, recs.N, self.num_edgetype + 1)
    return self._forward_impl(node_ids, bias, mask)


class TrainableGAT(GAT):
  """``GAT`` with a training path.  Under ``no_grad`` (or without trainable parameters) the forward is the
  fused inference path with its CUDA graphs; under autograd it is ``train.gat_train``.  Dropout > 0 in
  training mode is refused: the reference draws it at three sites per head (the head's input, the
  attention weights and Wh, model/gat.py:149-163), and per-head input masks rule out the one stacked
  projection per layer."""

  def forward(self, node_feat, L, label=None, mask=None):
    if self.training and self.dropout > 0.0:
      raise NotImplementedError(
          'TrainableGAT: dropout %g in training mode is not implemented (the reference drops the per-head '
          'input, the attention weights and Wh); train with dropout 0.0' % self.dropout)
    return self._forward((node_feat, L, mask), label)

  def _train_impl(self, node_feat, L, mask):
    from ..train import gat_train
    return gat_train(self, node_feat, L, mask)

  def _train_records(self, recs):
    from ..train import gat_train
    if self.training and self.dropout > 0.0:
      raise NotImplementedError('TrainableGAT: dropout %g in training mode is not implemented; train with '
                                'dropout 0.0' % self.dropout)
    _, node_ids, mask, _, _ = self._prepare_records(recs)
    bias = ops.gat_bias_sparse(recs.sizes, recs.edge_ptr, recs.edges, recs.N, self.num_edgetype + 1)
    return gat_train(self, node_ids, bias, mask)


class KeyedGAT(TrainableGAT):
  """``TrainableGAT`` (same constructor, parameters, initialisation, ``state_dict`` and checkpoints) that
  also trains with ``dropout > 0``, as the reference does: at every channel of every layer the input, the
  attention weights and Wh are dropped with p = ``dropout`` (model/gat.py:149-163).  The masks are drawn on
  the device from a key, so the step can be captured in a CUDA graph (``train.GraphedStep``, padded or
  ``sparse=True``): each channel's input mask inside the projection (``lnb_gat_dropout_project``, no masked
  copy of the input exists) and the other two inside the attention kernels (``lnb_gat_attention_dropout``);
  the adjoints draw them again.

  The key is an int64 tensor (seed, counter) of shape (2,); the rule is in the C header.  In training mode
  with dropout > 0, ``forward(..., dropout_key=None)`` reads the module's own key, the non-persistent buffer
  ``dropout_key`` initialised to (config.seed or 0, 0), and advances its counter on the device after the
  forward: eager calls and ``GraphedStep`` replays each draw new masks.  An explicit ``dropout_key`` is used
  as given and nothing is advanced.  The records entries take ``batch['dropout_key']`` when present, otherwise
  the module's key.  That forward is the dropout formulation with or without autograd (the reference's
  training-mode semantics).  In eval mode, or with dropout 0, this is ``TrainableGAT``: same code, same bits.
  Under ``nn.DataParallel`` the replicas share the module's key, so each replica draws the same masks for
  its own slice of the batch: pass distinct keys per replica if that matters.  The reference's torch
  dropout draws are not reproduced; the distribution is the same."""

  def __init__(self, config):
    super(KeyedGAT, self).__init__(config)
    seed = int(getattr(config, 'seed', 0) or 0)
    self.register_buffer('dropout_key', torch.tensor([seed, 0], dtype=torch.int64), persistent=False)

  def _drops(self):
    return self.training and self.dropout > 0.0

  def forward(self, node_feat, L, label=None, mask=None, dropout_key=None):
    """node_feat: long B x N; L: float B x N x N x (E+1) (data.gat_bias); label: B x P; mask: B x N;
    dropout_key: int64 (2,) (seed, counter), default the module's own key (advanced after the forward)."""
    if dropout_key is not None:
      ops.check_dropout_key('KeyedGAT', dropout_key)
    if not self._drops():
      return super(KeyedGAT, self).forward(node_feat, L, label, mask)
    dev = self._device()
    score = self._dropout_train(self._to(dev, node_feat), self._to(dev, L), self._to(dev, mask), dropout_key)
    return self._finish(score, self._to(dev, label))

  def _dropout_train(self, node_ids, bias, mask, dropout_key):
    from ..train import gat_train
    own = dropout_key is None
    key = self._to(node_ids.device, self.dropout_key if own else dropout_key)
    score = gat_train(self, node_ids, bias, mask, dropout_key=key)
    if own:
      with torch.no_grad():
        self.dropout_key[1:].add_(1)
    return score

  def _sparse_inputs(self, batch):
    inputs, impl, key = super(KeyedGAT, self)._sparse_inputs(batch)
    dk = batch.get('dropout_key')
    if dk is None:
      return inputs, impl, key
    ops.check_dropout_key('KeyedGAT', dk)
    return inputs + (dk,), lambda *a: impl(*a[:-1]), key        # inference draws no mask: the key rides along

  def _train_records(self, recs, dropout_key=None):
    if not self._drops():
      return super(KeyedGAT, self)._train_records(recs)
    _, node_ids, mask, _, _ = self._prepare_records(recs)
    bias = ops.gat_bias_sparse(recs.sizes, recs.edge_ptr, recs.edges, recs.N, self.num_edgetype + 1)
    return self._dropout_train(node_ids, bias, mask, dropout_key)
