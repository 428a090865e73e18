"""Drop-in for the reference ``model.GGNN`` (model/ggnn.py:10-197): gated graph neural network over the
bond channels.  Same constructor fields, parameter names, registration and initialisation order (so
``torch.manual_seed(s)`` gives the reference's initial weights and its checkpoints load by name), and the
same ``forward(node_feat, L, label=None, mask=None)``.

Per propagation step the reference runs E+1 message MLPs, E+1 bmm's against the binarised (and, for
``avg``, row-normalised) operators and a GRUCell (model/ggnn.py:143-171).  Here a step is three launches:
  * ``linear_tf32x3`` of h against the E+1 first message layers stacked into one [(E+1)*128, D] matrix
    (+ bias, ReLU);
  * ``linear_tf32x3_grouped`` for the E+1 second layers (block-diagonal), giving M [B*N, (E+1)*D];
  * ``lnb_ggnn_update``: the aggregation A_e M_e, gathered through the ELL rows of the 0/1 operators in
    the producer warps of a 3xTF32 wgmma GEMM against the re-laid-out GRU weights
    (``gru_gate_matrix``), with the GRU cell in its epilogue; h' goes to the other of two state buffers.
With the embedding gather, ``input_func``, one ``graph_prepare`` (binarising) and the readout, the whole
forward is captured as one CUDA graph.  The operators are read, never modified.

Differences from the reference, on purpose:
  * the reference binarises the caller's ``L`` in place (``L[L != 0] = 1``, :137); this module leaves it
    unchanged (the kernels read only its non-zero pattern);
  * ``update_func: MLP`` builds the same parameters as the reference, and the forward raises the
    reference's ``TypeError`` (nn.Sequential called with two arguments, :168) before touching the device;
  * the GRU gate pre-activations are one dot product over [messages | h] plus b_ih + b_hh instead of
    (W_i x + b_i) + (W_h h + b_h): the same sum in another order.
``update_func: RNN`` (relu RNNCell), shapes outside ``lnb_ggnn_update`` and ``input_dim % 4 != 0`` run the
training formulation of lanczosnetwork_b200.train under no_grad."""
import torch
import torch.nn as nn

from ._common import SpectralNetBase, init_cell, init_linears, loss_function
from .. import ops

__all__ = ['GGNN']

MSG_HIDDEN = 128                               # width of the message MLPs, fixed in the reference (:59-61)


def gru_gate_matrix(weight_ih, weight_hh, bias_ih, bias_hh):
  """The GRUCell as one GEMM over [x | h] (layout of lnb_ggnn_update): returns W [4D, Din + D] and
  b [4D] whose row (u // 4) * 16 + g * 4 + u % 4 is gate g of hidden unit u, with the gate blocks
  r = [W_ir | W_hr], z = [W_iz | W_hz], n_in = [W_in | 0], n_h = [0 | W_hn] and biases b_ir + b_hr,
  b_iz + b_hz, b_in, b_hn.  Works on any device."""
  D, Din = weight_hh.shape[1], weight_ih.shape[1]
  wi, wh = weight_ih.reshape(3, D, Din), weight_hh.reshape(3, D, D)
  W = weight_ih.new_zeros((4, D, Din + D))
  W[0, :, :Din], W[0, :, Din:] = wi[0], wh[0]
  W[1, :, :Din], W[1, :, Din:] = wi[1], wh[1]
  W[2, :, :Din] = wi[2]
  W[3, :, Din:] = wh[2]
  bi, bh = bias_ih.reshape(3, D), bias_hh.reshape(3, D)
  b = torch.stack([bi[0] + bh[0], bi[1] + bh[1], bi[2], bh[2]])
  W = W.reshape(4, D // 4, 4, Din + D).permute(1, 0, 2, 3).reshape(4 * D, Din + D).contiguous()
  b = b.reshape(4, D // 4, 4).permute(1, 0, 2).reshape(4 * D).contiguous()
  return W, b


def ggnn_step_params(cache, msg_func, cell):
  """Stacked message weights and the re-laid-out gate matrix of one GGNN propagation step (E1 message
  MLPs ``msg_func``, GRUCell ``cell``), split once per parameter version through ``cache``."""
  first = [seq[0] for seq in msg_func]
  second = [seq[2] for seq in msg_func]
  w1_hi, w1_lo, b1 = cache.split_stacked('msg_func.0', [l.weight for l in first], [l.bias for l in first])
  w2_hi, w2_lo, b2 = cache.split_stacked('msg_func.2', [l.weight for l in second], [l.bias for l in second])
  return (w1_hi, w1_lo, b1), (w2_hi, w2_lo, b2), cached_gates(cache, 'update_func.gates', cell)


def cached_gates(cache, name, cell):
  """(hi, lo, bias) of gru_gate_matrix of the GRUCell ``cell``, rebuilt through ``cache`` when its
  parameters change."""
  def build():
    W, b = gru_gate_matrix(cell.weight_ih.detach(), cell.weight_hh.detach(), cell.bias_ih.detach(),
                           cell.bias_hh.detach())
    return ops.split_tf32(W) + (b,)
  return cache.derived(name, [cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh], build)


def embed_input(model, node_feat, table):
  """h = input_func(table[node_feat]) [B*N, D] of GGNN / GPNN / MPNN: the embedding gather and one dense
  launch."""
  lin = model.input_func[0]
  w_hi, w_lo = model._wcache.split('input_func.0', lin.weight)
  x = ops.embedding_rows(node_feat.long().reshape(-1), table)
  return ops.linear_tf32x3(x, w_hi, w_lo, lin.bias)


def ggnn_step(h, prep, params, avg, out):
  """One GGNN propagation step in three launches (the E1 first message layers stacked, the grouped
  second layers, lnb_ggnn_update); ``params`` from ggnn_step_params, ``prep`` the binarised ELL rows.
  h' goes to ``out``, which must not alias h."""
  (w1_hi, w1_lo, b1), (w2_hi, w2_lo, b2), (g_hi, g_lo, g_b) = params
  E1 = prep[0].shape[1]
  hid = ops.linear_tf32x3(h, w1_hi, w1_lo, b1, relu=True)              # [B*N, E1*128]
  msg = ops.linear_tf32x3_grouped(hid, w2_hi, w2_lo, b2, E1)           # [B*N, E1*D]
  return ops.ggnn_update(msg, h, prep, g_hi, g_lo, g_b, avg, out=out)


class GGNN(SpectralNetBase):

  def __init__(self, config):
    super(GGNN, self).__init__()
    m = config.model
    self._setup_fields(config, config.dataset.num_bond_type)
    self.num_prop = m.num_prop
    self.aggregate_type = m.aggregate_type
    self.update_func_name = m.update_func
    assert self.num_layer == 1, "not implemented"
    assert self.aggregate_type in ['avg', 'sum'], 'not implemented'
    E1, D = self.num_edgetype + 1, self.hidden_dim

    self.embedding = nn.Embedding(self.num_atom, self.input_dim)
    if m.update_func == 'RNN':
      self.update_func = nn.RNNCell(input_size=D * E1, hidden_size=D, nonlinearity='relu')
    elif m.update_func == 'GRU':
      self.update_func = nn.GRUCell(input_size=D * E1, hidden_size=D)
    elif m.update_func == 'MLP':              # registered as in the reference; its forward raises
      self.update_func = nn.Sequential(nn.Linear(D * E1, D), nn.Tanh())
    if m.msg_func == 'MLP':
      self.msg_func = nn.ModuleList([
          nn.Sequential(nn.Linear(D, MSG_HIDDEN), nn.ReLU(), nn.Linear(MSG_HIDDEN, D)) for _ in range(E1)])
    else:
      self.msg_func = None
    self.att_func = nn.Sequential(nn.Linear(D, 1), nn.Sigmoid())
    self.input_func = nn.Sequential(nn.Linear(self.input_dim, D))
    self.output_func = nn.Sequential(nn.Linear(D, self.output_dim))
    self.loss_func = loss_function(m.loss)
    self._init_param()

  def _init_param(self):
    """The reference's order (model/ggnn.py:88-120): Xavier / zero bias for input_func, att_func and
    output_func (msg_func is a ModuleList, neither Sequential nor Linear, so it keeps PyTorch's default
    initialisation); then Xavier on weight_hh, weight_ih and zero biases of the GRU / RNN cell, or
    Xavier on the Linear of the MLP update."""
    init_linears([*self.input_func, *self.att_func, *self.output_func])
    if self.update_func_name in ('GRU', 'RNN'):
      init_cell(self.update_func)
    elif self.update_func_name == 'MLP':
      init_linears(self.update_func)

  def _param_device(self):
    return self.embedding.weight.device

  def forward(self, node_feat, L, label=None, mask=None):
    """
      node_feat: long B x N (atom ids); L: float B x N x N x (E+1) operators (only their non-zero
      pattern is read; L is not modified); label: B x P; mask: B x N (uint8 / bool / float).
      Returns score (B x P) or (score, loss).
    """
    self._check_runnable()
    return self._forward((node_feat, L, mask), label)

  def _check_runnable(self, N=None, E1=None):
    """The reference's errors of the configs its forward cannot run, before any launch."""
    if self.update_func_name == 'MLP':
      raise TypeError("forward() takes 2 positional arguments but 3 were given: update_func 'MLP' is an "
                      "nn.Sequential, which the reference calls with (messages, state) (model/ggnn.py:168)")
    if self.msg_func is None:
      raise UnboundLocalError("msg_func %r: the reference's propagation reads a message that is never "
                              "assigned (model/ggnn.py:147-154); only 'MLP' runs" % self.config.model.msg_func)

  def _train_impl(self, node_feat, L, mask):
    from ..train import ggnn_train
    return ggnn_train(self, node_feat, L, mask)

  def fused_supported(self, N, E1):
    """True when inference runs the three-launch step (GRU update, lnb_ggnn_update's shapes, an input
    width the dense kernel reads)."""
    return (self.update_func_name == 'GRU' and self.input_dim % 4 == 0 and
            self.update_func.weight_ih.shape[1] == E1 * self.hidden_dim and
            ops.ggnn_update_supported(N, self.hidden_dim, E1))

  def _step_params(self):
    return ggnn_step_params(self._wcache, self.msg_func, self.update_func)

  def _forward_impl(self, node_feat, L, mask):
    B, N = node_feat.shape
    E1 = L.shape[3]
    if not self.fused_supported(N, E1):
      return self._train_impl(node_feat, L, mask)        # RNN update / other shapes: the training formulation
    return self._propagate(node_feat, ops.graph_prepare(L, binarize=True), mask)

  def _forward_records(self, recs):
    fused = self.fused_supported(recs.N, self.num_edgetype + 1)
    prep, node_ids, mask, _, L = self._prepare_records(recs, binarize=True, want_dense=not fused)
    if not fused:
      return self._train_impl(node_ids, L, mask)
    return self._propagate(node_ids, prep, mask)

  def _train_records(self, recs):
    from ..train import ell_operator, ggnn_train
    prep, node_ids, mask, _, _ = self._prepare_records(recs, binarize=True)
    return ggnn_train(self, node_ids, ell_operator(prep), mask)

  def _propagate(self, node_feat, prep, mask):
    """The fused inference forward from the ELL rows of the 0/1 operators."""
    B, N = node_feat.shape
    D = self.hidden_dim
    h = embed_input(self, node_feat, self.embedding.weight)
    params = self._step_params()
    spare = torch.empty_like(h)
    avg = self.aggregate_type == 'avg'
    for _ in range(self.num_prop):
      h, spare = ggnn_step(h, prep, params, avg, out=spare), h
    head, att = self.output_func[0], self.att_func[0]
    return ops.readout(h.view(B, N, D), head.weight, head.bias, att.weight.reshape(-1), att.bias, mask)
