"""Drop-in for the reference ``model.MPNN`` (model/mpnn.py:14-212, Gilmer et al. 2017): message passing
with an edge network or per-channel edge embeddings, a GRU update and the Set2Vec readout
(model/set2set.py:60-100).  Same constructor fields, parameter names, registration and initialisation
order (so ``torch.manual_seed(s)`` gives the reference's initial weights and its checkpoints load by
name), and the same ``forward(node_feat, L, label=None, mask=None)``.

The reference runs the 2D -> 64 -> D edge MLP on all N^2 node pairs of every channel and then multiplies
by the 0/1 operator.  Here, with receiver i, neighbour j and P_e = h W1a_e^T, Q_e = h W1b_e^T + b1_e (the
first edge layer split at the two halves of its input [h_j | h_i], model/mpnn.py:132-134,158-164), the
second layer moves out of the sum and W_ih folds into it (see csrc/mpnn_update.cu).  A step of
``msg_func: MLP`` is two launches:
  * ``linear_tf32x3`` of h against the first edge layers stacked per channel as [W1a_e ; W1b_e] -> PQ;
  * ``lnb_mpnn_update``: S_e[i] = w_i sum_j A_e[i,j] relu(P_e[j] + Q_e[i]) gathered in the producer warps
    of a 3xTF32 wgmma GEMM against the folded gate matrix, the GRU cell in its epilogue.
``msg_func: embedding`` runs ``linear_tf32x3`` of h against the stacked E_e^T (the message is h E_e) and
``lnb_ggnn_update``.  With the embedding gather, ``input_func``, one binarising ``graph_prepare`` and
``lnb_set2vec`` (the readout and ``output_func`` in one launch), the forward is 2 * num_prop + 5 launches,
captured as one CUDA graph.

Differences from the reference, on purpose:
  * the reference binarises the caller's ``L`` in place (``L[L != 0] = 1``, :125); this module leaves it
    unchanged (the kernels read only its non-zero pattern);
  * the edge network's second layer and the GRU input weights are applied as one folded product
    (F = [W_ih,e W2_e]_e | [W_ih,e b2_e]_e, formed in fp64 and rounded once), and the gate sums run in
    another order: the same function, fp32 rounding apart.
Shapes outside the kernels' envelopes and ``input_dim % 4 != 0`` run the training formulation of
lanczosnetwork_b200.train under no_grad."""
import torch
import torch.nn as nn

from ._common import SpectralNetBase, init_cell, init_linears, loss_function
from .ggnn import cached_gates, embed_input, gru_gate_matrix
from .. import ops

__all__ = ['MPNN']

EDGE_HIDDEN = ops.MPNN_EDGE_HIDDEN             # model/mpnn.py:60


class Set2SetLSTM(nn.Module):
  """model/set2set.py:8-57: four gates on [h | read], each a Linear(2D, D) + activation."""

  def __init__(self, hidden_dim):
    super(Set2SetLSTM, self).__init__()
    self.hidden_dim = hidden_dim
    self.forget_gate = nn.Sequential(nn.Linear(2 * hidden_dim, hidden_dim), nn.Sigmoid())
    self.input_gate = nn.Sequential(nn.Linear(2 * hidden_dim, hidden_dim), nn.Sigmoid())
    self.output_gate = nn.Sequential(nn.Linear(2 * hidden_dim, hidden_dim), nn.Sigmoid())
    self.memory_gate = nn.Sequential(nn.Linear(2 * hidden_dim, hidden_dim), nn.Tanh())
    for seq in self.gates():
      nn.init.xavier_uniform_(seq[0].weight.data)
      seq[0].bias.data.zero_()

  def gates(self):
    return (self.forget_gate, self.input_gate, self.output_gate, self.memory_gate)


class Set2Vec(nn.Module):
  """Parameters of model/set2set.py:60-77 (``W_1`` [D, D] is used as [in, out], ``W_2`` [D, 1]); the
  forward is ``lnb_set2vec`` (inference) or train.set2vec_train."""

  def __init__(self, element_dim, num_step_encoder):
    super(Set2Vec, self).__init__()
    self.element_dim = element_dim
    self.num_step_encoder = num_step_encoder
    self.LSTM = Set2SetLSTM(element_dim)
    self.W_1 = nn.Parameter(torch.ones(element_dim, element_dim))
    self.W_2 = nn.Parameter(torch.ones(element_dim, 1))
    nn.init.xavier_uniform_(self.W_1.data)
    nn.init.xavier_uniform_(self.W_2.data)


class MPNN(SpectralNetBase):

  def __init__(self, config):
    super(MPNN, self).__init__()
    m = config.model
    self._setup_fields(config, config.dataset.num_bond_type)
    self.num_prop = m.num_prop
    self.msg_func_name = m.msg_func
    self.num_step_set2vec = m.num_step_set2vec
    self.aggregate_type = m.aggregate_type
    assert self.num_layer == 1, 'not implemented'
    assert self.aggregate_type in ['avg', 'sum'], 'not implemented'
    E1, D = self.num_edgetype + 1, self.hidden_dim

    self.node_embedding = nn.Embedding(self.num_atom, self.input_dim)
    self.input_func = nn.Sequential(nn.Linear(self.input_dim, D))
    self.update_func = nn.GRUCell(input_size=D * E1, hidden_size=D)
    if m.msg_func == 'embedding':
      self.edge_embedding = nn.Embedding(E1, D ** 2)
    elif m.msg_func == 'MLP':
      self.edge_func = nn.ModuleList([
          nn.Sequential(nn.Linear(2 * D, EDGE_HIDDEN), nn.ReLU(), nn.Linear(EDGE_HIDDEN, D)) for _ in range(E1)])
    else:
      raise ValueError('Non-supported message function')
    self.att_func = Set2Vec(D, self.num_step_set2vec)
    self.output_func = nn.Sequential(nn.Linear(2 * D, self.output_dim))
    self.loss_func = loss_function(m.loss)
    self._init_param()

  def _init_param(self):
    """The reference's order (model/mpnn.py:85-108): Xavier / zero bias for input_func and output_func
    (att_func is a Set2Vec, neither Sequential nor Linear: it keeps the initialisation of its own
    constructor; the edge network keeps PyTorch's default), then Xavier on weight_hh, weight_ih and zero
    biases of the GRU."""
    init_linears([*self.input_func, *self.output_func])
    init_cell(self.update_func)

  def _param_device(self):
    return self.node_embedding.weight.device

  def forward(self, node_feat, L, label=None, mask=None):
    """
      node_feat: long B x N (atom ids); L: float B x N x N x (E+1) operators (only their non-zero
      pattern is read; L is not modified); label: B x P; mask: B x N (uint8 / bool / float; the nodes
      of each graph's Set2Vec set).  Returns score (B x P) or (score, loss).
    """
    return self._forward((node_feat, L, mask), label)

  def _train_impl(self, node_feat, L, mask):
    from ..train import mpnn_train
    return mpnn_train(self, node_feat, L, mask)

  def fused_supported(self, N, E1):
    """True when inference runs the kernels (the update kernel's shapes, lnb_set2vec's shapes, an input
    width the dense kernel reads)."""
    D = self.hidden_dim
    step_ok = (ops.mpnn_update_supported(N, D, E1) if self.msg_func_name == 'MLP'
               else ops.ggnn_update_supported(N, D, E1))
    return (self.input_dim % 4 == 0 and E1 == self.num_edgetype + 1 and step_ok and
            ops.set2vec_supported(N, D, self.output_dim))

  def _step_params(self):
    """Split weights of a propagation step, rebuilt once per parameter version: for ``MLP`` the stacked
    first edge layers [W1a_e ; W1b_e] with bias [0 ; b1_e], and the gate matrix of the folded
    F = [W_ih,e W2_e]_e | [W_ih,e b2_e]_e (fp64, rounded once; degree columns zero padded to 32); for
    ``embedding`` the stacked E_e^T and the GRU gate matrix."""
    cache, cell = self._wcache, self.update_func
    E1, D = self.num_edgetype + 1, self.hidden_dim
    if self.msg_func_name == 'embedding':
      emb = self.edge_embedding.weight
      e_hi, e_lo = cache.derived('edge_embedding.stacked', [emb], lambda: ops.split_tf32(
          emb.detach().view(E1, D, D).transpose(1, 2).reshape(E1 * D, D)))
      return (e_hi, e_lo, None), cached_gates(cache, 'update_func.gates', cell)
    first = [seq[0] for seq in self.edge_func]
    second = [seq[2] for seq in self.edge_func]

    def build_pq():
      W = torch.cat([torch.cat([l.weight.detach()[:, :D], l.weight.detach()[:, D:]], dim=0) for l in first])
      b = torch.cat([torch.cat([torch.zeros_like(l.bias.detach()), l.bias.detach()]) for l in first])
      return ops.split_tf32(W.contiguous()) + (b.contiguous(),)
    pq = cache.derived('edge_func.0.pq', [l.weight for l in first] + [l.bias for l in first], build_pq)

    def build_gates():
      w_ih = cell.weight_ih.detach().double().view(3 * D, E1, D)
      F = w_ih.new_zeros((3 * D, EDGE_HIDDEN * E1 + 32))
      for e, l in enumerate(second):
        F[:, e * EDGE_HIDDEN:(e + 1) * EDGE_HIDDEN] = w_ih[:, e, :] @ l.weight.detach().double()
        F[:, EDGE_HIDDEN * E1 + e] = w_ih[:, e, :] @ l.bias.detach().double()
      W, b = gru_gate_matrix(F.float(), cell.weight_hh.detach(), cell.bias_ih.detach(), cell.bias_hh.detach())
      return ops.split_tf32(W) + (b,)
    gru = [cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh]
    gates = cache.derived('update_func.mpnn_gates',
                          gru + [l.weight for l in second] + [l.bias for l in second], build_gates)
    return pq, gates

  def _set2vec_params(self):
    """[2D, 4D] transposed gate weights (forget, input, output, memory) and their biases."""
    lin = [seq[0] for seq in self.att_func.LSTM.gates()]
    return self._wcache.derived(
        'att_func.LSTM.gates', [l.weight for l in lin] + [l.bias for l in lin],
        lambda: (torch.cat([l.weight.detach() for l in lin], dim=0).t().contiguous(),
                 torch.cat([l.bias.detach() for l in lin]).contiguous()))

  def _forward_impl(self, node_feat, L, mask):
    B, N = node_feat.shape
    E1 = L.shape[3]
    if not self.fused_supported(N, E1):
      return self._train_impl(node_feat, L, mask)        # other shapes: the training formulation
    return self._propagate(node_feat, ops.graph_prepare(L, binarize=True), mask)

  def _forward_records(self, recs):
    fused = self.fused_supported(recs.N, self.num_edgetype + 1)
    prep, node_ids, mask, _, L = self._prepare_records(recs, binarize=True, want_dense=not fused)
    if not fused:
      return self._train_impl(node_ids, L, mask)
    return self._propagate(node_ids, prep, mask)

  def _train_records(self, recs):
    from ..train import ell_operator, mpnn_train
    prep, node_ids, mask, _, _ = self._prepare_records(recs, binarize=True)
    return mpnn_train(self, node_ids, ell_operator(prep), mask)

  def _propagate(self, node_feat, prep, mask):
    """The fused inference forward from the ELL rows of the 0/1 operators."""
    B, N = node_feat.shape
    D = self.hidden_dim
    h = embed_input(self, node_feat, self.node_embedding.weight)
    (m_hi, m_lo, m_b), (g_hi, g_lo, g_b) = self._step_params()
    spare = torch.empty_like(h)
    avg = self.aggregate_type == 'avg'
    step = ops.mpnn_update if self.msg_func_name == 'MLP' else ops.ggnn_update
    for _ in range(self.num_prop):
      msg = ops.linear_tf32x3(h, m_hi, m_lo, m_b)       # PQ [B*N, E1*128] or h E_e [B*N, E1*D]
      h, spare = step(msg, h, prep, g_hi, g_lo, g_b, avg, out=spare), h
    wg_t, bg = self._set2vec_params()
    s2v, head = self.att_func, self.output_func[0]
    return ops.set2vec(h.view(B, N, D), mask, wg_t, bg, s2v.W_1, s2v.W_2, head.weight, head.bias,
                       self.num_step_set2vec)
