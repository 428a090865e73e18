"""Drop-in for the reference ``model.ChebyNet`` (model/cheby_net.py:8-124) -- SURVEY 8(f3).
Per layer (:86-100): the Chebyshev chain s_0 = L_0 X, s_k = 2 L_0 s_{k-1} - s_{k-2} (with
s_{-1} = X; k < polynomial_order), the products L_e X of the bond-type channels e >= 1, concatenated
as [edges | s_0 .. s_{order-1} | X], Linear + ReLU; then the shared gated readout.  Same constructor,
parameter names and ``forward(node_feat, L, label=None, mask=None)``.

Every piece is written straight into its column block of the message matrix by the strided
batched GEMM (the recurrence uses its alpha / beta-addend form), the Linear runs on the 3xTF32
wgmma dense layer; the whole forward is one CUDA-graph replay."""
import torch
import torch.nn as nn

from ._common import SpectralNetBase
from ..spectral_conv import dense
from .. import ops

__all__ = ['ChebyNet']


class ChebyNet(SpectralNetBase):

  def __init__(self, config):
    super(ChebyNet, self).__init__()
    self._setup_fields(config, config.dataset.num_bond_type)
    self.polynomial_order = config.model.polynomial_order
    self.short_diffusion_dist, self.long_diffusion_dist = [], []
    self.num_scale_short = self.num_scale_long = 0
    self.num_eig_vec = 0
    self.spectral_filter_kind = None
    dims = [self.input_dim] + list(self.hidden_dim) + [self.output_dim]
    C = self.polynomial_order + self.num_edgetype + 1
    self.filter = nn.ModuleList(
        [nn.Linear(dims[t] * C, dims[t + 1]) for t in range(self.num_layer)] +
        [nn.Linear(dims[-2], dims[-1])])
    self.embedding = nn.Embedding(self.num_atom, self.input_dim)
    self._build_head(dims)
    self._init_param()

  def forward(self, node_feat, L, label=None, mask=None):
    """
      node_feat: long B x N (atom ids); L: float B x N x N x (E+1) (channel 0: the rescaled
      simple-graph operator); label: B x P; mask: B x N.  Returns score or (score, loss).
    """
    return self._forward((node_feat, L, mask), label)

  def _train_impl(self, node_feat, L, mask):
    from ..train import cheby_train
    return cheby_train(self, node_feat, L, mask)

  def _forward_impl(self, node_feat, L, mask):
    L = L.float().contiguous()
    B, N, _, E1 = L.shape
    E, order = self.num_edgetype, self.polynomial_order
    state = ops.embedding_rows(node_feat.long(), self.embedding.weight)
    l0 = (N * N * E1, 0, N * E1, E1)                       # channel 0 of the operators, in place
    for t in range(self.num_layer):
      D = state.shape[2]
      C = E + order + 1
      CD = C * D
      msg = torch.empty((B, N, CD), device=state.device, dtype=torch.float32)
      blk = (N * CD, 0, CD, 1)                             # one column block of msg
      x_str = (N * D, 0, D, 1)
      # bond-type channels e = 1..E -> column blocks 0..E-1 (cheby_net.py:95-97)
      ops.bgemm(L, (N * N * E1, 1, N * E1, E1), state, x_str, msg, (N * CD, D, CD, 1),
                B, E, N, D, N, a_off=1)
      # s_0 = L_0 X (:90), then s_k = 2 L_0 s_{k-1} - s_{k-2} with s_{-1} = X (:91-93)
      if ops.operator_chain_supported(N, order):             # the whole chain in one launch
        ops.operator_chain(L, state, order, list(range(order)), msg, E, chebyshev=True)
      else:
        ops.bgemm(L, l0, state, x_str, msg, blk, B, 1, N, D, N, c_off=E * D)
      for k in range(1, order if not ops.operator_chain_supported(N, order) else 0):
        prev2 = (state, x_str, 0) if k == 1 else (msg, blk, (E + k - 2) * D)
        ops.bgemm(L, l0, msg, blk, msg, blk, B, 1, N, D, N, b_off=(E + k - 1) * D,
                  c_off=(E + k) * D, alpha=2.0, addend=prev2[0], add_str=(prev2[1][0], 0, prev2[1][2], 1),
                  add_off=prev2[2], beta=-1.0)
      msg[:, :, (E + order) * D:].copy_(state)             # the trailing X block (:89, :99)
      state = dense(msg.reshape(B * N, CD), self.filter[t].weight, self.filter[t].bias, True,
                    self._wcache, 'filter.%d' % t).reshape(B, N, -1)
    return self._readout(state, mask)

  def _forward_records(self, recs):
    _, node_ids, mask, _, L = self._prepare_records(recs, want_dense=True)
    return self._forward_impl(node_ids, L, mask)

  def _train_records(self, recs):
    from ..train import cheby_train, ell_operator
    prep, node_ids, mask, _, _ = self._prepare_records(recs)
    return cheby_train(self, node_ids, ell_operator(prep), mask)
