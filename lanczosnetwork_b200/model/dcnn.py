"""Drop-in for the reference ``model.DCNN`` (model/dcnn.py:8-124) -- SURVEY 8(f3): the LanczosNet
layer with short diffusion scales only.  Per layer (:86-100): the edge-type products ``L_e X`` and
the powers ``L_0^k X`` for k in diffusion_dist (a chain of max(diffusion_dist) sparse products),
concatenated edges-first, Linear + ReLU; then the shared gated readout.  Same constructor,
parameter names and ``forward(node_feat, L, label=None, mask=None)``.

The power chain needs every row of the previous walk, so this model does not fit the one-launch
stack: per layer one ``lnb_operator_chain`` launch runs all max(diffusion_dist) steps with the
operator and the walk on chip (N <= 32; larger graphs fall back to one batched GEMM per step), one
batched GEMM does the edge types, and the Linear runs on the 3xTF32 wgmma dense layer; the whole
forward is one CUDA-graph replay."""
import torch
import torch.nn as nn

from ._common import SpectralNetBase
from ..data import check_dist
from ..spectral_conv import dense, graph_conv_layer_unfused
from .. import ops

__all__ = ['DCNN']


class DCNN(SpectralNetBase):

  def __init__(self, config):
    super(DCNN, self).__init__()
    m = config.model
    self._setup_fields(config, config.dataset.num_bond_type)
    self.diffusion_dist = m.diffusion_dist
    self.num_scale = len(self.diffusion_dist)
    self.max_dist = max(self.diffusion_dist)
    # in the vocabulary of the shared layer: short scales = diffusion_dist, no long scales
    self.short_diffusion_dist = check_dist(list(self.diffusion_dist))
    self.long_diffusion_dist = []
    self.num_scale_short, self.num_scale_long = self.num_scale, 0
    self.num_eig_vec = 0
    self.spectral_filter_kind = None
    dims = self._build_layers()          # Linear(dims[t] * (num_scale + E + 1), dims[t+1])
    self.embedding = nn.Embedding(self.num_atom, self.input_dim)
    self._build_head(dims)
    self._init_param()

  def forward(self, node_feat, L, label=None, mask=None):
    """
      node_feat: long B x N (atom ids); L: float B x N x N x (E+1); label: B x P;
      mask: B x N (uint8 / bool / float).  Returns score (B x P) or (score, loss).
    """
    return self._forward((node_feat, L, mask), label)

  def _train_impl(self, node_feat, L, mask):
    from ..train import dcnn_train
    return dcnn_train(self, node_feat, L, mask)

  def _layer_weight(self, t):
    """The reference concatenates edge types first and diffusion scales last (dcnn.py:98); the
    shared layer orders scales first: permute the weight columns once per parameter version."""
    w = self.filter[t].weight
    split = (self.num_edgetype + 1) * (w.shape[1] // (self.num_scale + self.num_edgetype + 1))
    return self._wcache.derived(
        'filter.%d.scales_first' % t, [w],
        lambda: (torch.cat([w.detach()[:, split:], w.detach()[:, :split]], dim=1).contiguous(),))[0]

  def _forward_impl(self, node_feat, L, mask):
    L = L.float().contiguous()
    B, N, _, E1 = L.shape
    state = ops.embedding_rows(node_feat.long(), self.embedding.weight)
    if (ops.operator_chain_supported(N, self.max_dist) and
        not ops.graph_messages_supported(N, 0, E1, 0, self.max_dist)):
      # reference column order: [edge types | diffusion scales] (dcnn.py:98), no weight permutation
      # scales are emitted in ascending step order like the reference loop (dcnn.py:88-92) and the
      # general-shape path, whatever the order of the config list
      steps = sorted(set(self.diffusion_dist))
      sel = [steps.index(s) if s in steps else -1 for s in range(1, self.max_dist + 1)]
      for t in range(self.num_layer):
        D = state.shape[2]
        CD = (E1 + self.num_scale) * D
        msg = torch.empty((B, N, CD), device=state.device, dtype=torch.float32)
        ops.bgemm(L, (N * N * E1, 1, N * E1, E1), state, (N * D, 0, D, 1), msg, (N * CD, D, CD, 1),
                  B, E1, N, D, N)
        ops.operator_chain(L, state, self.max_dist, sel, msg, E1)
        state = dense(msg.reshape(B * N, CD), self.filter[t].weight, self.filter[t].bias, True,
                      self._wcache, 'filter.%d' % t).reshape(B, N, -1)
      return self._readout(state, mask)
    for t in range(self.num_layer):
      state = graph_conv_layer_unfused(state, L, None, None, False, self.short_diffusion_dist, 0,
                                       self._layer_weight(t), self.filter[t].bias, self._wcache,
                                       'filter.%d.perm' % t)
    return self._readout(state, mask)

  def _forward_records(self, recs):
    _, node_ids, mask, _, L = self._prepare_records(recs, want_dense=True)
    return self._forward_impl(node_ids, L, mask)

  def _train_records(self, recs):
    from ..train import dcnn_train, ell_operator
    prep, node_ids, mask, _, _ = self._prepare_records(recs)
    return dcnn_train(self, node_ids, ell_operator(prep), mask)
