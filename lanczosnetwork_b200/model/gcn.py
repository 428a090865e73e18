"""Drop-in for the reference ``model.GCN`` (model/gcn.py:8-119) -- SURVEY 8(f3): the sibling model
whose layer is the edge-type part of the LanczosNet layer (``msg = [L_e X]_e``, Linear, ReLU;
model/gcn.py:84-92) followed by the same gated readout (:95-110).  Same constructor, parameter
names and ``forward(node_feat, L, label=None, mask=None)``; the forward is ONE launch of the
fused convolution-stack kernel with no long scales (embedding gather + all layers + readout)."""
import torch
import torch.nn as nn

from ._common import SpectralNetBase

__all__ = ['GCN', 'GCNFP']


class GCN(SpectralNetBase):

  def __init__(self, config):
    super(GCN, self).__init__()
    self._setup_fields(config, config.dataset.num_bond_type)
    # no diffusion scales: the message is the E+1 edge-type products only
    self.short_diffusion_dist, self.long_diffusion_dist = [], []
    self.num_scale_short = self.num_scale_long = 0
    self.num_eig_vec = 0
    self.spectral_filter_kind = None
    dims = self._build_layers()
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
    from ..train import ritz_stack_train
    if getattr(self, '_binarize_operators', False):
      L = (L != 0).to(torch.float32)                 # model/gcnfp.py:83
    return ritz_stack_train(self, None, node_feat, L, None, None, mask)

  def _forward_impl(self, node_feat, L, mask):
    L = L.float().contiguous()
    B, N = node_feat.shape
    # no Ritz vectors: an all-zero block makes lnb_graph_prepare take the extents from L alone
    V = torch.zeros((B, N, 4), device=L.device, dtype=torch.float32)
    return self._ritz_conv_stack(None, node_feat.long(), L, None, V, mask)

  def _forward_records(self, recs):
    # the dense operators only when a layer falls off the stack kernel
    E1 = self.num_edgetype + 1
    prep, node_ids, mask, V, L = self._prepare_records(
        recs, binarize=getattr(self, '_binarize_operators', False),
        want_dense=not self._sparse_stack_ok(recs.N, E1, 4))
    return self._ritz_conv_stack(None, node_ids, L, None, V, mask, prep=prep, dims_hint=(recs.N, E1))

  def _train_records(self, recs):
    from ..train import ell_operator, ritz_stack_train
    prep, node_ids, mask, _, _ = self._prepare_records(recs, binarize=getattr(self, '_binarize_operators', False))
    return ritz_stack_train(self, None, node_ids, ell_operator(prep), None, None, mask)


class GCNFP(GCN):
  """Drop-in for the reference ``model.GCNFP`` (model/gcnfp.py:8-125): GCN on the non-zero pattern
  of the operators (``L[L != 0] = 1.0``, :83).  The 0/1 values are produced while the operators are
  compressed (lnb_graph_prepare flag), so the dense tensor is never rewritten -- unlike the
  reference, the caller's ``L`` is left untouched."""
  _binarize_operators = True
