"""Drop-in for the reference ``model.LanczosNet`` (model/lanczos_net.py:13-199): same
constructor, parameter names and ``forward(node_feat, L, D, V, label=None, mask=None)``;
the forward runs in hand-written sm_90a CUDA (no CPU path)."""
import torch
import torch.nn as nn

from .. import data as data_mod
from .. import ops
from ._common import RitzRecords, SpectralNetBase

__all__ = ['LanczosNet']


class LanczosNet(RitzRecords, SpectralNetBase):

  def __init__(self, config):
    super(LanczosNet, self).__init__()
    self._setup_common(config, config.dataset.num_bond_type,
                       len(config.model.long_diffusion_dist), 128)
    dims = self._build_layers()
    self.embedding = nn.Embedding(self.num_atom, self.input_dim)
    self._build_spectral_filter()
    self._build_head(dims)
    self._init_param()

  def forward(self, node_feat, L, D, V, label=None, mask=None):
    """
      node_feat: long B x N (atom ids); L: float B x N x N x (E+1); D: Ritz values B x K;
      V: Ritz vectors B x N x K; label: B x P; mask: B x N (uint8 / bool / float).
      Returns score (B x P) or (score, loss) when label is given.
    """
    return self._forward((node_feat, L, D, V, mask), label)

  def _train_impl(self, node_feat, L, D, V, mask):
    from ..train import ritz_stack_train
    return ritz_stack_train(self, None, node_feat, L, D, V, mask)

  def _forward_impl(self, node_feat, L, D, V, mask):
    return self._ritz_conv_stack(None, node_feat.long(), L.float().contiguous(),
                                 D.float().contiguous(), V.float().contiguous(), mask)

  def _forward_packed_impl(self, B, N, K, blob):
    E1 = self.num_edgetype + 1
    dense = not self._sparse_stack_ok(N, E1, K)
    off_D = data_mod.packed_offsets(B, K).D
    D = blob[off_D:off_D + 4 * B * K].view(torch.float32).reshape(B, K)     # fixed address in the buffer
    prep, node_ids, mask, V, L = ops.graph_prepare_sparse_packed(
        blob, B, N, E1, K, binarize=getattr(self, '_binarize_operators', False), want_dense=dense)
    return self._ritz_conv_stack(None, node_ids, L, D, V, mask, prep=prep, dims_hint=(N, E1))
