"""Drop-in for the reference ``model.LanczosNet`` (model/lanczos_net.py:13-199): same
constructor, parameter names and ``forward(node_feat, L, D, V, label=None, mask=None)``;
the forward runs in hand-written sm_90a CUDA (no CPU path)."""
import torch.nn as nn

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
