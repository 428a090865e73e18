"""Drop-in for the reference ``model.AdaLanczosNet`` (model/ada_lanczos_net.py:12-368): same
constructor, parameter names and ``forward(node_feat, L, label=None, mask=None)``.

Per batch it builds its own operator: Gaussian-kernel Laplacian from the learned embeddings
(:101-137), K-step Lanczos with double re-orthogonalisation (:139-247), the learned filter on
powers of the tridiagonal T (:250-286).  GPU mapping: one fused Laplacian kernel (no
B x N^2 x D pair tensors), one warp/CTA-per-graph Lanczos kernel (lnb_lanczos_ritz without the QL stage), T^p computed once per
forward instead of once per layer (the reference recomputes 30 bmm per layer, :266-270),
the 4096-wide MLP on the wgmma 3xTF32 kernel, and Q G (Q^T X) applied in factored form.
"""
import torch
import torch.nn as nn

from .. import ops
from ..spectral_conv import GraphContext, dense, graph_conv_layer
from ._common import SpectralNetBase

__all__ = ['AdaLanczosNet']


class AdaLanczosNet(SpectralNetBase):

  def __init__(self, config):
    super(AdaLanczosNet, self).__init__()
    K = config.model.num_eig_vec
    S = len(config.model.long_diffusion_dist)
    self._setup_common(config, config.dataset.num_bond_type, K * K * S, 4096)
    # The reference tests hasattr on the TOP-LEVEL config (ada_lanczos_net.py:35-38), so with
    # the shipped yaml both flags are always True; mirrored bit-for-bit.
    self.use_reorthogonalization = config.model.use_reorthogonalization if hasattr(
        config, 'use_reorthogonalization') else True
    self.use_power_iteration_cap = config.model.use_power_iteration_cap if hasattr(
        config, 'use_power_iteration_cap') else True
    if not self.use_reorthogonalization:
      raise NotImplementedError('the CUDA Lanczos kernel always re-orthogonalises '
                                '(the only behaviour reachable from the shipped configs)')
    self.input_dim = self.num_atom                    # ada_lanczos_net.py:40
    dims = self._build_layers()
    self.embedding = nn.Embedding(self.num_atom, self.input_dim)
    self._build_spectral_filter()
    self._build_head(dims)
    self._init_param()

  def forward(self, node_feat, L, label=None, mask=None):
    """
      node_feat: long B x N; L: float B x N x N x (E+1); label: B x P; mask: B x N.
      The Lanczos start vector is drawn exactly like the reference: torch.randn(B, N, 1) on
      the CPU generator (ada_lanczos_net.py:161), then copied to the device.
    """
    dev = self._device()
    B, N = node_feat.shape[0], node_feat.shape[1]
    if self._check_mode():
      q1 = torch.randn(B, N, 1)
      score = self._train_impl(self._to(dev, node_feat), self._to(dev, L), self._to(dev, mask), q1)
      return self._finish(score, self._to(dev, label))
    # drawn exactly like the reference (CPU generator, ada_lanczos_net.py:161); it enters the captured
    # CUDA graph as an input buffer
    q1 = torch.randn(B, N, 1) if self.num_scale_long > 0 else None
    score = self._graph_forward(self._forward_impl, (node_feat, L, mask, q1))
    return self._finish(score, self._to(dev, label))

  def _train_impl(self, node_feat, L, mask, q1):
    from ..train import ada_train
    return ada_train(self, node_feat, L, mask, q1)

  def _forward_impl(self, node_feat, L, mask, q1):
    dev = L.device
    L = L.float().contiguous()
    state = ops.embedding_rows(node_feat.long(), self.embedding.weight)
    B, N = state.shape[0], state.shape[1]
    K, S = self.num_eig_vec, self.num_scale_long

    Q = None
    powers = None
    if S > 0:
      Le = ops.gaussian_laplacian(state, L)
      # fused kernel, tridiagonalisation only (no QL / Ritz vectors for the learned filter)
      lz = ops.lanczos_ritz(Le, mask, q1, K, want_ritz=False)
      Q = lz['Q']
      powers = ops.tridiag_powers(lz['T'], self.long_diffusion_dist)     # [B,K,S,K], once
      self.last_lanczos = lz

    ctx = GraphContext(L, Q)
    for tt in range(self.num_layer):
      G = None
      if S > 0:
        if self.spectral_filter_kind == 'MLP':
          h = powers.reshape(B, K * S * K)
          seq = self.spectral_filter[tt]
          for i in (0, 2, 4, 6):
            h = dense(h, seq[i].weight, seq[i].bias, i != 6, self._wcache,
                      'spectral_filter.%d.%d' % (tt, i))
          G = ops.symmetrize_filters(h, K, S)                            # [B,S,K,K]
        else:
          G = powers.permute(0, 2, 1, 3).contiguous()
      state = graph_conv_layer(state, ctx, G, True, self.short_diffusion_dist, S,
                               self.filter[tt].weight, self.filter[tt].bias, self._wcache,
                               'filter.%d' % tt)
    return self._readout(state, mask)
