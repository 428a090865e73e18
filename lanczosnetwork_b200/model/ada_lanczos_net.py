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
from ._common import SparseRecords, SpectralNetBase

__all__ = ['AdaLanczosNet', 'KeyedAdaLanczosNet']


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
      # ascending powers, the order of the reference's T_list (ada_lanczos_net.py:266-268) whatever
      # the order of the config list
      powers = ops.tridiag_powers(lz['T'], sorted(self.long_diffusion_dist))   # [B,K,S,K], once
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


class KeyedAdaLanczosNet(AdaLanczosNet):
  """``AdaLanczosNet`` (same constructor, parameters, initialisation and ``state_dict``; construction
  consumes the same CPU random numbers) whose Lanczos start vector is drawn on the device from a key, so
  that it can be captured in a CUDA graph (``train.GraphedStep``, padded or ``sparse=True``) and run or
  trained from the bond-list records of data.sparse_collate (``forward_sparse``, ``forward_sparse_train``).

  The key is an int64 tensor (seed, counter) of shape (2,); ``ops.ada_start_vector(key, B, N)`` draws q1
  [B, N], one standard normal per (graph, padded node), from Philox4x32-10 (the rule is in the C header).
  ``forward(..., start_key=None)`` reads the module's own key, the non-persistent buffer ``start_key``
  initialised to (config.seed or 0, 0), and advances its counter on the device after each draw: eager
  calls, replays of a captured inference graph and ``GraphedStep`` replays each draw a new vector.  An
  explicit ``start_key`` is used as given and nothing is advanced.  The records entries take the key as
  ``batch['start_key']`` (required).  Under ``nn.DataParallel`` the replicas share the module's key, so each
  replica draws the same vectors for its own slice of the batch: pass distinct keys per replica if that
  matters.

  Contract: the scores of ``forward_sparse`` equal, bit for bit, those of the padded ``_forward_impl`` on
  data.collate(..., num_nodes=N) with q1 = ops.ada_start_vector(start_key, B, N), and
  ``forward_sparse_train`` computes this class's padded training formulation on the same q1.  The
  reference's torch.randn draws are not reproduced; the distribution is the same.  The training
  formulation is AdaLanczosNet's, except that the Lanczos recurrence runs on lnb_lanczos_tridiag_train and its
  adjoint lnb_lanczos_tridiag_backward (N <= 128, K <= 64), and the powers of T on lnb_tridiag_powers and its
  adjoint (when K and the powers fit that kernel), one launch each, instead of chains of GEMMs; outside those
  envelopes the GEMM chains of AdaLanczosNet run."""

  def __init__(self, config):
    super(KeyedAdaLanczosNet, self).__init__(config)
    seed = int(getattr(config, 'seed', 0) or 0)
    self.register_buffer('start_key', torch.tensor([seed, 0], dtype=torch.int64), persistent=False)

  def forward(self, node_feat, L, label=None, mask=None, start_key=None):
    """node_feat: long B x N; L: float B x N x N x (E+1); label: B x P; mask: B x N; start_key: int64 (2,)
    (seed, counter), default the module's own key (advanced after the draw)."""
    own = start_key is None
    key = self.start_key if own else start_key
    ops.check_start_key('KeyedAdaLanczosNet', key)
    dev = self._device()
    if self._check_mode():
      q1 = ops.ada_start_vector(self._to(dev, key), node_feat.shape[0], node_feat.shape[1])
      score = self._train_impl(self._to(dev, node_feat), self._to(dev, L), self._to(dev, mask), q1)
    else:
      score = self._graph_forward(self._keyed_impl, (node_feat, L, mask, key))
    if own:
      with torch.no_grad():
        self.start_key[1:].add_(1)
    return self._finish(score, self._to(dev, label))

  def _keyed_impl(self, node_feat, L, mask, key):
    q1 = ops.ada_start_vector(key, node_feat.shape[0], node_feat.shape[1])
    return self._forward_impl(node_feat, L, mask, q1)

  def _train_impl(self, node_feat, L, mask, q1):
    from ..train import ada_train, lanczos_tridiag, tridiag_powers
    K = self.num_eig_vec
    fits = ops.tridiag_powers_backward_supported(K, sorted(self.long_diffusion_dist) or [1])
    return ada_train(self, node_feat, L, mask, q1, powers_fn=tridiag_powers if fits else None,
                     lanczos_fn=lanczos_tridiag if ops.lanczos_tridiag_train_supported(L.shape[1], K) else None)

  def _sparse_inputs(self, batch):
    key = batch.get('start_key') if isinstance(batch, dict) else None
    if key is None:
      raise ValueError("KeyedAdaLanczosNet: the batch lacks 'start_key', the int64 (seed, counter) tensor of "
                       "the Lanczos start vector")
    ops.check_start_key('KeyedAdaLanczosNet', key)
    if 'blob' in batch:
      raise NotImplementedError('KeyedAdaLanczosNet takes data.sparse_collate records, not packed batches')
    inputs, _, _ = super(KeyedAdaLanczosNet, self)._sparse_inputs(batch)
    N = int(batch['N'])
    return (inputs + (key,), lambda *a: self._forward_records(SparseRecords(*a[:5], N=N), a[5]),
            ('keyed', N))

  def _takes_packed_training(self, batch):
    return False                                   # packed batches are refused (_sparse_inputs)

  def _records_inputs(self, recs, key):
    """node ids, dense operators and mask of the records (lnb_graph_prepare_sparse: the unfused conv
    layers read the dense L) and the start vector of ``key``."""
    _, node_ids, mask, _, L = self._prepare_records(recs, want_dense=True)
    return node_ids, L, mask, ops.ada_start_vector(key, node_ids.shape[0], recs.N)

  def _forward_records(self, recs, key):
    return self._forward_impl(*self._records_inputs(recs, key))

  def _train_records(self, recs, key):
    return self._train_impl(*self._records_inputs(recs, key))
