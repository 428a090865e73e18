"""Drop-in for the reference ``model.LanczosNetGeneral`` (model/lanczos_net_general.py:13-201):
LanczosNet with float node features instead of an atom embedding (:156) and the edge-type
count taken from ``config.dataset.num_edge_type`` (:24).  ``SparseLanczosNetGeneral`` adds the entries
from bond-list records with float feature rows."""

from ._common import RitzRecords, SpectralNetBase

__all__ = ['LanczosNetGeneral', 'SparseLanczosNetGeneral']


class LanczosNetGeneral(SpectralNetBase):

  def __init__(self, config):
    super(LanczosNetGeneral, self).__init__()
    self.node_emb_dim = config.dataset.node_emb_dim
    self.graph_emb_dim = config.dataset.graph_emb_dim
    self._setup_common(config, config.dataset.num_edge_type,
                       len(config.model.long_diffusion_dist), 128)
    dims = self._build_layers()
    assert self.input_dim == self.node_emb_dim      # lanczos_net_general.py:45-46
    assert self.output_dim == self.graph_emb_dim
    self._build_spectral_filter()
    self._build_head(dims)
    self._init_param()

  def forward(self, node_feat, L, D, V, label=None, mask=None):
    """
      node_feat: float B x N x D node features; L: B x N x N x (E+1); D: Ritz values B x K;
      V: Ritz vectors B x N x K; label: B x P; mask: B x N.
    """
    return self._forward((node_feat, L, D, V, mask), label)

  def _train_impl(self, node_feat, L, D, V, mask):
    from ..train import ritz_stack_train
    return ritz_stack_train(self, node_feat, None, L, D, V, mask)

  def _forward_impl(self, node_feat, L, D, V, mask):
    return self._ritz_conv_stack(node_feat.float().contiguous(), None, L.float().contiguous(),
                                 D.float().contiguous(), V.float().contiguous(), mask)


class SparseLanczosNetGeneral(RitzRecords, LanczosNetGeneral):
  """LanczosNetGeneral that also runs and trains from bond-list records (``data.sparse_collate`` of
  ``prepare_graph`` records with float features: ``node_feat`` float32 [sum n, input_dim]).  Same
  constructor, parameters, initial weights and ``state_dict`` as LanczosNetGeneral, and the same
  ``forward``; it adds ``forward_sparse``, ``forward_sparse_train`` and ``GraphedStep(sparse=True)``.

  lnb_graph_prepare_sparse_features pads the feature rows into X and builds the ELL rows, mask and V on the
  device; records without eigenpairs (``eigs=False``, only K) get them from one lnb_graph_eigs_sparse launch
  in front of it.  Layer 0 (input width 10 in the config) is not a fused-stack shape, so the prepare kernel
  also writes the dense operators on the device for it, as ``forward`` reads them; they never cross PCIe.
  Scores from records with eigenpairs equal ``forward`` on ``data.collate`` of the same samples, bit for
  bit.

  Packed batches of float feature rows (``data.pack_sparse`` of such records, ``data.PackedMolecules`` of
  GraphData samples; header slot F = input_dim) are taken too, by ``forward_sparse`` and by
  ``GraphedStep(packed=True)`` with labels in the blob: one copy per step.  A blob with eigenpairs runs
  lnb_graph_prepare_sparse_features_packed on the blob in place; one without them, and every training step, is
  split by lnb_records_unpack_features first.  The scores are those of the same records.  A packed batch of atom
  ids raises NotImplementedError, one of another feature width ValueError."""

  _feature_records = True
