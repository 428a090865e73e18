"""Drop-in for the reference ``model.LanczosNet`` (model/lanczos_net.py:13-199): same
constructor, parameter names and ``forward(node_feat, L, D, V, label=None, mask=None)``;
the forward runs in hand-written sm_90a CUDA (no CPU path)."""
import torch
import torch.nn as nn

from .. import data as data_mod
from .. import ops
from ._common import Ragged, SpectralNetBase

__all__ = ['LanczosNet']


class LanczosNet(SpectralNetBase):

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

  def _sparse_inputs(self, batch):
    """A sparse batch here also carries the Ritz pairs of the real nodes (``V_rows``, ``D``), or only K
    (``data.sparse_collate(..., eigs=False)``): the reference's eigenpairs then come from one
    lnb_graph_eigs_sparse launch in front of the batch construction, inside the same CUDA graph (no host
    eigh, no eigenvector bytes on the bus).  A packed batch (data.pack_sparse) crosses PCIe as ONE copy
    of exactly the bytes present."""
    if 'blob' in batch:
      B, N, K = int(batch['B']), int(batch['N']), int(batch['K'])
      cap = data_mod.packed_offsets(B, K)[4] + 16 * 3 + 4 * B * N + 4 * B * N * K + 4 * B * N * 4
      blob = batch['blob']
      return ((Ragged(blob, max(cap, int(blob.shape[0]))),),
              lambda b_: self._forward_packed_impl(B, N, K, b_), ('packed', B, N, K))
    N, B = int(batch['N']), int(batch['sizes'].shape[0])
    if 'V_rows' not in batch and 'D' not in batch:
      K = int(batch['K'])
      inputs = (batch['sizes'], batch['node_ptr'], Ragged(batch['node_feat'], B * N), batch['edge_ptr'],
                Ragged(batch['edges']))
      return inputs, lambda *a: self._forward_sparse_eigs_impl(N, K, *a), ('sparse_eigs', N, K)
    inputs = (batch['sizes'], batch['node_ptr'], Ragged(batch['node_feat'], B * N), batch['edge_ptr'],
              Ragged(batch['edges']), Ragged(batch['V_rows'], B * N), batch['D'])
    return inputs, lambda *a: self._forward_sparse_impl(N, *a), ('sparse', N)

  def _train_records(self, recs, V_rows=None, D=None):
    # records without eigenpairs get them from lnb_graph_eigs_sparse, as data (no gradient flows to them)
    from ..train import ell_operator, ritz_stack_train
    if V_rows is None:
      D, V_rows, _ = ops.graph_eigs_sparse(recs.sizes, recs.node_ptr, recs.edge_ptr, recs.edges, recs.N, recs.K,
                                           num_edgetype=self.num_edgetype, rows=recs.node_feat.shape[0])
    prep, node_ids, mask, V, _ = ops.graph_prepare_sparse(
        recs.sizes, recs.node_ptr, recs.node_feat, recs.edge_ptr, recs.edges, V_rows.float().contiguous(), recs.N,
        self.num_edgetype + 1)
    return ritz_stack_train(self, None, node_ids, ell_operator(prep), D, V, mask)

  def _forward_packed_impl(self, B, N, K, blob):
    E1 = self.num_edgetype + 1
    dense = not self._sparse_stack_ok(N, E1, K)
    off_D = data_mod.packed_offsets(B, K)[3]
    D = blob[off_D:off_D + 4 * B * K].view(torch.float32).reshape(B, K)     # fixed address in the buffer
    prep, node_ids, mask, V, L = ops.graph_prepare_sparse_packed(
        blob, B, N, E1, K, binarize=getattr(self, '_binarize_operators', False), want_dense=dense)
    return self._ritz_conv_stack(None, node_ids, L, D, V, mask, prep=prep, dims_hint=(N, E1))

  def _forward_sparse_impl(self, N, sizes, node_ptr, node_feat, edge_ptr, edges, V_rows, D):
    E1 = self.num_edgetype + 1
    K = V_rows.shape[1]
    dense = not self._sparse_stack_ok(N, E1, K)
    prep, node_ids, mask, V, L = ops.graph_prepare_sparse(
        sizes, node_ptr, node_feat, edge_ptr, edges, V_rows, N, E1,
        binarize=getattr(self, '_binarize_operators', False), want_dense=dense, defer_tiles=True)
    return self._ritz_conv_stack(None, node_ids, L, D.float().contiguous(), V, mask, prep=prep,
                                 dims_hint=(N, E1))

  def _forward_sparse_eigs_impl(self, N, K, sizes, node_ptr, node_feat, edge_ptr, edges):
    # V_rows has node_feat's rows (the static capacity under graph replay); rows past node_ptr[B] are
    # written by nobody and read by nobody
    D, V_rows, _ = ops.graph_eigs_sparse(sizes, node_ptr, edge_ptr, edges, N, K,
                                         num_edgetype=self.num_edgetype, rows=node_feat.shape[0])
    return self._forward_sparse_impl(N, sizes, node_ptr, node_feat, edge_ptr, edges, V_rows, D)
