"""Online (D, V) provider: Ritz pairs of the simple-graph operator computed on the GPU by the fused
Lanczos -> QL -> Ritz-vector kernel, in place of the offline fp64 ``eigh`` of the reference's
preprocessing (utils/data_helper.py:169-226 called from dataset/get_qm8_data.py:63-83, truncated /
padded to K at collate, dataset/qm8.py:265-291).

This is SURVEY 8(f4) and the paper's actual algorithm; it is a MODEL-INPUT CHANGE, never "reference
MAE": K Lanczos steps from one start vector span a Krylov space, so

  * a graph with n_b <= K real nodes and simple eigenvalues gets all its eigenpairs (to fp32
    rounding) -- but ordered / signed by QL, and the reference's (D, V) are only defined up to sign
    and to rotations inside degenerate eigenspaces anyway;
  * a repeated eigenvalue (symmetric molecules) contributes ONE Ritz vector (the projection of the
    start vector onto its eigenspace), so fewer than min(n_b, K) non-zero pairs come back where
    ``eigh`` returns an arbitrary basis of the eigenspace;
  * a graph with n_b > K gets K Ritz pairs approximating the extremal part of the spectrum, not
    the exact top-K by |lambda|.

``tools/study_online_eigs.py`` measures all three effects and what they do to LanczosNet's scores
(profiles/r2_online_eigs_study.md).

``exact_eigenpairs`` is the other provider: an fp64 Householder + QL eigensolver on the device
(lnb_sym_eigs) that reproduces the reference's preprocessing itself -- every eigenpair, the top K by
|lambda| in the reference's order -- so a checkpoint trained on the reference's inputs sees the same
inputs.

``spectral_partition`` is GPNN's graph partition (the collate's spectral clustering and partition
operators) for loaders that hand the model its operators themselves.
"""
import torch

from . import ops

__all__ = ['online_ritz_pairs', 'exact_eigenpairs', 'spectral_partition']


def online_ritz_pairs(L, mask, num_eigs, q1=None, generator=None):
  """(D [B,K], V [B,N,K], info) from channel 0 of the padded operator tensor L [B,N,N,E+1]
  (or a [B,N,N] operator), ready for ``LanczosNet.forward(node_feat, L, D, V, mask=mask)``.

  q1: start vectors [B,N] (device); default: standard normal draws from ``generator`` on the
  operator's device (masked and normalised by the kernel like model/ada_lanczos_net.py:159-167).
  info: dict(idx [B] retained Krylov directions, status [B] kernel status bits)."""
  A = L[..., 0] if L.dim() == 4 else L
  A = A.float().contiguous()
  B, N = A.shape[0], A.shape[1]
  if q1 is None:
    q1 = torch.randn(B, N, device=A.device, generator=generator)
  out = ops.lanczos_ritz(A, mask, q1, int(num_eigs), want_T=False, want_Q=False, proper=True)
  return out['theta'], out['V'], {'idx': out['idx'], 'status': out['status']}


def exact_eigenpairs(L, sizes_or_mask, num_eigs):
  """(D [B,K], V [B,N,K], info) from channel 0 of the padded operator tensor L [B,N,N,E+1] (or a
  [B,N,N] operator), ready for ``LanczosNet.forward`` / ``LanczosNetGeneral.forward``.

  Unlike ``online_ritz_pairs`` this REPRODUCES the reference's preprocessing (dense fp64 eigh,
  utils/data_helper.py:169-226, truncated / zero padded at collate, dataset/qm8.py:265-291): the
  eigenvalues of the leading n_b x n_b block by descending |lambda| (ties by ascending lambda), the
  first min(n_b, K), then zeros; repeated eigenvalues keep their whole eigenspace.  The eigenvectors
  match the reference's up to sign and up to a rotation inside a repeated eigenvalue's eigenspace,
  which the models do not see.  The solver reads the fp32 operator; the reference decomposed it in fp64
  before the cast, so eigenvalues agree to about 1e-7.

  sizes_or_mask: [B] real node counts, or a [B,N] node mask whose real nodes lead (the reference's
  padding).  info: dict(status [B] int32, bit 0 = QL did not converge)."""
  s = sizes_or_mask
  if s.dim() == 2:
    s = (s != 0).sum(dim=1)
  D, V, status = ops.sym_eigs(L, s.to(L.device), int(num_eigs))
  return D, V, {'status': status}


def spectral_partition(L, num_partition):
  """(L_cluster [B,N,N], L_cut [B,N,N], info) for ``GPNN.forward(node_feat, L, L_cluster, L_cut)`` from the
  padded operator tensor L [B,N,N,E+1] (channel 0 is read) or a [B,N,N] operator, on L's device.

  The reference's GPNN collate (dataset/qm8.py:123-136) as one kernel launch: the P = num_partition
  eigenvectors of largest |lambda| of each padded graph's operator, KMeans(n_clusters=P, random_state=1234)
  as scikit-learn >= 1.4 runs it (one k-means++ seeding), then the L4 operators of the within-cluster and
  the cut edges.  The partitions equal the reference's except where the reference itself is undetermined
  (an eigenvalue tie at the P-th |lambda|, flagged in status bit 1, or KMeans ties).  ``GPNN.forward``
  with ``L_cluster=L_cut=None`` runs the same launch inside its captured forward.
  info: dict(labels [B,N] int32 canonical (-1: no edge), status [B] int32, see ops.spectral_partition)."""
  labels, L_cluster, L_cut, status = ops.spectral_partition(L, int(num_partition))
  return L_cluster, L_cut, {'labels': labels, 'status': status}
