"""fp64 numpy restatement of the reference's GPNN partition, ``spectral_clustering(L, P, seed=1234)``
(utils/spectral_graph_partition.py:10-32), as it behaves with scikit-learn >= 1.4 (``n_init='auto'``: one
k-means++ run; ``algorithm='lloyd'``).  It is the oracle of ops.spectral_partition.

  * embedding: the P eigenvectors of largest |lambda| of the whole padded N x N operator (the padded zero
    rows included: the collate hands eigsh the padded matrix).  Column order and signs move the point set
    by an isometry only, so a dense ``eigh`` stands in for ARPACK's ``eigsh``;
  * KMeans.fit: tolerance mean(var(X, 0)) * 1e-4, X -= X.mean(0), k-means++ with 2 + int(log P) local trials
    drawn from a fresh RandomState(seed) (sklearn's _kmeans_plusplus), Lloyd as _kmeans_single_lloyd
    (E-step argmin of |c|^2 - 2 x.c, strict label convergence or a centre shift <= tol, 300 iterations, a
    final E-step when convergence was not strict, empty clusters relocated to the farthest points with
    ties broken by the lower index); it also reports KMeans ties (kmeans_tie), where the partition is
    decided by rounding;
  * labels in make_gpnn_golden.reference_partitions' canonical form.
"""
import numpy as np

TIE = 1e-9
KMEANS_TIE = 1e-9
MAX_ITER = 300


def canonical(labels, L):
  """Nodes without an edge get -1; the other clusters are numbered by first appearance."""
  L = np.asarray(L)
  linked = ((L != 0) & ~np.eye(L.shape[0], dtype=bool)).any(axis=1)
  first = {}
  return np.array([first.setdefault(int(v), len(first)) if ok else -1 for v, ok in zip(labels, linked)],
                  dtype=np.int32)


def embedding(L, P):
  """(V [N, P], tie): the eigenvectors of the P largest |lambda| and whether |lambda_P| and |lambda_P+1|
  are within TIE (the reference's choice is then open)."""
  w, V = np.linalg.eigh(np.asarray(L, dtype=np.float64))
  order = np.argsort(-np.abs(w), kind='mergesort')
  tie = P < len(w) and abs(abs(w[order[P - 1]]) - abs(w[order[P]])) < TIE
  return V[:, order[:P]], bool(tie)


def _sqdist(C, X, xx):
  """sklearn's _euclidean_distances(C, X, Y_norm_squared=xx, squared=True)."""
  d = -2 * (C @ X.T)
  d += np.einsum('ij,ij->i', C, C)[:, None]
  d += xx[None, :]
  np.maximum(d, 0, out=d)
  return d


def _near(a, b):
  return abs(a - b) <= KMEANS_TIE * max(abs(a), abs(b), 1e-300)


def kmeans_plusplus(X, P, rs, ties=None):
  """sklearn's _kmeans_plusplus with unit sample weights: (centres [P, d], indices [P]).  ``ties``, a list,
  collects the seeding steps whose best potential is within KMEANS_TIE of another candidate point's (the
  choice is then made by rounding)."""
  N = X.shape[0]
  T = 2 + int(np.log(P))
  xx = np.einsum('ij,ij->i', X, X)
  idx = [int(rs.choice(N, p=np.ones(N) / N))]
  w = np.ones(N)
  closest = _sqdist(X[idx], X, xx)
  pot = closest @ w                         # sklearn's potentials are BLAS products with the weights
  closest = closest[0]
  for _ in range(1, P):
    rv = rs.uniform(size=T) * pot
    cand = np.clip(np.searchsorted(np.cumsum(w * closest), rv), None, N - 1)
    d = np.minimum(closest, _sqdist(X[cand], X, xx))
    pots = (d @ w.reshape(-1, 1))[:, 0]
    b = int(np.argmin(pots))
    if ties is not None and any(not np.array_equal(X[cand[r]], X[cand[b]]) and _near(pots[r], pots[b])
                                 for r in range(T)):
      ties.append(len(idx))
    pot, closest = pots[b], d[b]
    idx.append(int(cand[b]))
  return X[idx].copy(), np.array(idx)


def _assign(X, C):
  return np.argmin((C * C).sum(axis=1)[None, :] - 2 * (X @ C.T), axis=1)


def lloyd(X, C, tol):
  """sklearn's _kmeans_single_lloyd: (labels, centres, inertia, hit_max_iter)."""
  N, P = X.shape[0], C.shape[0]
  labels_old = np.full(N, -1)
  strict = False
  it = 0
  for it in range(MAX_ITER):
    labels = _assign(X, C)
    counts = np.bincount(labels, minlength=P).astype(np.float64)
    Cn = np.zeros_like(C)
    np.add.at(Cn, labels, X)
    empty = np.flatnonzero(counts == 0)
    if len(empty):
      dist = ((X - C[labels]) ** 2).sum(axis=1)
      far = np.lexsort((np.arange(N), -dist))[:len(empty)]
      for j, f in zip(empty, far):
        Cn[labels[f]] -= X[f]
        Cn[j] = X[f]
        counts[j] = 1.0
        counts[labels[f]] -= 1.0
    nz = counts > 0
    Cn[nz] *= (1.0 / counts[nz])[:, None]
    shift = ((Cn - C) ** 2).sum()
    C = Cn
    if np.array_equal(labels, labels_old):
      strict = True
      break
    if shift <= tol:
      break
    labels_old = labels
  else:
    it = MAX_ITER
  if not strict:
    labels = _assign(X, C)
  inertia = float(((X - C[labels]) ** 2).sum())
  return labels, C, inertia, it == MAX_ITER


def centred_embedding(L, P):
  """(X centred [N, P], tol, tie) as KMeans.fit sees the embedding."""
  V, tie = embedding(L, P)
  X = V.copy()
  tol = float(np.mean(np.var(X, axis=0)) * 1e-4)
  X -= X.mean(axis=0)
  return X, tol, tie


def partition_inertia(L, P, labels):
  """Within-cluster sum of squares of a partition (raw labels, every node) in the centred embedding:
  KMeans' inertia at convergence, and invariant under the embedding's isometries."""
  X, _, _ = centred_embedding(L, P)
  labels = np.asarray(labels)
  return float(sum(((X[labels == c] - X[labels == c].mean(axis=0)) ** 2).sum() for c in np.unique(labels)))


def spectral_clustering(L, P, seed=1234):
  """dict(labels canonical [N] int32, raw [N], inertia, tie, maxed, kmeans_tie) of one padded operator
  L [N, N].  kmeans_tie: a seeding choice or a final assignment was decided within KMEANS_TIE, so rounding
  (or, in the reference, BLAS) picks the partition."""
  N = np.asarray(L).shape[0]
  assert P < N - 1
  X, tol, tie = centred_embedding(L, P)
  ties = []
  C, _ = kmeans_plusplus(X, P, np.random.RandomState(seed), ties)
  raw, C, inertia, maxed = lloyd(X, C, tol)
  pd = np.sort((C * C).sum(axis=1)[None, :] - 2 * (X @ C.T), axis=1)
  e_tie = bool(np.any(np.abs(pd[:, 1] - pd[:, 0]) <= KMEANS_TIE * np.maximum(np.abs(pd[:, 0]), 1e-300)))
  return {'labels': canonical(raw, L), 'raw': raw, 'inertia': inertia, 'tie': tie, 'maxed': maxed,
          'kmeans_tie': bool(ties) or e_tie}
