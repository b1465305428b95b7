"""Complete-linkage cosine agglomerative clustering on the device.

`CosineCompleteLinkage(n_clusters).fit_predict(X)` returns the labels of scikit-learn's
`AgglomerativeClustering(n_clusters, metric="cosine", linkage="complete").fit_predict(X)`,
integer for integer.  scikit-learn computes that as scipy `pdist(X, "cosine")` + scipy
`linkage(..., "complete")` (the NN-chain algorithm) + its own heap cut of the tree, all on the host:
O(N^2 d) single-threaded work and two N^2/2 float64 host arrays.  Here the distance matrix
(fp64 tensor cores) and every NN-chain merge (one cooperative launch) run on the GPU with the
matrix resident in HBM; the O(N log N) rest -- the stable sort of the merges by distance, scipy's
union-find relabelling and scikit-learn's heap cut -- runs on the host.

The device keeps a full fp64 N x ld matrix (8 N ld bytes: 34.4 GB at N = 65,536).  Only when that
and the input do not fit in free device memory does the scikit-learn call run instead.
"""

from __future__ import annotations

import heapq

import numpy as np

from . import device as dev


def linkage_matrix(merge_xy: np.ndarray, merge_dist: np.ndarray, n: int) -> np.ndarray:
  """scipy's `linkage` output Z [n-1, 4] from NN-chain merges in chain order: a stable sort by
  distance, then the union-find relabelling of scipy's `_hierarchy.label` (cluster k >= n is the
  one formed by row k - n; Z[i, 3] is its size)."""
  order = np.argsort(merge_dist, kind="mergesort")
  pairs = np.asarray(merge_xy)[order].tolist()
  z = np.empty((n - 1, 4), dtype=np.float64)
  z[:, 2] = np.asarray(merge_dist)[order]
  parent = list(range(2 * n - 1))
  size = [1] * (2 * n - 1)
  out, sizes = [], []

  def find(x):
    root = x
    while parent[root] != root:
      root = parent[root]
    while parent[x] != root:
      parent[x], x = root, parent[x]
    return root

  for label, (x, y) in enumerate(pairs, start=n):
    rx, ry = find(x), find(y)
    out.append((rx, ry) if rx < ry else (ry, rx))
    parent[rx] = parent[ry] = label
    size[label] = size[rx] + size[ry]
    sizes.append(size[label])
  z[:, :2] = np.asarray(out, dtype=np.float64).reshape(n - 1, 2)
  z[:, 3] = sizes
  return z


def hc_cut(n_clusters: int, children: np.ndarray, n_leaves: int) -> np.ndarray:
  """scikit-learn's `_hc_cut`: the n_clusters subtrees left after undoing the last merges, labelled
  in the order the heap leaves them; the label numbering is part of the result."""
  if n_clusters > n_leaves:
    raise ValueError("Cannot extract more clusters than samples: %s clusters were given for a "
                     "tree with %s leaves." % (n_clusters, n_leaves))
  nodes = [-(int(max(children[-1])) + 1)]
  for _ in range(n_clusters - 1):
    these = children[-nodes[0] - n_leaves]
    heapq.heappush(nodes, -int(these[0]))
    heapq.heappushpop(nodes, -int(these[1]))
  node_label = np.full(2 * n_leaves - 1, -1, dtype=np.intp)
  for i, node in enumerate(nodes):
    node_label[-node] = i
  # children have smaller ids than their parent: one descending pass hands each label down
  kids = children.tolist()
  for node in range(2 * n_leaves - 2, n_leaves - 1, -1):
    lab = node_label[node]
    if lab >= 0:
      a, b = kids[node - n_leaves]
      node_label[a] = node_label[b] = lab
  return node_label[:n_leaves].copy()


def distance_bytes(n: int) -> int:
  """Device bytes of the fp64 distance matrix (rows padded to 64 elements)."""
  return 8 * n * dev.round_up(n, 64)


class CosineCompleteLinkage:
  """AgglomerativeClustering(n_clusters, metric="cosine", linkage="complete") with the same
  `fit_predict`, `labels_`, `children_` and `n_leaves_`."""

  def __init__(self, n_clusters: int = 2):
    self.n_clusters = n_clusters

  def fit_predict(self, X) -> np.ndarray:
    x = np.asarray(X)
    if x.ndim != 2:
      raise ValueError("Expected 2D array, got %dD array instead." % x.ndim)
    if x.dtype not in (np.float32, np.float64):
      x = x.astype(np.float64)
    x = np.ascontiguousarray(x)
    n = x.shape[0]
    if n < 2:
      raise ValueError("Found array with %d sample(s) (shape=%s) while a minimum of 2 is required "
                       "by AgglomerativeClustering." % (n, x.shape))
    if not np.isfinite(x).all():
      raise ValueError("Input X contains NaN or infinity.")
    if int(self.n_clusters) < 1:
      raise ValueError("n_clusters must be >= 1, got %r" % (self.n_clusters,))
    if np.any(~np.any(x, axis=1)):
      raise ValueError("Cosine affinity cannot be used when X contains zero vectors")
    if self.n_clusters > n:
      raise ValueError("Cannot extract more clusters than samples: %s clusters were given for a "
                       "tree with %s leaves." % (self.n_clusters, n))
    eng = dev.Engine.get()
    free, _ = dev.torch().cuda.mem_get_info(eng.device)
    if distance_bytes(n) + x.nbytes > free:
      return self._fit_predict_host(x)
    t = dev.torch()
    x_dev = t.from_numpy(x).to(eng.device)
    dist, flag = eng.cosine_distances(x_dev)
    del x_dev
    if int(flag.item()):
      raise ValueError("The condensed distance matrix must contain only finite values.")
    xy, md, _ = eng.complete_linkage(dist, n)
    del dist
    z = linkage_matrix(xy, md, n)
    self.children_ = z[:, :2].astype(np.intp)
    self.n_leaves_ = n
    self.labels_ = hc_cut(int(self.n_clusters), self.children_, n)
    return self.labels_

  def _fit_predict_host(self, x: np.ndarray) -> np.ndarray:
    """Inputs whose distance matrix does not fit on the device: scikit-learn on the host."""
    from sklearn.cluster import AgglomerativeClustering
    ref = AgglomerativeClustering(n_clusters=self.n_clusters, metric="cosine",
                                  linkage="complete").fit(x)
    self.children_, self.n_leaves_, self.labels_ = ref.children_, ref.n_leaves_, ref.labels_
    return self.labels_
