"""Complete- and average-linkage cosine agglomerative clustering on the device.

`CosineCompleteLinkage(n_clusters).fit_predict(X)` returns the labels of scikit-learn's
`AgglomerativeClustering(n_clusters, metric="cosine", linkage="complete").fit_predict(X)`, and
`CosineAverageLinkage(t).fit_predict(X)` those of `AgglomerativeClustering(n_clusters=None,
metric="cosine", linkage="average", distance_threshold=t).fit_predict(X)`, integer for integer.
scikit-learn computes them as scipy `pdist(X, "cosine")` + scipy `linkage(..., "complete" /
"average")` (the NN-chain algorithm) + its own heap cut of the tree, all on the host: O(N^2 d)
single-threaded work and two N^2/2 float64 host arrays.  Here the distance matrix (fp64 tensor
cores) and every NN-chain merge (one cooperative launch) run on the GPU with the matrix resident in
HBM; the O(N log N) rest -- the stable sort of the merges by distance, scipy's union-find
relabelling and scikit-learn's heap cut -- runs on the host.

The device keeps a full fp64 N x ld matrix (8 N ld bytes: 34.4 GB at N = 65,536).  Only when that
and the input do not fit in free device memory does the scikit-learn call run instead.
"""

from __future__ import annotations

import heapq
import numbers

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


def threshold_cut(threshold: float, children: np.ndarray, distances: np.ndarray, n_leaves: int):
  """scikit-learn's distance-threshold cut (AgglomerativeClustering._fit): every merge at a distance
  >= threshold is undone, so there is one cluster more than such merges; those clusters are
  labelled by `hc_cut`.  -> (n_clusters, labels)."""
  n_clusters = np.count_nonzero(distances >= threshold) + 1
  return n_clusters, hc_cut(n_clusters, children, n_leaves)


def distance_bytes(n: int) -> int:
  """Device bytes of the fp64 distance matrix (rows padded to 64 elements)."""
  return 8 * n * dev.round_up(n, 64)


def device_fits(eng, nbytes: int) -> bool:
  """Whether `nbytes` more fit on the device.  When free device memory falls short, the torch
  caching allocator first hands back the blocks it holds without a live tensor and free memory is
  read again: inside predict() the previous call's matrices sit in that cache (two fp32 N x N at
  N = 65,536 are 34 GB), and an allocation could use them too."""
  t = dev.torch()
  if nbytes <= t.cuda.mem_get_info(eng.device)[0]:
    return True
  t.cuda.empty_cache()
  return nbytes <= t.cuda.mem_get_info(eng.device)[0]


def _checked_input(X):
  """scikit-learn's input checks for metric="cosine" -> (x, on_device): a CUDA tensor stays on the
  device, anything else becomes a C-contiguous float32/float64 ndarray."""
  t = dev.torch()
  on_device = isinstance(X, t.Tensor) and X.is_cuda
  x = X if on_device else np.asarray(X)
  if x.ndim != 2:
    raise ValueError("Expected 2D array, got %dD array instead." % x.ndim)
  n = int(x.shape[0])
  if on_device:
    if x.dtype not in (t.float32, t.float64):
      x = x.to(t.float64)
    if x.stride(1) != 1:
      x = x.contiguous()
  else:
    if x.dtype not in (np.float32, np.float64):
      x = x.astype(np.float64)
    x = np.ascontiguousarray(x)
  if n < 2:
    raise ValueError("Found array with %d sample(s) (shape=%s) while a minimum of 2 is required "
                     "by AgglomerativeClustering." % (n, tuple(x.shape)))
  finite = bool(t.isfinite(x).all()) if on_device else bool(np.isfinite(x).all())
  if not finite:
    raise ValueError("Input X contains NaN or infinity.")
  zero_row = bool((x == 0).all(dim=1).any()) if on_device else bool(np.any(~np.any(x, axis=1)))
  if zero_row:
    raise ValueError("Cosine affinity cannot be used when X contains zero vectors")
  return x, on_device


class _CosineLinkage:
  """What the cosine linkages share: the input checks, the choice between the device and
  scikit-learn, the distance matrix and the NN-chain on the device, and scipy's Z on the host.
  A subclass checks its parameters, runs its NN-chain entry, cuts the tree and names the
  scikit-learn estimator and attributes of the host path."""

  _fitted = ("children_", "n_leaves_", "labels_")

  def fit_predict(self, X) -> np.ndarray:
    x, on_device = _checked_input(X)
    n = int(x.shape[0])
    self._check_params(n)
    eng = dev.Engine.get()
    if not device_fits(eng, distance_bytes(n) + (0 if on_device else x.nbytes)):
      return self._fit_predict_host(x.cpu().numpy() if on_device else x)
    x_dev = x if on_device else dev.torch().from_numpy(x).to(eng.device)
    dist, flag = eng.cosine_distances(x_dev)
    del x_dev
    if int(flag.item()):
      raise ValueError("The condensed distance matrix must contain only finite values.")
    xy, md, _ = self._nn_chain(eng, dist, n)
    del dist
    z = linkage_matrix(xy, md, n)
    self.children_ = z[:, :2].astype(np.intp)
    self.n_leaves_ = n
    self.labels_ = self._cut(z, n)
    return self.labels_

  def _fit_predict_host(self, x: np.ndarray) -> np.ndarray:
    """Inputs whose distance matrix does not fit on the device: scikit-learn on the host."""
    ref = self._estimator().fit(x)
    for name in self._fitted:
      setattr(self, name, getattr(ref, name))
    return self.labels_


class CosineCompleteLinkage(_CosineLinkage):
  """AgglomerativeClustering(n_clusters, metric="cosine", linkage="complete") with the same
  `fit_predict`, `labels_`, `children_` and `n_leaves_`."""

  def __init__(self, n_clusters: int = 2):
    self.n_clusters = n_clusters

  def _check_params(self, n: int):
    if int(self.n_clusters) < 1:
      raise ValueError("n_clusters must be >= 1, got %r" % (self.n_clusters,))
    if self.n_clusters > n:
      raise ValueError("Cannot extract more clusters than samples: %s clusters were given for a "
                       "tree with %s leaves." % (self.n_clusters, n))

  def _nn_chain(self, eng, dist, n: int):
    return eng.complete_linkage(dist, n)

  def _cut(self, z: np.ndarray, n: int) -> np.ndarray:
    return hc_cut(int(self.n_clusters), self.children_, n)

  def _estimator(self):
    from sklearn.cluster import AgglomerativeClustering
    return AgglomerativeClustering(n_clusters=self.n_clusters, metric="cosine", linkage="complete")


class CosineAverageLinkage(_CosineLinkage):
  """AgglomerativeClustering(n_clusters=None, metric="cosine", linkage="average",
  distance_threshold) with the same `fit_predict`, `labels_`, `children_`, `n_leaves_`,
  `n_clusters_` and `distances_`: every merge at a distance >= distance_threshold is undone.
  `fit_predict` also takes the embeddings as a CUDA tensor, which it reads in place."""

  _fitted = _CosineLinkage._fitted + ("n_clusters_", "distances_")

  def __init__(self, distance_threshold: float):
    self.distance_threshold = distance_threshold

  def _check_params(self, n: int):
    t = self.distance_threshold
    if not isinstance(t, numbers.Real) or not t >= 0:
      from sklearn.utils._param_validation import InvalidParameterError
      raise InvalidParameterError(
          "The 'distance_threshold' parameter of AgglomerativeClustering must be a float in the "
          "range [0.0, inf) or None. Got %r instead." % (t,))

  def _nn_chain(self, eng, dist, n: int):
    return eng.average_linkage(dist, n)

  def _cut(self, z: np.ndarray, n: int) -> np.ndarray:
    self.distances_ = z[:, 2]
    self.n_clusters_, labels = threshold_cut(self.distance_threshold, self.children_,
                                             self.distances_, n)
    return labels

  def _estimator(self):
    from sklearn.cluster import AgglomerativeClustering
    return AgglomerativeClustering(n_clusters=None, metric="cosine", linkage="average",
                                   distance_threshold=self.distance_threshold)
