"""Affinity, eigen-analysis and eigengap utilities -- device-backed mirror of
/root/reference/spectralcluster/utils.py (compute_affinity_matrix :20-41,
compute_sorted_eigenvectors :44-71, compute_number_of_clusters :74-130,
enforce_ordered_labels :133-156)."""

from __future__ import annotations

import enum
import typing

import numpy as np

from . import _native as nat
from . import device as dev
from . import naive_clusterer

EPS = 1e-10


class EigenGapType(enum.Enum):
  Ratio = enum.auto()            # ratio of consecutive eigenvalues
  NormalizedDiff = enum.auto()   # difference of consecutive eigenvalues over the largest one


def compute_affinity_matrix(embeddings: np.ndarray) -> np.ndarray:
  """(cosine + 1) / 2 of all pairs of rows, computed on the device; result in [0, 1]."""
  eng = dev.Engine.get()
  t = dev.torch()
  x = np.ascontiguousarray(embeddings)
  if x.dtype not in (np.float32, np.float64):
    x = x.astype(np.float64)
  a, _ = eng.affinity(t.from_numpy(x).to(eng.device), want_crop_vector=False)
  return eng.download_matrix(a, x.shape[0])


def compute_sorted_eigenvectors(
    input_matrix: np.ndarray, descend: bool = True) -> typing.Tuple[np.ndarray, np.ndarray]:
  """All eigenpairs of a SYMMETRIC host matrix, sorted by eigenvalue (device Householder + QL).

  The reference calls the general np.linalg.eig; every matrix the hot path produces is
  symmetric or diagonally similar to a symmetric one, which is what the device solver handles
  (a genuinely non-symmetric input raises NotImplementedError)."""
  m = np.asarray(input_matrix, dtype=np.float64)
  if m.ndim != 2 or m.shape[0] != m.shape[1]:
    raise ValueError("input_matrix must be square")
  scale = np.max(np.abs(m)) if m.size else 0.0
  if m.size and np.max(np.abs(m - m.T)) > 1e-6 * max(scale, 1e-300):
    raise NotImplementedError(
        "general (non-symmetric) eigendecomposition is outside the GPU hot path "
        "(SURVEY.md 8(f) rank 1)")
  eng = dev.Engine.get()
  n = m.shape[0]
  s = eng.upload_matrix(m)
  w, v, _ = eng.eigh(s, n, None, None, None, 1.0,
                     nat.EIG_LARGEST if descend else nat.EIG_SMALLEST, n, n, dense=True)
  return w.copy(), v.to("cpu").numpy()


def compute_number_of_clusters(eigenvalues: np.ndarray,
                               max_clusters: typing.Optional[int] = None,
                               stop_eigenvalue: float = 1e-2,
                               eigengap_type: EigenGapType = EigenGapType.Ratio,
                               descend: bool = True,
                               eps: float = EPS,
                               max_eigenvalue: typing.Optional[float] = None
                               ) -> typing.Tuple[int, float]:
  """Maximum-eigengap estimate of the cluster count (host logic on <= max_clusters+1 values).

  Returns (number of clusters, the winning gap).  Descending spectra stop at the first
  eigenvalue below `stop_eigenvalue`; ascending spectra skip the (zero) first eigenvalue.
  `max_eigenvalue` stands in for np.max(eigenvalues) when `eigenvalues` is a prefix of the
  spectrum that lacks its largest value (NormalizedDiff normalises by it)."""
  if not isinstance(eigengap_type, EigenGapType):
    raise TypeError("eigengap_type must be a EigenGapType")
  if eigengap_type not in (EigenGapType.Ratio, EigenGapType.NormalizedDiff):
    raise ValueError("Unsupported eigengap_type")
  w = eigenvalues
  limit = len(w)
  if max_clusters and max_clusters + 1 < limit:
    limit = max_clusters + 1
  use_ratio = eigengap_type == EigenGapType.Ratio

  def gap(big, small):
    if use_ratio:
      return big / (small + eps)
    return (big - small) / (np.max(w) if max_eigenvalue is None else max_eigenvalue)

  winner, widest = 0, 0
  if descend:
    for count in range(1, limit):
      if w[count - 1] < stop_eigenvalue:
        break
      g = gap(w[count - 1], w[count])
      if g > widest:
        winner, widest = count, g
  else:
    for idx in range(1, limit - 1):
      g = gap(w[idx + 1], w[idx])
      if g > widest:
        winner, widest = idx + 1, g
  return winner, widest


def enforce_ordered_labels(labels: np.ndarray) -> np.ndarray:
  """Relabel so that labels appear in order of first occurrence (permutation-invariant form)."""
  _, first, inverse = np.unique(labels, return_index=True, return_inverse=True)
  rank = np.empty_like(first)
  rank[np.argsort(first)] = np.arange(len(first))
  out = labels.copy()
  out[...] = rank[inverse].reshape(labels.shape)
  return out


def get_cluster_centroids(embeddings, labels: np.ndarray):
  """Mean embedding of every cluster 0..max(labels) (utils.py:159-177), as one segmented sum.

  A CUDA tensor gives a device fp64 tensor (sc_cluster_centroids) whose host copy equals what the
  host function returns for the tensor's host twin, bit for bit."""
  if naive_clusterer._is_cuda_tensor(embeddings):
    x = dev.twin(dev.device_embeddings(embeddings))
    return dev.Engine.get(x.device.index).cluster_centroids(x, labels)
  labels = np.asarray(labels).astype(np.int64)
  k = int(labels.max()) + 1
  sums = np.zeros((k, embeddings.shape[1]), dtype=np.result_type(embeddings.dtype, np.float64))
  np.add.at(sums, labels, embeddings)
  counts = np.bincount(labels, minlength=k).astype(sums.dtype)
  return sums / counts[:, None]        # an empty cluster id gives NaN, like np.mean of no rows


def chain_labels(pre_labels: typing.Optional[np.ndarray], main_labels: np.ndarray) -> np.ndarray:
  """Compose pre-clusterer labels with the labels of its clusters (utils.py:180-206).  The result
  is float64 like the reference's (np.zeros default dtype, SURVEY.md A.4-5)."""
  if pre_labels is None:
    return main_labels
  groups = int(max(pre_labels) + 1)
  if groups != main_labels.shape[0]:
    raise ValueError("pre_labels has {} values while main_labels has {} rows.".format(
        groups, main_labels.shape[0]))
  return np.asarray(main_labels)[np.asarray(pre_labels).astype(np.int64)].astype(np.float64)
