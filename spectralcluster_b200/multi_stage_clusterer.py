"""Multi-stage streaming clusterer -- the outermost caller of the hot path
(/root/reference/spectralcluster/multi_stage_clusterer.py: Deflicker :19-28, match_labels :31-64,
MultiStageClusterer :67-180; Wang et al., arXiv:2210.13690).

Per incoming embedding: fallback clusterer for short inputs (L), the spectral clusterer up to U1
embeddings, beyond that an agglomerative pre-clusterer compresses the cache to U1 centroids which
the spectral clusterer (device path) labels; the cache itself is replaced by its centroids every
time it reaches U2.  Host logic around `SpectralClusterer.predict` exactly as in the reference; the
complete-linkage cosine pre-clusterer runs on the device with scikit-learn's labels
(agglomerative.py).
"""

from __future__ import annotations

import enum

import numpy as np

from . import agglomerative
from . import fallback_clusterer
from . import utils


class Deflicker(enum.Enum):
  NoDeflicker = enum.auto()      # raw labels
  OrderBased = enum.auto()       # first-appearance relabelling
  Hungarian = enum.auto()        # best assignment to the previous output


def match_labels(current: np.ndarray, previous: np.ndarray) -> np.ndarray:
  """Relabel `current` (one element longer than `previous`) so that it agrees with `previous` as
  much as an assignment of current labels to previous labels allows (multi_stage_clusterer.py:31-64)."""
  from scipy import optimize
  current = utils.enforce_ordered_labels(current).astype(np.int32)
  previous = previous.astype(np.int32)
  head = current[:-1]
  if head.shape != previous.shape:
    raise ValueError("current must have one more element than previous .")
  rows = int(head.max()) + 1
  cols = max(int(previous.max()) + 1, rows)
  overlap = np.zeros((rows, cols), dtype=np.int32)
  np.add.at(overlap, (head, previous), 1)
  row_ind, col_ind = optimize.linear_sum_assignment(overlap, maximize=True)
  table = np.arange(int(current.max()) + 1, dtype=current.dtype)
  table[row_ind] = col_ind
  return table[current]


class MultiStageClusterer:
  """multi_stage_clusterer.py:67-180."""

  def __init__(self, main_clusterer, fallback_threshold: float = 0.5, L: int = 50, U1: int = 100,
               U2: int = 600, deflicker: Deflicker = Deflicker.NoDeflicker):
    self.deflicker = deflicker
    self.main = main_clusterer
    if self.main.max_spectral_size:
      raise ValueError("Do not set max_spectral_size for SpectralClusterer when"
                       "using MultiStageClusterer.")
    options = self.main.fallback_options          # mutated, like the reference (:90-105)
    options.spectral_min_embeddings = L
    options.agglomerative_threshold = fallback_threshold
    options.single_cluster_condition = fallback_clusterer.SingleClusterCondition.FallbackClusterer
    options.fallback_clusterer_type = fallback_clusterer.FallbackClustererType.Agglomerative
    self.U1, self.U2 = U1, U2
    self.pre = agglomerative.CosineCompleteLinkage(n_clusters=U1)
    self.cache = None                    # embeddings, or centroids after a compression
    self.num_embeddings = 0
    self.compression_labels = None       # original embedding -> row of the cache
    self.previous_output = None

  def streaming_predict(self, embedding: np.ndarray) -> np.ndarray:
    """Labels of every embedding seen so far, earlier ones possibly corrected."""
    self.num_embeddings += 1
    if self.num_embeddings == 1:
      self.cache = embedding
      self.previous_output = np.array([0])
      return self.previous_output
    self.cache = np.vstack([self.cache, embedding])
    if self.num_embeddings <= self.U1:                        # fallback or main clusterer alone
      self.previous_output = self.main.predict(self.cache)
      return self.previous_output
    if self.compression_labels is not None:                   # the new embedding is its own row
      self.compression_labels = np.append(self.compression_labels,
                                          max(self.compression_labels) + 1)
    pre_labels = self.pre.fit_predict(self.cache)
    centroids = utils.get_cluster_centroids(self.cache, pre_labels)
    main_labels = self.main.predict(centroids)
    labels = utils.chain_labels(self.compression_labels,
                                utils.chain_labels(pre_labels, main_labels))
    if self.cache.shape[0] == self.U2:                        # dynamic compression
      self.cache = centroids
      self.compression_labels = utils.chain_labels(self.compression_labels, pre_labels)
    if self.deflicker == Deflicker.OrderBased:
      labels = utils.enforce_ordered_labels(labels)
    elif self.deflicker == Deflicker.Hungarian:
      labels = match_labels(labels, self.previous_output)
    self.previous_output = labels
    return labels
