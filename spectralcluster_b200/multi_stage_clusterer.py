"""Multi-stage streaming clusterer -- the outermost caller of the hot path
(/root/reference/spectralcluster/multi_stage_clusterer.py: Deflicker :19-28, match_labels :31-64,
MultiStageClusterer :67-180; Wang et al., arXiv:2210.13690).

Per incoming embedding: fallback clusterer for short inputs (L), the spectral clusterer up to U1
embeddings, beyond that an agglomerative pre-clusterer compresses the cache to U1 centroids which
the spectral clusterer (device path) labels; the cache itself is replaced by its centroids every
time it reaches U2.  Host logic around `SpectralClusterer.predict` exactly as in the reference; the
complete-linkage cosine pre-clusterer runs on the device with scikit-learn's labels
(agglomerative.py).  A stream of CUDA tensors keeps its cache on the device (torch.cat for
np.vstack, device centroids at a compression) and returns what the stream of their host twins
returns; labels stay host arrays.
"""

from __future__ import annotations

import enum

import numpy as np

from . import agglomerative
from . import device as dev
from . import fallback_clusterer
from . import naive_clusterer
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


def twin_dtype(x):
  """The numpy dtype of a tensor's host twin (x.cpu().numpy(); bfloat16 through float32)."""
  t = dev.torch()
  return np.dtype(np.float32) if x.dtype == t.bfloat16 else t.empty(0, dtype=x.dtype).numpy().dtype


def append_rows(cache, embedding):
  """np.vstack([cache, embedding]) for tensors: the rows of both, in the dtype np.vstack gives
  their host twins."""
  t = dev.torch()
  dtype = t.from_numpy(np.empty(0, np.result_type(twin_dtype(cache), twin_dtype(embedding)))).dtype
  return t.cat([t.atleast_2d(cache).to(dtype), t.atleast_2d(embedding.detach()).to(dtype)])


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
    self.stream_device = None            # the device of a stream of CUDA tensors

  def streaming_predict(self, embedding) -> np.ndarray:
    """Labels of every embedding seen so far, earlier ones possibly corrected.

    `embedding` is one row, (d,) or (1, d): an ndarray, or a CUDA tensor on the current device.
    A stream of CUDA tensors returns, step for step, what the stream of their host twins returns
    (X.cpu().numpy(); bfloat16: X.float().cpu().numpy()).  A stream that mixes host arrays and
    CUDA tensors, or CUDA tensors of two devices, raises TypeError, and the step changes nothing."""
    device = embedding.device if naive_clusterer._is_cuda_tensor(embedding) else None
    if self.num_embeddings and device != self.stream_device:
      raise TypeError("this stream takes %s, got %s" % (
          "host arrays" if self.stream_device is None else "CUDA tensors on %s" % self.stream_device,
          "a host array" if device is None else "a CUDA tensor on %s" % device))
    if device is not None and device.index != dev.torch().cuda.current_device():
      raise ValueError("the embedding is on %s, but streaming_predict() runs on cuda:%d (the "
                       "current device)" % (device, dev.torch().cuda.current_device()))
    self.num_embeddings += 1
    if self.num_embeddings == 1:
      self.stream_device = device
      # the first embedding is the cache as given (1-D stays 1-D); bfloat16 as its twin, float32
      self.cache = embedding
      if device is not None:
        self.cache = embedding.detach()
        if self.cache.dtype == dev.torch().bfloat16:
          self.cache = self.cache.float()
      self.previous_output = np.array([0])
      return self.previous_output
    if device is None:
      self.cache = np.vstack([self.cache, embedding])
    else:
      self.cache = append_rows(self.cache, embedding)
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
