"""Online "naive" clusterer -- the caller-side fallback of the hot path
(/root/reference/spectralcluster/naive_clusterer.py:5-105; used by FallbackClusterer,
fallback_clusterer.py:114-117).

Strictly sequential by definition (the label of frame t depends on the centroids after frames
0..t-1).  Host ndarrays run here, one matrix-vector product per embedding over the [clusters, d]
matrix of running means.  `predict` / `fit_predict` with a CUDA tensor run the whole sequence in
one device launch (`sc_naive_cluster`) with the same fp64 arithmetic and leave the same state, so
that `predict_next` continues where a host run would; the single-vs-multi cluster probe of
predict() uses that launch too (fallback_clusterer.check_single_cluster).
"""

from __future__ import annotations

import sys
import typing

import numpy as np


class NaiveCentroid:
  """One cluster of the naive algorithm as the reference exposes it (naive_clusterer.py:5-22):
  the running mean `embedding` of its `count` members."""

  def __init__(self, embedding: np.ndarray, count: int = 1):
    self.embedding = embedding
    self.count = count

  def merge(self, embedding: np.ndarray):
    total = self.count + 1
    self.embedding = (self.embedding * self.count + embedding) / total
    self.count = total

  def cosine(self, embedding: np.ndarray) -> float:
    norms = np.linalg.norm(self.embedding) * np.linalg.norm(embedding)
    return float(np.dot(self.embedding, embedding) / norms)


class NaiveClusterer:
  """Assign each embedding to the most similar running centroid, or open a new cluster."""

  def __init__(self, threshold: float, adaptation_threshold: typing.Optional[float] = None):
    if adaptation_threshold is not None and adaptation_threshold < threshold:
      raise ValueError("adaptation_threshold cannot be smaller than threshold")
    self.threshold = threshold
    self.adaptation_threshold = threshold if adaptation_threshold is None else adaptation_threshold
    self.reset()

  def reset(self):
    self._means = None                     # [clusters, d] running means
    self._counts = []                      # members merged into each mean

  @property
  def centroids(self) -> typing.List[NaiveCentroid]:
    """Snapshot of the clusters as NaiveCentroid objects (the reference keeps such a list)."""
    if self._means is None:
      return []
    return [NaiveCentroid(row.copy(), count) for row, count in zip(self._means, self._counts)]

  def _open(self, embedding) -> int:
    row = np.asarray(embedding, dtype=np.float64)[None, :]
    self._means = row.copy() if self._means is None else np.concatenate([self._means, row])
    self._counts.append(1)
    return len(self._counts) - 1

  def predict_next(self, embedding: np.ndarray) -> int:
    """Label of one new embedding (naive_clusterer.py:58-89)."""
    if self._means is None:
      return self._open(embedding)
    e = np.asarray(embedding, dtype=np.float64)
    cos = (self._means @ e) / (np.linalg.norm(self._means, axis=1) * np.linalg.norm(e))
    if cos.max() < self.threshold:
      return self._open(embedding)
    label = int(cos.argmax())
    if cos[label] > self.adaptation_threshold:
      c = self._counts[label]
      self._means[label] = (self._means[label] * c + e) / (c + 1)    # :14-18
      self._counts[label] = c + 1
    return label

  def predict(self, embeddings) -> np.ndarray:
    """Labels of the rows of `embeddings`, continuing the current state.  A CUDA tensor is read in
    place on the device; anything else runs on the host."""
    if _is_cuda_tensor(embeddings):
      return self._predict_device(embeddings)
    return np.array([self.predict_next(e) for e in embeddings])

  def _predict_device(self, x) -> np.ndarray:
    from . import device as dev
    t = dev.torch()
    if x.ndim != 2:
      raise ValueError("embeddings must be 2-dimensional")
    if x.dtype not in (t.float32, t.float64):
      x = x.to(t.float64)
    if x.stride(1) != 1:
      x = x.contiguous()
    eng = dev.Engine.get(x.device.index)
    means = counts = None
    if self._means is not None:
      means = t.from_numpy(self._means).to(eng.device)
      counts = t.tensor(self._counts, dtype=t.int64, device=eng.device)
    labels, _, k, means, counts = eng.naive_cluster(
        x, self.threshold, self.adaptation_threshold, means=means, counts=counts)
    if k:
      self._means = means.cpu().numpy()
      self._counts = counts.cpu().tolist()
    if x.shape[0] == 0:
      return np.array([])
    return labels.cpu().numpy()

  def fit_predict(self, embeddings: np.ndarray) -> np.ndarray:
    return self.predict(embeddings)


def _is_cuda_tensor(x) -> bool:
  torch = sys.modules.get("torch")       # a torch tensor implies torch is imported
  return torch is not None and isinstance(x, torch.Tensor) and x.is_cuda
