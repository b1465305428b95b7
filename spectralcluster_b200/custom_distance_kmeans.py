"""K-means with a custom distance on the spectral embeddings -- device-backed mirror of
/root/reference/spectralcluster/custom_distance_kmeans.py (run_kmeans :13-52, CustomKMeans
:55-141).  Seeding, the single scikit-learn Lloyd step and the custom-distance loop all run in
CUDA (csrc/kmeans.cu); only the MT19937 draws of RandomState(0) are taken on the host."""

from __future__ import annotations

import dataclasses
import typing

import numpy as np

from . import device as dev

# scipy.spatial.distance's numeric metrics and their spellings (scipy's _METRICS[name].aka) ->
# sc_kmeans metric code (SC_KMEANS_* in include/spectralcluster_b200.h).  A name can only carry
# minkowski's default p = 2, which scipy evaluates as euclidean.
_ALIASES = {
    "cosine": {"cosine", "cos"},
    "euclidean": {"euclidean", "euclid", "eu", "e"},
    "sqeuclidean": {"sqeuclidean", "sqeuclid", "sqe"},
    "cityblock": {"cityblock", "cblock", "cb", "c"},
    "chebyshev": {"chebyshev", "chebychev", "cheby", "cheb", "ch"},
    "minkowski": {"minkowski", "mi", "m", "pnorm"},
    "canberra": {"canberra"},
    "braycurtis": {"braycurtis"},
    "correlation": {"correlation", "co"},
    "jensenshannon": {"jensenshannon", "js"},
    "seuclidean": {"seuclidean", "se", "s"},
    "mahalanobis": {"mahalanobis", "mahal", "mah"},
}
_CODES = {"cosine": 0, "euclidean": 1, "sqeuclidean": 2, "cityblock": 3, "chebyshev": 4,
          "minkowski": 1, "canberra": 5, "braycurtis": 6, "correlation": 7, "jensenshannon": 8,
          "seuclidean": 9, "mahalanobis": 10}
_METRICS = {alias: _CODES[name] for name, akas in _ALIASES.items() for alias in akas}


def run_kmeans(spectral_embeddings, n_clusters: int,
               custom_dist: typing.Union[str, typing.Callable, None], max_iter: int) -> np.ndarray:
  """Cluster the rows of `spectral_embeddings` (host ndarray or device fp64 tensor) into
  `n_clusters` groups; returns int64 labels on the host.

  Every numeric scipy.spatial.distance metric name (cosine, euclidean, sqeuclidean, cityblock,
  chebyshev, minkowski, canberra, braycurtis, correlation, jensenshannon, seuclidean, mahalanobis,
  and scipy's other spellings of them) runs entirely on the device, with scipy's special values.
  A singular mahalanobis covariance raises numpy.linalg.LinAlgError, as np.linalg.inv does.  The
  other forms the reference accepts -- callables, hamming and the boolean metrics (degenerate on
  real-valued embeddings; custom_distance_kmeans.py:37-47; None fails in the reference, and
  here) -- are host code on the [n, k] embeddings, exactly like the reference."""
  eng = dev.Engine.get()          # no CUDA device -> RuntimeError, whatever the metric
  if isinstance(custom_dist, str) and custom_dist in _METRICS:
    t = dev.torch()
    if isinstance(spectral_embeddings, np.ndarray):
      e = t.from_numpy(np.ascontiguousarray(spectral_embeddings, dtype=np.float64)).to(eng.device)
    else:
      e = spectral_embeddings.contiguous()
    labels, _ = eng.kmeans(e, int(n_clusters), _METRICS[custom_dist], int(max_iter))
    return labels
  from sklearn.cluster import KMeans
  e = (spectral_embeddings if isinstance(spectral_embeddings, np.ndarray)
       else spectral_embeddings.to("cpu").numpy())
  if not custom_dist:
    # the reference builds this estimator and calls predict() without fitting it
    # (custom_distance_kmeans.py:33-36,51): scikit-learn raises NotFittedError.  Same here.
    return KMeans(n_clusters=n_clusters, init="k-means++", max_iter=300, random_state=0,
                  n_init="auto").predict(e)
  seed = KMeans(n_clusters=n_clusters, init="k-means++", max_iter=1, random_state=0,
                n_init="auto").fit(e)
  return CustomKMeans(n_clusters=n_clusters, centroids=seed.cluster_centers_, max_iter=max_iter,
                      custom_dist=custom_dist).predict(e)


@dataclasses.dataclass
class CustomKMeans:
  """Lloyd iterations under an arbitrary scipy distance (custom_distance_kmeans.py:55-141), host
  arrays; `run_kmeans` uses the CUDA implementation of the same loop for every numeric metric
  name."""
  n_clusters: typing.Optional[int] = None
  centroids: typing.Optional[np.ndarray] = None
  max_iter: int = 10
  tol: float = 0.001
  custom_dist: typing.Union[str, typing.Callable] = "cosine"

  def _init_centroids(self, embeddings: np.ndarray):
    pick = np.random.choice(np.arange(embeddings.shape[0]), size=self.n_clusters, replace=False)
    self.centroids = embeddings[pick, :]

  def predict(self, embeddings: np.ndarray) -> np.ndarray:
    from scipy.spatial import distance
    n, d = embeddings.shape
    if self.max_iter <= 0:
      raise ValueError("Number of iterations should be a positive number,"
                       " got %d instead" % self.max_iter)
    if n < self.n_clusters:
      raise ValueError("n_samples=%d should be >= n_clusters=%d" % (n, self.n_clusters))
    if self.centroids is None:
      self._init_centroids(embeddings)
    if self.centroids.shape[0] != self.n_clusters:
      raise ValueError("The shape of the initial centroids (%s)"
                       "does not match the number of clusters %d"
                       % (str(self.centroids.shape), self.n_clusters))
    if self.centroids.shape[1] != d:
      raise ValueError("The number of features of the initial centroids %d"
                       "does not match the number of features of the data %d."
                       % (self.centroids.shape[1], d))
    rows = np.arange(n)
    previous = 0
    for step in range(self.max_iter + 1):
      dist = distance.cdist(embeddings, self.centroids, metric=self.custom_dist)
      labels = dist.argmin(axis=1)
      mean = np.mean(dist[rows, labels])
      settled = mean <= previous and mean >= (1 - self.tol) * previous
      if settled or step == self.max_iter:
        break
      previous = mean
      for c in range(self.n_clusters):
        members = np.where(labels == c)[0]
        if members.any():          # sic: a cluster holding only sample 0 keeps its centroid (A.4-3)
          self.centroids[c] = np.mean(embeddings[members], axis=0)
    return labels
