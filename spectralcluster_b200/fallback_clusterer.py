"""Fallback clusterer and the single-vs-multi cluster decision around the hot path
(/root/reference/spectralcluster/fallback_clusterer.py: options :23-92, FallbackClusterer
:95-124, check_single_cluster :127-187).

What runs where:
  * AllAffinity / NeighborAffinity / AffinityStd are reductions over the N x N affinity: one
    streaming pass on the device (`sc_affinity_stats`), four doubles come back; on the factored
    route, whose affinity is never stored, one sweep of affinity row panels
    (FactoredAffinity.statistics) gives the same four doubles bit for bit;
  * AffinityGmmBic fits 1- and 2-component GMMs to the N^2/2 upper-band affinities: on the
    device for a device-resident affinity, one streaming pass per KMeans / EM step
    (`gmm_bic`, `sc_gmm_band_pass`), with scikit-learn's arithmetic and random draws; on the
    factored route over the packed band (FactoredAffinity.upper_band, `sc_gmm_band_pass_packed`),
    with the same sums bit for bit, held only while the check runs; a host ndarray still goes to
    scikit-learn;
  * FallbackClusterer as the probe of predict(), Agglomerative type: average-linkage cosine AHC
    on the device with scikit-learn's cluster count (agglomerative.CosineAverageLinkage); a host
    ndarray affinity still goes to scikit-learn;
  * FallbackClusterer as the probe of predict(), Naive type: the naive clusterer in one device
    launch that stops as soon as a second cluster opens (`sc_naive_cluster`); a host ndarray
    affinity still runs the host clusterer;
  * FallbackClusterer otherwise (inputs below `spectral_min_embeddings`,
    FallbackClusterer.predict): host for a host ndarray; a CUDA tensor stays on the device
    (sc_naive_cluster for the Naive type, agglomerative.CosineAverageLinkage for the Agglomerative
    type), with the labels the host call on its twin returns.
"""

from __future__ import annotations

import dataclasses
import enum
import typing

import numpy as np

from . import naive_clusterer


class SingleClusterCondition(enum.Enum):
  AffinityGmmBic = enum.auto()      # BIC of a 1- vs 2-component GMM on the affinities
  AllAffinity = enum.auto()         # every affinity above the threshold
  NeighborAffinity = enum.auto()    # every affinity[i, i+1] above the threshold
  AffinityStd = enum.auto()         # standard deviation of the affinities below the threshold
  FallbackClusterer = enum.auto()   # the fallback clusterer finds one cluster


class FallbackClustererType(enum.Enum):
  Agglomerative = enum.auto()
  Naive = enum.auto()


@dataclasses.dataclass
class FallbackOptions:
  spectral_min_embeddings: int = 1
  single_cluster_condition: SingleClusterCondition = SingleClusterCondition.AffinityGmmBic
  single_cluster_affinity_threshold: float = 0.75
  single_cluster_affinity_diagonal_offset: int = 1
  fallback_clusterer_type: FallbackClustererType = FallbackClustererType.Naive
  agglomerative_threshold: float = 0.5
  naive_threshold: float = 0.5
  naive_adaptation_threshold: typing.Optional[float] = None


class FallbackClusterer:
  """fallback_clusterer.py:95-124."""

  def __init__(self, options: FallbackOptions):
    self.options = options
    kind = options.fallback_clusterer_type
    if kind == FallbackClustererType.Agglomerative:
      from sklearn.cluster import AgglomerativeClustering
      self.clusterer = AgglomerativeClustering(
          n_clusters=None, metric="cosine", linkage="average",
          distance_threshold=options.agglomerative_threshold)
    elif kind == FallbackClustererType.Naive:
      self.clusterer = naive_clusterer.NaiveClusterer(
          threshold=options.naive_threshold,
          adaptation_threshold=options.naive_adaptation_threshold)
    # any other value: the reference builds a ValueError without raising it (:121, SURVEY.md
    # A.4-4) and fails later with AttributeError in predict(); same here.

  def predict(self, embeddings) -> np.ndarray:
    """Labels of the rows of an ndarray, or of a CUDA tensor on the device: what the host call on
    its twin (X.cpu().numpy(); for bfloat16, X.float().cpu().numpy()) returns."""
    if naive_clusterer._is_cuda_tensor(embeddings):
      from . import device as dev
      x = dev.twin(embeddings.detach())
      if self.options.fallback_clusterer_type == FallbackClustererType.Agglomerative:
        from . import agglomerative
        return agglomerative.CosineAverageLinkage(
            self.options.agglomerative_threshold).fit_predict(x)
      return self.clusterer.fit_predict(x)
    return self.clusterer.fit_predict(embeddings)


def affinity_statistics(affinity) -> typing.Dict[str, float]:
  """{min, neighbor_min, std} of a host ndarray, a device-resident affinity or the FactoredAffinity
  of the factored route."""
  if isinstance(affinity, np.ndarray):
    return dict(min=float(affinity.min()),
                neighbor_min=float(np.diag(affinity, k=1).min()) if affinity.shape[0] > 1 else np.inf,
                std=float(np.std(affinity)))
  import ctypes
  from . import device as dev
  eng = dev.Engine.get()
  if isinstance(affinity, dev.FactoredAffinity):
    return affinity.statistics(eng)
  out = np.zeros(4, dtype=np.float64)
  n = affinity.n
  eng.call("sc_affinity_stats", dev._ptr(affinity.matrix), n, affinity.matrix.stride(0),
           out.ctypes.data_as(ctypes.c_void_p), eng.stream)
  return statistics_from_sums(out, n)


def statistics_from_sums(out, n: int) -> typing.Dict[str, float]:
  """{min, neighbor_min, std} from sc_affinity_stats's (min, sum, sum of squares, neighbour min)."""
  count = float(n) * float(n)
  mean = out[1] / count
  var = max(out[2] / count - mean * mean, 0.0)
  return dict(min=float(out[0]), neighbor_min=float(out[3]), std=float(np.sqrt(var)))


def check_single_cluster(fallback_options: FallbackOptions,
                         embeddings: typing.Optional[np.ndarray], affinity,
                         details: typing.Optional[dict] = None,
                         embeddings_dev=None) -> bool:
  """True when the data form a single cluster (only consulted when min_clusters == 1).

  `affinity` is a host ndarray (reference signature), or the DeviceAffinity or FactoredAffinity
  predict() holds; the two device forms give the same verdict and `details`, bit for bit.
  For AffinityGmmBic on a device affinity, `details` (if given) receives the two BICs, both
  GMMs' EM iteration counts and the number of passes over the affinity.  Both fallback clusterer
  types on a device affinity run on the device too, on `embeddings_dev` (the embeddings as a CUDA
  tensor, read as its host twin's dtype: fp16 as fp64, bf16 as fp32) when given and on an uploaded
  copy of `embeddings` otherwise; the Naive type stops at the second cluster and records the
  embeddings it processed and the clusters it opened in `details`."""
  cond = fallback_options.single_cluster_condition
  thr = fallback_options.single_cluster_affinity_threshold
  if cond == SingleClusterCondition.AllAffinity:
    return affinity_statistics(affinity)["min"] > thr
  if cond == SingleClusterCondition.NeighborAffinity:
    return affinity_statistics(affinity)["neighbor_min"] > thr
  if cond == SingleClusterCondition.AffinityStd:
    return affinity_statistics(affinity)["std"] < thr
  if cond == SingleClusterCondition.AffinityGmmBic:
    n = affinity.shape[0] if isinstance(affinity, np.ndarray) else affinity.n
    offset = fallback_options.single_cluster_affinity_diagonal_offset
    if offset >= n - 1:
      raise ValueError("single_cluster_affinity_diagonal_offset must be significantly "
                       "smaller than affinity matrix dimension")
    if not isinstance(affinity, np.ndarray):
      from . import device as dev
      from . import gmm_bic
      eng = dev.Engine.get()
      if isinstance(affinity, dev.FactoredAffinity):
        # the packed band lives only for the check: refine() allocates Y_hi after it is freed
        band, row_off = affinity.upper_band(eng, offset)
        res = gmm_bic.gmm_bic(gmm_bic.DeviceOps(eng, band, n, offset, row_off))
        del band, row_off
      else:
        res = gmm_bic.gmm_bic(gmm_bic.DeviceOps(eng, affinity.matrix, n, offset))
      if details is not None:
        details.update(bic=res.bic, n_iter=res.n_iter, passes=res.passes)
      return res.single
    from sklearn.mixture import GaussianMixture
    values = affinity[np.triu_indices(n, offset)][:, None]
    bic = [GaussianMixture(n_components=c).fit(values).bic(values) for c in (1, 2)]
    return bool(bic[0] < bic[1])
  if cond == SingleClusterCondition.FallbackClusterer:
    kind = fallback_options.fallback_clusterer_type
    if kind == FallbackClustererType.Agglomerative and not isinstance(affinity, np.ndarray):
      from . import agglomerative
      from . import device as dev
      probe = agglomerative.CosineAverageLinkage(fallback_options.agglomerative_threshold)
      probe.fit_predict(embeddings if embeddings_dev is None else dev.twin(embeddings_dev))
      return probe.n_clusters_ == 1
    if kind == FallbackClustererType.Naive and not isinstance(affinity, np.ndarray):
      from . import device as dev
      probe = naive_clusterer.NaiveClusterer(fallback_options.naive_threshold,
                                             fallback_options.naive_adaptation_threshold)
      eng = dev.Engine.get()
      x = None if embeddings_dev is None else dev.twin(embeddings_dev)
      if x is None:
        x = np.ascontiguousarray(embeddings)
        if x.dtype not in (np.float32, np.float64):
          x = x.astype(np.float64)
        x = dev.torch().from_numpy(x).to(eng.device)
      _, processed, clusters, _, _ = eng.naive_cluster(x, probe.threshold,
                                                       probe.adaptation_threshold, stop_at=2)
      if details is not None:
        details.update(processed=processed, n_clusters=clusters)
      return clusters == 1
    labels = FallbackClusterer(fallback_options).predict(embeddings)
    return bool(np.unique(labels).size == 1)
  raise TypeError("Unsupported single_cluster_condition")
