"""CPU: the host half of CosineAverageLinkage (sort of the merges, scipy's relabelling, scikit-learn's
distance-threshold cut) on top of a NumPy restatement of the average-linkage NN-chain the device
kernel follows, against scipy `linkage(..., "average")` bit for bit and scikit-learn
`AgglomerativeClustering(linkage="average", distance_threshold=t)` integer for integer, including
exact ties and thresholds equal to a merge distance; input errors; the device/host choice by free
device memory; and which single-cluster checks stay on the host."""

import numpy as np
import pytest
from scipy.cluster import hierarchy
from scipy.spatial import distance
from sklearn.cluster import AgglomerativeClustering
from sklearn.utils._param_validation import InvalidParameterError

from spectralcluster_b200 import agglomerative as agg
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import fallback_clusterer as fb


def nn_chain_average(dist):
  """scipy's `_hierarchy.nn_chain` for average linkage with the chain rules of
  nn_chain_numpy.nn_chain_complete (the device kernel's); the update after merging x < y is scipy's
  `_average`, (nx d_xi + ny d_yi) / (nx + ny), with each product, the sum and the quotient rounded
  in turn.  Returns the merges in chain order, unsorted and unrelabelled."""
  d = np.array(dist, dtype=np.float64, copy=True)
  n = d.shape[0]
  size = np.ones(n, dtype=np.int64)
  xy = np.empty((n - 1, 2), dtype=np.int64)
  md = np.empty(n - 1, dtype=np.float64)
  ms = np.empty(n - 1, dtype=np.int64)
  chain = []
  for k in range(n - 1):
    if not chain:
      chain.append(int(np.flatnonzero(size)[0]))
    while True:
      x = chain[-1]
      if len(chain) > 1:
        y, best = chain[-2], d[x, chain[-2]]
      else:
        y, best = -1, np.inf
      cand = np.flatnonzero(size)
      cand = cand[cand != x]
      j = int(np.argmin(d[x, cand]))            # first index holding the minimum
      if d[x, cand[j]] < best:
        y, best = int(cand[j]), d[x, cand[j]]
      if len(chain) > 1 and y == chain[-2]:
        break
      chain.append(y)
    del chain[-2:]
    a, b = min(x, y), max(x, y)
    xy[k] = a, b
    md[k] = best
    ms[k] = size[a] + size[b]
    na, nb = float(size[a]), float(size[b])
    size[b] += size[a]
    size[a] = 0
    keep = size > 0
    keep[b] = False
    prod_a = np.multiply(na, d[a, keep])
    prod_b = np.multiply(nb, d[b, keep])
    d[b, keep] = d[keep, b] = np.divide(np.add(prod_a, prod_b), na + nb)
  return xy, md, ms


def integer_ties(n, top, seed):
  """Symmetric distances in {1..top}: masses of exact ties."""
  rng = np.random.default_rng(seed)
  d = np.triu(rng.integers(1, top + 1, size=(n, n)).astype(np.float64), 1)
  return d + d.T


def restated_z(dist):
  xy, md, _ = nn_chain_average(dist)
  return agg.linkage_matrix(xy, md, dist.shape[0])


def assert_bitwise(a, b):
  np.testing.assert_array_equal(np.asarray(a).view(np.int64), np.asarray(b).view(np.int64))


@pytest.mark.parametrize("n,d,seed", [(2, 3, 0), (3, 2, 1), (50, 8, 2), (300, 32, 3), (800, 64, 4)])
def test_random_data_matches_scipy_bitwise(n, d, seed):
  y = distance.pdist(np.random.default_rng(seed).standard_normal((n, d)), "cosine")
  assert_bitwise(restated_z(distance.squareform(y)), hierarchy.linkage(y, "average"))


@pytest.mark.parametrize("seed", range(10))
def test_exact_ties_match_scipy_bitwise(seed):
  n = 2 + seed * 7
  dist = integer_ties(n, 1 + seed % 4, seed)
  assert_bitwise(restated_z(dist), hierarchy.linkage(distance.squareform(dist), "average"))


def sklearn_precomputed(dist, t):
  return AgglomerativeClustering(n_clusters=None, metric="precomputed", linkage="average",
                                 distance_threshold=t).fit(dist)


def check_cut(dist, t):
  z = restated_z(dist)
  k, labels = agg.threshold_cut(t, z[:, :2].astype(np.intp), z[:, 2], dist.shape[0])
  ref = sklearn_precomputed(dist, t)
  assert k == ref.n_clusters_, t
  np.testing.assert_array_equal(labels, ref.labels_, err_msg=str(t))
  assert labels.dtype == ref.labels_.dtype
  return z


@pytest.mark.parametrize("seed", range(6))
def test_threshold_cut_matches_sklearn(seed):
  dist = integer_ties(20 + 13 * seed, 3 + seed % 3, 100 + seed)
  z = hierarchy.linkage(distance.squareform(dist), "average")
  merges = np.unique(z[:, 2])
  assert merges.size >= 3
  check_cut(dist, 0.0)                                   # every merge undone
  for lo, hi in zip(merges[:-1], merges[1:]):
    check_cut(dist, (lo + hi) / 2)                       # between two merge distances
  for m in merges:
    check_cut(dist, float(m))                            # exactly a merge distance: it is undone
  check_cut(dist, float(merges[-1]) + 0.5)               # one cluster


@pytest.mark.parametrize("t", [0.0, 0.3, 0.5, 0.9, 3.0])
def test_threshold_cut_on_cosine_data_matches_sklearn(t):
  x = np.random.default_rng(8).standard_normal((300, 16))
  dist = distance.squareform(distance.pdist(x, "cosine"))
  z = restated_z(dist)
  k, labels = agg.threshold_cut(t, z[:, :2].astype(np.intp), z[:, 2], 300)
  ref = AgglomerativeClustering(n_clusters=None, metric="cosine", linkage="average",
                                distance_threshold=t).fit(x)
  assert k == ref.n_clusters_
  np.testing.assert_array_equal(labels, ref.labels_)
  assert_bitwise(z[:, 2], ref.distances_)


class _NoDevice(Exception):
  pass


def _no_device(cls, device=None):
  raise _NoDevice()


def test_input_errors_match_sklearn_before_the_device(monkeypatch):
  monkeypatch.setattr(dev.Engine, "get", classmethod(_no_device))
  x = np.random.default_rng(0).standard_normal((6, 3))
  nan, inf = x.copy(), x.copy()
  nan[2, 1], inf[4, 0] = np.nan, np.inf
  cases = [(x[:1], 0.5), (nan, 0.5), (inf, 0.5), (np.vstack([x, np.zeros((1, 3))]), 0.5),
           (x, -0.1), (x, float("nan")), (x[None], 0.5)]
  for data, t in cases:
    with pytest.raises(Exception) as want:
      AgglomerativeClustering(n_clusters=None, metric="cosine", linkage="average",
                              distance_threshold=t).fit_predict(data)
    with pytest.raises(want.type):
      agg.CosineAverageLinkage(t).fit_predict(data)
  with pytest.raises(InvalidParameterError):
    agg.CosineAverageLinkage(-1e-300).fit_predict(x)


def test_constructor_needs_no_gpu():
  assert agg.CosineAverageLinkage(0.25).distance_threshold == 0.25


class _DeviceChosen(Exception):
  pass


class _StubEngine:
  device = "cpu"

  def cosine_distances(self, x_dev):
    raise _DeviceChosen()


def test_host_path_only_when_the_distances_do_not_fit(monkeypatch):
  import torch
  x = np.random.default_rng(4).standard_normal((60, 8))
  need = agg.distance_bytes(60) + x.nbytes
  monkeypatch.setattr(dev.Engine, "get", classmethod(lambda cls, device=None: _StubEngine()))
  monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (need, 80 << 30))
  with pytest.raises(_DeviceChosen):
    agg.CosineAverageLinkage(0.5).fit_predict(x)
  monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (need - 1, 80 << 30))
  c = agg.CosineAverageLinkage(0.5)
  ref = AgglomerativeClustering(n_clusters=None, metric="cosine", linkage="average",
                                distance_threshold=0.5).fit(x)
  np.testing.assert_array_equal(c.fit_predict(x), ref.labels_)
  np.testing.assert_array_equal(c.children_, ref.children_)
  np.testing.assert_array_equal(c.distances_, ref.distances_)
  assert (c.n_clusters_, c.n_leaves_) == (ref.n_clusters_, 60)


def test_device_fits_counts_the_allocator_cache(monkeypatch):
  """Free memory short of the request: the allocator's unused blocks are released and free memory
  is read again."""
  import torch
  state = dict(free=100, cached=50, emptied=0)

  def empty_cache():
    state["free"] += state["cached"]
    state["cached"] = 0
    state["emptied"] += 1

  monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (state["free"], 1000))
  monkeypatch.setattr(torch.cuda, "empty_cache", empty_cache)
  eng = _StubEngine()
  assert agg.device_fits(eng, 100) and state["emptied"] == 0        # enough: the cache is kept
  assert agg.device_fits(eng, 150) and state["emptied"] == 1
  assert not agg.device_fits(eng, 151) and state["emptied"] == 2


class _FakeDeviceAffinity:
  n = 40


@pytest.mark.parametrize("t", [0.2, 2.5])
def test_probe_choice(monkeypatch, t):
  """Agglomerative probe: a device affinity takes CosineAverageLinkage (here forced onto its host
  path), a host ndarray affinity and FallbackClusterer.predict take scikit-learn without touching
  the device; the verdicts agree."""
  import torch
  x = np.random.default_rng(5).standard_normal((40, 6))
  opts = fb.FallbackOptions(single_cluster_condition=fb.SingleClusterCondition.FallbackClusterer,
                            fallback_clusterer_type=fb.FallbackClustererType.Agglomerative,
                            agglomerative_threshold=t)
  want = AgglomerativeClustering(n_clusters=None, metric="cosine", linkage="average",
                                 distance_threshold=t).fit(x).n_clusters_ == 1
  monkeypatch.setattr(dev.Engine, "get", classmethod(_no_device))
  assert fb.check_single_cluster(opts, x, np.eye(40)) == want
  assert (np.unique(fb.FallbackClusterer(opts).predict(x)).size == 1) == want
  with pytest.raises(_NoDevice):
    fb.check_single_cluster(opts, x, _FakeDeviceAffinity())
  monkeypatch.setattr(dev.Engine, "get", classmethod(lambda cls, device=None: _StubEngine()))
  monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (0, 80 << 30))
  assert fb.check_single_cluster(opts, x, _FakeDeviceAffinity()) == want
