"""CPU: the host half of CosineCompleteLinkage (sort of the merges, scipy's relabelling,
scikit-learn's heap cut) on top of a NumPy restatement of the NN-chain rules the device kernel
follows, against scipy `linkage(..., "complete")` row for row and scikit-learn
`AgglomerativeClustering(linkage="complete")` integer for integer, including inputs with exact ties;
input errors; and the choice between the device and the scikit-learn path by free device memory."""

import numpy as np
import pytest
from scipy.cluster import hierarchy
from scipy.spatial import distance
from sklearn.cluster import AgglomerativeClustering

import spectralcluster_b200 as scb
from spectralcluster_b200 import agglomerative as agg
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import multi_stage_clusterer as ms

from nn_chain_numpy import nn_chain_complete


def integer_ties(n, top, seed):
  """Symmetric distances in {1..top}: masses of exact ties."""
  rng = np.random.default_rng(seed)
  d = rng.integers(1, top + 1, size=(n, n)).astype(np.float64)
  d = np.triu(d, 1)
  return d + d.T


def duplicated_points(n, distinct, dim, seed):
  rng = np.random.default_rng(seed)
  base = rng.standard_normal((distinct, dim))
  return base[rng.integers(0, distinct, size=n)]


def restated(dist, n_clusters):
  n = dist.shape[0]
  xy, md, _ = nn_chain_complete(dist)
  z = agg.linkage_matrix(xy, md, n)
  return z, agg.hc_cut(n_clusters, z[:, :2].astype(np.intp), n)


@pytest.mark.parametrize("n,d,seed", [(2, 3, 0), (3, 2, 1), (40, 8, 2), (257, 16, 3)])
def test_random_data_matches_scipy_and_sklearn(n, d, seed):
  x = np.random.default_rng(seed).standard_normal((n, d))
  dist = distance.squareform(distance.pdist(x, "cosine"))
  want = hierarchy.linkage(distance.pdist(x, "cosine"), "complete")
  for k in sorted({1, 2, min(5, n), min(17, n), n}):
    z, labels = restated(dist, k)
    np.testing.assert_array_equal(z, want)
    ref = AgglomerativeClustering(n_clusters=k, metric="cosine", linkage="complete").fit_predict(x)
    np.testing.assert_array_equal(labels, ref)
    assert labels.dtype == ref.dtype


@pytest.mark.parametrize("seed", range(12))
def test_exact_ties_match_scipy_and_sklearn(seed):
  n = 2 + seed * 3
  dist = integer_ties(n, 1 + seed % 4, seed)
  want = hierarchy.linkage(distance.squareform(dist), "complete")
  for k in sorted({1, 2, max(1, n // 3), n}):
    z, labels = restated(dist, k)
    np.testing.assert_array_equal(z, want)
    ref = AgglomerativeClustering(n_clusters=k, metric="precomputed",
                                  linkage="complete").fit_predict(dist)
    np.testing.assert_array_equal(labels, ref)


@pytest.mark.parametrize("n,distinct,seed", [(12, 3, 0), (30, 5, 1), (61, 4, 2), (90, 20, 3)])
def test_duplicated_points_match_scipy_and_sklearn(n, distinct, seed):
  x = duplicated_points(n, distinct, 6, seed)
  dist = distance.squareform(distance.pdist(x, "cosine"))
  want = hierarchy.linkage(distance.pdist(x, "cosine"), "complete")
  for k in sorted({1, distinct, n}):
    z, labels = restated(dist, k)
    np.testing.assert_array_equal(z, want)
    ref = AgglomerativeClustering(n_clusters=k, metric="cosine", linkage="complete").fit_predict(x)
    np.testing.assert_array_equal(labels, ref)


def test_constructors_need_no_gpu():
  c = agg.CosineCompleteLinkage(n_clusters=7)
  assert c.n_clusters == 7
  stream = ms.MultiStageClusterer(scb.SpectralClusterer(), U1=40)
  assert isinstance(stream.pre, agg.CosineCompleteLinkage) and stream.pre.n_clusters == 40


def test_input_errors_match_sklearn():
  x = np.random.default_rng(0).standard_normal((6, 3))
  cases = [(x[:1], 1), (x, 7), (np.vstack([x, np.zeros((1, 3))]), 2)]
  for data, k in cases:
    with pytest.raises(ValueError):
      AgglomerativeClustering(n_clusters=k, metric="cosine", linkage="complete").fit_predict(data)
    with pytest.raises(ValueError):
      agg.CosineCompleteLinkage(n_clusters=k).fit_predict(data)


class _DeviceChosen(Exception):
  pass


class _StubEngine:
  device = "cpu"

  def cosine_distances(self, x_dev):
    raise _DeviceChosen()


def test_host_path_only_when_the_distances_do_not_fit(monkeypatch):
  import torch
  x = np.random.default_rng(4).standard_normal((50, 8)).astype(np.float32)
  need = agg.distance_bytes(50) + x.nbytes
  assert need == 8 * 50 * 64 + x.nbytes
  monkeypatch.setattr(dev.Engine, "get", classmethod(lambda cls, device=None: _StubEngine()))
  monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (need, 80 << 30))
  with pytest.raises(_DeviceChosen):
    agg.CosineCompleteLinkage(n_clusters=4).fit_predict(x)
  monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (need - 1, 80 << 30))
  c = agg.CosineCompleteLinkage(n_clusters=4)
  ref = AgglomerativeClustering(n_clusters=4, metric="cosine", linkage="complete").fit(x)
  np.testing.assert_array_equal(c.fit_predict(x), ref.labels_)
  np.testing.assert_array_equal(c.children_, ref.children_)
  assert c.n_leaves_ == 50
