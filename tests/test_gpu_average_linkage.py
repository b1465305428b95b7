"""GPU: average-linkage cosine agglomerative clustering on the device (sc_average_linkage,
agglomerative.CosineAverageLinkage) against scipy `linkage(..., "average")` bit for bit and
scikit-learn `AgglomerativeClustering(linkage="average", distance_threshold=t)`, and the
FallbackClusterer / Agglomerative single-cluster check it runs inside predict() against the same
check in scikit-learn."""

import os

import numpy as np
import pytest
from scipy.cluster import hierarchy
from scipy.spatial import distance
from sklearn.cluster import AgglomerativeClustering
from sklearn.cluster._agglomerative import _hc_cut

import spectralcluster_b200 as scb
from spectralcluster_b200 import agglomerative as agg
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import synthetic

from test_average_linkage_cpu import nn_chain_average

pytestmark = pytest.mark.gpu


def upload(engine, dist):
  t = dev.torch()
  n = dist.shape[0]
  dm = engine.matrix(n, t.float64).fill_(float("nan"))
  dm[:, :n].copy_(t.from_numpy(np.ascontiguousarray(dist)))
  return dm


def assert_bitwise(a, b, msg=""):
  np.testing.assert_array_equal(np.asarray(a).view(np.int64), np.asarray(b).view(np.int64),
                                err_msg=msg)


@pytest.mark.parametrize("n", [2, 3, 63, 64, 65, 1000, 4097])
def test_scipy_distances_give_scipys_tree_bitwise(engine, n):
  y = distance.pdist(np.random.default_rng(n).standard_normal((n, 24)), "cosine")
  xy, md, sz = engine.average_linkage(upload(engine, distance.squareform(y)), n)
  z = agg.linkage_matrix(xy, md, n)
  assert_bitwise(z, hierarchy.linkage(y, "average"))
  np.testing.assert_array_equal(sz[np.argsort(md, kind="mergesort")], z[:, 3])


def tie_matrices():
  rng = np.random.default_rng(12)
  for n, top in ((2, 1), (3, 1), (9, 2), (29, 3), (64, 2), (200, 4), (2000, 5)):
    d = np.triu(rng.integers(1, top + 1, size=(n, n)).astype(np.float64), 1)
    yield d + d.T
  base = rng.standard_normal((6, 8))
  x = base[rng.integers(0, 6, size=1200)]            # duplicated points: zero distances tie
  yield distance.squareform(distance.pdist(x, "cosine"))


def test_chain_order_equals_restatement_on_exact_ties(engine):
  for dist in tie_matrices():
    n = dist.shape[0]
    xy, md, sz = engine.average_linkage(upload(engine, dist), n)
    want_xy, want_md, want_sz = nn_chain_average(dist)
    np.testing.assert_array_equal(xy, want_xy, err_msg=str(n))
    assert_bitwise(md, want_md, str(n))
    np.testing.assert_array_equal(sz, want_sz, err_msg=str(n))
    assert_bitwise(agg.linkage_matrix(xy, md, n),
                   hierarchy.linkage(distance.squareform(dist, checks=False), "average"), str(n))


def sklearn_average(t):
  return AgglomerativeClustering(n_clusters=None, metric="cosine", linkage="average",
                                 distance_threshold=t)


@pytest.mark.parametrize("n", [1000, 4096, 8192])
def test_end_to_end_matches_sklearn(n):
  x = synthetic.speaker_turn_dvectors(n, 256, 8, seed=n)
  src = x.astype(np.float32) if n == 4096 else x
  for t in (0.3, 0.5, 0.9):
    c = agg.CosineAverageLinkage(t)
    labels = c.fit_predict(src)
    ref = sklearn_average(t).fit(src)
    np.testing.assert_array_equal(labels, ref.labels_, err_msg=str(t))
    np.testing.assert_array_equal(c.children_, ref.children_, err_msg=str(t))
    assert c.n_clusters_ == ref.n_clusters_ and c.n_leaves_ == n
    assert np.abs(c.distances_ - ref.distances_).max() <= 1e-14
    assert labels.dtype == ref.labels_.dtype
  # a CUDA tensor is read in place and gives the same answer
  xd = dev.torch().from_numpy(src).to(dev.Engine.get().device)
  c2 = agg.CosineAverageLinkage(0.9)
  np.testing.assert_array_equal(c2.fit_predict(xd), labels)
  assert c2.n_clusters_ == c.n_clusters_


def test_16384_matches_scipy_tree_and_sklearn_cut():
  n = 16384
  x = synthetic.speaker_turn_dvectors(n, 256, 8, seed=n)
  want = hierarchy.linkage(distance.pdist(x, "cosine"), "average")
  children = want[:, :2].astype(np.intp)
  for t in (0.3, 0.5, 0.9):
    c = agg.CosineAverageLinkage(t)
    labels = c.fit_predict(x)
    np.testing.assert_array_equal(c.children_, children)
    assert np.abs(c.distances_ - want[:, 2]).max() <= 1e-14
    k = np.count_nonzero(want[:, 2] >= t) + 1
    assert c.n_clusters_ == k
    np.testing.assert_array_equal(labels, _hc_cut(k, children, n))


# ---- the single-cluster check inside predict()

def clusterer(threshold=0.5):
  return scb.SpectralClusterer(
      min_clusters=1, max_clusters=7, laplacian_type=scb.LaplacianType.GraphCut,
      fallback_options=scb.FallbackOptions(
          single_cluster_condition=scb.SingleClusterCondition.FallbackClusterer,
          fallback_clusterer_type=scb.FallbackClustererType.Agglomerative,
          agglomerative_threshold=threshold),
      refinement_options=scb.RefinementOptions(
          gaussian_blur_sigma=1, p_percentile=0.95,
          refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)))


def refuse_host(monkeypatch):
  def refuse(self, x):
    raise AssertionError("the scikit-learn path of CosineAverageLinkage ran")
  monkeypatch.setattr(agg.CosineAverageLinkage, "_fit_predict_host", refuse)


def inputs():
  z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "callers",
                           "predict_callers.npz"))
  yield "x1", z["x1"], True
  yield "x4", z["x4"], False
  yield "one speaker", synthetic.speaker_turn_dvectors(3000, 128, 1, seed=7), True
  yield "four speakers", synthetic.speaker_turn_dvectors(3000, 128, 4, seed=7), False


def test_predict_probe_matches_sklearn_probe_and_out_of_memory_fallback(monkeypatch):
  """The device probe against the same predict() with no free device memory, where the probe is
  scikit-learn's AgglomerativeClustering."""
  import torch
  host_calls = []
  host = agg.CosineAverageLinkage._fit_predict_host
  for name, x, single in inputs():
    with monkeypatch.context() as m:
      refuse_host(m)
      got = clusterer().predict(x)
    with monkeypatch.context() as m:
      m.setattr(torch.cuda, "mem_get_info", lambda device=None: (0, 80 << 30))
      m.setattr(agg.CosineAverageLinkage, "_fit_predict_host",
                lambda self, xh: host_calls.append(name) or host(self, xh))
      want = clusterer().predict(x)
    assert host_calls[-1] == name
    np.testing.assert_array_equal(got, want, err_msg=name)
    assert (np.unique(got).size == 1) == single, name


SINGLE = np.array([[1.0, 0.0], [1.1, 0.1], [1.0, 0.0], [1.1, 0.0], [0.9, -0.1], [1.0, 0.2]])
OUTLIER_MID = np.array([[1.0, 0.0], [1.1, 0.1], [1.0, 0.0], [1.0, 0.5], [1.1, 0.0], [0.9, -0.1]])


def test_reference_6x2_known_answers_with_the_agglomerative_probe(monkeypatch):
  # average-linkage merge distances: SINGLE tops out at 0.022, OUTLIER_MID at 0.109
  refuse_host(monkeypatch)
  ordered = scb.utils.enforce_ordered_labels
  for x, thr, want in ((SINGLE, 0.05, [0] * 6), (OUTLIER_MID, 0.05, [0, 0, 0, 1, 0, 0]),
                       (OUTLIER_MID, 0.2, [0] * 6)):
    assert (sklearn_average(thr).fit(x).n_clusters_ == 1) == (want == [0] * 6)
    c = scb.SpectralClusterer(
        min_clusters=1, laplacian_type=scb.LaplacianType.GraphCut, refinement_options=None,
        fallback_options=scb.FallbackOptions(
            single_cluster_condition=scb.SingleClusterCondition.FallbackClusterer,
            fallback_clusterer_type=scb.FallbackClustererType.Agglomerative,
            agglomerative_threshold=thr))
    np.testing.assert_array_equal(ordered(c.predict(x)), want)


def test_consecutive_predicts_at_32768_stay_on_the_device(monkeypatch):
  refuse_host(monkeypatch)
  x = synthetic.speaker_turn_dvectors(32768, 128, 4, seed=5)
  c = clusterer()
  first = c.predict(x)
  second = c.predict(x)
  np.testing.assert_array_equal(first, second)
  assert np.unique(first).size > 1


def test_blocks_cached_by_torch_count_as_free(monkeypatch, engine):
  """Free device memory one byte short of the distance matrix, but the allocator holds a released
  block as large: the probe still runs on the device."""
  import torch
  n = 8192
  x = synthetic.speaker_turn_dvectors(n, 128, 4, seed=2)
  want = agg.CosineAverageLinkage(0.5)
  want.fit_predict(x)
  need = agg.distance_bytes(n) + x.nbytes
  torch.cuda.empty_cache()                              # the block below gets a segment of its own
  blob = torch.empty(need, dtype=torch.uint8, device=engine.device)
  del blob                                              # cached by the allocator, not free
  real = torch.cuda.mem_get_info
  hidden = real(engine.device)[0] - (need - 1)
  monkeypatch.setattr(torch.cuda, "mem_get_info",
                      lambda device=None: (real(device)[0] - hidden, real(device)[1]))
  refuse_host(monkeypatch)
  c = agg.CosineAverageLinkage(0.5)
  np.testing.assert_array_equal(c.fit_predict(x), want.labels_)
  assert c.n_clusters_ == want.n_clusters_
