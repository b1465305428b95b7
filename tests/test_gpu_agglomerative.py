"""GPU: complete-linkage cosine agglomerative clustering on the device (sc_cosine_distances_f64,
sc_complete_linkage, agglomerative.CosineCompleteLinkage) against scipy pdist / linkage and
scikit-learn AgglomerativeClustering, and its two callers (max_spectral_size pre-clustering and
MultiStageClusterer) against the same callers with scikit-learn as the pre-clusterer."""

import ctypes

import numpy as np
import pytest
from scipy.cluster import hierarchy
from scipy.spatial import distance
from sklearn.cluster import AgglomerativeClustering

import spectralcluster_b200 as scb
from spectralcluster_b200 import agglomerative as agg
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import multi_stage_clusterer as ms
from spectralcluster_b200 import synthetic
from spectralcluster_b200 import utils

from nn_chain_numpy import nn_chain_complete

pytestmark = pytest.mark.gpu


def distances_prefilled(engine, x):
  """sc_cosine_distances_f64 into a NaN-prefilled buffer -> (host [n, n], flag)."""
  t = dev.torch()
  xd = t.from_numpy(np.ascontiguousarray(x)).to(engine.device)
  n, d = x.shape
  out = engine.matrix(n, t.float64).fill_(float("nan"))
  flag = t.full((1,), -1, dtype=t.int32, device=engine.device)
  engine.call("sc_cosine_distances_f64", ctypes.c_void_p(xd.data_ptr()),
              1 if x.dtype == np.float64 else 0, n, d, xd.stride(0),
              ctypes.c_void_p(out.data_ptr()), out.stride(0), ctypes.c_void_p(flag.data_ptr()),
              engine.stream)
  return out[:, :n].cpu().numpy(), int(flag.item())


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d", [2, 32, 256])
@pytest.mark.parametrize("n", [2, 63, 64, 65, 1000, 4097])
def test_cosine_distances_match_pdist(engine, n, d, dtype):
  x = np.random.default_rng(n * 7 + d).standard_normal((n, d)).astype(dtype)
  got, flag = distances_prefilled(engine, x)
  assert flag == 0
  assert np.isfinite(got).all()
  np.testing.assert_array_equal(got.view(np.int64), got.T.view(np.int64))   # bitwise symmetric
  want = distance.squareform(distance.pdist(x.astype(np.float64), "cosine"))
  # scipy's own summation order is not a plain loop: even a correctly rounded dot product lands up
  # to 2.5 units in the last place of the distance away from pdist at these sizes (5.6e-16 at
  # n = 4097, d = 32).  Three units, 6.7e-16 for distances in [1, 2), bound the difference.
  assert (np.abs(got - want) <= 3 * np.spacing(np.maximum(want, 1.0))).all()


def test_zero_row_sets_the_nonfinite_flag(engine):
  x = np.random.default_rng(1).standard_normal((100, 16))
  x[37] = 0.0
  _, flag = distances_prefilled(engine, x)
  assert flag == 1


def tie_matrices():
  rng = np.random.default_rng(11)
  for n, top in ((2, 1), (3, 1), (9, 2), (29, 3), (64, 2), (200, 4), (3000, 5)):
    d = np.triu(rng.integers(1, top + 1, size=(n, n)).astype(np.float64), 1)
    yield d + d.T
  base = rng.standard_normal((6, 8))
  x = base[rng.integers(0, 6, size=1500)]            # duplicated points: zero distances tie
  yield distance.squareform(distance.pdist(x, "cosine"))


def test_linkage_chain_order_equals_restatement_on_exact_ties(engine):
  t = dev.torch()
  for dist in tie_matrices():
    n = dist.shape[0]
    dm = engine.matrix(n, t.float64)
    dm[:, :n].copy_(t.from_numpy(dist))
    xy, md, sz = engine.complete_linkage(dm, n)
    want_xy, want_md, want_sz = nn_chain_complete(dist)
    np.testing.assert_array_equal(xy, want_xy, err_msg=str(n))
    np.testing.assert_array_equal(md, want_md, err_msg=str(n))
    np.testing.assert_array_equal(sz, want_sz, err_msg=str(n))


@pytest.mark.parametrize("n,k", [(1000, 30), (4096, 300), (8192, 1024), (16384, 300)])
def test_end_to_end_matches_scipy_and_sklearn(engine, n, k):
  t = dev.torch()
  x = synthetic.speaker_turn_dvectors(n, 256, 8, seed=n)
  want = hierarchy.linkage(distance.pdist(x, "cosine"), "complete")
  dist, flag = engine.cosine_distances(t.from_numpy(x).to(engine.device))
  assert int(flag.item()) == 0
  xy, md, _ = engine.complete_linkage(dist, n)
  z = agg.linkage_matrix(xy, md, n)
  np.testing.assert_array_equal(z[:, :2], want[:, :2])
  assert np.abs(z[:, 2] - want[:, 2]).max() <= 1e-14
  np.testing.assert_array_equal(z[:, 3], want[:, 3])
  c = agg.CosineCompleteLinkage(n_clusters=k)
  labels = c.fit_predict(x.astype(np.float32) if n == 4096 else x)
  if n <= 8192:
    ref = AgglomerativeClustering(n_clusters=k, metric="cosine", linkage="complete")
    src = x.astype(np.float32) if n == 4096 else x
    np.testing.assert_array_equal(labels, ref.fit_predict(src))
    np.testing.assert_array_equal(c.children_, ref.children_)
  else:
    # the same cut scikit-learn makes, applied to scipy's tree (saves a second 16 s host linkage)
    from sklearn.cluster._agglomerative import _hc_cut
    np.testing.assert_array_equal(labels, _hc_cut(k, want[:, :2].astype(np.intp), n))
  assert labels.dtype == np.intp and c.n_leaves_ == n


def clusterer(**kw):
  return scb.SpectralClusterer(
      min_clusters=2, max_clusters=7,
      refinement_options=scb.RefinementOptions(
          gaussian_blur_sigma=0, p_percentile=0.95,
          refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)), **kw)


@pytest.mark.parametrize("size", [300, 1024])
def test_max_spectral_size_matches_sklearn_composition(size):
  x = synthetic.speaker_turn_dvectors(8192, 256, 6, seed=3)
  got = clusterer(max_spectral_size=size).predict(x)
  pre = AgglomerativeClustering(n_clusters=size, metric="cosine",
                                linkage="complete").fit_predict(x)
  want = utils.chain_labels(pre, clusterer().predict(utils.get_cluster_centroids(x, pre)))
  assert got.dtype == want.dtype == np.float64
  np.testing.assert_array_equal(got, want)


def test_stream_matches_sklearn_preclusterer_step_for_step():
  x = synthetic.speaker_turn_dvectors(700, 128, 4, seed=9)

  def stream():
    main = scb.SpectralClusterer(
        min_clusters=1, max_clusters=5,
        refinement_options=scb.RefinementOptions(
            gaussian_blur_sigma=0, p_percentile=0.9,
            refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)))
    return ms.MultiStageClusterer(main, fallback_threshold=0.5, L=50, U1=100, U2=600,
                                  deflicker=ms.Deflicker.Hungarian)

  got, ref = stream(), stream()
  assert isinstance(got.pre, agg.CosineCompleteLinkage)
  ref.pre = AgglomerativeClustering(n_clusters=100, metric="cosine", linkage="complete")
  for i in range(len(x)):
    np.testing.assert_array_equal(got.streaming_predict(x[i]), ref.streaming_predict(x[i]),
                                  err_msg=str(i))
