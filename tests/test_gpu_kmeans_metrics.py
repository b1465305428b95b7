"""GPU: sc_kmeans with the scipy metrics beyond cosine and euclidean, against the margin-checked
float64 restatement in kmeans_metrics_restatement.py.

Every case is first certified on the host (every decision beats twice its rounding bound), then the
device must return the restatement's labels bit for bit and the same number of assignment passes.
The sizes sit on the kernels' edges (256-thread blocks, the 1,024-chunk scan, the batch of 4 passes
between host reads), and the special values are scipy's: NaN from zero rows and constant columns,
inf from negative entries, numpy's LinAlgError and scipy's ValueError for mahalanobis."""

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import custom_distance_kmeans as cdk
from spectralcluster_b200 import device as dev

import kmeans_metrics_restatement as km
import kmeans_restatement as kr

pytestmark = pytest.mark.gpu

METRICS = km.METRICS


def device_kmeans(engine, e, k, metric, max_iter):
  t = dev.torch()
  x = t.from_numpy(np.ascontiguousarray(e, dtype=np.float64)).to(engine.device)
  return engine.kmeans(x, int(k), cdk._METRICS[metric], int(max_iter))


def check(engine, e, k, metric, max_iter=300):
  want = km.restate(e, k, metric, max_iter)
  assert want.certified, "not certified: %s" % "; ".join(want.failures[:4])
  labels, iters = device_kmeans(engine, e, k, metric, max_iter)
  bad = np.flatnonzero(labels != want.labels)
  assert bad.size == 0, "%d labels differ, first at row %d" % (bad.size, bad[0])
  assert iters == want.iters, (iters, want.iters)
  return want


def rows_for(metric, n, k, kd, spread, seed):
  """Unit rows, or positive rows for jensenshannon (unit rows have negative entries: all inf)."""
  if metric == "jensenshannon":
    return km.positive_rows(n, k, kd, spread, seed)
  return kr.unit_rows(n, k, kd, spread, seed)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("n", [255, 256, 257, 1023, 1024, 1025, 2049, 65536])
def test_n_edges(engine, metric, n):
  check(engine, rows_for(metric, n, 8, 8, 0.6, seed=n), 8, metric)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("k", [1, 2, 7, 8, 20, 21, 54, 55])
def test_k_trial_steps(engine, metric, k):
  """k_dim = max(k, 3): below that, correlation (centred 2-vectors are +-(a, -a): cosines of
  exactly +-1) and jensenshannon (one column: p = q = 1, a divergence of rounding size whose sign
  decides NaN) are decided by rounding alone, in scipy as anywhere.  For k <= 2 the Lloyd step
  already gives the final labels, so the second pass repeats the first in exact arithmetic and
  only rounding decides the stop rule (see test_gpu_kmeans.py): those run with max_iter = 1."""
  kd = max(k, 3)
  check(engine, rows_for(metric, 4096, k, kd, 0.3, seed=k), k, metric, 1 if k <= 2 else 300)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("k,kd", [(12, 3), (5, 40)])
def test_k_dim_differs_from_k(engine, metric, k, kd):
  e = rows_for(metric, 3000, k, kd, 0.4, seed=k * kd)
  w = check(engine, e, k, metric)
  np.testing.assert_array_equal(cdk.run_kmeans(e, k, metric, 300), w.labels)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("max_iter", [1, 2, 3, 4, 5, 300])
def test_max_iter(engine, metric, max_iter):
  check(engine, rows_for(metric, 2049, 20, 20, 1.0, seed=7), 20, metric, max_iter)


@pytest.fixture(scope="module")
def eigenvectors_65536(engine):
  """The eigenvectors predict() computes at N = 65,536 (6 speakers, ICASSP, max_clusters=10), as
  they come off the device: the first 6, as predict() hands them to run_kmeans."""
  from oracle import spectral_oracle as orc
  x = orc.synthetic_dvectors(65536, 256, 6, seed=0)
  box = []
  orig = scb.SpectralClusterer._compute_eigenvectors_ncluster

  def spy(self, *a, **kw):
    out = orig(self, *a, **kw)
    box.append(out[0].clone())
    return out

  with pytest.MonkeyPatch.context() as mp:
    mp.setattr(scb.SpectralClusterer, "_compute_eigenvectors_ncluster", spy)
    opts = scb.RefinementOptions(gaussian_blur_sigma=1, p_percentile=0.95,
                                 thresholding_soft_multiplier=0.01,
                                 refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))
    scb.SpectralClusterer(max_clusters=10, refinement_options=opts).predict(x)
  return box.pop()[:, :6].contiguous().cpu().numpy()


@pytest.mark.parametrize("metric", METRICS)
def test_device_eigenvectors_65536(engine, eigenvectors_65536, metric):
  """max_iter = 1, as in test_gpu_kmeans.py.  canberra's bound is unbounded where a term's
  denominator |x_f| + |c_f| is within a centroid's rounding of 0, which eigenvector entries near 0
  reach: a case the restatement cannot certify is skipped, naming the margin."""
  want = km.restate(eigenvectors_65536, 6, metric, 1)
  if not want.certified:
    pytest.skip("not certified: %s" % want.failures[0])
  check(engine, eigenvectors_65536, 6, metric, max_iter=1)


# ---------------------------------------------------------------- special values
def zero_rows_case():
  rng = np.random.default_rng(11)
  e = kr.unit_rows(1000, 4, 6, 0.5, seed=11) * rng.uniform(0.5, 2.0, (1000, 1))
  e[[417, 700]] = 0.0
  return e


@pytest.mark.parametrize("metric", ["braycurtis", "correlation"])
def test_zero_rows(engine, metric):
  """braycurtis: a zero row is exactly 1 from every centroid (label 0); correlation: NaN against
  every centroid (the first NaN, label 0) and the mean distance is NaN, so the loop runs to
  max_iter as in the reference."""
  w = check(engine, zero_rows_case(), 4, metric, max_iter=20)
  assert w.labels[417] == 0 and w.labels[700] == 0
  if metric == "correlation":
    assert w.iters == 21


def test_constant_column_seuclidean(engine):
  """V = 0 in a column that is constant in every row and centroid: every distance is 0/0 = NaN."""
  e = kr.unit_rows(1000, 4, 6, 0.5, seed=12)
  e[:, 2] = 0.5
  w = check(engine, e, 4, "seuclidean", max_iter=7)
  assert w.iters == 8 and not w.labels.any()


def test_negative_entries_jensenshannon(engine):
  """Spectral embeddings have negative entries: every distance is inf, as in scipy."""
  w = check(engine, zero_rows_case(), 4, "jensenshannon", max_iter=20)
  assert not w.labels.any() and w.iters == 2


@pytest.mark.parametrize("bad", ["zero", "twin"])
def test_mahalanobis_singular(engine, bad):
  e = kr.unit_rows(2000, 4, 6, 0.5, seed=3)
  if bad == "zero":
    e[:, 3] = 0.0
  else:
    e[:, 4] = e[:, 1]
  with pytest.raises(np.linalg.LinAlgError, match="Singular matrix"):
    km.restate(e, 4, "mahalanobis")
  with pytest.raises(np.linalg.LinAlgError, match="^Singular matrix$"):
    device_kmeans(engine, e, 4, "mahalanobis", 300)
  with pytest.raises(np.linalg.LinAlgError, match="^Singular matrix$"):
    cdk.run_kmeans(e, 4, "mahalanobis", 300)


def test_mahalanobis_too_few_observations(engine):
  e = np.random.default_rng(4).standard_normal((4, 9))
  msg = ("^The number of observations \\(6\\) is too small; the covariance matrix is singular. "
         "For observations with 9 dimensions, at least 10 observations are required.$")
  with pytest.raises(ValueError, match=msg):
    km.restate(e, 2, "mahalanobis")
  with pytest.raises(ValueError, match=msg):
    cdk.run_kmeans(e, 2, "mahalanobis", 300)


# ---------------------------------------------------------------- public entry points
@pytest.mark.parametrize("metric", METRICS)
def test_run_kmeans_makes_no_host_call(engine, monkeypatch, metric):
  """With scipy's cdist and scikit-learn's KMeans replaced by functions that raise, every device
  metric and each of its scipy spellings still clusters, with the same labels."""
  import scipy.spatial.distance
  import sklearn.cluster

  def boom(*a, **kw):
    raise AssertionError("host path used")

  e = rows_for(metric, 2049, 6, 6, 0.5, seed=61)
  want = km.restate(e, 6, metric)
  monkeypatch.setattr(scipy.spatial.distance, "cdist", boom)
  monkeypatch.setattr(sklearn.cluster, "KMeans", boom)
  for alias in cdk._ALIASES[metric]:
    got = cdk.run_kmeans(e, 6, alias, 300)
    if want.certified:
      np.testing.assert_array_equal(got, want.labels)


@pytest.mark.parametrize("metric", METRICS)
def test_predict_matches_oracle(metric):
  """predict(custom_dist=m) at N = 2,400 gives the oracle's labels."""
  from oracle import spectral_oracle as orc
  from test_gpu_predict import make_clusterer
  x = orc.synthetic_dvectors(2400, 64, 4, seed=3)
  opt = orc.options(min_clusters=2, max_clusters=6, sequence=orc.ICASSP2018)
  want = orc.predict(x, dict(opt, custom_dist=metric))
  c = make_clusterer(opt)
  c.custom_dist = metric
  got = c.predict(x)
  np.testing.assert_array_equal(scb.utils.enforce_ordered_labels(got), orc.ordered(want))
