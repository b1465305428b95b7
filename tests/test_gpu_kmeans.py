"""GPU: sc_kmeans and sc_row_renorm at their launch edges against the margin-checked float64
restatement in kmeans_restatement.py.

Every k-means case is first certified on the host (every decision beats its rounding bound), then
the device must return the restatement's labels bit for bit and the same number of assignment
passes.  The sizes sit on the edges of the kernels: 256-thread blocks of k_assign, k_kpp_* and
k_cluster_sums (n = 255 .. 257, 1023 .. 1025, 2047, 2049, 65,536), the 1,024-chunk scan of
k_kpp_candidates, every step of the trial count 2 + int(ln k), the batch of 4 passes between
host reads (max_iter), and degenerate rows."""

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import device as dev

import kmeans_restatement as kr

pytestmark = pytest.mark.gpu

METRICS = {"cosine": 0, "euclidean": 1}


def device_kmeans(engine, e, k, metric, max_iter):
  t = dev.torch()
  x = t.from_numpy(np.ascontiguousarray(e, dtype=np.float64)).to(engine.device)
  return engine.kmeans(x, int(k), METRICS[metric], int(max_iter))


def check(engine, e, k, metric, max_iter=300, **kw):
  """Certify on the host, then compare labels and pass count with the device."""
  want = kr.restate(e, k, metric, max_iter)
  assert want.certified, "not certified: %s" % "; ".join(want.failures[:4])
  labels, iters = device_kmeans(engine, e, k, metric, max_iter)
  assert labels.dtype == np.int64
  bad = np.flatnonzero(labels != want.labels)
  assert bad.size == 0, "%d labels differ, first at row %d" % (bad.size, bad[0])
  assert iters == want.iters, (iters, want.iters)
  return want


# ---------------------------------------------------------------- n at block and grid edges
@pytest.mark.parametrize("metric", sorted(METRICS))
@pytest.mark.parametrize("n", [255, 256, 257, 1023, 1024, 1025, 2047, 2049, 65536])
@pytest.mark.parametrize("spread", [0.6, 1.0])
def test_n_edges_unit_rows(engine, metric, n, spread):
  check(engine, kr.unit_rows(n, 8, 8, spread, seed=n), 8, metric)


@pytest.mark.parametrize("metric", sorted(METRICS))
@pytest.mark.parametrize("n", [1, 2, 3, 256, 257])
def test_n_equals_k(engine, metric, n):
  """Every row is a seed and, after the Lloyd step, its own centroid: distances are exactly 0 and
  the loop stops after one pass.  Integer rows with integer norms keep the cosine exact."""
  e = kr.pythagorean_rows(n)
  w = check(engine, e, n, metric)
  assert w.iters == 1


# ---------------------------------------------------------------- k at every trial-count step
@pytest.mark.parametrize("metric", sorted(METRICS))
@pytest.mark.parametrize("k", [1, 2, 3, 7, 8, 20, 21, 54, 55, 148, 149, 403, 404])
def test_k_trial_steps(engine, metric, k):
  n = 4096
  check(engine, kr.unit_rows(n, k, k, 0.3, seed=k), k, metric)


@pytest.mark.parametrize("metric", sorted(METRICS))
@pytest.mark.parametrize("n,k", [(8192, 512), (65536, 64)])
def test_large_k(engine, metric, n, k):
  check(engine, kr.unit_rows(n, k, k, 0.3, seed=k), k, metric)


def test_k1_has_no_draws(engine):
  """k = 1 passes no uniforms (u_host NULL).  Integer rows with zero column sums put the one
  centroid exactly at the origin: euclidean stops when the second pass repeats the first, cosine
  is NaN against a zero centroid and runs to max_iter, as in the reference."""
  e = kr.integer_rows(1025, 5, seed=1)
  w = check(engine, e, 1, "euclidean", max_iter=12)
  assert not w.labels.any() and w.iters == 2
  w = check(engine, e, 1, "cosine", max_iter=12)
  assert not w.labels.any() and w.iters == 13


# ---------------------------------------------------------------- k_dim != k (public entry)
@pytest.mark.parametrize("metric", sorted(METRICS))
@pytest.mark.parametrize("k,kd", [(12, 3), (5, 40)])
def test_k_dim_differs_from_k(engine, metric, k, kd):
  e = kr.unit_rows(3000, k, kd, 0.4, seed=k * kd)
  w = check(engine, e, k, metric)
  got = scb.custom_distance_kmeans.run_kmeans(e, k, metric, 300)
  np.testing.assert_array_equal(got, w.labels)


# ---------------------------------------------------------------- max_iter around the batch of 4
@pytest.mark.parametrize("metric", sorted(METRICS))
@pytest.mark.parametrize("max_iter", [1, 2, 3, 4, 5, 8, 9, 300])
def test_max_iter(engine, metric, max_iter):
  """Overlapping clusters converge slowly, so every max_iter below the converged pass count stops
  the loop early (max_iter + 1 passes)."""
  e = kr.unit_rows(2049, 20, 20, 1.0, seed=7)
  w = check(engine, e, 20, metric, max_iter)
  full = kr.restate(e, 20, metric, 300)
  assert full.iters > 10                        # so max_iter <= 9 runs out of iterations
  if max_iter < full.iters:
    assert w.iters == max_iter + 1


# ---------------------------------------------------------------- small-integer embeddings
@pytest.mark.parametrize("metric", sorted(METRICS))
@pytest.mark.parametrize("n,kd", [(256, 6), (1024, 6), (2049, 4)])
def test_integer_rows_exact_ties(engine, metric, n, kd):
  """Every seeding product is exact, so squared distances tie exactly; the first minimum must win
  (np.argmin) in the k-means++ potentials and the Lloyd E-step."""
  e = kr.integer_rows(n, kd, seed=n + kd)
  w = check(engine, e, kd, metric)
  assert w.exact_ties > 0


# ---------------------------------------------------------------- the device's own eigenvectors
@pytest.mark.parametrize("renorm", [False, True])
def test_device_eigenvectors_65536(engine, monkeypatch, renorm):
  """The eigenvectors predict() computes at N = 65,536 (6 speakers, ICASSP), as they come off the
  device, with and without row_wise_renorm.

  max_clusters=None (windowed Lanczos) gives k = 6 vectors, max_clusters=10 gives 10.  These
  embeddings are so nearly piecewise constant that the Lloyd step already gives the final labels:
  the second pass's centroids then equal the first's in exact arithmetic, and only rounding
  decides the stop rule there, so the pass count is not certifiable beyond max_iter = 1 (see
  test_kmeans_restatement_cpu.py).  Both run with max_iter = 1, where both passes are decided."""
  from oracle import spectral_oracle as orc
  t = dev.torch()
  x = orc.synthetic_dvectors(65536, 256, 6, seed=0)
  box = []
  orig = scb.SpectralClusterer._compute_eigenvectors_ncluster

  def spy(self, *a, **kw):
    out = orig(self, *a, **kw)
    box.append((out[0].clone(), out[1]))
    return out

  monkeypatch.setattr(scb.SpectralClusterer, "_compute_eigenvectors_ncluster", spy)
  opts = scb.RefinementOptions(gaussian_blur_sigma=1, p_percentile=0.95,
                               thresholding_soft_multiplier=0.01,
                               refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))
  cases = []
  for max_clusters in (None, 10):
    c = scb.SpectralClusterer(max_clusters=max_clusters, refinement_options=opts,
                              row_wise_renorm=renorm)
    c.predict(x)
    vectors, k = box.pop()
    kk = k if max_clusters is None else max_clusters
    assert k == 6 and vectors.shape[1] >= kk
    cases.append((vectors[:, :kk].contiguous(), kk))
    del vectors
    t.cuda.empty_cache()
  for v, kk in cases:
    if renorm:
      engine.row_renorm(v)
    e = v.cpu().numpy()
    for metric in METRICS:
      check(engine, e, kk, metric, max_iter=1)


# ---------------------------------------------------------------- degenerate rows
def test_zero_row_cosine_runs_to_max_iter(engine):
  """An all-zero row is NaN against every centroid under cosine: label 0, the mean distance is
  NaN, so the stop rule never fires and the loop runs max_iter + 1 passes, as in the reference."""
  rng = np.random.default_rng(7)
  e = kr.unit_rows(1000, 4, 4, 0.6, seed=7) * rng.uniform(0.5, 2.0, (1000, 1))
  e[417] = 0.0              # (among unit rows it would tie exactly with every seed in the seeding)
  w = check(engine, e, 4, "cosine", max_iter=20)
  assert w.labels[417] == 0 and w.iters == 21
  w = check(engine, e, 4, "euclidean", max_iter=20)
  assert w.iters < 21


@pytest.mark.parametrize("bad,message", [(np.nan, "contains NaN"), (np.inf, "contains infinity"),
                                         (-np.inf, "contains infinity")])
def test_nonfinite_rows_raise_like_sklearn(engine, bad, message):
  """scikit-learn's fit refuses non-finite input (ValueError); so does sc_kmeans."""
  e = kr.unit_rows(1000, 4, 4, 0.3, seed=5)
  e[999, 2] = bad
  for metric in METRICS:
    with pytest.raises(ValueError, match=message):
      device_kmeans(engine, e, 4, metric, 300)
    with pytest.raises(ValueError, match=message):
      kr.restate(e, 4, metric)
  e[3, 0] = np.nan          # NaN anywhere takes precedence, as in scikit-learn
  with pytest.raises(ValueError, match="contains NaN"):
    device_kmeans(engine, e, 4, "cosine", 300)


def test_duplicate_rows_with_n_equal_k_raise(engine):
  """Known difference: with duplicate rows and n == k, k-means++ seeds the same point twice, a
  cluster is empty after the Lloyd step, and scikit-learn relocates it.  sc_kmeans does not
  restate the relocation and says so."""
  e = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 0.0], [0.5, 0.5]])
  assert kr.restate(e, 4, "cosine").empty_cluster
  with pytest.raises(ValueError, match="lost all members"):
    device_kmeans(engine, e, 4, "cosine", 300)


@pytest.mark.parametrize("seed", [148, 657])
def test_lonely_first_sample_quirk(engine, seed):
  """A cluster whose only member is sample 0 keeps its centroid (custom_distance_kmeans.py:137);
  the cases are chosen so that updating it would change the result."""
  e, k = kr.lonely_first_sample_rows(seed)
  w = check(engine, e, k, "cosine")
  other = kr.restate(e, k, "cosine", quirk=False)
  assert other.iters != w.iters or not np.array_equal(other.labels, w.labels)


# ---------------------------------------------------------------- sc_row_renorm
@pytest.mark.parametrize("n", [1, 255, 256, 257, 1023, 1025, 2049, 65536])
@pytest.mark.parametrize("k", [1, 6, 64])
def test_row_renorm(engine, n, k):
  """Against e / ||e||_2 in float64: within 2 ulps of 1 in norm (one kd-term sum, a sqrt and a
  division); k = 1 gives exactly +-1; zero rows give NaN and tiny rows stay finite, as numpy."""
  t = dev.torch()
  rng = np.random.default_rng(n * 7 + k)
  e = rng.standard_normal((n, k))
  if n > 3:
    e[1] = 0.0
    e[2] = 1e-300 * rng.standard_normal(k)
  x = t.from_numpy(e.copy()).to(engine.device)
  engine.row_renorm(x)
  got = x.cpu().numpy()
  with np.errstate(invalid="ignore", divide="ignore"):
    want = e / np.linalg.norm(e, axis=1, ord=2, keepdims=True)
  np.testing.assert_array_equal(np.isfinite(got), np.isfinite(want))
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
  fin = np.isfinite(want)
  err = np.abs(got - want)[fin]
  assert err.max(initial=0.0) <= kr.gamma(k + 4) * 1.0, err.max()
  if k == 1:
    np.testing.assert_array_equal(np.abs(got[fin]), 1.0)
