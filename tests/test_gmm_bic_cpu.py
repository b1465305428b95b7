"""CPU: the AffinityGmmBic recurrence (spectralcluster_b200/gmm_bic.py) with the NumPy backend
against scikit-learn's GaussianMixture(1) / (2) on the same band, under the same global seed; the
band indexing and the uniform-choice draw mapping against NumPy."""

import warnings

import numpy as np
import pytest
from sklearn.cluster import KMeans
from sklearn.exceptions import ConvergenceWarning
from sklearn.mixture import GaussianMixture

from spectralcluster_b200 import fallback_clusterer as fc
from spectralcluster_b200 import gmm_bic as gb


def seeded_affinity(n, speakers, seed):
  """Cosine affinity (x.y + 1) / 2 of noisy speaker embeddings, rounded through fp32 as the
  device holds it."""
  rng = np.random.default_rng(seed)
  centres = rng.normal(size=(speakers, 32))
  x = centres[rng.integers(0, speakers, n)] + 0.7 * rng.normal(size=(n, 32))
  x /= np.linalg.norm(x, axis=1, keepdims=True)
  return ((x @ x.T + 1.0) / 2.0).astype(np.float32).astype(np.float64)


def sklearn_fit(values, seed):
  """(GMM-1, GMM-2, bics, KMeans(2) init labels, RNG state after both fits, warnings)."""
  np.random.seed(seed)
  with warnings.catch_warnings(record=True) as caught:
    warnings.simplefilter("always")
    gms = [GaussianMixture(n_components=c).fit(values) for c in (1, 2)]
  state = np.random.get_state()
  bics = [g.bic(values) for g in gms]
  np.random.seed(seed)
  np.random.random_sample()                    # GMM-1's KMeans(1) draws its first centre
  labels = KMeans(n_clusters=2, n_init=1, random_state=np.random.mtrand._rand).fit(values).labels_
  return gms, bics, labels, state, [w.category for w in caught]


def ours(affinity, offset, seed):
  np.random.seed(seed)
  with warnings.catch_warnings(record=True) as caught:
    warnings.simplefilter("always")
    res = gb.gmm_bic(gb.NumpyOps(affinity, offset))
  return res, np.random.get_state(), [w.category for w in caught]


def assert_states_equal(a, b):
  assert a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def assert_matches_sklearn(affinity, offset, seed):
  n = affinity.shape[0]
  values = affinity[np.triu_indices(n, offset)][:, None]
  gms, bics, labels, state, warned = sklearn_fit(values, seed)
  res, state2, warned2 = ours(affinity, offset, seed)
  assert res.single == bool(bics[0] < bics[1])
  assert res.n_iter == [g.n_iter_ for g in gms]
  np.testing.assert_allclose(res.bic, bics, rtol=1e-9)
  for fit, g in zip(res.fits, gms):
    np.testing.assert_allclose(fit.weights, g.weights_, rtol=1e-9)
    np.testing.assert_allclose(fit.means, g.means_.ravel(), rtol=1e-9)
    np.testing.assert_allclose(fit.covariances, g.covariances_.ravel(), rtol=1e-9)
    assert fit.converged == g.converged_
  x = values[:, 0] - res.kmeans_mean
  np.testing.assert_array_equal(gb._assign(x, res.fits[1].kmeans_centres), labels)
  assert_states_equal(state, state2)
  assert warned2 == warned
  return res


@pytest.mark.parametrize("n,speakers,offset", [
    (5, 1, 0), (9, 2, 3), (40, 1, 1), (64, 2, -2), (150, 3, 0), (257, 4, 1), (300, 1, 3),
    (411, 2, -2), (600, 4, 0), (600, 3, 1)])
def test_gmm_bic_matches_sklearn(n, speakers, offset):
  a = seeded_affinity(n, speakers, seed=n + speakers)
  for seed in (0, 11):
    res = assert_matches_sklearn(a, offset, seed)
    assert res.passes < 100


def test_constant_samples_are_one_cluster():
  a = np.full((20, 20), 0.625)
  res = None
  with pytest.warns(ConvergenceWarning, match="distinct clusters"):
    np.random.seed(3)
    res = gb.gmm_bic(gb.NumpyOps(a, 1))
  assert res.single is True
  assert fc.check_single_cluster(fc.FallbackOptions(), None, a)      # scikit-learn agrees


def test_small_known_answer():
  a = np.array([[1, 2, 2], [2, 1, 1], [2, 1, 1]], dtype=np.float64)
  np.random.seed(0)
  assert gb.gmm_bic(gb.NumpyOps(a, 0)).single is False
  np.random.seed(0)
  assert fc.check_single_cluster(fc.FallbackOptions(single_cluster_affinity_diagonal_offset=0),
                                 None, a) is False


def test_nonfinite_sample_and_offset_raise():
  a = seeded_affinity(30, 2, 0)
  a[3, 10] = np.nan
  with pytest.raises(ValueError):
    gb.gmm_bic(gb.NumpyOps(a, 1))
  a[3, 10] = np.inf
  with pytest.raises(ValueError):
    gb.gmm_bic(gb.NumpyOps(a, 1))
  for offset in (29, 30, 45):
    with pytest.raises(ValueError, match="significantly"):
      fc.check_single_cluster(fc.FallbackOptions(single_cluster_affinity_diagonal_offset=offset),
                              None, seeded_affinity(30, 2, 0))


def test_band_indexing_matches_triu_indices():
  for n in (1, 2, 3, 4, 7, 10, 33):
    for offset in (-40, -3, -1, 0, 1, 2, n - 2):
      rows, cols = np.triu_indices(n, offset)
      assert gb.band_size(n, offset) == rows.size
      for k in range(rows.size):
        assert gb.band_position(n, offset, k) == (rows[k], cols[k])


@pytest.mark.parametrize("m", [3, 4, 5, 7, 100, 999, 12_345, 65_537, 1_048_583, 8_388_617,
                               33_554_467])
def test_uniform_choice_equals_numpy(m):
  """choice(m, p=uniform) from the closed-form running sum, at sizes up to the 33.6 M-sample band
  of N = 8,192 (a larger cumsum does not fit a test's memory budget)."""
  uc = gb.UniformChoice(m)
  cdf = np.cumsum(np.full(m, 1.0 / m))
  probe = np.unique(np.concatenate([np.arange(min(m, 64)), np.arange(max(0, m - 64), m),
                                    np.random.default_rng(m).integers(0, m, 4000)]))
  assert np.array_equal(np.array([uc.cum(int(i)) for i in probe]), cdf[probe])
  seeds = 400 if m < 10**6 else 60
  for seed in range(seeds):
    u = np.random.RandomState(seed).random_sample()
    assert uc.index(u) == np.random.RandomState(seed).choice(m, p=np.full(m, 1.0 / m))
