"""CPU: the margin-checked float64 k-means restatement (kmeans_restatement.py) against the oracle
(scikit-learn KMeans seeding + scipy cdist loop): same labels and the same number of assignment
passes on every certified case, and near ties reported as not certified."""

from unittest import mock

import numpy as np
import pytest

from oracle import spectral_oracle as orc

import kmeans_restatement as kr


def oracle(e, k, metric, max_iter):
  """orc.run_kmeans labels, and its pass count (one scipy cdist call per assignment pass)."""
  from scipy.spatial import distance
  calls = [0]
  cdist = distance.cdist

  def counted(*a, **kw):
    calls[0] += 1
    return cdist(*a, **kw)

  with mock.patch.object(distance, "cdist", counted):
    labels = orc.run_kmeans(e, k, metric, max_iter)
  return labels, calls[0]


def zero_row_case():
  rng = np.random.default_rng(7)
  e = kr.unit_rows(1000, 4, 4, 0.6, seed=7) * rng.uniform(0.5, 2.0, (1000, 1))
  e[417] = 0.0
  return e


CASES = {
    "unit_255_k8": lambda: (kr.unit_rows(255, 8, 8, 0.6, seed=255), 8, 300),
    "unit_1025_k8": lambda: (kr.unit_rows(1025, 8, 8, 1.0, seed=1025), 8, 300),
    "unit_2049_k8": lambda: (kr.unit_rows(2049, 8, 8, 0.6, seed=2049), 8, 300),
    "unit_4096_k21": lambda: (kr.unit_rows(4096, 21, 21, 0.3, seed=21), 21, 300),
    "unit_4096_k55": lambda: (kr.unit_rows(4096, 55, 55, 0.3, seed=55), 55, 300),
    "kd_below_k": lambda: (kr.unit_rows(3000, 12, 3, 0.4, seed=36), 12, 300),
    "kd_above_k": lambda: (kr.unit_rows(3000, 5, 40, 0.4, seed=200), 5, 300),
    "max_iter_3": lambda: (kr.unit_rows(2049, 20, 20, 1.0, seed=7), 20, 3),
    "max_iter_8": lambda: (kr.unit_rows(2049, 20, 20, 1.0, seed=7), 20, 8),
    "integer_256": lambda: (kr.integer_rows(256, 6, seed=262), 6, 300),
    "integer_2049": lambda: (kr.integer_rows(2049, 4, seed=2053), 4, 300),
    "n_equals_k_3": lambda: (kr.pythagorean_rows(3), 3, 300),
    "n_equals_k_256": lambda: (kr.pythagorean_rows(256), 256, 300),
    "k1_integer": lambda: (kr.integer_rows(1025, 5, seed=1), 1, 12),
    "zero_row": lambda: (zero_row_case(), 4, 20),
    "lonely_148": lambda: kr.lonely_first_sample_rows(148) + (300,),
    "lonely_657": lambda: kr.lonely_first_sample_rows(657) + (300,),
}


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_oracle(name, metric):
  e, k, max_iter = CASES[name]()
  got = kr.restate(e, k, metric, max_iter)
  if name.startswith("lonely") and metric == "euclidean":
    pass                              # these cases are built for cosine; certified or not
  else:
    assert got.certified, "; ".join(got.failures[:4])
  labels, passes = oracle(e, k, metric, max_iter)
  if got.certified:
    np.testing.assert_array_equal(got.labels, labels)
    assert got.iters == passes
  np.testing.assert_allclose(got.centers, orc.seed_centroids(e, k), rtol=0,
                             atol=1e-12 * max(1.0, np.abs(e).max()))


def test_integer_rows_decide_exact_ties():
  """The small-integer cases really exercise the first-minimum rule."""
  for name in ("integer_256", "integer_2049"):
    e, k, _ = CASES[name]()
    assert kr.restate(e, k, "euclidean").exact_ties > 0


@pytest.mark.parametrize("seed", [148, 657])
def test_lonely_first_sample_case_depends_on_the_quirk(seed):
  e, k = kr.lonely_first_sample_rows(seed)
  with_quirk = kr.restate(e, k, "cosine")
  without = kr.restate(e, k, "cosine", quirk=False)
  assert with_quirk.certified
  assert with_quirk.iters != without.iters or not np.array_equal(with_quirk.labels, without.labels)


def test_zero_row_among_unit_rows_is_a_near_tie():
  """Centred, a zero row is -mean and every unit seed c gives |c|^2 - 2 x.c = 1 - |mean|^2: an
  exact tie in the Lloyd E-step that rounding decides.  Not certified, and the E-step says so."""
  e = kr.unit_rows(1000, 4, 4, 0.3, seed=5)
  e[417] = 0.0
  got = kr.restate(e, 4, "cosine", 20)
  assert not got.certified
  assert got.failures[0].startswith("lloyd_estep") and "row[417]" in got.failures[0]


def test_k1_unit_rows_stop_rule_is_a_near_tie():
  """k = 1: the second pass's centroid (mean of all rows) equals the Lloyd centre in exact
  arithmetic, so the stop rule compares two equal means up to rounding.  Not certified."""
  got = kr.restate(kr.unit_rows(1025, 3, 5, 0.5, seed=1), 1, "euclidean")
  assert not got.certified
  assert any(f.startswith("stop_rule_prev") for f in got.failures)


@pytest.mark.parametrize("bad,message", [(np.nan, "contains NaN"), (np.inf, "contains infinity")])
def test_nonfinite_rows_raise_like_sklearn(bad, message):
  e = kr.unit_rows(100, 3, 3, 0.5, seed=1)
  e[50, 1] = bad
  with pytest.raises(ValueError, match=message):
    kr.restate(e, 3, "cosine")
  with pytest.raises(ValueError, match=message):
    orc.run_kmeans(e, 3, "cosine", 300)


def test_duplicate_rows_n_equal_k_flag_an_empty_cluster():
  e = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 0.0], [0.5, 0.5]])
  assert kr.restate(e, 4, "cosine").empty_cluster


def test_draws_match_engine_kmeans_order():
  """The draws are scikit-learn's: its k-means++ picks the restatement's seeds."""
  from sklearn.cluster import kmeans_plusplus
  e = kr.unit_rows(500, 7, 7, 0.5, seed=3)
  x = e - e.mean(axis=0)
  _, idx = kmeans_plusplus(x, 7, random_state=np.random.RandomState(0))
  np.testing.assert_array_equal(kr.restate(e, 7, "cosine").seeds, idx)
