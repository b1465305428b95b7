"""CPU: the margin-checked float64 restatement of the scipy-metric k-means passes
(kmeans_metrics_restatement.py) against the oracle (scikit-learn seeding + scipy cdist loop): the
same labels and pass count on every certified case, for every metric sc_kmeans evaluates beyond
cosine and euclidean; and run_kmeans's alias table against scipy's."""

from unittest import mock

import numpy as np
import pytest

from oracle import spectral_oracle as orc

import kmeans_metrics_restatement as km
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


def case(name):
  if name == "unit_1025_k8":
    return kr.unit_rows(1025, 8, 8, 0.6, seed=1025), 8, 300
  if name == "unit_2049_k6_kd12":
    return kr.unit_rows(2049, 6, 12, 0.5, seed=612), 6, 300
  if name == "unit_3000_k12_kd3":
    return kr.unit_rows(3000, 12, 3, 0.4, seed=36), 12, 300
  if name == "max_iter_2":
    return kr.unit_rows(2049, 20, 20, 1.0, seed=7), 20, 2
  if name == "positive_2049_k5":
    return km.positive_rows(2049, 5, 8, 0.3, seed=5), 5, 300
  raise KeyError(name)


NAMES = ["unit_1025_k8", "unit_2049_k6_kd12", "unit_3000_k12_kd3", "max_iter_2",
         "positive_2049_k5"]


@pytest.mark.parametrize("metric", km.METRICS)
@pytest.mark.parametrize("name", NAMES)
def test_restatement_matches_oracle(name, metric):
  e, k, max_iter = case(name)
  want = km.restate(e, k, metric, max_iter)
  labels, passes = oracle(e, k, metric, max_iter)
  if not want.certified:
    pytest.skip("not certified: %s" % "; ".join(want.failures[:2]))
  np.testing.assert_array_equal(want.labels, labels)
  assert want.iters == passes


def test_most_cases_are_certified():
  """The bounds are not so loose that nothing certifies: every metric certifies most cases."""
  for metric in km.METRICS:
    ok = 0
    for name in NAMES:
      e, k, max_iter = case(name)
      ok += km.restate(e, k, metric, max_iter).certified
    assert ok >= 3, (metric, ok)


def zero_rows_case():
  """Scaled unit rows (no exact ties in the seeding) with two zero rows."""
  rng = np.random.default_rng(11)
  e = kr.unit_rows(1000, 4, 6, 0.5, seed=11) * rng.uniform(0.5, 2.0, (1000, 1))
  e[[417, 700]] = 0.0
  return e


def test_special_values_match_oracle():
  """Zero rows (braycurtis NaN, correlation NaN), a constant column (seuclidean NaN everywhere)
  and negative entries (jensenshannon inf): labels and pass counts as scipy's."""
  e = zero_rows_case()
  for metric in ("braycurtis", "correlation"):
    want = km.restate(e, 4, metric, 20)
    assert want.certified, (metric, want.failures[:2])
    labels, passes = oracle(e, 4, metric, 20)
    np.testing.assert_array_equal(want.labels, labels)
    assert want.iters == passes
  c = kr.unit_rows(1000, 4, 6, 0.5, seed=12)
  c[:, 2] = 0.5
  want = km.restate(c, 4, "seuclidean", 7)
  assert want.certified and want.iters == 8 and not want.labels.any()
  labels, passes = oracle(c, 4, "seuclidean", 7)
  np.testing.assert_array_equal(want.labels, labels)
  assert passes == 8
  want = km.restate(e, 4, "jensenshannon", 20)   # unit rows have negative entries: inf
  assert want.certified and not want.labels.any() and want.iters == 2
  labels, passes = oracle(e, 4, "jensenshannon", 20)
  np.testing.assert_array_equal(want.labels, labels)
  assert passes == 2


def test_mahalanobis_errors_match_scipy():
  rng = np.random.default_rng(3)
  e = rng.standard_normal((200, 5))
  for bad in ("zero", "twin"):
    x = e.copy()
    if bad == "zero":
      x[:, 3] = 0.0
    else:
      x[:, 4] = x[:, 1]
    with pytest.raises(np.linalg.LinAlgError, match="Singular matrix"):
      km.restate(x, 3, "mahalanobis")
    with pytest.raises(np.linalg.LinAlgError, match="Singular matrix"):
      orc.run_kmeans(x, 3, "mahalanobis", 300)
  small = rng.standard_normal((4, 9))
  msg = ("The number of observations \\(6\\) is too small; the covariance matrix is singular. "
         "For observations with 9 dimensions, at least 10 observations are required.")
  with pytest.raises(ValueError, match=msg):
    km.restate(small, 2, "mahalanobis")
  with pytest.raises(ValueError, match=msg):
    orc.run_kmeans(small, 2, "mahalanobis", 300)


def test_alias_table_is_scipys():
  from scipy.spatial import distance
  from spectralcluster_b200 import custom_distance_kmeans as cdk
  for name, akas in cdk._ALIASES.items():
    assert akas == distance._METRICS[name].aka, name
  host = {"hamming", "dice", "jaccard", "rogerstanimoto", "russellrao", "sokalsneath", "yule"}
  assert set(cdk._ALIASES) | host == set(distance._METRICS)
  for name in host:
    assert not distance._METRICS[name].aka & set(cdk._METRICS)
