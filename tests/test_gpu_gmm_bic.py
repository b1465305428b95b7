"""GPU: `sc_gmm_band_pass`, each mode against the NumPy backend on the same fp32 matrix; the
device AffinityGmmBic check against scikit-learn; predict(min_clusters=1) at full size.

The device matrix has NaN everywhere outside the band (below it, in the padding and in extra
columns beyond the padding), so a pass that reads outside the band returns a non-finite sum.

Sums are compared within the fp64 reassociation bound |dev - ref| <= 2 (m + 4) eps sum |t_k|:
both sides add the same m terms t_k (up to one rounding of exp / log1p per term) in different
orders, and any order is within (m - 1) u sum |t_k| of the exact sum.  Counts, minima, maxima,
looked-up indices and values are exact."""

import math
import warnings

import numpy as np
import pytest
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import fallback_clusterer as fc
from spectralcluster_b200 import gmm_bic as gb
from spectralcluster_b200 import synthetic
from spectralcluster_b200.spectral_clusterer import DeviceAffinity

from test_gmm_bic_cpu import assert_states_equal, seeded_affinity, sklearn_fit

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps


def device_band(a, offset):
  """fp32 device copy of `a` with NaN outside the band, ld = padded n + 64 NaN columns."""
  n = a.shape[0]
  eng = dev.Engine.get()
  out = torch.full((n, dev.round_up(n, 64) + 64), float("nan"), dtype=torch.float32,
                   device=eng.device)
  masked = a.astype(np.float32)
  rows, cols = np.tril_indices(n, offset - 1)
  masked[rows, cols] = np.nan
  out[:, :n] = torch.from_numpy(masked).to(eng.device)
  return out


def close(got, want, abs_sum, m):
  assert abs(got - want) <= 2 * (m + 4) * EPS * abs_sum, (got, want, abs_sum)


@pytest.mark.parametrize("n,offset", [(3, 0), (5, -2), (67, 1), (130, 3), (1029, 0), (2051, -2),
                                      (4099, 1)])
def test_band_passes_against_numpy(n, offset):
  a = seeded_affinity(n, 3, seed=n)
  eng = dev.Engine.get()
  ref = gb.NumpyOps(a, offset)
  ops = gb.DeviceOps(eng, device_band(a, offset), n, offset)
  assert ops.m == ref.m
  x, m = ref.x, ref.m
  rng = np.random.default_rng(n)

  def twice(fn, *args):
    first = fn(*args)
    assert fn(*args) == first                   # bitwise repeatable
    return first

  # moments: about 0 and about the mean
  got = twice(ops.moments, 0.0)
  assert got[0] == m and got[3] == x.min() and got[4] == x.max() and got[5] == 0
  close(got[1], x.sum(), np.abs(x).sum(), m)
  close(got[2], (x * x).sum(), (x * x).sum(), m)
  mean = got[1] / m
  got = twice(ops.moments, mean)
  close(got[1], (x - mean).sum(), np.abs(x - mean).sum(), m)
  close(got[2], ((x - mean) ** 2).sum(), ((x - mean) ** 2).sum(), m)

  # flat index -> value, including both ends of the band
  for idx in ([0, m - 1], list(rng.integers(0, m, 2))):
    assert twice(ops.values, idx) == [float(x[i]) for i in idx]

  # KMeans++ potentials, then the cumulative lookup over the row sums they leave behind
  xc = x - mean
  c0, ca, cb = (float(v) - mean for v in x[rng.integers(0, m, 3)])
  d0 = gb._sqdist(xc, c0)
  got = twice(ops.kpp, mean, c0)
  close(got[0], d0.sum(), d0.sum(), m)
  for u in (rng.uniform(size=2), np.array([0.0, 0.999999999])):
    targets = u * got[0]
    vals = twice(ops.kpp_lookup, mean, c0, targets)
    want = np.clip(np.searchsorted(np.cumsum(d0), targets), None, m - 1)
    assert list(ops.last_lookup) == list(want)
    assert vals == [float(x[i]) for i in want]
  got = twice(ops.kpp, mean, c0, ca, cb)
  for g, c in zip(got[1:], (ca, cb)):
    t = np.minimum(d0, gb._sqdist(xc, c))
    close(g, t.sum(), t.sum(), m)

  # Lloyd: counts and changed labels exact, sums per side
  new = (min(ca, cb), max(ca, cb))
  old = (new[0] + 0.01, new[1] - 0.02)
  for prev in (None, old, new):
    got = twice(ops.lloyd, mean, new, prev)
    lab = gb._assign(xc, new)
    assert got[0] == lab.sum()
    assert got[3] == (m if prev is None else np.count_nonzero(lab != gb._assign(xc, prev)))
    close(got[1], xc[lab == 0].sum(), np.abs(xc[lab == 0]).sum(), m)
    close(got[2], xc[lab == 1].sum(), np.abs(xc[lab == 1]).sum(), m)

  # labels -> moments per side
  shifts = (new[0] + mean, new[1] + mean)
  got = twice(ops.label_moments, mean, new, shifts)
  want = ref.label_moments(mean, new, shifts)
  assert got[0] == want[0]
  lab = gb._assign(xc, new)
  for k in (0, 1):
    side = x[lab == k]
    close(got[1 + k], want[1 + k], np.abs(side).sum(), m)
    close(got[3 + k], want[3 + k], ((side - shifts[k]) ** 2).sum(), m)

  # EM and score, one and two components
  var = float(((x - mean) ** 2).mean()) + gb.REG_COVAR
  for weights, means, cov in (([1.0], [mean], [var]),
                              ([0.3, 0.7], [new[0] + mean, new[1] + mean], [var / 3, var / 2])):
    comps = gb._em_args(weights, means, cov)
    wlp, lse = ref._weighted(comps)
    r = np.exp(wlp - lse[:, None])
    got = twice(ops.em, comps)
    close(got[0], lse.sum(), np.abs(lse).sum(), m)
    for k, (mom, comp) in enumerate(zip(got[1], comps)):
      close(mom[0], r[:, k].sum(), r[:, k].sum(), m)
      close(mom[1], r[:, k] @ x, r[:, k] @ np.abs(x), m)
      close(mom[2], r[:, k] @ (x - comp[4]) ** 2, r[:, k] @ (x - comp[4]) ** 2, m)
    close(twice(ops.score, comps), lse.sum(), np.abs(lse).sum(), m)


def test_nonfinite_band_sample_raises():
  a = seeded_affinity(100, 2, seed=1)
  a[10, 50] = np.inf
  ops = gb.DeviceOps(dev.Engine.get(), device_band(a, 1), 100, 1)
  with pytest.raises(ValueError):
    gb.gmm_bic(ops)


@pytest.mark.parametrize("n,speakers,offset", [(5, 1, 0), (64, 2, -2), (300, 1, 3), (600, 4, 1),
                                               (1031, 3, 0), (2048, 2, 1), (2048, 4, -2)])
def test_device_check_matches_sklearn(n, speakers, offset, monkeypatch):
  a = seeded_affinity(n, speakers, seed=7 * n + speakers)
  eng = dev.Engine.get()
  mat = eng.upload_matrix(a)
  values = eng.download_matrix(mat, n)[np.triu_indices(n, offset)][:, None]
  seed = n + offset
  gms, bics, labels, state, warned = sklearn_fit(values, seed)

  np.random.seed(seed)
  with warnings.catch_warnings(record=True) as caught:
    warnings.simplefilter("always")
    res = gb.gmm_bic(gb.DeviceOps(eng, mat, n, offset))
  assert_states_equal(np.random.get_state(), state)
  assert [w.category for w in caught] == warned
  assert res.single == bool(bics[0] < bics[1])
  assert res.n_iter == [g.n_iter_ for g in gms]
  np.testing.assert_allclose(res.bic, bics, rtol=1e-9)
  for fit, g in zip(res.fits, gms):
    np.testing.assert_allclose(fit.weights, g.weights_, rtol=1e-9)
    np.testing.assert_allclose(fit.means, g.means_.ravel(), rtol=1e-9)
    np.testing.assert_allclose(fit.covariances, g.covariances_.ravel(), rtol=1e-9)
  np.testing.assert_array_equal(
      gb._assign(values[:, 0] - res.kmeans_mean, res.fits[1].kmeans_centres), labels)

  def no_download(*_args, **_kw):
    raise AssertionError("the device check must not download the affinity")

  monkeypatch.setattr(dev.Engine, "download_matrix", no_download)
  opts = fc.FallbackOptions(single_cluster_affinity_diagonal_offset=offset)
  details = {}
  np.random.seed(seed)
  with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    got = fc.check_single_cluster(opts, None, DeviceAffinity(mat, n), details)
  assert got == res.single
  assert details["bic"] == res.bic and details["n_iter"] == res.n_iter
  assert details["passes"] == res.passes
  with pytest.raises(ValueError, match="significantly"):
    fc.check_single_cluster(fc.FallbackOptions(single_cluster_affinity_diagonal_offset=n - 1),
                            None, DeviceAffinity(mat, n))


def test_constant_device_affinity_is_one_cluster():
  eng = dev.Engine.get()
  mat = eng.upload_matrix(np.full((50, 50), 0.8125))
  np.random.seed(0)
  with pytest.warns(Warning, match="distinct clusters"):
    assert fc.check_single_cluster(fc.FallbackOptions(), None, DeviceAffinity(mat, 50)) is True


@pytest.mark.parametrize("n", [16384, 65536])
def test_predict_min_clusters_one(n):
  """Identical embeddings give a constant affinity: one cluster.  (The synthetic generator's one
  speaker is not: its affinities are not one Gaussian, and scikit-learn's BIC prefers two
  components on them too.)  Four speakers: the labels of min_clusters=2."""
  opts = scb.configs.icassp2018_refinement_options
  one = np.tile(synthetic.speaker_turn_dvectors(1, 256, 1, seed=3), (n, 1))
  c1 = scb.SpectralClusterer(min_clusters=1, max_clusters=7, refinement_options=opts)
  np.random.seed(0)
  with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    labels = c1.predict(one)
  assert np.array_equal(labels, np.zeros(n, dtype=labels.dtype))
  assert c1.last_details["single_cluster"]["passes"] > 0

  four = synthetic.speaker_turn_dvectors(n, 256, 4, seed=n)
  np.random.seed(0)
  got = c1.predict(four)
  details = c1.last_details["single_cluster"]
  assert details["bic"][0] > details["bic"][1] and min(details["n_iter"]) >= 1
  want = scb.SpectralClusterer(min_clusters=2, max_clusters=7, refinement_options=opts).predict(four)
  assert np.array_equal(got, want)
  assert len(np.unique(got)) == 4
  assert math.isfinite(details["bic"][0])
