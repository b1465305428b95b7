"""GPU: the windowed solve on the factored operator (sc_eigh_extremal_locked_factored and
predict()'s windowed factored route) against the stored windows.

The route is forced at small N by setting Engine.factored_above_bytes = 0; at N = 131,072 it is
taken unforced.  "Routes agree" means within twice the float64 contract
|dw| <= 1e-5 |w| + 1e-6 lambda_max: the stored S is the fp32 tensor-core accumulation of the
product the factored operator applies exactly."""

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import eigen_windows as ew
from spectralcluster_b200 import laplacian as lap_lib
from oracle import spectral_oracle as orc

pytestmark = pytest.mark.gpu
GRAPHCUT = scb.LaplacianType.GraphCut


def icassp():
  return scb.RefinementOptions(gaussian_blur_sigma=1, p_percentile=0.95,
                               thresholding_soft_multiplier=0.01,
                               thresholding_type=scb.ThresholdType.RowMax,
                               refinement_sequence=list(scb.configs.ICASSP2018_REFINEMENT_SEQUENCE))


def assert_routes_agree(w, w_ref, lambda_max):
  w, w_ref = np.asarray(w), np.asarray(w_ref)
  assert w.shape == w_ref.shape
  np.testing.assert_allclose(w, w_ref, rtol=2e-5, atol=2e-6 * abs(lambda_max))


def factored_residuals(y_hi, n, terms, w, v, chunk=8192):
  """|M v_j - w_j v_j|max for M = diag(delta) + sign diag(left) Y Y^T diag(right), Y = Y_hi in
  float64, applied in row chunks."""
  t = dev.torch()
  delta, left, right, sign, _ = terms
  out = []
  for j in range(v.shape[1]):
    u = v[:, j] if right is None else right * v[:, j]
    z = t.empty(n, dtype=t.float64, device=v.device)
    for c0 in range(0, n, chunk):
      z[c0:c0 + chunk] = y_hi[c0:c0 + chunk, :n].double() @ u
    s = t.empty_like(z)
    for c0 in range(0, n, chunk):
      s[c0:c0 + chunk] = y_hi[c0:c0 + chunk, :n].double() @ z
    mv = sign * (s if left is None else left * s)
    if delta is not None:
      mv = mv + delta * v[:, j]
    out.append((mv - w[j] * v[:, j]).abs().max().item())
  return out


def test_locked_factored_entry_against_stored_windows(engine):
  t = dev.torch()
  n = 40000
  x = t.from_numpy(orc.synthetic_dvectors(n, 256, 6, seed=7).astype(np.float32)).to(engine.device)
  refined = dev.FactoredAffinity(engine, x).refine(engine, icassp())
  terms = lap_lib.operator_terms(engine, refined, GRAPHCUT)
  delta, left, right, sign, which = terms
  s, _, _ = engine.diffuse(n, hi=refined.y_hi, lo=None, precision=nat.GEMM_SINGLE)
  stored = ew.DeviceOps(engine, s, n, delta, left, right, sign, which, capacity=64)
  factored = ew.DeviceOps(engine, refined.y_hi, n, delta, left, right, sign, which, capacity=64,
                          factored=True)
  w_s = np.concatenate([stored.window(16) for _ in range(4)])
  w_f = np.concatenate([factored.window(16) for _ in range(4)])
  top = factored.lambda_max()
  assert_routes_agree(top, stored.lambda_max(), top)
  del stored, s
  assert_routes_agree(np.sort(w_f), np.sort(w_s), top)
  u = factored.locked[:64]
  gram = u @ u.T
  assert (gram - t.eye(64, dtype=t.float64, device=engine.device)).abs().max().item() <= 1e-10
  v = factored.vectors(list(range(64)))
  res = factored_residuals(refined.y_hi, n, terms, w_f, v)
  assert max(res) <= 1e-7 * max(1.0, float(np.abs(w_f).max())), max(res)
  assert factored.stats["windows"] == 4


@pytest.fixture
def lambda_maxes(monkeypatch):
  """The values of every DeviceOps.lambda_max() solve the test runs, in order."""
  tops = []
  inner = ew.DeviceOps.lambda_max

  def lambda_max(self):
    tops.append(inner(self))
    return tops[-1]

  monkeypatch.setattr(ew.DeviceOps, "lambda_max", lambda_max)
  return tops


CASES = {
    "graphcut-none": dict(laplacian_type=GRAPHCUT),
    "nolaplacian-none": dict(),
    "graphcut-normalizeddiff-none": dict(laplacian_type=GRAPHCUT,
                                         eigengap_type=scb.EigenGapType.NormalizedDiff),
    "graphcut-40": dict(laplacian_type=GRAPHCUT, max_clusters=40),
}


def clusterer(case):
  kw = dict(max_clusters=None)
  kw.update(CASES[case])
  return scb.SpectralClusterer(min_clusters=2, refinement_options=icassp(), custom_dist="cosine",
                               **kw)


def forced(engine, fn):
  saved = engine.factored_above_bytes
  engine.factored_above_bytes = 0
  try:
    return fn()
  finally:
    engine.factored_above_bytes = saved


@pytest.mark.parametrize("n,case", [(40000, c) for c in CASES] +
                         [(65536, "graphcut-none"), (65536, "nolaplacian-none")])
def test_predict_forced_factored_windows_equals_stored_windows(engine, lambda_maxes, n, case):
  tops = lambda_maxes
  x = orc.synthetic_dvectors(n, 256, 6, seed=11).astype(np.float32)
  c = clusterer(case)
  want = c.predict(x)
  ref = dict(c.last_details)
  assert not c._factored_windows_route(engine, n)
  got = forced(engine, lambda: c.predict(x))
  assert forced(engine, lambda: c._factored_windows_route(engine, n))
  assert ref["solver"] == "lanczos-windows"
  assert c.last_details["solver"] == "lanczos-factored-windows"
  assert c.last_details["n_clusters"] == ref["n_clusters"]
  assert np.array_equal(got, want)
  w, w_ref = c.last_details["eigenvalues"], ref["eigenvalues"]
  # lambda_max: the solve of each ascending route (its first value on a descending spectrum)
  top = max([abs(v) for v in tops] + [float(np.abs(w_ref).max())])
  n_common = min(len(w), len(w_ref))
  assert_routes_agree(w[:n_common], w_ref[:n_common], top)
  if len(tops) == 2:
    assert_routes_agree(tops[1], tops[0], top)


def test_window_cap_on_the_factored_route(engine, monkeypatch):
  monkeypatch.setattr(ew, "MAX_WINDOW_PAIRS", 4)
  x = orc.synthetic_dvectors(40000, 256, 6, seed=11).astype(np.float32)
  c = clusterer("graphcut-none")
  with pytest.raises(NotImplementedError, match="first 4 eigenvalues"):
    forced(engine, lambda: c.predict(x))


def test_device_input_equals_its_host_twin(engine):
  t = dev.torch()
  x = orc.synthetic_dvectors(40000, 256, 6, seed=3).astype(np.float32)
  c = clusterer("graphcut-none")
  want = forced(engine, lambda: c.predict(x))
  ref = dict(c.last_details)
  got = forced(engine, lambda: c.predict(t.from_numpy(x).to(engine.device)))
  assert ref["solver"] == c.last_details["solver"] == "lanczos-factored-windows"
  assert np.array_equal(got, want)
  assert np.array_equal(c.last_details["eigenvalues"], ref["eigenvalues"])


@pytest.mark.parametrize("laplacian", [GRAPHCUT, None])
def test_n131072_max_clusters_none_on_one_gpu(engine, lambda_maxes, laplacian):
  """max_clusters=None at BASELINE configs[3]'s size on one H100, route not forced.  Needs about
  40 GB of free device memory: Y_hi (34.4 GB), the locked set and the Lanczos scratch."""
  t = dev.torch()
  n = 131072
  x, truth = orc.synthetic_dvectors(n, 256, 6, seed=0, return_labels=True)
  c = scb.SpectralClusterer(min_clusters=2, max_clusters=None,
                            refinement_options=scb.configs.icassp2018_refinement_options,
                            laplacian_type=laplacian, custom_dist="cosine")
  assert c._factored_windows_route(engine, n)
  t.cuda.synchronize()
  t.cuda.reset_peak_memory_stats(engine.device)
  labels = c.predict(x.astype(np.float32))
  peak = t.cuda.max_memory_allocated(engine.device)
  ld = dev.round_up(n, 64)
  assert c.last_details["solver"] == "lanczos-factored-windows"
  assert c.last_details["n_clusters"] == 6
  assert np.array_equal(scb.utils.enforce_ordered_labels(labels), orc.ordered(truth))
  assert peak < 4 * n * ld, peak
  # the prefix against one factored Lanczos solve on the same Y_hi
  prefix = np.asarray(c.last_details["eigenvalues"])
  count = min(len(prefix), 32)
  fa = dev.FactoredAffinity(engine, t.from_numpy(x.astype(np.float32)).to(engine.device))
  refined = fa.refine(engine, c.refinement_options)
  del fa
  terms = lap_lib.operator_terms(engine, refined, laplacian)
  w, _, _ = engine.eigh_factored(refined.y_hi, n, *terms, count, 0)
  top = max([abs(v) for v in lambda_maxes] + [float(np.abs(prefix).max())])
  np.testing.assert_allclose(prefix[:count], w, rtol=1e-5, atol=1e-6 * top)
  stats = c.last_details["lanczos_stats"]
  print("N=131072 %s: %d values, %d windows, %d passes, peak %.1f GB (4 N ld = %.1f GB)" % (
      laplacian, len(prefix), stats["windows"], stats["passes"], peak / 1e9, 4 * n * ld / 1e9))
