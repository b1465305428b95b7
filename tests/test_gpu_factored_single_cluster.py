"""GPU: the single-cluster checks of predict(min_clusters=1) on the factored route, which never
stores the affinity, against the stored route.

The packed band's passes must equal the dense passes bit for bit in every mode; the panel sweep's
statistics must equal sc_affinity_stats bit for bit; predict() must return the stored route's
labels and the same `last_details["single_cluster"]` exactly, for every condition.  The route is
forced at small N by setting Engine.factored_above_bytes = 0."""

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

from test_gmm_bic_cpu import seeded_affinity
from test_gpu_factored import assert_routes_agree
from test_gpu_gmm_bic import device_band

pytestmark = pytest.mark.gpu
SCC = scb.SingleClusterCondition


def packed_from_panels(eng, dense, n, offset, rows=128):
  """The packed band of `dense` ([n, ld] fp32), packed in row panels of `rows` rows."""
  off = gb.packed_row_offsets(n, offset)
  band = torch.full((max(int(off[-1]), 4),), 7.0, dtype=torch.float32, device=eng.device)
  row_off = torch.from_numpy(off).to(eng.device)
  for r0 in range(0, gb.band_rows(n, offset), rows):
    r1 = min(n, r0 + rows)
    panel = dense[r0:r1]
    eng.call("sc_gmm_band_pack", dev._ptr(panel), panel.stride(0), r0, r1 - r0, n, offset,
             dev._ptr(row_off), dev._ptr(band), eng.stream)
  return band, row_off


def bits(o):
  return np.asarray(o, dtype=np.float64).copy().view(np.int64)


CASES = [(n, o) for n in (67, 130, 1029, 4099) for o in (-2, 0, 1, 3, n - 2)]


@pytest.mark.parametrize("n,offset", CASES)
def test_packed_passes_equal_dense_passes(n, offset):
  eng = dev.Engine.get()
  a = seeded_affinity(n, 3, seed=n + offset)
  dense = device_band(a, offset)
  band, row_off = packed_from_panels(eng, dense, n, offset)
  m = gb.band_size(n, offset)

  # the band holds the in-band values at their packed slots and NaN in every padding slot
  host = band.cpu().numpy()
  off = gb.packed_row_offsets(n, offset)
  rows, cols = np.triu_indices(n, offset)
  pos = off[rows] + cols - (np.maximum(rows + offset, 0) & ~3)
  assert np.array_equal(host[pos].view(np.int32), a[rows, cols].astype(np.float32).view(np.int32))
  assert int(np.isnan(host[:off[-1]]).sum()) == off[-1] - m

  d_ops = gb.DeviceOps(eng, dense, n, offset)
  p_ops = gb.DeviceOps(eng, band, n, offset, row_off)
  assert d_ops.m == p_ops.m == m

  def both(mode, *params):
    want = d_ops._pass(mode, *params).copy()
    got = p_ops._pass(mode, *params).copy()
    assert np.array_equal(bits(got), bits(want)), (mode, params, got, want)
    return want

  o = both(gb.MOMENTS, 0.0)
  assert o[0] == m and o[5] == 0
  mean = o[1] / m
  both(gb.MOMENTS, mean)
  rng = np.random.default_rng(n)
  x = a[rows, cols]
  c0, ca, cb = (float(v) - mean for v in x[rng.integers(0, m, 3)])
  pot = both(gb.KPP, mean, c0, 0.0, 0.0, 0.0)[0]
  for u in (rng.uniform(size=2), np.array([0.0, 0.999999999])):
    both(gb.KPP, mean, c0, 0.0, 0.0, 0.0)          # the row sums the lookup reads
    both(gb.LOOKUP, mean, c0, 1.0, *(u * pot))
  both(gb.KPP, mean, c0, ca, cb, 2.0)
  for idx in ([0, m - 1], list(rng.integers(0, m, 2))):
    both(gb.LOOKUP, 0.0, 0.0, 0.0, float(idx[0]), float(idx[1]))
  new = (min(ca, cb), max(ca, cb))
  both(gb.LLOYD, mean, *new, 0.0, 0.0, 0.0)
  both(gb.LLOYD, mean, *new, new[0] + 0.01, new[1] - 0.02, 1.0)
  both(gb.LABELS, mean, *new, new[0] + mean, new[1] + mean)
  var = float(((x - mean) ** 2).mean()) + gb.REG_COVAR
  for weights, means, cov in (([1.0], [mean], [var]),
                              ([0.3, 0.7], [new[0] + mean, new[1] + mean], [var / 3, var / 2])):
    params = [float(len(weights))] + [v for comp in gb._em_args(weights, means, cov) for v in comp]
    both(gb.EM, *params)
    both(gb.SCORE, *params)

  # the whole check: same draws, same fits, same passes
  results = []
  for ops in (d_ops, p_ops):
    np.random.seed(n)
    with warnings.catch_warnings():
      warnings.simplefilter("ignore")
      res = gb.gmm_bic(ops)
    results.append((res.single, res.bic, res.n_iter, res.passes, np.random.get_state()[1].copy()))
  (s0, b0, i0, p0, st0), (s1, b1, i1, p1, st1) = results
  assert (s0, b0, i0, p0) == (s1, b1, i1, p1) and np.array_equal(st0, st1)


def embeddings(eng, n, speakers=4, seed=7):
  return torch.from_numpy(synthetic.speaker_turn_dvectors(n, 256, speakers, seed=seed)
                          .astype(np.float32)).to(eng.device)


@pytest.mark.parametrize("n", [4099, 16384])
def test_panel_statistics_equal_the_stored_statistics(engine, n):
  x = embeddings(engine, n)
  a, _ = engine.affinity(x, want_crop_vector=False)
  want = fc.affinity_statistics(DeviceAffinity(a, n))
  del a
  for rows in (dev.PANEL_ALIGN, dev.PANEL_ALIGN * 3, None):
    got = fc.affinity_statistics(dev.FactoredAffinity(engine, x, panel_rows=rows))
    assert got == want, (rows, got, want)


def factored_and_stored(engine, make, x):
  """(labels, last_details) of the stored route, then of the forced factored route, with
  np.random.seed(0) before each call."""
  out = []
  for limit in (engine.factored_above_bytes, 0):
    saved = engine.factored_above_bytes
    engine.factored_above_bytes = limit
    try:
      c = make()
      n = x.shape[0]
      assert c._factored_single_cluster_route(engine, n) == (limit == 0)
      np.random.seed(0)
      with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        labels = c.predict(x)
    finally:
      engine.factored_above_bytes = saved
    out.append((labels, dict(c.last_details)))
  return out


CONDITIONS = {
    "gmm-bic": dict(single_cluster_condition=SCC.AffinityGmmBic),
    "all": dict(single_cluster_condition=SCC.AllAffinity),
    "neighbor": dict(single_cluster_condition=SCC.NeighborAffinity),
    "std": dict(single_cluster_condition=SCC.AffinityStd),
    "naive": dict(single_cluster_condition=SCC.FallbackClusterer,
                  fallback_clusterer_type=scb.FallbackClustererType.Naive),
    "agglomerative": dict(single_cluster_condition=SCC.FallbackClusterer,
                          fallback_clusterer_type=scb.FallbackClustererType.Agglomerative),
}


def clusterer(condition, max_clusters=10):
  return lambda: scb.SpectralClusterer(
      min_clusters=1, max_clusters=max_clusters,
      refinement_options=scb.configs.icassp2018_refinement_options,
      fallback_options=scb.FallbackOptions(**CONDITIONS[condition]), custom_dist="cosine")


def assert_same(stored, factored, windows=False):
  (want, ref), (got, det) = stored, factored
  assert np.array_equal(got, want)
  assert det.get("single_cluster") == ref.get("single_cluster")
  if "eigenvalues" in ref or "eigenvalues" in det:        # a multi verdict ran the eigen stage
    assert ref["solver"] == ("lanczos-windows" if windows else "lanczos")
    assert det["solver"] == ("lanczos-factored-windows" if windows else "lanczos-factored")
    assert det["n_clusters"] == ref["n_clusters"]
    assert_routes_agree(det["eigenvalues"], ref["eigenvalues"])


@pytest.mark.parametrize("condition", list(CONDITIONS))
@pytest.mark.parametrize("n", [16384, 65536])
def test_predict_factored_equals_stored(engine, n, condition):
  one = np.tile(synthetic.speaker_turn_dvectors(1, 256, 1, seed=3), (n, 1))
  stored, factored = factored_and_stored(engine, clusterer(condition), one)
  assert np.array_equal(factored[0], np.zeros(n, dtype=factored[0].dtype))
  assert_same(stored, factored)
  four = synthetic.speaker_turn_dvectors(n, 256, 4, seed=n)
  stored, factored = factored_and_stored(engine, clusterer(condition), four)
  assert_same(stored, factored)
  if condition == "gmm-bic":
    assert factored[1]["single_cluster"]["passes"] > 0
    assert "eigenvalues" in factored[1]                  # the BIC prefers two components here


def test_predict_windows_factored_equals_stored(engine):
  n = 65536
  four = synthetic.speaker_turn_dvectors(n, 256, 4, seed=n)
  stored, factored = factored_and_stored(engine, clusterer("gmm-bic", max_clusters=None), four)
  assert_same(stored, factored, windows=True)
  assert "eigenvalues" in factored[1]


def test_fp16_cuda_input_equals_its_host_twin(engine):
  n = 16384
  x16 = torch.from_numpy(synthetic.speaker_turn_dvectors(n, 256, 4, seed=1)
                         .astype(np.float16)).to(engine.device)
  out = []
  saved = engine.factored_above_bytes
  engine.factored_above_bytes = 0
  try:
    for x in (x16, x16.cpu().numpy()):
      c = clusterer("gmm-bic")()
      np.random.seed(0)
      with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out.append((c.predict(x), dict(c.last_details)))
  finally:
    engine.factored_above_bytes = saved
  (got, det), (want, ref) = out
  assert det["solver"] == "lanczos-factored"
  assert np.array_equal(got, want)
  assert det["single_cluster"] == ref["single_cluster"]
  np.testing.assert_array_equal(det["eigenvalues"], ref["eigenvalues"])


def test_n131072_on_one_gpu(engine):
  """Route not forced: the stored route's 172 GB peak does not fit, the factored route's does.
  The check holds the packed band and one panel; the refinement Y_hi and two panels."""
  n = 131072
  four = synthetic.speaker_turn_dvectors(n, 256, 4, seed=0).astype(np.float32)
  peaks, results = [], []
  for mc in (2, 1):
    c = scb.SpectralClusterer(min_clusters=mc, max_clusters=10,
                              refinement_options=scb.configs.icassp2018_refinement_options,
                              custom_dist="cosine")
    assert (c._factored_route(engine, n) if mc == 2 else
            c._factored_single_cluster_route(engine, n))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(engine.device)
    np.random.seed(0)
    results.append((c.predict(four), dict(c.last_details)))
    peaks.append(torch.cuda.max_memory_allocated(engine.device))
  (want, _), (got, det) = results
  assert np.array_equal(got, want)
  assert det["solver"] == "lanczos-factored"
  bic = det["single_cluster"]["bic"]
  assert bic[0] > bic[1]
  assert peaks[1] <= peaks[0] + (64 << 20), peaks
  print("N=131072: peak %.2f GB with min_clusters=1, %.2f GB with min_clusters=2; %d passes" % (
      peaks[1] / 1e9, peaks[0] / 1e9, det["single_cluster"]["passes"]))

  one = np.tile(synthetic.speaker_turn_dvectors(1, 256, 1, seed=3), (n, 1)).astype(np.float32)
  c = scb.SpectralClusterer(min_clusters=1, max_clusters=10,
                            refinement_options=scb.configs.icassp2018_refinement_options)
  np.random.seed(0)
  with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    labels = c.predict(one)
  assert np.array_equal(labels, np.zeros(n, dtype=labels.dtype))
