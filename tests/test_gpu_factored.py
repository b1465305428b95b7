"""GPU: the factored route of predict() (no N x N fp32 matrix) against the stored route.

Its panels must reproduce the stored route's affinity rows, crop values, blur maxima m and Y_hi bit
for bit; the statistics-only Diffuse its row statistics bit for bit; the fp16 block product a
float64 product of the upcast Y_hi to within its summation bound; and predict() the stored route's
labels and k.  The route is forced at small N by setting Engine.factored_above_bytes = 0 and a
single-MMA Diffuse."""

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import laplacian as lap_lib
from oracle import spectral_oracle as orc

RN = scb.RefinementName
pytestmark = pytest.mark.gpu


def icassp(seq=None, p=0.95):
  return scb.RefinementOptions(gaussian_blur_sigma=1, p_percentile=p,
                               thresholding_soft_multiplier=0.01,
                               thresholding_type=scb.ThresholdType.RowMax,
                               refinement_sequence=seq or list(scb.configs.ICASSP2018_REFINEMENT_SEQUENCE))


def embeddings(engine, n, speakers=5, seed=7):
  t = dev.torch()
  return t.from_numpy(orc.synthetic_dvectors(n, 256, speakers, seed=seed).astype(np.float32)).to(
      engine.device)


def stored_front(engine, x, opt):
  """Stored route: A, crop, m and Y_hi by the whole-matrix kernels."""
  n = int(x.shape[0])
  a, crop = engine.affinity(x, want_crop_vector=True)
  b, m = engine.blur_upper_rowmax(a, n, 1.0, crop, False)
  _, hi, _ = engine.threshold_symmetrize_upper(b, n, m, opt.p_percentile, 0.01, False, False,
                                               nat.SYMMETRIZE_MAX, False, True, want_lo=False)
  del b
  return a, crop, m, hi


def bits(t):
  return t.contiguous().view(dev.torch().int16 if t.element_size() == 2 else dev.torch().int32)


@pytest.mark.parametrize("n", [4097, 16384, 65536])
def test_panels_equal_the_whole_matrix(engine, n):
  t = dev.torch()
  x = embeddings(engine, n)
  opt = icassp()
  a, crop, m, hi = stored_front(engine, x, opt)
  ys = []
  for rows in (dev.PANEL_ALIGN * 3, dev.PANEL_ALIGN * 16):
    fa = dev.FactoredAffinity(engine, x, panel_rows=rows)
    diag = engine.vector(n, t.float32)
    for r0, r1, a0, a1 in dev.panel_plan(n, rows)[:3] + dev.panel_plan(n, rows)[-2:]:
      panel = engine.affinity_panel(fa.hi, fa.lo, n, fa.d, a0, a1, diag)
      assert t.equal(bits(panel[:, :n]), bits(a[a0:a1, :n])), (rows, a0, a1)
      assert t.equal(bits(diag[a0:a1]), bits(crop[a0:a1]))
    assert t.equal(bits(fa.rowmax(engine, opt)), bits(m))
    refined = fa.refine(engine, opt)
    y = refined.y_hi[:, :n]
    assert t.equal(bits(y), bits(hi[:, :n]))
    assert t.equal(bits(y), bits(y.T))
    ys.append(refined.y_hi)
    del fa, refined
  assert t.equal(bits(ys[0][:, :n]), bits(ys[1][:, :n]))


@pytest.mark.parametrize("n", [4097, 16384])
def test_stats_only_diffuse_equals_the_storing_call(engine, n):
  t = dev.torch()
  x = embeddings(engine, n)
  _, _, _, hi = stored_front(engine, x, icassp())
  _, mx, sm = engine.diffuse(n, hi=hi, lo=None, want_stats=True, precision=nat.GEMM_SINGLE)
  mx2, sm2 = engine.diffuse_stats(n, hi)
  assert t.equal(bits(mx2), bits(mx))
  assert t.equal(sm2.view(t.int64), sm.view(t.int64))


@pytest.mark.parametrize("b", [1, 5, 16])
@pytest.mark.parametrize("n", [4097, 16384])
def test_block_product_f16_vs_float64(engine, n, b):
  """y = Y_hi T against the float64 product of the upcast Y_hi.  Every product of an fp16 value and
  an fp64 value is exact in fp64 to one rounding; a sum of n such terms is off by at most
  gamma_n sum |y_ij t_j| with gamma_n = n u / (1 - n u), u = 2^-53."""
  t = dev.torch()
  x = embeddings(engine, n)
  _, _, _, hi = stored_front(engine, x, icassp())
  g = t.Generator(device=engine.device).manual_seed(n + b)
  ld = n + (n & 1)
  tv = t.zeros((b, ld), dtype=t.float64, device=engine.device)
  tv[:, :n] = t.randn((b, n), generator=g, dtype=t.float64, device=engine.device)
  y = t.empty((b, n), dtype=t.float64, device=engine.device)
  engine.block_product_f16(hi, n, n, tv, b, y)
  y64 = hi[:, :n].double()
  want = (y64 @ tv[:, :n].T).T
  bound = (y64.abs() @ tv[:, :n].abs().T).T
  u = 2.0 ** -53
  gamma = 2 * n * u / (1 - 2 * n * u)          # the reference product rounds too
  assert ((y - want).abs() <= gamma * bound + 1e-300).all()


def assert_routes_agree(w, w_stored):
  """Eigenvalues of the two routes.  The stored S is the fp32 tensor-core accumulation of the
  product the factored operator applies exactly, and both routes take the Laplacian degrees from
  that accumulation's row sums.  So they differ by up to ~1e-5 relative (8.3e-6 measured, N =
  16,384) and, through the degree/operator mismatch, ~1.4e-6 absolute on a GraphCut spectrum in
  [0, 1] (lambda_0: -1.3e-6 against 1e-11).  Each route is held to the project's float64 contract,
  |dw| <= 1e-5 |w| + 1e-6 max|w|, so two routes agree within twice it."""
  w, w_stored = np.asarray(w), np.asarray(w_stored)
  np.testing.assert_allclose(w, w_stored, rtol=2e-5, atol=2e-6 * np.abs(w_stored).max())


def factored_residuals(y_hi, n, terms, w, v, chunk=8192):
  """max_j |M v_j - w_j v_j| with M = diag(delta) + sign diag(left) Y Y^T diag(right), Y = Y_hi in
  float64, applied in row chunks of Y_hi."""
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


@pytest.mark.parametrize("laplacian", [None, scb.LaplacianType.GraphCut])
@pytest.mark.parametrize("n", [16384, 65536])
def test_factored_lanczos_vs_stored(engine, n, laplacian):
  x = embeddings(engine, n)
  refined = dev.FactoredAffinity(engine, x).refine(engine, icassp())
  terms = lap_lib.operator_terms(engine, refined, laplacian)
  delta, left, right, sign, which = terms
  w, v, stats = engine.eigh_factored(refined.y_hi, n, delta, left, right, sign, which, 11, 8)
  s, _, _ = engine.diffuse(n, hi=refined.y_hi, lo=None, precision=nat.GEMM_SINGLE)
  w2, _, _ = engine.eigh(s, n, delta, left, right, sign, which, 11, 8, dense=False)
  del s
  assert_routes_agree(w, w2)
  assert max(factored_residuals(refined.y_hi, n, terms, w, v)) <= 1e-7 * max(1.0, abs(w).max())
  assert stats[2] == 11


SEQ_NO_NORMALIZE = [RN.CropDiagonal, RN.GaussianBlur, RN.RowWiseThreshold, RN.Symmetrize,
                    RN.Diffuse]
CASES = {
    "icassp-graphcut": dict(laplacian_type=scb.LaplacianType.GraphCut),
    "icassp": dict(),
    "normalized-diff": dict(laplacian_type=scb.LaplacianType.GraphCut,
                            eigengap_type=scb.EigenGapType.NormalizedDiff),
    "no-normalize": dict(laplacian_type=scb.LaplacianType.GraphCut, seq=SEQ_NO_NORMALIZE),
}


def clusterer(case, autotune=None):
  kw = dict(CASES[case])
  seq = kw.pop("seq", None)
  return scb.SpectralClusterer(min_clusters=2, max_clusters=10, refinement_options=icassp(seq),
                               autotune=autotune, custom_dist="cosine", **kw)


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("n", [16384, 65536])
def test_predict_factored_equals_stored(engine, n, case):
  if n == 65536 and case in ("icassp", "no-normalize"):
    pytest.skip("covered at 16,384; two cases at 65,536 keep the file's run time down")
  x = orc.synthetic_dvectors(n, 256, 6, seed=11).astype(np.float32)
  saved = engine.diffuse_precision
  engine.diffuse_precision = nat.GEMM_SINGLE
  try:
    c = clusterer(case)
    want = c.predict(x)
    ref = dict(c.last_details)
    engine.factored_above_bytes, saved_limit = 0, engine.factored_above_bytes
    try:
      got = c.predict(x)
    finally:
      engine.factored_above_bytes = saved_limit
  finally:
    engine.diffuse_precision = saved
  assert ref["solver"] == "lanczos" and c.last_details["solver"] == "lanczos-factored"
  assert c.last_details["n_clusters"] == ref["n_clusters"]
  assert np.array_equal(got, want)
  assert_routes_agree(c.last_details["eigenvalues"], ref["eigenvalues"])


def test_autotune_factored_equals_stored(engine):
  n = 16384
  x = orc.synthetic_dvectors(n, 256, 6, seed=5).astype(np.float32)
  out = []
  for limit in (engine.factored_above_bytes, 0):
    saved = engine.factored_above_bytes
    engine.factored_above_bytes = limit
    try:
      c = clusterer("icassp-graphcut", autotune=scb.AutoTune(p_percentile_min=0.6,
                                                             p_percentile_max=0.95,
                                                             init_search_step=0.05,
                                                             search_level=1))
      labels = c.predict(x)
    finally:
      engine.factored_above_bytes = saved
    out.append((labels, c.last_details))
  (want, ref), (got, det) = out
  assert ref["solver"] == "lanczos" and det["solver"] == "lanczos-factored"
  assert det["best_p_percentile"] == ref["best_p_percentile"]
  assert det["n_clusters"] == ref["n_clusters"]
  assert np.array_equal(got, want)


@pytest.mark.parametrize("laplacian", [None, scb.LaplacianType.GraphCut])
def test_n131072_on_one_gpu(engine, laplacian):
  """BASELINE configs[3]'s size on one H100, route not forced.  Needs about 40 GB of free device
  memory: Y_hi (34.4 GB), two 1 GB panels and the fp64 row chunks of the residual check."""
  t = dev.torch()
  n = 131072
  x, truth = orc.synthetic_dvectors(n, 256, 6, seed=0, return_labels=True)
  c = scb.SpectralClusterer(min_clusters=2, max_clusters=10,
                            refinement_options=scb.configs.icassp2018_refinement_options,
                            laplacian_type=laplacian, custom_dist="cosine")
  assert c._factored_route(engine, n)
  t.cuda.synchronize()
  t.cuda.reset_peak_memory_stats(engine.device)
  labels = c.predict(x.astype(np.float32))
  peak = t.cuda.max_memory_allocated(engine.device)
  assert c.last_details["solver"] == "lanczos-factored"
  ld = dev.round_up(n, 64)
  assert peak < 4 * n * ld, peak
  assert np.array_equal(scb.utils.enforce_ordered_labels(labels), orc.ordered(truth))
  # eigenpair residuals on the same Y_hi, float64, in row chunks
  fa = dev.FactoredAffinity(engine, t.from_numpy(x.astype(np.float32)).to(engine.device))
  refined = fa.refine(engine, c.refinement_options)
  del fa
  terms = lap_lib.operator_terms(engine, refined, laplacian)
  w, v, _ = engine.eigh_factored(refined.y_hi, n, *terms, 11, 4)
  np.testing.assert_allclose(w, c.last_details["eigenvalues"], rtol=1e-9,
                             atol=1e-12 * np.abs(w).max())
  assert max(factored_residuals(refined.y_hi, n, terms, w, v)) <= 1e-7 * max(1.0, abs(w).max())
  print("N=131072 %s: peak %.1f GB (2 N ld = %.1f GB)" % (
      laplacian, peak / 1e9, 2 * n * ld / 1e9))
