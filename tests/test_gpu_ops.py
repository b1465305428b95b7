"""GPU: every CUDA operator against the CPU oracle on the same seeded inputs (through the
Python mirror of the reference API, i.e. through the C ABI).  fp32 storage => tolerances are a
few fp32 ulps of the matrix scale; integer-valued known answers must be exact."""

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from oracle import spectral_oracle as orc

pytestmark = pytest.mark.gpu

F32 = 2.0 ** -23


def rand_affinity(n, d=24, seed=0):
  rng = np.random.default_rng(seed)
  return orc.affinity(rng.standard_normal((n, d)))


def close(got, want, ulps=8, scale=None):
  scale = np.max(np.abs(want)) if scale is None else scale
  np.testing.assert_allclose(got, want, rtol=0, atol=ulps * F32 * scale)


# ---------------------------------------------------------------- known answers (reference tests)
def test_affinity_known_answer():            # tests/utils_test.py:10-15
  m = np.array([[3, 4], [-4, 3], [6, 8], [-3, -4]])
  want = np.array([[1, 0.5, 1, 0], [0.5, 1, 0.5, 0.5], [1, 0.5, 1, 0], [0, 0.5, 0, 1]])
  close(scb.utils.compute_affinity_matrix(m), want, ulps=2, scale=1.0)


def test_refinement_known_answers():         # tests/refinement_test.py:12-108
  m = np.array([[1, 2, 3], [3, 4, 5], [4, 2, 1]])
  np.testing.assert_equal(scb.refinement.CropDiagonal().refine(m),
                          np.array([[3, 2, 3], [3, 5, 5], [4, 2, 4]]))
  got = scb.refinement.GaussianBlur(sigma=1).refine(m.astype(float))
  np.testing.assert_allclose(got, [[2.12, 2.61, 3.10], [2.76, 2.90, 3.06], [3.16, 2.78, 2.46]],
                             atol=0.01)
  m3 = np.array([[0.5, 2.0, 3.0], [3.0, 4.0, 5.0], [4.0, 2.0, 1.0]])
  T, TT = scb.refinement.RowWiseThreshold, scb.ThresholdType
  np.testing.assert_allclose(T(0.5, 0.01, TT.Percentile).refine(m3),
                             [[0.005, 2.0, 3.0], [0.03, 4.0, 5.0], [4.0, 2.0, 0.01]], atol=0.001)
  np.testing.assert_allclose(T(0.5, 0.01, TT.RowMax).refine(m3),
                             [[0.005, 2.0, 3.0], [3.0, 4.0, 5.0], [4.0, 2.0, 0.01]], atol=0.001)
  np.testing.assert_allclose(T(0.5, 0.01, TT.RowMax, True).refine(m3),
                             [[0.005, 1.0, 1.0], [1.0, 1.0, 1.0], [1.0, 1.0, 0.01]], atol=0.001)
  np.testing.assert_allclose(T(0.5, 0.01, TT.RowMax, True, True).refine(m3), np.ones((3, 3)),
                             atol=0.001)
  np.testing.assert_equal(scb.refinement.Symmetrize().refine(m),
                          np.array([[1, 3, 4], [3, 4, 5], [4, 5, 1]]))
  np.testing.assert_equal(
      scb.refinement.Symmetrize(scb.SymmetrizeType.Average).refine(m),
      np.array([[1, 2.5, 3.5], [2.5, 4, 3.5], [3.5, 3.5, 1]]))
  np.testing.assert_equal(scb.refinement.Diffuse().refine(np.array([[1, 2], [3, 4]])),
                          np.array([[5, 11], [11, 25]]))
  np.testing.assert_allclose(scb.refinement.RowWiseNormalize().refine(m3),
                             [[0.167, 0.667, 1.0], [0.6, 0.8, 1.0], [1.0, 0.5, 0.25]], atol=0.001)


def test_laplacian_known_answers():          # tests/laplacian_test.py:13-45
  a = orc.affinity(np.array([[3, 4], [-4, 3], [6, 8], [-3, -4]]))
  L = scb.laplacian.compute_laplacian
  LT = scb.LaplacianType
  np.testing.assert_allclose(L(a, LT.Affinity), a, atol=1e-7)
  np.testing.assert_allclose(L(a, LT.Unnormalized),
                             [[1.5, -0.5, -1, 0], [-0.5, 1.5, -0.5, -0.5], [-1, -0.5, 1.5, 0],
                              [0, -0.5, 0, 0.5]], atol=1e-6)
  np.testing.assert_allclose(L(a, LT.GraphCut), orc.laplacian(a, "graphcut"), atol=1e-6)
  np.testing.assert_allclose(L(a, LT.RandomWalk), orc.laplacian(a, "randomwalk"), atol=1e-6)
  with pytest.raises(TypeError):
    L(a, "graphcut")


# ---------------------------------------------------------------- operators vs oracle, seeded
@pytest.mark.parametrize("n,d", [(5, 3), (63, 7), (64, 16), (200, 33), (777, 128), (1100, 256)])
def test_affinity_vs_oracle(n, d):
  rng = np.random.default_rng(n)
  x = rng.standard_normal((n, d))
  close(scb.utils.compute_affinity_matrix(x), orc.affinity(x), ulps=4, scale=1.0)
  close(scb.utils.compute_affinity_matrix(x.astype(np.float32)),
        orc.affinity(x.astype(np.float32).astype(np.float64)), ulps=4, scale=1.0)


@pytest.mark.parametrize("n", [3, 40, 257, 1000])
def test_crop_diagonal_vs_oracle(n):
  a = rand_affinity(n, seed=n).astype(np.float32).astype(np.float64)
  np.testing.assert_array_equal(scb.refinement.CropDiagonal().refine(a), orc.crop_diagonal(a))


@pytest.mark.parametrize("n,sigma", [(3, 1), (7, 2), (100, 1), (129, 0.7), (300, 2), (515, 1),
                                     (1000, 1), (64, 0), (50, 3.3)])
def test_gaussian_blur_vs_scipy(n, sigma):
  a = rand_affinity(n, seed=7 + n).astype(np.float32).astype(np.float64)
  close(scb.refinement.GaussianBlur(sigma).refine(a), orc.gaussian_blur(a, sigma), ulps=6,
        scale=1.0)


@pytest.mark.parametrize("kind", ["rowmax", "percentile"])
@pytest.mark.parametrize("binarize,keep_diag", [(False, False), (True, False), (False, True),
                                                (True, True)])
def test_row_threshold_vs_oracle(kind, binarize, keep_diag):
  TT = {"rowmax": scb.ThresholdType.RowMax, "percentile": scb.ThresholdType.Percentile}[kind]
  for n, p, mult in ((6, 0.95, 0.01), (211, 0.5, 0.0), (600, 0.3, 0.5), (1025, 0.9, 0.01)):
    a = rand_affinity(n, seed=n).astype(np.float32).astype(np.float64)
    got = scb.refinement.RowWiseThreshold(p, mult, TT, binarize, keep_diag).refine(a)
    want = orc.row_threshold(a, p, mult, kind, binarize, keep_diag)
    # elements within an fp32 ulp of the cut may legitimately land on the other side
    bad = np.abs(got - want) > 4 * F32
    assert bad.mean() <= 2e-5, "%d of %d elements differ" % (bad.sum(), bad.size)


@pytest.mark.parametrize("n", [3, 33, 500, 1030])
def test_symmetrize_vs_oracle(n):
  rng = np.random.default_rng(n)
  a = rng.random((n, n)).astype(np.float32).astype(np.float64)
  np.testing.assert_array_equal(scb.refinement.Symmetrize().refine(a), orc.symmetrize(a))
  close(scb.refinement.Symmetrize(scb.SymmetrizeType.Average).refine(a),
        orc.symmetrize(a, "average"), ulps=1, scale=1.0)


@pytest.mark.parametrize("n", [2, 40, 64, 130, 513, 1000, 1537])
def test_diffuse_vs_oracle(n):
  rng = np.random.default_rng(n)
  y = rng.random((n, n)).astype(np.float32).astype(np.float64)     # not symmetric on purpose
  want = orc.diffuse(y)
  got = scb.refinement.Diffuse().refine(y)
  # split-fp16 tensor-core product: ~2^-22 per term, fp32 accumulation over n terms
  np.testing.assert_allclose(got, want, rtol=3e-6, atol=0)


def test_diffuse_engines_agree(engine):
  n = 900
  rng = np.random.default_rng(3)
  y = rng.random((n, n)).astype(np.float32)
  yd = engine.upload_matrix(y)
  old = engine.simt_below
  try:
    engine.simt_below = 10 ** 9
    s_simt = engine.download_matrix(engine.diffuse(n, y=yd)[0], n)
    engine.simt_below = 0
    s_tc = engine.download_matrix(engine.diffuse(n, y=yd)[0], n)
  finally:
    engine.simt_below = old
  want = y.astype(np.float64) @ y.astype(np.float64).T
  np.testing.assert_allclose(s_simt, want, rtol=2 * F32, atol=0)   # fp64 accumulate: exact + rounding
  np.testing.assert_allclose(s_tc, want, rtol=3e-6, atol=0)


@pytest.mark.parametrize("n", [3, 100, 1024])
def test_row_normalize_vs_oracle(n):
  a = rand_affinity(n, seed=n).astype(np.float32).astype(np.float64)
  close(scb.refinement.RowWiseNormalize().refine(a), orc.row_normalize(a), ulps=1, scale=1.0)


@pytest.mark.parametrize("kind", ["unnormalized", "randomwalk", "graphcut"])
def test_laplacian_vs_oracle(kind):
  LT = {"unnormalized": scb.LaplacianType.Unnormalized, "randomwalk": scb.LaplacianType.RandomWalk,
        "graphcut": scb.LaplacianType.GraphCut}[kind]
  a = rand_affinity(500, seed=11).astype(np.float32).astype(np.float64)
  want = orc.laplacian(a, kind)
  close(scb.laplacian.compute_laplacian(a, LT), want, ulps=2)


@pytest.mark.parametrize("sigma,sym,binarize,keep_diag,crop", [
    (1, "max", False, False, True), (0, "max", False, False, True),
    (1, "average", False, False, True), (2, "max", True, False, False),
    (1, "max", False, True, True), (0, "average", True, True, False)])
def test_fused_chain_equals_operator_chain(engine, sigma, sym, binarize, keep_diag, crop):
  """crop? -> blur -> threshold(RowMax) -> symmetrize: fused kernels == oracle composition."""
  n = 700
  a = rand_affinity(n, d=40, seed=21).astype(np.float32).astype(np.float64)
  names = (["crop"] if crop else []) + ["blur", "threshold", "symmetrize"]
  opt = orc.options(sequence=tuple(names), sigma=sigma, p=0.9, mult=0.01, binarize=binarize,
                    preserve_diagonal=keep_diag, symmetrize_type=sym)
  want = orc.refine(a, opt)
  RN = scb.RefinementName
  ro = scb.RefinementOptions(
      gaussian_blur_sigma=sigma, p_percentile=0.9, thresholding_soft_multiplier=0.01,
      thresholding_with_binarization=binarize, thresholding_preserve_diagonal=keep_diag,
      symmetrize_type=scb.SymmetrizeType.Max if sym == "max" else scb.SymmetrizeType.Average,
      refinement_sequence=([RN.CropDiagonal] if crop else []) +
      [RN.GaussianBlur, RN.RowWiseThreshold, RN.Symmetrize])
  refined = dev.run_refinement(engine, engine.upload_matrix(a), n, ro)
  assert refined.symmetric and refined.row_scale is None
  got = engine.download_matrix(refined.s, n)
  bad = np.abs(got - want) > 8 * F32
  assert bad.mean() <= 2e-5, "%d elements differ" % bad.sum()


# ---------------------------------------------------------------- eigensolvers
def structured_problem(n, seed, kind):
  rng = np.random.default_rng(seed)
  x = orc.synthetic_dvectors(n, 32, 5, seed=seed)
  s = orc.affinity(x)
  s = (s @ s.T).astype(np.float32).astype(np.float64)
  left = 1.0 / s.max(axis=1)
  if kind == "rownorm":
    m = left[:, None] * s
    return s, None, left, None, 1.0, nat.EIG_LARGEST, m
  d = left * s.sum(axis=1)
  inv = 1.0 / (np.sqrt(d) + 1e-10)
  m = np.diag(inv * d * inv) - (inv * left)[:, None] * s * inv[None, :]
  return s, inv * d * inv, inv * left, inv, -1.0, nat.EIG_SMALLEST, m


def run_eigh(engine, s, delta, left, right, sign, which, nv, nvec, dense):
  t = dev.torch()
  up = lambda v: None if v is None else t.from_numpy(np.ascontiguousarray(v)).to(engine.device)
  n = s.shape[0]
  w, v, stats = engine.eigh(engine.upload_matrix(s), n, up(delta), up(left), up(right), sign,
                            which, nv, nvec, dense)
  return w, v.to("cpu").numpy(), stats


@pytest.mark.parametrize("n", [1, 2, 3, 6, 50, 301, 1000])
def test_dense_eigh_plain_symmetric(engine, n):
  rng = np.random.default_rng(n)
  a = rng.standard_normal((n, n))
  a = ((a + a.T) / 2).astype(np.float32).astype(np.float64)
  w, v, _ = run_eigh(engine, a, None, None, None, 1.0, nat.EIG_LARGEST, n, n, True)
  ref = np.linalg.eigvalsh(a)[::-1]
  np.testing.assert_allclose(w, ref, rtol=0, atol=1e-11 * max(1.0, np.abs(ref).max()))
  resid = a @ v - v * w[None, :]
  assert np.abs(resid).max() <= 1e-10 * max(1.0, np.abs(ref).max())
  np.testing.assert_allclose(v.T @ v, np.eye(n), atol=1e-10)


@pytest.mark.parametrize("kind", ["rownorm", "graphcut"])
def test_dense_eigh_similarity_form_matches_np_eig(engine, kind):
  """Eigenpairs of the NON-symmetric matrix the reference decomposes (utils.py:59)."""
  n = 400
  s, delta, left, right, sign, which, m = structured_problem(n, 5, kind)
  w, v, _ = run_eigh(engine, s, delta, left, right, sign, which, n, 12, True)
  wr, vr = orc.sorted_eig(m, descend=(which == nat.EIG_LARGEST))
  np.testing.assert_allclose(w[:12], wr[:12], rtol=1e-9, atol=1e-10 * np.abs(wr).max())
  np.testing.assert_allclose(np.linalg.norm(v, axis=0), 1.0, atol=1e-12)
  for c in range(8):     # up to sign; skip (near-)degenerate pairs by checking the residual
    r = m @ v[:, c] - w[c] * v[:, c]
    assert np.abs(r).max() <= 1e-9 * np.abs(wr).max()


@pytest.mark.parametrize("kind", ["rownorm", "graphcut"])
def test_lanczos_matches_dense(engine, kind):
  n = 3000
  s, delta, left, right, sign, which, m = structured_problem(n, 9, kind)
  wd, vd, _ = run_eigh(engine, s, delta, left, right, sign, which, n, 8, True)
  wl, vl, stats = run_eigh(engine, s, delta, left, right, sign, which, 11, 8, False)
  np.testing.assert_allclose(wl, wd[:11], rtol=1e-8, atol=1e-9 * np.abs(wd).max())
  for c in range(8):
    r = m @ vl[:, c] - wl[c] * vl[:, c]
    assert np.abs(r).max() <= 1e-6 * np.abs(wd).max()
  assert stats[0] > 0


@pytest.mark.parametrize("which", [nat.EIG_LARGEST, nat.EIG_SMALLEST])
def test_lanczos_thick_restart_on_dense_spectrum(engine, which):
  """A random symmetric matrix has no gaps at the edge of its spectrum: the 64-vector basis is not
  enough and the solver has to restart (several times) -- exercises k_combine / the arrowhead."""
  n = 1500
  rng = np.random.default_rng(1)
  b = rng.standard_normal((n, n))
  a = ((b + b.T) / 2).astype(np.float32).astype(np.float64)
  w, v, stats = run_eigh(engine, a, None, None, None, 1.0, which, 11, 11, False)
  ref = np.linalg.eigvalsh(a)
  ref = ref[::-1][:11] if which == nat.EIG_LARGEST else ref[:11]
  np.testing.assert_allclose(w, ref, rtol=0, atol=1e-8 * np.abs(ref).max())
  assert stats[1] >= 1 and stats[2] == 11          # restarted, and all 11 pairs converged
  resid = a @ v - v * w[None, :]
  assert np.abs(resid).max() <= 1e-6 * np.abs(ref).max()
  np.testing.assert_allclose(v.T @ v, np.eye(11), atol=1e-8)


# ---------------------------------------------------------------- k-means
@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
@pytest.mark.parametrize("n,k,seed", [(6, 2, 0), (450, 5, 1), (1000, 4, 2), (5000, 7, 3),
                                      (20000, 10, 4)])
def test_kmeans_vs_oracle(metric, n, k, seed):
  rng = np.random.default_rng(seed)
  if n == 6:
    e = np.array([[1.0, 0.0], [1.1, 0.1], [0.0, 1.0], [0.1, 1.0], [0.9, -0.1], [0.0, 1.2]])
  else:
    cent = rng.standard_normal((k, k)) * 2
    e = cent[rng.integers(0, k, n)] + 0.35 * rng.standard_normal((n, k))
  got = scb.custom_distance_kmeans.run_kmeans(e, k, metric, 300)
  want = orc.run_kmeans(e, k, metric, 300)
  np.testing.assert_array_equal(got, want)      # same seeds => same raw labels, not just up to order
  assert got.dtype == np.int64


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_kmeans_lonely_first_sample_quirk(metric):
  """Sample 0 alone in its cluster: `np.where(...)[0].any()` is False for array([0]), so the
  reference never updates that centroid (custom_distance_kmeans.py:137-138, SURVEY A.4-3)."""
  rng = np.random.default_rng(12)
  e = np.vstack([[[9.0, -7.0, 8.0]], rng.standard_normal((150, 3)) * 0.2 + [1, 1, 0],
                 rng.standard_normal((150, 3)) * 0.2 + [-1, 0.5, 1]])
  got = scb.custom_distance_kmeans.run_kmeans(e, 3, metric, 300)
  want = orc.run_kmeans(e, 3, metric, 300)
  np.testing.assert_array_equal(got, want)


def test_kmeans_errors():
  e = np.random.default_rng(0).random((10, 3))
  with pytest.raises(ValueError):
    scb.custom_distance_kmeans.run_kmeans(e, 3, "cosine", 0)
  with pytest.raises(ValueError):
    scb.custom_distance_kmeans.run_kmeans(e, 11, "cosine", 10)


@pytest.mark.parametrize("metric", ["cityblock", "chebyshev"])
def test_kmeans_generic_scipy_metric_matches_oracle(engine, metric):
  """Any other scipy metric name (custom_distance_kmeans.py:37-47) is the user-hook seam: host
  arrays in and out on the [n, k] embeddings, like the reference."""
  rng = np.random.default_rng(3)
  e = np.vstack([rng.standard_normal((120, 4)) * 0.2 + c for c in ([2, 0, 0, 0], [0, 2, 0, 1], [0, 0, 2, -1])])
  got = scb.custom_distance_kmeans.run_kmeans(e, 3, metric, 50)
  want = orc.run_kmeans(e, 3, metric, 50)
  np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("rows,n,b", [(1, 7, 1), (255, 33, 4), (256, 1000, 8), (1000, 1000, 12),
                                      (2304, 2304, 16), (777, 4099, 11), (8192, 16384, 12)])
def test_block_product_vs_float64(engine, rows, n, b):
  """sc_block_product (fp64 DMMA, cp.async ring, column splits) against the float64 product of the
  same fp32 matrix: ragged rows / columns / block widths; bit-reproducible from run to run."""
  import ctypes
  t = dev.torch()
  g = t.Generator(device="cpu").manual_seed(rows * 31 + n)
  ld = dev.round_up(n, 64)
  s = t.full((rows, ld), float("nan"), dtype=t.float32)          # the padding must never be read
  s[:, :n] = t.rand((rows, n), generator=g) - 0.3
  ldt = n + (n & 1) + 2
  tv = t.randn((b, ldt), generator=g, dtype=t.float64)
  s_d, t_d = s.to(engine.device), tv.to(engine.device)
  outs = []
  for _ in range(2):
    y = t.zeros((b, rows), dtype=t.float64, device=engine.device)
    engine.call("sc_block_product", dev._ptr(s_d), rows, n, ld, dev._ptr(t_d), ldt, ctypes.c_int(b),
                dev._ptr(y), rows, engine.stream)
    outs.append(y.cpu())
  want = tv[:, :n] @ s[:, :n].double().T
  scale = (tv[:, :n].abs() @ s[:, :n].double().abs().T).clamp_min(1e-300)
  assert float(((outs[0] - want).abs() / scale).max()) <= 1e-14
  assert t.equal(outs[0], outs[1])
