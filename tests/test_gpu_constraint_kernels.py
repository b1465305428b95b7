"""GPU: the constraint operators' kernels at their edges, and ConstraintPropagation against float64.

Every element-wise case calls the C ABI directly with NaN in the padding of its inputs and a
sentinel in the padding of its outputs.  The propagation is compared with a float64 restatement of
the reference's AffinityIntegration / ConstraintPropagation (constraint.py:95-164 of the reference:
np.linalg.inv of I - alpha Abar), and predict() with constraints with a float64 host composition of
that restatement and the oracle's refine / laplacian / sorted_eig / number_of_clusters / run_kmeans.

Error model of the propagation.  The device holds M = I - alpha Abar in fp32 (a backward error of
u = 2^-24 relative) and inverts it by Newton-Schulz, which corrects every earlier rounding, so the
inverse carries a forward error of about cond(M) u, cond(M) <= (1 + |a|) / (1 - |a|) since Abar's
spectrum lies in [-1, 1]; F = (1 - a)^2 X Q X holds X twice (2 cond u) and a fixed point of the
iteration has a backward error of its own last products (another 2 cond u).  The products after
the last correction (the last step's two, X Q and (X Q) X) each add the split-fp16 wgmma error
gamma_N = (40 + N / 128) 2^-24 of their scale (8 full-size wgmmas per 2-K-block chain, N / 128
chains, the 2^-22 of the operand split; test_gpu_affinity_tiles.py derives the chain terms), taken
twice.  The final combine has a derivative in [0, 1] with respect to F for an affinity in [0, 1],
and rounds once more.  So, element-wise,
    |adj - adj_ref| <= 4 u max(1, max|adj_ref|) + (4 cond u + 8 gamma_N) max|F_ref|.
Measured on an H100 (80 GB HBM3, 700 W), the relative error of F itself grows faster than
4 cond u -- about cond gamma_N / 2, the backward error of the fp32 products rather than of the
storage -- but up to |alpha| = 0.999 it stays inside the bound, which the fp32 floor of the
adjusted matrix dominates there.  At alpha = 0.9999 and N = 1,000 it is 1.6x outside, so
constraint.MAX_ABS_ALPHA = 0.999 and larger |alpha| raise NotImplementedError.
"""

import functools
import math
import re

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import constraint as ct
from spectralcluster_b200 import device as dev
from oracle import spectral_oracle as orc

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
NAN = float("nan")
SENTINEL = np.float32(-1234.5)


def t():
  return dev.torch()


def engine():
  return dev.Engine.get()


def device_buf(host, ld, fill):
  """Host [rows, cols] array in a device fp32 [rows, ld] buffer whose padding holds `fill`."""
  rows, cols = host.shape
  buf = t().full((rows, ld), float(fill), dtype=t().float32, device=engine().device)
  buf[:, :cols] = t().from_numpy(np.ascontiguousarray(host, dtype=np.float32)).to(engine().device)
  return buf


def host(buf):
  t().cuda.synchronize()
  return buf.cpu().numpy()


def bits(x):
  return np.ascontiguousarray(x, dtype=np.float32).view(np.int32)


def ulp32(x):
  return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def vec(h):
  return None if h is None else t().from_numpy(h).to(engine().device)


# ------------------------------------------------------------------ sc_transpose
TR = [1, 31, 32, 33, 95, 1000, 4097]


@pytest.mark.parametrize("cols", TR)
@pytest.mark.parametrize("rows", TR)
def test_transpose_is_exact_and_stays_in_bounds(rows, cols):
  rng = np.random.default_rng(rows * 8191 + cols)
  src_h = rng.standard_normal((rows, cols)).astype(np.float32)
  src_h.flat[::7] = -0.0
  src_h.flat[3::11] = np.inf
  lds, ldd = cols + 5, rows + 7                       # odd pitches: no alignment to lean on
  src = device_buf(src_h, lds, NAN)
  dst = t().full((cols, ldd), float(SENTINEL), dtype=t().float32, device=engine().device)
  e = engine()
  e.call("sc_transpose", dev._ptr(src), rows, cols, lds, dev._ptr(dst), ldd, e.stream)
  got = host(dst)
  np.testing.assert_array_equal(bits(got[:, :rows]), bits(src_h.T))
  assert (bits(got[:, rows:]) == bits(SENTINEL)).all(), "destination padding was written"


# ------------------------------------------------------------------ sc_scale_shift
SS_N = [1, 63, 64, 65, 255, 256, 257, 1000]


@pytest.mark.parametrize("alpha,beta", [(-0.37, 1.0), (0.0, 1.0), (1.7, 0.0), (-2.5, -0.75)])
@pytest.mark.parametrize("n", SS_N)
def test_scale_shift_matches_float64(n, alpha, beta):
  """out = ((alpha x) r_i) c_j (+ beta on the diagonal) in fp64, rounded once to fp32: bit for bit
  off the diagonal; 1 ulp on it, where nvcc may contract the + beta into an fp64 FMA."""
  rng = np.random.default_rng(n)
  x_h = rng.uniform(-2.0, 2.0, (n, n)).astype(np.float32)
  r_h = rng.uniform(0.1, 3.0, n)
  c_h = rng.uniform(0.1, 3.0, n)
  ld = dev.round_up(n, 64) + 64
  off = ~np.eye(n, dtype=bool)
  for use_r in (True, False):
    for use_c in (True, False):
      for alias in (False, True):
        x = device_buf(x_h, ld, NAN)
        out = x if alias else t().full((n, ld), float(SENTINEL), dtype=t().float32,
                                        device=engine().device)
        r, c = vec(r_h if use_r else None), vec(c_h if use_c else None)
        e = engine()
        e.call("sc_scale_shift", dev._ptr(x), ld, n, dev._ptr(r), dev._ptr(c), alpha, beta,
               dev._ptr(out), ld, e.stream)
        got = host(out)
        rr = r_h if use_r else np.ones(n)
        cc = c_h if use_c else np.ones(n)
        ref = ((alpha * x_h.astype(np.float64)) * rr[:, None]) * cc[None, :]
        ref[np.arange(n), np.arange(n)] += beta
        ref32 = ref.astype(np.float32)
        where = "n=%d r=%s c=%s alias=%s" % (n, use_r, use_c, alias)
        np.testing.assert_array_equal(bits(got[:, :n])[off], bits(ref32)[off], err_msg=where)
        d = np.arange(n)
        assert np.all(np.abs(got[d, d] - ref[d, d]) <= ulp32(ref32[d, d])), where
        pad = bits(got[:, n:])
        if alias:
          assert np.isnan(got[:, n:]).all(), where
        else:
          assert (pad == bits(SENTINEL)).all(), where


# ------------------------------------------------------------------ sc_constraint_combine
def reference_mode2(a, f):
  """constraint.py:158-163 of the reference, mask arithmetic and all, in float64."""
  is_positive = f > 0
  affinity1 = 1 - (1 - f * is_positive) * (1 - a * is_positive)
  affinity2 = (1 + f * np.invert(is_positive)) * (a * np.invert(is_positive))
  return affinity1 + affinity2


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n", [1, 63, 64, 257, 1000])
def test_constraint_combine(n, mode):
  rng = np.random.default_rng(10 * n + mode)
  a_h = rng.uniform(0.0, 1.0, (n, n)).astype(np.float32)
  f_h = rng.uniform(-3.0, 3.0, (n, n)).astype(np.float32)
  f_h.flat[0::11] = 0.0
  f_h.flat[1::11] = -0.0
  f_h.flat[2::13] = np.nan
  f_h.flat[4::19] = 1.0
  f_h.flat[5::19] = -1.0
  f_h.flat[6::23] = 1e-8                 # 1 - f rounds to 1: the cancellation case of mode 2
  a_h.flat[3::17] = np.nan
  a_h.flat[7::29] = 0.0
  ld = dev.round_up(n, 64) + 32
  for alias in (False, True):
    a = device_buf(a_h, ld, NAN)
    f = device_buf(f_h, ld, NAN)
    out = a if alias else t().full((n, ld), float(SENTINEL), dtype=t().float32,
                                    device=engine().device)
    e = engine()
    e.call("sc_constraint_combine", dev._ptr(a), ld, dev._ptr(f), ld, n, mode, dev._ptr(out), ld,
           e.stream)
    got = host(out)
    g = got[:, :n]
    if mode == 0:
      ref = np.maximum(a_h, f_h)
    elif mode == 1:
      ref = np.float32(0.5) * (a_h + f_h)
    else:
      ref = reference_mode2(a_h.astype(np.float64), f_h.astype(np.float64))
    nan = np.isnan(ref)
    np.testing.assert_array_equal(np.isnan(g), nan, err_msg="NaN does not propagate as np does")
    if mode < 2:                          # the same fp32 expression: bit for bit
      # except the sign of max(+-0, +-0), which differs between numpy's scalar and SIMD loops
      zeros = (a_h == 0) & (f_h == 0) if mode == 0 else np.zeros_like(nan)
      np.testing.assert_array_equal(bits(g)[~nan & ~zeros], bits(ref)[~nan & ~zeros])
      assert np.all(g[zeros] == 0)
    else:
      a64, f64 = a_h.astype(np.float64), f_h.astype(np.float64)
      pos = f64 > 0
      # f > 0: 1 - (1 - f)(1 - a): two operand roundings, the product's and (with or without an
      # FMA) the difference's, each <= 2^-24 of max(1, |(1 - f)(1 - a)|, |ref|) <= 2 ulps of it
      # once more for the fp32 spacing; f <= 0: (1 + f) a, two roundings of 2^-24 |ref|
      scale = np.where(pos, np.maximum(1.0, np.abs((1 - f64) * (1 - a64))), np.abs(ref))
      tol = np.where(pos, 4, 2) * ulp32(scale)
      err = np.abs(g.astype(np.float64) - ref)
      assert np.all(err[~nan] <= tol[~nan]), "mode 2: worst %g ulps" % np.max(
          (err / np.maximum(ulp32(scale), 1e-45))[~nan])
    if alias:
      assert np.isnan(got[:, n:]).all()
    else:
      assert (bits(got[:, n:]) == bits(SENTINEL)).all(), "output padding was written"


# ------------------------------------------------------------------ sc_gemm_nt_f32
@pytest.mark.parametrize("k", [1, 15, 16, 17, 300])
@pytest.mark.parametrize("n", [1, 63, 64, 65, 130])
@pytest.mark.parametrize("m", [1, 63, 64, 65, 130])
def test_gemm_nt_f32_against_exact_product(m, n, k):
  """fp32 x fp32 products are exact in fp64; the device sums them in fp64 (<= k 2^-53 sum|a||b|)
  and rounds once to fp32 (<= 1 ulp across a binade edge); the host's fp64 sum adds the same
  k 2^-53 sum|a||b| again."""
  rng = np.random.default_rng(m * 1000003 + n * 1009 + k)
  a_h = rng.standard_normal((m, k)).astype(np.float32)
  b_h = rng.standard_normal((n, k)).astype(np.float32)
  lda, ldb, ldc = k + 9, k + 3, n + 11
  a, b = device_buf(a_h, lda, NAN), device_buf(b_h, ldb, NAN)
  outs = []
  for _ in range(2):
    c = t().full((m, ldc), NAN, dtype=t().float32, device=engine().device)
    e = engine()
    e.call("sc_gemm_nt_f32", dev._ptr(a), lda, dev._ptr(b), ldb, m, n, k, dev._ptr(c), ldc,
           e.stream)
    outs.append(host(c))
  got = outs[0]
  assert np.isfinite(got[:, :n]).all(), "an output element was not written (or NaN padding read)"
  assert np.isnan(got[:, n:]).all(), "output padding was written"
  a64, b64 = a_h.astype(np.float64), b_h.astype(np.float64)
  exact = a64 @ b64.T
  tol = ulp32(exact) + 2 * k * 2.0 ** -53 * (np.abs(a64) @ np.abs(b64).T)
  assert np.all(np.abs(got[:, :n] - exact) <= tol)
  np.testing.assert_array_equal(bits(outs[1]), bits(got))


# ------------------------------------------------------------------ ConstraintPropagation
def restated_propagation(a, q, alpha, inv=None):
  """constraint.py:141-164 of the reference in float64 -> (adjusted affinity, final constraint F).
  The product inv Q inv runs over the rows/columns where Q is non-zero."""
  n = a.shape[0]
  if inv is None:
    degree_norm = 1 / (np.sqrt(a.sum(axis=1)) + ct.EPS)
    inv = np.linalg.inv(np.eye(n) - alpha * (degree_norm[:, None] * a * degree_norm[None, :]))
  s = np.flatnonzero(np.any(q != 0, axis=0) | np.any(q != 0, axis=1))
  f = (1 - alpha) ** 2 * (inv[:, s] @ (q[np.ix_(s, s)] @ inv[s, :]))
  return reference_mode2(a, f), f


@functools.lru_cache(maxsize=2)
def propagation_affinity(n):
  """Random unit vectors (d = 16), (x x^T + 1) / 2, rounded to the fp32 the device holds."""
  rng = np.random.default_rng(n)
  x = rng.standard_normal((n, 16))
  x /= np.linalg.norm(x, axis=1, keepdims=True)
  return ((x @ x.T + 1.0) / 2.0).astype(np.float32).astype(np.float64)


def inverse(n, alpha):
  a = propagation_affinity(n)
  dn = 1 / (np.sqrt(a.sum(axis=1)) + ct.EPS)
  return np.linalg.inv(np.eye(n) - alpha * (dn[:, None] * a * dn[None, :]))


def constraint_matrices(n):
  """Q of ConstraintMatrix from random speaker-turn scores, and a dense +-1 block Q."""
  rng = np.random.default_rng(n + 1)
  scores = rng.choice([0.0, 0.5, 2.0], n)
  turns = ct.ConstraintMatrix(list(scores), threshold=1).compute_diagonals()
  b, o = min(n, 32), (n - min(n, 32)) // 2
  blk = rng.choice([1.0, -1.0], (b, b))
  blk = np.triu(blk) + np.triu(blk, 1).T
  block = np.zeros((n, n))
  block[o:o + b, o:o + b] = blk
  return {"turns": turns, "block": block}


def propagation_tolerance(n, alpha, adj_ref, f_ref):
  cond = (1 + abs(alpha)) / (1 - abs(alpha))
  gamma = (40 + math.ceil(n / 128)) * U
  return 4 * U * max(1.0, np.abs(adj_ref).max()) + (4 * cond * U + 8 * gamma) * np.abs(f_ref).max()


def check_propagation(n, alpha, qname, q):
  a = propagation_affinity(n)
  got = ct.ConstraintPropagation(alpha).adjust_affinity(a, q)
  adj_ref, f_ref = restated_propagation(a, q, alpha, inverse(n, alpha))
  tol = propagation_tolerance(n, alpha, adj_ref, f_ref)
  err = np.abs(got - adj_ref).max()
  asym = np.abs(got - got.T).max()
  print("propagation n=%d alpha=%g q=%s max|F|=%.3g err=%.3g (%.3g of max|F|) asym=%.3g tol=%.3g"
        % (n, alpha, qname, np.abs(f_ref).max(), err, err / np.abs(f_ref).max(), asym, tol))
  assert err <= tol, "n=%d alpha=%g %s: error %g > %g" % (n, alpha, qname, err, tol)
  # predict() marks the propagated matrix symmetric and reads only its upper half downstream
  assert asym <= tol, "n=%d alpha=%g %s: asymmetry %g > %g" % (n, alpha, qname, asym, tol)


@pytest.mark.parametrize("alpha", [0.0, 0.1, 0.4, 0.6, 0.9, 0.99, -0.6])
@pytest.mark.parametrize("n", [3, 63, 64, 65, 300, 1000, 2500, 4096])
def test_propagation_matches_float64_inverse(n, alpha):
  for qname, q in constraint_matrices(n).items():
    check_propagation(n, alpha, qname, q)


@pytest.mark.parametrize("alpha", [0.995, 0.999, 0.9999, 1.0, 1.2, -1.5])
@pytest.mark.parametrize("n", [63, 1000])
def test_propagation_near_or_past_one_is_accurate_or_refused(n, alpha):
  """Either the same tolerance or NotImplementedError naming alpha; never a wrong matrix.  From
  X = I the iteration diverges for |alpha| >= 1, so those must be refused."""
  q = constraint_matrices(n)["turns"]
  name = re.escape(repr(float(alpha)))
  if abs(alpha) >= 1:
    with pytest.raises(NotImplementedError, match=name):
      ct.ConstraintPropagation(alpha).adjust_affinity(propagation_affinity(n), q)
    return
  try:
    check_propagation(n, alpha, "turns", q)
  except NotImplementedError as e:
    assert re.search(name, str(e))


# ------------------------------------------------------------------ AffinityIntegration
def turn_options(p=0.95):
  return scb.RefinementOptions(
      p_percentile=p, thresholding_soft_multiplier=0.01,
      thresholding_type=scb.ThresholdType.Percentile, thresholding_with_binarization=True,
      thresholding_preserve_diagonal=True, symmetrize_type=scb.SymmetrizeType.Average,
      refinement_sequence=list(scb.configs.TURNTODIARIZE_REFINEMENT_SEQUENCE))


def test_affinity_integration_with_nonsymmetric_q():
  n = 1000
  x = orc.synthetic_dvectors(n, 64, 4, seed=5)
  a = orc.affinity(x).astype(np.float32).astype(np.float64)
  rng = np.random.default_rng(6)
  q = rng.choice([-1.0, 0.0, 1.0], p=[0.01, 0.98, 0.01], size=(n, n))
  assert not np.array_equal(q, q.T)
  got = ct.AffinityIntegration(ct.IntegrationType.Max).adjust_affinity(a, q)
  np.testing.assert_array_equal(got, np.maximum(a, q))               # exact in fp32
  got = ct.AffinityIntegration(ct.IntegrationType.Average).adjust_affinity(a, q)
  ref = 0.5 * (a + q)                    # one rounding of a + q, halved exactly: 1/2 ulp
  assert np.all(np.abs(got - ref) <= 0.5 * ulp32(ref))
  c = scb.SpectralClusterer(
      min_clusters=2, max_clusters=7, refinement_options=turn_options(),
      constraint_options=scb.ConstraintOptions(
          constraint_name=scb.ConstraintName.AffinityIntegration, apply_before_refinement=False,
          integration_type=scb.IntegrationType.Max),
      laplacian_type=scb.LaplacianType.GraphCut, row_wise_renorm=True)
  labels = c.predict(x, q)
  assert c.last_details["solver"] == "krylov-schur"
  assert labels.shape == (n,)


# ------------------------------------------------------------------ predict() end to end
def turn_constraints(labels):
  """Speaker-turn scores from the true turns: 0 inside a turn (must-link), 2 > threshold at a
  change (cannot-link)."""
  scores = [0.0] + [0.0 if labels[i] == labels[i - 1] else 2.0 for i in range(1, len(labels))]
  return ct.ConstraintMatrix(scores, threshold=1).compute_diagonals()


def host_labels(w, v, k, opt):
  k = max(k, opt["min_clusters"])
  emb = v[:, :k]
  if opt["row_wise_renorm"]:
    emb = emb / np.linalg.norm(emb, axis=1, ord=2).reshape(-1, 1)
  return orc.run_kmeans(emb, k, opt["custom_dist"], opt["max_iter"])


def check_eigenvalues(got, want):
  """DESIGN.md section 3: |d| <= 1e-5 |lambda| + 1e-6 lambda_max."""
  m = min(len(got), len(want))
  scale = max(np.abs(want[:m]).max(), np.abs(got[:m]).max())
  err = np.abs(got[:m] - want[:m])
  assert np.all(err <= 1e-5 * np.abs(want[:m]) + 1e-6 * scale), err


@pytest.fixture(scope="module")
def speakers():
  x, lab = orc.synthetic_dvectors(2048, 128, 5, seed=3, return_labels=True)
  return x, turn_constraints(lab)


def test_turn_to_diarize_propagation_before_refinement(speakers):
  x, q = speakers
  opt = orc.options(min_clusters=2, max_clusters=7, sequence=("threshold", "symmetrize"),
                    p=0.95, mult=0.01, threshold_type="percentile", binarize=True,
                    preserve_diagonal=True, symmetrize_type="average", laplacian="graphcut",
                    row_wise_renorm=True)
  adj, _ = restated_propagation(orc.affinity(x), q, 0.4)             # spectral_clusterer.py:258-264
  w, v, k, _ = orc.eigenvectors_ncluster(adj, opt)
  want = host_labels(w, v, k, opt)
  c = scb.SpectralClusterer(
      min_clusters=2, max_clusters=7, refinement_options=turn_options(0.95),
      constraint_options=scb.ConstraintOptions(
          constraint_name=scb.ConstraintName.ConstraintPropagation, apply_before_refinement=True,
          constraint_propagation_alpha=0.4),
      laplacian_type=scb.LaplacianType.GraphCut, row_wise_renorm=True, custom_dist="cosine")
  got = c.predict(x, q)
  np.testing.assert_array_equal(orc.ordered(got), orc.ordered(want))
  check_eigenvalues(c.last_details["eigenvalues"], w[:8])


def test_icassp_with_integration_after_refinement(speakers):
  x, q = speakers
  opt = orc.options(min_clusters=2, max_clusters=7, sequence=orc.ICASSP2018)
  adj = np.maximum(orc.refine(orc.affinity(x), opt), q)             # spectral_clusterer.py:137-142
  w, v, k, _ = orc.eigenvectors_ncluster(adj, dict(opt, sequence=()))
  want = host_labels(w, v, k, opt)
  c = scb.SpectralClusterer(
      min_clusters=2, max_clusters=7, refinement_options=scb.configs.icassp2018_refinement_options,
      constraint_options=scb.ConstraintOptions(
          constraint_name=scb.ConstraintName.AffinityIntegration, apply_before_refinement=False,
          integration_type=scb.IntegrationType.Max),
      laplacian_type=None, custom_dist="cosine")
  got = c.predict(x, q)
  assert c.last_details["solver"] == "krylov-schur"
  np.testing.assert_array_equal(orc.ordered(got), orc.ordered(want))
  check_eigenvalues(c.last_details["eigenvalues"], w[:8])
