"""GPU: the blur family and the fused threshold/symmetrize passes, kernel by kernel, at their tile edges.

Every case calls the C ABI directly.  Inputs carry NaN in their padding columns (and NaN guard rows
around the row blocks), outputs are prefilled with NaN, and each case checks that every element in
[0, n) was written and is finite and that no padding was touched.  The blur is compared with
scipy's float64 correlate1d run with the kernel's own fp32 weights, so the only error left is the
kernel's fp32 rounding; everything downstream of the blur (row maxima, the threshold rule, the fp16
planes, the row-block entries, the upper-triangle pass) is compared bit for bit with the stored blur
or with the whole-matrix kernels.
"""

import math

import numpy as np
import pytest
import scipy.ndimage

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from oracle import spectral_oracle as orc

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24                      # unit roundoff of fp32
NAN = float("nan")
# n <= 2R + 1 reflects repeatedly; 260 is the first n with a fast (interior) tile of the radius-4
# kernel; 511 / 513 straddle the 4-tile column run of one CTA
SIZES = [1, 2, 3, 5, 8, 9, 31, 33, 127, 128, 129, 259, 260, 261, 511, 513, 1000, 2049, 4099]
# radius 4 (band kernel and upper pass) at sigma 1, 0.875 and 1.1249; radius 3 (generic) at 0.874;
# radius 0 (k_noblur) at 0.1; a copy at 1e-16; radius 8, 13 and 64 at 2, 3.3 and 16
SIGMAS = [1.0, 0.875, 1.1249, 0.874, 0.1, 1e-16, 2.0, 3.3, 16.0]
RADIUS4 = [1.0, 0.875, 1.1249]
# the float64 reference costs O(n^2 R) on the host: the two largest sizes take the three kernels
BLUR_CASES = [(n, s) for n in SIZES for s in SIGMAS if n < 2049 or s in (1.0, 0.874, 2.0)]
P, MULT = 0.95, 0.01                  # the ICASSP 2018 RowWiseThreshold


def ld_of(n):
  """Leading dimension with a whole 64-column block of (NaN) padding past the rounded-up width."""
  return dev.round_up(n, 64) + 64


def t():
  return dev.torch()


def nan_buf(rows, cols, device, dtype=None):
  return t().full((rows, cols), NAN, dtype=dtype or t().float32, device=device)


def nan_vector(n, device, zero=True):
  """n entries (zero-filled: the atomic maxima start from 0) and a NaN tail that must stay NaN."""
  v = t().full((n + 8,), NAN, dtype=t().float32, device=device)
  if zero:
    v[:n] = 0.0
  return v


def padded(a, device):
  """Host [n, n] -> device fp32 [n, ld_of(n)] with NaN padding columns."""
  n = a.shape[0]
  buf = nan_buf(n, ld_of(n), device)
  buf[:, :n] = t().from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)
  return buf


def assert_written(buf, n, rows=None):
  """[0, rows) x [0, n) finite, padding columns NaN."""
  rows = n if rows is None else rows
  assert t().isfinite(buf[:rows, :n].float()).all(), "an output element was not written"
  assert t().isnan(buf[:rows, n:].float()).all(), "a padding column was written"


def strong_diagonal(n, seed):
  """Non-symmetric, non-negative, with the largest entry of each row on the diagonal (so that the
  zero_diagonal statistics differ from the plain ones)."""
  rng = np.random.default_rng(seed)
  a = 0.5 * rng.random((n, n))
  np.fill_diagonal(a, 1.0)
  return a.astype(np.float32)


def structured_affinity(n, seed=0, d=32):
  """Symmetric affinity of seeded embeddings in four segments: speaker 0 clean, speaker 1 clean,
  speaker 1 noisy, speaker 0 noisy.  A noisy row is closer to the clean segment of its speaker than
  to its own neighbours, so the maximum of its blurred row lies far left of the diagonal, where
  the upper pass only sees it as a column maximum of an interior tile."""
  rng = np.random.default_rng(seed)
  cent = rng.standard_normal((2, d))
  cent /= np.linalg.norm(cent, axis=1, keepdims=True)
  seg = np.minimum(np.arange(n) * 4 // max(n, 1), 3)
  spk = np.array([0, 1, 1, 0])[seg]
  noise = np.where(seg < 2, math.sqrt((1 / 0.95 - 1) / d), math.sqrt((1 / 0.2 - 1) / d))
  x = cent[spk] + noise[:, None] * rng.standard_normal((n, d))
  return orc.affinity(x).astype(np.float32)


def blur_weights(sigma):
  """The kernel's weights: scipy's _gaussian_kernel1d in float64 (summed in index order, glibc
  exp like the host code), normalised, rounded to fp32."""
  r = int(4.0 * sigma + 0.5)
  w = [math.exp(-0.5 / (sigma * sigma) * float(k) * float(k)) for k in range(-r, r + 1)]
  s = 0.0
  for v in w:
    s += v
  return np.array([v / s for v in w], dtype=np.float32), r


def blur_ref(a, sigma):
  """float64 scipy correlate1d, axis 0 then axis 1, mode reflect, with the kernel's fp32 weights."""
  a = np.asarray(a, dtype=np.float64)
  if sigma <= 1e-15:
    return a.copy(), 0
  w, r = blur_weights(sigma)
  w = w.astype(np.float64)
  out = scipy.ndimage.correlate1d(a, w, axis=0, mode="reflect")
  return scipy.ndimage.correlate1d(out, w, axis=1, mode="reflect"), r


def blur_bound(r, scale):
  """Each output is two chains of 2R+1 fp32 FMAs (axis 0, then axis 1).  Every FMA rounds once,
  by at most u = 2^-24 of its partial sum, and a partial sum of non-negative weights (sum 1) times
  values of magnitude <= scale is <= scale: the first pass is off by <= (2R+1) u scale, which the
  second pass carries with weight 1 and adds its own (2R+1) u scale to.  Radius 0 is exact."""
  return 2 * (2 * r + 1) * U32 * scale * (1 + 1e-6)


def blur(engine, ab, n, sigma, diag=None):
  out = nan_buf(n + 1, ab.shape[1], engine.device)          # the last row is a guard
  engine.call("sc_gaussian_blur", dev._ptr(ab), n, ab.stride(0), dev._ptr(diag), float(sigma),
              dev._ptr(out), out.stride(0), None, engine.stream)
  t().cuda.synchronize()
  assert_written(out, n)
  assert t().isnan(out[n]).all()
  return out[:n]


def blur_rowmax(engine, ab, n, sigma, zero_diag, diag=None):
  m = nan_vector(n, engine.device)
  engine.call("sc_gaussian_blur_rowmax", dev._ptr(ab), n, ab.stride(0), dev._ptr(diag),
              float(sigma), int(zero_diag), dev._ptr(m), engine.stream)
  t().cuda.synchronize()
  assert t().isnan(m[n:]).all()
  return m[:n]


def same_bits(x, y):
  """Bit-for-bit equality of two buffers, NaN padding included."""
  ints = {2: t().int16, 4: t().int32}
  return x.shape == y.shape and t().equal(x.view(ints[x.element_size()]),
                                          y.view(ints[y.element_size()]))


def row_max(b, n, zero_diag):
  """max_j b[i, j] of a stored [n, n] blur (all >= 0), with the diagonal read as 0 if asked."""
  b = b[:, :n].clone()
  if zero_diag:
    b.fill_diagonal_(0.0)
  return b.clamp_min(0.0).max(dim=1).values


# ---------------------------------------------------------------- sc_gaussian_blur (EPI_STORE)
@pytest.mark.parametrize("n,sigma", BLUR_CASES)
def test_gaussian_blur(engine, n, sigma):
  a = strong_diagonal(n, seed=n)
  ab = padded(a, engine.device)
  out = nan_buf(n + 1, ab.shape[1], engine.device)
  rm = nan_vector(n, engine.device)
  engine.call("sc_gaussian_blur", dev._ptr(ab), n, ab.stride(0), None, float(sigma),
              dev._ptr(out), out.stride(0), dev._ptr(rm), engine.stream)
  t().cuda.synchronize()
  assert_written(out, n)
  assert t().isnan(out[n]).all() and t().isnan(rm[n:]).all()
  b = out[:n, :n]
  want, r = blur_ref(a, sigma)
  err = np.abs(b.double().cpu().numpy() - want).max()
  if r == 0:
    assert err == 0.0
  else:
    # measured on an H100 80GB HBM3 (700 W limit): at most 0.17 of the bound (n = 3, sigma = 0.874)
    assert err <= blur_bound(r, float(np.abs(a).max())), (err, blur_bound(r, 1.0))
  # the fused row maximum of the store epilogue and of the statistics-only pass describe the
  # stored output exactly: the epilogues share one FMA order
  assert t().equal(rm[:n], row_max(b, n, False))
  for zero_diag in (0, 1):
    assert t().equal(blur_rowmax(engine, ab, n, sigma, zero_diag), row_max(b, n, zero_diag))


def test_gaussian_blur_radius_over_64_is_rejected(engine):
  n = 300
  ab = padded(strong_diagonal(n, seed=1), engine.device)
  out = nan_buf(n, ab.shape[1], engine.device)
  launches = nat.load().sc_launch_count()
  with pytest.raises(nat.NativeError, match="radius"):
    engine.call("sc_gaussian_blur", dev._ptr(ab), n, ab.stride(0), None, 16.2, dev._ptr(out),
                out.stride(0), None, engine.stream)
  t().cuda.synchronize()
  assert nat.load().sc_launch_count() == launches
  assert t().isnan(out).all()


@pytest.mark.parametrize("sigma", [1.0, 0.874, 2.0])
@pytest.mark.parametrize("n", SIZES)
def test_diag_override_equals_cropped_matrix(engine, n, sigma):
  """blur(A with diag <- crop vector on read) == blur(CropDiagonal(A)), bit for bit: at n >= 1,000
  the radius-4 kernel patches the diagonal of interior tiles in shared memory, at small n the
  override meets the reflected edges."""
  a = structured_affinity(n, seed=3)
  ab = padded(a, engine.device)
  crop = nan_vector(n, engine.device, zero=False)
  engine.call("sc_crop_diagonal_values", dev._ptr(ab), n, ab.stride(0), dev._ptr(crop),
              engine.stream)
  cropped = nan_buf(n, ab.shape[1], engine.device)
  engine.call("sc_crop_diagonal", dev._ptr(ab), n, ab.stride(0), dev._ptr(cropped),
              cropped.stride(0), engine.stream)
  t().cuda.synchronize()
  assert t().isnan(crop[n:]).all()
  assert_written(cropped, n)
  assert t().equal(t().diagonal(cropped[:, :n]), crop[:n])
  assert same_bits(blur(engine, ab, n, sigma, diag=crop), blur(engine, cropped, n, sigma))
  for zero_diag in (0, 1):
    assert t().equal(blur_rowmax(engine, ab, n, sigma, zero_diag, diag=crop),
                     blur_rowmax(engine, cropped, n, sigma, zero_diag))


# ---------------------------------------------------------------- the symmetric upper pass
def upper_stored_mask(n, device):
  """The tiles sc_blur_upper_rowmax stores: row i from column 128 floor(32 floor(i/32) / 128)."""
  i = t().arange(n, device=device)
  first = (i // 32 * 32) // 128 * 128
  return t().arange(n, device=device)[None, :] >= first[:, None]


def blur_upper(engine, ab, n, sigma, zero_diag, diag=None):
  b = nan_buf(n, ab.shape[1], engine.device)
  m = nan_vector(n, engine.device, zero=False)        # the entry zero-fills m itself
  engine.call("sc_blur_upper_rowmax", dev._ptr(ab), n, ab.stride(0), dev._ptr(diag), float(sigma),
              int(zero_diag), dev._ptr(b), b.stride(0), dev._ptr(m), engine.stream)
  t().cuda.synchronize()
  assert t().isnan(m[n:]).all()
  return b, m[:n]


@pytest.mark.parametrize("sigma", RADIUS4)
@pytest.mark.parametrize("n", SIZES)
def test_blur_upper_rowmax(engine, n, sigma):
  a = structured_affinity(n, seed=n)
  ab = padded(a, engine.device)
  crop = engine.crop_values(ab, n)
  stored = upper_stored_mask(n, engine.device)
  for diag in (None, crop):
    full = blur(engine, ab, n, sigma, diag=diag)[:, :n]
    for zero_diag in (0, 1):
      b, m = blur_upper(engine, ab, n, sigma, zero_diag, diag=diag)
      assert t().isnan(b[:, n:]).all()
      bb = b[:, :n]
      assert t().equal(bb[stored], full[stored])
      assert t().isnan(bb[~stored]).all(), "the upper pass wrote left of its tiles"
      # m[i] = max over the stored b[i, .] and b[., i]
      z = t().where(stored, bb, t().zeros_like(bb))
      if zero_diag:
        z.fill_diagonal_(0.0)
      assert t().equal(m, t().maximum(z.max(dim=1).values, z.max(dim=0).values))


# ---------------------------------------------------------------- the threshold rule
def threshold_rule(b, m_row, m_col, binarize, keep_diag, sym_type):
  """The fused rule in fp32, operation by operation as the kernels do it: t = b * mult if
  b < m * p (m * p rounded to fp32) else (1 if binarize else b); y = fmax(t1, t2) or
  0.5 (t1 + t2); y[i, i] = 1 if the diagonal is preserved."""
  f32 = lambda v: t().tensor(v, dtype=t().float32, device=b.device)
  p, mult = f32(P), f32(MULT)
  small = b * mult
  keep = t().ones_like(b) if binarize else b
  t1 = t().where(b < (m_row * p)[:, None], small, keep)
  t2 = t().where(b < (m_col * p)[None, :], small, keep)
  y = t().maximum(t1, t2) if sym_type == nat.SYMMETRIZE_MAX else f32(0.5) * (t1 + t2)
  if keep_diag:
    y.fill_diagonal_(1.0)
  return y


def assert_planes(hi, lo, y, n):
  """hi == fp16(y) and lo == fp16(y - hi), bit for bit."""
  assert_written(hi, n)
  assert t().equal(hi[:, :n], y.half())
  if lo is not None:
    assert_written(lo, n)
    assert t().equal(lo[:, :n], (y - hi[:, :n].float()).half())


RULES = [(bz, st) for bz in (0, 1) for st in (nat.SYMMETRIZE_MAX, nat.SYMMETRIZE_AVERAGE)]


def run_upper(engine, b, m, n, binarize, keep_diag, sym_type, want_y, want_hi, want_lo):
  ld = b.shape[1]
  y = nan_buf(n, ld, engine.device) if want_y else None
  hi = nan_buf(n, ld, engine.device, t().float16) if want_hi else None
  lo = nan_buf(n, ld, engine.device, t().float16)     # stays NaN when not passed
  engine.call("sc_threshold_symmetrize_upper", dev._ptr(b), n, b.stride(0), dev._ptr(m), P, MULT,
              binarize, keep_diag, sym_type, dev._ptr(y), 0 if y is None else y.stride(0),
              dev._ptr(hi), dev._ptr(lo if want_lo else None), 0 if hi is None else hi.stride(0),
              engine.stream)
  t().cuda.synchronize()
  return y, hi, lo


@pytest.mark.parametrize("n", SIZES)
def test_threshold_symmetrize_upper(engine, n):
  """Y(i, j) = Y(j, i) = rule(b[min(i, j), max(i, j)], m_i, m_j) from the stored upper tiles."""
  a = structured_affinity(n, seed=n + 1)
  ab = padded(a, engine.device)
  crop = engine.crop_values(ab, n)
  for keep_diag in (0, 1):
    b, m = blur_upper(engine, ab, n, 1.0, keep_diag, diag=crop)
    upper = t().triu(b[:, :n])
    bsym = upper + t().triu(b[:, :n], diagonal=1).T
    for binarize, sym_type in RULES:
      want = threshold_rule(bsym, m, m, binarize, keep_diag, sym_type)
      y, hi, lo = run_upper(engine, b, m, n, binarize, keep_diag, sym_type, True, True, True)
      assert_written(y, n)
      yy = y[:, :n]
      assert t().equal(yy, want), "%d elements differ" % (yy != want).sum().item()
      assert t().equal(yy, yy.T)
      assert_planes(hi, lo, want, n)
      _, hi2, lo2 = run_upper(engine, b, m, n, binarize, keep_diag, sym_type, False, True, True)
      assert same_bits(hi2, hi) and same_bits(lo2, lo)
      # hi plane only (a single-MMA Diffuse): the lo buffer is not touched
      _, hi3, lo3 = run_upper(engine, b, m, n, binarize, keep_diag, sym_type, False, True, False)
      assert same_bits(hi3, hi)
      assert t().isnan(lo3).all()


def run_two_pass(engine, ab, n, sigma, diag, m, binarize, keep_diag, sym_type, want_y, want_planes):
  ld = ab.shape[1]
  y = nan_buf(n, ld, engine.device) if want_y else None
  hi = nan_buf(n, ld, engine.device, t().float16) if want_planes else None
  lo = nan_buf(n, ld, engine.device, t().float16) if want_planes else None
  engine.call("sc_blur_threshold_symmetrize", dev._ptr(ab), n, ab.stride(0), dev._ptr(diag),
              float(sigma), dev._ptr(m), P, MULT, binarize, keep_diag, sym_type, dev._ptr(y),
              0 if y is None else y.stride(0), dev._ptr(hi), dev._ptr(lo),
              0 if hi is None else hi.stride(0), engine.stream)
  t().cuda.synchronize()
  return y, hi, lo


@pytest.mark.parametrize("sigma", [1.0, 2.0, 0.0])
@pytest.mark.parametrize("n", SIZES)
def test_blur_threshold_symmetrize(engine, n, sigma):
  """The two-pass fused kernel: Y(i, j) = rule(blur[i, j], m_i, m_j) of the stored
  sc_gaussian_blur output, with m from sc_gaussian_blur_rowmax."""
  a = structured_affinity(n, seed=n + 2)
  ab = padded(a, engine.device)
  crop = engine.crop_values(ab, n)
  bfull = blur(engine, ab, n, sigma, diag=crop)[:, :n]
  for keep_diag in (0, 1):
    m = blur_rowmax(engine, ab, n, sigma, keep_diag, diag=crop)
    m16 = t().full((n + 8,), NAN, dtype=t().float32, device=engine.device)
    m16[:n] = m           # a 16-byte aligned copy with a NaN tail the kernel must not read
    for binarize, sym_type in RULES:
      want = threshold_rule(bfull, m, m, binarize, keep_diag, sym_type)
      y, hi, lo = run_two_pass(engine, ab, n, sigma, crop, m16, binarize, keep_diag, sym_type,
                               True, True)
      assert_written(y, n)
      assert t().equal(y[:, :n], want), "%d elements differ" % (y[:, :n] != want).sum().item()
      assert_planes(hi, lo, want, n)
      _, hi2, lo2 = run_two_pass(engine, ab, n, sigma, crop, m16, binarize, keep_diag, sym_type,
                                 False, True)
      assert same_bits(hi2, hi) and same_bits(lo2, lo)


# ---------------------------------------------------------------- row-block entries
def halo_block(a_dev, n, rb, re, r, guard=8):
  """Rows [rb - R, re + R) & [0, n) of the padded matrix in a buffer with NaN guard rows."""
  lo, hi = max(rb - r, 0), min(re + r, n)
  buf = t().full((hi - lo + 2 * guard, a_dev.shape[1]), NAN, dtype=t().float32,
                 device=a_dev.device)
  buf[guard:guard + hi - lo] = a_dev[lo:hi]
  return buf[guard:], lo, hi - lo


@pytest.mark.parametrize("sigma", [1.0, 2.0])
@pytest.mark.parametrize("n", [129, 1000, 2049])
def test_row_block_entries(engine, n, sigma):
  """Row blocks with exactly their blur halo resident give the whole-matrix results bit for bit."""
  a = structured_affinity(n, seed=5)
  ab = padded(a, engine.device)
  crop = engine.crop_values(ab, n)
  r = int(4.0 * sigma + 0.5)
  ld = ab.shape[1]
  m_whole = blur_rowmax(engine, ab, n, sigma, 1, diag=crop)
  m16 = t().zeros((n + 8,), dtype=t().float32, device=engine.device)
  m16[:n] = m_whole
  y_whole, hi_whole, lo_whole = run_two_pass(engine, ab, n, sigma, crop, m16, 0, 1,
                                             nat.SYMMETRIZE_MAX, True, True)
  for rb, re in ((0, 32), (32, 96), (96, n), (0, n)):
    blk, in_base, in_rows = halo_block(ab, n, rb, re, r)
    m = t().full((n + 8,), NAN, dtype=t().float32, device=engine.device)
    m[rb:re] = 0.0
    engine.call("sc_gaussian_blur_rowmax_block", dev._ptr(blk), n, ld, in_base, in_rows, rb, re,
                dev._ptr(crop), float(sigma), 1, dev._ptr(m), engine.stream)
    y = nan_buf(re - rb, ld, engine.device)
    hi = nan_buf(re - rb, ld, engine.device, t().float16)
    lo = nan_buf(re - rb, ld, engine.device, t().float16)
    engine.call("sc_blur_threshold_symmetrize_block", dev._ptr(blk), n, ld, in_base, in_rows, rb,
                re, dev._ptr(crop), float(sigma), dev._ptr(m16), P, MULT, 0, 1,
                nat.SYMMETRIZE_MAX, dev._ptr(y), y.stride(0), dev._ptr(hi), dev._ptr(lo),
                hi.stride(0), engine.stream)
    t().cuda.synchronize()
    assert t().equal(m[rb:re], m_whole[rb:re])
    assert t().isnan(m[:rb]).all() and t().isnan(m[re:]).all()
    assert_written(y, n)
    assert same_bits(y, y_whole[rb:re])
    assert same_bits(hi, hi_whole[rb:re]) and same_bits(lo, lo_whole[rb:re])
  # a block that does not end the matrix must span whole 32-row bands
  blk, in_base, in_rows = halo_block(ab, n, 32, 80, r)
  m = t().zeros((n + 8,), dtype=t().float32, device=engine.device)
  with pytest.raises(nat.NativeError, match="multiple of 32"):
    engine.call("sc_gaussian_blur_rowmax_block", dev._ptr(blk), n, ld, in_base, in_rows, 32, 80,
                dev._ptr(crop), float(sigma), 1, dev._ptr(m), engine.stream)
  with pytest.raises(nat.NativeError, match="multiple of 32"):
    engine.call("sc_blur_threshold_symmetrize_block", dev._ptr(blk), n, ld, in_base, in_rows, 32,
                80, dev._ptr(crop), float(sigma), dev._ptr(m16), P, MULT, 0, 1,
                nat.SYMMETRIZE_MAX, dev._ptr(y), y.stride(0), None, None, 0, engine.stream)


# ---------------------------------------------------------------- symmetry of the fused chain
def icassp_chain(sigma, diffuse=False):
  RN = scb.RefinementName
  return scb.RefinementOptions(
      gaussian_blur_sigma=sigma, p_percentile=P, thresholding_soft_multiplier=MULT,
      thresholding_type=scb.ThresholdType.RowMax,
      refinement_sequence=[RN.CropDiagonal, RN.GaussianBlur, RN.RowWiseThreshold, RN.Symmetrize] +
      ([RN.Diffuse] if diffuse else []))


def dvector_affinity(engine, n):
  x = orc.synthetic_dvectors(n, 64, 4, seed=n)
  a, _ = engine.affinity(t().from_numpy(x).to(engine.device), want_crop_vector=False)
  return a


@pytest.mark.parametrize("n", [700, 2049, 4099])
def test_fused_chain_output_is_symmetric(engine, n):
  """The upper pass (sigma 1) evaluates each pair (i, j), (j, i) from one stored blur value, so Y
  and the planes handed to Diffuse are exactly symmetric, as numpy's maximum(a, a.T) is."""
  a = dvector_affinity(engine, n)
  refined = dev.run_refinement(engine, a, n, icassp_chain(1.0))
  y = refined.s[:, :n]
  assert t().equal(y, y.T), "%d elements differ" % (y != y.T).sum().item()
  # with Diffuse after it the chain emits planes: hi + lo (two and three MMAs) or hi alone (one)
  crop = engine.crop_values(a, n)
  b, m = engine.blur_upper_rowmax(a, n, 1.0, crop, False)
  for want_lo in (True, False):
    _, hi, lo = engine.threshold_symmetrize_upper(b, n, m, P, MULT, False, False,
                                                  nat.SYMMETRIZE_MAX, False, True, want_lo)
    t().cuda.synchronize()
    assert t().equal(hi[:, :n], hi[:, :n].T)
    assert t().equal(hi[:, :n].float(), y.half().float())
    if want_lo:
      assert t().equal(lo[:, :n], lo[:, :n].T)
  s = dev.run_refinement(engine, a, n, icassp_chain(1.0, diffuse=True)).s[:, :n]
  assert t().isfinite(s).all() and t().equal(s, s.T)


@pytest.mark.parametrize("n", [700, 2049])
def test_two_pass_chain_symmetry(engine, n):
  """The two-pass kernels (radius != 4) blur (i, j) and (j, i) separately: Y is symmetric to the
  blur tolerance wherever both orientations take the same threshold decisions.  Pairs whose two
  blur values straddle a cut are counted and reported; their blur values agree to the tolerance."""
  sigma = 2.0
  a = dvector_affinity(engine, n)
  y = dev.run_refinement(engine, a, n, icassp_chain(sigma)).s[:, :n]
  crop = engine.crop_values(a, n)
  b = blur(engine, a, n, sigma, diag=crop)[:, :n]
  m = blur_rowmax(engine, a, n, sigma, 0, diag=crop)
  tol = 2 * blur_bound(int(4 * sigma + 0.5), 1.0)     # both orientations within the bound
  assert (b - b.T).abs().max().item() <= tol
  cut = m * t().tensor(P, dtype=t().float32, device=b.device)
  d_row, d_col = b < cut[:, None], b < cut[None, :]
  differs = (d_row != d_col.T) | (d_col != d_row.T)
  same = ~differs
  assert ((y - y.T).abs()[same].max().item() if same.any() else 0.0) <= tol
  pairs = int(t().triu(differs, diagonal=1).sum().item())
  print("two-pass chain, n = %d, sigma = %g: %d of %d pairs take different threshold decisions"
        % (n, sigma, pairs, n * (n - 1) // 2))
