"""GPU: row normalisation, the affinity GEMM and the 128 x 128 split3 products, tile edge by tile edge.

The affinity (`TC_EPI_AFFINITY`) and the split3 Diffuse run on 128 x 128 wgmma tiles; the
single/split2 Diffuse tiles (128 x 192) are covered by test_gpu_gemm_tiles.py.  Every case calls the
C ABI directly, puts NaN in the padding columns of its inputs, prefills its outputs with NaN, checks
that every element in [0, n) was written and no padding was touched, and compares with an exact
float64 evaluation of what the kernel computes from the very fp16 planes it reads.

Error model of the tensor-core products.  The products of fp16 planes are exact and the reference
sums them exactly, so the only error is the fp32 accumulation.  Inside a register chain every wgmma
(k = 16) adds into the accumulator with truncation, by at most 1 ulp = 2^-23 of the partial sum.
A K block issues 8 cross-term wgmmas (hi lo, lo hi; split3 only) and then 4 hi hi wgmmas.  In the
first K block of a chain the cross terms go into an accumulator 2^-11 the size of the result, so
they cost nothing; every later wgmma of the chain adds at full size:
    full-size wgmmas per chain = 4 CHAIN_KB + 8 (CHAIN_KB - 1)   (split3; single: 4 CHAIN_KB)
At the end of a chain the chain is added, rounded to nearest (2^-24), into the tile sum.  With
T[i, j] = sum_k (|hi| + |lo|)_ik (|hi| + |lo|)_jk bounding every partial sum of element (i, j):
    |error| <= (2 x full-size wgmmas per chain + number of chains) 2^-24 T[i, j]
The affinity uses 1-K-block chains (`aff_chunk_kb`), so (8 + K blocks) 2^-24 T; it then halves
that with (x + 1) / 2 and adds one rounding of the fmaf.  For d <= 256 (T <= 1 + 2^-10) that is at
most 7 x 2^-24, below the 4 fp32 ulps (8 x 2^-24) that test_gpu_ops.py allows against the unsplit
float64 affinity.  Split3 Diffuse uses 2-K-block chains.
"""

import numpy as np
import pytest

from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
NAN = float("nan")
AFF_N = [64, 65, 127, 128, 129, 255, 257, 2047, 2049, 4097]
AFF_D = [3, 33, 64, 65, 256]
# 4,160 = 65 K blocks: at least 2 x 32 K blocks and more tiles than SMs, so producer pacing runs
AFF_SHAPES = [(n, d) for n in AFF_N for d in AFF_D] + [(2049, 4160)]
PRECISIONS = {"split3": nat.GEMM_SPLIT3, "single": nat.GEMM_SINGLE}
DIFFUSE_SIZES = [1, 63, 127, 128, 129, 191, 192, 193, 320, 383, 640, 1000, 2049, 4097]


def t():
  return dev.torch()


def nan_buf(rows, cols, device, dtype=None):
  return t().full((rows, cols), NAN, dtype=dtype or t().float32, device=device)


def pad_cols(k):
  return dev.round_up(k, 64) + 64


def assert_written(buf, cols, rows=None):
  rows = buf.shape[0] if rows is None else rows
  assert t().isfinite(buf[:rows, :cols].float()).all(), "an output element was not written"
  assert t().isnan(buf[:rows, cols:].float()).all(), "a padding column was written"


def embeddings(n, d, seed, device, dtype):
  """Seeded speaker-like embeddings (a few shared directions plus noise) in a NaN-padded buffer."""
  rng = np.random.default_rng(seed)
  cent = rng.standard_normal((4, d))
  x = cent[rng.integers(0, 4, n)] + 0.7 * rng.standard_normal((n, d))
  buf = t().full((n, pad_cols(d)), NAN, dtype=dtype, device=device)
  buf[:, :d] = t().from_numpy(x).to(device=device, dtype=dtype)
  return buf


def normalize(engine, x, n, d, want_xn=True, want_planes=True):
  is64 = 1 if x.dtype == t().float64 else 0
  xn = nan_buf(n, pad_cols(d), engine.device) if want_xn else None
  hi = nan_buf(n, pad_cols(d), engine.device, t().float16) if want_planes else None
  lo = nan_buf(n, pad_cols(d), engine.device, t().float16) if want_planes else None
  engine.call("sc_normalize_rows", dev._ptr(x), is64, n, d, x.stride(0), dev._ptr(xn),
              0 if xn is None else xn.stride(0), dev._ptr(hi), dev._ptr(lo),
              0 if hi is None else hi.stride(0), engine.stream)
  t().cuda.synchronize()
  return xn, hi, lo


def product_terms(a_hi, a_lo, b_hi, b_lo, k, precision):
  """Exact float64 sum of the products the kernel issues, and the bound T of its partial sums."""
  ah, bh = a_hi[:, :k].double(), b_hi[:, :k].double()
  want = ah @ bh.T
  if precision == nat.GEMM_SPLIT3:
    al, bl = a_lo[:, :k].double(), b_lo[:, :k].double()
    want += ah @ bl.T + al @ bh.T
    mag_a, mag_b = ah.abs() + al.abs(), bh.abs() + bl.abs()
  else:
    mag_a, mag_b = ah.abs(), bh.abs()
  return want, mag_a @ mag_b.T


def chain_bound(k, chain_kb, precision, mag):
  kb = (k + 63) // 64
  chains = (kb + chain_kb - 1) // chain_kb
  per_chain = min(chain_kb, kb)
  full_size = 4 * per_chain + (8 * (per_chain - 1) if precision == nat.GEMM_SPLIT3 else 0)
  return (2 * full_size + chains) * U32 * mag


# ---------------------------------------------------------------- sc_normalize_rows
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("n,d", [(1, 3), (65, 33), (257, 64), (1000, 256), (300, 4160)])
def test_normalize_rows(engine, dtype, n, d):
  x = embeddings(n, d, seed=d, device=engine.device, dtype=getattr(t(), dtype))
  zero = n // 2
  x[zero, :d] = 0.0
  xn, hi, lo = normalize(engine, x, n, d)
  ok = t().ones(n, dtype=t().bool, device=engine.device)
  ok[zero] = False
  for buf in (xn, hi, lo):
    assert t().isnan(buf[:, d:].float()).all(), "a padding column was written"
    assert t().isfinite(buf[ok, :d].float()).all()
    assert t().isnan(buf[zero, :d].float()).all(), "a zero row gives NaN like the reference"
  xd = x[:, :d].double()
  want = xd / xd.pow(2).sum(dim=1, keepdim=True).sqrt()
  got = xn[ok, :d]
  ulp = t().nextafter(got.abs(), t().full_like(got, float("inf"))) - got.abs()
  assert ((got.double() - want[ok]).abs() <= ulp.double()).all()
  assert t().equal(hi[ok, :d], got.half())
  assert t().equal(lo[ok, :d], (got - hi[ok, :d].float()).half())
  # a call for the planes alone writes the same planes
  _, hi2, lo2 = normalize(engine, x, n, d, want_xn=False)
  assert t().equal(hi2[ok, :d], hi[ok, :d]) and t().equal(lo2[ok, :d], lo[ok, :d])
  assert t().isnan(hi2[:, d:]).all() and t().isnan(lo2[:, d:]).all()


# ---------------------------------------------------------------- sc_affinity_cosine
def crop_of(a, n, diag_shift=0):
  """max(0, max_{j != i} a[i, j]) with row i's diagonal at column i + diag_shift."""
  rows = a.shape[0]
  v = a[:, :n].clone()
  r = t().arange(rows, device=a.device)
  v[r, r + diag_shift] = -float("inf")
  return v.max(dim=1).values.clamp_min(0.0)


def affinity_bound(k, precision, mag, a):
  # 1-K-block chains: (8 + K blocks) 2^-24 T on the product, halved by (x + 1) / 2, plus one
  # rounding of the fmaf.  Measured on an H100 80GB HBM3 (700 W limit): at most 0.93 of this bound
  # for the whole matrix (n = 4,097), 0.59 for the row blocks.
  return 0.5 * chain_bound(k, 1, precision, mag) + U32 * a.abs()


def affinity(engine, precision, hi, lo, n, d):
  a = nan_buf(n, pad_cols(n), engine.device)
  crop = t().full((n + 8,), NAN, dtype=t().float32, device=engine.device)
  crop[:n] = 0.0                                              # zero-filled by the caller
  engine.call("sc_affinity_cosine", nat.GEMM_TCGEN05, precision, None, 0, dev._ptr(hi),
              dev._ptr(lo), hi.stride(0), n, d, dev._ptr(a), a.stride(0), dev._ptr(crop),
              engine.stream)
  t().cuda.synchronize()
  assert t().isnan(crop[n:]).all()
  assert_written(a, n)
  return a[:, :n], crop[:n]


@pytest.mark.parametrize("precision", sorted(PRECISIONS))
@pytest.mark.parametrize("n,d", AFF_SHAPES)
def test_affinity_tiles(engine, n, d, precision):
  prec = PRECISIONS[precision]
  x = embeddings(n, d, seed=n + d, device=engine.device, dtype=t().float32)
  _, hi, lo = normalize(engine, x, n, d, want_xn=False)
  a, crop = affinity(engine, prec, hi, lo, n, d)
  prod, mag = product_terms(hi, lo, hi, lo, d, prec)
  want = (prod + 1.0) / 2.0
  err = (a.double() - want).abs()
  bound = affinity_bound(d, prec, mag, want)
  assert (err <= bound).all(), ((err / bound).max().item(), err.max().item())
  # the product of one plane set with itself is symmetric: tiles off the 128-tile diagonal are
  # mirrored (bitwise), the square diagonal tiles store both orientations from their own sums
  tile = t().arange(n, device=engine.device) // 128
  off = tile[:, None] != tile[None, :]
  assert t().equal(a[off], a.T[off])
  assert ((a - a.T).abs().double() <= bound + bound.T).all()
  assert t().equal(crop, crop_of(a, n))


@pytest.mark.parametrize("n", [1, 2, 63])
def test_affinity_simt(engine, n):
  d = 33
  x = embeddings(n, d, seed=n, device=engine.device, dtype=t().float64)
  xn, _, _ = normalize(engine, x, n, d, want_planes=False)
  a = nan_buf(n, pad_cols(n), engine.device)
  crop = t().full((n + 8,), NAN, dtype=t().float32, device=engine.device)
  crop[:n] = 0.0
  engine.call("sc_affinity_cosine", nat.GEMM_SIMT, nat.GEMM_SPLIT3, dev._ptr(xn), xn.stride(0),
              None, None, 0, n, d, dev._ptr(a), a.stride(0), dev._ptr(crop), engine.stream)
  t().cuda.synchronize()
  assert_written(a, n)
  assert t().isnan(crop[n:]).all()
  a = a[:, :n]
  xd = xn[:, :d].double()
  want = (xd @ xd.T + 1.0) / 2.0
  # fp64 accumulation of exact fp32 x fp32 products, one rounding to fp32: within 1 ulp
  ulp = t().nextafter(a.abs(), t().full_like(a, float("inf"))) - a.abs()
  assert ((a.double() - want).abs() <= ulp.double()).all()
  assert t().equal(crop[:n], crop_of(a, n))
  if n == 1:
    assert crop[0].item() == 0.0


@pytest.mark.parametrize("n", [2049, 4097])
@pytest.mark.parametrize("d", [65, 256])
def test_affinity_row_blocks(engine, n, d):
  x = embeddings(n, d, seed=7, device=engine.device, dtype=t().float32)
  _, hi, lo = normalize(engine, x, n, d, want_xn=False)
  prod, mag = product_terms(hi, lo, hi, lo, d, nat.GEMM_SPLIT3)
  want = (prod + 1.0) / 2.0
  for rb, rc in ((0, 300), (300, 1000), (n - 77, 77), (0, n)):
    blk = nan_buf(rc, pad_cols(n), engine.device)
    crop = t().full((rc + 8,), NAN, dtype=t().float32, device=engine.device)
    crop[:rc] = 0.0
    engine.call("sc_affinity_cosine_block", nat.GEMM_SPLIT3, dev._ptr(hi), dev._ptr(lo),
                hi.stride(0), n, d, rb, rc, dev._ptr(blk), blk.stride(0), dev._ptr(crop),
                engine.stream)
    t().cuda.synchronize()
    assert_written(blk, n)
    assert t().isnan(crop[rc:]).all()
    got = blk[:, :n]
    w = want[rb:rb + rc]
    err = (got.double() - w).abs()
    bound = affinity_bound(d, nat.GEMM_SPLIT3, mag[rb:rb + rc], w)
    assert (err <= bound).all(), ((err / bound).max().item(), err.max().item())
    assert t().equal(crop[:rc], crop_of(got, n, diag_shift=rb))


# ---------------------------------------------------------------- split3 Diffuse (128 x 128 tiles)
def split_planes(rows, k, seed, device):
  """Seeded Y in [0, 1) as fp16 planes with NaN padding columns."""
  g = t().Generator(device=device).manual_seed(seed)
  y = t().rand((rows, k), generator=g, device=device, dtype=t().float32)
  hi = nan_buf(rows, pad_cols(k), device, t().float16)
  lo = nan_buf(rows, pad_cols(k), device, t().float16)
  hi[:, :k] = y.half()
  lo[:, :k] = (y - hi[:, :k].float()).half()
  return hi, lo


def diffuse_bound(k, mag):
  # 2-K-block chains (split3 Diffuse).  Measured on an H100 80GB HBM3 (700 W limit): at most 0.64
  # of this bound for the symmetric product (n = 63), 0.47 for the general one.
  return chain_bound(k, 2, nat.GEMM_SPLIT3, mag)


@pytest.mark.parametrize("n", DIFFUSE_SIZES)
def test_symmetric_split3_diffuse(engine, n):
  hi, lo = split_planes(n, n, seed=n, device=engine.device)
  s = nan_buf(n, pad_cols(n), engine.device)
  mx = t().full((n + 8,), NAN, dtype=t().float32, device=engine.device)
  sm = t().full((n + 8,), NAN, dtype=t().float64, device=engine.device)
  engine.call("sc_diffuse", nat.GEMM_TCGEN05, nat.GEMM_SPLIT3, None, 0, dev._ptr(hi),
              dev._ptr(lo), hi.stride(0), n, dev._ptr(s), s.stride(0), dev._ptr(mx), dev._ptr(sm),
              engine.stream)
  t().cuda.synchronize()
  assert_written(s, n)
  assert t().isnan(mx[n:]).all() and t().isnan(sm[n:]).all()
  s = s[:, :n]
  assert t().equal(s, s.T)
  want, mag = product_terms(hi, lo, hi, lo, n, nat.GEMM_SPLIT3)
  err = (s.double() - want).abs()
  bound = diffuse_bound(n, mag)
  assert (err <= bound).all(), ((err / bound).max().item(), err.max().item())
  assert t().equal(mx[:n], s.max(dim=1).values)
  t().testing.assert_close(sm[:n], s.double().sum(dim=1), rtol=1e-6, atol=0)


@pytest.mark.parametrize("m,n,k", [(300, 457, 1000), (1000, 193, 2049), (129, 4097, 383)])
def test_split3_general_product_with_mirror(engine, m, n, k):
  a_hi, a_lo = split_planes(m, k, seed=1, device=engine.device)
  b_hi, b_lo = split_planes(n, k, seed=2, device=engine.device)
  c = nan_buf(m, pad_cols(n), engine.device)
  mirror = nan_buf(n, pad_cols(m), engine.device)
  engine.call("sc_gemm_nt_planes", nat.GEMM_SPLIT3, dev._ptr(a_hi), dev._ptr(a_lo),
              a_hi.stride(0), m, dev._ptr(b_hi), dev._ptr(b_lo), b_hi.stride(0), n, k,
              dev._ptr(c), c.stride(0), dev._ptr(mirror), mirror.stride(0), engine.stream)
  t().cuda.synchronize()
  assert_written(c, n)
  assert_written(mirror, m)
  c, mirror = c[:, :n], mirror[:, :m]
  assert t().equal(mirror, c.T)
  want, mag = product_terms(a_hi, a_lo, b_hi, b_lo, k, nat.GEMM_SPLIT3)
  err = (c.double() - want).abs()
  bound = diffuse_bound(k, mag)
  assert (err <= bound).all(), ((err / bound).max().item(), err.max().item())
