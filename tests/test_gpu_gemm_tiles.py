"""GPU: the wgmma GEMM's tile enumeration and epilogue at every shape class of its two tile widths.

The one- and two-MMA Diffuse products run on 128 x 192 tiles, so the symmetric enumeration has
tiles that straddle the diagonal, a ragged last column block and several tile groups.  Each case
checks that every element of S is written (NaN prefill), that S is bitwise symmetric, that S agrees
with an exact float64 product of the very fp16 planes the kernel reads, and that the fused row
statistics describe the stored S.  The general (non-symmetric) product with a mirrored copy is
checked the same way on ragged M != N."""

import pytest

from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev

pytestmark = pytest.mark.gpu

SIZES = [1, 63, 127, 128, 129, 191, 192, 193, 320, 383, 640, 1000, 2049, 4097]
PRECISIONS = {"single": nat.GEMM_SINGLE, "split2": nat.GEMM_SPLIT2}


def split_planes(rows, k, seed, device):
  """Seeded Y in [0, 1) as fp16 planes hi = fp16(y), lo = fp16(y - hi), rows padded to 64."""
  t = dev.torch()
  g = t.Generator(device=device).manual_seed(seed)
  y = t.rand((rows, k), generator=g, device=device, dtype=t.float32)
  hi = t.zeros((rows, dev.round_up(k, 64)), dtype=t.float16, device=device)
  lo = t.zeros_like(hi)
  hi[:, :k] = y.half()
  lo[:, :k] = (y - hi[:, :k].float()).half()
  return hi, lo


def exact_product(a_hi, a_lo, b_hi, k, precision):
  """float64 of what the kernel computes: hi.hi^T (single), + lo.hi^T (split2)."""
  ah, bh = a_hi[:, :k].double(), b_hi[:, :k].double()
  want = ah @ bh.T
  if precision == nat.GEMM_SPLIT2:
    want += a_lo[:, :k].double() @ bh.T
  return want


def assert_close(got, want, precision):
  rel = (got.double() - want).abs() / want.abs().clamp_min(1e-300)
  rms, worst = rel.pow(2).mean().sqrt().item(), rel.max().item()
  # the tensor core's fp32 accumulation truncates within a register chain; single-MMA chains are 4
  # K-blocks long, split2 chains 2, so single gets twice the bound (measured rms 1.1e-6 at
  # N = 1,000 to 4,097)
  scale = 2.0 if precision == nat.GEMM_SINGLE else 1.0
  assert rms <= 1e-6 * scale, (rms, worst)
  assert worst <= 3e-6 * scale, (rms, worst)


@pytest.mark.parametrize("precision", sorted(PRECISIONS))
@pytest.mark.parametrize("n", SIZES)
def test_symmetric_diffuse_tiles(engine, n, precision):
  t = dev.torch()
  prec = PRECISIONS[precision]
  hi, lo = split_planes(n, n, seed=n, device=engine.device)
  s = engine.matrix(n)
  s.fill_(float("nan"))
  mx = engine.vector(n, t.float32)
  sm = engine.vector(n, t.float64)
  engine.call("sc_diffuse", nat.GEMM_TCGEN05, prec, None, 0, dev._ptr(hi), dev._ptr(lo),
              hi.stride(0), n, dev._ptr(s), s.stride(0), dev._ptr(mx), dev._ptr(sm), engine.stream)
  t.cuda.synchronize()
  s = s[:, :n]
  assert t.isfinite(s).all()
  assert t.equal(s, s.T)
  # split2 computes hi_r.hi_c + lo_r.hi_c, which is not symmetric in (r, c): the upper triangle is
  # the computed half, the lower one is its mirror (checked bitwise above)
  want = exact_product(hi, lo, hi, n, prec)
  upper = t.triu(t.ones((n, n), dtype=t.bool, device=engine.device))
  assert_close(s[upper], want[upper], prec)
  assert t.equal(mx, s.max(dim=1).values)
  t.testing.assert_close(sm, s.double().sum(dim=1), rtol=1e-6, atol=0)


@pytest.mark.parametrize("precision", sorted(PRECISIONS))
@pytest.mark.parametrize("m,n,k", [(300, 457, 1000), (1000, 193, 2049), (129, 4097, 383)])
def test_general_product_with_mirror(engine, m, n, k, precision):
  t = dev.torch()
  prec = PRECISIONS[precision]
  a_hi, a_lo = split_planes(m, k, seed=1, device=engine.device)
  b_hi, b_lo = split_planes(n, k, seed=2, device=engine.device)
  c = t.full((m, dev.round_up(n, 64)), float("nan"), device=engine.device)
  mirror = t.full((n, dev.round_up(m, 64)), float("nan"), device=engine.device)
  engine.call("sc_gemm_nt_planes", prec, dev._ptr(a_hi), dev._ptr(a_lo), a_hi.stride(0), m,
              dev._ptr(b_hi), dev._ptr(b_lo), b_hi.stride(0), n, k, dev._ptr(c), c.stride(0),
              dev._ptr(mirror), mirror.stride(0), engine.stream)
  t.cuda.synchronize()
  c, mirror = c[:, :n], mirror[:, :m]
  assert t.isfinite(c).all()
  assert t.equal(mirror, c.T)
  assert_close(c, exact_product(a_hi, a_lo, b_hi, k, prec), prec)
