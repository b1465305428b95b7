"""GPU: the symmetric blur pair without a stored B, against the pair that stores it, bit for bit.

Pass 1 (sc_blur_upper_rowmax with b_out == NULL) must give the row maxima of the storing pass, and
pass 2 (sc_blur_threshold_symmetrize_upper, which blurs A's upper triangle again) the fp32 Y and
the fp16 planes that sc_threshold_symmetrize_upper writes from the stored B.  Outputs and padding
start as NaN, and whole buffers are compared, so an element written by one and not the other, or a
padding element written by either, fails.  Sizes cover the 256-row bands and 120-column strips of
the recomputing kernels at their edges (n = 1 and 5 reflect repeatedly; 16,385 has interior,
diagonal and ragged-edge strips), with and without the crop vector, the diagonal folded as 0 or
not, the diagonal preserved or not, binarization and both symmetrize types.
"""

import numpy as np
import pytest

from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from test_gpu_refinement_kernels import (RULES, blur_upper, nan_buf, nan_vector, padded,
                                         run_upper, same_bits, structured_affinity, P, MULT)

pytestmark = pytest.mark.gpu

SIZES = [1, 5, 63, 64, 65, 127, 700, 2049, 4099, 16385]


def t():
  return dev.torch()


def pass1(engine, ab, n, diag, zero_diag):
  m = nan_vector(n, engine.device, zero=False)        # the entry zero-fills m itself
  engine.call("sc_blur_upper_rowmax", dev._ptr(ab), n, ab.stride(0), dev._ptr(diag), 1.0,
              int(zero_diag), None, 0, dev._ptr(m), engine.stream)
  t().cuda.synchronize()
  assert t().isnan(m[n:]).all()
  return m[:n]


def pass2(engine, ab, n, diag, m, binarize, keep_diag, sym_type, want_y, want_hi, want_lo):
  ld = ab.shape[1]
  y = nan_buf(n, ld, engine.device) if want_y else None
  hi = nan_buf(n, ld, engine.device, t().float16) if want_hi else None
  lo = nan_buf(n, ld, engine.device, t().float16)     # stays NaN when not passed
  engine.call("sc_blur_threshold_symmetrize_upper", dev._ptr(ab), n, ab.stride(0), dev._ptr(diag),
              1.0, dev._ptr(m), P, MULT, binarize, keep_diag, sym_type, dev._ptr(y),
              0 if y is None else y.stride(0), dev._ptr(hi), dev._ptr(lo if want_lo else None),
              0 if hi is None else hi.stride(0), engine.stream)
  t().cuda.synchronize()
  return y, hi, lo


def check_pair(engine, ab, n, seed_rules):
  crop = engine.crop_values(ab, n)
  for diag in (None, crop):
    for zero_diag in (0, 1):
      b, m_ref = blur_upper(engine, ab, n, 1.0, zero_diag, diag=diag)
      m = pass1(engine, ab, n, diag, zero_diag)
      assert same_bits(m, m_ref), "%d row maxima differ" % (m != m_ref).sum().item()
      for keep_diag in (0, 1):
        for binarize, sym_type in seed_rules:
          want = run_upper(engine, b, m_ref, n, binarize, keep_diag, sym_type, True, True, True)
          got = pass2(engine, ab, n, diag, m, binarize, keep_diag, sym_type, True, True, True)
          for name, g, w in zip(("y", "hi", "lo"), got, want):
            assert same_bits(g, w), "%s: %d elements differ" % (
                name, (g.float() != w.float()).sum().item())
      # the hi plane alone (a single-MMA Diffuse): the lo buffer is not touched
      _, hi_ref, _ = run_upper(engine, b, m_ref, n, 0, zero_diag, nat.SYMMETRIZE_MAX, False, True,
                               False)
      _, hi, lo = pass2(engine, ab, n, diag, m, 0, zero_diag, nat.SYMMETRIZE_MAX, False, True,
                        False)
      assert same_bits(hi, hi_ref)
      assert t().isnan(lo).all()
      yy = got[0][:, :n]
      assert t().equal(yy, yy.T)


@pytest.mark.parametrize("n", SIZES)
def test_pair_matches_stored_blur(engine, n):
  a = structured_affinity(n, seed=n + 11)
  check_pair(engine, padded(a, engine.device), n, RULES)


def test_pair_unaligned_input(engine):
  """A at an odd leading dimension and a base 4 bytes past alignment: no 128-bit loads."""
  n = 700
  a = structured_affinity(n, seed=5)
  ld = dev.round_up(n, 64) + 64
  base = nan_buf(n, ld + 1, engine.device)
  base[:, 1:n + 1] = t().from_numpy(np.ascontiguousarray(a)).to(engine.device)
  ab = base[:, 1:]
  assert ab.stride(0) % 4 == 1 and ab.data_ptr() % 16 == 4
  check_pair(engine, ab, n, RULES[:1])


def test_engine_pair_matches_stored_route(engine):
  """Engine.blur_upper_rowmax's record through threshold_symmetrize_upper == the stored B."""
  n = 4099
  ab = padded(structured_affinity(n, seed=9), engine.device)
  crop = engine.crop_values(ab, n)
  rec, m = engine.blur_upper_rowmax(ab, n, 1.0, crop, True)
  assert isinstance(rec, dev.DeferredBlur)
  b, m_ref = engine.blur_upper_rowmax(ab, n, 1.0, crop, True, store_b=True)
  assert same_bits(m, m_ref)
  for want_lo in (True, False):
    got = engine.threshold_symmetrize_upper(rec, n, m, P, MULT, False, True, nat.SYMMETRIZE_MAX,
                                            True, True, want_lo)
    want = engine.threshold_symmetrize_upper(b, n, m_ref, P, MULT, False, True,
                                             nat.SYMMETRIZE_MAX, True, True, want_lo)
    t().cuda.synchronize()
    for g, w in zip(got, want):
      assert (g is None) == (w is None)
      if g is not None:
        assert t().equal(g[:, :n], w[:, :n])
