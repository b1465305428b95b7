"""GPU: the sc_krylov_* primitives of the general eigen path (csrc/eigh_lanczos.cu) at the launch
edges of their kernels, against float64.

Every output and every padding starts as NaN, so an element that is never written, or a read past
the data, shows up; every primitive runs twice and must repeat bit for bit.  u = 2^-53: a sum of
n fp64 products has an error <= n u sum|a_i b_i| however it is ordered (fma chains and tree
reductions alike), and the host's float64 restatement has the same bound again.
"""

import ctypes
import math

import numpy as np
import pytest

from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
NAN = float("nan")


def t():
  return dev.torch()


def to_dev(a):
  return t().from_numpy(np.ascontiguousarray(a)).to(dev.Engine.get().device)


def host(x):
  t().cuda.synchronize()
  return x.cpu().numpy()


def nan_buf(shape, dtype=None):
  return t().full(shape, NAN, dtype=dtype or t().float64, device=dev.Engine.get().device)


def host_ptr(a):
  return a.ctypes.data_as(ctypes.c_void_p)


def bits(x):
  return np.ascontiguousarray(x, dtype=np.float64).view(np.int64)


# ------------------------------------------------------------------ sc_krylov_matvec
MV = [1, 7, 8, 9, 255, 2047, 2048, 2049, 4097, 6145]


@pytest.mark.parametrize("n", MV)
def test_matvec_against_float64(engine, n):
  """k_symv_f32_f64: 8 rows per CTA, 2048-column chunks of x in shared memory, 8 loads per lane.
  The fp32 entries are exact in fp64, so |y - S x| <= n u (|S| |x|) on the device and again on
  the host: 2 n u (|S| |x|) elementwise."""
  rng = np.random.default_rng(n)
  s_h = rng.uniform(-1.0, 1.0, (n, n)).astype(np.float32)
  lda = n + 5                                         # odd pitch, NaN padding
  s = nan_buf((n, lda), t().float32)
  s[:, :n] = to_dev(s_h)
  s64 = s_h.astype(np.float64)
  for rows in sorted({n, max(1, n // 2 + 1)}):        # the whole matrix and a row slab
    x_h = rng.standard_normal(n)
    x = to_dev(x_h)
    outs = []
    for _ in range(2):
      y = nan_buf((rows + 3,))
      engine.call("sc_krylov_matvec", dev._ptr(s), rows, n, lda, dev._ptr(x), dev._ptr(y),
                  engine.stream)
      outs.append(host(y))
    got = outs[0]
    assert np.isnan(got[rows:]).all(), "wrote past `rows`"
    assert np.isfinite(got[:rows]).all(), "a row was not written (or NaN padding was read)"
    ref = s64[:rows] @ x_h
    tol = 2 * n * U * (np.abs(s64[:rows]) @ np.abs(x_h))
    assert np.all(np.abs(got[:rows] - ref) <= tol), (rows, np.max(np.abs(got[:rows] - ref) / tol))
    np.testing.assert_array_equal(bits(outs[1]), bits(got))


# ------------------------------------------------------------------ sc_krylov_orthogonalize
ORTHO = [(n, c) for n in (1, 255, 257, 4097) for c in (0, 1, 31, 32, 33, 160, 1024) if c <= n]


def orthonormal(n, count, rng):
  if count == 0:
    return np.zeros((0, n))
  q, _ = np.linalg.qr(rng.standard_normal((n, count)))
  return q.T.copy()


def orthogonalize(engine, v_dev, n, count, w_h):
  w = nan_buf((n + 4,))
  w[:n] = to_dev(w_h)
  h = np.full(max(count, 1), NAN)
  nrm2 = ctypes.c_double(NAN)
  engine.call("sc_krylov_orthogonalize", dev._ptr(v_dev), n, count, dev._ptr(w), host_ptr(h),
              ctypes.byref(nrm2), engine.stream)
  out = host(w)
  assert np.isnan(out[n:]).all(), "wrote past n"
  return out[:n], h[:count], nrm2.value


@pytest.mark.parametrize("n,count", ORTHO)
def test_orthogonalize_against_float64(engine, n, count):
  """Classical Gram-Schmidt twice.  One sweep: each coefficient <v_j, w> is off by <= n u |w|
  (Cauchy-Schwarz on sum |v_ji w_i|) and the update w - V h by <= count u (|w| + sum |h_j|) <=
  count (1 + sqrt(count)) u |w|; so the part of w left in span(V) after a sweep is
  <= B |w_in|, B = (sqrt(count) n + count (1 + sqrt(count))) u.  After the second sweep
  |V^T w| <= B |w_1| <= B (|w| + B |w_0|); the host adds sqrt(count) n u |w| computing V^T w.
  The coefficients h = h_1 + h_2 differ from the float64 restatement by the first sweep's
  rounding on both sides and the second sweep's inputs: <= 4 (n u + B) |w_0|."""
  rng = np.random.default_rng(n * 7919 + count)
  v_h = orthonormal(n, count, rng)
  v = nan_buf((count + 2, n))                           # rows past `count` are NaN
  if count:
    v[:count] = to_dev(v_h)
  c = rng.standard_normal(count)
  r = rng.standard_normal(n)
  cases = {"random": r}
  if count:
    cases["in span"] = v_h.T @ c                        # leaves only rounding: nrm2 near zero
    if count < n:
      cases["near span"] = v_h.T @ c + 1e-8 * r / np.linalg.norm(r)
  b = (math.sqrt(count) * n + count * (1 + math.sqrt(count))) * U
  for name, w0 in cases.items():
    (w, h, nrm2), (w_b, h_b, nrm2_b) = (orthogonalize(engine, v, n, count, w0) for _ in range(2))
    np.testing.assert_array_equal(bits(w_b), bits(w), err_msg=name)
    np.testing.assert_array_equal(bits(h_b), bits(h), err_msg=name)
    assert bits(np.array([nrm2_b])) == bits(np.array([nrm2])), name
    assert np.isfinite(w).all(), name
    norm0, norm = np.linalg.norm(w0), np.linalg.norm(w)
    # |w|^2: n products summed twice (device, host)
    assert abs(nrm2 - norm * norm) <= 2 * n * U * norm * norm, name
    if count == 0:
      np.testing.assert_array_equal(bits(w), bits(w0), err_msg=name)
      continue
    h1 = v_h @ w0
    h2 = v_h @ (w0 - v_h.T @ h1)
    assert np.all(np.abs(h - (h1 + h2)) <= 4 * (n * U + b) * norm0), (name, np.abs(h - h1 - h2).max())
    left = np.linalg.norm(v_h @ w)
    assert left <= 2 * b * (norm + b * norm0) + math.sqrt(count) * n * U * norm, (name, left)


# ------------------------------------------------------------------ sc_krylov_combine
@pytest.mark.parametrize("m", [1, 2, 64, 161])
@pytest.mark.parametrize("k", [1, 7, 8, 9, 63, 64])
def test_combine_against_float64(engine, k, m):
  """out[p] = sum_q z[q, p] V_q: m fp64 fmas per element, <= m u (|Z|^T |V|) on each side."""
  n = 1003                                              # ragged against the 256-thread rows
  rng = np.random.default_rng(k * 1000 + m)
  v_h = rng.standard_normal((m, n))
  z = rng.standard_normal((m, k))
  v = nan_buf((m + 2, n))
  v[:m] = to_dev(v_h)
  outs = []
  for _ in range(2):
    out = nan_buf((k + 1, n))
    engine.call("sc_krylov_combine", dev._ptr(v), n, m, host_ptr(z), k, dev._ptr(out),
                engine.stream)
    outs.append(host(out))
  got = outs[0]
  assert np.isnan(got[k]).all(), "wrote past k vectors"
  assert np.isfinite(got[:k]).all(), "an output element was not written (or a NaN row was read)"
  ref = z.T @ v_h
  tol = 2 * m * U * (np.abs(z).T @ np.abs(v_h))
  assert np.all(np.abs(got[:k] - ref) <= tol)
  np.testing.assert_array_equal(bits(outs[1]), bits(got))


def test_combine_refuses_more_than_64_columns_and_aliasing(engine):
  n, m = 300, 4
  v = to_dev(np.ones((m + 1, n)))
  out = nan_buf((65, n))
  z = np.ones((m, 65))
  with pytest.raises(nat.NativeError):
    engine.call("sc_krylov_combine", dev._ptr(v), n, m, host_ptr(z), 65, dev._ptr(out), engine.stream)
  z = np.ones((m, 1))
  with pytest.raises(nat.NativeError):
    engine.call("sc_krylov_combine", dev._ptr(v), n, m, host_ptr(z), 1, dev._ptr(v), engine.stream)


# ------------------------------------------------------------------ sc_krylov_scale / _random
RAGGED = [1, 255, 256, 257, 1000, 4097]


@pytest.mark.parametrize("n", RAGGED)
def test_scale_is_one_rounded_product(engine, n):
  rng = np.random.default_rng(n)
  w_h = rng.standard_normal(n)
  w = to_dev(w_h)
  for alpha in (0.0, -1.0, 3.0 / 7.0, 1e300, 1e-300):
    out = nan_buf((n + 3,))
    engine.call("sc_krylov_scale", dev._ptr(w), n, alpha, dev._ptr(out), engine.stream)
    got = host(out)
    np.testing.assert_array_equal(bits(got[:n]), bits(alpha * w_h))   # one IEEE product
    assert np.isnan(got[n:]).all()


def splitmix_vector(n, seed):
  """k_random_vec restated: splitmix64 of seed' + golden * (i + 1), top 53 bits in [-0.5, 0.5),
  seed' = 0x5CB200 + 7919 seed (sc_krylov_random)."""
  m = np.uint64(0xFFFFFFFFFFFFFFFF)
  with np.errstate(over="ignore"):
    base = np.uint64((0x5CB200 + 7919 * seed) & 0xFFFFFFFFFFFFFFFF)
    z = base + np.uint64(0x9E3779B97F4A7C15) * np.arange(1, n + 1, dtype=np.uint64)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = (z ^ (z >> np.uint64(31))) & m
  return (z >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0) - 0.5


@pytest.mark.parametrize("n", RAGGED)
def test_random_is_seeded_splitmix_in_half_open_interval(engine, n):
  got = {}
  for seed in (1, 2, 1):
    w = nan_buf((n + 3,))
    engine.call("sc_krylov_random", dev._ptr(w), n, seed, engine.stream)
    out = host(w)
    assert np.isnan(out[n:]).all()
    out = out[:n]
    assert np.all(out >= -0.5) and np.all(out < 0.5)
    np.testing.assert_array_equal(bits(out), bits(splitmix_vector(n, seed)))
    if seed in got:
      np.testing.assert_array_equal(bits(out), bits(got[seed]))
    got[seed] = out
  if n > 1:
    assert not np.array_equal(got[1], got[2])


# ------------------------------------------------------------------ sc_krylov_columns
@pytest.mark.parametrize("n,k", [(1, 1), (1, 64), (300, 7), (4097, 3), (257, 1024)])
def test_columns_are_unit_and_parallel(engine, n, k):
  """k_mapback without left / right terms: v[i, c] = u_c[i] / |u_c|, row-major [n, k].  The norm
  sums n squares (<= n u relative), its square root halves that, the reciprocal and the product
  add a rounding each: <= (n / 2 + 3) u |v| per element, and the host's restatement as much."""
  rng = np.random.default_rng(n + k)
  u_h = rng.standard_normal((k, n)) * np.exp(rng.uniform(-20, 20, (k, 1)))
  u = nan_buf((k + 1, n))
  u[:k] = to_dev(u_h)
  outs = []
  for _ in range(2):
    out = nan_buf((n * k + 5,))
    engine.call("sc_krylov_columns", dev._ptr(u), n, k, dev._ptr(out), engine.stream)
    outs.append(host(out))
  got = outs[0]
  assert np.isnan(got[n * k:]).all(), "wrote past the [n, k] array"
  v = got[:n * k].reshape(n, k)
  ref = (u_h / np.linalg.norm(u_h, axis=1, keepdims=True)).T
  assert np.all(np.abs(v - ref) <= (n + 6) * U * np.abs(ref)), np.max(np.abs(v - ref))
  assert np.all(np.abs(np.linalg.norm(v, axis=0) - 1.0) <= (2 * n + 6) * U)
  np.testing.assert_array_equal(bits(outs[1]), bits(got))
