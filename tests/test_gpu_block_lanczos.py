"""GPU: the thick-restart block Lanczos solver (csrc/eigh_lanczos.cu) against float64 LAPACK.

Every result is compared with scipy.linalg.eigh on exactly the operator the device sees, in its
symmetrised form T = diag(delta) + sign * c S c, c = sqrt(left * right):
  * stored operator: S is the uploaded fp32 matrix, converted to float64;
  * factored operator: S = Y Y^T in float64, Y the fp16 matrix converted exactly.  The device
    computes Y (Y T), which is S T only for a symmetric Y, so every Y here is symmetric.
The eigenvectors the solver returns are those of the non-symmetric M = diag(delta) + sign *
diag(left) S diag(right), v = E u / |E u| with E = sqrt(left / right).

Bounds (derived once here, used below):
  * The solver stops when every wanted residual satisfies |r| <= tol * Theta, Theta = max(largest
    |Ritz value| of the basis, scale) <= ||T||_2 = max |lambda| (Ritz values lie inside the
    spectrum, and `scale` is a magnitude of an earlier Ritz value).  For a symmetric operator each
    Ritz value lies within |r| of an eigenvalue, so a solve that misses none of the wanted
    eigenvalues has |theta_i - lambda_i| <= tol * ||T||_2.
  * The block product is fp64 with fp64 accumulation: per product, |fl(T x) - T x| <=
    gamma_{n + splits} |T| |x| elementwise, so its 2-norm error is at most (n + 64) u || |T| ||_inf
    for a unit x (u = 2^-53, || |T| ||_2 <= the largest row sum of |T| for symmetric |T|; at most
    64 column splits).  The factored operator takes two such products: ROUND = 2 (n + 64) u ||
    |T| ||_inf, with |T| <= |delta| + |c| |Y| |Y|^T |c|.
  * A Ritz vector x = V z is a combination of at most jmax = 7 b basis vectors, each product
    carrying the error above: ||T x - theta x|| <= tol ||T||_2 + sqrt(jmax) ROUND.  A window on the
    complement of L locked vectors adds ||L^T T x|| = ||R_L^T x|| <= ||R_L||_F <= sqrt(L) tol
    ||T||_2 (R_L: the locked vectors' residuals).
  * M v - theta v = E (T u - theta u) / |E u|, so the residual of v is at most max(E) / min(E)
    times that of u.
  * Orthonormality: classical Gram-Schmidt applied twice keeps the basis orthonormal to
    O(jmax n u); ORTH = 4 (jmax + L) n u allows a factor 4 over that.
"""

import ctypes
import math

import numpy as np
import pytest
import scipy.linalg as sla
from scipy.sparse.csgraph import connected_components

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import eigen_windows as ew
from spectralcluster_b200 import laplacian as lap
from oracle import spectral_oracle as orc

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
TOL = 1e-9                 # the solver's default tolerance (tol <= 0)
NAN = float("nan")
LARGEST, SMALLEST = nat.EIG_LARGEST, nat.EIG_SMALLEST


# ---------------------------------------------------------------- restated host rules
def block_size(n_values):
  """sc_eigh_block_size: vectors per block for n_values pairs."""
  return 4 if n_values <= 4 else 8 if n_values <= 8 else 12 if n_values <= 12 else 16


def smallest_n(n_values, n_locked=0):
  """Smallest n the solver takes: n - n_locked >= 2 * 7 * b (six processed blocks and the one in
  flight, twice)."""
  return n_locked + 2 * 7 * block_size(n_values)


def product_plan(rows, n, sm_count):
  """block_product_scratch_doubles: (column splits, columns per split)."""
  row_blocks = -(-rows // 256)
  splits = -(-6 * sm_count // row_blocks)
  splits = max(1, min(splits, -(-n // 2048)))
  cps = -(-n // splits)
  cps = -(-cps // 32) * 32
  return -(-n // cps), cps


def sm_count(engine):
  return int(nat.load().sc_context_sm_count(engine.ctx))


def up(x):
  return None if x is None else dev.torch().from_numpy(np.ascontiguousarray(x)).to("cuda")


def host(x, n, fill):
  return np.full(n, fill) if x is None else x.cpu().numpy()


# ---------------------------------------------------------------- operators and references
FORMS = ("none", "rownorm", "unnormalized", "randomwalk", "graphcut")
LAPLACIAN = {"unnormalized": lap.LaplacianType.Unnormalized,
             "randomwalk": lap.LaplacianType.RandomWalk, "graphcut": lap.LaplacianType.GraphCut}


class Operator:
  """One operator on the device (NaN-padded operand, Laplacian terms) and on the host in float64
  (T, M, E), with its LAPACK spectrum computed once."""

  def __init__(self, engine, kind, mat, form="none", sign=None):
    t = dev.torch()
    self.engine, self.kind, self.form = engine, kind, form
    n = self.n = mat.shape[0]
    ld = dev.round_up(n, 64)
    dtype = t.float32 if kind == "stored" else t.float16
    self.dev = t.full((n, ld), NAN, dtype=dtype, device=engine.device)
    self.dev[:, :n] = t.from_numpy(np.ascontiguousarray(mat).astype(
        np.float32 if kind == "stored" else np.float16)).to(engine.device)
    m64 = self.dev[:, :n].double()
    if kind == "stored":
      s_dev, abs_s = m64, m64.abs()
    else:
      s_dev, abs_s = m64 @ m64.T, m64.abs() @ m64.abs().T
    if form in ("none", "rownorm"):
      r = None if form == "none" else 1.0 / s_dev.max(dim=1).values
      delta, left, right, sgn = None, r, None, 1.0
    else:
      r = 1.0 / s_dev.max(dim=1).values
      delta, left, right, sgn, _ = lap.terms_from_row_sums(s_dev.sum(dim=1), r, LAPLACIAN[form])
    self.sign = float(sgn if sign is None else sign)
    self.delta, self.left, self.right = delta, left, right
    d, lf, rt = host(delta, n, 0.0), host(left, n, 1.0), host(right, n, 1.0)
    s = s_dev.cpu().numpy()
    c = np.sqrt(lf * rt)
    self.e = np.sqrt(lf / rt)
    self.t = np.diag(d) + self.sign * c[:, None] * s * c[None, :]
    self.m = np.diag(d) + self.sign * lf[:, None] * s * rt[None, :]
    absrow = np.abs(d) + np.abs(c) * (abs_s.cpu().numpy() @ np.abs(c))
    self.round = 2 * (n + 64) * U * float(absrow.max())
    self.lam, self.q = sla.eigh(self.t)             # ascending
    self.norm = float(np.abs(self.lam).max())
    self.cond_e = float(self.e.max() / self.e.min())
    del s_dev, abs_s, m64

  @property
  def terms(self):
    return (self.delta, self.left, self.right, self.sign)

  def want(self, which, count):
    return self.lam[::-1][:count] if which == LARGEST else self.lam[:count]

  def solve(self, which, n_values, n_vectors):
    """sc_eigh_extremal(_factored) into NaN-filled outputs -> (w, v host, stats)."""
    t = dev.torch()
    n = self.n
    w = np.full(max(n_values, 1), NAN)
    v = t.full((n, max(n_vectors, 1)), NAN, dtype=t.float64, device=self.engine.device)
    stats = np.full(4, -1, dtype=np.int64)
    entry = "sc_eigh_extremal" if self.kind == "stored" else "sc_eigh_extremal_factored"
    self.engine.call(entry, dev._ptr(self.dev), n, self.dev.stride(0), dev._ptr(self.delta),
                     dev._ptr(self.left), dev._ptr(self.right), self.sign, int(which), n_values,
                     n_vectors, 0.0, 0, w.ctypes.data_as(ctypes.c_void_p), dev._ptr(v),
                     stats.ctypes.data_as(ctypes.c_void_p), self.engine.stream)
    vh = v.cpu().numpy()
    if n_vectors == 0:
      assert np.isnan(vh).all()                     # nothing asked, nothing written
    return w[:n_values], vh[:, :n_vectors], stats

  def check_vectors(self, w, v, locked_before=0, b=16):
    """Residual, unit norm and symmetrised-space orthonormality of M-eigenvectors v."""
    k = v.shape[1]
    if k == 0:
      return
    assert np.isfinite(v).all()
    jmax = 7 * b
    np.testing.assert_allclose(np.linalg.norm(v, axis=0), 1.0, rtol=0, atol=4 * self.n * U)
    bound_u = (1 + math.sqrt(locked_before)) * TOL * self.norm + math.sqrt(jmax) * self.round
    resid = np.linalg.norm(self.m @ v - v * w[None, :k], axis=0)
    assert resid.max() <= self.cond_e * bound_u, (resid.max(), self.cond_e * bound_u)
    u = v / self.e[:, None]
    u /= np.linalg.norm(u, axis=0, keepdims=True)
    orth = 4 * (jmax + locked_before) * self.n * U
    assert np.abs(u.T @ u - np.eye(k)).max() <= orth


def random_symmetric(n, seed, shift=0.0):
  rng = np.random.default_rng(seed)
  g = rng.standard_normal((n, n))
  return (g + g.T) / (2 * math.sqrt(n)) + shift * np.eye(n)


def speaker_matrix(n, seed, kind):
  """Stored: S = A A with A the cosine affinity of 6 synthetic speakers (d = 32).  Factored: Y = A
  (symmetric), so that the device's S = Y Y^T is the same product."""
  a = orc.affinity(orc.synthetic_dvectors(n, 32, 6, seed=seed))
  if kind == "stored":
    return (a @ a) / n
  return a


class Cache:
  def __init__(self, engine):
    self.engine, self.ops = engine, {}

  def get(self, key, make):
    if key not in self.ops:
      self.ops[key] = make()
    return self.ops[key]


@pytest.fixture(scope="module")
def cache(engine):
  c = Cache(engine)
  yield c
  c.ops.clear()
  dev.torch().cuda.empty_cache()


def random_operator(cache, kind, n=1281):
  # factored: Y shifted to eigenvalues in about [1, 5] so that S = Y^2 keeps both ends gap-free
  # (the smallest end of an unshifted Y^2 would pile up at 0)
  mat = random_symmetric(n, 7 + n, 0.0 if kind == "stored" else 3.0)
  return cache.get(("random", kind, n), lambda: Operator(cache.engine, kind, mat))


def speaker_operator(cache, kind, form, n=1279):
  return cache.get(("speaker", kind, form, n),
                   lambda: Operator(cache.engine, kind, speaker_matrix(n, 3, kind), form))


def check_values(op, which, w):
  want = op.want(which, len(w))
  bound = TOL * op.norm + op.round
  err = np.abs(w - want)
  assert err.max() <= bound, (int(err.argmax()), w[err.argmax()], want[err.argmax()], bound)


def check_values_in_a_cluster(op, which, w):
  """Values at an end where the spectrum is a cluster narrower than the stopping rule resolves
  (the bulk of a speaker-like spectrum, whose width is ~1e-7 ||T||): each Ritz value lies within
  |r| <= tol ||T|| of an eigenvalue, and the Rayleigh quotient on the returned vectors is diag(w)
  up to that residual, so by Weyl and Cauchy interlacing the i-th value from the wanted end does not
  pass the i-th eigenvalue by more than tol ||T||."""
  bound = TOL * op.norm + op.round
  assert np.abs(w[:, None] - op.lam[None, :]).min(axis=1).max() <= bound
  want = op.want(which, len(w))
  assert np.all(w <= want + bound) if which == LARGEST else np.all(w >= want - bound)


def check_solve(op, which, nv, nvec, w, v, stats, resolved=True):
  b = block_size(nv)
  (check_values if resolved else check_values_in_a_cluster)(op, which, w)
  assert stats[0] == b * stats[3] and stats[2] >= nv, stats
  op.check_vectors(w, v, b=b)


# ---------------------------------------------------------------- A. block products
def test_block_size_restatement(engine):
  lib = nat.load()
  assert [lib.sc_eigh_block_size(k) for k in range(1, 33)] == [block_size(k) for k in range(1, 33)]


BP_SHAPES = [(255, 1000), (1, 2049), (2049, 2049), (4097, 4097), (511, 6000)]


def test_block_product_shapes_cover_the_split_edges(engine):
  """The shapes below, on this device's SM count: one split, several splits whose width is an odd
  multiple of 32 columns, a short last split, and rows % 256 of 1 and 255."""
  plans = [product_plan(rows, n, sm_count(engine)) for rows, n in BP_SHAPES]
  assert any(s == 1 for s, _ in plans)
  assert any(s > 1 and c % 64 == 32 for s, c in plans)
  assert any(s > 1 and n - (s - 1) * c < c for (s, c), (_, n) in zip(plans, BP_SHAPES))
  assert {rows % 256 for rows, _ in BP_SHAPES} >= {1, 255}


@pytest.mark.parametrize("rows,n", BP_SHAPES)
def test_block_products_against_float64(engine, rows, n):
  """sc_block_product and sc_block_product_f16 for every b in 1..16: within the float64 summation
  bound of the exact product, the fp16 kernel bit for bit the fp32 kernel on the upcast matrix
  (fp16 -> fp32 -> fp64 is exact), two calls identical.  NaN in the padding of S, T and Y."""
  t = dev.torch()
  g = t.Generator(device="cpu").manual_seed(rows * 131 + n)
  splits, _ = product_plan(rows, n, sm_count(engine))
  ld32, ld16 = dev.round_up(n, 4) + 4, dev.round_up(n, 8) + 8
  s16 = (t.rand((rows, n), generator=g) - 0.3).half()
  s32 = t.full((rows, ld32), NAN, dtype=t.float32)
  s32[:, :n] = t.rand((rows, n), generator=g) - 0.3
  h32 = t.full((rows, ld32), NAN, dtype=t.float32)
  h32[:, :n] = s16.float()
  h16 = t.full((rows, ld16), NAN, dtype=t.float16)
  h16[:, :n] = s16
  ldt = n + (n & 1) + 2
  tv = t.full((16, ldt), NAN, dtype=t.float64)
  tv[:, :n] = t.randn((16, n), generator=g, dtype=t.float64)
  s32_d, h32_d, h16_d, t_d = (x.to(engine.device) for x in (s32, h32, h16, tv))
  ldy = rows + 3
  # gamma_{n + splits} for the device sum and for the float64 reference, each bounded by the
  # product of absolute values
  gamma = 2 * (n + splits) * U / (1 - (n + splits) * U)

  def product(entry, s_d, b):
    y = t.full((b, ldy), NAN, dtype=t.float64, device=engine.device)
    engine.call(entry, dev._ptr(s_d), rows, n, s_d.stride(0), dev._ptr(t_d), ldt, ctypes.c_int(b),
                dev._ptr(y), ldy, engine.stream)
    y = y.cpu()
    assert t.isnan(y[:, rows:]).all()            # nothing past `rows`
    return y[:, :rows]

  exact = {"sc_block_product": s32[:, :n].double(), "sc_block_product_f16": h32[:, :n].double()}
  for b in range(1, 17):
    for entry, s_d in (("sc_block_product", s32_d), ("sc_block_product_f16", h16_d)):
      y = product(entry, s_d, b)
      want = tv[:b, :n] @ exact[entry].T
      scale = tv[:b, :n].abs() @ exact[entry].abs().T
      assert bool(((y - want).abs() <= gamma * scale).all()), (entry, b)
      assert t.equal(y, product(entry, s_d, b)), (entry, b)
    assert t.equal(product("sc_block_product_f16", h16_d, b),
                   product("sc_block_product", h32_d, b)), b


# ---------------------------------------------------------------- B. one solve
N_VALUES = [1, 4, 5, 8, 9, 12, 13, 16, 17, 24, 32]


def vector_count(nv, i):
  return (0, max(1, nv // 2), nv)[i % 3]


@pytest.mark.parametrize("which", [LARGEST, SMALLEST])
@pytest.mark.parametrize("nv", N_VALUES)
@pytest.mark.parametrize("kind", ["stored", "factored"])
def test_one_solve_on_a_random_spectrum(cache, kind, nv, which):
  """A random symmetric matrix (no gap at either end: the solver restarts), every width at both
  ends of its range, n = 1281 (n % 256 == 1).  Values, vectors, statistics, and a repeated call
  identical bit for bit."""
  op = random_operator(cache, kind)
  nvec = vector_count(nv, N_VALUES.index(nv) + which + (kind == "factored"))
  w, v, stats = op.solve(which, nv, nvec)
  check_solve(op, which, nv, nvec, w, v, stats)
  w2, v2, stats2 = op.solve(which, nv, nvec)
  assert np.array_equal(w, w2) and np.array_equal(v, v2) and np.array_equal(stats, stats2)


@pytest.mark.parametrize("nv", [5, 16, 24])
@pytest.mark.parametrize("which", [LARGEST, SMALLEST])
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", ["stored", "factored"])
def test_one_solve_under_every_operator_form(cache, kind, form, which, nv):
  """A speaker-like S (6 synthetic speakers, n = 1279: n % 256 == 255) under every operator form
  of laplacian.terms_from_row_sums, at both ends.  At the end predict() reads (largest without a
  Laplacian, smallest with one) the values are resolved and compared in order; the other end is
  the rank-deficient bulk, clustered within ~1e-7 ||T||, where the stopping rule only places each
  value within tol ||T|| of an eigenvalue (check_values_in_a_cluster)."""
  op = speaker_operator(cache, kind, form)
  nvec = vector_count(nv, [5, 16, 24].index(nv) + which)
  w, v, stats = op.solve(which, nv, nvec)
  resolved = which == (LARGEST if form in ("none", "rownorm") else SMALLEST)
  check_solve(op, which, nv, nvec, w, v, stats, resolved)


@pytest.mark.parametrize("nv", [1, 4, 5, 12, 16, 17, 32])
@pytest.mark.parametrize("kind", ["stored", "factored"])
def test_smallest_legal_n(engine, kind, nv):
  """n = 2 * 7 * b is accepted and solved right; one row fewer is refused."""
  n = smallest_n(nv)
  op = Operator(engine, kind, random_symmetric(n, n, 0.0 if kind == "stored" else 3.0))
  w, v, stats = op.solve(LARGEST, nv, nv)
  check_solve(op, LARGEST, nv, nv, w, v, stats)
  small = Operator(engine, kind, random_symmetric(n - 1, n, 0.0 if kind == "stored" else 3.0))
  with pytest.raises(nat.NativeError, match="too small for the Lanczos basis"):
    small.solve(LARGEST, nv, 0)


def test_more_than_32_values_refused(cache):
  op = random_operator(cache, "stored")
  with pytest.raises(nat.NativeError, match="n_values <= 32"):
    op.solve(LARGEST, 33, 0)


# ---------------------------------------------------------------- C. repeated eigenvalues
BLOCK_ROWS, REST = 48, 200


def repeated_matrix(m, kind):
  """kron(I_m, B) (+) 0.5 C: B the cosine affinity of 48 random d-vectors, so its top eigenvalue
  (simple) repeats exactly m times; C the affinity of 200 more, scaled so that its top eigenvalue
  equals B's, so the next eigenvalue sits at half the repeated one.  The factored Y is this matrix
  (symmetric, block diagonal) and S = Y^2 repeats the square."""
  rng = np.random.default_rng(m)
  b = orc.affinity(rng.standard_normal((BLOCK_ROWS, 16)))
  c = orc.affinity(rng.standard_normal((REST, 16)))
  top = np.linalg.eigvalsh(b)[-1]
  c *= top / np.linalg.eigvalsh(c)[-1]
  if kind == "factored":
    b, c = b.astype(np.float16).astype(np.float64), c.astype(np.float16).astype(np.float64)
  return sla.block_diag(np.kron(np.eye(m), b), 0.5 * c)


REPEATS = [(4, 4), (5, 8), (5, 5), (8, 8), (11, 12), (11, 11), (12, 12), (13, 16), (13, 13),
           (16, 16), (21, 20), (26, 20), (32, 20)]


@pytest.mark.parametrize("which", [LARGEST, SMALLEST])
@pytest.mark.parametrize("nv,m", REPEATS)
@pytest.mark.parametrize("kind", ["stored", "factored"])
def test_every_copy_of_a_repeated_value(cache, kind, nv, m, which):
  """An eigenvalue repeated m times at the wanted end (m = b and m = n_values, and m = 20 with 21
  to 32 pairs, more copies than the 16-vector block holds: in exact arithmetic its Krylov space
  sees only 16 of them, and the rest must come from rounding before the solve stops): every copy is
  found, and the vectors span the LAPACK eigenspace to 1e-8.  The smallest end is the same matrix
  with sign -1.  1e-8: sin(angle) <= |r| / gap <= tol ||T|| / (||T|| / 2) = 2e-9."""
  sign = 1.0 if which == LARGEST else -1.0
  op = cache.get(("repeated", kind, m, sign),
                 lambda: Operator(cache.engine, kind, repeated_matrix(m, kind), sign=sign))
  want = op.want(which, op.n)
  top = want[0]
  cluster = np.flatnonzero(np.abs(op.lam - top) <= 1e-10 * op.norm)
  assert len(cluster) == m and abs(want[m] - top) >= 0.4 * op.norm   # the matrix is as built
  w, v, stats = op.solve(which, nv, nv)
  check_solve(op, which, nv, nv, w, v, stats)
  found = min(m, nv)
  assert np.all(np.abs(w[:found] - top) <= TOL * op.norm + op.round)
  q = op.q[:, cluster]
  u = v[:, :found]                                  # left = right = 1: v is u
  assert np.linalg.norm(u - q @ (q.T @ u), axis=0).max() <= 1e-8
  if nv >= m:
    assert np.linalg.svd(q.T @ u, compute_uv=False).min() >= 1 - 1e-8


@pytest.mark.parametrize("diffuse,max_clusters", [(False, 21), (True, 25)])
def test_predict_finds_twenty_components(engine, diffuse, max_clusters):
  """20 well-separated speakers, no soft threshold: the refined affinity has exactly 20 connected
  components, so the Unnormalized Laplacian has eigenvalue 0 twenty times, and max_clusters=21 or
  25 asks for more pairs than the 16-vector block.  predict() must count all 20 and match the
  oracle's labels.
    * Without Diffuse (the values after the zeros are 3.27, 3.61, 3.66, then 17.2 and up) one
      Lanczos solve finds them.
    * With the ICASSP sequence, Diffuse makes every component a near-complete graph whose nonzero
      Laplacian eigenvalues crowd within 1e-2 of each other; 26 pairs do not converge to
      tol * lambda_max in 20,000 products, and predict() falls back to the dense solver."""
  x = orc.synthetic_dvectors(2000, 64, 20, seed=0, intra_cos=0.9, turn=(20, 60))
  rn = scb.RefinementName
  if diffuse:
    sequence, names = orc.ICASSP2018, list(scb.ICASSP2018_REFINEMENT_SEQUENCE)
  else:
    sequence = ("crop", "blur", "threshold", "symmetrize")
    names = [rn.CropDiagonal, rn.GaussianBlur, rn.RowWiseThreshold, rn.Symmetrize]
  opt = orc.options(sequence=sequence, mult=0.0, laplacian="unnormalized",
                    max_clusters=max_clusters)
  refined = orc.refine(orc.affinity(x), opt)
  assert connected_components(refined != 0, directed=False)[0] == 20
  c = scb.SpectralClusterer(
      max_clusters=max_clusters, laplacian_type=scb.LaplacianType.Unnormalized,
      refinement_options=scb.RefinementOptions(
          gaussian_blur_sigma=1, p_percentile=0.95, thresholding_soft_multiplier=0.0,
          refinement_sequence=names))
  labels = c.predict(x)
  if diffuse:
    assert c.last_details["solver"] == "dense"
    assert "eigenpairs converged" in c.last_details["lanczos_fallback"]
  else:
    assert c.last_details["solver"] == "lanczos" and "lanczos_fallback" not in c.last_details
  assert c.last_details["n_clusters"] == 20
  assert np.array_equal(scb.utils.enforce_ordered_labels(labels), orc.ordered(orc.predict(x, opt)))


# ---------------------------------------------------------------- D. rank deficiency
def rank5_matrix(kind, n=2000):
  """S = Y Y^T with Y made of 5 distinct integer rows, each repeated: rank 5, every entry an exact
  small integer in fp32.  Factored: the symmetric Y = Z Z^T of such a Z (exact in fp16)."""
  rng = np.random.default_rng(5)
  proto = rng.integers(-3, 4, size=(5, 8)).astype(np.float64)
  assert np.linalg.matrix_rank(proto) == 5
  z = proto[rng.integers(0, 5, size=n)]
  return z @ z.T


@pytest.mark.parametrize("kind", ["stored", "factored"])
def test_rank_deficient_single_solve(cache, kind):
  """11 pairs of a rank-5 operator: the 5 nonzero eigenvalues, then 6 values within tol * lambda_max
  (+ rounding) of 0, with orthonormal vectors and no convergence error."""
  op = cache.get(("rank5", kind), lambda: Operator(cache.engine, kind, rank5_matrix(kind)))
  w, v, stats = op.solve(LARGEST, 11, 11)
  check_solve(op, LARGEST, 11, 11, w, v, stats)
  assert np.sum(np.abs(op.lam) > 1e-6 * op.norm) == 5          # the operator is as built
  assert np.all(np.abs(w[5:]) <= TOL * op.norm + op.round)


@pytest.mark.parametrize("kind", ["stored", "factored"])
def test_rank_deficient_windows_continue_past_the_rank(cache, kind):
  """Three windows of 16 on the same operator: the first holds the 5 nonzero values, the rest are
  zeros, and the 48 locked vectors stay orthonormal."""
  op = cache.get(("rank5", kind), lambda: Operator(cache.engine, kind, rank5_matrix(kind)))
  ops = ew.DeviceOps(op.engine, op.dev, op.n, *op.terms, LARGEST, capacity=48,
                     factored=(kind == "factored"))
  ops.locked.fill_(NAN)
  found = np.concatenate([ops.window(16) for _ in range(3)])
  check_values(op, LARGEST, np.sort(found)[::-1])
  assert np.all(np.abs(found[5:]) <= TOL * op.norm + op.round)
  u = ops.locked.cpu().numpy().T
  assert np.abs(u.T @ u - np.eye(48)).max() <= 4 * (112 + 48) * op.n * U


# ---------------------------------------------------------------- E. locked windows
@pytest.mark.parametrize("kind", ["stored", "factored"])
def test_ten_windows_cross_the_lock_chunk(cache, kind):
  """Nine windows of 16 and one of 5 on n = 3000 lock 149 vectors, past the 128-vector chunk of
  the locked-set deflation.  Sorted values against LAPACK's first 149; the locked vectors
  orthonormal eigenvectors of T."""
  op = random_operator(cache, kind, n=3000)
  ops = ew.DeviceOps(op.engine, op.dev, op.n, *op.terms, LARGEST, capacity=149,
                     factored=(kind == "factored"))
  ops.locked.fill_(NAN)
  found = np.concatenate([ops.window(16) for _ in range(9)] + [ops.window(5)])
  assert ops.count == 149
  check_values(op, LARGEST, np.sort(found)[::-1])
  u = ops.locked.cpu().numpy().T
  assert np.abs(u.T @ u - np.eye(149)).max() <= 4 * (112 + 149) * op.n * U
  resid = np.linalg.norm(op.t @ u - u * found[None, :], axis=0)
  assert resid.max() <= (1 + math.sqrt(149)) * TOL * op.norm + math.sqrt(112) * op.round


@pytest.mark.parametrize("kind", ["stored", "factored"])
def test_window_at_the_basis_edge(engine, kind):
  """n = 3 * 16 + 224: the fourth window of 16 leaves exactly n - n_locked = 2 * 7 * 16 free
  directions and is accepted; the fifth is refused."""
  n = 3 * 16 + 2 * 7 * 16
  op = Operator(engine, kind, random_symmetric(n, 11, 0.0 if kind == "stored" else 3.0))
  ops = ew.DeviceOps(engine, op.dev, n, *op.terms, LARGEST, capacity=80,
                     factored=(kind == "factored"))
  ops.locked.fill_(NAN)
  found = np.concatenate([ops.window(16) for _ in range(4)])
  assert n - (ops.count - 16) == smallest_n(16)
  check_values(op, LARGEST, np.sort(found)[::-1])
  with pytest.raises(nat.NativeError, match="too small for the Lanczos basis"):
    ops.window(16)


def test_mapback_permuted_columns_with_left_ne_right(engine):
  """sc_eigh_mapback: v[:, j] = E u_{cols[j]} / |E u_{cols[j]}|, E = sqrt(left / right), against
  NumPy (each element within a few ulps: one sqrt, one division, a sum of n squares)."""
  t = dev.torch()
  rng = np.random.default_rng(4)
  n, k = 1537, 12
  u = rng.standard_normal((k, n))
  left, right = rng.uniform(0.1, 3.0, n), rng.uniform(0.1, 3.0, n)
  cols = np.array([7, 0, 11, 3, 3, 9], dtype=np.int32)
  out = t.full((n, len(cols)), NAN, dtype=t.float64, device=engine.device)
  u_d, left_d, right_d = up(u), up(left), up(right)       # alive until the call returns
  engine.call("sc_eigh_mapback", dev._ptr(u_d), n, cols.ctypes.data_as(ctypes.c_void_p),
              len(cols), dev._ptr(left_d), dev._ptr(right_d), dev._ptr(out), engine.stream)
  e = np.sqrt(left / right)
  want = (e[:, None] * u[cols].T)
  want /= np.linalg.norm(want, axis=0, keepdims=True)
  np.testing.assert_allclose(out.cpu().numpy(), want, rtol=4 * n * U, atol=0)
  got = engine.eigh_mapback(u_d, n, cols, left_d, right_d).cpu().numpy()
  np.testing.assert_array_equal(got, out.cpu().numpy())
