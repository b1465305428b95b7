"""CPU: the Krylov-Schur recurrence of arnoldi.py (thick-restart Arnoldi for the eigenvalues of
largest real part of a non-symmetric matrix) on its float64 NumPy backend, against LAPACK's dgeev
through scipy.linalg.eig, and the dgeev normalisation that lapack_real_part restates.

Error model.  u = 2^-53.  LAPACK returns the exact eigenvalues of A + E with |E|_F <= c n u |A|_F
(Householder Hessenberg reduction and Francis QR are backward stable with a modest c; c = 8 is
generous).  A computed Ritz pair (theta, x), |x| = 1, is an exact eigenpair of A - r x^H with
r = A x - theta x.  To first order an eigenvalue with left and right unit vectors y, x moves by at
most kappa |E|, kappa = 1 / |y^H x|, under a perturbation E, so
    |theta_i - lambda_i| <= kappa_i (|r_i| + c n u |A|_F),
doubled to cover the second-order term while kappa |E| stays far below the gap to the next
eigenvalue.  Where LAPACK cannot tell two eigenvalues apart (their discs of that radius overlap),
the largest kappa of the cluster bounds them all: for a semisimple eigenvalue of multiplicity k
with right and left bases X, Y (Y^H X = I) the copies move by the eigenvalues of Y^H E X, at most
|Y| |E| |X| = max kappa |E| when the copies have disjoint supports as below.
"""

import math

import numpy as np
import pytest
import scipy.linalg

from spectralcluster_b200 import arnoldi
from oracle import spectral_oracle as orc

U = 2.0 ** -53
C_LAPACK = 8
TOL = 1e-9                # the tolerance eig_extremal_device passes


def capacity(n, n_values):
  """The basis capacity eig_extremal_device chooses."""
  return n if n_values >= n else min(n, max(2 * n_values + 40, 64))


class RecordingOps(arnoldi.NumpyOps):
  """NumpyOps that records [basis size, kept columns, locked] of every restart; a restart that
  locks the converged block continues from a fresh random vector."""

  def __init__(self, matrix, cap):
    super().__init__(matrix, cap)
    self.kept = []
    self.last = None

  def rotate(self, q, next_index):
    self.kept.append([q.shape[0], q.shape[1], False])
    self.last = "rotate"
    super().rotate(q, next_index)

  def randomize(self, seed):
    if self.last == "rotate":
      self.kept[-1][2] = True
    self.last = "randomize"
    super().randomize(seed)

  def apply(self, j):
    self.last = "apply"
    super().apply(j)


def solve(a, n_values):
  n = a.shape[0]
  nv = min(n_values, n)
  cap = capacity(n, n_values)
  ops = RecordingOps(a, cap)
  res = arnoldi.krylov_schur(ops, n, nv, tol=TOL, basis=cap)
  return res, ops


def lapack(a, blocks=None):
  """(eigenvalues, kappa) of a by scipy.linalg.eig with left and right vectors; block by block
  when a is block diagonal with the given (start, stop) blocks (the spectrum is their union and a
  repeated eigenvalue spread over blocks keeps the kappa of each copy)."""
  if blocks is not None:
    parts = [lapack(a[b0:b1, b0:b1]) for b0, b1 in blocks]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
  w, vl, vr = scipy.linalg.eig(a, left=True, right=True)
  dots = np.abs(np.einsum("ij,ij->j", vl.conj(), vr))
  dots /= np.linalg.norm(vl, axis=0) * np.linalg.norm(vr, axis=0)
  return w, 1.0 / np.maximum(dots, np.finfo(float).tiny)


def check(a, n_values, res, ops, blocks=None, want_restarts=False, spectrum=None):
  n = a.shape[0]
  nv = min(n_values, n)
  assert res.converged == nv, "converged %d of %d" % (res.converged, nv)
  if want_restarts:
    assert res.restarts >= 1
  p = res.basis_size
  v = ops.v[:p]
  # Gram-Schmidt applied twice keeps the basis orthonormal to a few u per entry (a basis of at
  # most 1024 vectors of length <= 3000 whose inner products sum <= n products of unit vectors:
  # |V V^T - I| <= (n + 2 p) u < 1e-12)
  assert np.abs(v @ v.T - np.eye(p)).max() <= 1e-12
  norm_a = np.linalg.norm(a)
  a_2 = math.sqrt(np.abs(a).sum(axis=0).max() * np.abs(a).sum(axis=1).max())   # >= |A|_2
  backward = C_LAPACK * n * U * norm_a
  theta = res.values
  x = v.T @ res.coefficients
  x = x / np.linalg.norm(x, axis=0)
  resid = np.linalg.norm(a @ x - x * theta, axis=0)
  # The stopping test is |beta z_p| <= tol max|theta| and every Ritz value lies in the field of
  # values (|theta| <= |A|_2); the Arnoldi relation A V = V H + f e^T itself holds to the
  # rounding of the products and the two Gram-Schmidt sweeps, inside c n u |A|_F.
  assert np.all(resid <= TOL * a_2 + backward), resid
  lam, kappa = spectrum if spectrum is not None else lapack(a, blocks)
  # clusters LAPACK cannot resolve: eigenvalues whose discs of radius 2 kappa |E| overlap
  radius = 2 * kappa * backward
  kappa_c = np.array([kappa[np.abs(lam - lam[j]) <= radius + radius[j]].max()
                      for j in range(len(lam))])
  order = np.argsort(-lam.real, kind="stable")
  edge = lam[order[nv - 1]].real
  used = set()
  for i in range(nv):
    bound = 2 * kappa_c * (resid[i] + backward)
    dist = np.abs(lam - theta[i])
    ok = [j for j in np.argsort(dist) if j not in used and dist[j] <= bound[j]]
    assert ok, "theta[%d] = %r: nearest LAPACK value %r, bound %g" % (
        i, theta[i], lam[np.argmin(dist)], bound[np.argmin(dist)])
    j = ok[0]
    used.add(j)
    # matched by real part: every value found belongs to the wanted end of the spectrum (a tie at
    # its edge may be matched by either copy)
    assert lam[j].real >= edge - bound[j], (i, theta[i], edge)
  return x, resid


def check_restarts(ops, n_values):
  """Every thick restart keeps at least nv + max(8, nv / 2) Ritz values and every locking restart
  the nv converged ones (fewer than the basis either way), more only to keep a conjugate pair (or
  a tie) together.  Every solve that does not span the whole space ends with a locked pass."""
  for p, k, locked in ops.kept:
    base = n_values if locked else min(p - 2, n_values + max(8, n_values // 2))
    assert base <= k < p, (p, k, locked, base)


def gaussian(n, seed):
  return np.random.default_rng(seed).standard_normal((n, n)) / math.sqrt(n)


# ------------------------------------------------------------------ Gaussian random
@pytest.mark.parametrize("n,n_values", [
    (1, 1),          # one vector spans the space
    (2, 1), (2, 2),
    (6, 3), (6, 6),  # every eigenvalue
    (50, 5), (50, 50),
    (64, 5),         # n == max(2 nv + 40, 64): the Krylov space spans everything
    (65, 5)])        # one past it: a 64-vector basis with a residual coupling
def test_gaussian_small(n, n_values):
  a = gaussian(n, n)
  res, ops = solve(a, n_values)
  check(a, n_values, res, ops)
  check_restarts(ops, n_values)


@pytest.mark.parametrize("n", [300, 1024, 2000])
def test_gaussian_restarts(n):
  """The rightmost eigenvalues of a Ginibre matrix crowd the edge of the unit disc: no gap, so the
  64-vector basis restarts."""
  a = gaussian(n, n)
  res, ops = solve(a, 8)
  check(a, 8, res, ops, want_restarts=True)
  check_restarts(ops, 8)


# ------------------------------------------------------------------ conjugate pairs
def pairs_matrix(n, seed):
  """Q T Q^T, Q orthogonal, T block diagonal of 2 x 2 blocks [[a, b], [-b, a]]: every eigenvalue
  is half of a conjugate pair a +- ib, a uniform in (-1, 1], b in [0.1, 0.6)."""
  rng = np.random.default_rng(seed)
  t = np.zeros((n, n))
  for k in range(n // 2):
    re, im = 1 - 2 * k / (n // 2), 0.1 + 0.5 * rng.random()
    t[2 * k:2 * k + 2, 2 * k:2 * k + 2] = [[re, im], [-im, re]]
  q, _ = np.linalg.qr(rng.standard_normal((n, n)))
  return q @ t @ q.T


@pytest.mark.parametrize("n_values", [1, 3, 5])
def test_conjugate_pairs_cut_by_n_values(n_values):
  """n_values odd cuts the last wanted pair; the restarts keep nv + 8 (odd) Ritz values, so a pair
  of Ritz values straddles the cut and the Schur reordering must keep it whole."""
  a = pairs_matrix(400, 7)
  res, ops = solve(a, n_values)
  check(a, n_values, res, ops, want_restarts=True)
  check_restarts(ops, n_values)
  assert any(k == min(p - 2, n_values + 8) + 1 for p, k, locked in ops.kept if not locked), \
      "no restart had to extend its kept block over a conjugate pair"
  assert np.abs(res.values.imag).min() > 0.05           # every wanted value is complex


# ------------------------------------------------------------------ exact multiplicity
def thresholded_components(n, k, seed):
  """Block-diagonal [CropDiagonal, RowWiseThreshold] affinity (p = 0.95, multiplier 0.01) of k
  disconnected groups of random embeddings: the cut follows each row's own maximum, so it is not
  symmetric; every block is dense, so strongly connected."""
  rng = np.random.default_rng(seed)
  cuts = np.sort(rng.choice(np.arange(20, n - 20), k - 1, replace=False))
  bounds = np.concatenate([[0], cuts, [n]])
  blocks = list(zip(bounds[:-1], bounds[1:]))
  w = np.zeros((n, n))
  for b0, b1 in blocks:
    x = rng.standard_normal((b1 - b0, 16))
    w[b0:b1, b0:b1] = orc.row_threshold(orc.crop_diagonal(orc.affinity(x)), 0.95, 0.01)
  assert not np.array_equal(w, w.T)
  return w, blocks


@pytest.mark.parametrize("n,k", [(300, 3), (1000, 5), (3000, 8)])
def test_laplacian_zero_repeated_k_times(n, k):
  """L = D - W has eigenvalue 0 exactly k times (one per component, L 1_block = 0).  One start
  vector sees only one copy in exact arithmetic; rounding must seed the rest and every copy must
  be found: the smallest end through flip = -1, as eig_extremal_device runs it."""
  w, blocks = thresholded_components(n, k, n + k)
  a = -(np.diag(w.sum(axis=1)) - w)
  n_values = k + 2
  res, ops = solve(a, n_values)
  x, resid = check(a, n_values, res, ops, blocks=blocks)
  check_restarts(ops, n_values)
  # every copy is in the basis: the k block indicators (the null space) lie in span(V).  A Ritz
  # vector of residual r is within r / gap of the eigenspace, gap the distance from 0 to the rest
  # of the spectrum, so the cosines of the angles are >= 1 - sqrt(k) tol |A|_2 / gap
  ind = np.zeros((n, k))
  for c, (b0, b1) in enumerate(blocks):
    ind[b0:b1, c] = 1.0 / math.sqrt(b1 - b0)
  lam, _ = lapack(a, blocks)
  gap = np.sort(np.abs(lam))[k]
  a_2 = math.sqrt(np.abs(a).sum(axis=0).max() * np.abs(a).sum(axis=1).max())
  cosines = np.linalg.svd(ops.v[:res.basis_size] @ ind, compute_uv=False)
  assert cosines.min() >= 1 - math.sqrt(k) * TOL * a_2 / gap, cosines


@pytest.mark.parametrize("n,k", [(300, 3), (1000, 5), (3000, 8)])
def test_row_normalized_components_close_top_values(n, k):
  """The RowWiseNormalize form W / rowmax(W): one Perron root per block, k close but distinct."""
  w, blocks = thresholded_components(n, k, 2 * n + k)
  a = orc.row_normalize(w)
  res, ops = solve(a, k + 2)
  check(a, k + 2, res, ops, blocks=blocks)
  check_restarts(ops, k + 2)


# ------------------------------------------------------------------ invariant subspaces
def rank3(n, seed):
  """X diag(3, 2, 1) Y^T with Y^T X = I: eigenvalues 3, 2, 1 and 0 (n - 3 times, semisimple)."""
  rng = np.random.default_rng(seed)
  x = rng.standard_normal((n, 3))
  y = rng.standard_normal((n, 3))
  y = y @ np.linalg.inv(x.T @ y)
  return x @ np.diag([3.0, 2.0, 1.0]) @ y.T, x, y


@pytest.mark.parametrize("n", [50, 300])
@pytest.mark.parametrize("kind", ["rank3", "zero", "identity"])
def test_invariant_subspaces(kind, n):
  """A Krylov space that closes (beta <= 1e-12 scale) continues from a fresh random vector; the
  zero matrix closes at once, with no scale at all."""
  n_values = 3
  # exact spectra and condition numbers: the semisimple zero of the rank-3 matrix has no unique
  # left / right vectors for LAPACK to report
  if kind == "rank3":
    a, x, y = rank3(n, n)
    kappa = np.linalg.norm(x, axis=0) * np.linalg.norm(y, axis=0)     # y_i^T x_i = 1
    spectrum = (np.array([3.0, 2.0, 1.0]), kappa)
  else:
    a = np.zeros((n, n)) if kind == "zero" else np.eye(n)
    spectrum = (np.full(n, 0.0 if kind == "zero" else 1.0), np.ones(n))   # normal: kappa = 1
  res, ops = solve(a, n_values)
  check(a, n_values, res, ops, spectrum=spectrum)


# ------------------------------------------------------------------ lapack_real_part
@pytest.mark.parametrize("n", [5, 40, 200])
def test_lapack_real_part_restates_dgeev(n):
  """Eigenvectors of a random real matrix, each column multiplied by a random complex scale, come
  back as dgeev's `.real` (unit norm, component of largest modulus real) up to the sign of each
  column.  Either side rounds each component through a handful of operations (the scale, its
  inverse through the norm, the phase; about 8 roundings of u relative) and a norm summed
  pairwise (log2 n roundings): |difference| <= 2 (8 + log2 n) u per component of a unit vector."""
  rng = np.random.default_rng(n)
  for trial in range(3):
    a = rng.standard_normal((n, n))
    w, v = np.linalg.eig(a)
    assert np.abs(w.imag).max() > 0                   # complex columns are present
    scale = rng.uniform(0.1, 10.0, n) * np.exp(2j * np.pi * rng.random(n))
    got = arnoldi.lapack_real_part(v * scale)
    want = v.real
    sign = np.sign(np.einsum("ij,ij->j", got, want))
    tol = 2 * (8 + math.ceil(math.log2(n))) * U
    assert np.abs(got * sign - want).max() <= tol, (trial, np.abs(got * sign - want).max())


# ------------------------------------------------------------------ refusal
@pytest.mark.parametrize("n,n_values", [(1025, 1025), (1025, 4000), (5000, 5000)])
def test_full_spectrum_above_limit_is_refused_before_any_device_work(n, n_values):
  assert n > arnoldi.FULL_SPECTRUM_LIMIT

  class Untouchable:
    def __getattr__(self, name):
      raise AssertionError("the engine was used: %s" % name)

  with pytest.raises(NotImplementedError, match="full spectrum"):
    arnoldi.eig_extremal_device(Untouchable(), Untouchable(), n, None, None, None, 1.0, False,
                                n_values, n_values)
