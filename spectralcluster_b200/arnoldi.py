"""General (non-symmetrisable) eigen path: extremal eigenpairs of a real non-symmetric operator by
Krylov-Schur (thick-restart Arnoldi), with the reference's `.real` semantics.

The reference hands every matrix to np.linalg.eig and keeps the real parts (utils.py:59-61).  The
hot path never needs that generality -- its matrices are diagonally similar to symmetric ones
(SURVEY.md A.2) -- but sequences such as [RowWiseThreshold] alone (reference
tests/spectral_clusterer_test.py:166-184, autotune_test.py:49-52) leave a genuinely non-symmetric
matrix M = diag(delta) + sign * diag(left) S diag(right) with S itself non-symmetric.

Division of labour: every length-n operation (products with the fp32 matrix, Gram-Schmidt against
the basis, assembling Ritz vectors) is a CUDA kernel behind the C ABI (`sc_krylov_*`); this module
holds the recurrence, whose only arithmetic is on the m x m Rayleigh quotient (m <= 160): its
eigen-decomposition and, at a restart, an ordered real Schur form (scipy.linalg.schur).  `ops`
abstracts the vector backend so that the recurrence is unit-tested on the CPU with NumPy.
"""

from __future__ import annotations

import numpy as np


class Result:
  def __init__(self, values, basis_size, coefficients, matvecs, restarts, converged):
    self.values = values                # complex Ritz values, ordered (wanted end first)
    self.basis_size = basis_size        # P: the Ritz vectors are V[:P] @ coefficients
    self.coefficients = coefficients    # complex [P, n_values]
    # restarts counts the locking restarts too
    self.matvecs, self.restarts, self.converged = matvecs, restarts, converged


def krylov_schur(ops, n: int, n_values: int, tol: float = 1e-9, basis: int = 0,
                 max_matvecs: int = 20000) -> Result:
  """The `n_values` eigenvalues of largest REAL PART of the operator behind `ops`.

  ops.apply(j) -> None          w <- Op V[j]
  ops.orthogonalize(count)      w <- (I - V V^T)^2 w over V[:count]; returns (h[count], |w|^2)
  ops.store(j, alpha)           V[j] <- alpha * w
  ops.randomize(seed)           w <- pseudo-random vector
  ops.rotate(q, next_index)     V[:k] <- V[:P] q (q is [P, k]);  V[k] <- V[next_index]
  """
  full = n <= max(basis, 2 * n_values + 40, 64)        # the Krylov space can span everything
  m = n if full else max(basis, 2 * n_values + 40, 64)
  h = np.zeros((m + 1, m))
  seed = 1

  def fresh(j):
    nonlocal seed
    ops.randomize(seed)
    seed += 1
    _, nrm2 = ops.orthogonalize(j)
    ops.store(j, 1.0 / np.sqrt(nrm2))

  def schur_keep(hm, theta, keep, ref):
    """Ordered real Schur form of hm whose leading block holds the `keep` Ritz values of largest
    real part, more if the cut would split a conjugate pair (or a tie)."""
    import scipy.linalg
    p = hm.shape[0]
    re_sorted = np.sort(theta.real)[::-1]
    while keep < p - 1 and abs(re_sorted[keep - 1] - re_sorted[keep]) <= 1e-14 * ref:
      keep += 1                                        # never split a conjugate pair
    cut = 0.5 * (re_sorted[keep - 1] + re_sorted[keep])
    t, q, sdim = scipy.linalg.schur(hm, output="real", sort=lambda re, im: re > cut)
    if sdim < 1 or sdim >= p:
      raise RuntimeError("krylov_schur: Schur reordering kept %d of %d" % (sdim, p))
    return t, q, sdim

  fresh(0)
  p, matvecs, restarts, converged = 0, 0, 0, 0
  values = coeffs = None
  # Locking.  One start vector sees a single copy of a repeated eigenvalue in exact arithmetic;
  # rounding seeds the other copies only slowly, so the wanted set can converge without them.
  # Once it has converged, its Schur vectors are locked: their residual coupling (each Ritz
  # vector's share of it within the tolerance) is dropped from H and kept in `drop`, one row per
  # lock in the coordinates of the current basis, and the basis continues from a fresh random
  # vector orthogonal to them, i.e. Arnoldi on the complement.  A copy that was missing enters the
  # wanted set there; the solve ends when such a pass adds nothing to it.  A Ritz pair (theta, V z)
  # has the residual |coupling z[p-1]| + sum_l |drop_l . z|.
  drop, probed = np.zeros((0, m)), None
  while True:
    j = p
    while j < m:
      ops.apply(j)
      matvecs += 1
      coef, nrm2 = ops.orthogonalize(j + 1)
      h[:j + 1, j] = coef
      beta = float(np.sqrt(nrm2))
      scale = max(float(np.abs(coef).max()), 1e-300)
      if j + 1 == n:                                   # the basis spans the whole space
        j += 1
        break
      if beta > 1e-12 * scale:
        h[j + 1, j] = beta
        ops.store(j + 1, 1.0 / beta)
      else:                                            # invariant subspace: continue orthogonally
        h[j + 1, j] = 0.0
        fresh(j + 1)
      j += 1
    p = j
    hm = h[:p, :p]
    theta, z = np.linalg.eig(hm)
    order = np.argsort(-theta.real, kind="stable")
    theta, z = theta[order], z[:, order]
    coupling = h[p, p - 1] if p < n else 0.0           # residual_i = |coupling * z[p-1, i]|
    resid = np.abs(coupling * z[p - 1, :]) + np.abs(drop[:, :p] @ z).sum(axis=0)
    ref = max(float(np.abs(theta).max()), 1e-300)
    converged = 0
    for i in range(min(n_values, p)):
      if resid[i] <= tol * ref:
        converged += 1
      else:
        break
    values, coeffs = theta[:n_values], z[:, :n_values]
    done = converged >= min(n_values, p)
    if p >= n or matvecs >= max_matvecs:
      break
    if done and (probed is not None and values[-1].real <= probed + tol * ref or
                 theta[-1].real >= values[-1].real - 1e-14 * ref):
      break            # the locked pass found nothing new, or nothing else is there to find
    # ---- thick restart (or, once converged, locking): ordered real Schur form, keep the
    # leading block
    keep = n_values if done else min(p - 2, n_values + max(8, n_values // 2))
    t, q, sdim = schur_keep(hm, theta, keep, ref)
    row = coupling * q[p - 1, :sdim]
    ops.rotate(np.ascontiguousarray(q[:, :sdim]), p)
    kept = drop[:, :p] @ q[:, :sdim]
    drop = np.zeros((len(kept) + done, m))
    drop[:len(kept), :sdim] = kept
    h[:, :] = 0.0
    h[:sdim, :sdim] = t[:sdim, :sdim]
    if done:
      drop[-1, :sdim] = row
      probed = values[-1].real
      fresh(sdim)
    else:
      h[sdim, :sdim] = row
    p = sdim
    restarts += 1
  return Result(values, p, coeffs, matvecs, restarts, converged)


class NumpyOps:
  """Reference vector backend (CPU tests of the recurrence)."""

  def __init__(self, matrix, capacity):
    self.a = np.asarray(matrix, dtype=np.float64)
    n = self.a.shape[0]
    self.v = np.zeros((capacity + 1, n))
    self.w = np.zeros(n)

  def apply(self, j):
    self.w = self.a @ self.v[j]

  def orthogonalize(self, count):
    h = np.zeros(count)
    for _ in range(2):
      c = self.v[:count] @ self.w
      self.w = self.w - self.v[:count].T @ c
      h += c
    return h, float(self.w @ self.w)

  def store(self, j, alpha):
    self.v[j] = alpha * self.w

  def randomize(self, seed):
    self.w = np.random.default_rng(seed).standard_normal(self.a.shape[0])

  def rotate(self, q, next_index):
    k = q.shape[1]
    nxt = self.v[next_index].copy()
    self.v[:k] = q.T @ self.v[:q.shape[0]]
    self.v[k] = nxt


def lapack_real_part(vectors: np.ndarray) -> np.ndarray:
  """Real parts of complex eigenvectors under dgeev's normalisation (unit 2-norm, component of
  largest magnitude real) -- what `eigenvectors.real` (utils.py:61) sees."""
  out = np.empty(vectors.shape, dtype=np.float64)
  for c in range(vectors.shape[1]):
    v = vectors[:, c] / np.linalg.norm(vectors[:, c])
    if np.iscomplexobj(v) and np.abs(v.imag).max() > 0:
      big = v[np.argmax(np.abs(v))]
      v = v * (np.conj(big) / abs(big))
    out[:, c] = v.real
  return out


class DeviceOps:
  """CUDA vector backend over the C ABI (`sc_krylov_*`): the operator is
  x -> flip * (delta .* x + sign * left .* (S (right .* x))) with S an fp32 device matrix."""

  def __init__(self, eng, s, n, delta, left, right, sign, flip, capacity):
    import ctypes
    from . import device as dev
    self.eng, self.s, self.n = eng, s, n
    self.delta, self.left, self.right, self.sign, self.flip = delta, left, right, sign, flip
    self.t = dev.torch()
    self.ptr, self.ct = dev._ptr, ctypes
    f64 = self.t.float64
    self.v = self.t.zeros((capacity + 1, n), dtype=f64, device=eng.device)
    self.v2 = self.t.zeros((capacity + 1, n), dtype=f64, device=eng.device)
    self.w = self.t.zeros((n,), dtype=f64, device=eng.device)
    self.y = self.t.zeros((n,), dtype=f64, device=eng.device)

  def apply(self, j):
    x = self.v[j]
    tvec = x * self.right if self.right is not None else x
    self.eng.call("sc_krylov_matvec", self.ptr(self.s), self.n, self.n, self.s.stride(0),
                  self.ptr(tvec.contiguous()), self.ptr(self.y), self.eng.stream)
    y = self.y * self.left if self.left is not None else self.y
    w = self.sign * y
    if self.delta is not None:
      w = w + self.delta * x
    self.w.copy_(self.flip * w)

  def orthogonalize(self, count):
    h = np.zeros(max(count, 1), dtype=np.float64)
    nrm2 = self.ct.c_double(0.0)
    self.eng.call("sc_krylov_orthogonalize", self.ptr(self.v), self.n, count, self.ptr(self.w),
                  h.ctypes.data_as(self.ct.c_void_p), self.ct.byref(nrm2), self.eng.stream)
    return h[:count], float(nrm2.value)

  def store(self, j, alpha):
    self.eng.call("sc_krylov_scale", self.ptr(self.w), self.n, float(alpha), self.ptr(self.v[j]),
                  self.eng.stream)

  def randomize(self, seed):
    self.eng.call("sc_krylov_random", self.ptr(self.w), self.n, int(seed), self.eng.stream)

  def _combine(self, coeffs, count, out):
    """out[:k] <- V[:count] @ coeffs (real [count, k]), 64 columns at a time."""
    k = coeffs.shape[1]
    for c0 in range(0, k, 64):
      z = np.ascontiguousarray(coeffs[:, c0:c0 + 64], dtype=np.float64)
      self.eng.call("sc_krylov_combine", self.ptr(self.v), self.n, count,
                    z.ctypes.data_as(self.ct.c_void_p), z.shape[1], self.ptr(out[c0]),
                    self.eng.stream)

  def rotate(self, q, next_index):
    k = q.shape[1]
    self._combine(q, q.shape[0], self.v2)
    self.v2[k].copy_(self.v[next_index])
    self.v, self.v2 = self.v2, self.v

  def ritz_vectors(self, coeffs, count):
    """Unit-norm real parts of V[:count] @ coeffs as a row-major device [n, k] fp64 array
    (eigenvectors.real of utils.py:61 under LAPACK's normalisation)."""
    k = coeffs.shape[1]
    out = self.t.empty((self.n, k), dtype=self.t.float64, device=self.eng.device)
    u = self.t.empty((k, self.n), dtype=self.t.float64, device=self.eng.device)
    self._combine(np.ascontiguousarray(coeffs.real), count, u)
    complex_cols = [c for c in range(k) if np.abs(coeffs[:, c].imag).max() > 0]
    if complex_cols:
      # rare: a wanted Ritz pair is complex.  Its imaginary part is assembled too and the dgeev
      # phase convention applied on the host copy of just those columns.
      ui = self.t.empty((len(complex_cols), self.n), dtype=self.t.float64, device=self.eng.device)
      self._combine(np.ascontiguousarray(coeffs[:, complex_cols].imag), count, ui)
      vec = u[complex_cols].cpu().numpy().T + 1j * ui.cpu().numpy().T
      u[complex_cols] = self.t.from_numpy(lapack_real_part(vec).T.copy()).to(self.eng.device)
    self.eng.call("sc_krylov_columns", self.ptr(u), self.n, k, self.ptr(out), self.eng.stream)
    if complex_cols:        # the real part of a unit complex vector is not a unit vector: undo
      scale = self.t.from_numpy(np.linalg.norm(lapack_real_part(vec), axis=0)).to(self.eng.device)
      out[:, complex_cols] *= scale
    return out


FULL_SPECTRUM_LIMIT = 1024      # max n for which every eigenvalue may be requested on this path


def eig_extremal_device(eng, s, n, delta, left, right, sign, smallest, n_values, n_vectors,
                        tol=1e-9):
  """(real parts of the n_values extremal eigenvalues, device [n, n_vectors] eigenvectors, stats)
  of M = diag(delta) + sign diag(left) S diag(right), S a general fp32 device matrix."""
  flip = -1.0 if smallest else 1.0
  capacity = n if n_values >= n else min(n, max(2 * n_values + 40, 64))
  if n_values >= n and n > FULL_SPECTRUM_LIMIT:
    raise NotImplementedError(
        "the full spectrum of a non-symmetrisable %d x %d matrix (max_clusters=None) is outside "
        "the device path; set max_clusters" % (n, n))
  ops = DeviceOps(eng, s, n, delta, left, right, sign, flip, capacity)
  res = krylov_schur(ops, n, min(n_values, n), tol=tol, basis=capacity)
  if res.converged < min(n_values, res.basis_size) and res.basis_size < n:
    raise RuntimeError("general eigensolver: %d of %d eigenpairs converged in %d products"
                       % (res.converged, n_values, res.matvecs))
  w = flip * res.values.real
  v = ops.ritz_vectors(res.coefficients[:, :n_vectors], res.basis_size) if n_vectors else None
  return w, v, [res.matvecs, res.restarts, res.converged, res.basis_size]
