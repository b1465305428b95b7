"""Eigenvalue prefixes for max_clusters=None (and max_clusters >= 32) above the dense solver's N.

utils.compute_number_of_clusters (reference utils.py:74-130) scans the whole sorted spectrum when
max_clusters is None, but only a prefix of it can change its answer:

  * descending (no Laplacian, or LaplacianType.Affinity): the scan stops at the first value below
    stop_eigenvalue, so the prefix up to and including that value decides k (NormalizedDiff
    normalises by w[0], the first value of the prefix);
  * ascending (any Laplacian): with the m smallest values w[0..m-1] and lambda_max known and
    w[m-1] + eps > 0, every later index i >= m-1 has
        Ratio           w[i+1] / (w[i] + eps)      <= lambda_max / (w[m-1] + eps)
        NormalizedDiff  (w[i+1] - w[i]) / lambda_max <= (lambda_max - w[m-1]) / lambda_max,
    and a later index replaces the running best only when strictly greater, so once the best gap
    over the exact indices 1 .. m-2 exceeds that bound, k and the gap are final.

Such a prefix is "settled".  `solve` grows the prefix a window of WINDOW_PAIRS eigenpairs at a
time until it is: on the device each window is a block Lanczos solve on the complement of the
pairs already found (sc_eigh_extremal_locked, or sc_eigh_extremal_locked_factored on the factored
operator), on the CPU a NumPy backend stands in (tests).
`grow_krylov_schur` applies the same rule to the general (non-symmetrisable) path, whose
Krylov-Schur solver is restarted with twice the pairs until the prefix settles.
"""

from __future__ import annotations

import typing

import numpy as np

from . import utils

WINDOW_PAIRS = 16             # eigenpairs per window: one 16-vector block product per pass over S
MAX_WINDOW_PAIRS = 512        # most eigenpairs a windowed solve finds before it gives up
SETTLE_RTOL = 1e-5            # relative eigenvalue tolerance: a near tie asks for another window
GROW_START, GROW_CAP = 16, 256   # Krylov-Schur pairs: first solve, most before it gives up
# Lanczos basis of one window (sc_eigh_extremal_locked*): a 16-vector block, six blocks processed
# before a thick restart plus the block being processed.  A window needs
# n - (vectors already locked) >= 2 x this basis.
WINDOW_BASIS = 7 * WINDOW_PAIRS


def capacity(n: int, max_clusters, min_clusters) -> int:
  """Rows of the locked set of a windowed solve: the eigenvalues it may need (all n when
  max_clusters is None, capped at MAX_WINDOW_PAIRS), plus one window that may overshoot them."""
  limit = min(n, max_clusters + 1) if max_clusters else n
  return min(n, MAX_WINDOW_PAIRS, max(limit, min_clusters or 0) + WINDOW_PAIRS)


def settled(prefix, descend: bool, max_clusters: typing.Optional[int], stop_eigenvalue: float,
            eigengap_type, lambda_max: typing.Optional[float]) -> bool:
  """Whether compute_number_of_clusters on the sorted `prefix` equals it on the whole spectrum
  (same k, same gap).  `lambda_max` is the spectrum's largest value; only ascending spectra use it.
  Decisions need a margin of SETTLE_RTOL, so values that tie up to rounding ask for more."""
  w = np.asarray(prefix, dtype=np.float64)
  m = len(w)
  if max_clusters and m >= max_clusters + 1:
    return True                         # the scan never reads past w[max_clusters]
  if descend:
    return bool(np.any(w < stop_eigenvalue - SETTLE_RTOL * abs(stop_eigenvalue)))
  if m < 3 or lambda_max is None or not lambda_max > 0:
    return False
  floor = w[-1] + utils.EPS
  if not floor > 0:
    return False
  if eigengap_type == utils.EigenGapType.Ratio:
    bound = lambda_max / floor
  else:
    bound = (lambda_max - w[-1]) / lambda_max
  _, widest = utils.compute_number_of_clusters(w, max_clusters=max_clusters,
                                               eigengap_type=eigengap_type, descend=False,
                                               max_eigenvalue=lambda_max)
  return bool(widest > bound + SETTLE_RTOL * abs(bound))


def _cap_error(max_clusters, cap):
  if max_clusters:
    return NotImplementedError(
        "max_clusters=%d needs %d eigenpairs, more than the windowed eigensolver finds "
        "(MAX_WINDOW_PAIRS = %d)" % (max_clusters, max_clusters + 1, cap))
  return NotImplementedError(
      "max_clusters=None: the eigengap is not settled within the first %d eigenvalues "
      "(MAX_WINDOW_PAIRS); set max_clusters" % cap)


class Prefix:
  def __init__(self, values, order, lambda_max, windows):
    self.values = values          # sorted as the reference sorts, wanted end first
    self.order = order            # values[j] was found as pair order[j] (the ops' numbering)
    self.lambda_max = lambda_max  # largest eigenvalue (ascending spectra), else None
    self.windows = windows


def solve(ops, descend: bool, max_clusters, min_clusters, stop_eigenvalue, eigengap_type,
          n: typing.Optional[int] = None) -> Prefix:
  """Windows of eigenpairs until the prefix decides the eigengap.

  ops.window(count) -> the next `count` eigenvalues at the wanted end (fewer only when the
                       spectrum is exhausted); the ops keep the vectors, numbered as found
  ops.lambda_max()  -> the largest eigenvalue (ascending spectra only)

  A bounded solve (max_clusters set) returns max_clusters + 1 values, as every other route does;
  an unbounded one stops as soon as the prefix is settled.  Either also covers min_clusters
  columns.  More than MAX_WINDOW_PAIRS values needed -> NotImplementedError."""
  cap = MAX_WINDOW_PAIRS
  need = max(min_clusters or 0, 1)
  if max_clusters:
    need = max(need, max_clusters + 1)
  if n is not None:
    need = min(need, n)
  ndiff = eigengap_type == utils.EigenGapType.NormalizedDiff
  lam = None
  found: typing.List[float] = []
  windows = 0
  while True:
    if len(found) >= cap:
      raise _cap_error(max_clusters, cap)
    count = min(WINDOW_PAIRS, cap - len(found))
    got = np.asarray(ops.window(count), dtype=np.float64)
    windows += 1
    found.extend(got.tolist())
    values = np.asarray(found)
    order = np.argsort(-values if descend else values, kind="stable")
    prefix = values[order]
    if not descend and lam is None and (ndiff or not max_clusters):
      lam = float(ops.lambda_max())
    if len(got) < count:                # the whole spectrum is in the prefix
      break
    if len(prefix) < need:
      continue
    if max_clusters or settled(prefix, descend, None, stop_eigenvalue, eigengap_type,
                               prefix[0] if descend else lam):
      break
  return Prefix(prefix, order, lam, windows)


class NumpyOps:
  """Reference backend (CPU tests): exact windows of a symmetric matrix restricted to the
  complement of the pairs already found."""

  def __init__(self, matrix, descend: bool):
    self.a = np.asarray(matrix, dtype=np.float64)
    self.descend = descend
    self.u = np.zeros((self.a.shape[0], 0))

  def window(self, count):
    n = self.a.shape[0]
    if self.u.shape[1]:
      q = np.linalg.svd(np.eye(n) - self.u @ self.u.T)[0][:, :n - self.u.shape[1]]
    else:
      q = np.eye(n)
    w, z = np.linalg.eigh(q.T @ self.a @ q)
    idx = np.argsort(-w if self.descend else w, kind="stable")[:count]
    self.u = np.concatenate([self.u, q @ z[:, idx]], axis=1)
    return w[idx]

  def lambda_max(self):
    return float(np.linalg.eigvalsh(self.a)[-1])

  def vectors(self, cols):
    return self.u[:, np.asarray(cols)]


class DeviceOps:
  """Windows on the device: sc_eigh_extremal_locked on the implicit operator
  diag(delta) + sign * diag(left) S diag(right), its Ritz vectors kept in HBM.  `factored`: `s` is
  the fp16 Y_hi of S = Y_hi Y_hi^T, never formed, and the windows and the lambda_max solve run on
  the factored operator (sc_eigh_extremal_locked_factored, sc_eigh_extremal_factored)."""

  def __init__(self, eng, s, n, delta, left, right, sign, which, capacity, factored=False):
    from . import device as dev
    from . import _native as nat
    t = dev.torch()
    self.eng, self.op, self.which, self.largest = eng, (s, n, delta, left, right, sign), which, nat.EIG_LARGEST
    # Engine.eigh_window picks the locked entry from the operand's dtype (fp16: Y_hi)
    assert not factored or s.dtype == t.float16
    self.factored = factored
    self.locked = t.empty((capacity, n), dtype=t.float64, device=eng.device)
    self.count, self.scale = 0, 0.0
    self.stats = dict(windows=0, passes=0, matvecs=0, restarts=0)

  def window(self, count):
    w, st = self.eng.eigh_window(*self.op, self.which, count, self.locked, self.count, self.scale)
    self.count += count
    self.scale = max(self.scale, float(np.abs(w).max()))
    self.stats["windows"] += 1
    self.stats["matvecs"] += int(st[0])
    self.stats["restarts"] += int(st[1])
    self.stats["passes"] += int(st[3])
    return w

  def lambda_max(self):
    if self.factored:
      w, _, st = self.eng.eigh_factored(*self.op, self.largest, 1, 0)
    else:
      w, _, st = self.eng.eigh(*self.op, self.largest, 1, 0, False)
    self.scale = max(self.scale, abs(float(w[0])))
    self.stats["passes"] += int(st[3])
    return float(w[0])

  def vectors(self, cols):
    s, n, delta, left, right, sign = self.op
    return self.eng.eigh_mapback(self.locked, n, cols, left, right)


def grow_krylov_schur(eng, op, descend: bool, min_clusters, stop_eigenvalue, eigengap_type):
  """The general (non-symmetrisable) path with max_clusters=None: Krylov-Schur for GROW_START
  pairs, doubled until the real parts settle (the bounds above use only their order and
  lambda_max) -> (values, device vectors, stats, lambda_max or None)."""
  from . import arnoldi
  lam = None
  count = max(GROW_START, min_clusters or 0)
  while True:
    w, v, stats = arnoldi.eig_extremal_device(eng, *op, not descend, count, count)
    if not descend and lam is None:
      lam = float(arnoldi.eig_extremal_device(eng, *op, False, 1, 0)[0][0])
    if settled(w, descend, None, stop_eigenvalue, eigengap_type, w[0] if descend else lam):
      return w, v, stats, lam
    if count >= GROW_CAP:
      raise NotImplementedError(
          "max_clusters=None: the eigengap of a non-symmetrisable matrix is not settled within "
          "the first %d eigenvalues (GROW_CAP); set max_clusters" % GROW_CAP)
    count = min(2 * count, GROW_CAP)
