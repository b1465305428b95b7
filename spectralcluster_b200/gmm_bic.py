"""The AffinityGmmBic single-cluster check (fallback_clusterer.py:158-178) as a streaming
recurrence: scikit-learn 1.9.0's GaussianMixture(n_components=1) and (n_components=2), default
options, fitted to the strict upper band `affinity[np.triu_indices(n, offset)]`, and their BICs.

The samples are never gathered.  Every step of KMeans initialisation, EM and scoring is one
reduction over the band, done by a backend (`ops`); this module holds the O(1) state between
reductions (centres, parameters, sums) and restates scikit-learn's control flow around them:

  * KMeans(n_clusters=c, n_init=1, random_state=<global RandomState>) (mixture/_base.py:119-128):
    samples centred by their mean (cluster/_kmeans.py:1486-1493); k-means++ with 2 + int(log c)
    local trials (:180-278) on expanded-form squared distances x^2 - 2xc + c^2 clipped at 0;
    Lloyd (:630-758) with labels argmin(c^2 - 2xc), first minimum winning, stopping on unchanged
    labels or center_shift_tot <= var * 1e-4 (:285-292), then one final assignment unless the
    stop was strict.  In 1-D "labels unchanged" is counted in one pass by evaluating the rule
    under the previous and the current centres, so no per-sample labels are stored.
  * Initial parameters from the one-hot labels, EM with tol 1e-3 and max_iter 100, reg_covar
    1e-6, nk + 10 eps (mixture/_gaussian_mixture.py:282-320, 490-553, 849-898; _base.py:251-312).
  * bic = -2 score m + p log m with p = 2 and 5, the score under the final parameters (:945-980).

Random draws come from the global np.random state in scikit-learn's order, so the caller's stream
advances exactly as scikit-learn advances it: random_sample() for GMM-1's first centre,
random_sample() for GMM-2's first centre, uniform(size=2) for GMM-2's local trials.

Second moments are taken about a shift close to the mean (the previous mean, the Lloyd centre) and
moved to the mean exactly: sum r (x - mu)^2 = Q - 2 (mu - s) (R1 - s R0) + (mu - s)^2 R0.

`NumpyOps` evaluates each reduction on a host copy of the band with NumPy in scikit-learn's order
(the CPU tests compare the recurrence with scikit-learn itself); `DeviceOps` calls
`sc_gmm_band_pass`, one streaming pass over the fp32 device matrix, or `sc_gmm_band_pass_packed`
over the packed band (`packed_row_offsets`) of an affinity that is never stored; both return the
same sums bit for bit.
"""

from __future__ import annotations

import bisect
import ctypes
import math
import warnings

import numpy as np

EPS10 = 10 * np.finfo(np.float64).eps
REG_COVAR = 1e-6
EM_TOL, EM_MAX_ITER = 1e-3, 100
KMEANS_TOL, KMEANS_MAX_ITER = 1e-4, 300
LOG_2PI = math.log(2 * math.pi)

# modes of sc_gmm_band_pass (include/spectralcluster_b200.h)
MOMENTS, KPP, LOOKUP, LLOYD, LABELS, EM, SCORE = range(7)


# ---- the band np.triu_indices(n, offset), row-major -----------------------------------------
def band_rows(n: int, offset: int) -> int:
  """Number of rows with at least one band element."""
  return max(0, min(n, n - offset))


def band_start(n: int, offset: int, i: int) -> int:
  """Flat index of the first band element of row i (= band size for i >= band_rows)."""
  full = min(max(-offset, 0), n)               # rows whose band starts at column 0
  a = min(i, full)
  b = min(i, band_rows(n, offset))
  s = a * n
  if b > a:
    s += (b - a) * (n - offset) - (b * (b - 1) // 2 - a * (a - 1) // 2)
  return s


def band_size(n: int, offset: int) -> int:
  return band_start(n, offset, n)


def band_position(n: int, offset: int, idx: int):
  """(i, j) of flat band index idx: np.triu_indices(n, offset)[0][idx], [1][idx]."""
  lo, hi = 0, band_rows(n, offset) - 1
  while lo < hi:                               # last row whose start is <= idx
    mid = (lo + hi + 1) // 2
    if band_start(n, offset, mid) <= idx:
      lo = mid
    else:
      hi = mid - 1
  return lo, max(0, lo + offset) + idx - band_start(n, offset, lo)


def packed_row_offsets(n: int, offset: int) -> np.ndarray:
  """row_off [n + 1] (int64) of the packed band: row i (j0 = max(0, i + offset) < n) keeps columns
  [c0, n), c0 = j0 & ~3, at band[row_off[i] ...], padded to a multiple of 4 so that column j sits
  at the position mod 4 it has in a dense matrix with ld % 4 == 0; rows without band elements take
  no room.  row_off[n] is the packed length in elements."""
  j0 = np.maximum(np.arange(n, dtype=np.int64) + offset, 0)
  width = np.where(j0 < n, (n - (j0 & ~3) + 3) & ~3, 0)
  out = np.zeros(n + 1, dtype=np.int64)
  np.cumsum(width, out=out[1:])
  return out


# ---- RandomState.choice(m, p=uniform) without m values ------------------------------------------
class UniformChoice:
  """numpy's `choice(m, p=np.full(m, 1 / m))` is `searchsorted(cumsum(p) / cumsum(p)[-1], u,
  'right')` with the sequential fp64 cumsum of m copies of p = fl(1 / m).  Within one binade of
  the running sum every addition rounds the same way (a tie can change only the first step), so
  the running sum is piecewise arithmetic: a handful of segments per binade, built in O(log m).
  `index(u)` binary-searches the normalised sum, as numpy does, without materialising it."""

  def __init__(self, m: int):
    self.m = m
    p = 1.0 / m
    self.starts, self.segs = [], []            # segment k covers indices starts[k] .. + count - 1
    i, s = 0, p
    self._add(0, p, 0.0, 1)
    while i + 1 < m:
      top = math.ldexp(1.0, math.frexp(s)[1])  # the binade of s is [top / 2, top)
      t1 = s + p
      if t1 >= top or i + 2 >= m:
        self._add(i + 1, t1, 0.0, 1)
        i, s = i + 1, t1
        continue
      t2 = t1 + p
      if t2 >= top:
        self._add(i + 1, t1, 0.0, 1)
        i, s = i + 1, t1
        continue
      delta = t2 - t1                          # every later step in this binade adds delta
      ulp = math.ulp(t1)
      steps = -(-round((top - t1) / ulp) // round(delta / ulp))   # t1 + k delta < top
      steps = min(steps, m - 1 - i)
      self._add(i + 1, t1, delta, steps)
      i, s = i + steps, t1 + (steps - 1) * delta
    self.total = self.cum(m - 1)

  def _add(self, start, value, delta, count):
    self.starts.append(start)
    self.segs.append((start, value, delta, count))

  def cum(self, i: int) -> float:
    """The i-th element of np.cumsum(np.full(m, 1 / m))."""
    start, value, delta, _ = self.segs[bisect.bisect_right(self.starts, i) - 1]
    return value + (i - start) * delta

  def index(self, u: float) -> int:
    lo, hi = 0, self.m                         # count of i with cum(i) / total <= u
    while lo < hi:
      mid = (lo + hi) // 2
      if self.cum(mid) / self.total <= u:
        lo = mid + 1
      else:
        hi = mid
    return lo


# ---- the recurrence ------------------------------------------------------------------------------
class Fit:
  """One fitted GaussianMixture: parameters, n_iter_, converged_, its BIC and its KMeans init."""

  def __init__(self, weights, means, covariances, n_iter, converged, bic, kmeans_centres):
    self.weights, self.means, self.covariances = weights, means, covariances
    self.n_iter, self.converged, self.bic = n_iter, converged, bic
    self.kmeans_centres = kmeans_centres       # centred centres of the final KMeans assignment


class Result:
  def __init__(self, single, fits, mean, passes):
    self.single = single                       # bic1 < bic2
    self.fits = fits                           # [GMM-1, GMM-2]
    self.kmeans_mean = mean                    # the mean KMeans centres the samples by
    self.passes = passes                       # band reductions run

  @property
  def bic(self):
    return [f.bic for f in self.fits]

  @property
  def n_iter(self):
    return [f.n_iter for f in self.fits]


def _deviation(q, r0, r1, mu, s):
  """sum r (x - mu)^2 from Q = sum r (x - s)^2, R1 = sum r x, R0 = sum r."""
  d = mu - s
  return q - 2.0 * d * (r1 - s * r0) + d * d * r0


def _params(nk, means, dev):
  cov = [dv / k + REG_COVAR for dv, k in zip(dev, nk)]
  if any(not c > 0.0 for c in cov):
    raise ValueError("Fitting the mixture model failed because some components have ill-defined "
                     "empirical covariance (for instance caused by singleton or collapsed "
                     "samples). Try to decrease the number of components, increase reg_covar, "
                     "or scale the input data.")
  return cov


def _em_args(weights, means, cov):
  """Per component: log weight, mu * pc, pc, log pc, shift (= mu) for the EM / score pass."""
  out = []
  for w, mu, c in zip(weights, means, cov):
    pc = 1.0 / math.sqrt(c)                    # cholesky(cov) -> solve(L, I).T in 1-D
    out.append((math.log(w) if w > 0 else -math.inf, mu * pc, pc, math.log(pc), mu))
  return out


def _kmeans2(ops, mean, tol, draws):
  """Centred centres of the final Lloyd assignment of KMeans(2)."""
  m = ops.m
  u0 = draws.random_sample()
  c0 = ops.values([UniformChoice(m).index(u0)])[0] - mean
  pot = ops.kpp(mean, c0)[0]
  rand_vals = draws.uniform(size=2) * pot
  vals = ops.kpp_lookup(mean, c0, rand_vals)
  cand = [v - mean for v in vals]
  pots = ops.kpp(mean, c0, cand[0], cand[1])[1:]
  centres = (c0, cand[0] if pots[0] <= pots[1] else cand[1])
  old = None
  for _ in range(KMEANS_MAX_ITER):
    count1, s0, s1, changed = ops.lloyd(mean, centres, old)
    count0 = m - count1
    if count0 == 0 or count1 == 0:
      # In 1-D a side empties only for constant samples: both centres are the one value, so
      # every sample keeps label 0 whatever the empty-cluster relocation moves, and the next
      # iteration stops strictly with these labels.
      return centres
    if old is not None and changed == 0:
      return centres                           # strict convergence: labels under these centres
    new = (s0 / count0, s1 / count1)
    shift = (new[0] - centres[0]) ** 2 + (new[1] - centres[1]) ** 2
    old, centres = centres, new
    if shift <= tol:
      break
  return centres                               # the final assignment runs under the new centres


def _fit(ops, c, mean, moments, tol, draws):
  """GaussianMixture(n_components=c).fit on the band; `moments` = (count, sum(x - mean),
  sum (x - mean)^2) from the validation passes."""
  from sklearn.exceptions import ConvergenceWarning
  m = ops.m
  if c == 1:
    draws.random_sample()                      # KMeans(1)'s first centre: every label is 0
    _, d1, q = moments
    r0, r1 = [float(m)], [d1 + mean * m]
    qs, shifts = [q], [mean]
    centres = (0.0,)
  else:
    centres = _kmeans2(ops, mean, tol, draws)
    shifts = [centres[0] + mean, centres[1] + mean]
    count1, s0, s1, q0, q1 = ops.label_moments(mean, centres, shifts)
    r0 = [float(m - count1), float(count1)]
    r1, qs = [s0, s1], [q0, q1]
    if count1 == 0 or count1 == m:
      warnings.warn("Number of distinct clusters (1) found smaller than n_clusters (2). "
                    "Possibly due to duplicate points in X.", ConvergenceWarning, stacklevel=3)
  nk = [k + EPS10 for k in r0]
  means = [s / k for s, k in zip(r1, nk)]
  cov = _params(nk, means, [_deviation(q, a, b, mu, s)
                            for q, a, b, mu, s in zip(qs, r0, r1, means, shifts)])
  weights = [k / m for k in nk]                # initial weights: nk / n_samples
  lower = -math.inf
  converged = False
  for n_iter in range(1, EM_MAX_ITER + 1):
    prev = lower
    slse, mom = ops.em(_em_args(weights, means, cov))
    lower = slse / m
    nk = [mm[0] + EPS10 for mm in mom]
    new_means = [mm[1] / k for mm, k in zip(mom, nk)]
    cov = _params(nk, new_means, [_deviation(mm[2], mm[0], mm[1], mu, s)
                                  for mm, mu, s in zip(mom, new_means, means)])
    means = new_means
    total = sum(nk)
    weights = [k / total for k in nk]
    if abs(lower - prev) < EM_TOL:
      converged = True
      break
  if not converged:
    warnings.warn("Best performing initialization did not converge. Try different init "
                  "parameters, or increase max_iter, tol, or check for degenerate data.",
                  ConvergenceWarning, stacklevel=3)
  score = ops.score(_em_args(weights, means, cov)) / m
  n_params = 3 * c - 1
  bic = -2 * score * m + n_params * math.log(m)
  return Fit(np.array(weights), np.array(means), np.array(cov), n_iter, converged, bic, centres)


def gmm_bic(ops, draws=None) -> Result:
  """bic(GMM-1) < bic(GMM-2) on the band behind `ops`, drawing from `draws` (default: the global
  np.random state, as scikit-learn's random_state=None does)."""
  draws = np.random.mtrand._rand if draws is None else draws
  ops.passes = 0
  count, s, _, _, _, bad = ops.moments(0.0)
  if bad:
    raise ValueError("Input X contains NaN or infinity.")
  mean = s / count                             # X.mean(axis=0) of KMeans
  _, d1, d2, _, _, _ = ops.moments(mean)
  var = d2 / count - (d1 / count) ** 2         # np.var(X, axis=0)
  tol = var * KMEANS_TOL
  fits = [_fit(ops, c, mean, (count, d1, d2), tol, draws) for c in (1, 2)]
  return Result(bool(fits[0].bic < fits[1].bic), fits, mean, ops.passes)


# ---- backends ------------------------------------------------------------------------------------
def _assign(x, centres):
  """sklearn's Lloyd label rule in 1-D: argmin_k c_k^2 - 2 x c_k, first minimum wins."""
  d0 = centres[0] * centres[0] - 2.0 * (x * centres[0])
  d1 = centres[1] * centres[1] - 2.0 * (x * centres[1])
  return (d1 < d0).astype(np.int64)


def _sqdist(x, c):
  """_euclidean_distances(squared=True) in 1-D: -2 x c + c^2 + x^2, clipped at 0."""
  return np.maximum(-2.0 * (x * c) + c * c + x * x, 0.0)


class NumpyOps:
  """Reference backend over a host copy of the band (CPU tests of the recurrence)."""

  def __init__(self, affinity, offset):
    a = np.asarray(affinity)
    n = a.shape[0]
    self.x = np.asarray(a[np.triu_indices(n, offset)], dtype=np.float64)
    self.m = self.x.size
    self.passes = 0

  def moments(self, shift):
    self.passes += 1
    x = self.x
    bad = int(np.count_nonzero(~np.isfinite(x)))
    d = x - shift
    with np.errstate(invalid="ignore", over="ignore"):
      return (self.m, float(d.sum()), float((d * d).sum()), float(np.min(x)), float(np.max(x)),
              bad)

  def values(self, idx):
    self.passes += 1
    return [float(self.x[i]) for i in idx]

  def kpp(self, mean, c0, ca=None, cb=None):
    self.passes += 1
    xc = self.x - mean
    d0 = _sqdist(xc, c0)
    self._closest = d0
    ones = np.ones(self.m)
    if ca is None:
      return float(d0 @ ones), 0.0, 0.0
    return (float(d0 @ ones), float(np.minimum(d0, _sqdist(xc, ca)) @ ones),
            float(np.minimum(d0, _sqdist(xc, cb)) @ ones))

  def kpp_lookup(self, mean, c0, targets):
    self.passes += 1
    ids = np.searchsorted(np.cumsum(self._closest), targets)
    ids = np.clip(ids, None, self.m - 1)
    return [float(self.x[i]) for i in ids]

  def lloyd(self, mean, centres, old):
    self.passes += 1
    xc = self.x - mean
    lab = _assign(xc, centres)
    changed = self.m if old is None else int(np.count_nonzero(lab != _assign(xc, old)))
    return (int(lab.sum()), float(xc[lab == 0].sum()), float(xc[lab == 1].sum()), changed)

  def label_moments(self, mean, centres, shifts):
    self.passes += 1
    lab = _assign(self.x - mean, centres)
    x0, x1 = self.x[lab == 0], self.x[lab == 1]
    return (int(lab.sum()), float(x0.sum()), float(x1.sum()),
            float(((x0 - shifts[0]) ** 2).sum()), float(((x1 - shifts[1]) ** 2).sum()))

  def _weighted(self, comps):
    x = self.x
    wlp = np.stack([-0.5 * (LOG_2PI + (x * pc - mupc) ** 2) + logpc + logw
                    for logw, mupc, pc, logpc, _ in comps], axis=1)
    mx = wlp.max(axis=1)
    with np.errstate(under="ignore", divide="ignore"):
      lse = np.log(np.exp(wlp - mx[:, None]).sum(axis=1)) + mx
    return wlp, lse

  def em(self, comps):
    self.passes += 1
    wlp, lse = self._weighted(comps)
    with np.errstate(under="ignore"):
      r = np.exp(wlp - lse[:, None])
    out = []
    for k, (_, _, _, _, s) in enumerate(comps):
      out.append((float(r[:, k].sum()), float(r[:, k] @ self.x),
                  float(r[:, k] @ (self.x - s) ** 2)))
    return float(lse.sum()), out

  def score(self, comps):
    self.passes += 1
    return float(self._weighted(comps)[1].sum())


class DeviceOps:
  """CUDA backend: each reduction is one `sc_gmm_band_pass` over the fp32 device matrix
  [n, lda]; only the band j >= max(0, i + offset), j < n is read.  With `row_off` (the device copy
  of packed_row_offsets(n, offset)), `matrix` is the packed band and each reduction is one
  `sc_gmm_band_pass_packed`."""

  def __init__(self, eng, matrix, n, offset, row_off=None):
    from . import device as dev
    self.eng, self.a, self.n, self.offset = eng, matrix, int(n), int(offset)
    self.row_off = row_off
    self.m = band_size(self.n, self.offset)
    self.ptr = dev._ptr
    # per-row partials of up to 8 fields; the KMeans++ row sums stay here for the lookup
    self.work = dev.torch().empty((8 * self.n + 16,), dtype=dev.torch().float64,
                                  device=eng.device)
    self.params = np.zeros(16, dtype=np.float64)
    self.out = np.zeros(16, dtype=np.float64)
    self.passes = 0

  def _pass(self, mode, *params):
    self.passes += 1
    self.params[:] = 0.0
    self.params[:len(params)] = params
    tail = (self.params.ctypes.data_as(ctypes.c_void_p), self.ptr(self.work),
            self.out.ctypes.data_as(ctypes.c_void_p), self.eng.stream)
    if self.row_off is None:
      self.eng.call("sc_gmm_band_pass", self.ptr(self.a), self.n, self.a.stride(0), self.offset,
                    mode, *tail)
    else:
      self.eng.call("sc_gmm_band_pass_packed", self.ptr(self.a), self.ptr(self.row_off), self.n,
                    self.offset, mode, *tail)
    return self.out

  def moments(self, shift):
    o = self._pass(MOMENTS, shift)
    return int(o[0]), float(o[1]), float(o[2]), float(o[3]), float(o[4]), int(o[5])

  def values(self, idx):
    o = self._pass(LOOKUP, 0.0, 0.0, 0.0, float(idx[0]), float(idx[-1]))
    return [float(o[2]), float(o[3])][:len(idx)]

  def kpp(self, mean, c0, ca=None, cb=None):
    trials = 0.0 if ca is None else 2.0
    o = self._pass(KPP, mean, c0, ca or 0.0, cb or 0.0, trials)
    return float(o[0]), float(o[1]), float(o[2])

  def kpp_lookup(self, mean, c0, targets):
    o = self._pass(LOOKUP, mean, c0, 1.0, float(targets[0]), float(targets[1]))
    self.last_lookup = (int(o[0]), int(o[1]))
    return [float(o[2]), float(o[3])]

  def lloyd(self, mean, centres, old):
    o = self._pass(LLOYD, mean, centres[0], centres[1], *(old or (0.0, 0.0)),
                   0.0 if old is None else 1.0)
    return int(o[0]), float(o[1]), float(o[2]), self.m if old is None else int(o[3])

  def label_moments(self, mean, centres, shifts):
    o = self._pass(LABELS, mean, centres[0], centres[1], shifts[0], shifts[1])
    return int(o[0]), float(o[1]), float(o[2]), float(o[3]), float(o[4])

  def em(self, comps):
    o = self._pass(EM, float(len(comps)), *[v for comp in comps for v in comp])
    return float(o[0]), [tuple(float(v) for v in o[1 + 3 * k:4 + 3 * k])
                         for k in range(len(comps))]

  def score(self, comps):
    return float(self._pass(SCORE, float(len(comps)), *[v for comp in comps for v in comp])[0])
