"""Float64 restatement of `custom_distance_kmeans.run_kmeans` (cosine / euclidean) that records the
margin of every decision it takes, so that a case can be *certified*: every decision is far enough
from its threshold that any float64 evaluation of the same operation takes it the same way.

TEST INFRASTRUCTURE ONLY (NumPy/SciPy).  What it restates, in order:

1. scikit-learn 1.9's `KMeans(k, init="k-means++", max_iter=1, random_state=0).fit(E)`
   (sklearn/cluster/_kmeans.py): X = E - mean(E); `_kmeans_plusplus` (:224-267) with the
   RandomState(0) draws of `Engine.kmeans` -- first centre `choice(n, p=1/n)`, then per centre
   `u = uniform(size=2 + int(ln k))`, candidates `searchsorted(cumsum(closest), u * pot)` clipped to
   n - 1, `np.minimum` with the candidates' squared distances, first argmin of the potentials;
   one Lloyd E-step (argmin of |c|^2 - 2 x.c, first minimum) and M-step (member sum times
   1 / count, plus the mean).  An empty cluster is flagged (`Result.empty_cluster`): scikit-learn
   relocates it, and neither this module nor `sc_kmeans` restates that.
2. `CustomKMeans.predict` (custom_distance_kmeans.py:118-141): at most max_iter + 1 passes of
   scipy `cdist` + argmin, mean distance, the relative stop rule, centroid = mean of members,
   including the quirk that a cluster whose only member is sample 0 keeps its centroid.

Margins and their bounds.  u = 2^-53 and gamma_m = m u / (1 - m u) bounds the rounding of a sum
of m terms in any order (with or without fused multiply-adds): |fl(sum) - sum| <= gamma_m sum|t|.
Each bound below is on the distance between a computed value and a value both float64
implementations are within that bound of; a decision is certified when the computed margin beats
twice the sum of the bounds of the two quantities compared (either implementation can be off by
one bound on each side).  kd is the embedding width and R = max_i |x_i|.

* Squared distances in the seeding, d2(x_i, x_j) = |x_j|^2 - 2 x_i.x_j + |x_i|^2 on centred rows:
  three kd-term sums and two additions give gamma_{kd+2} (|x_i| + |x_j|)^2; the centring
  x = fl(e - mean) perturbs each element by u|x| and the difference of two rows by
  2u (|x_i| + |x_j|)^2 in d2 (the mean itself cancels in x_i - x_j, so the two implementations
  may centre by different means).  Bound r_i = gamma_{kd+5} (|x_i| + R)^2, which also covers the
  closest distance min(...) over any set of centres.
* Potential and cumulative sums: sum_i r_i + gamma_n * pot (n terms, any order -- the device sums
  1,024 chunks and scans them, numpy goes left to right).  The draw u*pot adds u*bound(pot) +
  u*|u pot|.  Margin: distance from u*pot to the nearest cumsum value.
* Trial potentials: gap between the best trial and each trial with a different candidate row
  (the same row gives the same potential in every implementation).
* Lloyd E-step: |c|^2 - 2 x.c, bound gamma_{kd+5} (|x_i| + |c|)^2 as for d2 (only differences
  between centres are compared, so |x_i|^2 and the mean cancel).  Margin: second-best minus best.
* Stage-1 centres: mean of the member rows of E, computed as (sum of centred rows) * fl(1/m) +
  mean; bound gamma_{m+3} (mean_i |x_i| + |c|) in norm.
* Custom-distance passes: euclidean sqrt(sum (x - c)^2) has relative error gamma_{kd+4};
  cosine 1 - x.c / (|x||c|) has absolute error 2 gamma_{kd+4}.  A centroid off by dc moves a
  euclidean distance by at most dc and a cosine distance by at most 2 dc / |c|.  Centroid update:
  gamma_{m+2} mean_i |e_i| over the m members.  Margin per row: second-best minus best.
* Stop rule: the mean distance is off by sum_i bound_i / n + gamma_{n+1} mean.  Margins:
  |mean - prev| and |mean - (1 - tol) prev|.  When the two passes before a pass gave the same labels,
  that pass uses the same centroids as the one before it, so its mean equals prev bit for bit in
  every implementation and the rule fires: counted as decided.

Exact cases.  When a value is provably computed without rounding (every operand and partial sum on
a grid of 2^-q that fits in 53 bits), or by the same single correctly rounded operation on
identical operands, every implementation produces the same bits: its bound is 0 and an exact tie
is decided by the first-minimum rule of `np.argmin`.  Small-integer embeddings whose column means
are exact (columns summing to zero, say) are exact throughout the seeding and the Lloyd E-step.

A certified case must give the same labels and pass count in every float64 implementation; an
uncertified one names the margin that was too small in `Result.failures`."""

from __future__ import annotations

import dataclasses

import numpy as np

U = 2.0 ** -53
TOL = 1e-3


def gamma(m):
  return m * U / (1.0 - m * U)


def draws(n, k):
  """The RandomState(0) draws of `Engine.kmeans` (= scikit-learn's order): first centre, then one
  row of `trials` uniforms per further centre."""
  rs = np.random.RandomState(0)
  first = int(rs.choice(n, p=np.full(n, 1.0 / n)))
  trials = 2 + int(np.log(k))
  u = np.array([rs.uniform(size=trials) for _ in range(k - 1)], dtype=np.float64)
  return first, u.reshape(k - 1, trials)


def grid_exponent(a):
  """Smallest q >= 0 with a * 2^q all integers (finite float64 input)."""
  a = np.asarray(a, dtype=np.float64).ravel()
  a = a[a != 0]
  if a.size == 0:
    return 0
  m, ex = np.frexp(np.abs(a))                       # |a| = m 2^ex, m in [0.5, 1)
  mi = (m * 2.0 ** 53).astype(np.int64)             # exact 53-bit integer mantissa
  tz = np.log2((mi & -mi).astype(np.float64)).astype(np.int64)
  return max(0, int((53 - ex - tz).max()))


def _fits(total_abs, q):
  """A sum whose terms lie on the 2^-q grid and whose sum of magnitudes is total_abs is exact in
  any order: every partial sum is an integer multiple of 2^-q below 2^53 * 2^-q."""
  return q <= 1000 and float(total_abs) * 2.0 ** q < 2.0 ** 53


def _exact_centring(e, mean, q_e):
  """The column sums, their division by n and e - mean are all exact (same bits anywhere)."""
  from fractions import Fraction
  n = e.shape[0]
  if not _fits(np.abs(e).sum(axis=0).max(), q_e):
    return False
  sums = e.sum(axis=0)
  if any(Fraction(float(m)) * n != Fraction(float(s)) for m, s in zip(mean, sums)):
    return False
  q = max(q_e, grid_exponent(mean))
  return _fits((np.abs(e) + np.abs(mean)).max(), q)


@dataclasses.dataclass
class Margin:
  margin: float          # smallest margin of this kind (where the bound is non-zero)
  bound: float           # the bound it had to beat
  where: str


@dataclasses.dataclass
class Result:
  labels: np.ndarray
  iters: int
  certified: bool
  failures: list
  margins: dict                    # kind -> Margin with the smallest margin - bound
  centers: np.ndarray              # stage-1 centres (scikit-learn's cluster_centers_)
  seeds: np.ndarray                # k-means++ row indices
  empty_cluster: bool = False
  exact_ties: int = 0              # argmin decisions taken on an exact tie (first minimum)
  counts: dict = dataclasses.field(default_factory=dict)   # decisions checked per kind


class _Ledger:
  def __init__(self):
    self.margins, self.failures, self.counts = {}, [], {}

  def note(self, kind, margin, bound, where):
    """One decision, or the worst of a vector of them (margin and bound arrays)."""
    margin = np.atleast_1d(np.asarray(margin, dtype=np.float64))
    bound = np.atleast_1d(np.asarray(bound, dtype=np.float64))
    margin, bound = np.broadcast_arrays(margin, bound)
    self.counts[kind] = self.counts.get(kind, 0) + margin.size
    live = bound > 0                                   # bound 0: identical bits everywhere
    if not live.any():
      return
    slack = np.where(live, margin - bound, np.inf)
    j = int(np.argmin(slack))
    old = self.margins.get(kind)
    if old is None or slack[j] < old.margin - old.bound:
      self.margins[kind] = Margin(float(margin.flat[j]), float(bound.flat[j]), "%s[%d]" % (where, j))
    if not slack[j] > 0:
      self.failures.append("%s at %s[%d]: margin %.3e <= bound %.3e" % (
          kind, where, j, margin.flat[j], bound.flat[j]))


def _argmin_margins(d, r, ledger, kind, where):
  """First-minimum argmin of each row of d (n x k) with per-entry bounds r.  Returns labels and the
  number of exact ties decided by the first-minimum rule."""
  n, k = d.shape
  lab = np.argmin(d, axis=1)
  if k == 1:
    return lab, 0
  rows = np.arange(n)
  best = d[rows, lab][:, None]
  rb = r[rows, lab][:, None]
  diff = d - best                                     # >= 0; > 0 left of the winner
  bound = 2.0 * (r + rb)
  exact = bound == 0
  diff[rows, lab] = np.inf
  ties = int(np.count_nonzero(exact & (diff == 0)))
  bound = np.where(exact, 0.0, bound)
  margin = np.where(exact, np.inf, diff)
  # worst entry per row keeps the ledger small
  slack = margin - bound
  j = np.argmin(slack, axis=1)
  ledger.note(kind, margin[rows, j], bound[rows, j], where)
  return lab, ties


def restate(e, k, metric="cosine", max_iter=300, tol=TOL, quirk=True):
  """Labels, pass count and margins of run_kmeans(e, k, metric, max_iter).  `quirk=False` updates
  a cluster whose only member is sample 0 (what the reference does not do), so a test can show
  that a case depends on the quirk."""
  from scipy.spatial import distance
  e = np.ascontiguousarray(e, dtype=np.float64)
  n, kd = e.shape
  if not np.isfinite(e).all():
    raise ValueError("Input X contains NaN." if np.isnan(e).any() else
                     "Input X contains infinity or a value too large for dtype('float64').")
  if max_iter <= 0 or n < k:
    raise ValueError("run_kmeans: bad arguments")
  led = _Ledger()
  ties = 0

  # ---- stage 1: centring
  q_e = grid_exponent(e)
  mean = e.mean(axis=0)
  x = e - mean
  xsq = np.einsum("ij,ij->i", x, x)
  xn = np.sqrt(xsq)
  big_r = float(xn.max())
  exact1 = _exact_centring(e, mean, q_e) and _fits(
      n * 4.0 * big_r ** 2, 2 * max(q_e, grid_exponent(mean)))   # every d2, potential, cumsum
  r_row = np.zeros(n) if exact1 else gamma(kd + 5) * (xn + big_r) ** 2
  r_sum = float(r_row.sum())

  def d2(rows_idx):
    c = x[rows_idx]
    dd = (xsq[rows_idx][:, None] - 2.0 * (c @ x.T)) + xsq[None, :]
    return np.maximum(dd, 0.0)

  def pot_bound(p):
    return 0.0 if exact1 else r_sum + gamma(n) * p

  # ---- k-means++
  first, u = draws(n, k)
  seeds = [first]
  closest = d2(np.array([first]))[0]
  pot = closest.sum()
  for c in range(1, k):
    vals = u[c - 1] * pot
    cum = np.cumsum(closest)
    cand = np.searchsorted(cum, vals)
    # margin to the nearest cumsum value on either side of each draw
    lo = np.clip(cand - 1, 0, n - 1)
    hi = np.clip(cand, 0, n - 1)
    gap = np.minimum(np.abs(cum[lo] - vals), np.abs(cum[hi] - vals))
    b_pot = pot_bound(pot)
    b_val = u[c - 1] * b_pot + (0.0 if exact1 else U * vals)
    led.note("kpp_cumsum", gap, 2.0 * (b_pot + b_val), "centre %d trial" % c)
    np.clip(cand, None, n - 1, out=cand)
    newd = np.minimum(closest[None, :], d2(cand))
    pots = newd.sum(axis=1)
    best = int(np.argmin(pots))
    if len(cand) > 1:
      other = cand != cand[best]
      pb = np.array([pot_bound(p) for p in pots])
      diff = pots - pots[best]
      bnd = 2.0 * (pb + pb[best])
      if exact1:
        ties += int(np.count_nonzero(other & (diff == 0)))
      led.note("kpp_trial", np.where(other, diff, np.inf), np.where(other, bnd, 0.0),
               "centre %d trial" % c)
    seeds.append(int(cand[best]))
    closest = newd[best]
    pot = pots[best]
  seeds = np.array(seeds)

  # ---- one Lloyd iteration (E-step on centred rows, M-step, + mean)
  cen = x[seeds]
  dist = np.sum(cen * cen, axis=1)[None, :] - 2.0 * (x @ cen.T)
  cn = np.sqrt(np.sum(cen * cen, axis=1))
  r_e = np.zeros_like(dist) if exact1 else gamma(kd + 5) * (xn[:, None] + cn[None, :]) ** 2
  lab, t = _argmin_margins(dist, r_e, led, "lloyd_estep", "row")
  ties += t
  counts = np.bincount(lab, minlength=k)
  if (counts == 0).any():
    return Result(lab, 0, False, ["empty cluster after the Lloyd E-step"], led.margins, None,
                  seeds, empty_cluster=True, exact_ties=ties, counts=led.counts)
  sums = np.zeros((k, kd))
  np.add.at(sums, lab, x)
  centers = sums * (1.0 / counts)[:, None] + mean
  if exact1:        # the device divides: its centre equals this one unless fl(S/m) differs
    alt = sums / counts[:, None] + mean
    rc = np.linalg.norm(centers - alt, axis=1)
  else:
    mean_norm = np.bincount(lab, weights=xn, minlength=k) / counts
    rc = gamma(counts + 3) * (mean_norm + np.linalg.norm(centers, axis=1))
  stage1 = centers.copy()

  # ---- stage 2: custom-distance passes
  en = np.sqrt(np.einsum("ij,ij->i", e, e))
  q_rows = q_e
  prev, r_prev = 0.0, 0.0
  prev_labels = None
  same_centroids = False
  c_cur = centers.copy()
  labels = None
  passes = 0
  for it in range(max_iter + 1):
    d = distance.cdist(e, c_cur, metric=metric)
    cnorm = np.linalg.norm(c_cur, axis=1)
    q_c = grid_exponent(c_cur)
    q = max(q_rows, q_c)
    exact_pass = _fits(kd * (float(en.max()) + float(cnorm.max())) ** 2, 2 * q)
    if metric == "euclidean":
      r = (0.0 if exact_pass else gamma(kd + 4)) * d + rc[None, :]
    else:
      with np.errstate(divide="ignore", invalid="ignore"):
        prop = np.where(rc > 0, 2.0 * rc / cnorm, 0.0)
      r = np.full(d.shape, 2.0 * gamma(kd + 4)) + prop[None, :]
      if exact_pass:   # x.c, |x|^2, |c|^2 exact; perfect squares and cos in {-1, 0, 1}: exact
        dot = e @ c_cur.T
        xx = np.einsum("ij,ij->i", e, e) * 4.0 ** q
        cc = np.einsum("ij,ij->i", c_cur, c_cur) * 4.0 ** q
        sx, sc = np.sqrt(xx), np.sqrt(cc)
        sq = (np.rint(sx) ** 2 == xx)[:, None] & (np.rint(sc) ** 2 == cc)[None, :]
        dd = dot * 4.0 ** q
        unit = (dd == 0) | (dd * dd == xx[:, None] * cc[None, :])
        r = np.where(sq & unit, prop[None, :], r)
    nanrow = np.isnan(d).any(axis=1)
    if nanrow.any():
      # a zero row (0/0) is NaN against every centroid: label 0 in numpy and on the device.  A NaN
      # against some centroids only (a zero centroid) is taken differently: not certified.
      partial = nanrow & ~np.isnan(d).all(axis=1)
      if partial.any():
        led.failures.append("pass %d: NaN distance to some centroids only, row %d" % (
            it, int(np.flatnonzero(partial)[0])))
    ok = ~nanrow
    labels = np.zeros(n, dtype=np.int64)
    if ok.any():
      lab_ok, t = _argmin_margins(d[ok], r[ok], led, "pass_argmin", "pass %d row" % it)
      labels[ok] = lab_ok
      ties += t
    rows = np.arange(n)
    sel = d[rows, labels]
    mean_d = np.mean(sel)
    passes = it + 1
    rsel = np.where(ok, r[rows, labels], 0.0)
    if not rsel.any() and _fits(np.abs(sel[ok]).sum(), grid_exponent(sel[ok])):
      r_mean = 0.0                    # exact sum, one correctly rounded division
    else:
      r_mean = float(rsel.sum()) / n + gamma(n + 1) * abs(mean_d)
    # centroids of this pass == those of the previous pass when the two passes before produced
    # the same labels: then the mean repeats bit for bit
    repeat = same_centroids
    settled = mean_d <= prev and mean_d >= (1 - tol) * prev
    if it < max_iter and not repeat and not (np.isnan(mean_d) or np.isnan(prev)):
      b_a = 2.0 * (r_mean + r_prev)
      q_prev = (1 - tol) * prev
      r_q = 0.0 if r_prev == 0 else (1 - tol) * r_prev + U * abs(q_prev)
      b_b = 2.0 * (r_mean + r_q)
      m_a, m_b = abs(mean_d - prev), abs(mean_d - q_prev)
      dec_a = b_a == 0 or m_a > b_a
      dec_b = b_b == 0 or m_b > b_b
      a_true, b_true = mean_d <= prev, mean_d >= q_prev
      decided = (dec_a and not a_true) or (dec_b and not b_true) or (dec_a and dec_b)
      led.counts["stop_rule"] = led.counts.get("stop_rule", 0) + 1
      if not decided:
        kind = "stop_rule_prev" if not dec_a else "stop_rule_tol"
        m, b = (m_a, b_a) if not dec_a else (m_b, b_b)
        led.failures.append("%s at pass %d: margin %.3e <= bound %.3e" % (kind, it, m, b))
      for kind, m, b in (("stop_rule_prev", m_a, b_a), ("stop_rule_tol", m_b, b_b)):
        if b > 0:
          old = led.margins.get(kind)
          if old is None or m - b < old.margin - old.bound:
            led.margins[kind] = Margin(float(m), float(b), "pass %d" % it)
    if settled or it == max_iter:
      break
    prev, r_prev = mean_d, r_mean
    c_before, rc_before = c_cur.copy(), rc.copy()
    for c in range(k):
      members = np.where(labels == c)[0]
      if members.any() or (not quirk and members.size):
        c_cur[c] = np.mean(e[members], axis=0)
        s_abs = np.abs(e[members]).sum(axis=0).max()
        if _fits(s_abs, q_rows):
          rc[c] = 0.0                 # exact member sum, one correctly rounded division
        else:
          rc[c] = gamma(members.size + 2) * float(en[members].mean())
    # the next pass uses the same centroids as this one (so repeats its mean bit for bit) when
    # this pass repeated the labels of the one before, or when the update reproduced them
    # exactly with identical bits in every implementation
    same_centroids = (prev_labels is not None and np.array_equal(labels, prev_labels)) or (
        np.array_equal(c_cur, c_before) and not rc.any() and not rc_before.any())
    prev_labels = labels
  return Result(labels, passes, not led.failures, led.failures, led.margins, stage1, seeds,
                exact_ties=ties, counts=led.counts)


# ---------------------------------------------------------------- case generators
def unit_rows(n, k, kd, spread, seed):
  """n unit rows around k random unit directions in kd dimensions; `spread` sets the overlap."""
  rng = np.random.default_rng(seed)
  cent = rng.standard_normal((k, kd))
  e = cent[rng.integers(0, k, n)] / np.sqrt(kd) * 3.0 + spread * rng.standard_normal((n, kd))
  return e / np.linalg.norm(e, axis=1, keepdims=True)


def integer_rows(n, kd, seed, span=2):
  """Rows with entries in [-span, span] whose columns sum to zero (each row and its negation; a
  zero row makes n odd), so the mean is exactly 0 and every seeding product is exact."""
  rng = np.random.default_rng(seed)
  half = rng.integers(-span, span + 1, (n // 2, kd)).astype(np.float64)
  rows = [half, -half] + ([np.zeros((1, kd))] if n % 2 else [])
  e = np.vstack(rows)
  return e[rng.permutation(n)]


def pythagorean_rows(n, kd=4):
  """n distinct small-integer rows with integer norms, no two with the same direction, and columns
  summing to zero (pairs +-v, and for odd n one triple a + b + c = 0): centring and every cosine
  of a row with itself are exact."""
  import itertools
  import math
  vecs = []
  for v in itertools.product(range(-6, 7), repeat=kd):
    s = sum(t * t for t in v)
    r = math.isqrt(s)
    if s and r * r == s and math.gcd(*v) == 1:
      vecs.append(np.array(v, dtype=np.float64))
  rng = np.random.default_rng(n)
  rows = []
  if n == 1:
    return np.array([[2.0, 3.0, 6.0, 0.0][:kd]])
  if n % 2:
    for a, b in itertools.combinations(vecs, 2):
      c = -(a + b)
      s = int(c @ c)
      if s and math.isqrt(s) ** 2 == s:
        rows += [a, b, c]
        break

  def direction(v):
    return tuple((v // math.gcd(*v.astype(int))).astype(int))

  seen = {direction(r) for r in rows}
  for i in rng.permutation(len(vecs)):
    if len(rows) >= n:
      break
    v = vecs[i]
    if direction(v) in seen or direction(-v) in seen:
      continue
    rows += [v, -v]
    seen |= {direction(v), direction(-v)}
  return np.array(rows[:n])


def lonely_first_sample_rows(seed):
  """A small 2-D case in which, under cosine, a cluster is left holding only sample 0 while its
  centroid is elsewhere: updating that centroid (what the reference does not do) changes the
  labels or the pass count.  Returns (embeddings, k)."""
  rng = np.random.default_rng(seed)
  n, k = int(rng.integers(6, 13)), int(rng.integers(2, 4))
  return rng.standard_normal((n, 2)) + [1.5, 0.5], k
