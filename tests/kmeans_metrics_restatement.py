"""Float64 restatement of stage 2 of `custom_distance_kmeans.run_kmeans` for the scipy metrics
beyond cosine and euclidean, recording the margin of every decision so that a case can be
certified (see kmeans_restatement.py, whose stage 1, ledger and stop-rule accounting this reuses).

TEST INFRASTRUCTURE ONLY (NumPy/SciPy).  Stage 1 (k-means++ seeding and one Lloyd step) does not
depend on the metric: `kmeans_restatement.restate` runs it, and only its stage-1 decisions are kept.
Stage 2 is the reference's loop with scipy's `cdist(E, C, metric)`, its per-pass parameters
recomputed from vstack([E, C]) as scipy's validators do.

Bounds.  u = 2^-53, gamma_m as in kmeans_restatement.  Each distance carries a bound on its
rounding (any order of the same operations, with or without fused multiply-adds, log within
2 ulps) plus the effect of a centroid off by rc in norm and of the per-pass parameters' own error.
Subtraction and abs are correctly rounded and take identical bits everywhere, and so does a max of
them: chebyshev's rounding bound is 0.
* sqeuclidean: gamma_{kd+1} d; centroid rc (2 sqrt(d) + rc).
* cityblock: gamma_{kd} d; centroid sqrt(kd) rc.  chebyshev: 0; centroid rc.
* canberra: gamma_{kd+3} d; centroid 2 rc / (|x_f| + |c_f| - rc) per term (unbounded where a term's
  denominator is within rc of 0: a 0/0 term adds 0 but a perturbed one adds 1).
* braycurtis: gamma_{2kd+3} d; centroid sqrt(kd) rc (1 + d) / (den - sqrt(kd) rc).  NaN where
  sum |x + c| is exactly 0 (x = -c exactly), which every implementation decides alike.
* correlation: cosine of the row-centred vectors, 2 gamma_{kd+4} plus 2 |dv| / |v| for each
  centred vector v off by dv (the row mean's rounding, and rc for a centroid).  NaN where a
  centred vector is exactly 0: a constant vector whose mean is exact.
* jensenshannon: inf where an entry is negative (a sign test: exact, unless a centroid entry lies
  within its rounding of 0).  Otherwise the divergence s is off by gamma_{2kd+8} sum (p + q)
  (1 + |log(p/m)| + |log(q/m)|) from rounding, and by sum |log(2 q/(p + q))| |dq| for a centroid
  perturbation dq (doubled for the second order); the distance sqrt(s/2) by min(ds/(2 d),
  sqrt(ds/2)).
* seuclidean: V over the n + k rows is off by dV = gamma_{m+3} V + m dmu^2/(m - 1) + the centroid
  terms (2 |c - mu| rc + rc^2)/(m - 1); the distance by gamma_{kd+4} d + d max(dV/V) + rc /
  sqrt(min V).  A column that is exactly constant in every row (its mean exact) has V = 0 and every
  distance NaN (0/0), in every implementation.
* mahalanobis: CV is off by dCV (rounding gamma_{m+3} |X - mu|^T |X - mu| / (m - 1), and the
  centroid terms), VI by |VI|^2 (dCV + 2 kd^2 u |CV|) / (1 - ...) in the 2-norm (the inverse's
  own error, for any pivot growth up to kd); s = d^T VI d by gamma_{2kd+2} |d|^T |VI| |d| +
  |dVI| |d|^2 and the distance by min(ds / sqrt(s), sqrt(ds)) + u d + sqrt(|VI|) rc.  An exactly
  singular CV raises numpy's LinAlgError here (np.linalg.inv), as in the reference.

Argmin: np.argmin, the first NaN wins, otherwise the first minimum.  NaN and inf entries are only
accepted where the conditions above prove them in every implementation; a row whose every entry
is inf is label 0.  The stop rule takes non-finite means as exact (inf or NaN compare alike
everywhere)."""

from __future__ import annotations

import numpy as np

import kmeans_restatement as kr

U, TOL, gamma = kr.U, kr.TOL, kr.gamma

# the metrics sc_kmeans evaluates beyond cosine / euclidean (minkowski with p = 2 is euclidean)
METRICS = ["sqeuclidean", "cityblock", "chebyshev", "minkowski", "canberra", "braycurtis",
           "correlation", "jensenshannon", "seuclidean", "mahalanobis"]
STAGE1_KINDS = ("kpp_cumsum", "kpp_trial", "lloyd_estep", "empty cluster")


def stage1(e, k):
  """Stage-1 centres, their bound rc (norm, per centre) and stage-1 failures, from
  kmeans_restatement.restate; its euclidean stage 2 is discarded."""
  w = kr.restate(e, k, "euclidean", max_iter=1)
  fails = [f for f in w.failures if f.startswith(STAGE1_KINDS)]
  if w.empty_cluster:
    return None, None, fails, w
  n, kd = e.shape
  mean = e.mean(axis=0)
  x = e - mean
  xn = np.sqrt(np.einsum("ij,ij->i", x, x))
  q_e = kr.grid_exponent(e)
  exact1 = kr._exact_centring(e, mean, q_e) and kr._fits(
      n * 4.0 * float(xn.max()) ** 2, 2 * max(q_e, kr.grid_exponent(mean)))
  cen = x[w.seeds]
  lab = np.argmin(np.sum(cen * cen, axis=1)[None, :] - 2.0 * (x @ cen.T), axis=1)
  counts = np.bincount(lab, minlength=k)
  sums = np.zeros((k, kd))
  np.add.at(sums, lab, x)
  centers = sums * (1.0 / counts)[:, None] + mean
  if exact1:
    rc = np.linalg.norm(centers - (sums / counts[:, None] + mean), axis=1)
  else:
    mean_norm = np.bincount(lab, weights=xn, minlength=k) / counts
    rc = gamma(counts + 3) * (mean_norm + np.linalg.norm(centers, axis=1))
  assert np.array_equal(centers, w.centers)
  return centers, rc, fails, w


def _constant_exact(v):
  """Rows of v (2-D) that are constant with a mean computed exactly in any order."""
  v = np.atleast_2d(v)
  const = (v == v[:, :1]).all(axis=1)
  kd = v.shape[1]
  out = np.zeros(v.shape[0], dtype=bool)
  for i in np.flatnonzero(const):
    out[i] = kr._fits(kd * abs(float(v[i, 0])), kr.grid_exponent(v[i, :1]))
  return out


def distances(e, c, rc, metric):
  """scipy's cdist(e, c, metric), per-entry bounds r (inf: undecidable) and `sure`, the entries
  whose NaN / inf status is the same in every implementation.  May raise scipy's ValueError or
  numpy's LinAlgError, as the reference does."""
  from scipy.spatial import distance
  d = distance.cdist(e, c, metric=metric)
  n, kd = e.shape
  k = c.shape[0]
  rcc = rc[None, :]
  sure = np.isfinite(d)
  with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
    if metric == "sqeuclidean":
      r = gamma(kd + 1) * d + rcc * (2.0 * np.sqrt(d) + rcc)
    elif metric == "cityblock":
      r = gamma(kd) * d + np.sqrt(kd) * rcc
    elif metric == "chebyshev":
      r = np.broadcast_to(rcc, d.shape).copy()
    elif metric == "minkowski":
      r = gamma(kd + 4) * d + rcc
    elif metric == "canberra":
      den = np.abs(e)[:, None, :] + np.abs(c)[None, :, :]
      slack = den - rc[None, :, None]
      pert = np.where(slack > 0, 2.0 * rc[None, :, None] / slack, np.inf)
      pert = np.where(rc[None, :, None] == 0, 0.0, pert).sum(axis=2)
      r = gamma(kd + 3) * d + pert
    elif metric == "braycurtis":
      den = np.abs(e[:, None, :] + c[None, :, :]).sum(axis=2)
      slack = den - np.sqrt(kd) * rcc
      pert = np.where(rcc == 0, 0.0, np.where(slack > 0, np.sqrt(kd) * rcc * (1.0 + d) / slack,
                                             np.inf))
      r = gamma(2 * kd + 3) * d + pert
      # a zero row sums |c| twice in the same order: exactly 1 against every nonzero centroid
      r[~e.any(axis=1)] = 0.0
      sure = sure | ((den == 0) & (rcc == 0))
    elif metric == "correlation":
      ec = e - e.mean(axis=1, keepdims=True)
      cc = c - c.mean(axis=1, keepdims=True)
      en, cn = np.linalg.norm(ec, axis=1), np.linalg.norm(cc, axis=1)
      de = np.sqrt(kd) * gamma(kd + 1) * np.abs(e).mean(axis=1) + U * en
      dc = np.sqrt(kd) * gamma(kd + 1) * np.abs(c).mean(axis=1) + U * cn + rc
      r = 2.0 * gamma(kd + 4) + 2.0 * (de / en)[:, None] + 2.0 * (dc / cn)[None, :]
      zero_e = _constant_exact(e)
      zero_c = _constant_exact(c) & (rc == 0)
      sure = sure | zero_e[:, None] | zero_c[None, :]
    elif metric == "jensenshannon":
      neg_e = (e < 0).any(axis=1)
      elem = rc[:, None] * np.ones((1, kd))               # |dc_f| <= rc
      neg_c = (c < 0) & (np.abs(c) > elem)
      unsure_c = (np.abs(c) <= elem) & (elem > 0) & (c != 0) | ((c == 0) & (elem > 0))
      inf_sure = neg_e[:, None] | neg_c.any(axis=1)[None, :]
      p = e / e.sum(axis=1, keepdims=True)
      q = c / c.sum(axis=1, keepdims=True)
      pp, qq = p[:, None, :], q[None, :, :]
      m = (pp + qq) / 2.0
      lp = np.where(pp > 0, np.abs(np.log(pp / m)), 0.0)
      lq = np.where(qq > 0, np.abs(np.log(qq / m)), 0.0)
      ds = gamma(2 * kd + 8) * ((pp + qq) * (1.0 + lp + lq)).sum(axis=2)
      csum = c.sum(axis=1)
      dq = (elem + q * np.sqrt(kd) * rc[:, None]) / (csum - np.sqrt(kd) * rc)[:, None]
      near0 = (q < 2.0 * dq) & (dq > 0)
      ds_c = 2.0 * (np.abs(np.log(2.0 * qq / (pp + qq))) * dq[None, :, :]).sum(axis=2)
      ds_c = np.where(near0.any(axis=1)[None, :], np.inf, ds_c)
      ds = ds + np.where(rcc == 0, 0.0, ds_c)
      r = np.minimum(ds / (2.0 * np.where(d > 0, d, np.inf)), np.sqrt(ds / 2.0)) + U * d
      r = np.where(inf_sure, 0.0, r)
      r = np.where(~inf_sure & unsure_c.any(axis=1)[None, :], np.inf, r)
      sure = (sure & ~unsure_c.any(axis=1)[None, :]) | inf_sure
    elif metric == "seuclidean":
      x = np.vstack([e, c])
      m = n + k
      mu = x.mean(axis=0)
      v = np.var(x, axis=0, ddof=1)
      dmu = gamma(m + 1) * np.abs(x).mean(axis=0)
      dv = gamma(m + 3) * v + m * dmu ** 2 / (m - 1) + (
          2.0 * (np.abs(c - mu) * rc[:, None]).sum(axis=0) + k * rc.max() ** 2) / (m - 1)
      zero_col = (x == x[:1]).all(axis=0)
      zero_col &= np.array([kr._fits(m * abs(float(x[0, f])), kr.grid_exponent(x[:1, f]))
                            for f in range(kd)])
      if zero_col.any():
        # every row and centroid holds the column's value, and a mean of equal values that sums
        # exactly reproduces it: every term of that column is 0/0 and every distance NaN
        return d, np.zeros_like(d), np.ones(d.shape, dtype=bool)
      rel = dv / v
      r = gamma(kd + 4) * d + d * rel.max() / max(1.0 - rel.max(), 0.0) + rcc / np.sqrt(
          max(v.min() - dv.max(), 0.0))
    elif metric == "mahalanobis":
      x = np.vstack([e, c])
      m = n + k
      cv = np.atleast_2d(np.cov(x.T))
      vi = np.linalg.inv(cv).T                  # LinAlgError("Singular matrix") as scipy
      xc = np.abs(x - x.mean(axis=0))
      dcv = np.linalg.norm(gamma(m + 3) * (xc.T @ xc) / (m - 1), 2)
      dcv += (2.0 * np.sqrt(k) * rc.max() * float(np.abs(c - x.mean(axis=0)).max()) * np.sqrt(kd)
              + k * rc.max() ** 2) / (m - 1)
      nvi, ncv = np.linalg.norm(vi, 2), np.linalg.norm(cv, 2)
      eta = nvi * (dcv + 2.0 * kd * kd * U * ncv)
      dvi = nvi * eta / (1.0 - eta) if eta < 0.5 else np.inf
      diff = e[:, None, :] - c[None, :, :]
      absd = np.abs(diff)
      s = d * d
      ds = gamma(2 * kd + 2) * np.einsum("ikf,fg,ikg->ik", absd, np.abs(vi), absd) + dvi * (
          absd ** 2).sum(axis=2)
      r = np.minimum(ds / np.where(s > 0, np.sqrt(s), np.inf), np.sqrt(ds)) + U * d + np.sqrt(
          nvi) * rcc
    else:
      raise ValueError(metric)
  r = np.where(np.isfinite(d), r, 0.0)
  return d, r, sure


def _argmin_nan_first(d, r, sure, led, where):
  """np.argmin with margins: the first NaN wins, otherwise the first minimum.  Non-finite entries
  must be `sure`; a finite winner must beat every other finite entry by twice the bounds."""
  n, k = d.shape
  lab = np.argmin(d, axis=1)
  bad = ~np.isfinite(d) & ~sure
  if bad.any():
    i, j = np.argwhere(bad)[0]
    led.failures.append("%s: non-finite distance not certain at row %d, centroid %d" % (where, i, j))
  if k == 1:
    return lab
  rows = np.arange(n)
  best = d[rows, lab]
  fin = np.isfinite(best)
  with np.errstate(invalid="ignore"):
    diff = d - best[:, None]
  bound = 2.0 * (r + r[rows, lab][:, None])
  margin = np.where(np.isfinite(d), diff, np.inf)
  margin[rows, lab] = np.inf
  margin = np.where(fin[:, None], margin, np.inf)     # NaN / all-inf rows: decided by `sure`
  bound = np.where(np.isfinite(margin), bound, 0.0)
  live = bound > 0
  if live.any():
    slack = np.where(live, margin - bound, np.inf)
    j = np.argmin(slack, axis=1)
    led.note("pass_argmin", margin[rows, j], bound[rows, j], where)
  return lab


def restate(e, k, metric, max_iter=300, tol=TOL):
  """Labels, pass count and margins of run_kmeans(e, k, metric, max_iter)."""
  e = np.ascontiguousarray(e, dtype=np.float64)
  n, kd = e.shape
  if not np.isfinite(e).all():
    raise ValueError("Input X contains NaN." if np.isnan(e).any() else
                     "Input X contains infinity or a value too large for dtype('float64').")
  if max_iter <= 0 or n < k:
    raise ValueError("run_kmeans: bad arguments")
  centers, rc, fails, w1 = stage1(e, k)
  led = kr._Ledger()
  led.failures += fails
  if centers is None:
    return kr.Result(w1.labels, 0, False, led.failures, led.margins, None, w1.seeds,
                     empty_cluster=True)
  c_cur, rc = centers.copy(), rc.copy()
  en = np.sqrt(np.einsum("ij,ij->i", e, e))
  prev, r_prev = 0.0, 0.0
  prev_labels, same_centroids, labels, passes = None, False, None, 0
  for it in range(max_iter + 1):
    d, r, sure = distances(e, c_cur, rc, metric)
    labels = _argmin_nan_first(d, r, sure, led, "pass %d row" % it)
    rows = np.arange(n)
    sel = d[rows, labels]
    mean_d = np.mean(sel)
    passes = it + 1
    rsel = r[rows, labels]
    r_mean = float(rsel.sum()) / n + gamma(n + 1) * abs(mean_d) if np.isfinite(mean_d) else 0.0
    settled = mean_d <= prev and mean_d >= (1 - tol) * prev
    if it < max_iter and not same_centroids and np.isfinite(mean_d) and np.isfinite(prev):
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
    if settled or it == max_iter:
      break
    prev, r_prev = mean_d, r_mean
    c_before, rc_before = c_cur.copy(), rc.copy()
    for c in range(k):
      members = np.where(labels == c)[0]
      if members.any():          # sic: a cluster holding only sample 0 keeps its centroid
        c_cur[c] = np.mean(e[members], axis=0)
        if kr._fits(np.abs(e[members]).sum(axis=0).max(), kr.grid_exponent(e)):
          rc[c] = 0.0
        else:
          rc[c] = gamma(members.size + 2) * float(en[members].mean())
    same_centroids = (prev_labels is not None and np.array_equal(labels, prev_labels)) or (
        np.array_equal(c_cur, c_before) and not rc.any() and not rc_before.any())
    prev_labels = labels
  return kr.Result(labels, passes, not led.failures, led.failures, led.margins, centers, w1.seeds,
                   counts=led.counts)


# ---------------------------------------------------------------- case generators
def positive_rows(n, k, kd, spread, seed):
  """n rows of positive weights around k random profiles (jensenshannon's finite case).  Not
  normalised: rows summing to 1 would make mahalanobis's covariance singular."""
  rng = np.random.default_rng(seed)
  prof = rng.gamma(1.0, 1.0, (k, kd)) + 0.05
  return prof[rng.integers(0, k, n)] * np.exp(spread * rng.standard_normal((n, kd)))
