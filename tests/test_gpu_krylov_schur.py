"""GPU: the general eigen path end to end -- arnoldi.eig_extremal_device (Krylov-Schur over the
sc_krylov_* primitives) on non-symmetric fp32 refined matrices, under every Laplacian, against
LAPACK's dgeev (scipy.linalg.eig) of the float64 matrix M built from the same fp32 S.

Error model (test_krylov_schur_cpu.py states it in full).  u = 2^-53.  The device applies M
exactly up to its fp64 sums (<= n u |M| |x|) and the solver stops at a Ritz residual
<= tol max|theta| <= tol |A|_2, A = flip M.  LAPACK has a backward error <= c n u |A|_F.  So, to
first order and doubled for the second,
    |theta_i - lambda_i| <= 2 kappa_i (tol |A|_2 + 2 c n u |A|_F),   kappa = 1 / |y^H x|.
A simple eigenvector moves under a perturbation E by sum_{l != j} kappa_l |E| / |lambda_j - lambda_l|
(first order); dgeev's normalisation (the largest component made real) turns that into a phase
error of at most |dx| / |x_max|.  Both sides carry such a perturbation.
"""

import math

import numpy as np
import pytest
import scipy.linalg
import scipy.sparse.linalg

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import arnoldi
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import laplacian as lap
from oracle import spectral_oracle as orc

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
C_LAPACK = 8
TOL = 1e-9
LAPLACIANS = [None, lap.LaplacianType.Unnormalized, lap.LaplacianType.RandomWalk,
              lap.LaplacianType.GraphCut]


def t():
  return dev.torch()


def refined_nonsymmetric(n, seed):
  """[CropDiagonal, RowWiseThreshold] of synthetic d-vectors, in fp32: each row's cut follows its
  own maximum, so S is not symmetric nor diagonally similar to a symmetric matrix.  Below 64 rows
  a uniform random matrix, which is no more symmetric."""
  if n < 64:
    return np.random.default_rng(seed).uniform(0.0, 1.0, (n, n)).astype(np.float32)
  x = orc.synthetic_dvectors(n, 32, 4, seed=seed)
  s = orc.row_threshold(orc.crop_diagonal(orc.affinity(x)), 0.9, 0.01).astype(np.float32)
  assert not np.array_equal(s, s.T)
  return s


def operator(engine, s32, laplacian):
  """Device terms from laplacian.terms_from_row_sums and the float64 M they stand for."""
  n = s32.shape[0]
  s64 = s32.astype(np.float64)
  rowsum = t().from_numpy(s64.sum(axis=1)).to(engine.device)
  delta, left, right, sign, which = lap.terms_from_row_sums(rowsum, None, laplacian)
  hv = lambda x: np.ones(n) if x is None else x.cpu().numpy()
  m = sign * (hv(left)[:, None] * s64 * hv(right)[None, :])
  if delta is not None:
    m[np.arange(n), np.arange(n)] += hv(delta)
  s = engine.upload_matrix(s32)
  return (s, n, delta, left, right, sign), which == nat.EIG_SMALLEST, m


def lapack(a):
  w, vl, vr = scipy.linalg.eig(a, left=True, right=True)
  dots = np.abs(np.einsum("ij,ij->j", vl.conj(), vr))
  dots /= np.linalg.norm(vl, axis=0) * np.linalg.norm(vr, axis=0)
  return w, 1.0 / np.maximum(dots, np.finfo(float).tiny), vr


def norms(a):
  n = a.shape[0]
  a_2 = math.sqrt(np.abs(a).sum(axis=0).max() * np.abs(a).sum(axis=1).max())   # >= |A|_2
  return a_2, 2 * C_LAPACK * n * U * np.linalg.norm(a)


def spans_everything(n, n_values):
  """The basis of eig_extremal_device spans the whole space: no residual coupling is left, the
  Ritz values are those of an orthogonal similarity, and only rounding separates them from A's."""
  cap = n if n_values >= n else min(n, max(2 * n_values + 40, 64))
  return n <= max(cap, 2 * n_values + 40, 64)


def error_radius(a, n_values):
  a_2, backward = norms(a)
  return backward if spans_everything(a.shape[0], n_values) else TOL * a_2 + backward


def match(w, a, lam, kappa):
  """Matches the device's real parts w (of A = flip M) with LAPACK's eigenvalues by real part,
  a tie at the edge of the wanted set by either copy.  Returns the matched indices."""
  _, backward = norms(a)
  radius = 2 * kappa * backward
  kappa_c = np.array([kappa[np.abs(lam - lam[j]) <= radius + radius[j]].max()
                      for j in range(len(lam))])
  bound = 2 * kappa_c * error_radius(a, len(w))
  edge = np.sort(lam.real)[::-1][len(w) - 1]
  used = []
  for i, wi in enumerate(w):
    dist = np.abs(lam.real - wi)
    ok = [j for j in np.argsort(dist, kind="stable") if j not in used and dist[j] <= bound[j]]
    assert ok, "w[%d] = %r: nearest %r, bound %g" % (i, wi, lam[np.argmin(dist)],
                                                      bound[np.argmin(dist)])
    used.append(ok[0])
    assert lam[ok[0]].real >= edge - bound[ok[0]], (i, wi, edge)
  return np.array(used), bound


def check_vectors(v, a, lam, kappa, vr, used):
  """Every matched eigenvalue that is simple, with LAPACK's `.real` vector: equal up to sign."""
  e = error_radius(a, len(used))
  checked = 0
  for c, j in enumerate(used):
    d = np.abs(lam - lam[j])
    d[j] = np.inf
    if np.iscomplex(lam[j]):
      d[np.argmin(np.abs(lam - np.conj(lam[j])))] = np.inf    # its conjugate: same real part
    dx = float(np.sum(kappa * e / d))
    x = vr[:, j] / np.linalg.norm(vr[:, j])
    mods = np.sort(np.abs(x))[::-1]
    if dx > 1e-2 or (len(mods) > 1 and mods[0] - mods[1] <= 4 * dx):
      continue                        # no gap, or the largest component is ambiguous
    bound = 2 * dx * (1 + 1 / mods[0]) * 2
    want = x.real if np.iscomplex(lam[j]) else np.real(x)
    got = v[:, c]
    sign = 1.0 if got @ want >= 0 else -1.0
    assert np.linalg.norm(got - sign * want) <= bound, (c, lam[j], np.linalg.norm(got - sign * want), bound)
    checked += 1
  return checked


def solve_twice(engine, op, smallest, n_values):
  runs = [arnoldi.eig_extremal_device(engine, *op, smallest, n_values, n_values) for _ in range(2)]
  (w, v, stats), (w2, v2, stats2) = runs
  np.testing.assert_array_equal(w2, w)
  vh, vh2 = v.cpu().numpy(), v2.cpu().numpy()
  np.testing.assert_array_equal(vh2.view(np.int64), vh.view(np.int64))
  assert stats == stats2
  assert stats[2] == min(n_values, op[1])
  return w, vh, stats


@pytest.mark.parametrize("laplacian", LAPLACIANS, ids=lambda x: "none" if x is None else x.name)
@pytest.mark.parametrize("n,n_values", [(2, 2), (6, 3), (64, 8), (65, 8), (1024, 8), (2049, 8)])
def test_eig_extremal_device_against_lapack(engine, n, n_values, laplacian):
  s32 = refined_nonsymmetric(n, n)
  op, smallest, m = operator(engine, s32, laplacian)
  flip = -1.0 if smallest else 1.0
  w, v, stats = solve_twice(engine, op, smallest, n_values)
  a = flip * m
  lam, kappa, vr = lapack(a)
  used, _ = match(flip * w, a, lam, kappa)
  check_vectors(v, a, lam, kappa, vr, used)


def test_full_spectrum_at_the_limit(engine):
  """n = 1024 = FULL_SPECTRUM_LIMIT, every eigenpair: 16 combine chunks of 64 vectors, most of
  them complex pairs (the complex branch of ritz_vectors)."""
  n = arnoldi.FULL_SPECTRUM_LIMIT
  s32 = np.random.default_rng(5).uniform(0.0, 1.0, (n, n)).astype(np.float32)
  op, smallest, m = operator(engine, s32, None)
  w, v, stats = solve_twice(engine, op, smallest, n)
  lam, kappa, vr = lapack(m)
  assert np.sum(np.abs(lam.imag) > 0) > n // 2
  used, _ = match(w, m, lam, kappa)
  checked = check_vectors(v, m, lam, kappa, vr, used)
  assert checked >= n // 2, checked


def components(n, k, seed):
  """Block-diagonal [CropDiagonal, RowWiseThreshold] affinity of k groups, in fp32."""
  rng = np.random.default_rng(seed)
  cuts = np.sort(rng.choice(np.arange(20, n - 20), k - 1, replace=False))
  bounds = np.concatenate([[0], cuts, [n]])
  s = np.zeros((n, n), dtype=np.float32)
  for b0, b1 in zip(bounds[:-1], bounds[1:]):
    x = rng.standard_normal((b1 - b0, 16))
    s[b0:b1, b0:b1] = orc.row_threshold(orc.crop_diagonal(orc.affinity(x)), 0.95, 0.01)
  return s, list(zip(bounds[:-1], bounds[1:]))


@pytest.mark.parametrize("n,k", [(300, 3), (1000, 5), (3000, 8)])
def test_unnormalized_laplacian_zero_repeated_k_times(engine, n, k):
  """L = D - S has eigenvalue 0 exactly k times: every copy must be found on the device too,
  where the rounding that seeds the copies differs from the host's.  No gap, so the vectors are
  checked by residual: |L x - w x| <= tol |A|_2 + rounding."""
  s32, blocks = components(n, k, n + k)
  op, smallest, m = operator(engine, s32, lap.LaplacianType.Unnormalized)
  assert smallest
  w, v, stats = solve_twice(engine, op, smallest, k + 2)
  lam = np.concatenate([scipy.linalg.eigvals(m[b0:b1, b0:b1]) for b0, b1 in blocks])
  kappa = np.concatenate([lapack(-m[b0:b1, b0:b1])[1] for b0, b1 in blocks])
  match(-w, -m, -lam, kappa)
  a_2, backward = norms(m)
  assert np.all(np.abs(w[:k]) <= 2 * kappa.max() * (TOL * a_2 + backward))
  resid = np.linalg.norm(m @ v[:, :k] - v[:, :k] * w[:k], axis=0)
  assert np.all(resid <= 2 * (TOL * a_2 + backward)), resid


def test_restarting_solve_against_arpack(engine):
  """n = 6000, [RowWiseThreshold] alone, no Laplacian: the basis restarts.  LAPACK would be slow
  here, so ARPACK (float64) on M and on M^T gives the eigenvalues of largest real part and their
  left and right vectors, hence kappa."""
  n, nv = 6000, 8
  x = orc.synthetic_dvectors(n, 32, 6, seed=11)
  s32 = orc.row_threshold(orc.affinity(x), 0.9, 0.01, kind="percentile").astype(np.float32)
  op, smallest, m = operator(engine, s32, None)
  w, v, stats = solve_twice(engine, op, smallest, nv)
  assert stats[1] >= 1
  k = nv + 4
  lam, xr = scipy.sparse.linalg.eigs(m, k=k, which="LR", tol=1e-13, ncv=80)
  lam_l, yl = scipy.sparse.linalg.eigs(m.T, k=k, which="LR", tol=1e-13, ncv=80)
  kappa = np.empty(k)
  for j in range(k):
    l = np.argmin(np.abs(lam_l - np.conj(lam[j])))
    y, xx = yl[:, l], xr[:, j]
    kappa[j] = np.linalg.norm(y) * np.linalg.norm(xx) / abs(np.vdot(y, xx))
  # ARPACK's own residual (tol 1e-13 of |lambda|) is inside the LAPACK-sized backward term's
  # order; the wanted end must not be cut by the k found
  order = np.argsort(-lam.real)
  lam, kappa = lam[order], kappa[order]
  assert lam[nv].real < lam[nv - 1].real
  match(w, m, lam, kappa)


def test_predict_threshold_only_grows_against_float64():
  """predict() with [RowWiseThreshold] and max_clusters=None at N = 3000 > FULL_SPECTRUM_LIMIT takes
  grow_krylov_schur.  The float64 restatement: the oracle's refinement and Laplacian and
  scipy.linalg.eig.  The device matrix differs from the oracle's by its fp32 affinity: no entry
  may lie within 2^-20 of its row's cut (so both take the same thresholding decisions), and
  then |E| <= 8 2^-24 |M|_F (the affinity's few fp32 roundings and S's storage) joins the bound."""
  n = 3000
  x = orc.synthetic_dvectors(n, 128, 4, seed=4, intra_cos=0.8)
  aff = orc.affinity(x)
  cut = aff.max(axis=1, keepdims=True) * 0.95
  assert np.abs(aff - cut).min() > 2.0 ** -20
  c = scb.SpectralClusterer(
      refinement_options=scb.RefinementOptions(refinement_sequence=[scb.RefinementName.RowWiseThreshold]),
      laplacian_type=scb.LaplacianType.GraphCut)
  c.predict(x)
  assert c.last_details["solver"] == "krylov-schur"
  w = np.asarray(c.last_details["eigenvalues"])
  m = orc.laplacian(orc.row_threshold(aff, 0.95, 0.01), "graphcut")
  lam, kappa, _ = lapack(m)
  a_2, backward = norms(m)
  e = TOL * a_2 + backward + 8 * 2.0 ** -24 * np.linalg.norm(m)
  # smallest first: the device's values are the prefix of the ascending real parts
  order = np.argsort(lam.real, kind="stable")
  want = lam.real[order][:len(w)]
  assert np.all(np.abs(w - want) <= 2 * kappa[order][:len(w)].max() * e), np.abs(w - want).max()
  k_ref, _ = orc.number_of_clusters(lam.real[order], None, eigengap="ratio", descend=False)
  assert c.last_details["n_clusters"] == k_ref
