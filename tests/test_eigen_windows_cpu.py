"""CPU: the settlement rule of the windowed eigensolve (eigen_windows.settled) against the eigengap
of the whole spectrum, the window loop on a NumPy backend, and which route _eigen_on_device takes
for max_clusters=None / >= 32 above the dense solver's n (a recording fake engine)."""

import functools

import numpy as np
import pytest
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import eigen_windows as ew
from spectralcluster_b200 import laplacian as lap
from spectralcluster_b200 import utils
from oracle import spectral_oracle as orc

from test_host_logic import FakeEngine

RATIO, NDIFF = utils.EigenGapType.Ratio, utils.EigenGapType.NormalizedDiff
LT = scb.LaplacianType
L, S = nat.EIG_LARGEST, nat.EIG_SMALLEST


def count(w, descend, eigengap, lambda_max=None, max_clusters=None):
  stop = dict(stop_eigenvalue=1e-2) if descend else {}
  return utils.compute_number_of_clusters(w, max_clusters=max_clusters, eigengap_type=eigengap,
                                          descend=descend, max_eigenvalue=lambda_max, **stop)


def check_every_settled_prefix(w, descend, eigengap, max_clusters=None, upto=None):
  """For every m at which settled() holds, (k, gap) of the prefix equal those of the whole
  spectrum.  Returns the first such m (None if never)."""
  lam = float(np.max(w))
  full = count(w, descend, eigengap, max_clusters=max_clusters)
  first = None
  for m in range(1, min(len(w), upto or len(w)) + 1):
    if ew.settled(w[:m], descend, max_clusters, 1e-2, eigengap, lam):
      got = count(w[:m], descend, eigengap, None if descend else lam, max_clusters)
      assert got == full, (m, got, full)
      first = first or m
  return first


@functools.lru_cache(maxsize=None)
def oracle_matrix(n, speakers, refined):
  """(S, row scale or None) of the oracle's float64 chain on synthetic d-vectors, d = 256."""
  x = orc.synthetic_dvectors(n, 256, speakers, seed=0)
  a = orc.affinity(x)
  if not refined:
    return a, None
  s = orc.refine(a, orc.options(sequence=orc.ICASSP2018[:-1]))   # RowWiseNormalize: row scale
  return s, 1.0 / s.max(axis=1)


@functools.lru_cache(maxsize=None)
def reference_spectrum(n, speakers, refined, laplacian):
  """The sorted spectrum of the matrix the reference decomposes, through its symmetrised form."""
  s, r = oracle_matrix(n, speakers, refined)
  delta, left, right, sign, which = lap.terms_from_row_sums(
      torch.from_numpy(s.sum(axis=1)), None if r is None else torch.from_numpy(r), laplacian)
  le = np.ones(n) if left is None else left.numpy()
  ri = np.ones(n) if right is None else right.numpy()
  c = np.sqrt(le * ri)
  t = sign * c[:, None] * s * c[None, :]
  if delta is not None:
    t[np.diag_indices(n)] += delta.numpy()
  w = np.linalg.eigvalsh(t)
  descend = which == nat.EIG_LARGEST
  return (w[::-1] if descend else w), descend


@pytest.mark.parametrize("eigengap", [RATIO, NDIFF])
@pytest.mark.parametrize("laplacian", [None, LT.GraphCut, LT.RandomWalk, LT.Unnormalized])
@pytest.mark.parametrize("refined", [False, True])
@pytest.mark.parametrize("n,speakers", [(2000, 4), (3000, 6)])
def test_settled_prefixes_decide_like_the_whole_spectrum(n, speakers, refined, laplacian, eigengap):
  w, descend = reference_spectrum(n, speakers, refined, laplacian)
  first = check_every_settled_prefix(w, descend, eigengap, upto=600)
  if descend and not refined:
    # raw cosine affinity (X^X^T + 1) / 2: rank d + 1, the first value below stop_eigenvalue is d + 2
    assert first == 256 + 2
  elif refined and laplacian in (None, LT.GraphCut, LT.RandomWalk):
    assert first is not None and first <= 2 * speakers + 1, first
  # with max_clusters the rule is the bounded scan's: settled at max_clusters + 1 at the latest
  first = check_every_settled_prefix(w, descend, eigengap, max_clusters=7, upto=20)
  assert first is not None and first <= 8


@pytest.mark.parametrize("seed", range(40))
@pytest.mark.parametrize("eigengap", [RATIO, NDIFF])
@pytest.mark.parametrize("descend", [True, False])
def test_settled_on_random_spectra(seed, eigengap, descend):
  """Negative, near-zero and exactly tied values: settled prefixes never change (k, gap)."""
  rng = np.random.default_rng(seed)
  n = int(rng.integers(5, 60))
  w = np.concatenate([rng.exponential(1.0, n) * 10.0 ** rng.integers(-3, 2),
                      rng.normal(0.0, 1e-9, int(rng.integers(0, 5))),        # near zero
                      -rng.exponential(1e-3, int(rng.integers(0, 3)))])     # negative
  w = np.concatenate([w, rng.choice(w, int(rng.integers(0, 6)))])           # exact ties
  if seed % 4 == 0:
    w = np.concatenate([w, np.full(5, 0.01)])                               # at stop_eigenvalue
  w = np.sort(w)[::-1] if descend else np.sort(w)
  check_every_settled_prefix(w, descend, eigengap)
  check_every_settled_prefix(w, descend, eigengap, max_clusters=int(rng.integers(1, 12)))


def test_settled_needs_a_margin():
  # a value one rounding step under stop_eigenvalue does not settle a descending prefix
  assert not ew.settled([5.0, 1.0, 1e-2 * (1 - 1e-9)], True, None, 1e-2, RATIO, None)
  assert ew.settled([5.0, 1.0, 1e-3], True, None, 1e-2, RATIO, None)
  # ascending: best gap 3/1.5 = 2 against the bound lambda_max / w[-1] = 2 (a tie) -> not settled
  w = [0.0, 1.5, 3.0]
  assert not ew.settled(w, False, None, 1e-2, RATIO, 6.0)
  assert ew.settled(w, False, None, 1e-2, RATIO, 5.9)
  # lambda_max unknown, or w[-1] + eps <= 0: never settled
  assert not ew.settled(w, False, None, 1e-2, RATIO, None)
  assert not ew.settled([0.0, -1e-3, -1e-3], False, None, 1e-2, RATIO, 1.0)


def spectrum_matrix(values, seed=0):
  rng = np.random.default_rng(seed)
  q, _ = np.linalg.qr(rng.standard_normal((len(values), len(values))))
  return (q * np.asarray(values)) @ q.T


@pytest.mark.parametrize("descend", [True, False])
def test_window_loop_finds_a_value_repeated_more_often_than_a_window_is_wide(descend):
  n = 300
  rng = np.random.default_rng(1)
  if descend:     # 20 copies of the top value, a slow decay, then values under stop_eigenvalue
    values = np.concatenate([np.full(20, 50.0), 5.0 * 0.8 ** np.arange(30), rng.uniform(0, 1e-3, n - 50)])
  else:           # Laplacian-like: 20 nearly disconnected components, then the rest
    values = np.concatenate([np.full(20, 0.01), rng.uniform(0.5, 2.0, n - 20)])
  a = spectrum_matrix(values)
  ops = ew.NumpyOps(a, descend)
  got = ew.solve(ops, descend, None, None, 1e-2, RATIO, n=n)
  want = np.sort(values)[::-1] if descend else np.sort(values)
  m = len(got.values)
  assert m % ew.WINDOW_PAIRS == 0 and m > 20
  np.testing.assert_allclose(got.values, want[:m], atol=1e-9)
  assert ew.settled(got.values, descend, None, 1e-2, RATIO, float(values.max()))
  k, gap = count(got.values, descend, RATIO, None if descend else got.lambda_max)
  k_full, gap_full = count(want, descend, RATIO)
  assert k == k_full and gap == pytest.approx(gap_full, rel=1e-9)   # values exact to rounding
  if not descend:
    assert count(want, descend, RATIO)[0] == 20
  v = ops.vectors(got.order)
  np.testing.assert_allclose(v.T @ v, np.eye(m), atol=1e-9)
  np.testing.assert_allclose(a @ v, v * got.values[None, :], atol=1e-8)


def test_window_loop_bounded_min_clusters_and_cap(monkeypatch):
  n = 200
  values = np.concatenate([[9.0, 8.0, 7.0], np.linspace(1.0, 0.5, n - 3)])   # never < 1e-2
  a = spectrum_matrix(values, seed=2)
  got = ew.solve(ew.NumpyOps(a, True), True, 40, None, 1e-2, RATIO, n=n)
  assert len(got.values) == 48 and got.windows == 3                          # >= 41 values
  got = ew.solve(ew.NumpyOps(a, True), True, 5, 20, 1e-2, RATIO, n=n)
  assert len(got.values) == 32                                               # min_clusters = 20
  monkeypatch.setattr(ew, "MAX_WINDOW_PAIRS", 64)
  with pytest.raises(NotImplementedError, match="first 64 eigenvalues"):
    ew.solve(ew.NumpyOps(a, True), True, None, None, 1e-2, RATIO, n=n)
  with pytest.raises(NotImplementedError, match="max_clusters=70 .* 64"):
    ew.solve(ew.NumpyOps(a, True), True, 70, None, 1e-2, RATIO, n=n)
  monkeypatch.setattr(ew, "MAX_WINDOW_PAIRS", 4)      # windows never pass the cap
  ops = ew.NumpyOps(a, True)
  with pytest.raises(NotImplementedError, match="first 4 eigenvalues"):
    ew.solve(ops, True, None, None, 1e-2, RATIO, n=n)
  assert ops.u.shape[1] == 4
  # the whole spectrum found: the loop ends even though nothing settles
  monkeypatch.setattr(ew, "MAX_WINDOW_PAIRS", 512)
  got = ew.solve(ew.NumpyOps(a[:40, :40], True), True, None, None, -1.0, RATIO, n=40)
  assert len(got.values) == 40


# ---- routing: which solver _eigen_on_device runs above the dense solver's n


class WindowEngine(FakeEngine):
  """FakeEngine plus the windowed solve; its spectrum falls under stop_eigenvalue at value 10."""
  device = "cpu"

  @staticmethod
  def _spectrum(count, which):
    w = np.array([5.0, 4.0, 3.0] + [0.5 * 0.5 ** i for i in range(max(count - 3, 0))])[:count]
    return w if which == nat.EIG_LARGEST else 5.0 - w

  def eigh_window(self, s, n, delta, left, right, sign, which, n_values, locked, n_locked, scale):
    self._rec("window", which, n_values, n_locked)
    return self._spectrum(n_locked + n_values, which)[n_locked:], np.array([16, 0, 16, 1])

  def eigh_mapback(self, u, n, cols, left, right):
    self._rec("mapback", list(cols))
    return "V"


@pytest.mark.parametrize("case,calls,solver", [
    ((40000, None, None, None, RATIO, True),
     [("window", L, 16, 0), ("mapback", [0, 1, 2])], "lanczos-windows"),
    ((40000, None, None, LT.GraphCut, NDIFF, True),
     [("window", S, 16, 0), ("eigh", L, 1, 0, False), ("mapback", [0, 1, 2])], "lanczos-windows"),
    ((40000, 40, None, None, RATIO, True),
     [("window", L, 16, 0), ("window", L, 16, 16), ("window", L, 16, 32), ("mapback", [0, 1, 2])],
     "lanczos-windows"),
    ((40000, None, 20, None, RATIO, True),
     [("window", L, 16, 0), ("window", L, 16, 16), ("mapback", list(range(20)))], "lanczos-windows"),
    ((40000, 10, None, None, RATIO, True), [("eigh", L, 11, 11, False)], "lanczos"),
    ((32768, None, None, None, RATIO, True), [("eigh_dense_pick", L, 3)], "dense"),
    ((2000, None, None, None, RATIO, False), [("arnoldi", False, 16, 16)], "krylov-schur"),
    ((2000, None, None, LT.GraphCut, RATIO, False),
     [("arnoldi", True, 16, 16), ("arnoldi", False, 1, 0)], "krylov-schur"),
    ((1024, None, None, None, RATIO, False), [("arnoldi", False, 1024, 1024)], "krylov-schur"),
])
def test_eigen_stage_routes_above_the_dense_limit(monkeypatch, case, calls, solver):
  from spectralcluster_b200 import arnoldi
  n, max_clusters, min_clusters, laplacian, eigengap, symmetric = case
  eng = WindowEngine(n)

  def fake_arnoldi(eng_, s, n_, delta, left, right, sign, smallest, n_values, n_vectors):
    eng_._rec("arnoldi", smallest, n_values, n_vectors)
    return WindowEngine._spectrum(n_values, S if smallest else L), "V", [0, 0, 0, 0]

  monkeypatch.setattr(arnoldi, "eig_extremal_device", fake_arnoldi)
  sc = scb.SpectralClusterer(min_clusters=min_clusters, max_clusters=max_clusters,
                             laplacian_type=laplacian, eigengap_type=eigengap)
  w, v, k, gap = sc._eigen_on_device(eng, scb.spectral_clusterer.DeviceAffinity("A", n, None,
                                                                                 symmetric))
  solves = [c for c in eng.calls if c[0] != "row_stats"]
  assert solves == calls
  assert v == "V" and k == 3
  assert sc.last_details["solver"] == solver
  limit = n if not max_clusters else min(n, max_clusters + 1)
  assert len(sc.last_details["eigenvalues"]) == min(limit, len(w))
  if solver == "lanczos-windows":
    want = WindowEngine._spectrum(len(w), L if laplacian is None else S)
    np.testing.assert_array_equal(sc.last_details["eigenvalues"], want)
    assert sc.last_details["lanczos_stats"]["windows"] == sum(c[0] == "window" for c in calls)
    if max_clusters:
      assert len(w) == max_clusters + 1



def test_dense_limit_mirrors_the_native_guard():
  import os
  src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                          "spectralcluster_b200", "csrc", "eigh_dense.cu")).read()
  assert "SC_REQUIRE(n <= %d," % scb.spectral_clusterer.DENSE_MAX_N in src


def lanczos_block_size(n_values):
  """sc_eigh_block_size restated: vectors per block for n_values pairs."""
  return 4 if n_values <= 4 else 8 if n_values <= 8 else 12 if n_values <= 12 else 16


@pytest.mark.parametrize("limit", range(1, scb.spectral_clusterer.LANCZOS_MAX_PAIRS + 1))
def test_lanczos_fits_implies_the_native_basis_requirement(limit):
  """Whenever predict() picks one Lanczos solve (lanczos_fits), sc_eigh_extremal takes it: with
  b = sc_eigh_block_size(limit) it needs n >= 2 * 7 * b (six processed blocks and the one in
  flight, twice)."""
  fits = [n for n in range(1, 2048) if scb.spectral_clusterer.lanczos_fits(n, limit)]
  assert fits and fits == list(range(fits[0], 2048))           # monotone in n
  assert fits[0] >= 2 * 7 * lanczos_block_size(limit)
