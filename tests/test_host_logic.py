"""CPU: host-side logic of the GPU path that needs no GPU -- the symbolic Laplacian terms
(SURVEY.md A.2) against the oracle's materialised Laplacians, and the refinement planner's fusion
decisions against a recording fake engine."""

import numpy as np
import pytest
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import laplacian as lap
from oracle import spectral_oracle as orc

RN = scb.RefinementName


@pytest.mark.parametrize("kind,ltype", [
    (None, None), ("unnormalized", scb.LaplacianType.Unnormalized),
    ("randomwalk", scb.LaplacianType.RandomWalk), ("graphcut", scb.LaplacianType.GraphCut)])
@pytest.mark.parametrize("row_normalised", [False, True])
def test_operator_terms_reproduce_the_reference_matrix(kind, ltype, row_normalised):
  """diag(delta) + sign*diag(left) S diag(right) == what the reference hands to np.linalg.eig, and
  its symmetrised form has the same spectrum; v = E u / |E u| are its eigenvectors."""
  rng = np.random.default_rng(0)
  x = rng.standard_normal((60, 8))
  s = orc.diffuse(orc.symmetrize(orc.row_threshold(orc.affinity(x), 0.9, 0.01)))
  r = 1.0 / s.max(axis=1) if row_normalised else None
  w_ref = s if r is None else orc.row_normalize(s)
  m_ref = w_ref if kind is None else orc.laplacian(w_ref, kind)
  rowsum = torch.from_numpy(s.sum(axis=1))
  rt = None if r is None else torch.from_numpy(r)
  delta, left, right, sign, which = lap.terms_from_row_sums(rowsum, rt, ltype)
  one = np.ones(60)
  d = np.zeros(60) if delta is None else delta.numpy()
  le = one if left is None else left.numpy()
  ri = one if right is None else right.numpy()
  m = np.diag(d) + sign * le[:, None] * s * ri[None, :]
  np.testing.assert_allclose(m, m_ref, rtol=1e-12, atol=1e-12)
  assert which == (nat.EIG_LARGEST if kind is None else nat.EIG_SMALLEST)
  c = np.sqrt(le * ri)
  t = np.diag(d) + sign * c[:, None] * s * c[None, :]
  np.testing.assert_allclose(t, t.T, atol=1e-12)
  wt, u = np.linalg.eigh(t)
  wm = np.sort(np.linalg.eigvals(m).real)
  np.testing.assert_allclose(wt, wm, rtol=1e-8, atol=1e-9)
  e = np.sqrt(le / ri)
  v = e[:, None] * u
  v /= np.linalg.norm(v, axis=0)
  np.testing.assert_allclose(m @ v, v * wt[None, :], atol=1e-8 * max(1.0, np.abs(wt).max()))


class FakeEngine:
  """Records the device calls run_refinement() makes; returns opaque tokens."""

  def __init__(self, n, tensor_cores=True):
    self.calls, self.n, self.tc = [], n, tensor_cores

  def gemm_engine(self, n):
    return nat.GEMM_TCGEN05 if self.tc else nat.GEMM_SIMT

  def _rec(self, name, *info):
    self.calls.append((name,) + info)
    return name

  def crop_values(self, a, n): return self._rec("crop_values")
  def crop_diagonal(self, a, n): return self._rec("crop_diagonal")
  def gaussian_blur(self, a, n, sigma, diag=None): return self._rec("gaussian_blur", sigma)
  def row_threshold(self, a, n, *args): return self._rec("row_threshold", args[0])
  def symmetrize(self, a, n, kind): return self._rec("symmetrize", kind)
  def blur_rowmax(self, a, n, sigma, diag, zero_diag): return self._rec("blur_rowmax", sigma, diag)

  gemm_precision = nat.GEMM_SPLIT3

  def upper_pass_ok(self, sigma):
    return dev.Engine.upper_pass_ok(sigma)

  def blur_upper_rowmax(self, a, n, sigma, diag, zero_diag):
    self._rec("blur_upper", sigma, diag)
    return "B", "m"

  def threshold_symmetrize_upper(self, b, n, m, p, mult, binarize, keep, sym, want_f32, want_planes,
                                 want_lo=True):
    self._rec("thrsym_upper", b, m, sym, want_f32, want_planes)
    return ("y" if want_f32 else None, "hi" if want_planes else None, "lo" if want_planes else None)

  def blur_threshold_symmetrize(self, a, n, sigma, diag, m, p, mult, binarize, keep, sym, want_f32,
                                want_planes):
    self._rec("blur_thrsym", sigma, diag, sym, want_f32, want_planes)
    return ("y" if want_f32 else None, "hi" if want_planes else None, "lo" if want_planes else None)

  def diffuse(self, n, y=None, hi=None, lo=None, want_stats=False, precision=None):
    self._rec("diffuse", y, hi, want_stats)
    if want_stats:    # (rowmax fp32, rowsum fp64) from the GEMM epilogue
      return "S", torch.ones(self.n, dtype=torch.float32) * 2.0, torch.ones(self.n, dtype=torch.float64) * 3.0
    return "S", None, None
  def row_normalize(self, a, n): return self._rec("row_normalize")

  def row_stats(self, a, n, want_max=True, want_sum=True):
    self._rec("row_stats", want_max, want_sum)
    return (torch.ones(self.n, dtype=torch.float64) * 2.0,
            torch.ones(self.n, dtype=torch.float64) * 3.0 if want_sum else None)

  # ---- eigen stage: which solver runs, with which arguments
  dense_eig_max = 0

  def diffuse_precision_for(self, n):
    return None

  @staticmethod
  def _spectrum(count, which):
    # a clear gap after the third value, in the order the solver returns them
    w = np.array([5.0, 4.0, 3.0] + [0.5 * 0.999 ** i for i in range(max(count - 3, 0))])[:count]
    return w if which == nat.EIG_LARGEST else 5.0 - w

  def eigh(self, s, n, delta, left, right, sign, which, n_values, n_vectors, dense, tol=1e-9,
           max_matvecs=0):
    self._rec("eigh", which, n_values, n_vectors, dense)
    return self._spectrum(n_values, which), "V", np.zeros(4, dtype=np.int64)

  def eigh_dense_pick(self, s, n, delta, left, right, sign, which, picker):
    w = self._spectrum(n, which)
    self._rec("eigh_dense_pick", which, picker(w))
    return w, "V"


def names(eng):
  return [c[0] for c in eng.calls]


def test_planner_fuses_the_icassp_sequence():
  eng = FakeEngine(1000)
  opt = scb.RefinementOptions(refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))
  out = dev.run_refinement(eng, "A", 1000, opt, crop_vector="cropvec")
  # sigma = 1: the symmetric blur pair (upper tiles blurred once, result mirrored);
  # RowWiseNormalize's row maxima (and the degree) come out of the Diffuse epilogue: no row_stats
  assert names(eng) == ["blur_upper", "thrsym_upper", "diffuse"]
  assert eng.calls[0][1:] == (1.0, "cropvec")            # crop vector from the affinity epilogue
  assert eng.calls[1][1:] == ("B", "m", nat.SYMMETRIZE_MAX, False, True)   # planes only: Diffuse follows
  assert eng.calls[2][1:] == (None, "hi", True)          # tensor-core Diffuse on the planes
  assert out.symmetric and torch.allclose(out.row_scale, torch.full((1000,), 0.5, dtype=torch.float64))
  assert torch.allclose(out.rowsum, torch.full((1000,), 3.0, dtype=torch.float64))


def test_planner_variants():
  # no crop vector supplied -> crop values computed; sigma 0 -> fused chain without blur
  eng = FakeEngine(500)
  opt = scb.RefinementOptions(gaussian_blur_sigma=0, symmetrize_type=scb.SymmetrizeType.Average,
                              refinement_sequence=[RN.CropDiagonal, RN.RowWiseThreshold,
                                                   RN.Symmetrize])
  out = dev.run_refinement(eng, "A", 500, opt)
  assert names(eng) == ["crop_values", "blur_rowmax", "blur_thrsym"]
  assert eng.calls[2][1] == 0.0 and eng.calls[2][3:] == (nat.SYMMETRIZE_AVERAGE, True, False)
  assert out.symmetric and out.row_scale is None
  # small matrices use the SIMT GEMM: fp32 Y is kept instead of planes
  eng = FakeEngine(20, tensor_cores=False)
  opt = scb.RefinementOptions(refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))
  dev.run_refinement(eng, "A", 20, opt, crop_vector="c")
  assert eng.calls[1][4:] == (True, False) and eng.calls[2][1:] == ("y", None, False)
  assert names(eng)[-1] == "row_stats"                   # SIMT GEMM: separate reduction pass
  # a blur radius other than 4 keeps the two-pass form (blur recomputed in both passes)
  eng = FakeEngine(1000)
  opt = scb.RefinementOptions(gaussian_blur_sigma=2, refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))
  dev.run_refinement(eng, "A", 1000, opt, crop_vector="c")
  assert names(eng)[:2] == ["blur_rowmax", "blur_thrsym"]
  # Percentile thresholding and threshold-without-symmetrize are not fusable
  eng = FakeEngine(300)
  opt = scb.RefinementOptions(thresholding_type=scb.ThresholdType.Percentile,
                              refinement_sequence=[RN.RowWiseThreshold, RN.Symmetrize])
  out = dev.run_refinement(eng, "A", 300, opt)
  assert names(eng) == ["row_threshold", "symmetrize"] and out.symmetric
  eng = FakeEngine(300)
  out = dev.run_refinement(eng, "A", 300, scb.RefinementOptions(
      refinement_sequence=[RN.GaussianBlur, RN.RowWiseThreshold]))
  assert names(eng) == ["gaussian_blur", "row_threshold"] and not out.symmetric
  # RowWiseNormalize in the middle is materialised and breaks symmetry until Diffuse restores it
  eng = FakeEngine(300)
  out = dev.run_refinement(eng, "A", 300, scb.RefinementOptions(
      refinement_sequence=[RN.RowWiseNormalize, RN.Diffuse]))
  assert names(eng) == ["row_normalize", "diffuse"] and out.symmetric
  with pytest.raises(ValueError):
    dev.run_refinement(FakeEngine(10), "A", 10, scb.RefinementOptions(refinement_sequence=["x"]))


L, S = nat.EIG_LARGEST, nat.EIG_SMALLEST
UNNORM = scb.LaplacianType.Unnormalized
RATIO, NDIFF = scb.EigenGapType.Ratio, scb.EigenGapType.NormalizedDiff


# (n, max_clusters, min_clusters, laplacian, eigengap, symmetric, dense_eig_max) ->
# (solver calls in order, last_details["solver"]).  max_clusters = 10: the Lanczos basis is 64
# vectors, so Lanczos needs n >= 256; max_clusters = 31: basis 96, n >= 384.
@pytest.mark.parametrize("case,calls,solver", [
    ((2000, 10, None, None, RATIO, True, 0), [("eigh", L, 11, 11, False)], "lanczos"),
    ((256, 10, None, None, RATIO, True, 0), [("eigh", L, 11, 11, False)], "lanczos"),
    ((255, 10, None, None, RATIO, True, 0), [("eigh", L, 255, 11, True)], "dense"),
    ((2000, 10, 15, None, RATIO, True, 0), [("eigh", L, 11, 15, False)], "lanczos"),
    ((2000, 10, None, None, RATIO, True, 2000), [("eigh", L, 2000, 11, True)], "dense"),
    ((2000, 31, None, None, RATIO, True, 0), [("eigh", L, 32, 32, False)], "lanczos"),
    ((383, 31, None, None, RATIO, True, 0), [("eigh", L, 383, 32, True)], "dense"),
    ((2000, 32, None, None, RATIO, True, 0), [("eigh", L, 2000, 33, True)], "dense"),
    ((2000, None, None, None, RATIO, True, 0), [("eigh_dense_pick", L, 3)], "dense"),
    ((2000, None, 5, UNNORM, RATIO, True, 0), [("eigh_dense_pick", S, 5)], "dense"),
    ((200, None, None, None, RATIO, True, 0), [("eigh", L, 200, 200, True)], "dense"),
    ((2000, 10, None, UNNORM, RATIO, True, 0), [("eigh", S, 11, 11, False)], "lanczos"),
    ((2000, 10, None, UNNORM, NDIFF, True, 0),
     [("eigh", S, 11, 11, False), ("eigh", L, 1, 0, False)], "lanczos"),
    ((2000, 10, None, None, NDIFF, True, 0), [("eigh", L, 11, 11, False)], "lanczos"),
    ((200, 10, None, UNNORM, NDIFF, True, 0), [("eigh", S, 200, 11, True)], "dense"),
    ((2000, None, None, UNNORM, NDIFF, True, 0), [("eigh_dense_pick", S, 3)], "dense"),
    ((2000, 10, None, None, RATIO, False, 0), [("arnoldi", False, 11, 11)], "krylov-schur"),
    ((2000, 10, 15, None, NDIFF, False, 0), [("arnoldi", False, 11, 15)], "krylov-schur"),
    ((2000, 10, None, UNNORM, RATIO, False, 0), [("arnoldi", True, 11, 11)], "krylov-schur"),
    ((2000, 10, None, UNNORM, NDIFF, False, 0),
     [("arnoldi", True, 11, 11), ("arnoldi", False, 1, 0)], "krylov-schur"),
    ((200, None, None, UNNORM, NDIFF, False, 0), [("arnoldi", True, 200, 200)], "krylov-schur"),
])
def test_eigen_stage_solver_choice(monkeypatch, case, calls, solver):
  """Which eigensolver _eigen_on_device() runs, with which arguments, and whether it adds the
  lambda_max solve NormalizedDiff needs on an ascending spectrum."""
  from spectralcluster_b200 import arnoldi
  n, max_clusters, min_clusters, laplacian, eigengap, symmetric, dense_eig_max = case
  eng = FakeEngine(n)
  eng.dense_eig_max = dense_eig_max

  def fake_arnoldi(eng_, s, n_, delta, left, right, sign, smallest, n_values, n_vectors):
    eng_._rec("arnoldi", smallest, n_values, n_vectors)
    return FakeEngine._spectrum(n_values, S if smallest else L), "V", [0, 0, 0, 0]

  monkeypatch.setattr(arnoldi, "eig_extremal_device", fake_arnoldi)
  sc = scb.SpectralClusterer(min_clusters=min_clusters, max_clusters=max_clusters,
                             laplacian_type=laplacian, eigengap_type=eigengap)
  w, v, k, gap = sc._eigen_on_device(eng, scb.spectral_clusterer.DeviceAffinity("A", n, None,
                                                                                 symmetric))
  solves = [c for c in eng.calls if c[0] != "row_stats"]
  assert solves == calls
  assert v == "V" and k == 3
  assert sc.last_details["solver"] == solver
  assert sc.last_details["n_clusters_raw"] == k and sc.last_details["max_gap"] == gap
  limit = n if not max_clusters else min(n, max_clusters + 1)
  assert len(sc.last_details["eigenvalues"]) == min(limit, len(w))
  assert (sc.last_details["lanczos_stats"] is None) == (solver == "dense")


class StallingEngine(FakeEngine):
  """A FakeEngine whose Lanczos solves of more than one pair stop short of convergence."""

  def __init__(self, n, message="sc_eigh_extremal: only 7 of 26 eigenpairs converged to 1e-09 in "
               "20000 matrix-vector products"):
    super().__init__(n)
    self.message = message

  def eigh(self, s, n, delta, left, right, sign, which, n_values, n_vectors, dense, tol=1e-9,
           max_matvecs=0):
    if not dense and n_values > 1:
      self._rec("eigh", which, n_values, n_vectors, dense)
      raise nat.NativeError(self.message)
    return super().eigh(s, n, delta, left, right, sign, which, n_values, n_vectors, dense)


@pytest.mark.parametrize("eigengap", [RATIO, NDIFF])
def test_unconverged_lanczos_falls_back_to_the_dense_solver(eigengap):
  """A stored S whose Lanczos solve does not converge is solved by the dense solver, as on the
  dense route (the whole spectrum, so no lambda_max solve), and last_details says why."""
  eng = StallingEngine(2000)
  sc = scb.SpectralClusterer(max_clusters=25, laplacian_type=UNNORM, eigengap_type=eigengap)
  w, v, k, gap = sc._eigen_on_device(eng, scb.spectral_clusterer.DeviceAffinity("A", 2000))
  solves = [c for c in eng.calls if c[0] != "row_stats"]
  assert solves == [("eigh", S, 26, 26, False), ("eigh", S, 2000, 26, True)]
  assert sc.last_details["solver"] == "dense" and sc.last_details["lanczos_stats"] is None
  assert "eigenpairs converged" in sc.last_details["lanczos_fallback"]
  assert len(sc.last_details["eigenvalues"]) == 26 and k == 3 and v == "V"


def test_other_lanczos_errors_and_large_n_still_raise():
  """Only non-convergence falls back, and only where the dense solver takes n."""
  sc = scb.SpectralClusterer(max_clusters=25, laplacian_type=UNNORM)
  eng = StallingEngine(2000, message="sc_eigh_extremal: bad arguments")
  with pytest.raises(nat.NativeError, match="bad arguments"):
    sc._eigen_on_device(eng, scb.spectral_clusterer.DeviceAffinity("A", 2000))
  n = scb.spectral_clusterer.DENSE_MAX_N + 1
  with pytest.raises(nat.NativeError, match="eigenpairs converged"):
    sc._eigen_on_device(StallingEngine(n), scb.spectral_clusterer.DeviceAffinity("A", n))
