"""GPU: the windowed block Lanczos solve (sc_eigh_extremal_locked + eigen_windows.py) that serves
max_clusters=None and max_clusters >= 32 above the dense solver's N, and the growing Krylov-Schur
solve of the non-symmetrisable path with max_clusters=None.

Tolerance on eigenvalues, as elsewhere in the suite: |dw| <= 1e-5 |w| + 1e-6 lambda_max."""

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import eigen_windows as ew
from oracle import spectral_oracle as orc

import fp64_checker

pytestmark = pytest.mark.gpu

RN = scb.RefinementName


def assert_values_close(w, want):
  w, want = np.asarray(w), np.asarray(want)
  np.testing.assert_allclose(w, want, rtol=1e-5, atol=1e-6 * np.abs(want).max())


def icassp_options():
  return scb.RefinementOptions(
      gaussian_blur_sigma=1, p_percentile=0.95, thresholding_soft_multiplier=0.01,
      refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))


def test_windows_against_dense_on_a_value_repeated_20_times(engine):
  """Four windows of 16 on a block-diagonal affinity whose top eigenvalue repeats 20 times (more
  often than one window is wide) against the dense solver."""
  rng = np.random.default_rng(20)
  size, copies, n = 400, 20, 8192
  block = orc.affinity(rng.standard_normal((size, 16)))
  a = np.zeros((n, n))
  for i in range(copies):
    a[i * size:(i + 1) * size, i * size:(i + 1) * size] = block
  rest = n - copies * size
  a[copies * size:, copies * size:] = 0.5 * orc.affinity(rng.standard_normal((rest, 16)))
  s = engine.upload_matrix(a)
  ops = ew.DeviceOps(engine, s, n, None, None, None, 1.0, nat.EIG_LARGEST, capacity=64)
  found = np.concatenate([ops.window(16) for _ in range(4)])
  order = np.argsort(-found, kind="stable")
  w = found[order]
  w_dense, v_dense, _ = engine.eigh(s, n, None, None, None, 1.0, nat.EIG_LARGEST, 64, 64, True)
  lam = float(np.abs(w_dense).max())
  np.testing.assert_allclose(w, w_dense, rtol=1e-5, atol=1e-6 * lam)
  top = np.linalg.eigvalsh(block)[-1]
  assert np.all(np.abs(w[:copies] - top) <= 1e-5 * top)              # every copy found
  assert abs(w[copies] - top) > 1e-3 * top
  v = ops.vectors(order).cpu().numpy()
  vd = v_dense.cpu().numpy()
  for j in range(64):
    sep = min([abs(w_dense[j] - w_dense[i]) for i in (j - 1, j + 1) if 0 <= i < 64] or [np.inf])
    if j < 63 and sep > 1e-3 * lam:                                 # the 64th has no right neighbour here
      assert abs(v[:, j] @ vd[:, j]) >= 1 - 1e-6, j
  assert ops.stats["windows"] == 4


def checker_prefix(s, laplacian, count):
  terms = fp64_checker.operator_terms(s, laplacian)
  return fp64_checker.extremal_eigh(s, terms, count)


def checker_labels(w, v, descend, max_clusters=None):
  if descend:
    k, _ = orc.number_of_clusters(w, max_clusters, 1e-2, "ratio", descend=True)
  else:
    k, _ = orc.number_of_clusters(w, max_clusters, eigengap="ratio", descend=False)
  return k, orc.run_kmeans(v[:, :k], k)


def test_icassp_max_clusters_none_at_65536(engine):
  """N = 65,536, d = 256, 6 speakers, ICASSP sequence, max_clusters=None: no Laplacian and
  GraphCut against the float64 GPU checker and the generator's ground truth."""
  t = dev.torch()
  n = 65536
  x, truth = orc.synthetic_dvectors(n, 256, 6, seed=0, return_labels=True)
  runs = {}
  for laplacian in (None, "graphcut"):
    c = scb.SpectralClusterer(refinement_options=icassp_options(),
                              laplacian_type=scb.LaplacianType.GraphCut if laplacian else None)
    labels = c.predict(x)
    assert c.last_details["solver"] == "lanczos-windows"
    runs[laplacian] = (labels, np.array(c.last_details["eigenvalues"]), c.last_details["n_clusters"])
  t.cuda.synchronize()
  t.cuda.empty_cache()
  s = fp64_checker.refine_through_diffuse(x, engine.device)
  for laplacian, (labels, w, k) in runs.items():
    w_ref, v_ref = checker_prefix(s, laplacian, len(w))
    assert_values_close(w, w_ref)
    k_ref, labels_ref = checker_labels(w_ref, v_ref, laplacian is None)
    assert k == k_ref == 6, (laplacian, k, k_ref)
    assert np.array_equal(scb.utils.enforce_ordered_labels(labels), orc.ordered(labels_ref))
    assert np.array_equal(scb.utils.enforce_ordered_labels(labels), orc.ordered(truth))
  del s
  t.cuda.empty_cache()


def test_graphcut_max_clusters_40_at_40000(engine, monkeypatch):
  """max_clusters >= 32 above the dense solver's N: all 41 values, k and labels against the
  checker.  Then the same case with the cap lowered to 4 values: it needs at least 7 (6
  speakers), so it raises, naming the cap."""
  t = dev.torch()
  n = 40000
  x = orc.synthetic_dvectors(n, 256, 6, seed=1)
  c = scb.SpectralClusterer(max_clusters=40, refinement_options=icassp_options(),
                            laplacian_type=scb.LaplacianType.GraphCut)
  labels = c.predict(x)
  assert c.last_details["solver"] == "lanczos-windows"
  w = np.array(c.last_details["eigenvalues"])
  assert len(w) == 41
  monkeypatch.setattr(ew, "MAX_WINDOW_PAIRS", 4)
  c_none = scb.SpectralClusterer(refinement_options=icassp_options(),
                                 laplacian_type=scb.LaplacianType.GraphCut)
  with pytest.raises(NotImplementedError, match="first 4 eigenvalues"):
    c_none.predict(x)
  t.cuda.synchronize()
  t.cuda.empty_cache()
  s = fp64_checker.refine_through_diffuse(x, engine.device)
  w_ref, v_ref = checker_prefix(s, "graphcut", 41)
  del s
  t.cuda.empty_cache()
  assert_values_close(w, w_ref)
  k_ref, labels_ref = checker_labels(w_ref, v_ref, False, max_clusters=40)
  assert c.last_details["n_clusters"] == k_ref
  assert np.array_equal(scb.utils.enforce_ordered_labels(labels), orc.ordered(labels_ref))


def test_default_clusterer_at_40000_d64(engine):
  """SpectralClusterer() (no refinement, max_clusters=None) on N = 40,000, d = 64.  The raw
  affinity (X^X^T + 1) / 2 = B B^T with B = [1/sqrt2, X^/sqrt2] has rank d + 1 = 65: its nonzero
  eigenvalues are those of the 65 x 65 matrix B^T B, exactly, in float64.  The eigengap scan stops
  at value d + 2, a rounding artefact in both implementations (fp32 storage of the affinity here,
  float64 in the reference), so k and the labels are not compared."""
  n, d = 40000, 64
  x = orc.synthetic_dvectors(n, d, 5, seed=2)
  c = scb.SpectralClusterer()
  c.predict(x)
  assert c.last_details["solver"] == "lanczos-windows"
  w = np.array(c.last_details["eigenvalues"])
  xh = x / np.linalg.norm(x, axis=1, keepdims=True)
  b = np.concatenate([np.full((n, 1), 1.0), xh], axis=1) / np.sqrt(2.0)
  want = np.linalg.eigvalsh(b.T @ b)[::-1]
  assert len(w) > d + 1
  assert_values_close(w[:d + 1], want)
  assert w[-1] < c.stop_eigenvalue
  assert np.all(w[:d + 1] >= c.stop_eigenvalue)


@pytest.mark.parametrize("laplacian", [None, "graphcut"])
def test_threshold_only_max_clusters_none_at_2500(laplacian):
  """[RowWiseThreshold] alone (non-symmetrisable), N = 2,500 > 1,024, max_clusters=None: the
  growing Krylov-Schur solve against the host oracle (np.linalg.eig, as the reference).  Without a
  Laplacian the scan runs to the first value below stop_eigenvalue; on these inputs (d = 32,
  intra-speaker cosine 0.95) that is value 216 of the oracle's spectrum, within the 256 pairs of the
  largest Krylov-Schur solve (at d = 128 and cosine 0.8 no such value comes before 600)."""
  n = 2500
  d, intra = (32, 0.95) if laplacian is None else (128, 0.8)
  x = orc.synthetic_dvectors(n, d, 4, seed=4, intra_cos=intra)
  c = scb.SpectralClusterer(
      refinement_options=scb.RefinementOptions(refinement_sequence=[RN.RowWiseThreshold]),
      laplacian_type=scb.LaplacianType.GraphCut if laplacian else None)
  labels = c.predict(x)
  assert c.last_details["solver"] == "krylov-schur"
  w = np.array(c.last_details["eigenvalues"])
  assert len(w) < n
  opt = orc.options(sequence=("threshold",), laplacian=laplacian)
  labels_ref, det = orc.predict(x, opt, return_details=True)
  w_ref = np.asarray(det["eigenvalues"])
  np.testing.assert_allclose(w, w_ref[:len(w)], rtol=1e-5, atol=1e-6 * np.abs(w_ref).max())
  assert c.last_details["n_clusters"] == det["n_clusters"]
  assert np.array_equal(scb.utils.enforce_ordered_labels(labels), orc.ordered(labels_ref))
