"""GPU: SpectralClusterer.predict() on the GPU against the golden fixtures produced by the
unmodified reference (tests/golden/make_golden.py) and against the oracle run side by side.

Parity bar (BASELINE.json north_star): labels identical after utils.enforce_ordered_labels;
eigenvalues within 1e-5 relative.  fp32 storage of the N x N matrices adds an absolute floor of
1e-6 * lambda_max to that tolerance (near-zero eigenvalues -- the Laplacian's lambda_0 and
tail values far below lambda_max -- have no meaningful relative error)."""

import numpy as np
import pytest

import spectralcluster_b200 as scb
from conftest import golden_names, load_golden
from oracle import spectral_oracle as orc

pytestmark = pytest.mark.gpu

RN = scb.RefinementName
NAME = {"crop": RN.CropDiagonal, "blur": RN.GaussianBlur, "threshold": RN.RowWiseThreshold,
        "symmetrize": RN.Symmetrize, "diffuse": RN.Diffuse, "rownorm": RN.RowWiseNormalize}
LAP = {None: None, "affinity": scb.LaplacianType.Affinity,
       "unnormalized": scb.LaplacianType.Unnormalized,
       "randomwalk": scb.LaplacianType.RandomWalk, "graphcut": scb.LaplacianType.GraphCut}
GAP = {"ratio": scb.EigenGapType.Ratio, "normalizeddiff": scb.EigenGapType.NormalizedDiff}
TT = {"rowmax": scb.ThresholdType.RowMax, "percentile": scb.ThresholdType.Percentile}
ST = {"max": scb.SymmetrizeType.Max, "average": scb.SymmetrizeType.Average}


def make_clusterer(opt):
  """Fresh objects from an oracle option bag (reads like the reference's own tests)."""
  ro = scb.RefinementOptions(
      gaussian_blur_sigma=opt["sigma"], p_percentile=opt["p"],
      thresholding_soft_multiplier=opt["mult"], thresholding_type=TT[opt["threshold_type"]],
      thresholding_with_binarization=opt["binarize"],
      thresholding_preserve_diagonal=opt["preserve_diagonal"],
      symmetrize_type=ST[opt["symmetrize_type"]],
      refinement_sequence=[NAME[s] for s in opt["sequence"]])
  at = None
  if opt["autotune"]:
    a = opt["autotune"]
    at = scb.AutoTune(p_percentile_min=a["p_min"], p_percentile_max=a["p_max"],
                      init_search_step=a["step"], search_level=a.get("level", 1),
                      proxy=scb.AutoTuneProxy.PercentileSqrtOverNME if a.get("proxy", "sqrt") == "sqrt"
                      else scb.AutoTuneProxy.PercentileOverNME)
  return scb.SpectralClusterer(
      min_clusters=opt["min_clusters"], max_clusters=opt["max_clusters"], refinement_options=ro,
      autotune=at, laplacian_type=LAP[opt["laplacian"]], stop_eigenvalue=opt["stop_eigenvalue"],
      row_wise_renorm=opt["row_wise_renorm"], custom_dist=opt["custom_dist"],
      max_iter=opt["max_iter"], eigengap_type=GAP[opt["eigengap"]])


def check_eigenvalues(got, want, opt):
  m = len(want) if not opt["max_clusters"] else min(len(want), opt["max_clusters"] + 1)
  m = min(m, len(got))
  scale = max(np.max(np.abs(want)), np.max(np.abs(got)))
  tol = 1e-5 * np.abs(want[:m]) + 1e-6 * scale
  err = np.abs(got[:m] - want[:m])
  assert np.all(err <= tol), "eigenvalue mismatch: rel %s" % (err / np.maximum(np.abs(want[:m]), 1e-300))


@pytest.mark.parametrize("name", golden_names())
def test_predict_matches_reference_fixture(name):
  case = load_golden(name)
  opt = case["options"]
  clusterer = make_clusterer(opt)
  labels = clusterer.predict(case["embeddings"])
  assert labels.dtype == np.int64 and labels.shape == case["labels"].shape
  np.testing.assert_array_equal(scb.utils.enforce_ordered_labels(labels),
                                scb.utils.enforce_ordered_labels(case["labels"]))
  if "eigenvalues_head" in case:
    assert clusterer.last_details["n_clusters_raw"] == int(case["n_clusters_raw"])
    check_eigenvalues(clusterer.last_details["eigenvalues"], case["eigenvalues_head"], opt)
  else:
    assert clusterer.last_details["best_p_percentile"] == float(case["p_best"])


@pytest.mark.parametrize("solver", ["dense", "lanczos"])
@pytest.mark.parametrize("lap", [None, "graphcut"])
def test_predict_vs_oracle_side_by_side(engine, solver, lap):
  """Same seeded d-vectors through both implementations, both eigensolvers."""
  n, d, k = 2400, 256, 5
  x = orc.synthetic_dvectors(n, d, k, seed=11)
  opt = orc.options(min_clusters=2, max_clusters=9, sequence=orc.ICASSP2018, laplacian=lap)
  want, det = orc.predict(x, opt, return_details=True)
  old = engine.dense_eig_max
  engine.dense_eig_max = 10 ** 9 if solver == "dense" else 0
  try:
    clusterer = make_clusterer(opt)
    got = clusterer.predict(x)
  finally:
    engine.dense_eig_max = old
  assert clusterer.last_details["solver"] == solver
  np.testing.assert_array_equal(scb.utils.enforce_ordered_labels(got), orc.ordered(want))
  check_eigenvalues(clusterer.last_details["eigenvalues"], det["eigenvalues"][:10], opt)


def test_predict_float32_input_and_preset():
  x = orc.synthetic_dvectors(1000, 128, 4, seed=0).astype(np.float32)
  want = orc.predict(x.astype(np.float64), orc.options(
      min_clusters=2, max_clusters=7, sequence=orc.ICASSP2018))
  got = scb.configs.icassp2018_clusterer.predict(x)
  np.testing.assert_array_equal(scb.utils.enforce_ordered_labels(got), orc.ordered(want))


def test_compute_eigenvectors_ncluster_host_api():
  """The private-but-tested entry point (autotune_test.py:72): host affinity in, host out."""
  x = np.array([[1.0, 0.0], [1.1, 0.1], [0.0, 1.0], [0.1, 1.0], [0.9, -0.1], [0.0, 1.2]])
  c = scb.SpectralClusterer(max_clusters=2, laplacian_type=scb.LaplacianType.GraphCut,
                            refinement_options=scb.RefinementOptions(refinement_sequence=[]))
  v, k, gap = c._compute_eigenvectors_ncluster(orc.affinity(x))
  assert isinstance(v, np.ndarray) and v.shape[0] == 6 and k == 2
  w, vr, kr, gr = orc.eigenvectors_ncluster(orc.affinity(x), orc.options(
      max_clusters=2, laplacian="graphcut"))
  assert kr == k and abs(gap - gr) <= 1e-4 * gr
  for col in range(2):
    assert min(np.abs(v[:, col] - vr[:, col]).max(), np.abs(v[:, col] + vr[:, col]).max()) < 1e-5


def test_option_errors_and_host_side_metrics():
  x = orc.synthetic_dvectors(300, 32, 3, seed=0)
  with pytest.raises(ValueError):        # AutoTune without RowWiseThreshold (spectral_clusterer.py:268-272)
    scb.SpectralClusterer(autotune=scb.AutoTune(), refinement_options=scb.RefinementOptions(
        refinement_sequence=[RN.CropDiagonal])).predict(x)
  # metrics beyond cosine / euclidean follow the reference on the host ([n, k] embeddings)
  opt = orc.options(min_clusters=2, max_clusters=6, sequence=orc.ICASSP2018)
  c = make_clusterer(opt)
  c.custom_dist = "cityblock"
  want = orc.predict(x, dict(opt, custom_dist="cityblock"))
  assert np.array_equal(scb.utils.enforce_ordered_labels(c.predict(x)), orc.ordered(want))
  import sklearn.exceptions
  c.custom_dist = None                   # the reference never fits this estimator (:33-36,51)
  with pytest.raises(sklearn.exceptions.NotFittedError):
    c.predict(x)


def test_user_hooks_still_work():
  x = orc.synthetic_dvectors(500, 64, 3, seed=2)
  calls = {}

  def my_affinity(e):
    calls["aff"] = e.shape
    return orc.affinity(e)

  def my_cluster(spectral_embeddings, n_clusters, custom_dist, max_iter):
    calls["post"] = (spectral_embeddings.shape, n_clusters, custom_dist, max_iter)
    return orc.run_kmeans(spectral_embeddings, n_clusters, custom_dist, max_iter)

  opt = orc.options(min_clusters=2, max_clusters=6, sequence=orc.ICASSP2018)
  want = orc.predict(x, opt)
  c = make_clusterer(opt)
  c.affinity_function = my_affinity
  c.post_eigen_cluster_function = my_cluster
  got = c.predict(x)
  assert calls["aff"] == (500, 64) and calls["post"][1:] == (3, "cosine", 300)
  np.testing.assert_array_equal(scb.utils.enforce_ordered_labels(got), orc.ordered(want))
