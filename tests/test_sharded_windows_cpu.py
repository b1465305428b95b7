"""CPU: which options predict_sharded() takes now that it solves in eigenvalue windows
(max_clusters None or >= 32), and what it still refuses -- all before any launch."""

import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import eigen_windows, sharded

GC = scb.LaplacianType.GraphCut
N = 40000


def clusterer(**kw):
  kw.setdefault("min_clusters", 2)
  return scb.SpectralClusterer(refinement_options=scb.configs.icassp2018_refinement_options,
                               custom_dist="cosine", **kw)


@pytest.mark.parametrize("max_clusters", [None, 32, 511])
@pytest.mark.parametrize("laplacian_type", [None, GC])
def test_windows_accepted(max_clusters, laplacian_type):
  c = clusterer(max_clusters=max_clusters, laplacian_type=laplacian_type)
  sharded.check_sharded_options(c, N)
  assert sharded.windowed(c)


@pytest.mark.parametrize("max_clusters", [None, 10, 40])
def test_normalized_diff_on_a_laplacian_accepted(max_clusters):
  c = clusterer(max_clusters=max_clusters, laplacian_type=GC,
                eigengap_type=scb.EigenGapType.NormalizedDiff)
  sharded.check_sharded_options(c, N)
  assert sharded.windowed(c) == (max_clusters != 10)


def test_up_to_31_keeps_the_single_solve():
  assert not sharded.windowed(clusterer(max_clusters=31))
  assert sharded.windowed(clusterer(max_clusters=32))


@pytest.mark.parametrize("max_clusters", [512, 600])
def test_bounded_above_the_cap_refused_with_the_windows_wording(max_clusters):
  c = clusterer(max_clusters=max_clusters, laplacian_type=GC)
  want = str(eigen_windows._cap_error(max_clusters, eigen_windows.MAX_WINDOW_PAIRS))
  with pytest.raises(NotImplementedError) as err:
    sharded.check_sharded_options(c, N)
  assert str(err.value) == want
  assert "needs %d eigenpairs" % (max_clusters + 1) in want


def test_cap_is_read_when_checked(monkeypatch):
  monkeypatch.setattr(eigen_windows, "MAX_WINDOW_PAIRS", 4)
  with pytest.raises(NotImplementedError, match="MAX_WINDOW_PAIRS = 4"):
    sharded.check_sharded_options(clusterer(max_clusters=32, laplacian_type=GC), N)
  # the single Lanczos solve and an unbounded solve are not refused up front
  sharded.check_sharded_options(clusterer(max_clusters=10, laplacian_type=GC), N)
  sharded.check_sharded_options(clusterer(max_clusters=None, laplacian_type=GC), N)


@pytest.mark.parametrize("kw, match", [
    (dict(autotune=scb.AutoTune(p_percentile_min=0.6, p_percentile_max=0.95,
                                init_search_step=0.05, search_level=1)), "AutoTune"),
    (dict(min_clusters=1), "single-cluster"),
    (dict(constraint_options=scb.ConstraintOptions(
        constraint_name=scb.ConstraintName.ConstraintPropagation,
        apply_before_refinement=True)), "constraints"),
    (dict(affinity_function=lambda x: x @ x.T), "affinity"),
    (dict(max_spectral_size=1000), "max_spectral_size"),
])
@pytest.mark.parametrize("max_clusters", [None, 40])
def test_still_refused(kw, match, max_clusters):
  c = clusterer(max_clusters=max_clusters, laplacian_type=GC, **kw)
  with pytest.raises(NotImplementedError, match=match):
    sharded.check_sharded_options(c, N)


def test_n_below_the_windows_basis_refused():
  # max_clusters=None locks up to min(n, 512) pairs; the last window starts with 16 fewer and
  # needs 2 x 112 more rows than it locks
  basis = 2 * eigen_windows.WINDOW_BASIS
  assert basis == 224
  smallest = basis - eigen_windows.WINDOW_PAIRS + eigen_windows.MAX_WINDOW_PAIRS
  sharded.check_sharded_options(clusterer(max_clusters=None, laplacian_type=GC), smallest)
  with pytest.raises(ValueError, match="too small for the windowed Lanczos basis"):
    sharded.check_sharded_options(clusterer(max_clusters=None, laplacian_type=GC), smallest - 1)
  # bounded: 41 values + one window of overshoot
  c = clusterer(max_clusters=40, laplacian_type=GC)
  sharded.check_sharded_options(c, 57 - 16 + basis)
  with pytest.raises(ValueError, match="too small for the windowed Lanczos basis"):
    sharded.check_sharded_options(c, 57 - 16 + basis - 1)


def test_locked_set_capacity():
  # predict() and predict_sharded() size their locked sets with it
  assert eigen_windows.capacity(40000, None, 2) == 512
  assert eigen_windows.capacity(40000, 40, 2) == 57
  assert eigen_windows.capacity(40000, 40, 60) == 76
  assert eigen_windows.capacity(40000, 600, 2) == 512
  assert eigen_windows.capacity(300, None, 2) == 300
