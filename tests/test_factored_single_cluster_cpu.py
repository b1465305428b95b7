"""CPU: host logic of the single-cluster checks on the factored route -- the packed band's row
offsets against a plain restatement, its size against Y_hi, and which predict(min_clusters=1)
calls take the factored route (a fake engine stands in for an 80 GB H100)."""

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import gmm_bic as gb

from test_factored_route_cpu import ICASSP, FakeEngine, _not_affinity, _seq

RN = scb.RefinementName
SIZES = [2, 3, 67, 130, 4099, 131072]


def offsets_for(n):
  return [o for o in (-2, 0, 1, 3, 64, n - 2) if o < n - 1]


def restated_row_offsets(n, offset):
  """Row i of np.triu_indices(n, offset): columns [j0, n) stored from c0 = j0 & ~3, in slots of 4."""
  out = [0]
  for i in range(n):
    j0 = max(0, i + offset)
    width = 0
    if j0 < n:
      c0 = j0 - j0 % 4
      width = -(-(n - c0) // 4) * 4
    out.append(out[-1] + width)
  return np.array(out, dtype=np.int64)


CASES = [(n, o) for n in SIZES for o in offsets_for(n)]


@pytest.mark.parametrize("n,offset", CASES)
def test_row_offsets_match_the_restatement(n, offset):
  off = gb.packed_row_offsets(n, offset)
  assert off.dtype == np.int64 and off.shape == (n + 1,)
  np.testing.assert_array_equal(off, restated_row_offsets(n, offset))
  assert (off % 4 == 0).all() and (np.diff(off) >= 0).all()


@pytest.mark.parametrize("n,offset", CASES)
def test_in_band_elements_make_the_band(n, offset):
  off = gb.packed_row_offsets(n, offset)
  j0 = np.maximum(np.arange(n) + offset, 0)
  inband = np.where(j0 < n, n - j0, 0)
  assert int(inband.sum()) == gb.band_size(n, offset)
  # every in-band slot lies inside its row's packed range; padding is at most 3 + 3 slots per row
  c0 = j0 & ~3
  rows = j0 < n
  assert (off[1:][rows] - off[:-1][rows] - inband[rows] == (j0 - c0)[rows] +
          (-n % 4)).all()
  assert (off[1:][~rows] == off[:-1][~rows]).all()


@pytest.mark.parametrize("n,offset", [(n, o) for n, o in CASES if n <= 130])
def test_packed_positions_keep_the_dense_alignment(n, offset):
  """Column j of row i lands at row_off[i] + j - c0: distinct slots, j's position mod 4."""
  off = gb.packed_row_offsets(n, offset)
  rows, cols = np.triu_indices(n, offset)
  c0 = np.maximum(rows + offset, 0) & ~3
  pos = off[rows] + cols - c0
  assert np.unique(pos).size == pos.size
  assert ((pos - cols) % 4 == 0).all()
  assert (pos >= off[rows]).all() and (pos < off[rows + 1]).all()


@pytest.mark.parametrize("n", [4099, 65536, 98304, 131000, 131072, 150000, 190000])
@pytest.mark.parametrize("offset", [0, 1, 3, 64])
def test_packed_band_fits_in_y_hi(n, offset):
  """The check holds the band and one panel before refine() allocates Y_hi (2 N ld bytes) and two
  panels, so a band within Y_hi + 8 N bytes leaves the route's peak where it was."""
  band_bytes = 4 * int(gb.packed_row_offsets(n, offset)[-1])
  assert band_bytes <= 2 * n * dev.round_up(n, 64) + 8 * n


def single_clusterer(condition, **kw):
  args = dict(min_clusters=1, max_clusters=10,
              refinement_options=scb.configs.icassp2018_refinement_options,
              fallback_options=scb.FallbackOptions(single_cluster_condition=condition),
              custom_dist="cosine")
  args.update(kw)
  return scb.SpectralClusterer(**args)


def routes(c, eng, n, matrix=None):
  return (c._factored_route(eng, n, matrix), c._factored_windows_route(eng, n, matrix),
          c._bounded_route(eng, n, matrix), c._factored_single_cluster_route(eng, n, matrix))


@pytest.mark.parametrize("max_clusters", [10, None])
@pytest.mark.parametrize("condition", list(scb.SingleClusterCondition))
def test_min_clusters_one_takes_the_factored_route_at_131072(condition, max_clusters):
  c = single_clusterer(condition, max_clusters=max_clusters)
  assert routes(c, FakeEngine(), 131072) == (False, False, False, True)
  assert routes(c, FakeEngine(), 98304) == (False, False, False, True)
  c.min_clusters = 2                        # the same call without the check: one of the two routes
  assert c._factored_route(FakeEngine(), 131072) == (max_clusters == 10)
  assert c._factored_windows_route(FakeEngine(), 131072) == (max_clusters is None)


@pytest.mark.parametrize("max_clusters", [10, None])
@pytest.mark.parametrize("condition", list(scb.SingleClusterCondition))
def test_min_clusters_one_keeps_the_stored_route_at_65536(condition, max_clusters):
  c = single_clusterer(condition, max_clusters=max_clusters)
  assert routes(c, FakeEngine(), 65536) == (False, False, False, False)


def test_other_min_clusters_never_take_it():
  for mc in (None, 2, 3):
    c = single_clusterer(scb.SingleClusterCondition.AffinityGmmBic, min_clusters=mc)
    assert not c._factored_single_cluster_route(FakeEngine(), 131072)


@pytest.mark.parametrize("change", [
    dict(affinity_function=_not_affinity), dict(autotune_group=True),
    dict(refinement_options=_seq(*ICASSP, sigma=2.0)),
    dict(refinement_options=_seq(RN.CropDiagonal, RN.RowWiseThreshold, RN.Symmetrize,
                                 RN.Diffuse, RN.RowWiseNormalize)),
    dict(refinement_options=_seq(*ICASSP, ttype=scb.ThresholdType.Percentile)),
    dict(refinement_options=_seq(*ICASSP[:-1], RN.CropDiagonal)),
    dict(refinement_options=_seq(RN.RowWiseThreshold, RN.Symmetrize)),
    dict(refinement_options=_seq(*ICASSP, RN.Diffuse)),
    dict(constraint=True), dict(diffuse_precision=nat.GEMM_SPLIT2), dict(dense_eig_max=1 << 20)])
def test_out_of_scope_options_keep_the_stored_route(change):
  change = dict(change)
  eng = FakeEngine()
  eng.diffuse_precision = change.pop("diffuse_precision", None)
  if "dense_eig_max" in change:
    eng.dense_eig_max = change.pop("dense_eig_max")
  constraint = change.pop("constraint", False)
  group = change.pop("autotune_group", None)
  c = single_clusterer(scb.SingleClusterCondition.AffinityGmmBic, **change)
  c.autotune_group = group
  matrix = None
  if constraint:
    c.constraint_options = scb.ConstraintOptions(
        constraint_name=scb.ConstraintName.ConstraintPropagation, apply_before_refinement=False)
    matrix = [[0]]
  assert routes(c, eng, 131072, matrix) == (False, False, False, False)
