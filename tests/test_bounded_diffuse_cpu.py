"""CPU: the bounded Diffuse's tile rule (NumPy restatement, tests/bounded_diffuse_numpy.py) on
ragged N and non-negative fp16 inputs -- no skipped tile holds an element that reaches its row's
maximum, the rasterised enumeration is the launch's -- and which calls take the route."""

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev

import bounded_diffuse_numpy as bd
from test_factored_route_cpu import FakeEngine, icassp_clusterer, _seq, ICASSP


def speaker_y(n, speakers, seed):
  """A symmetric non-negative fp16 Y of speaker turns that is large only on same-speaker pairs, as
  RowMax thresholding leaves it."""
  rng = np.random.default_rng(seed)
  turns = rng.integers(40, 300, n)                # speaker turns: runs of one speaker
  lab = np.repeat(rng.integers(0, speakers, n), turns)[:n]
  y = rng.uniform(0.0, 0.01, (n, n))
  y[lab[:, None] == lab[None, :]] += rng.uniform(0.5, 1.0, (n, n))[lab[:, None] == lab[None, :]]
  y = np.maximum(y, y.T)
  return y.astype(np.float16), lab


def skipped_hold_no_maximum(y16, perm, kept):
  y = y16.astype(np.float64)
  s = y @ y.T
  n = len(perm)
  sp = s[np.ix_(perm, perm)]
  covered = np.zeros((n, n), dtype=bool)
  for m, c in kept:
    covered[bd.BM * m:bd.BM * m + bd.BM, bd.BN * c:bd.BN * c + bd.BN] = True
  covered |= covered.T
  row_max = sp.max(axis=1)
  # every element that reaches its row's maximum lies in a kept tile (or its mirror)
  hits = sp >= row_max[:, None] * (1 - 4 * bd.EPS)
  return bool(covered[hits].all())


@pytest.mark.parametrize("n", [1000, 2500, 4097])
def test_skipped_tiles_hold_no_row_maximum(n):
  y16, lab = speaker_y(n, 5, seed=n)
  norms, diag, _ = bd.row_bounds(y16)
  for perm in (np.argsort(lab, kind="stable"), np.arange(n)):
    kept = bd.kept_tiles(norms, diag, perm)
    assert skipped_hold_no_maximum(y16, perm, kept)
  # grouped by speaker, most off-diagonal tiles go (at 1,000 there are only 32 tiles)
  assert n < 2500 or len(bd.kept_tiles(norms, diag, np.argsort(lab, kind="stable"))) < 0.6 * len(
      bd.rasterised_tiles(n))


def test_identical_rows_skip_nothing():
  n = 1300
  y16 = np.full((n, n), 0.25, dtype=np.float16)
  norms, diag, _ = bd.row_bounds(y16)
  assert len(bd.kept_tiles(norms, diag, np.arange(n))) == len(bd.rasterised_tiles(n))


def test_block_diagonal_skips_every_off_diagonal_tile():
  n, b = 1536, 384                         # blocks aligned with both tile sizes
  rng = np.random.default_rng(1)
  y = np.zeros((n, n))
  for s in range(0, n, b):
    blk = rng.uniform(0.1, 1.0, (b, b))
    y[s:s + b, s:s + b] = np.maximum(blk, blk.T)
  y16 = y.astype(np.float16)
  norms, diag, _ = bd.row_bounds(y16)
  kept = bd.kept_tiles(norms, diag, np.arange(n))
  for m, c in kept:
    rows = range(bd.BM * m, bd.BM * m + bd.BM)
    cols = range(bd.BN * c, min(n, bd.BN * c + bd.BN))
    same_block = {r // b for r in rows} & {c_ // b for c_ in cols}
    assert same_block or bd.BN * c < bd.BM * m + bd.BM


@pytest.mark.parametrize("n", [1000, 4097, 16384, 40000, 65536])
def test_rasterised_enumeration_is_the_launch(n):
  tiles = bd.rasterised_tiles(n)
  assert len(tiles) == len(set(tiles)) == dev.bounded_tile_count(n)


def test_scope_bounded_and_factored_split_the_lanczos_calls():
  eng = FakeEngine()
  c = icassp_clusterer()
  for n in (dev.BOUNDED_FROM, 40000, 65536):
    assert c._bounded_route(eng, n) and not c._factored_route(eng, n)
  assert c._factored_route(eng, 131072) and not c._bounded_route(eng, 131072)
  # below BOUNDED_FROM the storing Diffuse is faster; below N = 16,384 it takes two MMAs
  assert not c._bounded_route(eng, dev.BOUNDED_FROM - 1)
  assert not c._bounded_route(eng, 16384)


@pytest.mark.parametrize("change", [
    dict(min_clusters=1), dict(max_clusters=None), dict(max_clusters=32),
    dict(refinement_options=_seq(*ICASSP, sigma=2.0)),
    dict(refinement_options=_seq(*ICASSP, ttype=scb.ThresholdType.Percentile)),
    dict(refinement_options=_seq(*ICASSP, scb.RefinementName.Diffuse)),
    dict(constraint=True), dict(diffuse_precision=nat.GEMM_SPLIT2)])
def test_out_of_scope_calls_keep_the_storing_diffuse(change):
  change = dict(change)
  eng = FakeEngine()
  eng.diffuse_precision = change.pop("diffuse_precision", None)
  constraint = change.pop("constraint", False)
  kw = dict(min_clusters=2, max_clusters=10,
            refinement_options=scb.configs.icassp2018_refinement_options)
  kw.update(change)
  c = scb.SpectralClusterer(custom_dist="cosine", **kw)
  matrix = None
  if constraint:
    c.constraint_options = scb.ConstraintOptions(
        constraint_name=scb.ConstraintName.ConstraintPropagation, apply_before_refinement=False)
    matrix = [[0]]
  assert not c._bounded_route(eng, 65536, matrix)
