"""CPU: the hub-first bounded Diffuse restated in NumPy (tests/hub_bounded_numpy.py) -- the order is
a permutation that keeps every cluster contiguous and leads it with its hub, and no tile that phase
1 and phase 2 both leave out holds an element that reaches its row's maximum, on speaker data and on
block-diagonal, identical, zero and ragged inputs."""

import numpy as np
import pytest

import bounded_diffuse_numpy as bd
import hub_bounded_numpy as hb
from test_bounded_diffuse_cpu import speaker_y


def run(y16, labels, k):
  """(perm, starts, phase-1 tiles, phase-2 tiles, the permuted exact product)."""
  n = y16.shape[0]
  norms, diag, _ = bd.row_bounds(y16)
  perm, starts = hb.hub_order(diag, labels, k)
  y = y16.astype(np.float64)[perm]
  sp = y @ y.T
  p1 = hb.hub_tiles(starts, n)
  p2 = hb.phase2_tiles(norms[perm], hb.fold(sp, p1, n), p1)
  return perm, starts, p1, p2, sp


def maxima_covered(sp, tiles):
  n = sp.shape[0]
  covered = np.zeros((n, n), dtype=bool)
  for m, c in tiles:
    covered[bd.BM * m:bd.BM * m + bd.BM, bd.BN * c:bd.BN * c + bd.BN] = True
  covered |= covered.T
  # every element within the product's rounding of its row's maximum lies in a computed tile
  hits = sp >= sp.max(axis=1)[:, None] * (1 - 4 * bd.EPS)
  return bool(covered[hits].all())


def check_order(perm, starts, labels, diag):
  n = len(perm)
  assert np.array_equal(np.sort(perm), np.arange(n))
  key = hb.diag_key(diag)
  for c, (a, b) in enumerate(zip(starts[:-1], starts[1:])):
    assert (labels[perm[a:b]] == c).all()                   # contiguous clusters, in label order
    if b > a:
      assert np.all(np.diff(key[perm[a:b]].astype(np.float64)) <= 0)   # hub first, then descending
  assert starts[-1] == n


@pytest.mark.parametrize("n", [1000, 2500, 4097])
def test_speaker_data(n):
  y16, lab = speaker_y(n, 5, seed=n)
  perm, starts, p1, p2, sp = run(y16, lab, 5)
  check_order(perm, starts, lab, bd.row_bounds(y16)[1])
  assert not set(p1) & set(p2)
  assert maxima_covered(sp, p1 + p2)
  assert n < 2500 or len(p1) + len(p2) < 0.6 * len(bd.rasterised_tiles(n))


def test_speaker_data_in_fewer_clusters_than_speakers():
  # a cluster holding two speakers: its hub serves only one of them, the rule still holds
  n = 3000
  y16, lab = speaker_y(n, 6, seed=7)
  merged = np.minimum(lab, 3)
  _, _, p1, p2, sp = run(y16, merged, 4)
  assert maxima_covered(sp, p1 + p2)


@pytest.mark.parametrize("kind,n", [("block", 2000), ("identical", 1300), ("zeros", 777),
                                    ("ragged", 1501)])
def test_edge_inputs(kind, n):
  rng = np.random.default_rng(n)
  if kind == "identical":
    y = np.full((n, n), 0.25)
  elif kind == "zeros":
    y = np.zeros((n, n))
  else:
    y = np.zeros((n, n))
    edges = np.linspace(0, n, 7).astype(int)
    for a, b in zip(edges[:-1], edges[1:]):
      blk = rng.uniform(0.1, 1.0, (b - a, b - a))
      y[a:b, a:b] = np.maximum(blk, blk.T)
    if kind == "ragged":
      y[n - 50:, :] = 0
      y[:, n - 50:] = 0
  y16 = y.astype(np.float16)
  labels = np.zeros(n, dtype=np.int64)
  if kind in ("block", "ragged"):
    labels = np.searchsorted(np.linspace(0, n, 7).astype(int)[1:], np.arange(n), side="right")
  k = int(labels.max()) + 1
  perm, starts, p1, p2, sp = run(y16, labels, k)
  check_order(perm, starts, labels, bd.row_bounds(y16)[1])
  assert maxima_covered(sp, p1 + p2)
  if kind in ("identical", "zeros"):
    assert len(p1) + len(p2) == len(bd.rasterised_tiles(n))


def test_hub_tiles_cover_every_row_with_its_hub():
  n = 5000
  starts = np.array([0, 130, 1900, 1901, 1901, 5000])       # with a one-row and an empty cluster
  tiles = hb.hub_tiles(starts, n)
  covered = np.zeros((n, n), dtype=bool)
  for m, c in tiles:
    covered[bd.BM * m:bd.BM * m + bd.BM, bd.BN * c:bd.BN * c + bd.BN] = True
  for a, b in zip(starts[:-1], starts[1:]):
    assert covered[a, a:b].all()
  assert len(tiles) == len(set(tiles)) <= -(-n // bd.BN) + len(starts)
