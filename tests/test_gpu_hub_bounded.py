"""GPU: the hub-first bounded Diffuse (sc_bound_order_hubs + sc_diffuse_hub_tiles +
sc_diffuse_tile_list_rows) -- row maxima bit for bit those of sc_diffuse on speaker data and on edge
inputs, both device tile lists equal to the NumPy restatement (tests/hub_bounded_numpy.py) over the
same norms and phase-1 maxima, a repeatable order and count, and the tile share on the bench input."""

import numpy as np
import pytest

from spectralcluster_b200 import device as dev

import bounded_diffuse_numpy as bd
import hub_bounded_numpy as hb
from test_gpu_bounded_diffuse import bits, edge_y
from test_gpu_factored import embeddings, icassp, stored_front

pytestmark = pytest.mark.gpu
# the hub rule computes under 13 % of the tiles on the bench input at N = 65,536 (the tile-wide
# rule of sc_diffuse_tile_list computes 19 %)
SHARE_CEILING_65536 = 0.13


def speaker_hi(engine, n):
  return stored_front(engine, embeddings(engine, n, speakers=6, seed=0), icassp())[3]


def device_lists(engine, n, hi):
  """(perm, starts, phase-1 list, phase-1 maxima, phase-2 list, total, final maxima) from the
  entries themselves."""
  t = dev.torch()
  norms, diag, _ = engine.row_group_bounds(hi, n)
  perm, starts = engine.bound_order_hubs(norms, diag)
  mx, counts, l1 = engine.hub_rowmax_tiles(hi, n, norms, perm, starts, want_phase1=True)
  size = -(-n // bd.BM) * -(-n // bd.BN)
  k = int(starts.shape[0]) - 1
  tiles = t.empty(size, dtype=t.int32, device=engine.device)
  c = t.empty(3, dtype=t.int32, device=engine.device)
  engine.call("sc_diffuse_hub_tiles", dev._ptr(starts), k, n, dev._ptr(tiles), dev._ptr(c),
              engine.stream)
  n1 = int(c[0].item())
  list1 = [(v >> 16, v & 0xFFFF) for v in tiles[:n1].cpu().numpy().tolist()]
  engine.call("sc_diffuse_tile_list_rows", dev._ptr(norms), int(norms.shape[1]), dev._ptr(perm), n,
              dev._ptr(l1), dev._ptr(starts), k, dev._ptr(tiles), dev._ptr(c[1:]),
              dev._ptr(c[2:]), engine.stream)
  n2, total = int(c[1].item()), int(c[2].item())
  list2 = [(v >> 16, v & 0xFFFF) for v in tiles[:n2].cpu().numpy().tolist()]
  assert counts.tolist() == [n1, n2, total]
  return dict(norms=norms, perm=perm, starts=starts, list1=list1, l1=l1, list2=list2, total=total,
              mx=mx)


def check(engine, n, hi, expect_all=False):
  t = dev.torch()
  mx_ref, _ = engine.diffuse_stats(n, hi)
  r = device_lists(engine, n, hi)
  assert t.equal(bits(r["mx"]), bits(mx_ref))
  assert r["total"] == dev.bounded_tile_count(n)
  perm = r["perm"].long().cpu().numpy()
  starts = r["starts"].long().cpu().numpy()
  assert np.array_equal(np.sort(perm), np.arange(n))
  assert r["list1"] == hb.hub_tiles(starts, n)
  pn = r["norms"].double().cpu().numpy()[perm]
  l1 = r["l1"].double().cpu().numpy()[perm]
  assert r["list2"] == hb.phase2_tiles(pn, l1, r["list1"])
  _, _, counts = engine.bounded_diffuse(n, hi)
  computed = len(r["list1"]) + len(r["list2"])
  assert counts.tolist() == [computed, r["total"]]
  if expect_all:
    assert computed == r["total"]
  return computed, r["total"]


@pytest.mark.parametrize("n", [32768, 65536])
def test_rowmax_bitwise_on_speaker_data(engine, n):
  computed, total = check(engine, n, speaker_hi(engine, n))
  assert computed < 0.2 * total


@pytest.mark.parametrize("kind,n", [("identical", 20000), ("block", 12345), ("zeros", 5000),
                                    ("ragged", 7001)])
def test_rowmax_bitwise_on_edge_inputs(engine, kind, n):
  t = dev.torch()
  if kind == "zeros":
    hi = t.zeros((n, dev.round_up(n, 64)), dtype=t.float16, device=engine.device)
  elif kind == "ragged":                 # block-diagonal with a zero row block at the ragged end
    hi = edge_y(engine, n, "block")
    hi[n - 100:, :] = 0
    hi[:, n - 100:n] = 0
  else:
    hi = edge_y(engine, n, kind)
  check(engine, n, hi, expect_all=kind in ("identical", "zeros"))


def test_order_and_counts_repeat(engine):
  t = dev.torch()
  n = 40003
  hi = speaker_hi(engine, n)
  norms, diag, _ = engine.row_group_bounds(hi, n)
  p1, s1 = engine.bound_order_hubs(norms, diag)
  p2, s2 = engine.bound_order_hubs(norms, diag)
  assert t.equal(p1, p2) and t.equal(s1, s2)
  # the clusters are those of bound_order, each led by its largest diagonal
  old = engine.bound_order(norms).long().cpu().numpy()
  perm, starts = p1.long().cpu().numpy(), s1.long().cpu().numpy()
  key = hb.diag_key(diag.cpu().numpy())
  for a, b in zip(starts[:-1], starts[1:]):
    assert set(perm[a:b]) == set(old[a:b])
    if b > a:
      assert key[perm[a]] == key[perm[a:b]].max()
  _, c1 = engine.hub_rowmax_tiles(hi, n, norms, p1, s1)
  _, c2 = engine.hub_rowmax_tiles(hi, n, norms, p1, s1)
  assert c1.tolist() == c2.tolist()


def test_tile_share_on_bench_input(engine):
  n = 65536
  hi = speaker_hi(engine, n)
  _, _, counts = engine.bounded_diffuse(n, hi)
  computed, total = counts.tolist()
  assert total == dev.bounded_tile_count(n)
  assert computed < SHARE_CEILING_65536 * total, computed / total
