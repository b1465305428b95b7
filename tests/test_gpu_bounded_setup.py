"""GPU: the set-up of the bounded Diffuse and the factored operator around the tile GEMM.

- sc_block_product_f16 (k_symm_dmma_f16) equals sc_block_product on the fp32 upcast bit for bit
  (torch.equal): the same column splits and k order, and fp16 -> fp64 is exact -- at ragged n,
  row slabs (rows != n), every b in 1..16 and padded leading dimensions, on signed data with
  zeros and fp16 subnormals.
- sc_bound_order (the device row order) returns a permutation, the same one on every call, keeps
  the natural order where all profiles are alike, and on the bench's input at N = 65,536 leaves the
  tile count of the bounded Diffuse within half a point of the k-means order it replaced.
"""

import ctypes

import numpy as np
import pytest

from spectralcluster_b200 import device as dev

from test_gpu_factored import embeddings, icassp, stored_front

pytestmark = pytest.mark.gpu

# Tiles the bounded Diffuse computed at N = 65,536 on the bench's speaker turns (6 speakers, seed 0)
# with the scikit-learn-exact k-means order (H100 80GB HBM3): 16,371 of 88,064.  The device order
# may cost at most half a point of the total more.
KMEANS_ORDER_TILES_65536, TOTAL_TILES_65536 = 16371, 88064
TILE_CEILING_65536 = KMEANS_ORDER_TILES_65536 + int(0.005 * TOTAL_TILES_65536)


def signed_f16(engine, rows, ld, seed):
  """rows x ld fp16, signed, about 1/8 zeros and 1/16 fp16 subnormals."""
  t = dev.torch()
  g = t.Generator(device=engine.device).manual_seed(seed)
  x = t.rand((rows, ld), generator=g, device=engine.device, dtype=t.float16).mul_(2).sub_(1)
  u = t.rand((rows, ld), generator=g, device=engine.device, dtype=t.float16)
  x.masked_fill_(u < 0.125, 0.0)
  sub = (u >= 0.125) & (u < 0.1875)
  del u
  x[sub] *= 2.0 ** -16
  return x


def product(engine, name, s, rows, n, t_, b):
  t = dev.torch()
  y = t.full((b, rows), float("nan"), dtype=t.float64, device=engine.device)
  engine.call(name, dev._ptr(s), rows, n, s.stride(0), dev._ptr(t_), t_.stride(0), ctypes.c_int(b),
              dev._ptr(y), y.stride(0), engine.stream)
  return y


@pytest.mark.parametrize("n", [1, 7, 255, 257, 2049, 4097, 40003, 65536])
def test_block_product_f16_equals_fp32_upcast(engine, n):
  t = dev.torch()
  ld = dev.round_up(n, 8) + 8                          # padded: the columns past n are never read
  slab0 = n // 3
  slabs = [(0, n), (slab0, max(1, min(n - slab0, n // 3 + 5)))]
  s16 = signed_f16(engine, n, ld, n)
  s16[:, n:] = float("inf")                            # a stray read past n would poison the result
  s32 = s16.float()
  g = t.Generator(device=engine.device).manual_seed(n + 1)
  ldt = dev.round_up(n, 2)
  t_ = t.rand((16, ldt), generator=g, dtype=t.float64, device=engine.device) - 0.5
  for r0, rows in slabs:
    for b in range(1, 17):
      want = product(engine, "sc_block_product", s32[r0:], rows, n, t_, b)
      got = product(engine, "sc_block_product_f16", s16[r0:], rows, n, t_, b)
      assert t.equal(got, want), (n, r0, rows, b)
      assert bool(t.isfinite(got).all())


def bound_order(engine, norms):
  perm = engine.bound_order(norms)
  assert perm.dtype == dev.torch().int32 and perm.numel() == norms.shape[0]
  return perm


def is_permutation(perm):
  p = perm.long().cpu().numpy()
  return np.array_equal(np.sort(p), np.arange(p.size))


@pytest.mark.parametrize("n", [40003, 65536])
def test_bound_order_is_a_repeatable_permutation(engine, n):
  t = dev.torch()
  _, _, _, hi = stored_front(engine, embeddings(engine, n, speakers=6, seed=0), icassp())
  norms, _, _ = engine.row_group_bounds(hi, n)
  p1 = bound_order(engine, norms)
  p2 = bound_order(engine, norms)
  assert is_permutation(p1)
  assert t.equal(p1, p2)


@pytest.mark.parametrize("kind", ["identical", "zeros", "block", "one-row"])
def test_bound_order_edge_profiles(engine, kind):
  t = dev.torch()
  if kind == "identical":
    x = t.full((5000, 20), 0.5, device=engine.device)
  elif kind == "zeros":
    x = t.zeros((3001, 12), device=engine.device)
  elif kind == "one-row":
    x = t.rand((1, 3), device=engine.device)
  else:                                                # block-diagonal: 5 disjoint supports
    x = t.block_diag(*[t.ones(700, 8, device=engine.device)] * 5)
    x = x[t.randperm(x.shape[0], generator=t.Generator().manual_seed(1)).to(engine.device)]
  x = x.float().contiguous()
  p = bound_order(engine, x)
  assert is_permutation(p)
  assert t.equal(p, bound_order(engine, x))
  if kind in ("identical", "zeros", "one-row"):        # all alike: the natural order
    assert t.equal(p.long(), t.arange(x.shape[0], device=engine.device))
  else:                                                # rows of one support end up contiguous
    support = x[p.long()].argmax(dim=1).cpu().numpy()
    assert int((np.diff(support) != 0).sum()) == 4


def test_bound_order_tile_count_on_bench_input(engine):
  n = 65536
  _, _, _, hi = stored_front(engine, embeddings(engine, n, speakers=6, seed=0), icassp())
  norms, diag, _ = engine.row_group_bounds(hi, n)
  mx_ref, _ = engine.diffuse_stats(n, hi)
  mx, counts = engine.rowmax_tiles(hi, n, norms, diag, engine.bound_order(norms))
  computed, total = counts.tolist()
  assert total == TOTAL_TILES_65536 == dev.bounded_tile_count(n)
  assert computed <= TILE_CEILING_65536, computed
  assert dev.torch().equal(mx.view(dev.torch().int32), mx_ref.view(dev.torch().int32))
