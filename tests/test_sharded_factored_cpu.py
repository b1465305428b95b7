"""CPU: the factored route of predict_sharded() -- which calls take it (a fake engine stands in for
an 80 GB H100), that the option checks still refuse what they refused, and, under gloo with two
ranks and a NumPy backend, the factored orchestration: panel front end, S's row statistics
streamed through the staging buffers, and the eigensolve's two half-products (the first summed
over the ranks, the second all-gathered)."""

import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import spectralcluster_b200 as scb  # noqa: E402
from spectralcluster_b200 import _native as nat  # noqa: E402
from spectralcluster_b200 import device as dev  # noqa: E402
from spectralcluster_b200 import sharded  # noqa: E402

H100_80GB = 85_520_809_984          # torch.cuda.get_device_properties(0).total_memory


class FakeEngine:
  """What factored_sharded_route reads from an Engine, for a device with `total` bytes."""

  def __init__(self, total=H100_80GB):
    self.factored_above_bytes = total - dev.FACTORED_ROUTE_RESERVE
    self.diffuse_precision = None

  diffuse_precision_for = dev.Engine.diffuse_precision_for


def clusterer(**kw):
  kw.setdefault("min_clusters", 2)
  kw.setdefault("max_clusters", 10)
  return scb.SpectralClusterer(refinement_options=scb.configs.icassp2018_refinement_options,
                               custom_dist="cosine", **kw)


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_65536_keeps_the_stored_route_at_every_world(world):
  assert not sharded.factored_sharded_route(FakeEngine(), 65536, world)


def test_131072_stored_at_8_factored_at_2():
  eng = FakeEngine()
  assert not sharded.factored_sharded_route(eng, 131072, 8)
  assert sharded.factored_sharded_route(eng, 131072, 2)
  assert sharded.factored_sharded_route(eng, 131072, 1)


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_262144_factored_at_every_world(world):
  assert sharded.factored_sharded_route(FakeEngine(), 262144, world)


def test_threshold_follows_the_byte_formula():
  n, world = 100000, 4
  block = dev.round_up(-(-n // world), 128)
  ld = dev.round_up(n, 64)
  peak = 4 * world * block * ld + 4 * (block + 2 * dev.BLUR_HALO + 128) * ld
  assert sharded.sharded_stored_peak_bytes(n, world) == peak
  eng = FakeEngine()
  eng.factored_above_bytes = peak
  assert not sharded.factored_sharded_route(eng, n, world)
  eng.factored_above_bytes = peak - 1
  assert sharded.factored_sharded_route(eng, n, world)


def test_only_a_single_mma_diffuse_is_factored():
  eng = FakeEngine()
  eng.diffuse_precision = nat.GEMM_SPLIT3
  assert not sharded.factored_sharded_route(eng, 262144, 8)


def test_factored_buffers_fit_where_the_stored_ones_do_not():
  above = FakeEngine().factored_above_bytes
  for n, world in ((131072, 2), (262144, 8)):
    assert sharded.sharded_stored_peak_bytes(n, world) > above
    assert sharded.sharded_factored_peak_bytes(n, world) < above / 2


def test_staging_is_a_fixed_size_not_a_peer_block():
  for n in (65536, 131072, 262144):
    rows = sharded.staging_rows_for(n)
    assert rows % 128 == 0
    assert 2 * rows * dev.round_up(n, 64) <= sharded.STAGING_BYTES
    assert rows < dev.round_up(n // 8, 128)


@pytest.mark.parametrize("kw, message", [
    (dict(autotune=scb.AutoTune(p_percentile_min=0.6, p_percentile_max=0.95,
                                init_search_step=0.05, search_level=1)),
     "predict_sharded: AutoTune is not sharded"),
    (dict(min_clusters=1), "predict_sharded: single-cluster detection is not sharded"),
    (dict(constraint_options=scb.ConstraintOptions(
        constraint_name=scb.ConstraintName.ConstraintPropagation, apply_before_refinement=True)),
     "predict_sharded: constraints are not sharded"),
    (dict(affinity_function=lambda x: x @ x.T),
     "predict_sharded: only the built-in cosine affinity is sharded"),
    (dict(max_spectral_size=1000),
     "predict_sharded: max_spectral_size pre-clustering is not sharded (sharding is the exact "
     "alternative to it)"),
])
def test_refusals_unchanged_where_the_factored_route_would_run(kw, message):
  with pytest.raises(NotImplementedError) as err:
    sharded.check_sharded_options(clusterer(**kw), 262144)
  assert str(err.value) == message


# ---- two gloo ranks: the factored orchestration with a NumPy backend

def free_port():
  s = socket.socket()
  s.bind(("127.0.0.1", 0))
  port = s.getsockname()[1]
  s.close()
  return port


def _numpy_backend(staging_rows):
  from sharded_numpy_backend import NumpyBackend

  class FactoredNumpyBackend(NumpyBackend):
    """NumpyBackend plus the factored route's block interface (float64 torch CPU buffers)."""

    def affinity_block(self, xn, n, row_begin, row_count, want_crop, capacity=None):
      return super().affinity_block(xn, n, row_begin, row_count, want_crop)

    def thrsym_rows(self, a_ext, n, rows, crop, sigma, m_full, opt, sym_max, hi, lo, first_row):
      full = (torch.zeros((rows.row_end, n), dtype=torch.float64),)
      self.thrsym_block(a_ext, n, rows, crop, sigma, m_full, opt, sym_max, full)
      hi[rows.row_begin - first_row:rows.row_end - first_row] = full[0][rows.row_begin:]

    def new_rows(self, rows, n):
      return torch.zeros((rows, n), dtype=torch.float64)

    def new_stats(self, rows):
      return (torch.zeros(rows, dtype=torch.float64), torch.zeros(rows, dtype=torch.float64))

    def stats_block(self, a, a_rows, b, b_rows, n, mx, sm):
      s = a[:a_rows].numpy() @ b[:b_rows].numpy().T
      mx.copy_(torch.maximum(mx, torch.from_numpy(s.max(axis=1))))
      sm += torch.from_numpy(s.sum(axis=1))

    def staging(self, n):
      return [torch.zeros((staging_rows, n), dtype=torch.float64) for _ in range(2)], staging_rows

  return FactoredNumpyBackend()


def _half_products(y_rows, plan, t_full, slabs, group=None):
  """One pass of the sharded factored operator as sc_eigh_extremal_factored_sharded runs it: this
  rank's share of Z = Y^T T summed over the ranks in the slab buffer (gather(-b)); then Y[R,:] Z
  into this rank's slab, all-gathered (gather(b)).  Returns S T = Y Y^T T."""
  b = t_full.shape[1]
  per = b * plan.block
  n = plan.n
  rows = slice(plan.row_begin, plan.row_end)
  z = slabs[:b * n].view(b, n)
  z.copy_((y_rows.T @ t_full[rows]).T)
  dist.all_reduce(slabs[:b * n], group=group)
  local = y_rows @ z.T.clone()
  mine = slabs[plan.rank * per:(plan.rank + 1) * per].view(b, plan.block)
  mine.zero_()
  mine[:, :plan.rows] = local.T
  dist.all_gather_into_tensor(slabs[:plan.world * per], mine.reshape(-1).clone(), group=group)
  full = slabs[:plan.world * per].view(plan.world, b, plan.block).permute(0, 2, 1)
  return full.reshape(plan.world * plan.block, b)[:n]


def _orchestration_worker(rank, world, port, n, laplacian, out):
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  dist.init_process_group("gloo", rank=rank, world_size=world)
  from oracle import spectral_oracle as orc
  from spectralcluster_b200 import laplacian as lap
  RN = scb.RefinementName
  opt = scb.RefinementOptions(gaussian_blur_sigma=1, p_percentile=0.9, refinement_sequence=[
      RN.CropDiagonal, RN.GaussianBlur, RN.RowWiseThreshold, RN.Symmetrize, RN.Diffuse,
      RN.RowWiseNormalize])
  x = orc.synthetic_dvectors(n, 16, 3, seed=5)
  refiner = sharded.FactoredShardedRefiner(_numpy_backend(staging_rows=48), opt, dist=dist,
                                           panel_rows=96)
  res = refiner.run(x, world, rank)
  plan = res["plan"]
  y_rows = res["y_rows"]
  # rank 0's rows take several panels and several staging chunks
  ok = refiner.last_transport == "gloo" and (rank > 0 or len(refiner.panels(plan)) > 1)
  # Y rows and S's row statistics against the oracle's unsharded refinement
  y_want = orc.refine(orc.affinity(x), orc.options(
      sequence=("crop", "blur", "threshold", "symmetrize"), sigma=1, p=0.9))
  s_want = y_want @ y_want.T
  rows = slice(plan.row_begin, plan.row_end)
  ok &= np.allclose(y_rows.numpy(), y_want[rows], rtol=1e-12, atol=1e-12)
  ok &= np.allclose(res["rowmax"].numpy(), s_want[rows].max(axis=1), rtol=1e-11)
  ok &= np.allclose(res["rowsum"].numpy(), s_want[rows].sum(axis=1), rtol=1e-11)

  def gathered(local):
    full = torch.zeros(world * plan.block, dtype=torch.float64)
    full[rows] = local
    dist.all_gather_into_tensor(full, full[rank * plan.block:(rank + 1) * plan.block].clone())
    return full[:n]

  rowmax, rowsum = gathered(res["rowmax"]), gathered(res["rowsum"])
  delta, left, right, sign, _ = lap.terms_from_row_sums(rowsum, 1.0 / rowmax, laplacian)
  c = torch.sqrt((left if left is not None else 1.0) * (right if right is not None else 1.0)
                 * torch.ones(n, dtype=torch.float64))
  # the operator diag(delta) + sign diag(c) S diag(c), assembled column block by column block
  # through the sharded half-products only
  b = 8
  slabs = torch.zeros(world * b * plan.block, dtype=torch.float64)
  op = np.zeros((n, n))
  for j0 in range(0, n, b):
    eye = torch.zeros((n, b), dtype=torch.float64)
    cols = list(range(j0, min(n, j0 + b)))
    eye[cols, range(len(cols))] = 1.0
    prod = c[:, None] * _half_products(y_rows, plan, c[:, None] * eye, slabs)
    op[:, j0:j0 + len(cols)] = sign * prod[:, :len(cols)].numpy()
  if delta is not None:
    op += np.diag(delta.numpy())
  w = np.linalg.eigh(0.5 * (op + op.T))[0]
  # the same operator from the oracle's S
  r = 1.0 / s_want.max(axis=1)
  d, l_, r_, sg, _ = lap.terms_from_row_sums(torch.from_numpy(s_want.sum(axis=1)),
                                             torch.from_numpy(r), laplacian)
  cw = np.sqrt((l_.numpy() if l_ is not None else 1.0) * (r_.numpy() if r_ is not None else 1.0)
               * np.ones(n))
  ref = sg * cw[:, None] * s_want * cw[None, :] + (np.diag(d.numpy()) if d is not None else 0.0)
  w_ref = np.linalg.eigh(0.5 * (ref + ref.T))[0]
  ok &= np.allclose(w, w_ref, rtol=1e-9, atol=1e-9 * np.abs(w_ref).max())
  # every rank holds bitwise the same w
  every = [torch.zeros(n, dtype=torch.float64) for _ in range(world)]
  dist.all_gather(every, torch.from_numpy(w))
  ok &= all(torch.equal(every[0], e) for e in every)
  flags = torch.tensor([1 if ok else 0])
  dist.all_reduce(flags, op=dist.ReduceOp.MIN)
  if rank == 0:
    out.put(int(flags[0]))
  dist.destroy_process_group()


@pytest.mark.parametrize("n,laplacian", [(300, scb.LaplacianType.GraphCut), (257, None)])
def test_factored_orchestration_two_ranks_gloo(n, laplacian):
  ctx = mp.get_context("spawn")
  out = ctx.Queue()
  mp.spawn(_orchestration_worker, args=(2, free_port(), n, laplacian, out), nprocs=2, join=True)
  assert out.get(timeout=10) == 1
