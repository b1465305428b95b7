"""GPU: the factored route of predict_sharded() (owned Y_hi rows only, S never stored) against the
stored sharded route, with the route forced by factored_above_bytes = 0.

At world = 1 the owned Y_hi rows are bit for bit the hi plane of the stored route, and the row
maxima of S are too: the own block is the same symmetric launch of the same GEMM, so every element
comes from the same accumulator.  The row sums are folded from the GEMM epilogue's fp32 partial sums
over a 192-column tile row (the stored route sums the stored fp32 elements in fp64), so they agree
within 2 * 191 * 2^-24 of the row sum.

Y_hi is not bitwise symmetric on either sharded route (the row-block blur sums B[i, j] and B[j, i]
in different orders), so the eigenpair residuals are taken against Y_hi Y_hi^T itself."""

import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

D, SPEAKERS = 256, 6


@pytest.fixture(autouse=True, scope="module")
def release_sharded_buffers():
  """Give the engine's persistent sharded buffers back when the module ends."""
  yield
  free_engine_buffers()


def free_engine_buffers():
  import torch
  from spectralcluster_b200 import device as dev
  eng = dev.Engine.get()
  if getattr(eng, "_sharded_backend", None) is not None:
    del eng._sharded_backend
  torch.cuda.synchronize()
  torch.cuda.empty_cache()


def icassp_options(scb):
  return scb.RefinementOptions(
      gaussian_blur_sigma=1, p_percentile=0.95, thresholding_soft_multiplier=0.01,
      refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))


def make(scb, case):
  GC = scb.LaplacianType.GraphCut
  kw = dict(graphcut_10=dict(laplacian_type=GC, max_clusters=10),
            nolaplacian_none=dict(),
            graphcut_none=dict(laplacian_type=GC),
            graphcut_ndiff_10=dict(laplacian_type=GC, max_clusters=10,
                                   eigengap_type=scb.EigenGapType.NormalizedDiff))[case]
  return scb.SpectralClusterer(min_clusters=2, refinement_options=icassp_options(scb), **kw)


def data(n, seed=7):
  from oracle import spectral_oracle as orc
  return orc.synthetic_dvectors(n, D, SPEAKERS, seed=seed, return_labels=True)


class forced_factored:
  """predict_sharded() on the factored route whatever N: factored_above_bytes = 0."""

  def __enter__(self):
    from spectralcluster_b200 import device as dev
    self.eng = dev.Engine.get()
    self.saved = self.eng.factored_above_bytes
    self.eng.factored_above_bytes = 0
    return self

  def __exit__(self, *exc):
    self.eng.factored_above_bytes = self.saved


@pytest.mark.parametrize("n", [40000, 65536])
def test_y_rows_and_row_statistics_match_the_stored_route(engine, n):
  import torch
  import spectralcluster_b200 as scb
  from spectralcluster_b200 import sharded
  free_engine_buffers()
  x, _ = data(n)
  x_dev = torch.from_numpy(x).to(engine.device)
  opt = icassp_options(scb)
  be = sharded.DeviceBackend(engine)
  res = sharded.ShardedRefiner(be, opt).run(x_dev, 1, 0)
  y_stored = res["y_planes"][0][:n, :n].clone()
  mx_stored, sm_stored = res["rowmax"].clone(), res["rowsum"].clone()
  del res
  be._buffers.clear()
  torch.cuda.empty_cache()
  # a panel height that gives several panels at these N
  refiner = sharded.FactoredShardedRefiner(be, opt, panel_rows=8192)
  got = refiner.run(x_dev, 1, 0)
  assert len(refiner.panels(got["plan"])) > 1
  y = got["y_rows"]
  assert y.dtype == torch.float16 and y.shape[0] == n
  assert torch.equal(y[:, :n], y_stored)
  # The row-block blur sums B[i, j] and B[j, i] in different orders, so Y is symmetric only to
  # rounding: the factored operator applies Y (Y^T T) and never assumes Y = Y^T.
  asym = 0
  for i in range(0, n, 8192):
    asym += int((y[i:i + 8192, :n] != y[:n, i:i + 8192].T).sum())
  print("N=%d: %d of %d elements of Y_hi differ from their mirror" % (n, asym, n * n))
  assert asym < n * n // 1000
  del y_stored
  assert torch.equal(got["rowmax"].double(), mx_stored)
  bound = 2 * 191 * 2.0 ** -24 * sm_stored
  assert bool(((got["rowsum"] - sm_stored).abs() <= bound).all())
  del got, be
  torch.cuda.empty_cache()


def factored_residual(y_rows, terms, v, w):
  """max_j |M v_j - w_j v_j|_inf in float64, M = diag(delta) + sign diag(left) Y Y^T diag(right)
  with Y the fp16 hi plane (world = 1: all rows), applied as Y (Y^T x) in row chunks."""
  import torch
  delta, left, right, sign, _ = terms
  v = v.double()
  n, cols = v.shape
  x = v if right is None else v * right[:, None]
  z = torch.zeros_like(v)
  for i in range(0, n, 4096):
    z += y_rows[i:i + 4096, :n].double().T @ x[i:i + 4096]
  sx = torch.empty_like(v)
  for i in range(0, n, 4096):
    sx[i:i + 4096] = y_rows[i:i + 4096, :n].double() @ z
  mv = sign * (sx if left is None else sx * left[:, None])
  if delta is not None:
    mv += delta[:, None] * v
  lam = torch.as_tensor(np.asarray(w[:cols]), dtype=torch.float64, device=v.device)
  return float((mv - v * lam[None, :]).abs().max())


@pytest.mark.parametrize("n", [40000, 65536])
@pytest.mark.parametrize("case, windows", [
    ("graphcut_10", False), ("nolaplacian_none", True), ("graphcut_none", True),
    ("graphcut_ndiff_10", False)])
def test_pipeline_matches_the_stored_route(engine, monkeypatch, n, case, windows):
  import torch
  import spectralcluster_b200 as scb
  from spectralcluster_b200 import laplacian, sharded
  x, truth = data(n)
  stored = make(scb, case)
  want = sharded.predict_sharded(stored, x)
  free_engine_buffers()
  c = make(scb, case)
  grabbed = {}
  run, terms, cluster = sharded.FactoredShardedRefiner.run, laplacian.terms_from_row_sums, \
      c._cluster_embeddings

  def grab_run(refiner, *a, **kw):
    grabbed["res"] = run(refiner, *a, **kw)
    return grabbed["res"]

  def grab_terms(*a, **kw):
    grabbed["terms"] = terms(*a, **kw)
    return grabbed["terms"]

  def grab_vectors(eng, v, k):
    grabbed["v"] = v.clone()
    return cluster(eng, v, k)

  monkeypatch.setattr(sharded.FactoredShardedRefiner, "run", grab_run)
  monkeypatch.setattr(laplacian, "terms_from_row_sums", grab_terms)
  monkeypatch.setattr(c, "_cluster_embeddings", grab_vectors)
  with forced_factored():
    got = sharded.predict_sharded(c, x)
  kind = "windows-" if windows else ""
  assert stored.last_details["solver"] == "lanczos-%ssharded x1" % kind
  assert c.last_details["solver"] == "lanczos-%sfactored-sharded x1" % kind
  w, w_ref = np.asarray(c.last_details["eigenvalues"]), np.asarray(stored.last_details["eigenvalues"])
  assert len(w) == len(w_ref)
  np.testing.assert_allclose(w, w_ref, rtol=2e-5, atol=2e-6 * np.abs(w_ref).max())
  assert c.last_details["n_clusters"] == stored.last_details["n_clusters"] == SPEAKERS
  assert np.array_equal(scb.utils.enforce_ordered_labels(got), scb.utils.enforce_ordered_labels(want))
  assert np.array_equal(scb.utils.enforce_ordered_labels(got), scb.utils.enforce_ordered_labels(truth))
  residual = factored_residual(grabbed["res"]["y_rows"], grabbed["terms"], grabbed["v"], w)
  assert residual <= 1e-7 * max(1.0, float(np.abs(w).max())), residual
  grabbed.clear()
  free_engine_buffers()


def test_peak_memory_below_the_formula(engine):
  """The refinement's torch allocations beyond what was live before: the formula's buffers plus
  the embeddings' split planes and a few vectors of N."""
  import torch
  import spectralcluster_b200 as scb
  from spectralcluster_b200 import sharded
  n = 65536
  free_engine_buffers()
  x, _ = data(n)
  x_dev = torch.from_numpy(x).to(engine.device)
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  be = sharded.DeviceBackend(engine)
  sharded.FactoredShardedRefiner(be, icassp_options(scb)).run(x_dev, 1, 0)
  torch.cuda.synchronize()
  peak = torch.cuda.max_memory_allocated() - base
  formula = sharded.sharded_factored_peak_bytes(n, 1)
  extra = 2 * 2 * n * D + 64 * 8 * n
  print("factored sharded refinement N=%d world=1: peak %.2f GB, formula %.2f GB (+%.2f GB "
        "planes and vectors)" % (n, peak / 1e9, formula / 1e9, extra / 1e9))
  assert peak <= formula + extra
  del be
  torch.cuda.empty_cache()


def _free_port():
  s = socket.socket()
  s.bind(("127.0.0.1", 0))
  port = s.getsockname()[1]
  s.close()
  return port


def _worker(rank, world, port, use_nccl, n, cases, want, out):
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  import torch
  import torch.distributed as dist
  torch.cuda.set_device(rank if use_nccl else 0)
  dist.init_process_group("nccl" if use_nccl else "gloo", rank=rank, world_size=world)
  import spectralcluster_b200 as scb
  from spectralcluster_b200 import device as dev
  from spectralcluster_b200 import sharded
  eng = dev.Engine.get()
  if want is not None:
    eng.factored_above_bytes = 0
  x, truth = data(n, seed=7 if want is not None else 0)
  report = []
  for case in cases:
    c = make(scb, case)
    torch.cuda.reset_peak_memory_stats()
    labels = sharded.predict_sharded(c, x, dist=dist)
    w = np.asarray(c.last_details["eigenvalues"], dtype=np.float64)
    everyone = [None] * world
    dist.all_gather_object(everyone, w.tobytes())
    ref = want[case] if want is not None else (truth, SPEAKERS)
    report.append(dict(
        case=case, solver=c.last_details["solver"], transport=c.last_details["transport"],
        identical=all(b == everyone[0] for b in everyone),
        labels=bool(np.array_equal(scb.utils.enforce_ordered_labels(labels),
                                   scb.utils.enforce_ordered_labels(ref[0]))),
        k=int(c.last_details["n_clusters"]), k_ref=int(ref[1]),
        peak_gb=torch.cuda.max_memory_allocated() / 1e9))
  peaks = [None] * world
  dist.all_gather_object(peaks, [r["peak_gb"] for r in report])
  if rank == 0:
    out.put((report, peaks))
  dist.destroy_process_group()


def _spawn(world, use_nccl, n, cases, want, timeout=120):
  import torch.multiprocessing as mp
  ctx = mp.get_context("spawn")
  out = ctx.Queue()
  mp.spawn(_worker, args=(world, _free_port(), use_nccl, n, cases, want, out), nprocs=world,
           join=True)
  return out.get(timeout=timeout)


def test_two_ranks_bitwise_identical_and_match_world_1(engine):
  """Two ranks (over NCCL on two GPUs when the box has them, else both on GPU 0 over gloo): the
  exchange and staging code runs, every rank holds the same eigenvalues bit for bit, and the
  labels are those of the world = 1 factored run."""
  import torch
  import spectralcluster_b200 as scb
  from spectralcluster_b200 import sharded
  n = 40000
  x, _ = data(n)
  cases = ["graphcut_10", "graphcut_none"]
  want = {}
  with forced_factored():
    for case in cases:
      c = make(scb, case)
      want[case] = (sharded.predict_sharded(c, x), c.last_details["n_clusters"])
  free_engine_buffers()
  use_nccl = torch.cuda.device_count() >= 2
  report, _ = _spawn(2, use_nccl, n, cases, want)
  assert [r["case"] for r in report] == cases
  for r, windows in zip(report, (False, True)):
    assert r["solver"] == "lanczos-%sfactored-sharded x2" % ("windows-" if windows else ""), r
    assert r["transport"] == ("nccl" if use_nccl else "gloo"), r
    assert r["identical"], r
    assert r["labels"], r
    assert r["k"] == r["k_ref"] == SPEAKERS, r


@pytest.mark.parametrize("n, world", [(131072, 2), (262144, 8)])
def test_beyond_the_stored_route_over_several_gpus(n, world):
  """Sizes the stored sharded route cannot hold on 80 GB cards; the factored route is chosen by
  itself.  Labels must equal the generator's ground truth."""
  import torch
  if torch.cuda.device_count() < world:
    pytest.skip("N = %d over %d GPUs needs %d GPUs; this box has %d"
                % (n, world, world, torch.cuda.device_count()))
  free_engine_buffers()
  report, peaks = _spawn(world, True, n, ["graphcut_10"], None, timeout=600)
  print("N=%d world=%d peak allocated per rank (GB): %s" % (n, world, peaks))
  r = report[0]
  assert r["solver"] == "lanczos-factored-sharded x%d" % world, r
  assert r["identical"] and r["labels"] and r["k"] == SPEAKERS, r
