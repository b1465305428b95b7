"""GPU: predict_sharded() in eigenvalue windows (max_clusters None or >= 32, and NormalizedDiff on
a Laplacian) against single-GPU predict().  N = 40,000 is above the dense solver's N, so predict()
takes its windowed route too.

The sharded and unsharded S agree to 2e-6 relative element-wise, not bitwise
(test_gpu_sharded.py::test_two_ranks_match_unsharded), so eigenvalues are compared within twice
the project's contract, |dw| <= 2e-5 |w| + 2e-6 max|w|, and the eigenpair residuals are taken
against the sharded S itself.  world = 2 runs over NCCL on two GPUs when the box has them, else
both ranks on GPU 0 with gloo, as test_gpu_sharded.py does."""

import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

N, D, SPEAKERS = 40000, 256, 6


@pytest.fixture(autouse=True, scope="module")
def release_sharded_buffers():
  """predict_sharded() keeps its N x N-scale buffers on the engine for the next call (13 GB at
  N = 40,000); give them back so that later tests have the whole card."""
  yield
  import torch
  from spectralcluster_b200 import device as dev
  eng = dev.Engine.get()
  if getattr(eng, "_sharded_backend", None) is not None:
    del eng._sharded_backend
  torch.cuda.empty_cache()


def icassp_options(scb):
  return scb.RefinementOptions(
      gaussian_blur_sigma=1, p_percentile=0.95, thresholding_soft_multiplier=0.01,
      refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))


def make(scb, case):
  GC = scb.LaplacianType.GraphCut
  kw = dict(graphcut_none=dict(laplacian_type=GC),
            nolaplacian_none=dict(),
            graphcut_40=dict(laplacian_type=GC, max_clusters=40),
            graphcut_ndiff_10=dict(laplacian_type=GC, max_clusters=10,
                                   eigengap_type=scb.EigenGapType.NormalizedDiff))[case]
  return scb.SpectralClusterer(min_clusters=2, refinement_options=icassp_options(scb), **kw)


def data():
  from oracle import spectral_oracle as orc
  return orc.synthetic_dvectors(N, D, SPEAKERS, seed=7, return_labels=True)


def assert_values_close(w, want):
  w, want = np.asarray(w), np.asarray(want)
  np.testing.assert_allclose(w, want, rtol=2e-5, atol=2e-6 * np.abs(want).max())


class Captured:
  """The sharded S, the operator terms and the eigenvectors predict_sharded() hands to k-means."""

  def __init__(self, monkeypatch, clusterer):
    from spectralcluster_b200 import laplacian, sharded
    run, terms = sharded.ShardedRefiner.run, laplacian.terms_from_row_sums
    cluster = clusterer._cluster_embeddings

    def grab_run(refiner, *a, **kw):
      self.res = run(refiner, *a, **kw)
      return self.res

    def grab_terms(*a, **kw):
      self.terms = terms(*a, **kw)
      return self.terms

    def grab_vectors(eng, v, k):
      self.v = v.clone()
      return cluster(eng, v, k)

    monkeypatch.setattr(sharded.ShardedRefiner, "run", grab_run)
    monkeypatch.setattr(laplacian, "terms_from_row_sums", grab_terms)
    monkeypatch.setattr(clusterer, "_cluster_embeddings", grab_vectors)

  def residual(self, w):
    """max_j |M v_j - w_j v_j|_inf in float64, M = diag(delta) + sign diag(left) S diag(right)
    with the sharded S (world = 1: the whole matrix)."""
    import torch
    s = self.res["s_block"]
    delta, left, right, sign, _ = self.terms
    v = self.v.double()
    n, cols = v.shape
    x = v if right is None else v * right[:, None]
    sx = torch.empty_like(v)
    for i in range(0, n, 4096):
      sx[i:i + 4096] = s[i:i + 4096, :n].double() @ x
    mv = sign * (sx if left is None else sx * left[:, None])
    if delta is not None:
      mv += delta[:, None] * v
    lam = torch.as_tensor(np.asarray(w[:cols]), dtype=torch.float64, device=v.device)
    return float((mv - v * lam[None, :]).abs().max())


@pytest.mark.parametrize("case, solver", [
    ("graphcut_none", "lanczos-windows"),
    ("nolaplacian_none", "lanczos-windows"),
    ("graphcut_40", "lanczos-windows"),
    ("graphcut_ndiff_10", "lanczos"),
])
def test_world1_matches_predict(engine, monkeypatch, case, solver):
  import torch
  import spectralcluster_b200 as scb
  from spectralcluster_b200 import sharded
  x, truth = data()
  single = make(scb, case)
  want = single.predict(x)
  torch.cuda.empty_cache()
  c = make(scb, case)
  cap = Captured(monkeypatch, c)
  got = sharded.predict_sharded(c, x)
  sharded_solver = ("lanczos-windows-sharded x1" if solver == "lanczos-windows"
                    else "lanczos-sharded x1")
  assert single.last_details["solver"] == solver
  assert c.last_details["solver"] == sharded_solver
  w, w_ref = np.asarray(c.last_details["eigenvalues"]), np.asarray(single.last_details["eigenvalues"])
  assert len(w) == len(w_ref)
  assert_values_close(w, w_ref)
  assert c.last_details["n_clusters"] == single.last_details["n_clusters"] == SPEAKERS
  assert np.array_equal(scb.utils.enforce_ordered_labels(got), scb.utils.enforce_ordered_labels(want))
  assert np.array_equal(scb.utils.enforce_ordered_labels(got), scb.utils.enforce_ordered_labels(truth))
  if case == "graphcut_40":
    assert len(w) == 41
  if case == "graphcut_ndiff_10":
    # the gap is normalised by the appended sharded lambda_max solve
    assert np.isclose(c.last_details["max_gap"], single.last_details["max_gap"], rtol=1e-4, atol=0)
  stats = c.last_details["lanczos_stats"]
  if solver == "lanczos-windows":
    assert stats["windows"] == single.last_details["lanczos_stats"]["windows"]
  residual = cap.residual(w)
  assert residual <= 1e-7 * max(1.0, float(np.abs(w).max())), residual
  del cap
  torch.cuda.empty_cache()


def test_world1_cap(engine, monkeypatch):
  """GraphCut with max_clusters=None needs at least 7 values (6 speakers): a cap of 4 raises from
  the windows driver, naming the cap, as predict() does."""
  import spectralcluster_b200 as scb
  from spectralcluster_b200 import eigen_windows as ew
  from spectralcluster_b200 import sharded
  x, _ = data()
  monkeypatch.setattr(ew, "MAX_WINDOW_PAIRS", 4)
  with pytest.raises(NotImplementedError, match="first 4 eigenvalues"):
    sharded.predict_sharded(make(scb, "graphcut_none"), x)


def _free_port():
  s = socket.socket()
  s.bind(("127.0.0.1", 0))
  port = s.getsockname()[1]
  s.close()
  return port


def _worker(rank, world, port, use_nccl, cases, want, out):
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  import torch
  import torch.distributed as dist
  torch.cuda.set_device(rank if use_nccl else 0)
  dist.init_process_group("nccl" if use_nccl else "gloo", rank=rank, world_size=world)
  import spectralcluster_b200 as scb
  from spectralcluster_b200 import sharded
  x, _ = data()
  report = []
  for case in cases:
    c = make(scb, case)
    labels = sharded.predict_sharded(c, x, dist=dist)
    w = np.asarray(c.last_details["eigenvalues"], dtype=np.float64)
    everyone = [None] * world
    dist.all_gather_object(everyone, w.tobytes())
    labels_ref, k_ref = want[case]
    report.append(dict(
        case=case, solver=c.last_details["solver"],
        identical=all(b == everyone[0] for b in everyone),
        labels=bool(np.array_equal(scb.utils.enforce_ordered_labels(labels),
                                   scb.utils.enforce_ordered_labels(labels_ref))),
        k=int(c.last_details["n_clusters"]), k_ref=int(k_ref)))
  if rank == 0:
    out.put(report)
  dist.destroy_process_group()


def test_two_ranks_bitwise_identical_and_match_single_gpu(engine):
  import torch
  import torch.multiprocessing as mp
  import spectralcluster_b200 as scb
  x, _ = data()
  cases = ["graphcut_none", "graphcut_40"]
  want = {}
  for case in cases:
    c = make(scb, case)
    want[case] = (c.predict(x), c.last_details["n_clusters"])
  torch.cuda.synchronize()
  torch.cuda.empty_cache()
  use_nccl = torch.cuda.device_count() >= 2
  ctx = mp.get_context("spawn")
  out = ctx.Queue()
  mp.spawn(_worker, args=(2, _free_port(), use_nccl, cases, want, out), nprocs=2, join=True)
  report = out.get(timeout=60)
  assert [r["case"] for r in report] == cases
  for r in report:
    assert r["solver"] == "lanczos-windows-sharded x2", r
    assert r["identical"], r
    assert r["labels"], r
    assert r["k"] == r["k_ref"] == SPEAKERS, r


def _large_worker(rank, world, port, out):
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  import torch
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group("nccl", rank=rank, world_size=world)
  import spectralcluster_b200 as scb
  from spectralcluster_b200 import sharded
  from oracle import spectral_oracle as orc
  x, truth = orc.synthetic_dvectors(131072, D, SPEAKERS, seed=0, return_labels=True)
  c = make(scb, "graphcut_none")
  labels = sharded.predict_sharded(c, x, dist=dist)
  if rank == 0:
    out.put(dict(k=int(c.last_details["n_clusters"]), solver=c.last_details["solver"],
                 labels=bool(np.array_equal(scb.utils.enforce_ordered_labels(labels),
                                            scb.utils.enforce_ordered_labels(truth)))))
  dist.destroy_process_group()


def test_131072_over_every_gpu_graphcut_max_clusters_none():
  import torch
  import torch.multiprocessing as mp
  from spectralcluster_b200 import sharded
  world = torch.cuda.device_count()
  if world < 2:
    pytest.skip("N = 131,072 row-sharded needs at least 2 GPUs; this box has %d" % world)
  n = 131072
  block = sharded.ShardPlan(n, world, 0, 4).block
  ld = (n + 63) // 64 * 64
  # per rank: the full-size Y planes (2 x fp16), the S row block (fp32), the locked set
  need = 2 * 2 * world * block * ld + 4 * (block + 128) * ld + 8 * 512 * n
  total = torch.cuda.get_device_properties(0).total_memory
  if need > total - (4 << 30):
    pytest.skip("N = 131,072 over %d GPUs needs %.1f GB per GPU on the sharded path; each has "
                "%.1f GB" % (world, need / 1e9, total / 1e9))
  ctx = mp.get_context("spawn")
  out = ctx.Queue()
  mp.spawn(_large_worker, args=(world, _free_port(), out), nprocs=world, join=True)
  r = out.get(timeout=60)
  assert r["solver"] == "lanczos-windows-sharded x%d" % world
  assert r["k"] == SPEAKERS
  assert r["labels"]
