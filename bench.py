#!/usr/bin/env python
"""Benchmark of the SpectralClusterer.predict() hot path (BASELINE.json metric:
embeddings/sec through predict() at N=65,536 d=256; eigensolve ms).

    python bench.py --gpus N --steps K --warmup W [--impl reference] [--n 65536]

One "step" = one predict() over one batch of N synthetic speaker-turn d-vectors
(SURVEY.md 8(d)).  Workload (BASELINE.json configs[2], the configuration the metric is quoted
on): N=65,536, d=256, ICASSP-2018 refinement sequence, GraphCut Laplacian, eigengap in [2,10].

  value : embeddings/s with the embeddings already resident in HBM (CUDA events)
  e2e   : the same metric through the public API -- predict(np.ndarray) -> np.ndarray, the H2D
          copy of the embeddings and the D2H copy of the labels inside the timed region
  roofline : the dominant kernel (Diffuse, wgmma GEMM) against the tensor peak
  cpu_baseline / --impl reference : the NumPy/SciPy/scikit-learn oracle (a restatement of the
          pure-Python reference, which cannot travel to the GPU box) on a bounded sample

With --gpus N > 1 (torchrun) the default is STRONG scaling of ONE N=65,536 problem: every
N x N matrix is row-sharded over the ranks (spectralcluster_b200/sharded.py, north_star's
split), value = N / time of one predict_sharded(); the labels are checked against the generator's
ground truth inside the run (exit code 3 on a mismatch).  `--workload replicas` runs one
independent batch per GPU instead (weak scaling), `--workload sharded-refine` is BASELINE
configs[3] (N=131,072 through Diffuse + row statistics).
"""

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def parse():
  ap = argparse.ArgumentParser()
  ap.add_argument("--gpus", type=int, default=1)
  ap.add_argument("--steps", type=int, default=3)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
  ap.add_argument("--n", "--size", dest="n", type=int, default=65536)
  ap.add_argument("--d", type=int, default=256)
  ap.add_argument("--speakers", type=int, default=6)
  ap.add_argument("--cpu-sample-n", type=int, default=2048)
  ap.add_argument("--no-cpu-baseline", action="store_true")
  ap.add_argument("--workload", default="auto",
                  choices=["auto", "predict", "replicas", "sharded-refine", "sharded-predict"],
                  help="auto: predict on 1 GPU, sharded-predict (ONE problem, strong scaling) on "
                       "more; replicas: one independent batch per GPU; sharded-refine: configs[3], "
                       "timed region = affinity -> ... -> Diffuse -> row statistics (no eigensolve)")
  ap.add_argument("--cpu-stagewise-n", type=int, default=8192,
                  help="--impl reference: also time the CPU path stage by stage at this N, once, "
                       "outside the timed steps (BASELINE.md section 3 planned 16384: ~70 s; the "
                       "default 8192 takes ~15 s; 0 = skip)")
  ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                  help="predict workload: after the timed steps, write what the last timed step "
                       "computed (labels, eigenvalues) as DIR/<name>.npy in float64")
  args = ap.parse_args()
  if args.dump_outputs and (args.impl != "b200" or args.workload not in ("auto", "predict")):
    ap.error("--dump-outputs covers the single-process predict workload")
  return args


def workload_name(n, d):
  return ("N=%d d=%d synthetic speaker-turn d-vectors; ICASSP2018 refinement "
          "(Crop,Blur,RowMax-Threshold,Symmetrize,Diffuse,RowNormalize) + GraphCut Laplacian + "
          "eigengap k in [2,10] + cosine k-means" % (n, d))


def oracle_options():
  from oracle import spectral_oracle as orc
  return orc.options(min_clusters=2, max_clusters=10, sequence=orc.ICASSP2018,
                     laplacian="graphcut")


def make_clusterer():
  import spectralcluster_b200 as scb
  return scb.SpectralClusterer(
      min_clusters=2, max_clusters=10, laplacian_type=scb.LaplacianType.GraphCut,
      refinement_options=scb.RefinementOptions(
          gaussian_blur_sigma=1, p_percentile=0.95, thresholding_soft_multiplier=0.01,
          thresholding_type=scb.ThresholdType.RowMax,
          refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)),
      custom_dist="cosine")


class ClockSampler(threading.Thread):
  """nvidia-smi clocks / throttle reasons during the timed region."""

  def __init__(self, index):
    super().__init__(daemon=True)
    self.index = index
    self.rows = []
    self.stop_flag = threading.Event()

  def run(self):
    q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")
    while not self.stop_flag.is_set():
      try:
        out = subprocess.run(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q,
                              "--format=csv,noheader,nounits"], capture_output=True, text=True,
                             timeout=5).stdout.strip()
        if out:
          self.rows.append([c.strip() for c in out.split(",")])
      except Exception:
        pass
      self.stop_flag.wait(0.2)

  def summary(self):
    if not self.rows:
      return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
    sm = sorted(int(r[0]) for r in self.rows if r[0].isdigit())
    names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
    reasons = [n for i, n in enumerate(names)
               if any(len(r) > 2 + i and r[2 + i].lower().startswith("active") for r in self.rows)]
    return {"sm_mhz": sm[len(sm) // 2] if sm else None,
            "sm_max_mhz": int(self.rows[0][1]) if self.rows[0][1].isdigit() else None,
            "reasons": reasons, "samples": len(self.rows)}


def all_host_threads():
  """Context manager: let NumPy/OpenBLAS and scikit-learn's OpenMP use every host core, even when
  the launcher exported OMP_NUM_THREADS=1 (torchrun does)."""
  import contextlib
  try:
    import threadpoolctl
    return threadpoolctl.threadpool_limits(limits=os.cpu_count())
  except Exception:
    return contextlib.nullcontext()


def host_threads():
  try:
    import threadpoolctl
    return max((p.get("num_threads", 1) for p in threadpoolctl.threadpool_info()), default=1)
  except Exception:
    return os.cpu_count()


def cpu_baseline(sample_n, d, speakers, repeats=1):
  """Oracle predict() (NumPy/OpenBLAS, SciPy, scikit-learn; all host cores) on a bounded
  sample of the same workload.  eig is ~N^3, so the full N=65,536 is out of reach of the CPU
  path (SURVEY.md section 6: >=137 GB and ~19 h); the sample size is reported."""
  from oracle import spectral_oracle as orc
  x = orc.synthetic_dvectors(sample_n, d, speakers, seed=0)
  opt = oracle_options()
  best = None
  with all_host_threads():
    for _ in range(repeats):
      t0 = time.perf_counter()
      orc.predict(x, opt)
      dt = time.perf_counter() - t0
      best = dt if best is None else min(best, dt)
    threads = host_threads()
  return {"value": sample_n / best, "unit": "embeddings/s", "cores": int(threads), "kind": "port",
          "sample": "oracle predict() on N=%d d=%d of the same generator (%.2f s); the CPU path "
                    "scales ~N^3 and cannot run N=65,536" % (sample_n, d, best),
          "seconds": best}


def run_reference(args, rank):
  if rank != 0:
    return
  total = args.warmup + args.steps
  from oracle import spectral_oracle as orc
  x = orc.synthetic_dvectors(args.cpu_sample_n, args.d, args.speakers, seed=0)
  opt = oracle_options()
  times = []
  with all_host_threads():
    for i in range(total):
      t0 = time.perf_counter()
      orc.predict(x, opt)
      times.append(time.perf_counter() - t0)
    threads = host_threads()
  timed = times[args.warmup:]
  sec = sum(timed) / len(timed)
  val = args.cpu_sample_n / sec
  line = {
      "impl": "reference", "metric": "embeddings/sec through predict()", "value": val,
      "unit": "embeddings/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
      "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "weak",
      "vs_baseline": None, "dtype": "f64", "data": "synthetic",
      "config": {"workload": workload_name(args.n, args.d),
                 "sample": "each step = the CPU path on N=%d of the same generator" % args.cpu_sample_n},
      "cpu_baseline": {"value": val, "unit": "embeddings/s", "cores": int(threads),
                       "kind": "port",
                       "sample": "oracle (NumPy/SciPy/scikit-learn restatement of the pure-Python "
                                 "reference) predict() on N=%d d=%d per step" % (args.cpu_sample_n, args.d)},
      "e2e": {"value": val, "unit": "embeddings/s", "h2d_bytes_per_step": 0,
              "d2h_bytes_per_step": 0},
      "gpu_launches": 0,
  }
  if args.cpu_stagewise_n > 0:
    line["cpu_stagewise"] = cpu_stagewise(args.cpu_stagewise_n, args.d, args.speakers)
  emit(line)


def cpu_stagewise(n, d, speakers):
  """Seconds per stage of the CPU path (oracle = NumPy/SciPy restatement of the reference) at a
  size where the N x N stages still fit the host (BASELINE.md section 3: N=16,384; the O(N^3)
  np.linalg.eig is excluded -- SURVEY.md section 6 measured 138 s at N=8,192, exponent 2.96)."""
  from oracle import spectral_oracle as orc
  x = orc.synthetic_dvectors(n, d, speakers, seed=0)
  out = {}
  with all_host_threads():
    def timed(name, fn):
      t0 = time.perf_counter()
      r = fn()
      out[name] = time.perf_counter() - t0
      return r
    a = timed("affinity", lambda: orc.affinity(x))
    a = timed("crop_diagonal", lambda: orc.crop_diagonal(a))
    a = timed("gaussian_blur", lambda: orc.gaussian_blur(a, 1.0))
    a = timed("row_threshold", lambda: orc.row_threshold(a, 0.95, 0.01))
    a = timed("symmetrize", lambda: orc.symmetrize(a))
    a = timed("diffuse", lambda: orc.diffuse(a))
    a = timed("row_normalize", lambda: orc.row_normalize(a))
    threads = host_threads()
  return {"n": n, "seconds": out, "cores": int(threads),
          "note": "eig (utils.py:59) and the Laplacian's two dense N^3 dots (laplacian.py:53,57) "
                  "are not run at this size"}


def run_sharded(args, eng, rank, world, dist):
  """configs[3]: one N x N problem, rows sharded over the ranks (spectralcluster_b200/sharded.py)."""
  import torch
  import spectralcluster_b200 as scb
  from spectralcluster_b200 import _native as nat
  from spectralcluster_b200 import sharded, synthetic
  n, d = args.n, args.d
  x = torch.from_numpy(synthetic.speaker_turn_dvectors(n, d, 8, seed=0).astype(np.float32)).to(eng.device)
  opt = scb.RefinementOptions(gaussian_blur_sigma=1, p_percentile=0.95,
                              thresholding_soft_multiplier=0.01,
                              refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))
  refiner = sharded.ShardedRefiner(sharded.DeviceBackend(eng), opt,
                                   dist=dist if world > 1 else None)

  def barrier():
    if world > 1:
      dist.barrier()
    torch.cuda.synchronize()

  for _ in range(args.warmup):
    res = refiner.run(x, world, rank)
    del res
  barrier()
  launches0 = nat.load().sc_launch_count()
  eng.start_profile()
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for step in range(args.steps):
    if step == args.steps - 1:
      refiner.trace = []
    res = refiner.run(x, world, rank)
    del res
  stop.record()
  barrier()
  ms = start.elapsed_time(stop)
  stages = eng.stop_profile()
  trace = refiner.trace or []
  timeline = {trace[i][0]: trace[0][1].elapsed_time(trace[i][1]) for i in range(1, len(trace))}
  launches = nat.load().sc_launch_count() - launches0
  if world > 1:
    tt = torch.tensor([ms], dtype=torch.float64, device=eng.device)
    dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    ms = float(tt[0])
  if rank == 0:
    per = ms / args.steps
    gemm_ms = stages.get("sc_gemm_nt_planes", 0.0) / args.steps
    emit(({
        "metric": "embeddings/sec through the row-sharded refinement (affinity..Diffuse..row stats)",
        "value": n / (per / 1e3), "unit": "embeddings/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": per, "higher_is_better": True, "scaling": "strong",
        "vs_baseline": None, "dtype": "f32 storage; fp16x3 split tensor-core products", "data": "synthetic",
        "config": {"workload": "N=%d d=%d ICASSP2018 refinement through Diffuse + row statistics, "
                               "row-sharded over %d GPU(s) (BASELINE configs[3])" % (n, d, world),
                   "parallelism": "row-shard x%d, broadcast of Y row blocks overlapped with per-peer GEMMs" % world},
        "gpu_launches": int(launches),
        "stage_ms_rank0": {k: v / args.steps for k, v in sorted(stages.items())},
        "timeline_ms_rank0_last_step": timeline,
        "roofline": {"kernel": "k_gemm_wgmma (per-peer Diffuse blocks, rank 0)", "bound": "tensor",
                     "achieved": (2.0 * n * n * n / world) / (gemm_ms * 1e-3) / 1e12 if gemm_ms else None,
                     "unit": "TFLOP/s", "traffic": None}}))
  if world > 1:
    dist.destroy_process_group()


def dtype_string(eng, n):
  from spectralcluster_b200 import _native as nat
  scheme = {nat.GEMM_SPLIT3: "fp16x3 split (hi*hi + hi*lo + lo*hi)",
            nat.GEMM_SPLIT2: "fp16x2 split ((hi+lo)*hi)",
            nat.GEMM_SINGLE: "fp16 single (hi*hi)"}[eng.diffuse_precision_for(n)]
  return ("f32 storage; affinity: fp16x3 split wgmma MMAs; Diffuse: %s wgmma MMAs, f32 "
          "two-level accumulate; f64 eigensolve and k-means" % scheme)


def mma_per_product(eng, n):
  from spectralcluster_b200 import _native as nat
  return {nat.GEMM_SPLIT3: 3, nat.GEMM_SPLIT2: 2, nat.GEMM_SINGLE: 1}[eng.diffuse_precision_for(n)]


def roofline_diffuse(eng, n, diffuse_ms, tensor_peak, peak_note, traffic):
  """The dominant kernel against the measured tensor peak.  `achieved` counts the fp16 MMA flop the
  kernel EXECUTES: it computes only the tiles that touch the upper triangle of S = Y Y^T and
  mirrors them (N^3 multiply-adds x 2 / 2 per MMA plane), times the MMAs issued per product.
  SURVEY.md 8(d) quotes 2 N^3 for the full product: reported beside it, not as the fraction."""
  if not diffuse_ms:
    return {"kernel": "k_gemm_wgmma (Diffuse, Y Y^T)", "bound": "tensor", "achieved": None,
            "peak": tensor_peak, "unit": "TFLOP/s", "frac": None, "traffic": traffic}
  mmas = mma_per_product(eng, n)
  tri = 1.0 * n * n * n / (diffuse_ms * 1e-3) / 1e12          # N^3: the triangle, one MMA per product
  return {"kernel": "k_gemm_wgmma (Diffuse, Y Y^T)", "bound": "tensor",
          "achieved": tri * mmas, "peak": tensor_peak, "unit": "TFLOP/s",
          "frac": tri * mmas / tensor_peak, "traffic": traffic, "peak_source": peak_note,
          "basis": "executed fp16 MMA flop = %d x N^3 (upper-triangle tiles only, %d MMA(s) per "
                   "product) / CUDA-event time of sc_diffuse" % (mmas, mmas),
          "triangle_basis": {"achieved": tri, "frac": tri / tensor_peak,
                             "note": "N^3 algorithmic flop of the triangle (SURVEY.md 8(d))"},
          "full_product_basis": {"achieved": 2 * tri, "ratio_to_peak": 2 * tri / tensor_peak,
                                 "note": "2 N^3 of the full product Y Y^T; the mirrored half is "
                                         "stored, not computed, so this is a speed-up figure, "
                                         "not a pipe utilisation"}}


def roofline_refinement(eng, n, stages, steps, hbm_peak):
  """Crop -> Blur -> RowMax threshold -> Symmetrize against the measured HBM bandwidth, on the
  contract basis of SURVEY.md 8(d) (12 B per affinity element) and on the bytes the kernels
  actually move."""
  from spectralcluster_b200 import _native as nat
  t1 = (stages.get("sc_blur_upper_rowmax", 0) + stages.get("sc_gaussian_blur_rowmax", 0)) / steps
  t2 = (stages.get("sc_threshold_symmetrize_upper", 0) + stages.get("sc_blur_threshold_symmetrize", 0)) / steps
  symmetric_pair = "sc_blur_upper_rowmax" in stages
  if symmetric_pair:
    # pass 1 reads the upper tiles of A and stores the upper tiles of B (2 + 2 B per matrix
    # element); pass 2 reads them (2) and writes every element of Y: fp16 hi (+ lo) plane
    y_bytes = 2 if eng.diffuse_precision_for(n) == nat.GEMM_SINGLE else 4
    moved = 2 + 2 + 2 + y_bytes
    how = "symmetric pair: blur the upper tiles once (read 2 + write 2 B/element), element-wise " \
          "threshold/symmetrize with mirrored stores (read 2 + write %d B/element)" % y_bytes
  else:
    moved = 12
    how = "two blur passes over the whole matrix (read 4, read 4 + write 4 B/element)"
  tot = t1 + t2
  gb = n * n / 1e9
  return {"blur_rowmax_pass_ms": t1 or None, "threshold_symmetrize_pass_ms": t2 or None,
          "fused_chain_GBps": 12 * gb / (tot / 1e3) if tot else None,
          "fused_chain_frac": 12 * gb / (tot / 1e3) / hbm_peak if tot else None,
          "basis": "12 B per affinity element (SURVEY.md 8(d)): read A, read A, write Y planes",
          "moved_bytes_per_element": moved,
          "moved_GBps": moved * gb / (tot / 1e3) if tot else None,
          "moved_frac": moved * gb / (tot / 1e3) / hbm_peak if tot else None,
          "kernels": how, "peak_GBps": hbm_peak}


# NVIDIA's H100 SXM data sheet (700 W card): dense fp16/bf16 tensor rate and HBM3 bandwidth, the
# denominators when no measured peaks are given
H100_FP16_DENSE_TFLOPS = 989.0
H100_HBM_GBPS = 3350.0


def load_peaks():
  try:
    return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
  except Exception:
    return {}


def run_sharded_predict(args, eng, rank, world, dist):
  """ONE N x N problem end to end (predict) with every matrix row-sharded over the ranks: the
  north_star split, strong scaling.  value = N / device time of predict_sharded() with the
  embeddings resident in HBM (CUDA events, max over ranks); e2e = the same call fed a host
  ndarray (H2D of the embeddings and D2H of the labels inside the timed region)."""
  import torch
  from spectralcluster_b200 import _native as nat
  from spectralcluster_b200 import sharded, synthetic, utils
  n, d = args.n, args.d
  x, truth = synthetic.speaker_turn_dvectors(n, d, args.speakers, seed=0, return_labels=True)
  x = x.astype(np.float32)
  x_pinned = torch.from_numpy(x).pin_memory()
  x_dev = torch.from_numpy(x).to(eng.device)
  clusterer = make_clusterer()
  group = dist if world > 1 else None

  def barrier():
    if world > 1:
      dist.barrier()
    torch.cuda.synchronize()

  def check(labels, what):
    if not np.array_equal(utils.enforce_ordered_labels(labels), utils.enforce_ordered_labels(truth)):
      sys.stderr.write("bench: %s labels differ from the generator's ground truth\n" % what)
      sys.stderr.flush()
      os._exit(3)

  # ---------------- e2e: host ndarray in, host labels out
  labels = None
  for _ in range(args.warmup):
    labels = sharded.predict_sharded(clusterer, x_pinned.numpy(), dist=group)
  barrier()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    labels = sharded.predict_sharded(clusterer, x_pinned.numpy(), dist=group)
  barrier()
  e2e_s = time.perf_counter() - t0
  check(labels, "e2e")

  # ---------------- device-resident: embeddings already in HBM, CUDA events
  for _ in range(max(1, args.warmup - 2)):
    sharded.predict_sharded(clusterer, x_dev, dist=group)
  barrier()
  sampler = ClockSampler(int(os.environ.get("LOCAL_RANK", "0")))
  sampler.start()
  launches0 = nat.load().sc_launch_count()
  eng.start_profile()
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(args.steps):
    labels = sharded.predict_sharded(clusterer, x_dev, dist=group)
  stop.record()
  barrier()
  dev_ms = start.elapsed_time(stop)
  stages = eng.stop_profile()
  launches = nat.load().sc_launch_count() - launches0
  sampler.stop_flag.set()
  sampler.join(timeout=2)
  check(labels, "device-resident")
  # one more step with the timeline markers on (outside the timed region)
  refiner_trace = {}
  if True:
    from spectralcluster_b200 import device as dev
    be = eng._sharded_backend
    r = sharded.ShardedRefiner(be, clusterer.refinement_options, dist=group)
    r.trace = []
    r.run(x_dev, world, rank)
    torch.cuda.synchronize()
    refiner_trace = {r.trace[i][0]: r.trace[0][1].elapsed_time(r.trace[i][1])
                     for i in range(1, len(r.trace))}
  if world > 1:
    tt = torch.tensor([dev_ms, e2e_s], dtype=torch.float64, device=eng.device)
    dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    dev_ms, e2e_s = float(tt[0]), float(tt[1])
  if rank == 0:
    per = dev_ms / args.steps
    peaks = load_peaks()
    tensor_peak = peaks.get("bf16_tflops_sustained") or H100_FP16_DENSE_TFLOPS
    gemm_ms = stages.get("sc_gemm_nt_planes", 0.0) / args.steps
    # per rank: G/2 of the G^2 block products of the full 2 N^3 flop product (symmetry across ranks)
    flops_rank = 2.0 * n * n * n / (2.0 * world) if world > 1 else 2.0 * n * n * n / 2.0
    achieved = flops_rank / (gemm_ms * 1e-3) / 1e12 if gemm_ms else None
    emit({
        "metric": "embeddings/sec through predict()", "value": n / (per / 1e3),
        "unit": "embeddings/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": per, "higher_is_better": True, "scaling": "strong",
        "vs_baseline": None, "dtype": dtype_string(eng, n), "data": "synthetic",
        "config": {"workload": workload_name(n, d),
                   "l2": "inputs larger than L2 (N x N fp32 = %.1f GB over %d GPUs)" % (n * n * 4 / 1e9, world),
                   "parallelism": "ONE problem, N x N matrices row-sharded x%d (strong scaling)" % world,
                   "transport": clusterer.last_details.get("transport"),
                   "labels_match_generator_truth": True,
                   "clusters_found": clusterer.last_details.get("n_clusters"),
                   "eigensolver": clusterer.last_details.get("solver"),
                   "lanczos_stats[matvecs,restarts,converged,passes_over_S]": clusterer.last_details.get("lanczos_stats")},
        "e2e": {"value": n * args.steps / e2e_s, "unit": "embeddings/s",
                "h2d_bytes_per_step": int(x.nbytes) * world, "d2h_bytes_per_step": int(labels.nbytes) * world},
        "gpu_launches": int(launches),
        "eigensolve_ms": stages.get("sc_eigh_extremal_sharded", 0.0) / args.steps,
        "stage_ms_rank0": {k: v / args.steps for k, v in sorted(stages.items())},
        "timeline_ms_rank0": refiner_trace,
        "roofline": {"kernel": "k_gemm_wgmma (rank 0's Diffuse block products)", "bound": "tensor",
                     "achieved": achieved, "peak": tensor_peak, "unit": "TFLOP/s",
                     "frac": (achieved / tensor_peak) if achieved else None, "traffic": None,
                     "note": "achieved = this rank's share of the N^3 triangle-basis flop / CUDA-event "
                             "time of its sc_gemm_nt_planes calls; %d MMAs issued per product"
                             % mma_per_product(eng, n)},
        "clocks": sampler.summary()})
  if world > 1:
    dist.destroy_process_group()


class StdoutGuard:
  """Keeps stdout to the single JSON line: NCCL prints its version banner on fd 1 when the first
  communicator is created, whatever NCCL_DEBUG says.  Everything written to fd 1 while the guard
  is active goes to stderr; result() restores fd 1 and prints."""

  def __init__(self):
    sys.stdout.flush()
    self.saved = os.dup(1)
    os.dup2(2, 1)

  def result(self, line: str):
    sys.stdout.flush()
    os.dup2(self.saved, 1)
    sys.stdout.write(line + "\n")
    sys.stdout.flush()
    # ... and back to stderr: with NCCL_DEBUG=INFO the communicator teardown logs on fd 1 too
    os.dup2(2, 1)


GUARD = None


def emit(obj):
  line = json.dumps(obj)
  if GUARD is not None:
    GUARD.result(line)
  else:
    print(line)


def main():
  global GUARD
  args = parse()
  GUARD = StdoutGuard()
  rank = int(os.environ.get("RANK", "0"))
  local_rank = int(os.environ.get("LOCAL_RANK", "0"))
  world = int(os.environ.get("WORLD_SIZE", "1"))
  if args.impl == "reference":
    run_reference(args, rank)
    return

  import torch
  import torch.distributed as dist
  from spectralcluster_b200 import _native as nat
  from spectralcluster_b200 import device as dev
  from spectralcluster_b200 import synthetic

  torch.cuda.set_device(local_rank)
  if world > 1:
    # NCCL's own log stays on (the StdoutGuard keeps fd 1 clean for the JSON line): the driver
    # reads the communicator size from it
    if os.environ.get("NCCL_DEBUG", "").upper() not in ("INFO", "TRACE"):
      os.environ["NCCL_DEBUG"] = "INFO"          # images preset VERSION/WARN: the init lines matter
      os.environ.setdefault("NCCL_DEBUG_SUBSYS", "INIT")
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
  eng = dev.Engine.get(local_rank)
  n, d = args.n, args.d
  workload = args.workload
  if workload == "auto":
    workload = "predict" if world == 1 else "sharded-predict"
  if workload == "sharded-refine":
    run_sharded(args, eng, rank, world, dist)
    return
  if workload == "sharded-predict":
    run_sharded_predict(args, eng, rank, world, dist)
    return
  # every rank clusters its own batch (different seed): weak scaling over independent units
  x = synthetic.speaker_turn_dvectors(n, d, args.speakers, seed=rank).astype(np.float32)
  x_pinned = torch.from_numpy(x).pin_memory()
  clusterer = make_clusterer()

  def barrier():
    if world > 1:
      dist.barrier()
    torch.cuda.synchronize()

  # ---------------- e2e: host ndarray in, host labels out
  labels = None
  for _ in range(args.warmup):
    labels = clusterer.predict(x_pinned.numpy())
  barrier()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    labels = clusterer.predict(x_pinned.numpy())
  barrier()
  e2e_s = time.perf_counter() - t0
  k_found = clusterer.last_details.get("n_clusters")

  # ---------------- device-resident: embeddings already in HBM, CUDA events
  from spectralcluster_b200 import spectral_clusterer as sc_mod
  x_dev = torch.from_numpy(x).to(eng.device)
  seq = clusterer.refinement_options.refinement_sequence

  def device_step():
    a, crop = eng.affinity(x_dev, want_crop_vector=True)
    aff = sc_mod.DeviceAffinity(a, n, crop, True)
    v, k, _ = clusterer._compute_eigenvectors_ncluster(aff)
    k = max(k, clusterer.min_clusters)
    emb = v[:, :k].contiguous()
    return eng.kmeans(emb, k, 0, clusterer.max_iter)[0]

  def dump_outputs(labels):
    # the labels predict() returns and the eigenvalues it decided k from (last_details)
    os.makedirs(args.dump_outputs, exist_ok=True)
    out = {"labels": labels, "eigenvalues": clusterer.last_details["eigenvalues"]}
    for name, arr in out.items():
      np.save(os.path.join(args.dump_outputs, name + ".npy"), np.asarray(arr, dtype=np.float64))

  for _ in range(max(1, args.warmup - 2)):     # the e2e loop above already warmed everything
    device_step()
  barrier()
  sampler = ClockSampler(local_rank)
  sampler.start()
  launches0 = nat.load().sc_launch_count()
  eng.start_profile()
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(args.steps):
    labels = device_step()
  stop.record()
  barrier()
  dev_ms = start.elapsed_time(stop)
  stages = eng.stop_profile()
  launches = nat.load().sc_launch_count() - launches0
  sampler.stop_flag.set()
  sampler.join(timeout=2)
  if args.dump_outputs and rank == 0:
    dump_outputs(labels)

  if world > 1:
    tt = torch.tensor([dev_ms, e2e_s], dtype=torch.float64, device=eng.device)
    dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    dev_ms, e2e_s = float(tt[0]), float(tt[1])
  if rank != 0:
    if world > 1:
      dist.destroy_process_group()
    return

  ms_per_step = dev_ms / args.steps
  value = world * n / (ms_per_step / 1e3)
  e2e_value = world * n * args.steps / e2e_s
  peaks = {}
  try:
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
  except Exception:
    pass
  tensor_peak = peaks.get("bf16_tflops_sustained") or H100_FP16_DENSE_TFLOPS
  peak_note = "measured (MEASURED_PEAKS.json, sustained fp16/bf16 dense)" if peaks else \
      "H100 SXM data sheet, dense fp16 (not a measured rate)"
  diffuse_ms = stages.get("sc_diffuse", 0.0) / args.steps
  hbm_peak = peaks.get("hbm_gbs") or H100_HBM_GBPS
  traffic = None
  line = {
      "metric": "embeddings/sec through predict()", "value": value, "unit": "embeddings/s",
      "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step,
      "higher_is_better": True, "scaling": "weak" if world > 1 else "strong", "vs_baseline": None,
      "dtype": dtype_string(eng, n),
      "data": "synthetic",
      "config": {"workload": workload_name(n, d), "l2": "inputs larger than L2 (N x N fp32 = %.1f GB)"
                 % (n * n * 4 / 1e9), "parallelism": "replicas x%d" % world,
                 "clusters_found": k_found,
                 "eigensolver": clusterer.last_details.get("solver"),
                 "lanczos_stats[matvecs,restarts,converged,passes_over_S]": clusterer.last_details.get("lanczos_stats")},
      "e2e": {"value": e2e_value, "unit": "embeddings/s", "h2d_bytes_per_step": int(x.nbytes),
              "d2h_bytes_per_step": int(labels.nbytes) + 8 * 16},
      "gpu_launches": int(launches),
      "eigensolve_ms": (stages.get("sc_eigh_extremal", 0.0) + stages.get("sc_eigh_dense", 0.0)) / args.steps,
      "stage_ms": {k: v / args.steps for k, v in sorted(stages.items())},
      "roofline": roofline_diffuse(eng, n, diffuse_ms, tensor_peak, peak_note, traffic),
      "roofline_hbm_stages": roofline_refinement(eng, n, stages, args.steps, hbm_peak),
      "clocks": sampler.summary(),
  }
  if not args.no_cpu_baseline:
    line["cpu_baseline"] = cpu_baseline(args.cpu_sample_n, d, args.speakers)
  emit(line)
  if world > 1:
    dist.destroy_process_group()


if __name__ == "__main__":
  main()
