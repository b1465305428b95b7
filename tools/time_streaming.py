#!/usr/bin/env python
"""Times MultiStageClusterer.streaming_predict per step, fed host ndarrays and fed CUDA tensors
(and host ndarrays with the cooperative NN-chain at every size, the kernel choice before
sc_nn_chain_small), and the two NN-chain kernels per call (sc_nn_chain_small, one thread block,
against the cooperative sc_complete_linkage / sc_average_linkage) on the same matrices.

A step's time is the host clock around streaming_predict, which returns host labels (so the
device work of the step has finished).  Steps are reported in the stream's three phases: up to L
(the fallback clusterer), up to U1 (the main clusterer alone) and past U1 (pre-clusterer,
centroids, main clusterer).  A kernel call is the host clock around the synchronous C-ABI entry
(launch, merges, copy of the merges to the host), on a fresh copy of the distance matrix.

    python tools/time_streaming.py [--steps 2000] [--d 256] [--repeats 1]
                                   [--kernel-sizes 100,600,<NN_SMALL_MAX>] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import multi_stage_clusterer as ms
from spectralcluster_b200 import synthetic

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=2000)
ap.add_argument("--d", type=int, default=256)
ap.add_argument("--speakers", type=int, default=4)
ap.add_argument("--L", type=int, default=50)
ap.add_argument("--U1", type=int, default=100)
ap.add_argument("--U2", type=int, default=600)
ap.add_argument("--repeats", type=int, default=1, help="alternating host / device streams")
ap.add_argument("--kernel-sizes", default="100,600,%d" % nat.NN_SMALL_MAX)
ap.add_argument("--reps", type=int, default=20, help="timed calls per kernel and size")
a = ap.parse_args()


def query(fields):
  out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  return out.splitlines()[torch.cuda.current_device()] if out else "nvidia-smi unavailable"


def emit(obj):
  print(json.dumps(obj), flush=True)


emit({"card": query("name,power.limit,clocks.max.sm"), "torch_name": torch.cuda.get_device_name()})
eng = dev.Engine.get()


def make_stream():
  main = scb.SpectralClusterer(
      min_clusters=2, max_clusters=7,
      refinement_options=scb.RefinementOptions(
          gaussian_blur_sigma=0, p_percentile=0.9,
          refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)))
  return ms.MultiStageClusterer(main, fallback_threshold=0.5, L=a.L, U1=a.U1, U2=a.U2,
                                deflicker=ms.Deflicker.Hungarian)


def run_stream(rows):
  """Per-step milliseconds and the labels of the last step."""
  s = make_stream()
  out = []
  for e in rows:
    t0 = time.perf_counter()
    labels = s.streaming_predict(e)
    out.append(1e3 * (time.perf_counter() - t0))
  torch.cuda.synchronize()
  return np.array(out), labels


def phases(ms_per_step):
  step = np.arange(1, len(ms_per_step) + 1)
  out = {}
  for name, sel in (("<=L", step <= a.L), ("<=U1", (step > a.L) & (step <= a.U1)),
                    (">U1", step > a.U1)):
    v = ms_per_step[sel]
    out[name] = {"steps": int(v.size), "median_ms": round(float(np.median(v)), 3),
                 "p99_ms": round(float(np.percentile(v, 99)), 3)} if v.size else None
  return out


x = synthetic.speaker_turn_dvectors(a.steps, a.d, a.speakers, seed=0)
xd = torch.from_numpy(x).to(eng.device)
host_rows = [x[i] for i in range(a.steps)]
device_rows = [xd[i] for i in range(a.steps)]
warm = min(a.steps, a.U1 + 20)
run_stream(host_rows[:warm])                       # module loads, first allocations
run_stream(device_rows[:warm])
one_block = dev.nn_chain_entry


def cooperative_only(linkage, n):
  """The kernel choice before sc_nn_chain_small: the cooperative grid at every n."""
  return one_block(linkage, 1 << 30)


for r in range(a.repeats):
  t_host, l_host = run_stream(host_rows)
  t_dev, l_dev = run_stream(device_rows)
  dev.nn_chain_entry = cooperative_only
  try:
    t_grid, l_grid = run_stream(host_rows)
  finally:
    dev.nn_chain_entry = one_block
  for name, t_ms, labels in (("host ndarray", t_host, l_host), ("CUDA tensor", t_dev, l_dev),
                             ("host ndarray, cooperative NN-chain only", t_grid, l_grid)):
    emit({"stream": name, "repeat": r, "steps": a.steps, "d": a.d, "phases": phases(t_ms),
          "total_s": round(float(t_ms.sum()) / 1e3, 3),
          "labels_equal_host": bool(np.array_equal(labels, l_host))})

KERNELS = [("sc_nn_chain_small", "complete", nat.LINKAGE_COMPLETE),
           ("sc_complete_linkage", "complete", nat.LINKAGE_COMPLETE),
           ("sc_nn_chain_small", "average", nat.LINKAGE_AVERAGE),
           ("sc_average_linkage", "average", nat.LINKAGE_AVERAGE)]
for n in [int(s) for s in a.kernel_sizes.split(",")]:
  dist0, flag = eng.cosine_distances(
      torch.from_numpy(synthetic.speaker_turn_dvectors(n, a.d, 8, seed=n)).to(eng.device))
  assert int(flag.item()) == 0
  results = {}
  for entry, method, linkage in KERNELS:
    if entry == "sc_nn_chain_small" and n > nat.NN_SMALL_MAX:
      emit({"kernel": entry, "linkage": method, "n": n, "per_call_ms": "refused (n > NN_SMALL_MAX)"})
      continue
    times = []
    for rep in range(a.reps + 2):                  # two untimed warm-up calls
      dist = dist0.clone()
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      out = eng.nn_chain(entry, dist, n, linkage)
      if rep >= 2:
        times.append(1e3 * (time.perf_counter() - t0))
    results[(entry, method)] = out
    emit({"kernel": entry, "linkage": method, "n": n,
          "per_call_ms": {"median": round(float(np.median(times)), 4),
                          "min": round(float(np.min(times)), 4),
                          "max": round(float(np.max(times)), 4)}})
  for method, grid in (("complete", "sc_complete_linkage"), ("average", "sc_average_linkage")):
    if ("sc_nn_chain_small", method) in results:
      same = all(np.array_equal(p, q) for p, q in zip(results[("sc_nn_chain_small", method)],
                                                      results[(grid, method)]))
      emit({"n": n, "linkage": method, "same_merges": same})
emit({"card_after": query("clocks.sm,temperature.gpu,power.draw,clocks_event_reasons.sw_power_cap")})
