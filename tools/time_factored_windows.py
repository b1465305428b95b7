#!/usr/bin/env python
"""Times predict()'s windowed solve on the factored operator (max_clusters=None or >= 32) against
the stored windows at N = 65,536 on one GPU (the factored route forced by
Engine.factored_above_bytes = 0), alternating, then the factored route unforced at N = 131,072,
where the stored route does not fit.  For each call: the wall time (host clock; predict() ends in
a device synchronise), the windows, the passes over the operator, the passes spent in the
lambda_max solve, and the peak torch allocation.  The card name and power limit are read in the
same run.

    python tools/time_factored_windows.py [--n 65536] [--large 131072] [--reps 2]
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
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import eigen_windows

CASES = {
    "graphcut_max_none": dict(laplacian_type=scb.LaplacianType.GraphCut),
    "nolaplacian_max_none": dict(),
    "graphcut_max_64": dict(laplacian_type=scb.LaplacianType.GraphCut, max_clusters=64),
}


def card_name():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  return out.splitlines()[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def count_lambda_max_passes():
  """Record, in each DeviceOps' stats, the passes over the operator its lambda_max() solve took."""
  inner = eigen_windows.DeviceOps.lambda_max

  def lambda_max(self):
    before = self.stats["passes"]
    value = inner(self)
    self.stats["lambda_max_passes"] = self.stats["passes"] - before
    return value
  eigen_windows.DeviceOps.lambda_max = lambda_max


def clusterer(name):
  kw = dict(max_clusters=None)
  kw.update(CASES[name])
  return scb.SpectralClusterer(min_clusters=2,
                               refinement_options=scb.configs.icassp2018_refinement_options,
                               custom_dist="cosine", **kw)


def run(eng, name, x, truth, route, rep):
  c = clusterer(name)
  saved = eng.factored_above_bytes
  if route == "factored-forced":
    eng.factored_above_bytes = 0
  try:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(eng.device)
    t0 = time.perf_counter()
    labels = c.predict(x)
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
  finally:
    eng.factored_above_bytes = saved
  stats = c.last_details["lanczos_stats"]
  rec = dict(route=route, case=name, n=len(x), rep=rep, wall_ms=round(1e3 * seconds, 1),
             solver=c.last_details["solver"], values=len(c.last_details["eigenvalues"]),
             k=int(c.last_details["n_clusters"]), windows=stats["windows"],
             passes=stats["passes"], lambda_max_passes=stats.get("lambda_max_passes", 0),
             peak_gb=round(torch.cuda.max_memory_allocated(eng.device) / 1e9, 2),
             labels_match_truth=bool(np.array_equal(scb.utils.enforce_ordered_labels(labels),
                                                    scb.utils.enforce_ordered_labels(truth))))
  print(json.dumps(rec), flush=True)
  del c, labels
  torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=65536)
  ap.add_argument("--large", type=int, default=131072)
  ap.add_argument("--reps", type=int, default=2)
  a = ap.parse_args()
  from oracle import spectral_oracle as orc
  print("card: %s" % card_name(), flush=True)
  count_lambda_max_passes()
  eng = dev.Engine.get()
  warm, warm_truth = orc.synthetic_dvectors(40000, 256, 6, seed=1, return_labels=True)
  for route in ("stored", "factored-forced"):               # rep -1: warm-up
    run(eng, "graphcut_max_none", warm.astype(np.float32), warm_truth, route, -1)
  x, truth = orc.synthetic_dvectors(a.n, 256, 6, seed=0, return_labels=True)
  x = x.astype(np.float32)
  for rep in range(a.reps):
    for name in CASES:
      for route in ("stored", "factored-forced"):
        run(eng, name, x, truth, route, rep)
  del x
  x, truth = orc.synthetic_dvectors(a.large, 256, 6, seed=0, return_labels=True)
  x = x.astype(np.float32)
  for name in CASES:
    run(eng, name, x, truth, "factored", 0)


if __name__ == "__main__":
  main()
