#!/usr/bin/env python
"""Times predict_sharded() on its factored route (owned Y_hi rows, S never stored; forced with
factored_above_bytes = 0) against its stored route at N = 65,536 on one GPU, alternating the two
in the same process.  For each call: the wall time (host clock; every call ends in a device
synchronise), the refinement time to the row statistics (CUDA events), the passes over the
operator, the peak of torch's allocations and whether the labels match the generator's.  The card
name and power limit are read in the same run.

    python tools/time_sharded_factored.py [--n 65536] [--reps 3]
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
from spectralcluster_b200 import sharded


def card_name():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  return out.splitlines()[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def clusterer(name):
  kw = dict(graphcut_10=dict(laplacian_type=scb.LaplacianType.GraphCut, max_clusters=10),
            graphcut_none=dict(laplacian_type=scb.LaplacianType.GraphCut))[name]
  return scb.SpectralClusterer(min_clusters=2, refinement_options=scb.RefinementOptions(
      refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)), **kw)


def release(eng):
  if getattr(eng, "_sharded_backend", None) is not None:
    del eng._sharded_backend
  torch.cuda.synchronize()
  torch.cuda.empty_cache()


def timed_refiners():
  """Record, on every refiner, the device time from its start to its row statistics."""
  for cls in (sharded.ShardedRefiner, sharded.FactoredShardedRefiner):
    def run(self, *a, _inner=cls.run, **kw):
      self.trace = []
      out = _inner(self, *a, **kw)
      torch.cuda.synchronize()
      marks = dict(self.trace)
      end = marks.get("row stats")
      timed_refiners.last_ms = marks["start"].elapsed_time(end) if end is not None else None
      return out
    cls.run = run


def main(n, reps):
  from oracle import spectral_oracle as orc
  eng = dev.Engine.get()
  natural = eng.factored_above_bytes
  x, truth = orc.synthetic_dvectors(n, 256, 6, seed=0, return_labels=True)
  warm = orc.synthetic_dvectors(4096, 256, 6, seed=1)
  timed_refiners()
  for route in ("stored", "factored"):
    eng.factored_above_bytes = 0 if route == "factored" else natural
    sharded.predict_sharded(clusterer("graphcut_10"), warm)
  for rep in range(reps):
    for name in ("graphcut_10", "graphcut_none"):
      for route in ("stored", "factored"):
        eng.factored_above_bytes = 0 if route == "factored" else natural
        release(eng)
        torch.cuda.reset_peak_memory_stats()
        c = clusterer(name)
        t0 = time.perf_counter()
        labels = sharded.predict_sharded(c, x)
        torch.cuda.synchronize()
        seconds = time.perf_counter() - t0
        stats = c.last_details["lanczos_stats"]
        passes = stats["passes"] if isinstance(stats, dict) else int(stats[3])
        print(json.dumps(dict(
            route=route, case=name, n=n, world=1, rep=rep, wall_ms=round(1e3 * seconds, 1),
            refinement_ms=round(timed_refiners.last_ms, 1), solver=c.last_details["solver"],
            passes=passes, k=int(c.last_details["n_clusters"]),
            peak_allocated_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2),
            labels_match_truth=bool(np.array_equal(scb.utils.enforce_ordered_labels(labels),
                                                   scb.utils.enforce_ordered_labels(truth))))),
              flush=True)
  eng.factored_above_bytes = natural
  release(eng)


if __name__ == "__main__":
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=65536)
  ap.add_argument("--reps", type=int, default=3)
  a = ap.parse_args()
  print("card: %s; GPUs: %d" % (card_name(), torch.cuda.device_count()), flush=True)
  main(a.n, a.reps)
