#!/usr/bin/env python
"""Times sc_kmeans (Engine.kmeans: seeding, Lloyd step and the custom-distance passes, ending in a
host read) at N = 65,536 with k = k_dim in {8, 64, 256, 512}, on unit rows around k directions.
Reports the median and spread over --repeats calls after a warm-up call, the pass count, and the
per-kernel share of one call from torch.profiler (run separately, after the timed calls).
Measurement only.

    python tools/time_kmeans.py [--n 65536] [--ks 8,64,256,512] [--repeats 5] [--metric cosine]
"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from spectralcluster_b200 import device as dev

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=65536)
ap.add_argument("--ks", default="8,64,256,512")
ap.add_argument("--repeats", type=int, default=5)
ap.add_argument("--metric", default="cosine", choices=["cosine", "euclidean"])
a = ap.parse_args()


def query(fields):
  out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  return out.splitlines()[torch.cuda.current_device()] if out else "nvidia-smi unavailable"


def unit_rows(n, k, seed):
  rng = np.random.default_rng(seed)
  cent = rng.standard_normal((k, k))
  e = cent[rng.integers(0, k, n)] / np.sqrt(k) * 3.0 + 0.6 * rng.standard_normal((n, k))
  return e / np.linalg.norm(e, axis=1, keepdims=True)


print("card: %s (%s)" % (query("name,power.limit,clocks.max.sm"), torch.cuda.get_device_name()),
      flush=True)
eng = dev.Engine.get()
metric = {"cosine": 0, "euclidean": 1}[a.metric]
for k in [int(s) for s in a.ks.split(",")]:
  e = torch.from_numpy(unit_rows(a.n, k, seed=k)).to(eng.device)
  labels, iters = eng.kmeans(e, k, metric, 300)          # warm-up
  times = []
  for _ in range(a.repeats):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    got, it = eng.kmeans(e, k, metric, 300)              # ends in a host read of the labels
    times.append(time.perf_counter() - t0)
    assert it == iters and np.array_equal(got, labels)
  times = np.array(times) * 1e3
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    eng.kmeans(e, k, metric, 300)
    torch.cuda.synchronize()
  per = {}
  for ev in prof.key_averages():
    if ev.device_type == torch.autograd.DeviceType.CUDA:
      per[ev.key] = per.get(ev.key, 0.0) + ev.device_time_total / 1e3
  total = sum(per.values()) or 1.0
  top = sorted(per.items(), key=lambda kv: -kv[1])[:4]
  print("N=%d k=k_dim=%d %s: %d passes, median %.2f ms (min %.2f, max %.2f, %d calls); kernels: %s"
        % (a.n, k, a.metric, iters, np.median(times), times.min(), times.max(), a.repeats,
           ", ".join("%s %.2f ms (%.0f%%)" % (name.split("(")[0], ms, 100 * ms / total)
                     for name, ms in top)), flush=True)
  del e
print("clocks at end (sm MHz, C, W): %s" % query("clocks.sm,temperature.gpu,power.draw"))
