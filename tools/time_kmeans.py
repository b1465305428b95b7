#!/usr/bin/env python
"""Times sc_kmeans (Engine.kmeans: seeding, Lloyd step and the custom-distance passes, ending in a
host read) at N = 65,536 with k = k_dim in {8, 64, 256, 512}, on unit rows around k directions
(positive rows for jensenshannon, whose distance is inf on negative entries).  Reports the median
and spread over --repeats calls after a warm-up call, the pass count, and the per-kernel share of
one call from torch.profiler (run separately, after the timed calls).

--host also times the host path the reference takes for that metric (scikit-learn's KMeans
seeding and the scipy cdist loop, oracle.run_kmeans) once per k.  --predict times
predict(custom_dist=metric) against predict(custom_dist="cosine") at --predict-n rows, the two
alternating, --repeats calls each.  Measurement only.

    python tools/time_kmeans.py [--n 65536] [--ks 8,64,256,512] [--repeats 5] [--metric cosine]
                                [--host] [--predict] [--predict-n 65536]
"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from spectralcluster_b200 import custom_distance_kmeans as cdk
from spectralcluster_b200 import device as dev

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=65536)
ap.add_argument("--ks", default="8,64,256,512")
ap.add_argument("--repeats", type=int, default=5)
ap.add_argument("--metric", default="cosine", choices=sorted(cdk._ALIASES))
ap.add_argument("--host", action="store_true")
ap.add_argument("--predict", action="store_true")
ap.add_argument("--predict-n", type=int, default=65536)
a = ap.parse_args()


def query(fields):
  out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  return out.splitlines()[torch.cuda.current_device()] if out else "nvidia-smi unavailable"


def unit_rows(n, k, seed):
  rng = np.random.default_rng(seed)
  cent = rng.standard_normal((k, k))
  e = cent[rng.integers(0, k, n)] / np.sqrt(k) * 3.0 + 0.6 * rng.standard_normal((n, k))
  if a.metric == "jensenshannon":
    return np.abs(e)
  return e / np.linalg.norm(e, axis=1, keepdims=True)


print("card: %s (%s)" % (query("name,power.limit,clocks.max.sm"), torch.cuda.get_device_name()),
      flush=True)
eng = dev.Engine.get()
metric = cdk._METRICS[a.metric]
for k in [int(s) for s in a.ks.split(",")] if a.ks else []:
  host = unit_rows(a.n, k, seed=k)
  e = torch.from_numpy(host).to(eng.device)
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
  if a.host:
    from oracle import spectral_oracle as orc
    t0 = time.perf_counter()
    want = orc.run_kmeans(host, k, a.metric, 300)
    th = time.perf_counter() - t0
    print("  host path (scikit-learn seeding + scipy cdist, %d CPUs): %.1f ms; labels %s"
          % (os.cpu_count(), th * 1e3, "equal" if np.array_equal(want, labels) else "DIFFER"),
          flush=True)
  del e
if a.predict:
  import spectralcluster_b200 as scb
  from oracle import spectral_oracle as orc
  x = orc.synthetic_dvectors(a.predict_n, 256, 6, seed=0)
  opts = scb.RefinementOptions(gaussian_blur_sigma=1, p_percentile=0.95,
                               thresholding_soft_multiplier=0.01,
                               refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))
  runs = {"cosine": [], a.metric: []}
  for rep in range(a.repeats + 1):                        # the first round is a warm-up
    for name in runs:
      c = scb.SpectralClusterer(max_clusters=10, refinement_options=opts, custom_dist=name)
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      c.predict(x)
      if rep:
        runs[name].append(time.perf_counter() - t0)
  for name, ts in runs.items():
    ts = np.array(ts) * 1e3
    print("predict N=%d custom_dist=%s: median %.1f ms (min %.1f, max %.1f, %d calls)"
          % (a.predict_n, name, np.median(ts), ts.min(), ts.max(), len(ts)), flush=True)
print("clocks at end (sm MHz, C, W): %s" % query("clocks.sm,temperature.gpu,power.draw"))
