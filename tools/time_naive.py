#!/usr/bin/env python
"""Times the naive online clusterer: the device launch (`sc_naive_cluster`, CUDA events) against the
host NaiveClusterer loop on the same embeddings, alternating, for thresholds that give one cluster,
about ten and thousands (speaker_turn_dvectors, 8 speakers); the stop-at-the-second-cluster run the
single-cluster check makes; and predict(min_clusters=1) with the FallbackClusterer / Naive check
against predict(min_clusters=2).

    python tools/time_naive.py [--sizes 8192,65536] [--thresholds=-0.5,0.5,0.87]
"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import naive_clusterer as nc
from spectralcluster_b200 import synthetic

ap = argparse.ArgumentParser()
ap.add_argument("--sizes", default="8192,65536")
ap.add_argument("--d", type=int, default=256)
ap.add_argument("--thresholds", default="-0.5,0.5,0.87")
ap.add_argument("--predict-n", type=int, default=65536)
a = ap.parse_args()


def query(fields):
  out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  return out.splitlines()[torch.cuda.current_device()] if out else "nvidia-smi unavailable"


def clocks(when):
  """SM clock, temperature and active clock-limiting reasons (a throttled card is slower)."""
  print("clocks %s (sm MHz, C, W, sw power cap, sw thermal, hw slowdown): %s" % (
      when, query("clocks.sm,temperature.gpu,power.draw,clocks_event_reasons.sw_power_cap,"
                  "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.hw_slowdown")),
      flush=True)


print("card: %s (%s)" % (query("name,power.limit,clocks.max.sm"), torch.cuda.get_device_name()))
clocks("at start")
eng = dev.Engine.get()


def timed(fn):
  st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  st.record()
  out = fn()
  en.record()
  torch.cuda.synchronize()
  return out, st.elapsed_time(en)


warm = torch.from_numpy(synthetic.speaker_turn_dvectors(512, a.d, 8, seed=0)).to(eng.device)
eng.naive_cluster(warm, 0.5, 0.5)
eng.naive_cluster(warm, 0.5, 0.5, stop_at=2)
for n in [int(s) for s in a.sizes.split(",")]:
  x = synthetic.speaker_turn_dvectors(n, a.d, 8, seed=n)
  xd = torch.from_numpy(x).to(eng.device)
  for thr in [float(s) for s in a.thresholds.split(",")]:
    dev_ms = []
    for turn in ("device", "host", "device"):
      if turn == "device":
        (labels, _, k, _, _), t_ms = timed(lambda: eng.naive_cluster(xd, thr, thr))
        dev_ms.append(t_ms)
      else:
        t0 = time.perf_counter()
        want = nc.NaiveClusterer(thr).predict(x)
        host_s = time.perf_counter() - t0
        assert np.array_equal(want, labels.cpu().numpy())
    (_, processed, k2, _, _), stop_ms = timed(lambda: eng.naive_cluster(xd, thr, thr, stop_at=2))
    print("N=%6d d=%d t=%5.2f  %5d clusters  device %9.2f / %9.2f ms (%.2f us per embedding)  "
          "host loop %.3f s (%d CPUs)  stop at 2: %d embeddings, %.3f ms" % (
              n, a.d, thr, k, dev_ms[0], dev_ms[1], 1e3 * min(dev_ms) / n, host_s, os.cpu_count(),
              processed, stop_ms), flush=True)
  clocks("after N=%d" % n)
  del xd

if a.predict_n:
  x = synthetic.speaker_turn_dvectors(a.predict_n, a.d, 8, seed=1)
  opts = scb.FallbackOptions(single_cluster_condition=scb.SingleClusterCondition.FallbackClusterer,
                             fallback_clusterer_type=scb.FallbackClustererType.Naive)
  for mc in (1, 2, 1, 2):
    c = scb.SpectralClusterer(min_clusters=mc, max_clusters=7,
                              refinement_options=scb.configs.icassp2018_refinement_options,
                              fallback_options=opts)
    c.predict(x[:2048])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    labels = c.predict(x)
    torch.cuda.synchronize()
    print("predict(min_clusters=%d%s) N=%d d=%d: %.3f s wall, %d clusters%s" % (
        mc, ", FallbackClusterer/Naive" if mc == 1 else "", a.predict_n, a.d,
        time.perf_counter() - t0, len(np.unique(labels)),
        "  check: %s" % c.last_details.get("single_cluster") if mc == 1 else ""), flush=True)
clocks("at end")
