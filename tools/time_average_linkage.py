#!/usr/bin/env python
"""Times the average-linkage cosine clustering behind the FallbackClusterer / Agglomerative
single-cluster check: device distances + NN-chain (CUDA events per kernel entry), scikit-learn on
this host for comparison, predict(min_clusters=1) with that check against predict(min_clusters=2),
and the per-step latency of a MultiStageClusterer stream (whose main clusterer runs the check) with
the check on the device and in scikit-learn.

    python tools/time_average_linkage.py [--sizes 8192,16384,65536] [--sklearn-max 16384]
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
from spectralcluster_b200 import agglomerative as agg
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import multi_stage_clusterer as ms
from spectralcluster_b200 import synthetic

ap = argparse.ArgumentParser()
ap.add_argument("--sizes", default="8192,16384,65536")
ap.add_argument("--d", type=int, default=256)
ap.add_argument("--threshold", type=float, default=0.5)
ap.add_argument("--sklearn-max", type=int, default=16384)
ap.add_argument("--predict-n", type=int, default=65536)
ap.add_argument("--stream-steps", type=int, default=700)
a = ap.parse_args()


def query(fields):
  out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  return out.splitlines()[torch.cuda.current_device()] if out else "nvidia-smi unavailable"


def clocks(when):
  """SM clock, temperature and active clock-limiting reasons (a throttled card is slower)."""
  print("clocks %s (sm MHz, C, W, sw power cap, sw thermal, hw slowdown): %s" % (
      when, query("clocks.sm,temperature.gpu,power.draw,clocks_event_reasons.sw_power_cap,"
                  "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.hw_slowdown")))


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


def sklearn_average():
  from sklearn.cluster import AgglomerativeClustering
  return AgglomerativeClustering(n_clusters=None, metric="cosine", linkage="average",
                                 distance_threshold=a.threshold)


warm = torch.from_numpy(synthetic.speaker_turn_dvectors(1024, a.d, 8, seed=0)).to(eng.device)
eng.average_linkage(eng.cosine_distances(warm)[0], 1024)
for n in [int(s) for s in a.sizes.split(",")]:
  x = synthetic.speaker_turn_dvectors(n, a.d, 8, seed=n)
  xd = torch.from_numpy(x).to(eng.device)
  dist_ms = []
  for _ in range(3):                               # the first call at a size also allocates
    (dist, _), t_ms = timed(lambda: eng.cosine_distances(xd))
    dist_ms.append(t_ms)
    if len(dist_ms) < 3:
      del dist
  t_dist = min(dist_ms)
  (xy, md, _), t_link = timed(lambda: eng.average_linkage(dist, n))
  del dist
  k = np.count_nonzero(md >= a.threshold) + 1
  print("N=%6d d=%d  distances %8.2f ms  average linkage %9.1f ms  (%.2f us per merge)  "
        "%d clusters at t=%g" % (n, a.d, t_dist, t_link, 1e3 * t_link / (n - 1), k, a.threshold))
  clocks("after N=%d" % n)
  if n <= a.sklearn_max:
    t0 = time.perf_counter()
    ref = sklearn_average().fit(x)
    print("N=%6d scikit-learn fit on this host: %.2f s (%d CPUs), %d clusters" % (
        n, time.perf_counter() - t0, os.cpu_count(), ref.n_clusters_))
  del xd


def fallback_agglomerative():
  return scb.FallbackOptions(
      single_cluster_condition=scb.SingleClusterCondition.FallbackClusterer,
      fallback_clusterer_type=scb.FallbackClustererType.Agglomerative,
      agglomerative_threshold=a.threshold)


if a.predict_n:
  x = synthetic.speaker_turn_dvectors(a.predict_n, a.d, 8, seed=1)
  opts = scb.configs.icassp2018_refinement_options
  for mc in (1, 2, 1, 2):
    c = scb.SpectralClusterer(min_clusters=mc, max_clusters=7, refinement_options=opts,
                              fallback_options=fallback_agglomerative())
    c.predict(x[:2048])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    labels = c.predict(x)
    torch.cuda.synchronize()
    print("predict(min_clusters=%d%s) N=%d d=%d: %.3f s wall, %d clusters" % (
        mc, ", FallbackClusterer/Agglomerative" if mc == 1 else "", a.predict_n, a.d,
        time.perf_counter() - t0, len(np.unique(labels))))


def host_fit_predict(self, X):
  """The check as scikit-learn runs it (the embeddings as predict() holds them, on the host)."""
  return self._fit_predict_host(X.cpu().numpy() if torch.is_tensor(X) else np.asarray(X))


if a.stream_steps:
  x = synthetic.speaker_turn_dvectors(a.stream_steps, 128, 4, seed=9)
  device_fit_predict = agg.CosineAverageLinkage.fit_predict

  def stream(host_check):
    agg.CosineAverageLinkage.fit_predict = host_fit_predict if host_check else device_fit_predict
    main = scb.SpectralClusterer(
        min_clusters=1, max_clusters=5,
        refinement_options=scb.RefinementOptions(
            gaussian_blur_sigma=0, p_percentile=0.9,
            refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)))
    s = ms.MultiStageClusterer(main, fallback_threshold=0.5, L=50, U1=100, U2=600,
                               deflicker=ms.Deflicker.Hungarian)
    steps, out = [], None
    for i in range(len(x)):
      t0 = time.perf_counter()
      out = s.streaming_predict(x[i])
      steps.append(time.perf_counter() - t0)
    agg.CosineAverageLinkage.fit_predict = device_fit_predict
    return np.array(steps) * 1e3, out

  results = {}
  for label, flag in (("device", False), ("scikit-learn", True), ("device", False),
                      ("scikit-learn", True)):
    s, out = stream(flag)
    results.setdefault(label, out)
    print("stream of %d (L=50 U1=100 U2=600), check on %-12s: steps 50..100 median %.2f ms, "
          "steps past 100 median %.2f ms, all steps median %.2f ms" % (
              a.stream_steps, label, np.median(s[49:100]), np.median(s[100:]), np.median(s)))
  print("final stream labels equal: %s" % np.array_equal(results["device"], results["scikit-learn"]))
clocks("at end")
