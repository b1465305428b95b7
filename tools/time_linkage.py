#!/usr/bin/env python
"""Times the complete-linkage cosine pre-clustering on the device (CUDA events per kernel entry),
the max_spectral_size predict() that uses it, scikit-learn on this host for comparison, and the
per-step latency of a MultiStageClusterer stream with the device and the scikit-learn pre-clusterer.

    python tools/time_linkage.py [--sizes 8192,16384,32768,65536] [--sklearn-max 16384]
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
from spectralcluster_b200 import multi_stage_clusterer as ms
from spectralcluster_b200 import synthetic

PEAK_FP64_TFLOPS, PEAK_HBM_TBS = 67.0, 3.35      # H100 SXM data sheet (700 W)

ap = argparse.ArgumentParser()
ap.add_argument("--sizes", default="8192,16384,32768,65536")
ap.add_argument("--d", type=int, default=256)
ap.add_argument("--sklearn-max", type=int, default=16384)
ap.add_argument("--predict-n", type=int, default=65536)
ap.add_argument("--stream-steps", type=int, default=700)
a = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                       "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card: %s" % card.splitlines()[torch.cuda.current_device()] if card else torch.cuda.get_device_name())

eng = dev.Engine.get()


def timed(fn):
  st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  st.record()
  out = fn()
  en.record()
  torch.cuda.synchronize()
  return out, st.elapsed_time(en)


warm = torch.from_numpy(synthetic.speaker_turn_dvectors(1024, a.d, 8, seed=0)).to(eng.device)
eng.complete_linkage(eng.cosine_distances(warm)[0], 1024)
for n in [int(s) for s in a.sizes.split(",")]:
  x = synthetic.speaker_turn_dvectors(n, a.d, 8, seed=n)
  xd = torch.from_numpy(x).to(eng.device)
  dist_ms = []
  for _ in range(3):
    (dist, _), t_ms = timed(lambda: eng.cosine_distances(xd))
    dist_ms.append(t_ms)
    if len(dist_ms) < 3:
      del dist
  t_dist = min(dist_ms)
  (xy, md, sz), t_link = timed(lambda: eng.complete_linkage(dist, n))
  del dist
  flops = 2.0 * a.d * n * (n + 1) / 2            # upper triangle, one FMA per element and k
  bytes_ = 8.0 * n * n + x.nbytes                # full matrix stored once, input read once
  print("N=%6d d=%d  distances %8.2f ms  %5.1f TFLOP/s (%4.1f %% of %g)  %5.2f TB/s (%4.1f %% of %g)"
        "  linkage %9.1f ms  (%.2f us per merge)" % (
            n, a.d, t_dist, flops / t_dist / 1e9, 100 * flops / t_dist / 1e9 / PEAK_FP64_TFLOPS,
            PEAK_FP64_TFLOPS, bytes_ / t_dist / 1e9, 100 * bytes_ / t_dist / 1e9 / PEAK_HBM_TBS,
            PEAK_HBM_TBS, t_link, 1e3 * t_link / (n - 1)))
  if n <= a.sklearn_max:
    from sklearn.cluster import AgglomerativeClustering
    t0 = time.perf_counter()
    AgglomerativeClustering(n_clusters=1024, metric="cosine", linkage="complete").fit_predict(x)
    print("N=%6d scikit-learn fit_predict on this host: %.2f s (%d CPUs)" % (
        n, time.perf_counter() - t0, os.cpu_count()))
  del xd

if a.predict_n:
  x = synthetic.speaker_turn_dvectors(a.predict_n, a.d, 8, seed=1)
  c = scb.SpectralClusterer(min_clusters=2, max_clusters=7, max_spectral_size=1024,
                            refinement_options=scb.configs.icassp2018_refinement_options)
  c.predict(x[:4096])
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  c.predict(x)
  torch.cuda.synchronize()
  print("predict(max_spectral_size=1024) N=%d d=%d: %.2f s wall" % (
      a.predict_n, a.d, time.perf_counter() - t0))

if a.stream_steps:
  from sklearn.cluster import AgglomerativeClustering
  x = synthetic.speaker_turn_dvectors(a.stream_steps, 128, 4, seed=9)

  def stream(sklearn_pre):
    main = scb.SpectralClusterer(
        min_clusters=1, max_clusters=5,
        refinement_options=scb.RefinementOptions(
            gaussian_blur_sigma=0, p_percentile=0.9,
            refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)))
    s = ms.MultiStageClusterer(main, fallback_threshold=0.5, L=50, U1=100, U2=600,
                               deflicker=ms.Deflicker.Hungarian)
    if sklearn_pre:
      s.pre = AgglomerativeClustering(n_clusters=100, metric="cosine", linkage="complete")
    steps = []
    for i in range(len(x)):
      t0 = time.perf_counter()
      s.streaming_predict(x[i])
      steps.append(time.perf_counter() - t0)
    return np.array(steps[100:]) * 1e3         # the steps that run the pre-clusterer

  for label, flag in (("device", False), ("scikit-learn", True), ("device", False),
                      ("scikit-learn", True)):
    s = stream(flag)
    print("stream of %d (L=50 U1=100 U2=600), steps past U1, %-12s pre-clusterer: median %.2f ms"
          "  mean %.2f ms  at cache 500..600: median %.2f ms" % (
              a.stream_steps, label, np.median(s), s.mean(), np.median(s[400:500])))
