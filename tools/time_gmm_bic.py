#!/usr/bin/env python
"""Times the device AffinityGmmBic single-cluster check (CUDA events per pass type, a host clock
around the synchronised call), reports the bytes each pass reads and the number of passes,
compares predict(min_clusters=1) with predict(min_clusters=2), and times scikit-learn on this
host up to --sklearn-max.

    python tools/time_gmm_bic.py [--sizes 8192,16384,65536] [--predict-n 65536] [--sklearn-max 4096]
"""
import argparse
import os
import subprocess
import sys
import time
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import gmm_bic as gb
from spectralcluster_b200 import synthetic

PEAK_HBM_TBS = 3.35      # H100 SXM data sheet (700 W)
MODE_NAMES = {gb.MOMENTS: "moments", gb.KPP: "kmeans++", gb.LOOKUP: "lookup", gb.LLOYD: "lloyd",
              gb.LABELS: "labels", gb.EM: "em", gb.SCORE: "score"}

ap = argparse.ArgumentParser()
ap.add_argument("--sizes", default="8192,16384,65536")
ap.add_argument("--d", type=int, default=256)
ap.add_argument("--speakers", type=int, default=4)
ap.add_argument("--offset", type=int, default=1)
ap.add_argument("--predict-n", type=int, default=65536)
ap.add_argument("--sklearn-max", type=int, default=4096)
a = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                       "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card: %s" % card.splitlines()[torch.cuda.current_device()] if card else torch.cuda.get_device_name())
eng = dev.Engine.get()


class TimedOps(gb.DeviceOps):
  """DeviceOps that brackets every pass with CUDA events, per mode."""

  def __init__(self, *args):
    super().__init__(*args)
    self.times = {}

  def _pass(self, mode, *params):
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.record()
    out = super()._pass(mode, *params)       # synchronous: the entry copies its result back
    en.record()
    en.synchronize()
    self.times.setdefault(mode, []).append(st.elapsed_time(en))
    return out


def affinity(n, seed):
  x = torch.from_numpy(synthetic.speaker_turn_dvectors(n, a.d, a.speakers, seed=seed))
  return eng.affinity(x.to(eng.device), want_crop_vector=False)[0]


warm = affinity(1024, 0)
np.random.seed(0)
gb.gmm_bic(gb.DeviceOps(eng, warm, 1024, a.offset))
for n in [int(s) for s in a.sizes.split(",")]:
  mat = affinity(n, n)
  m = gb.band_size(n, a.offset)
  for rep in range(2):
    ops = TimedOps(eng, mat, n, a.offset)
    np.random.seed(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with warnings.catch_warnings():
      warnings.simplefilter("ignore")
      res = gb.gmm_bic(ops)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
  band_bytes = 4.0 * m
  print("N=%6d offset=%d m=%d: check %.1f ms wall, %d passes, single=%s, bic=%s, EM iterations "
        "%s; %.2f GB read per streaming pass (%.2f ms at %.2f TB/s)" % (
            n, a.offset, m, 1e3 * wall, res.passes, res.single,
            ["%.6e" % b for b in res.bic], res.n_iter, band_bytes / 1e9,
            1e3 * band_bytes / PEAK_HBM_TBS / 1e12, PEAK_HBM_TBS))
  for mode, ts in sorted(ops.times.items()):
    med = float(np.median(ts))
    line = "    %-9s x%3d  median %8.3f ms  total %8.1f ms" % (MODE_NAMES[mode], len(ts), med,
                                                                sum(ts))
    if mode != gb.LOOKUP:
      line += "  %.2f TB/s (%.0f %% of %.2f)" % (band_bytes / med / 1e9,
                                                   100 * band_bytes / med / 1e9 / PEAK_HBM_TBS,
                                                   PEAK_HBM_TBS)
    print(line)
  del mat

if a.predict_n:
  x = synthetic.speaker_turn_dvectors(a.predict_n, a.d, a.speakers, seed=1)
  opts = scb.configs.icassp2018_refinement_options
  for mc in (1, 2, 1, 2):
    c = scb.SpectralClusterer(min_clusters=mc, max_clusters=7, refinement_options=opts)
    c.predict(x[:2048])
    torch.cuda.synchronize()
    np.random.seed(0)
    t0 = time.perf_counter()
    labels = c.predict(x)
    torch.cuda.synchronize()
    print("predict(min_clusters=%d) N=%d d=%d: %.3f s wall, %d clusters%s" % (
        mc, a.predict_n, a.d, time.perf_counter() - t0, len(np.unique(labels)),
        ", check: %s" % c.last_details.get("single_cluster") if mc == 1 else ""))

for n in (1024, 2048, 4096, 8192):
  if n > a.sklearn_max:
    break
  from sklearn.mixture import GaussianMixture
  mat = affinity(n, n)
  values = eng.download_matrix(mat, n)[np.triu_indices(n, a.offset)][:, None]
  np.random.seed(0)
  t0 = time.perf_counter()
  bic = [GaussianMixture(n_components=c).fit(values).bic(values) for c in (1, 2)]
  print("N=%6d scikit-learn on this host (%d CPUs): %.2f s, bic=%s" % (
      n, os.cpu_count(), time.perf_counter() - t0, ["%.6e" % b for b in bic]))
