#!/usr/bin/env python
"""Per-stage device times (CUDA events around each C-ABI call) of predict() at one N, for A/B runs
of kernel variants under environment switches on ONE box (box-to-box clocks differ by ~10 %):

    SCB_GEMM_PACE_KB=16 python tools/time_stages.py --n 65536 --tag pace16
"""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import bench
from spectralcluster_b200 import device as dev, synthetic
from spectralcluster_b200 import spectral_clusterer as sc_mod

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=65536)
ap.add_argument("--steps", type=int, default=4)
ap.add_argument("--tag", default="")
a = ap.parse_args()
eng = dev.Engine.get(0)
x = torch.from_numpy(synthetic.speaker_turn_dvectors(a.n, 256, 6, seed=0).astype(np.float32)).to(eng.device)
c = bench.make_clusterer()


def step():
  aff, crop = eng.affinity(x, want_crop_vector=True)
  v, k, _ = c._compute_eigenvectors_ncluster(sc_mod.DeviceAffinity(aff, a.n, crop, True))
  k = max(k, c.min_clusters)
  return eng.kmeans(v[:, :k].contiguous(), k, 0, c.max_iter)[0]


for _ in range(2):
  step()
torch.cuda.synchronize()
eng.start_profile()
st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
st.record()
for _ in range(a.steps):
  step()
en.record()
stages = eng.stop_profile()
out = {k: round(v / a.steps, 3) for k, v in sorted(stages.items())}
out["step_ms"] = round(st.elapsed_time(en) / a.steps, 2)
print(json.dumps({"tag": a.tag, "n": a.n, **out}))
