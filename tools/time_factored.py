"""Time predict() on the factored route (no N x N fp32 matrix) against the stored route.

N = 65,536: both routes, alternating, predict() wall time (host clock around a synchronised call)
and per-stage device time from collect_timings.  Larger N: the factored route alone (the stored
one does not fit an 80 GB card), with peak torch memory and embeddings/s.  Prints the device name
and power limit of the same run.  Usage: python tools/time_factored.py [--reps 3] [--n 98304 131072]
"""

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import spectralcluster_b200 as scb  # noqa: E402
from spectralcluster_b200 import device as dev  # noqa: E402
from oracle import spectral_oracle as orc  # noqa: E402


def device_line():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else torch.cuda.get_device_name(0)
  except (OSError, subprocess.SubprocessError):
    return torch.cuda.get_device_name(0)


def run(c, x, eng, factored):
  saved = eng.factored_above_bytes
  if factored:
    eng.factored_above_bytes = 0
  try:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    labels = c.predict(x)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
  finally:
    eng.factored_above_bytes = saved
  return dict(wall_s=wall, peak_gb=torch.cuda.max_memory_allocated() / 1e9,
              solver=c.last_details["solver"], k=int(c.last_details["n_clusters"]),
              stages_ms={k: round(v, 1) for k, v in sorted(c.last_timings.items(),
                                                            key=lambda kv: -kv[1])[:8]}), labels


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--n", type=int, nargs="*", default=[98304, 131072])
  args = ap.parse_args()
  print("device:", device_line())
  eng = dev.Engine.get()
  c = scb.SpectralClusterer(min_clusters=2, max_clusters=10,
                            refinement_options=scb.configs.icassp2018_refinement_options,
                            custom_dist="cosine")
  c.collect_timings = True
  n = 65536
  x = orc.synthetic_dvectors(n, 256, 6, seed=0).astype(np.float32)
  run(c, x, eng, False)                                  # warm up both routes
  run(c, x, eng, True)
  for rep in range(args.reps):
    for factored in (False, True):
      r, labels = run(c, x, eng, factored)
      r.update(n=n, rep=rep, route="factored" if factored else "stored")
      print(json.dumps(r))
  for n in args.n:
    x = orc.synthetic_dvectors(n, 256, 6, seed=0).astype(np.float32)
    for rep in range(2):
      r, _ = run(c, x, eng, False)
      r.update(n=n, rep=rep, route="auto", embeddings_per_s=round(n / r["wall_s"]))
      print(json.dumps(r))


if __name__ == "__main__":
  main()
