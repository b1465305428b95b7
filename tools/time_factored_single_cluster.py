#!/usr/bin/env python
"""Times the AffinityGmmBic single-cluster check of predict(min_clusters=1) on the factored route
(affinity row panels packed into the upper band, then the GMM passes over the packed band) against
the stored route's check at N = 65,536 (the factored route forced by
Engine.factored_above_bytes = 0), alternating, then on the factored route unforced at N = 98,304
and 131,072, where the stored route does not fit.  For each call: the check's wall time, split
into the panel sweep + pack and the passes, the pass count, predict(min_clusters=1) against
predict(min_clusters=2) on the same route, and the peak torch allocation of each.  Wall times are
host clocks around work that ends in a device synchronise.  The card name and power limit are read
in the same run.

    python tools/time_factored_single_cluster.py [--n 65536] [--large 98304 131072] [--reps 2]
"""
import argparse
import json
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
from spectralcluster_b200 import fallback_clusterer
from spectralcluster_b200 import synthetic

TIMES = {}


def card_name():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  return out.splitlines()[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def timed(owner, name, key):
  """Wrap owner.name so that each call adds its synchronised wall time to TIMES[key]."""
  inner = getattr(owner, name)

  def wrapper(*args, **kw):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    try:
      return inner(*args, **kw)
    finally:
      torch.cuda.synchronize()
      TIMES[key] = TIMES.get(key, 0.0) + time.perf_counter() - t0
  setattr(owner, name, wrapper)


def run(eng, x, route, min_clusters, rep):
  c = scb.SpectralClusterer(min_clusters=min_clusters, max_clusters=10,
                            refinement_options=scb.configs.icassp2018_refinement_options,
                            custom_dist="cosine")
  saved = eng.factored_above_bytes
  if route == "factored-forced":
    eng.factored_above_bytes = 0
  TIMES.clear()
  try:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(eng.device)
    np.random.seed(0)
    t0 = time.perf_counter()
    with warnings.catch_warnings():
      warnings.simplefilter("ignore")
      labels = c.predict(x)
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
  finally:
    eng.factored_above_bytes = saved
  rec = dict(route=route, n=len(x), min_clusters=min_clusters, rep=rep,
             predict_ms=round(1e3 * seconds, 1), solver=c.last_details.get("solver"),
             k=int(c.last_details.get("n_clusters", 1)),
             peak_gb=round(torch.cuda.max_memory_allocated(eng.device) / 1e9, 2))
  if min_clusters == 1:
    check = TIMES.get("check", 0.0)
    pack = TIMES.get("pack", 0.0)
    single = c.last_details["single_cluster"]
    rec.update(check_ms=round(1e3 * check, 1), sweep_pack_ms=round(1e3 * pack, 1),
               passes_ms=round(1e3 * (check - pack), 1), passes=single["passes"],
               bic=single["bic"], n_iter=single["n_iter"])
  print(json.dumps(rec), flush=True)
  del c, labels
  torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=65536)
  ap.add_argument("--large", type=int, nargs="*", default=[98304, 131072])
  ap.add_argument("--reps", type=int, default=2)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("time_factored_single_cluster: needs a CUDA device")
  print("card: %s" % card_name(), flush=True)
  timed(fallback_clusterer, "check_single_cluster", "check")
  timed(dev.FactoredAffinity, "upper_band", "pack")
  eng = dev.Engine.get()
  warm = synthetic.speaker_turn_dvectors(20000, 256, 4, seed=1).astype(np.float32)
  for route in ("stored", "factored-forced"):                 # rep -1: warm-up
    for mc in (1, 2):
      run(eng, warm, route, mc, -1)
  x = synthetic.speaker_turn_dvectors(a.n, 256, 4, seed=a.n).astype(np.float32)
  for rep in range(a.reps):
    for route in ("stored", "factored-forced"):
      for mc in (1, 2):
        run(eng, x, route, mc, rep)
  del x
  for n in a.large:
    x = synthetic.speaker_turn_dvectors(n, 256, 4, seed=n).astype(np.float32)
    for mc in (1, 2):
      run(eng, x, "factored", mc, 0)
    del x


if __name__ == "__main__":
  main()
