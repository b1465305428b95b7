#!/usr/bin/env python
"""Times predict() on the windowed eigensolve (max_clusters=None and max_clusters >= 32 above the
dense solver's N) with CUDA events: the whole call, and the device time of its eigensolver entry
points (collect_timings).  Cases alternate within the run; the card name and power limit are
read in the same run.

    python tools/time_eigen_windows.py [--n 65536] [--reps 2] [--out eigen_windows.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import synthetic

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=65536)
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--out", default=None)
a = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                       "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
card = card.splitlines()[torch.cuda.current_device()] if card else torch.cuda.get_device_name()
print("card: %s" % card)

GC = scb.LaplacianType.GraphCut
EIGEN_ENTRIES = ("sc_eigh_extremal_locked", "sc_eigh_extremal", "sc_eigh_mapback", "sc_eigh_dense",
                 "sc_krylov_matvec", "sc_krylov_orthogonalize")


def icassp():
  return scb.RefinementOptions(refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))


CASES = [
    ("icassp_graphcut_max_none", dict(refinement_options=icassp(), laplacian_type=GC)),
    ("icassp_graphcut_max_10", dict(max_clusters=10, refinement_options=icassp(), laplacian_type=GC)),
    ("icassp_nolaplacian_max_none", dict(refinement_options=icassp())),
    ("icassp_graphcut_max_64", dict(max_clusters=64, refinement_options=icassp(), laplacian_type=GC)),
    ("default_clusterer", dict()),
]

x = synthetic.speaker_turn_dvectors(a.n, 256, 6, seed=0)
warm = synthetic.speaker_turn_dvectors(4096, 256, 6, seed=1)
scb.SpectralClusterer(max_clusters=10, refinement_options=icassp(), laplacian_type=GC).predict(warm)
records = []
for rep in range(a.reps):
  for name, kw in CASES:
    c = scb.SpectralClusterer(**kw)
    c.collect_timings = True
    torch.cuda.synchronize()
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.record()
    labels = c.predict(x)
    en.record()
    en.synchronize()
    eig_ms = sum(v for k, v in c.last_timings.items() if k in EIGEN_ENTRIES)
    stats = c.last_details.get("lanczos_stats")
    rec = dict(case=name, n=a.n, rep=rep, card=card, predict_ms=round(st.elapsed_time(en), 1),
               eigensolver_ms=round(eig_ms, 1), solver=c.last_details["solver"],
               values=len(c.last_details["eigenvalues"]), k=int(c.last_details["n_clusters"]),
               clusters_found=int(len(np.unique(labels))),
               stats=stats if isinstance(stats, dict) else (list(map(int, stats)) if stats is not None else None))
    print(json.dumps(rec), flush=True)
    records.append(rec)
    del c, labels
    torch.cuda.empty_cache()
if a.out:
  os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
  with open(a.out, "w") as f:
    for rec in records:
      f.write(json.dumps(rec) + "\n")
