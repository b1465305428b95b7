"""Count the tiles of S = Y Yᵀ the bounded Diffuse computes under the tile-wide rule (row maxima
bounded by the diagonal) and under the hub-first rule (phase 1: every cluster's rows against its
hub, the row of largest diagonal; phase 2: the per-row rule against the maxima phase 1 found).
Tile counts only, no times.

    python tools/count_hub_tiles.py [--sizes 8192 16384]            # CPU, NumPy front end
    python tools/count_hub_tiles.py --gpu [--sizes 32768 65536]     # device front end and order

CPU: Y is the ICASSP front end (crop, blur σ = 1, RowMax p = 0.95, max-symmetrize) of the bench's
speaker-turn generator (d = 256, 6 speakers, seed 0) in NumPy; rows are clustered by the true
speaker label.  The hub rule's phase 2 is also counted with L taken against every cluster's hub
(an upper bound on what pairing clusters with other clusters' hubs could gain).
GPU: Y, the group norms, both row orders and the phase-1 maxima come from the device; the rules
are restated here over them, and the device's own counts are printed beside them.
"""

import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "tests"))

import bounded_diffuse_numpy as bd  # noqa: E402
import hub_bounded_numpy as hb  # noqa: E402
from spectralcluster_b200 import synthetic  # noqa: E402


def numpy_front(n):
  from scipy import ndimage
  x, lab = synthetic.speaker_turn_dvectors(n, 256, 6, seed=0, return_labels=True)
  u = (x / np.linalg.norm(x, axis=1)[:, None]).astype(np.float32)
  a = (u @ u.T + 1.0) / 2.0
  np.fill_diagonal(a, 0.0)
  np.fill_diagonal(a, a.max(axis=1))
  a = ndimage.gaussian_filter(a, sigma=1.0)
  cut = a.max(axis=1)[:, None] * 0.95
  a = np.where(a < cut, a * 0.01, a)
  a = np.maximum(a, a.T)
  return a.astype(np.float16), lab


def shares(n, norms, diag, old_perm, labels, k, sp_of, extra_hubs=False):
  total = len(bd.rasterised_tiles(n))
  old = len(bd.kept_tiles(norms, diag, old_perm))
  perm, starts = hb.hub_order(diag, labels, k)
  sp = sp_of(perm)
  p1 = hb.hub_tiles(starts, n)
  big_l = hb.fold(sp, p1, n)
  pn = norms[perm]
  p2 = hb.phase2_tiles(pn, big_l, p1)
  out = {"n": n, "tiles": total, "old_rule": old / total, "hub_phase1": len(p1) / total,
         "hub_phase2": len(p2) / total, "hub_rule": (len(p1) + len(p2)) / total}
  if extra_hubs:
    hubs = [starts[c] for c in range(k) if starts[c + 1] > starts[c]]
    l_all = np.maximum(big_l, sp[:, hubs].max(axis=1))
    p1_all = {(h // bd.BM, c) for h in hubs for c in range(-(-n // bd.BN))}
    p1_all |= {(m, h // bd.BN) for h in hubs for m in range(-(-n // bd.BM))}
    p1_all = [t for t in bd.rasterised_tiles(n) if t in p1_all]
    out["all_hubs_phase1"] = len(p1_all) / total
    out["all_hubs_phase2"] = len(hb.phase2_tiles(pn, l_all, p1)) / total
  return out


def run_cpu(sizes):
  for n in sizes:
    y16, lab = numpy_front(n)
    norms, diag, _ = bd.row_bounds(y16)
    y32 = y16.astype(np.float32)
    labels = lab.astype(np.int64)
    k = int(labels.max()) + 1
    sp_of = lambda perm: (y32[perm] @ y32[perm].T).astype(np.float64)  # noqa: E731
    print(json.dumps(shares(n, norms, diag, np.argsort(labels, kind="stable"), labels, k, sp_of,
                            extra_hubs=True)), flush=True)


def run_gpu(sizes):
  import torch
  from spectralcluster_b200 import device as dev
  sys.path.insert(0, HERE)
  from time_bounded_diffuse import front
  eng = dev.Engine.get()
  print(json.dumps({"device": torch.cuda.get_device_name(0)}), flush=True)
  for n in sizes:
    hi = front(eng, n)
    norms_d, diag_d, _ = eng.row_group_bounds(hi, n)
    old_perm = eng.bound_order(norms_d)
    _, old_counts = eng.rowmax_tiles(hi, n, norms_d, diag_d, old_perm)
    perm_d, starts_d = eng.bound_order_hubs(norms_d, diag_d)
    mx, counts, big_l_d = eng.hub_rowmax_tiles(hi, n, norms_d, perm_d, starts_d, want_phase1=True)
    norms = norms_d.double().cpu().numpy()
    diag = diag_d.cpu().numpy()
    perm, starts = perm_d.cpu().numpy(), starts_d.cpu().numpy()
    big_l = big_l_d.double().cpu().numpy()[perm]
    total = len(bd.rasterised_tiles(n))
    p1 = hb.hub_tiles(starts, n)
    p2 = hb.phase2_tiles(norms[perm], big_l, p1)
    old = len(bd.kept_tiles(norms, diag, old_perm.cpu().numpy()))
    c1, c2, tot = counts.tolist()
    print(json.dumps({"n": n, "tiles": total, "old_rule": old / total,
                      "old_rule_device": int(old_counts[0]) / total,
                      "hub_phase1": len(p1) / total, "hub_phase2": len(p2) / total,
                      "hub_rule": (len(p1) + len(p2)) / total,
                      "hub_rule_device": (c1 + c2) / tot}), flush=True)
    del hi, mx
    torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--gpu", action="store_true")
  ap.add_argument("--sizes", type=int, nargs="+", default=None)
  args = ap.parse_args()
  if args.gpu:
    run_gpu(args.sizes or [32768, 65536])
  else:
    run_cpu(args.sizes or [8192, 16384])


if __name__ == "__main__":
  main()
