"""Time the bounded Diffuse against the storing one, alternating in one process.

    python tools/time_bounded_diffuse.py [--sizes 16384 32768 65536] [--reps 3] [--out FILE]

For each N: Y_hi of the ICASSP front end on the bench's speaker-turn generator (seed 0), then per
repetition the old back end (storing sc_diffuse with its epilogue statistics + sc_eigh_extremal on
S) and the new one (row bounds + row sums, row order, gather + tile list + listed GEMM, then
sc_eigh_extremal_factored), and the hub-first route (hub order, phase-1 and phase-2 lists and
GEMMs), each stage bracketed by CUDA events.  Reports per-stage ms, the share of
tiles computed and the TFLOP/s of the computed tiles (128 x 192 x N multiply-adds each), and the
same for an input where nothing can be skipped (identical rows), the worst-case overhead.
"""

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import torch  # noqa: E402

import spectralcluster_b200 as scb  # noqa: E402
from spectralcluster_b200 import _native as nat  # noqa: E402
from spectralcluster_b200 import device as dev  # noqa: E402
from spectralcluster_b200 import laplacian as lap  # noqa: E402
from spectralcluster_b200 import synthetic  # noqa: E402


def timed(stages, name, fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  out = fn()
  b.record()
  torch.cuda.synchronize()
  stages[name] = stages.get(name, 0.0) + a.elapsed_time(b)
  return out


def front(eng, n):
  x = synthetic.speaker_turn_dvectors(n, 256, 6, seed=0).astype(np.float32)
  a, crop = eng.affinity(torch.from_numpy(x).to(eng.device), want_crop_vector=True)
  b, m = eng.blur_upper_rowmax(a, n, 1.0, crop, False)
  del a
  _, hi, _ = eng.threshold_symmetrize_upper(b, n, m, 0.95, 0.01, False, False, nat.SYMMETRIZE_MAX,
                                            False, True, want_lo=False)
  return hi


def old_route(eng, n, hi):
  st = {}
  s, mx, sm = timed(st, "diffuse", lambda: eng.diffuse(n, hi=hi, lo=None, want_stats=True,
                                                       precision=nat.GEMM_SINGLE))
  r = dev.Refined(s, n, True, 1.0 / mx.double(), sm)
  delta, left, right, sign, which = lap.operator_terms(eng, r, scb.LaplacianType.GraphCut)
  timed(st, "eigensolve", lambda: eng.eigh(s, n, delta, left, right, sign, which, 11, 11, False))
  del s
  return st


def new_route(eng, n, hi):
  st = {}
  norms, diag, c = timed(st, "bounds", lambda: eng.row_group_bounds(hi, n))
  rowsum = torch.empty((1, n), dtype=torch.float64, device=eng.device)
  timed(st, "rowsum", lambda: eng.block_product_f16(hi, n, n, c.view(1, -1), 1, rowsum))
  perm = timed(st, "order", lambda: eng.bound_order(norms))
  mx, counts = timed(st, "tiles+gemm", lambda: eng.rowmax_tiles(hi, n, norms, diag, perm))
  r = dev.Refined(None, n, True, 1.0 / mx.double(), rowsum.view(n), y_hi=hi)
  delta, left, right, sign, which = lap.operator_terms(eng, r, scb.LaplacianType.GraphCut)
  timed(st, "eigensolve", lambda: eng.eigh_factored(hi, n, delta, left, right, sign, which, 11, 11))
  computed, total = counts.tolist()
  st["tiles"], st["of"] = computed, total
  return st


def hub_route(eng, n, hi):
  st = {}
  norms, diag, c = timed(st, "bounds", lambda: eng.row_group_bounds(hi, n))
  rowsum = torch.empty((1, n), dtype=torch.float64, device=eng.device)
  timed(st, "rowsum", lambda: eng.block_product_f16(hi, n, n, c.view(1, -1), 1, rowsum))
  perm, starts = timed(st, "order", lambda: eng.bound_order_hubs(norms, diag))
  mx, counts = timed(st, "tiles+gemm", lambda: eng.hub_rowmax_tiles(hi, n, norms, perm, starts))
  r = dev.Refined(None, n, True, 1.0 / mx.double(), rowsum.view(n), y_hi=hi)
  delta, left, right, sign, which = lap.operator_terms(eng, r, scb.LaplacianType.GraphCut)
  timed(st, "eigensolve", lambda: eng.eigh_factored(hi, n, delta, left, right, sign, which, 11, 11))
  p1, p2, total = counts.tolist()
  st["tiles"], st["of"], st["phase1"] = p1 + p2, total, p1
  return st


def summarise(runs):
  keys = [k for k in runs[0] if k not in ("tiles", "of", "phase1")]
  out = {k: float(np.median([r[k] for r in runs])) for k in keys}
  out["total"] = float(np.median([sum(r[k] for k in keys) for r in runs]))
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--sizes", type=int, nargs="+", default=[16384, 32768, 65536])
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  eng = dev.Engine.get()
  prop = torch.cuda.get_device_properties(0)
  report = {"device": prop.name, "sizes": {}}
  for n in args.sizes:
    for kind in ("speaker-turns", "identical-rows"):
      if kind == "speaker-turns":
        hi = front(eng, n)
      else:
        hi = torch.zeros((n, dev.round_up(n, 64)), dtype=torch.float16, device=eng.device)
        hi[:, :n] = 0.125
      old_route(eng, n, hi), new_route(eng, n, hi), hub_route(eng, n, hi)   # warm-up
      olds, news, hubs = [], [], []
      for _ in range(args.reps):
        olds.append(old_route(eng, n, hi))
        news.append(new_route(eng, n, hi))
        hubs.append(hub_route(eng, n, hi))
      entry = {"old_ms": summarise(olds)}
      for name, runs in (("tile_wide", news), ("hub", hubs)):
        ms = summarise(runs)
        computed, total = runs[-1]["tiles"], runs[-1]["of"]
        flop = 2.0 * dev.LIST_BM * dev.LIST_BN * n * computed
        entry[name] = {"ms": ms, "tiles": computed, "of": total, "tile_fraction": computed / total,
                       "computed_tile_TFLOPs": flop / (ms["tiles+gemm"] * 1e-3) / 1e12}
        if name == "hub":
          entry[name]["phase1_tiles"] = runs[-1]["phase1"]
      report["sizes"].setdefault(str(n), {})[kind] = entry
      print(json.dumps({str(n): {kind: report["sizes"][str(n)][kind]}}), flush=True)
      del hi
      torch.cuda.empty_cache()
  if args.out:
    with open(args.out, "w") as f:
      json.dump(report, f, indent=1)


if __name__ == "__main__":
  main()
