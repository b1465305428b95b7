#!/usr/bin/env python
"""VERDICT r01 item 4: how many fp16 MMAs per product does Diffuse need?

For split3 (hi*hi + hi*lo + lo*hi), split2 ((hi+lo)*hi) and single (hi*hi):
  * N=2,400, configs[1] (ICASSP, no Laplacian) and configs[2] (GraphCut), seeds 0-4, against the
    float64 oracle: max relative eigenvalue error over the values the eigengap reads, labels equal?
  * N=16,384, seeds 0-1: element-wise error of 512 sampled rows of S against the float64 product
    (fraction of elements beyond 3e-6, max), eigenvalues against split3, labels against truth.
Writes a markdown table to stdout."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import spectralcluster_b200 as scb                    # noqa: E402
from spectralcluster_b200 import _native as nat       # noqa: E402
from spectralcluster_b200 import device as dev        # noqa: E402
from oracle import spectral_oracle as orc             # noqa: E402

MODES = [("split3", nat.GEMM_SPLIT3), ("split2", nat.GEMM_SPLIT2), ("single", nat.GEMM_SINGLE)]


def options():
  return scb.RefinementOptions(gaussian_blur_sigma=1, p_percentile=0.95,
                               thresholding_soft_multiplier=0.01,
                               refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))


def clusterer(cfg):
  if cfg == 2:
    return scb.SpectralClusterer(min_clusters=2, max_clusters=7, refinement_options=options())
  return scb.SpectralClusterer(min_clusters=2, max_clusters=10, refinement_options=options(),
                               laplacian_type=scb.LaplacianType.GraphCut)


def oracle_opts(cfg):
  if cfg == 2:
    return orc.options(min_clusters=2, max_clusters=7, sequence=orc.ICASSP2018)
  return orc.options(min_clusters=2, max_clusters=10, sequence=orc.ICASSP2018, laplacian="graphcut")


def relerr(w, ref):
  """Error in units of the parity tolerance |dw| <= 1e-5 |w| + 1e-6 max|w| (<= 1 passes)."""
  return float(np.max(np.abs(w - ref) / (1e-5 * np.abs(ref) + 1e-6 * np.abs(ref).max())))


def main():
  eng = dev.Engine.get()
  t = dev.torch()
  print("# Diffuse: MMAs per product vs parity (tests/diffuse_precision_study.py)\n")
  print("## N=2,400 against the float64 oracle (eigenvalue error in units of the parity tolerance: max |dw| / (1e-5 |w| + 1e-6 max|w|); <= 1 passes)\n")
  print("| config | seed | " + " | ".join("%s eig err / labels" % m for m, _ in MODES) + " |")
  print("|---|---|" + "---|" * len(MODES))
  worst = {m: 0.0 for m, _ in MODES}
  label_fail = {m: 0 for m, _ in MODES}
  for cfg, speakers in ((2, 4), (3, 6)):
    for seed in range(5):
      x = orc.synthetic_dvectors(2400, 256, speakers, seed=seed)
      want, det = orc.predict(x, oracle_opts(cfg), return_details=True)
      nv = 8 if cfg == 2 else 11
      cells = []
      for name, mode in MODES:
        eng.diffuse_precision = mode
        c = clusterer(cfg)
        got = c.predict(x)
        e = relerr(c.last_details["eigenvalues"][:nv], np.real(det["eigenvalues"][:nv]))
        same = bool(np.array_equal(scb.utils.enforce_ordered_labels(got), orc.ordered(want)))
        worst[name] = max(worst[name], e)
        label_fail[name] += 0 if same else 1
        cells.append("%.2e / %s" % (e, "same" if same else "DIFFER"))
      print("| %d | %d | %s |" % (cfg, seed, " | ".join(cells)))
  print("\nworst eigenvalue error: " + ", ".join("%s %.2e" % (m, worst[m]) for m, _ in MODES))
  print("label mismatches: " + ", ".join("%s %d" % (m, label_fail[m]) for m, _ in MODES))

  print("\n## N=16,384: 512 sampled rows of S against the float64 product; eigenvalues against split3 (tolerance units)\n")
  print("| config | seed | mode | max rel err | frac > 3e-6 | eig err vs split3 | labels == truth | Diffuse ms |")
  print("|---|---|---|---|---|---|---|---|")
  n = 16384
  for cfg, speakers in ((2, 4), (3, 6)):
    for seed in range(2):
      x, truth = orc.synthetic_dvectors(n, 256, speakers, seed=seed, return_labels=True)
      xd = t.from_numpy(x.astype(np.float32)).to(eng.device)
      a, crop = eng.affinity(xd, want_crop_vector=True)
      pre = scb.RefinementOptions(**{**options().__dict__, "refinement_sequence":
                                     list(scb.ICASSP2018_REFINEMENT_SEQUENCE[:4])})
      y = dev.run_refinement(eng, a, n, pre, crop_vector=crop).s
      hi, lo = eng.split_planes(y, n)
      rows = t.from_numpy(np.sort(np.random.default_rng(seed).choice(n, 512, replace=False))).to(eng.device)
      want = y[rows, :n].double() @ y[:n, :n].double().T
      base = None
      for name, mode in MODES:
        st, en = t.cuda.Event(enable_timing=True), t.cuda.Event(enable_timing=True)
        eng.diffuse(n, hi=hi, lo=lo, precision=mode)     # warm
        st.record()
        s, _, _ = eng.diffuse(n, hi=hi, lo=lo, precision=mode)
        en.record()
        t.cuda.synchronize()
        rel = ((s[rows, :n].double() - want).abs() / want.abs().clamp_min(1e-300))
        eng.diffuse_precision = mode
        c = clusterer(cfg)
        got = c.predict(x)
        w = c.last_details["eigenvalues"]
        base = w if base is None else base
        same = bool(np.array_equal(scb.utils.enforce_ordered_labels(got), orc.ordered(truth)))
        print("| %d | %d | %s | %.2e | %.2e | %.2e | %s | %.2f |" % (
            cfg, seed, name, rel.max().item(), (rel > 3e-6).double().mean().item(),
            relerr(w, base), same, st.elapsed_time(en)))
        del s
      del y, hi, lo, want, a


if __name__ == "__main__":
  main()
