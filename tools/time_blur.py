#!/usr/bin/env python
"""Times the refinement pair (CUDA events, L2 flushed by the matrix size) for one N: the two passes
of the two-pass form (statistics, blur + threshold/symmetrize) and the symmetric pair predict()
runs (upper-tile blur + row maxima, threshold/symmetrize writing the hi plane only, as for a
single-MMA Diffuse), with B stored and with the blur recomputed in pass 2:
python tools/time_blur.py --n 65536"""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from spectralcluster_b200 import device as dev
ap = argparse.ArgumentParser(); ap.add_argument("--n", type=int, default=65536); ap.add_argument("--iters", type=int, default=5)
a = ap.parse_args()
eng = dev.Engine.get(0); n = a.n
A = eng.matrix(n); A.uniform_(0.3, 1.0)
crop = torch.rand(n, device=eng.device, dtype=torch.float32)
res = {}


def timed(name, fn, bytes_per_element):
  for _ in range(2): fn()
  torch.cuda.synchronize()
  s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  s.record()
  for _ in range(a.iters): fn()
  e.record(); torch.cuda.synchronize()
  ms = s.elapsed_time(e) / a.iters
  res[name] = (ms, n * n * bytes_per_element / ms / 1e6)


m = eng.blur_rowmax(A, n, 1.0, crop, False)
timed("stats_4B", lambda: eng.blur_rowmax(A, n, 1.0, crop, False), 4)
timed("thrsym_8B", lambda: eng.blur_threshold_symmetrize(A, n, 1.0, crop, m, 0.95, 0.01, False, False, 0,
                                                         False, True), 8)
# upper pair with B stored: half of A read and half of B written; half of B read and the hi plane
# written
timed("upper_blur_4B", lambda: eng.blur_upper_rowmax(A, n, 1.0, crop, False, store_b=True), 4)
b, mu = eng.blur_upper_rowmax(A, n, 1.0, crop, False, store_b=True)
timed("upper_thrsym_4B", lambda: eng.threshold_symmetrize_upper(b, n, mu, 0.95, 0.01, False, False, 0,
                                                                False, True, want_lo=False), 4)
del b
# upper pair with the blur recomputed: half of A read; half of A read again and the hi plane written
timed("pair_rowmax_2B", lambda: eng.blur_upper_rowmax(A, n, 1.0, crop, False), 2)
rec, mu = eng.blur_upper_rowmax(A, n, 1.0, crop, False)
timed("pair_thrsym_4B", lambda: eng.threshold_symmetrize_upper(rec, n, mu, 0.95, 0.01, False, False, 0,
                                                               False, True, want_lo=False), 4)
print("%s N=%d tiles_per_cta=%s " % (torch.cuda.get_device_name(0), n,
                                     os.environ.get("SCB_BLUR_TILES_PER_CTA", "default")) +
      "  ".join("%s %.2f ms %.0f GB/s" % (k, v[0], v[1]) for k, v in res.items()))
