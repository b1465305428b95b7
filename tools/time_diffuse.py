#!/usr/bin/env python
"""Times sc_diffuse (wgmma GEMM, Y Y^T) for one N with CUDA events."""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from spectralcluster_b200 import device as dev
ap = argparse.ArgumentParser(); ap.add_argument("--n", type=int, default=65536); ap.add_argument("--iters", type=int, default=3); ap.add_argument("--precision", default="single", choices=["split3", "split2", "single"])
a = ap.parse_args()
from spectralcluster_b200 import _native as nat
eng = dev.Engine.get(0); n = a.n
prec = {"split3": nat.GEMM_SPLIT3, "split2": nat.GEMM_SPLIT2, "single": nat.GEMM_SINGLE}[a.precision]
y = eng.matrix(n); y.uniform_(0.0, 1.0)
hi, lo = eng.split_planes(y, n); del y
for _ in range(1): s = eng.diffuse(n, hi=hi, lo=lo, precision=prec)[0]; del s
torch.cuda.synchronize()
st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
st.record()
for _ in range(a.iters): s = eng.diffuse(n, hi=hi, lo=lo, precision=prec)[0]; del s
en.record(); torch.cuda.synchronize()
ms = st.elapsed_time(en) / a.iters
print("N=%d %s pacing=%s diffuse %.1f ms  %.0f TFLOP/s algorithmic (2N^3)" % (
    n, a.precision, "off" if os.environ.get("SCB_NO_GEMM_PACING") else "on", ms, 2.0 * n ** 3 / ms / 1e9))
