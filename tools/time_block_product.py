"""Time the fp64-tensor-core block product Y = S T on an fp16 matrix (sc_block_product_f16, the
operator of the factored Lanczos route and of the bounded Diffuse's row sums) and, for comparison,
on an fp32 matrix (sc_block_product, the stored route).

    python tools/time_block_product.py [--sizes 65536 131072] [--b 1 4 8 12 16] [--reps 20] [--out FILE]

For each N and block size b: CUDA events around --reps launches after warm-up.  Reports ms per
product, GB/s of matrix bytes (N^2 x 2 or 4 B: each product is one pass over the matrix) and the
executed DMMA TFLOP/s (the kernels issue 8 vectors' worth of fp64 MMA per 4 columns for b <= 8 and
16 above, whatever b is), with the card's name and power limit read in the same run.  The fp32
matrix is skipped where it does not fit beside the fp16 one.
"""

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import torch  # noqa: E402

from spectralcluster_b200 import device as dev  # noqa: E402


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return out.stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    return torch.cuda.get_device_properties(0).name + ", power limit not read"


def time_product(eng, name, s, n, t, b, y, reps):
  def run():
    eng.call(name, dev._ptr(s), n, n, s.stride(0), dev._ptr(t), t.stride(0), b, dev._ptr(y),
             y.stride(0), eng.stream)
  for _ in range(3):
    run()
  a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(reps):
    run()
  e.record()
  torch.cuda.synchronize()
  return a.elapsed_time(e) / reps


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--sizes", type=int, nargs="+", default=[65536, 131072])
  ap.add_argument("--b", type=int, nargs="+", default=[1, 4, 8, 12, 16])
  ap.add_argument("--reps", type=int, default=20)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  eng = dev.Engine.get()
  report = {"card": card(), "rows": []}
  print(report["card"], flush=True)
  g = torch.Generator(device=eng.device).manual_seed(0)
  for n in args.sizes:
    ld = dev.round_up(n, 64)
    s16 = torch.rand((n, ld), dtype=torch.float16, device=eng.device, generator=g)
    free = torch.cuda.mem_get_info()[0]
    s32 = s16.float() if free > 4 * n * ld + (2 << 30) else None
    t = torch.rand((16, n), dtype=torch.float64, device=eng.device, generator=g)
    y = torch.empty((16, n), dtype=torch.float64, device=eng.device)
    for b in args.b:
      dmma_flop = 2.0 * n * n * (16 if b > 8 else 8)
      for name, s, eb in (("sc_block_product_f16", s16, 2), ("sc_block_product", s32, 4)):
        if s is None:
          continue
        ms = time_product(eng, name, s, n, t, b, y, args.reps)
        row = {"n": n, "b": b, "kernel": name, "ms": ms,
               "matrix_GBps": eb * n * n / (ms * 1e-3) / 1e9,
               "dmma_TFLOPs": dmma_flop / (ms * 1e-3) / 1e12}
        report["rows"].append(row)
        print(json.dumps(row), flush=True)
    del s16, s32, t, y
    torch.cuda.empty_cache()
  if args.out:
    with open(args.out, "w") as f:
      json.dump(report, f, indent=1)


if __name__ == "__main__":
  main()
