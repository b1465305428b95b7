"""Time predict() on embeddings already in HBM against the host-array call and bench.py's composition.

    python tools/time_device_inputs.py [--n 65536] [--d 256] [--reps 5] [--out FILE]

On bench.py's workload (speaker-turn d-vectors, seed 0; GraphCut, ICASSP refinement,
max_clusters=10), each repetition runs, in turn, with CUDA events around the call:
  * predict(X) for an fp32 CUDA tensor X,
  * predict(X16) for its fp16 cast,
  * predict(H) for the host ndarray H = X.cpu().numpy() (one upload inside the call),
  * device_step: the private-part composition bench.py's `value` times (eng.affinity,
    DeviceAffinity, _compute_eigenvectors_ncluster, eng.kmeans).
Each call ends in a host array of labels, so the stop event follows the device work it waits for.
Labels of the three predict() calls are checked equal (X16 against its own host twin).
"""

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import torch  # noqa: E402

import spectralcluster_b200 as scb  # noqa: E402
from spectralcluster_b200 import device as dev  # noqa: E402
from spectralcluster_b200 import spectral_clusterer as sc_mod  # noqa: E402
from spectralcluster_b200 import synthetic  # noqa: E402


def make_clusterer():
  return scb.SpectralClusterer(
      min_clusters=2, max_clusters=10, laplacian_type=scb.LaplacianType.GraphCut,
      refinement_options=scb.RefinementOptions(
          gaussian_blur_sigma=1, p_percentile=0.95, thresholding_soft_multiplier=0.01,
          thresholding_type=scb.ThresholdType.RowMax,
          refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)),
      custom_dist="cosine")


def timed(fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  a.record()
  out = fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b), out


def gpu_description():
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
  except Exception:
    return torch.cuda.get_device_name()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=65536)
  ap.add_argument("--d", type=int, default=256)
  ap.add_argument("--reps", type=int, default=5)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("needs a CUDA device")
  n, d = args.n, args.d
  eng = dev.Engine.get()
  host = synthetic.speaker_turn_dvectors(n, d, 6, seed=0).astype(np.float32)
  x = torch.from_numpy(host).to(eng.device)
  x16 = x.half()
  h16 = x16.cpu().numpy()
  clusterer = make_clusterer()

  def device_step():
    a, crop = eng.affinity(x, want_crop_vector=True)
    aff = sc_mod.DeviceAffinity(a, n, crop, True)
    v, k, _ = clusterer._compute_eigenvectors_ncluster(aff)
    k = max(k, clusterer.min_clusters)
    return eng.kmeans(v[:, :k].contiguous(), k, 0, clusterer.max_iter)[0]

  cases = {"predict(X) fp32": lambda: clusterer.predict(x),
           "predict(X) fp16": lambda: clusterer.predict(x16),
           "predict(H) fp32": lambda: clusterer.predict(host),
           "device_step": device_step}
  labels = {name: fn() for name, fn in cases.items()}           # warm-up
  assert np.array_equal(labels["predict(X) fp32"], labels["predict(H) fp32"])
  assert np.array_equal(labels["predict(X) fp16"], clusterer.predict(h16))
  ms = {name: [] for name in cases}
  for _ in range(args.reps):
    for name, fn in cases.items():
      ms[name].append(timed(fn)[0])
  result = {"gpu": gpu_description(), "n": n, "d": d, "reps": args.reps,
            "ms": {name: [round(v, 2) for v in vals] for name, vals in ms.items()},
            "median_ms": {name: round(float(np.median(vals)), 2) for name, vals in ms.items()},
            "labels_equal": True}
  text = json.dumps(result, indent=1)
  print(text)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
