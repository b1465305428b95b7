#!/usr/bin/env python
"""Times the windowed eigensolve of predict_sharded() (max_clusters=None) against predict()'s at
N = 65,536 on one GPU, alternating, then predict_sharded() at N = 131,072 over every GPU of the
box.  For each call: the wall time (host clock; both calls end in a device synchronise), the
windows, the passes over S and the passes spent in the lambda_max solve.  The card name and
power limit are read in the same run.

    python tools/time_sharded_windows.py [--n 65536] [--large 131072] [--reps 2]
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import eigen_windows, sharded


def card_name():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  return out.splitlines()[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def count_lambda_max_passes():
  """Record, in each ops object's stats, the passes over S its lambda_max() solve took."""
  for cls in (eigen_windows.DeviceOps, sharded.ShardedOps):
    def lambda_max(self, _inner=cls.lambda_max):
      before = self.stats["passes"]
      value = _inner(self)
      self.stats["lambda_max_passes"] = self.stats["passes"] - before
      return value
    cls.lambda_max = lambda_max


def clusterer(name):
  kw = dict(laplacian_type=scb.LaplacianType.GraphCut) if name == "graphcut_max_none" else {}
  return scb.SpectralClusterer(
      refinement_options=scb.RefinementOptions(
          refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)), **kw)


def record(route, name, n, world, rep, c, labels, truth, seconds):
  stats = c.last_details["lanczos_stats"]
  rec = dict(route=route, case=name, n=n, world=world, rep=rep, wall_ms=round(1e3 * seconds, 1),
             solver=c.last_details["solver"], values=len(c.last_details["eigenvalues"]),
             k=int(c.last_details["n_clusters"]), windows=stats["windows"],
             passes=stats["passes"], lambda_max_passes=stats.get("lambda_max_passes", 0),
             labels_match_truth=bool(np.array_equal(scb.utils.enforce_ordered_labels(labels),
                                                    scb.utils.enforce_ordered_labels(truth))))
  print(json.dumps(rec), flush=True)


def one_gpu(n, reps):
  from oracle import spectral_oracle as orc
  x, truth = orc.synthetic_dvectors(n, 256, 6, seed=0, return_labels=True)
  warm = orc.synthetic_dvectors(4096, 256, 6, seed=1)
  clusterer("graphcut_max_none").predict(warm)
  sharded.predict_sharded(clusterer("graphcut_max_none"), warm)
  for rep in range(reps):
    for name in ("graphcut_max_none", "nolaplacian_max_none"):
      for route in ("predict", "predict_sharded"):
        c = clusterer(name)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        labels = c.predict(x) if route == "predict" else sharded.predict_sharded(c, x)
        torch.cuda.synchronize()
        record(route, name, n, 1, rep, c, labels, truth, time.perf_counter() - t0)
        del c, labels
        torch.cuda.empty_cache()


def _large_worker(rank, world, port, n, reps):
  os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
  torch.cuda.set_device(rank)
  import torch.distributed as dist
  dist.init_process_group("nccl", rank=rank, world_size=world)
  count_lambda_max_passes()
  from oracle import spectral_oracle as orc
  x, truth = orc.synthetic_dvectors(n, 256, 6, seed=0, return_labels=True)
  for rep in range(reps + 1):                      # the first call warms up
    c = clusterer("graphcut_max_none")
    dist.barrier()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    labels = sharded.predict_sharded(c, x, dist=dist)
    torch.cuda.synchronize()
    if rank == 0 and rep > 0:
      record("predict_sharded", "graphcut_max_none", n, world, rep - 1, c, labels, truth,
             time.perf_counter() - t0)
  dist.destroy_process_group()


def many_gpus(n, reps):
  world = torch.cuda.device_count()
  if world < 2:
    print(json.dumps(dict(route="predict_sharded", case="graphcut_max_none", n=n,
                          world=world, result="not measured: one GPU holds neither the sharded "
                          "path's N x N buffers nor predict()'s stored route at this N")),
          flush=True)
    return
  s = socket.socket()
  s.bind(("127.0.0.1", 0))
  port = s.getsockname()[1]
  s.close()
  import torch.multiprocessing as mp
  mp.spawn(_large_worker, args=(world, port, n, reps), nprocs=world, join=True)


if __name__ == "__main__":
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=65536)
  ap.add_argument("--large", type=int, default=131072)
  ap.add_argument("--reps", type=int, default=2)
  a = ap.parse_args()
  print("card: %s; GPUs: %d" % (card_name(), torch.cuda.device_count()), flush=True)
  count_lambda_max_passes()
  one_gpu(a.n, a.reps)
  torch.cuda.empty_cache()
  many_gpus(a.large, a.reps)
