"""In-tree build of libspectralcluster_b200.so (sm_90a only).

    python -m spectralcluster_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  Objects and the shared library are written to
spectralcluster_b200/lib/ (git-ignored build products).
"""

from __future__ import annotations

import concurrent.futures
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
LIBNAME = "libspectralcluster_b200.so"
INCLUDE = os.path.join(os.path.dirname(PKG), "include")

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-O2",
              "--expt-relaxed-constexpr", "-I", INCLUDE]


def nvcc_path() -> str:
  for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
    if cand and os.path.exists(cand):
      return cand
  raise RuntimeError("nvcc not found: spectralcluster_b200 needs the CUDA toolkit to build")


def sources():
  return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def headers():
  hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
  hs.append(os.path.join(INCLUDE, "spectralcluster_b200.h"))
  return hs


def _stale(target: str, deps) -> bool:
  if not os.path.exists(target):
    return True
  t = os.path.getmtime(target)
  return any(os.path.getmtime(d) > t for d in deps)


def _compile(nvcc: str, src: str, obj: str, verbose: bool):
  cmd = [nvcc] + ARCH_FLAGS + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + [
      "-c", os.path.join(CSRC, src), "-o", obj]
  res = subprocess.run(cmd, capture_output=True, text=True)
  if res.returncode != 0:
    raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, res.stdout, res.stderr))
  return src, res.stderr


def build(force: bool = False, verbose: bool = False) -> str:
  os.makedirs(LIBDIR, exist_ok=True)
  nvcc = nvcc_path()
  hdrs = headers()
  jobs = []
  objs = []
  for src in sources():
    obj = os.path.join(LIBDIR, src[:-3] + ".o")
    objs.append(obj)
    if force or _stale(obj, [os.path.join(CSRC, src)] + hdrs):
      jobs.append((src, obj))
  with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as pool:
    for src, log in pool.map(lambda j: _compile(nvcc, j[0], j[1], verbose), jobs):
      if verbose:
        print("== %s\n%s" % (src, log))
  lib = os.path.join(LIBDIR, LIBNAME)
  if force or jobs or _stale(lib, objs):
    cmd = [nvcc] + ARCH_FLAGS + ["-shared", "-o", lib] + objs + ["-cudart", "static"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
      raise RuntimeError("link failed:\n%s\n%s" % (res.stdout, res.stderr))
  return lib


if __name__ == "__main__":
  path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
  print(path)
