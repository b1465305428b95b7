#!/usr/bin/env python
"""Opcode histogram of the built library's SASS (cuobjdump -sass), per kernel family: the evidence
that the hot kernels are Hopper-native (HGMMA = wgmma, UTMALDG = TMA loads, SYNCS = mbarrier,
LDGSTS = cp.async, DMMA = fp64 tensor cores; no HMMA mma.sync fp16 path).

    python tools/sass_histogram.py
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "spectralcluster_b200", "lib", "libspectralcluster_b200.so")
INTERESTING = ("HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "LDGSTS", "HMMA", "DMMA", "DFMA", "FFMA", "FFMA2", "SHFL", "ATOMG", "RED", "SYNCS", "BAR",
               "LDG", "STG", "LDS", "STS", "MUFU")

out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
per = collections.OrderedDict()
name = None
for line in out.splitlines():
  m = re.search(r"Function : (\S+)", line)
  if m:
    name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
    name = re.sub(r"\(.*", "", name)
    per[name] = collections.Counter()
    continue
  m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_]+)", line)
  if m and name:
    per[name][m.group(1).split(".")[0]] += 1
print("# SASS opcode histogram of %s (sm_90a), cuobjdump -sass" % os.path.basename(LIB))
total = collections.Counter()
for k, c in per.items():
  total.update(c)
print("# whole library: " + ", ".join("%s %d" % (op, total[op]) for op in INTERESTING if total[op]))
print("# mma.sync fp16 tensor path (HMMA): %d instructions" % total["HMMA"])
for k, c in per.items():
  n = sum(c.values())
  keys = [op for op in INTERESTING if c[op]]
  print("%-72s %6d instr | %s" % (k[:72], n, " ".join("%s:%d" % (op, c[op]) for op in keys)))
