#!/usr/bin/env python
# Measurement script (not product code): times the GPU path NEXT TO the CPU oracle, like bench.py's
# cpu_baseline leg.
"""BASELINE.json configs[0]: configs.icassp2018_clusterer.predict on N=1,000 d=128 (k=4): wall time
of the GPU path and of the CPU oracle on the same box, medians of 5 after 2 warm-ups."""
import os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import spectralcluster_b200 as scb
from oracle import spectral_oracle as orc
out = []
for n, d, k in ((1000, 128, 4), (2048, 256, 4), (4096, 256, 4)):
  x = orc.synthetic_dvectors(n, d, k, seed=0)
  c = scb.SpectralClusterer(min_clusters=2, max_clusters=7,
                            refinement_options=scb.configs.icassp2018_refinement_options)
  ts = []
  for i in range(7):
    t0 = time.perf_counter(); lab = c.predict(x); ts.append(time.perf_counter() - t0)
  gpu = float(np.median(ts[2:]))
  cpu = None
  if n <= 2048:
    opt = orc.options(min_clusters=2, max_clusters=7, sequence=orc.ICASSP2018)
    orc.predict(x, opt)
    t0 = time.perf_counter(); ref = orc.predict(x, opt); cpu = time.perf_counter() - t0
    assert np.array_equal(orc.ordered(ref), scb.utils.enforce_ordered_labels(lab))
  out.append("N=%d d=%d: GPU %.1f ms (%s, %.0f emb/s)%s" % (
      n, d, gpu * 1e3, c.last_details["solver"], n / gpu,
      "" if cpu is None else "; CPU oracle %.0f ms (%.0f emb/s); labels equal" % (cpu * 1e3, n / cpu)))
print("\n".join(out))
