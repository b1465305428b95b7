#!/bin/bash
# compute-sanitizer racecheck + synccheck on the wgmma GEMM (affinity, Diffuse), the cp.async blur
# pipeline (fused chain), the symmetric blur pair and the block matvec, at small N (VERDICT r01
# item 9).  Writes gpurun_out/<tag>_sanitizer_{racecheck,synccheck}.txt
tag=${1:-r02}
sel='affinity_vs_oracle and 200 or diffuse_vs_oracle and 513 or fused_chain_equals_operator_chain or lanczos_matches_dense'
for tool in racecheck synccheck; do
  timeout 420 compute-sanitizer --tool $tool --print-limit 20 \
    python -m pytest tests/test_gpu_ops.py -x -q -k "$sel" > gpurun_out/${tag}_sanitizer_${tool}.txt 2>&1
  echo "exit code: $?" >> gpurun_out/${tag}_sanitizer_${tool}.txt
done
