#!/bin/bash
# One gpurun call's worth of evidence (1 GPU): launch list of a predict() step at N=65,536, one
# `ncu --set full` capture per hot kernel, the Diffuse precision study, and the summaries.
#   gpurun --timeout 1500 -- 'bash tools/gpu_profile_pack.sh r02'
# Everything lands in gpurun_out/; copy what should be judged into profiles/.
tag=${1:-r02}
n=${2:-65536}
out=gpurun_out
mkdir -p $out
NCU="ncu --profile-from-start off --clock-control none"

# 1. launch list (share of each kernel in the step; cold-cache, serialised times)
timeout 600 $NCU --metrics gpu__time_duration.sum --csv --log-file $out/${tag}_launches_n${n}.csv \
  python tools/profile_step.py --n $n > $out/${tag}_launches_n${n}.log 2>&1
python tools/summarize_launches.py $out/${tag}_launches_n${n}.csv > $out/${tag}_launches_n${n}.txt 2>&1

# 2. full captures: refinement pair, both GEMMs, the block matvec
timeout 900 $NCU --set full --import-source on -k regex:'k_blur_band|k_thrsym_upper|k_gemm_wgmma|k_symm_dmma|k_block_proj' \
  -c 7 -o $out/${tag}_full_n${n} -f python tools/profile_step.py --n $n > $out/${tag}_full_n${n}.log 2>&1
python tools/ncu_summary.py $out/${tag}_full_n${n}.ncu-rep > $out/${tag}_ncu_full_n${n}.txt 2>&1

# 3. MMAs per Diffuse product vs parity (only on request: PRECISION_STUDY=1)
if [ "$PRECISION_STUDY" = "1" ]; then
  timeout 900 python tests/diffuse_precision_study.py > $out/${tag}_diffuse_precision.md 2> $out/${tag}_diffuse_precision.err
fi
tail -5 $out/${tag}_launches_n${n}.txt
