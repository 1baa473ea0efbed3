#!/bin/bash
# ncu evidence for one training step (N_rand = 1024), run on the GPU:  scripts/profile_step.sh <tag> [<out dir>]
# 1. launch list of an eager (non-graph) bench run: per-launch gpu__time_duration
# 2. --set full capture of one step's big launches (forward x2, DGRAD x2, WGRAD x3 + reductions, divergence fwd/bwd/G)
tag=${1:-h100}
out=${2:-ncu_out}
mkdir -p "$out"
ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file $out/${tag}_launches_step.csv \
    python bench.py --steps 2 --warmup 3 --no-graph --no-cpu-baseline --no-breakdown > $out/${tag}_ncu_launches.log 2>&1
# warm-up = 3 steps; every step has 2 + 2 + 3 + 3 + 3 = 13 launches matching the filter: skip 3 steps, capture one
ncu --set full --clock-control none --import-source on -k regex:'field_fwd_kernel|field_bwd_kernel|wgrad_kernel|wgrad_reduce_kernel|div_fwd_kernel|div_bwd_kernel|div_G_kernel' \
    --launch-skip 39 -c 13 -f -o $out/${tag}_full_step \
    python bench.py --steps 1 --warmup 3 --no-graph --no-cpu-baseline --no-breakdown > $out/${tag}_ncu_full.log 2>&1
ncu -i $out/${tag}_full_step.ncu-rep --page raw --csv > $out/${tag}_ncu_full_step_raw.csv 2>> $out/${tag}_ncu_full.log
python scripts/ncu_summary.py $out/${tag}_ncu_full_step_raw.csv $out/${tag}
