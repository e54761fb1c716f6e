#!/bin/bash
# ncu launch lists and captures (ONE GPU): launch lists + one --set full capture of the
# solve kernels for the two batch workloads.  Numbers printed by bench.py under ncu are NOT bench values.
R=${1:-rd2}
MODE=${2:-full}   # "launches": launch lists only
mkdir -p gpurun_out
B="python bench.py --steps 3 --warmup 3 --no-cpu-baseline"
ncu --metrics gpu__time_duration.sum --clock-control none -c 150 --csv --log-file gpurun_out/${R}_m3500_batch_launches.csv $B --workload m3500_batch > gpurun_out/${R}_ncu_m3500_a.log 2>&1
[ $MODE = full ] && ncu --set full --clock-control none --import-source on -k regex:"k_factor|k_backsolve|k_linearize" -s 12 -c 3 -o gpurun_out/${R}_m3500_batch_prof $B --workload m3500_batch > gpurun_out/${R}_ncu_m3500_b.log 2>&1
ncu --metrics gpu__time_duration.sum --clock-control none -c 150 --csv --log-file gpurun_out/${R}_100k_batch_launches.csv $B --workload manhattan_batch > gpurun_out/${R}_ncu_100k_a.log 2>&1
[ $MODE = full ] && ncu --set full --clock-control none --import-source on -k regex:"k_factor|k_backsolve|k_linearize" -s 20 -c 5 -o gpurun_out/${R}_100k_batch_prof $B --workload manhattan_batch > gpurun_out/${R}_ncu_100k_b.log 2>&1
# launch list of a stretch of the M3500 replay (k_step = one fused small step; single-pass metric only: the host
# spins on k_step's completion flag and re-uses its pinned payload, which a multi-pass replay would read again)
ncu --metrics gpu__time_duration.sum --clock-control none -s 400 -c 400 --csv --log-file gpurun_out/${R}_m3500_replay_launches.csv python bench.py --workload m3500_replay --steps 600 --no-cpu-baseline > gpurun_out/${R}_ncu_replay.log 2>&1
ls -la gpurun_out/${R}_*
