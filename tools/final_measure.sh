#!/bin/bash
# Evidence run on ONE GPU: bench lines of every BASELINE config with their CPU legs, the reference arm,
# one `ncu --set full` capture of the tier-0 and prep kernels and the launch list of the bench command.
#   tools/final_measure.sh <tag>
set -u
tag=${1:-r2}
mkdir -p gpurun_out
(timeout 500 python bench.py --steps 20 --warmup 3 2>&1 | tail -1) > gpurun_out/bench_${tag}_c4.json
(timeout 400 python bench.py --impl reference --steps 5 --warmup 1 2>&1 | tail -1) > gpurun_out/bench_${tag}_c4_reference.json
(timeout 300 python bench.py --config C2 --steps 20 2>&1 | tail -1) > gpurun_out/bench_${tag}_c2.json
(timeout 400 python bench.py --config C3 --steps 20 2>&1 | tail -1) > gpurun_out/bench_${tag}_c3.json
(timeout 300 python bench.py --config C5 --steps 20 2>&1 | tail -1) > gpurun_out/bench_${tag}_c5.json
(timeout 300 python bench.py --steps 20 --warmup 3 --no-cpu-baseline --max-pfanout 4 --max-gfanout 4 2>&1 | tail -1) > gpurun_out/bench_${tag}_c4_caps44.json
timeout 300 ncu --set full --clock-control none --import-source on -k regex:"match_topics_lane|order_prep" -s 8 -c 2 -o gpurun_out/prof_${tag} \
    python bench.py --steps 2 --warmup 3 --no-cpu-baseline > gpurun_out/ncu_${tag}.log 2>&1
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -s 40 -c 80 --csv --log-file gpurun_out/launches_${tag}.csv \
    python bench.py --steps 6 --warmup 3 --no-cpu-baseline > gpurun_out/launch_${tag}.log 2>&1
timeout 200 ncu --set full --clock-control none -k regex:"rmatch_kernel" -s 3 -c 1 -o gpurun_out/prof_${tag}_rmatch \
    python bench.py --config C5 --steps 2 --no-cpu-baseline > gpurun_out/ncu_${tag}_rmatch.log 2>&1
ls -la gpurun_out | tail -12
