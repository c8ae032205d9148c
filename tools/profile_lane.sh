#!/bin/bash
# One-stop profile of the tier-0 kernel on ONE GPU:
#   tools/profile_lane.sh <tag>
# writes gpurun_out/prof_<tag>.ncu-rep (ncu --set full, source counters), gpurun_out/launches_<tag>.csv (launch list of the
# bench command) and, when ncu can export here, the JSON summaries tools/ncu_summary.py makes.
set -u
tag=${1:-lane}
mkdir -p gpurun_out
ncu --set full --clock-control none --import-source on -k regex:match_topics_lane -s 3 -c 1 -o gpurun_out/prof_$tag \
    python bench.py --steps 3 --warmup 3 --no-cpu-baseline > gpurun_out/ncu_$tag.log 2>&1
ncu --metrics gpu__time_duration.sum --clock-control none -s 60 -c 120 --csv --log-file gpurun_out/launches_$tag.csv \
    python bench.py --steps 6 --warmup 3 --no-cpu-baseline > gpurun_out/launch_$tag.log 2>&1
ncu -i gpurun_out/prof_$tag.ncu-rep --page raw --csv > gpurun_out/raw_$tag.csv 2>/dev/null && \
    python tools/ncu_summary.py kernel gpurun_out/raw_$tag.csv gpurun_out/summary_$tag.ncu.json "ncu --set full --clock-control none, tier-0 kernel, bench.py C4 full size ($tag)"
python tools/ncu_summary.py launches gpurun_out/launches_$tag.csv gpurun_out/launches_$tag.json "launch list of bench.py --steps 6 --warmup 3 ($tag); cold-cache serialised times, compare shares"
ls -la gpurun_out | tail -6
