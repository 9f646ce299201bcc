#!/bin/bash
# Validates a built tree on an H100 and collects the evidence in the output directory it creates:
#   bash tools/gpu_check.sh        (from the repository root)
# 1. the whole GPU test-suite (oracle parity first, then the reference-sources fixtures), 2. bench fast + exact,
# 3. the ncu launch list of one fast-mode bench step.  Every stage has its own timeout so a hang cannot eat the box.
mkdir -p gpurun_out
timeout 900 python -m pytest tests -m gpu -q -x 2>&1 | tail -25 > gpurun_out/gpu_tests.log
tail -3 gpurun_out/gpu_tests.log
timeout 300 python bench.py 2>gpurun_out/bench_fast.err | tail -1 > gpurun_out/bench_fast.json
timeout 300 python bench.py --mode exact 2>gpurun_out/bench_exact.err | tail -1 > gpurun_out/bench_exact.json
python tools/show_bench.py gpurun_out/bench_fast.json 2>/dev/null; python tools/show_bench.py gpurun_out/bench_exact.json 2>/dev/null
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/launches.csv \
    python bench.py --steps 1 --warmup 1 --streams 1 --pairs 64 > gpurun_out/ncu_bench.log 2>&1
python tools/launch_summary.py gpurun_out/launches.csv 2>/dev/null | head -20
