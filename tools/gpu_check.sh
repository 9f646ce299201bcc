#!/bin/bash
# Validates a built tree on an H100 and collects the evidence in an output directory:
#   bash tools/gpu_check.sh [OUT_DIR]        (from the repository root; default: a new temporary directory)
# 1. the whole GPU test-suite (oracle parity first, then the reference-sources fixtures), 2. bench fast + exact,
# 3. the per-kernel device times of the bench workload with one group in flight (tools/solver_kernel_times.py,
# torch.profiler).  Every stage has its own timeout so a hang cannot eat the box.
OUT=${1:-$(mktemp -d)}
mkdir -p "$OUT"
echo "evidence in $OUT"
timeout 900 python -m pytest tests -m gpu -q -x 2>&1 | tail -25 > "$OUT/gpu_tests.log"
tail -3 "$OUT/gpu_tests.log"
timeout 300 python bench.py 2>"$OUT/bench_fast.err" | tail -1 > "$OUT/bench_fast.json"
timeout 300 python bench.py --mode exact 2>"$OUT/bench_exact.err" | tail -1 > "$OUT/bench_exact.json"
python tools/show_bench.py "$OUT/bench_fast.json" 2>/dev/null; python tools/show_bench.py "$OUT/bench_exact.json" 2>/dev/null
timeout 300 python tools/solver_kernel_times.py > "$OUT/kernel_times.txt" 2>&1
grep -v '^{' "$OUT/kernel_times.txt"
