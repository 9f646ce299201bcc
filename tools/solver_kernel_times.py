"""Per-kernel device time of the headline workload with one lock-step group in flight.

The workload is bench.py's: --pairs C2 image pairs (relpose_5pt, 10 000 correspondences, 30 % inliers, max 100 000
iterations), resident in device memory, run through one cabi.Batch with streams=1, so that no kernel shares the GPU
with a kernel of another group.  After --warmup untimed runs, --steps runs are traced with torch.profiler (CUDA
activities) and the kernels are listed with their launches, total device time per step and share of the traced kernel
time.  Prints the table, then one JSON line with the card's name, power limit and max SM clock beside the numbers.

    python tools/solver_kernel_times.py [--pairs 256] [--n 10000] [--steps 1] [--warmup 1]
"""
import argparse
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from poselib_b200 import problem_generator as G  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return dict(card=name, power_limit=power, max_sm_clock=clock)


def short_name(name):
    """'void plb::k5_roots(int, plb::HypOut)' -> 'k5_roots'; template arguments are kept: 'k_screen<2, 512>'."""
    name = re.sub(r"^void\s+", "", name)
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            cut = i
            break
    return name[:cut].replace("plb::", "").strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--n", type=int, default=10000, help="correspondences per pair (above 12 288 k_screen does not stage)")
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from poselib_b200 import cabi
    if not torch.cuda.is_available() or cabi.device_count() == 0:
        sys.exit("no CUDA device: nothing is measured")
    cabi.set_device(0)
    ropt = dict(max_iterations=100000, min_iterations=1000, seed=0)
    handles, probs = [], []
    for i in range(a.pairs):
        p = G.config_c2(i, n=a.n)
        h = cabi.resident_create("relpose", p["x1"] / G.FOCAL, p["x2"] / G.FOCAL)
        handles.append(h)
        probs.append(dict(kind="relpose", resident=h, n=len(p["x1"]), ransac=cabi.RansacOpt(**ropt),
                          max_error=1.0 / G.FOCAL))
    batch = cabi.Batch(probs)
    for _ in range(max(a.warmup, 1)):
        batch.run(streams=1)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            batch.run(streams=1)
        torch.cuda.synchronize()
    launches, us = defaultdict(int), defaultdict(float)
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        n = short_name(ev.name)
        if n.startswith("Memcpy") or n.startswith("Memset"):
            continue
        launches[n] += 1
        us[n] += ev.device_time
    total = sum(us.values())
    rows = sorted(us, key=lambda k: -us[k])
    print(f"{'kernel':<40} {'launches/step':>14} {'ms/step':>10} {'share':>7}")
    for k in rows:
        print(f"{k:<40} {launches[k] / a.steps:>14.1f} {us[k] / 1e3 / a.steps:>10.3f} {100 * us[k] / total:>6.1f}%")
    solver = sum(us[k] for k in rows if k == "k_sample" or k.startswith("k5_"))
    print(f"{'all kernels':<40} {sum(launches.values()) / a.steps:>14.1f} {total / 1e3 / a.steps:>10.3f}")
    print(f"{'5-point solver chain':<40} {'':>14} {solver / 1e3 / a.steps:>10.3f} {100 * solver / total:>6.1f}%")
    out = dict(card(), pairs=a.pairs, n=a.n, steps=a.steps, streams=1,
               kernels={k: dict(launches_per_step=launches[k] / a.steps, ms_per_step=us[k] / 1e3 / a.steps)
                        for k in rows},
               total_ms_per_step=total / 1e3 / a.steps, solver_5pt_ms_per_step=solver / 1e3 / a.steps)
    print(json.dumps(out))
    for h in handles:
        cabi.resident_free(h)


if __name__ == "__main__":
    main()
