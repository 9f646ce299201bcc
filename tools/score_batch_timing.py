"""Throughput of plb_score_batch: scored correspondences per second (the sum of n * m over a call), host form against
device form, masks off and on, on seeded inputs.

Workloads:
  relpose   64 problems x 10 000 correspondences x 256 relative poses
  pnp       1 024 problems x 200 correspondences x 64 absolute poses
  homog     16 problems x 20 000 correspondences x 256 homographies
Each workload runs through
  host      cabi.score_batch on numpy float64 arrays (n_gpus -1)
  device    cabi.score_batch_device on CUDA float64 tensors
with masks off and on.  The variants alternate, --warmup calls of each first; each timing is the host clock around one
call, which returns after its device work is done.  Before timing, the device form is checked against the host form
(scores, counts and masks equal bit for bit).  Prints one JSON line with the card's name, power limit and max SM clock,
then one line per workload and variant: the median, min and max call time in ms over --reps calls and the median rate.

    python tools/score_batch_timing.py [--reps 15] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from poselib_b200 import cabi  # noqa: E402
from test_score_batch import _scene  # noqa: E402

WORKLOADS = {"relpose": ("relpose", 64, 10000, 256), "pnp": ("pnp", 1024, 200, 64),
             "homog": ("homography", 16, 20000, 256)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return dict(card=name, power_limit=power, max_sm_clock=clock)


def to_device(probs):
    return [dict(p, a=torch.tensor(p["a"], device="cuda:0"), b=torch.tensor(p["b"], device="cuda:0"),
                 models=torch.tensor(np.asarray(p["models"]), device="cuda:0")) for p in probs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    assert cabi.device_count() > 0, "no CUDA device"
    cabi.set_device(0)
    print(json.dumps(card()), flush=True)
    for name, (kind, count, n, m) in WORKLOADS.items():
        base = [_scene(kind, n, m, 1000 + i) for i in range(count)]
        corrs = sum(len(p["a"]) * len(p["models"]) for p in base)
        for masks in (False, True):
            host = [dict(p, inliers=masks) for p in base]
            dev = to_device(host)
            h = cabi.score_batch(host)
            d = cabi.score_batch_device(dev)
            torch.cuda.synchronize()
            for x, y in zip(h, d):
                assert np.array_equal(x["scores"].view(np.uint64), y["scores"].cpu().numpy().view(np.uint64))
                assert np.array_equal(x["num_inliers"], y["num_inliers"].cpu().numpy())
                assert (x["inliers"] is None) == (y["inliers"] is None)
                if masks:
                    assert np.array_equal(x["inliers"], y["inliers"].cpu().numpy())
            del h, d
            calls = {"host": lambda: cabi.score_batch(host), "device": lambda: cabi.score_batch_device(dev)}
            times = {k: [] for k in calls}
            for _ in range(args.warmup):
                for f in calls.values():
                    f()
            for _ in range(args.reps):
                for k, f in calls.items():
                    t0 = time.perf_counter()
                    f()
                    if k == "device":
                        torch.cuda.synchronize()
                    times[k].append(time.perf_counter() - t0)
            for k, ts in times.items():
                ms = 1e3 * np.array(ts)
                print(json.dumps(dict(workload=name, form=k, masks=masks, problems=count, n=n, m=m,
                                      median_ms=round(float(np.median(ms)), 3), min_ms=round(float(ms.min()), 3),
                                      max_ms=round(float(ms.max()), 3),
                                      gcorr_per_s=round(corrs / float(np.median(ms)) / 1e6, 2))), flush=True)
            del dev
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
