"""Single-call latency of the relative-pose camera refinement on the GPU.

Inputs: C2-sized two-view problems (10 000 correspondences, 30 % inliers) with the --models cameras on both images
(RADIAL and OPENCV by default; RADIAL_FISHEYE and DIVISION are the test cameras of
tests/golden/make_camera_models_golden.py).  Timed, each as the median of --reps synchronised calls after --warmup
calls (host clock; every call returns after its device work is done):
  * plb_estimate_relative_pose_pair with tangent_sampson, refine flags 0 and 7;
  * plb_refine_relpose_pair with flags 0 and 7 on the inlier set of the flags-0 estimate;
  * with --pnp, plb_estimate_absolute_pose_image with refine flags 0 and 7 on a 10 000-point PnP problem (30 % inliers)
    of the same camera.
Prints one JSON line per measurement, after one line with the card's name, power limit and max SM clock.

    python tools/relpose_pair_timing.py [--reps 9] [--warmup 3] [--models RADIAL,OPENCV,RADIAL_FISHEYE,DIVISION] [--pnp]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from poselib_b200 import cabi  # noqa: E402
import make_relpose_intrinsics_golden as RG  # noqa: E402
import make_camera_models_golden as CG  # noqa: E402

N, INLIER_RATIO, MAX_ERROR = 10000, 0.3, 1.0
NEW_MODELS = {"RADIAL_FISHEYE": "RADIAL_FISHEYE", "DIVISION": "DIVISION-"}  # model -> test camera of CG.CAMERAS


def pair_inputs(model):
    if model in NEW_MODELS:
        x1, x2, pose0, c1, c2 = CG.pair_problem(NEW_MODELS[model], NEW_MODELS[model], N, 1234 + cabi.CAMERA[model],
                                                outliers=1.0 - INLIER_RATIO)
    else:
        mid = RG.MODELS[model]
        x1, x2, pose0, c1, c2 = RG.pair_problem(mid, mid, N, 1234 + mid, outliers=1.0 - INLIER_RATIO)
    return x1, x2, cabi.Camera(model, tuple(c1)), cabi.Camera(model, tuple(c2))


def pnp_inputs(model):
    if model in NEW_MODELS:
        x, X, _, p0 = CG.problem(NEW_MODELS[model], N, 4321, outliers=1.0 - INLIER_RATIO)
    else:
        x, X, _, p0, _ = RG.MG.problem(RG.MODELS[model], N, 4321, outliers=1.0 - INLIER_RATIO)
    return x, X, cabi.Camera(model, tuple(p0))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return dict(card=name, power_limit=power, max_sm_clock=clock)


def median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(t)), float(min(t)), float(max(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--models", default="RADIAL,OPENCV", help="comma-separated: RADIAL, OPENCV, RADIAL_FISHEYE, DIVISION")
    ap.add_argument("--pnp", action="store_true", help="also time plb_estimate_absolute_pose_image")
    a = ap.parse_args()
    models = a.models.split(",")
    for m in models:
        if m not in ("RADIAL", "OPENCV") and m not in NEW_MODELS:
            sys.exit("unknown --models entry %r" % m)
    if a.reps < 7:
        sys.exit("--reps must be at least 7")
    if cabi.device_count() == 0:
        sys.exit("no CUDA device: nothing is measured")
    print(json.dumps(card()))
    ro = cabi.RansacOpt(max_iterations=10000, min_iterations=100, seed=0)
    for model in models:
        x1, x2, cam1, cam2 = pair_inputs(model)
        base = cabi.estimate_relative_pose_pair(x1, x2, cam1, cam2, ro, cabi.BundleOpt(), MAX_ERROR)
        keep = base["inliers"].astype(bool)
        for flags in (0, 7):
            b = cabi.BundleOpt(refine_intrinsics=flags)
            med, lo, hi = median_ms(lambda: cabi.estimate_relative_pose_pair(x1, x2, cam1, cam2, ro, b, MAX_ERROR),
                                    a.reps, a.warmup)
            print(json.dumps(dict(call="plb_estimate_relative_pose_pair", camera=model, n=N, flags=flags,
                                  num_inliers=int(keep.sum()), median_ms=med, min_ms=lo, max_ms=hi)))
        for flags in (0, 7):
            b = cabi.BundleOpt(refine_intrinsics=flags)
            med, lo, hi = median_ms(lambda: cabi.refine_relpose_pair(base["model"], x1[keep], x2[keep], cam1, cam2, b),
                                    a.reps, a.warmup)
            print(json.dumps(dict(call="plb_refine_relpose_pair", camera=model, n=int(keep.sum()), flags=flags,
                                  median_ms=med, min_ms=lo, max_ms=hi)))
        if a.pnp:
            x, X, cam = pnp_inputs(model)
            for flags in (0, 7):
                b = cabi.BundleOpt(refine_intrinsics=flags)
                med, lo, hi = median_ms(lambda: cabi.estimate_image(x, X, cam, ro, b, 4.0), a.reps, a.warmup)
                print(json.dumps(dict(call="plb_estimate_absolute_pose_image", camera=model, n=N, flags=flags,
                                      median_ms=med, min_ms=lo, max_ms=hi)))


if __name__ == "__main__":
    main()
