"""Single-call latency of the LM refiners with and without PoseLib's per-residual weights on the GPU.

Inputs: the problems of tests/golden/make_weights_golden.py (inputs(), CAUCHY loss) at n = 500, 6000 and 20000 with
their weights.  For every refiner the weighted and the unweighted call alternate, each timed as the median of --reps
synchronised calls after --warmup calls of both (host clock; every call returns after its device work is done):
  bundle_adjust_image on a PINHOLE camera, flags 0 and 7; refine_relpose; refine_relpose_cameras and
  refine_relpose_pair (flags 0 and 7) on a SIMPLE_RADIAL / RADIAL pair; refine_fundamental; refine_homography.
Prints one JSON line per measurement, after one line with the card's name, power limit and max SM clock.

    python tools/weighted_refine_timing.py [--reps 15] [--warmup 3] [--sizes 500,6000,20000]
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
import make_weights_golden as WG  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return dict(card=name, power_limit=power, max_sm_clock=clock)


def medians_ms(fns, reps, warmup):
    """Median, min and max of each of fns, called in turn (alternating) reps times after warmup calls of each."""
    for _ in range(warmup):
        for fn in fns:
            fn()
    t = [[] for _ in fns]
    for _ in range(reps):
        for i, fn in enumerate(fns):
            t0 = time.perf_counter()
            fn()
            t[i].append(1e3 * (time.perf_counter() - t0))
    return [(float(np.median(v)), float(min(v)), float(max(v))) for v in t]


def calls(n):
    """(name, flags, fn(weights)) for every refiner at n points."""
    out = []
    I = WG.inputs("image", "PINHOLE", n, 1000 + n)
    cam = cabi.Camera(I["model1"], tuple(I["params1"]))
    for flags in (0, 7):
        b = cabi.BundleOpt(loss_scale=I["loss_scale"], refine_intrinsics=flags)
        out.append(("plb_bundle_adjust_image", flags, I["weights"],
                    lambda w, I=I, b=b: cabi.refine_image(I["model0"], I["a"], I["b"], cam, b, weights=w)))
    P = WG.inputs("pair", "", n, 2000 + n)
    c1, c2 = cabi.Camera(P["model1"], tuple(P["params1"])), cabi.Camera(P["model2"], tuple(P["params2"]))
    b0 = cabi.BundleOpt(loss_scale=P["loss_scale"])
    out.append(("plb_refine_relpose_cameras", 0, P["weights"],
                lambda w: cabi.refine_relpose_cameras(P["model0"], P["a"], P["b"], c1, c2, b0, weights=w)))
    for flags in (0, 7):
        b = cabi.BundleOpt(loss_scale=P["loss_scale"], refine_intrinsics=flags)
        out.append(("plb_refine_relpose_pair", flags, P["weights"],
                    lambda w, b=b: cabi.refine_relpose_pair(P["model0"], P["a"], P["b"], c1, c2, b, weights=w)))
    for kind, name in (("relpose", "plb_refine_relpose"), ("fundamental", "plb_refine_fundamental"),
                       ("homography", "plb_refine_homography")):
        K = WG.inputs(kind, "", n, 3000 + n)
        b = cabi.BundleOpt(loss_scale=K["loss_scale"])
        out.append((name, 0, K["weights"],
                    lambda w, K=K, b=b, kind=kind: cabi.refine(kind, K["model0"], K["a"], K["b"], b, weights=w)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="500,6000,20000")
    a = ap.parse_args()
    if a.reps < 7:
        sys.exit("--reps must be at least 7")
    if cabi.device_count() == 0:
        sys.exit("no CUDA device: nothing is measured")
    cabi.set_device(0)
    print(json.dumps(card()))
    for n in [int(s) for s in a.sizes.split(",")]:
        for name, flags, w, fn in calls(n):
            (mw, lw, hw), (mu, lu, hu) = medians_ms([lambda: fn(w), lambda: fn(None)], a.reps, a.warmup)
            iters = int(fn(w)[-1][0]), int(fn(None)[-1][0])
            print(json.dumps(dict(call=name, n=n, flags=flags, weighted_median_ms=mw, unweighted_median_ms=mu,
                                  weighted_min_max_ms=[lw, hw], unweighted_min_max_ms=[lu, hu],
                                  iterations_weighted_unweighted=list(iters))))


if __name__ == "__main__":
    main()
