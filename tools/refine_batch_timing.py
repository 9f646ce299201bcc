"""End-to-end time of a batch of refinements: a loop of single refiner calls, plb_refine_batch and
plb_refine_batch_device, on the same seeded inputs.

Workloads:
  relpose500     4096 calibrated refine_relpose problems of 500 points (CAUCHY)
  relpose10000   256 calibrated refine_relpose problems of 10 000 points
  image200       1024 bundle_adjust_image problems of 200 pixels on a PINHOLE camera, focal length refined, with weights
Each workload runs through
  single         a host loop of the single entry point (cabi.refine / cabi.refine_image)
  batch          cabi.refine_batch on numpy float64 arrays (n_gpus -1)
  device         cabi.refine_batch_device on CUDA float64 tensors
The variants alternate, --warmup calls of each first; each timing is the host clock around one call, which returns after
its device work is done.  Before timing, both batch forms are checked against the single calls: models, bundle stats and
cameras equal bit for bit.  Prints one JSON line with the card's name, power limit and max SM clock, then one line per
workload and variant with the median, min and max in ms over --reps runs.

    python tools/refine_batch_timing.py [--reps 15] [--warmup 2] [--scale 1.0]
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from poselib_b200 import cabi  # noqa: E402
import make_intrinsics_golden as MG  # noqa: E402
import make_weights_golden as WG  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return dict(card=name, power_limit=power, max_sm_clock=clock)


def relpose(count, n):
    out = []
    for i in range(count):
        I = WG.inputs("relpose", "", n, 7000 + i)
        out.append({"refiner": "relpose", "a": I["a"], "b": I["b"], "model": I["model0"],
                    "bundle": cabi.BundleOpt(loss_scale=I["loss_scale"])})
    return out


def image(count, n):
    out = []
    for i in range(count):
        x, X, pose0, p0, _ = MG.problem(1, n, 9000 + i, outliers=0.1)
        w = np.random.default_rng(i).uniform(0.2, 1.5, n)
        out.append({"refiner": "bundle_image", "a": x, "b": X, "model": pose0, "weights": w,
                    "cam1": cabi.Camera("PINHOLE", tuple(p0)),
                    "bundle": cabi.BundleOpt(loss_scale=MG.LOSS_SCALE, refine_intrinsics=cabi.REFINE_FOCAL_LENGTH)})
    return out


def singles(probs):
    out = []
    for p in probs:
        if p["refiner"] == "bundle_image":
            m, c, bs = cabi.refine_image(p["model"], p["a"], p["b"], p["cam1"], p["bundle"], weights=p.get("weights"))
        else:
            m, bs = cabi.refine(p["refiner"], p["model"], p["a"], p["b"], p["bundle"], weights=p.get("weights"))
            c = np.zeros(0)
        out.append((m, bs, c))
    return out


def on_device(probs):
    return [dict(p, **{k: torch.as_tensor(p[k]).cuda() for k in ("a", "b", "weights") if k in p}) for p in probs]


def same(ref, out):
    bits = lambda v: np.ascontiguousarray(np.asarray(v, dtype=np.float64)).view(np.uint64)
    for (m, bs, c), r in zip(ref, out):
        cam = r["camera1"] if len(c) else np.zeros(0)
        if not (np.array_equal(bits(m), bits(r["model"])) and np.array_equal(bits(bs), bits(r["bundle_stats"])) and
                np.array_equal(bits(c), bits(cam))):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every workload's problem count")
    args = ap.parse_args()
    if cabi.device_count() == 0:
        sys.exit("refine_batch_timing: no CUDA device")
    cabi.set_device(0)
    print(json.dumps(card()), flush=True)
    k = lambda c: max(1, int(c * args.scale))
    workloads = {"relpose500": relpose(k(4096), 500), "relpose10000": relpose(k(256), 10000),
                 "image200": image(k(1024), 200)}
    for name, probs in workloads.items():
        dev = on_device(probs)
        variants = {"single": lambda: singles(probs), "batch": lambda: cabi.refine_batch(probs),
                    "device": lambda: cabi.refine_batch_device(dev)}
        ref = variants["single"]()
        ok = same(ref, variants["batch"]()) and same(ref, variants["device"]())
        times = {v: [] for v in variants}
        for rep in range(args.warmup + args.reps):
            for v, fn in variants.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                if rep >= args.warmup:
                    times[v].append(1e3 * dt)
        for v, t in times.items():
            print(json.dumps(dict(workload=name, problems=len(probs), n=len(probs[0]["a"]), variant=v,
                                  median_ms=round(float(np.median(t)), 3), min_ms=round(min(t), 3),
                                  max_ms=round(max(t), 3), equal_to_single=ok)), flush=True)
        if not ok:
            sys.exit(f"refine_batch_timing: {name}: batch outputs differ from the single calls")


if __name__ == "__main__":
    main()
