"""Times plb_camera_batch[_device]: 1 024 cameras x 8 192 points of one model per call, for PINHOLE, OPENCV,
RADIAL_FISHEYE and DIVISION, every op, without and with both Jacobians, host and device (fp64) form.

Per case: the call's wall time (median of the timed calls, host clock around a call that ends in a synchronisation),
the k_camera kernel time (torch.profiler, CUDA activities, in a run of its own), and bytes moved (inputs read plus
outputs written, computed from the shapes) over the kernel time, against the H100 SXM's 3.35 TB/s.  The card's name,
power limit and maximum SM clock are read in the same run.

    python tools/camera_batch_timing.py [--cams 1024] [--points 8192] [--reps 3] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from poselib_b200 import cabi  # noqa: E402

PEAK_BW = 3.35e12
MODELS = {"PINHOLE": (500.0, 510.0, 320.0, 240.0), "OPENCV": (500.0, 510.0, 320.0, 240.0, -0.3, 0.1, 1e-3, 2e-3),
          "RADIAL_FISHEYE": (400.0, 320.0, 240.0, -0.04, -0.005), "DIVISION": (500.0, 510.0, 320.0, 240.0, -0.2)}
CALLS = [("project", False), ("project", True), ("unproject", False), ("unproject", True), ("unproject_2d", False)]


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def problems(model, op, jac, cams, pts, rng):
    P = cabi.CAMERA_NUM_PARAMS[cabi.CAMERA[model]]
    base = np.array(MODELS[model])
    out = []
    for _ in range(cams):
        p = base * (1.0 + 1e-3 * rng.normal(size=len(base)))
        if op == "project":
            x = np.c_[rng.uniform(-1, 1, (pts, 2)), rng.uniform(2, 6, pts)]
        else:
            x = np.c_[rng.uniform(0, 640, pts), rng.uniform(0, 480, pts)]
        out.append(dict(op=op, cam=cabi.Camera(model, tuple(p)), x=x, jac=jac, jac_params=jac))
    rows = 2 if op == "project" else 3
    in_w, out_w = (3 if op == "project" else 2), (3 if op == "unproject" else 2)
    nbytes = cams * pts * 8 * (in_w + out_w + ((6 + rows * P) if jac else 0))
    return out, nbytes


def kernel_ms(torch, fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if "k_camera" in e.name]
    return sum(e.device_time_total for e in ev) / 1e3 if ev else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cams", type=int, default=1024)
    ap.add_argument("--points", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the rows as JSON to this file")
    a = ap.parse_args()
    import torch
    if cabi.device_count() == 0:
        sys.exit("no CUDA device")
    cabi.set_device(0)
    rng = np.random.default_rng(0)
    gpu = card()
    print("card (name, power limit, max SM clock):", gpu)
    rows = []
    for model in MODELS:
        for op, jac in CALLS:
            probs, nbytes = problems(model, op, jac, a.cams, a.points, rng)
            dprobs = [dict(p, x=torch.tensor(p["x"], device="cuda:0")) for p in probs]
            torch.cuda.synchronize()
            for form, call in (("host", lambda: cabi.camera_batch(probs, streams=1)),
                               ("device", lambda: cabi.camera_batch_device(dprobs, streams=1))):
                call()  # warm-up: module load and buffer growth
                torch.cuda.synchronize()
                ts = []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    call()
                    torch.cuda.synchronize()
                    ts.append(time.perf_counter() - t0)
                kms = kernel_ms(torch, call)
                r = dict(model=model, op=op, jac=jac, form=form, call_ms=1e3 * float(np.median(ts)), kernel_ms=kms,
                         bytes=nbytes, tb_s=nbytes / (kms * 1e-3) / 1e12, frac_bw=nbytes / (kms * 1e-3) / PEAK_BW)
                rows.append(r)
                print("%-15s %-13s jac=%d %-6s call %8.2f ms  kernel %7.3f ms  %6.3f TB/s  %5.1f %% of 3.35 TB/s" %
                      (model, op, jac, form, r["call_ms"], kms, r["tb_s"], 100 * r["frac_bw"]), flush=True)
            del dprobs
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=gpu, cams=a.cams, points=a.points, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
