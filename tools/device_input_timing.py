"""End-to-end time of one estimate batch from host arrays and from GPU tensors, on the same seeded inputs.

Batches: C2-sized (--c2 pairs of config_c2: relpose_5pt, 10 000 correspondences, 30 % inliers) and C1-sized (--c1
problems of config_c1: p3p, 200 correspondences, exactly 1000 iterations), both in pixels with a PINHOLE camera through
the estimate_* path.  Each batch runs through
  pageable      estimate_batch on numpy float64 arrays (staged by the engine into its pinned buffer)
  pinned        estimate_batch on float64 arrays in page-locked memory (DMA straight from them)
  device_fp64   estimate_batch_device on CUDA float64 tensors (masks returned as CUDA bool tensors)
  device_fp32   estimate_batch_device on CUDA float32 tensors
  roundtrip_fp32  what a caller with float32 CUDA tensors does without the device call: synchronise, copy to the host,
                widen to float64, estimate_batch, upload the masks again
The variants alternate, --warmup calls of each first; each timing is the host clock around one call, which returns after
its device work is done.  Prints one JSON line with the card's name, power limit and max SM clock, then one line per
batch and variant with the median, min and max in ms.  Before timing, the device variants are checked against
estimate_batch on the same values (the fp32 ones against the widened values): stats, models and masks equal.

    python tools/device_input_timing.py [--reps 9] [--warmup 2] [--c2 64] [--c1 1024]
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
from poselib_b200 import cabi, problem_generator as G  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return dict(card=name, power_limit=power, max_sm_clock=clock)


def batch(name, count):
    cam = cabi.Camera("PINHOLE", (G.FOCAL, G.FOCAL, 0.0, 0.0))
    bo = cabi.BundleOpt()
    probs = []
    for i in range(count):
        if name == "C2":
            p = G.config_c2(problem_idx=i)
            probs.append(dict(kind="relpose", a=p["x1"], b=p["x2"], cam1=cam, cam2=cam, max_error=p["max_error"],
                              ransac=cabi.RansacOpt(seed=i, **p["ransac"]), bundle=bo))
        else:
            p = G.config_c1(problem_idx=i)
            probs.append(dict(kind="pnp", a=p["x"], b=p["X"], cam1=cam, max_error=p["max_error"],
                              ransac=cabi.RansacOpt(seed=i, **p["ransac"]), bundle=bo))
    return probs


def pinned(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).pin_memory().numpy()


def on_device(probs, dtype):
    return [dict(p, a=torch.tensor(p["a"], dtype=dtype, device="cuda:0"),
                 b=torch.tensor(p["b"], dtype=dtype, device="cuda:0")) for p in probs]


def roundtrip(dev32, streams):
    torch.cuda.synchronize()
    host = [dict(p, a=p["a"].cpu().double().numpy(), b=p["b"].cpu().double().numpy()) for p in dev32]
    out = cabi.estimate_batch(host, streams=streams, n_gpus=-1)
    for o in out:
        o["inliers"] = torch.from_numpy(o["inliers"]).to("cuda:0").bool()
    torch.cuda.synchronize()
    return out


def same(ref, out):
    for r, o in zip(ref, out):
        m = o["inliers"]
        m = m.cpu().numpy() if isinstance(m, torch.Tensor) else m
        if not (r["stats"] == o["stats"] and np.array_equal(r["model"], o["model"])
                and np.array_equal(r["inliers"].astype(bool), m.astype(bool))):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--c2", type=int, default=64)
    ap.add_argument("--c1", type=int, default=1024)
    ap.add_argument("--streams", type=int, default=8)
    a = ap.parse_args()
    if a.reps < 5:
        sys.exit("--reps must be at least 5")
    if cabi.device_count() == 0 or not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing is measured")
    cabi.set_device(0)
    print(json.dumps(card()), flush=True)
    for name, count in (("C2", a.c2), ("C1", a.c1)):
        probs = batch(name, count)
        pin = [dict(p, a=pinned(p["a"]), b=pinned(p["b"])) for p in probs]
        d64, d32 = on_device(probs, torch.float64), on_device(probs, torch.float32)
        widened = [dict(p, a=d["a"].double().cpu().numpy(), b=d["b"].double().cpu().numpy()) for p, d in zip(probs, d32)]
        s = a.streams
        variants = {
            "pageable": lambda: cabi.estimate_batch(probs, streams=s, n_gpus=-1),
            "pinned": lambda: cabi.estimate_batch(pin, streams=s, n_gpus=-1),
            "device_fp64": lambda: cabi.estimate_batch_device(d64, streams=s),
            "device_fp32": lambda: cabi.estimate_batch_device(d32, streams=s),
            "roundtrip_fp32": lambda: roundtrip(d32, s),
        }
        ref64, ref32 = variants["pageable"](), cabi.estimate_batch(widened, streams=s, n_gpus=-1)
        checks = dict(device_fp64=same(ref64, variants["device_fp64"]()), device_fp32=same(ref32, variants["device_fp32"]()),
                      roundtrip_fp32=same(ref32, variants["roundtrip_fp32"]()))
        for _ in range(a.warmup):
            for fn in variants.values():
                fn()
        t = {k: [] for k in variants}
        for _ in range(a.reps):
            for k, fn in variants.items():
                t0 = time.perf_counter()
                fn()
                t[k].append(1e3 * (time.perf_counter() - t0))
        n = len(probs[0]["a"])
        for k, v in t.items():
            print(json.dumps(dict(batch=name, problems=count, n=n, variant=k, median_ms=float(np.median(v)),
                                  min_ms=float(min(v)), max_ms=float(max(v)), results_equal=checks.get(k, True))),
                  flush=True)


if __name__ == "__main__":
    main()
