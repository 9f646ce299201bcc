"""Throughput of plb_generate_batch: hypotheses (models generated and scored) and scored correspondences (the sum of
n over every model) per second, host form against device form, on seeded inputs, beside the RANSAC path's own
hypothesis stage on the same scenes.

Workloads (samples drawn by PoseLib's RandomSampler, plb_host_sample_table):
  relpose   64 problems x 10 000 correspondences x 1 024 samples
  homog     16 problems x 20 000 correspondences x 1 024 samples
  pnp       256 problems x 2 000 correspondences x 1 024 samples
Each workload runs through
  host      cabi.generate_batch on numpy arrays (n_gpus -1), including the binding's allocation of the padded outputs
  host_c    plb_generate_batch alone on the same problems, outputs allocated once before timing
  device    cabi.generate_batch_device on CUDA tensors (float64 points, int32 samples)
Before timing, the device form is checked against the host form (counts, models and records equal bit for bit).  The
variants alternate, --warmup calls of each first; each timing is the host clock around one call, which returns after its
device work is done (the device form is followed by a device synchronise as well).
The same kernels in mode 0 are the RANSAC path's all-fp64 hypothesis stage: `ransac` runs plb_ransac_batch in mode 0 on
the same scenes (1 024 iterations, one stream, so that the groups' event times do not overlap) and reports that stage's
rate from plb_counters: samples_evaluated and models_evaluated over gpu_seconds - gpu_seconds_select (sampling, solve
and exact scoring of the rounds).
Prints one JSON line with the card's name, power limit and max SM clock, then one line per workload and variant.

    python tools/generate_batch_timing.py [--reps 9] [--warmup 2]
"""
import argparse
import ctypes as C
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
from test_generate_batch import problem  # noqa: E402

WORKLOADS = {"relpose": ("relpose", 64, 10000, 1024), "homog": ("homography", 16, 20000, 1024),
             "pnp": ("pnp", 256, 2000, 1024)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return dict(card=name, power_limit=power, max_sm_clock=clock)


def to_device(probs):
    return [dict(p, a=torch.tensor(p["a"], device="cuda:0"), b=torch.tensor(p["b"], device="cuda:0"),
                 samples=torch.tensor(p["samples"], device="cuda:0")) for p in probs]


def c_problems(probs):
    """The plb_generate_problem array of cabi.generate_batch with its outputs allocated once, so that `host_c` times the C
    call alone: the binding's allocation of the padded outputs (s x M slots) is part of `host`."""
    arr = (cabi.GenerateProblem * len(probs))()
    keep = []
    for q, p in zip(arr, probs):
        aa, ap = cabi._d(p["a"])
        ba, bp = cabi._d(p["b"])
        smp = np.ascontiguousarray(p["samples"], dtype=np.int32)
        s, M = len(smp), cabi.GENERATE_M[p["kind"]]
        msz = 7 if p["kind"] in ("pnp", "relpose") else 9
        out = (np.zeros(s, np.int32), np.zeros(s * M * msz), np.zeros(s * M), np.zeros(s * M, np.int64))
        keep.append((aa, ba, smp, out))
        cabi._fill_generate_problem(q, p, len(aa), s)
        q.a, q.b, q.samples = ap, bp, smp.ctypes.data_as(C.POINTER(C.c_int32))
        q.n_models, q.models = out[0].ctypes.data_as(C.POINTER(C.c_int32)), out[1].ctypes.data_as(cabi._P)
        q.scores, q.num_inliers = out[2].ctypes.data_as(cabi._P), out[3].ctypes.data_as(C.POINTER(C.c_int64))
    return arr, keep


def ransac_stage(probs):
    """The hypothesis stage of plb_ransac_batch in mode 0 on the same scenes, from its counters."""
    cabi.set_mode("exact")
    try:
        batch = cabi.Batch([{"kind": p["kind"], "a": p["a"], "b": p["b"], "max_error": float(np.sqrt(p["sq_threshold"])),
                             "ransac": cabi.RansacOpt(max_iterations=1024, min_iterations=1024, seed=i)}
                            for i, p in enumerate(probs)])
        batch.run(streams=1)
        c = batch.counter_sums()
    finally:
        cabi.set_mode("fast")
    secs = c["gpu_seconds"] - c["gpu_seconds_select"]
    mean_n = float(np.mean([len(p["a"]) for p in probs]))
    return dict(samples=c["samples_evaluated"], hypotheses=c["models_evaluated"], stage_ms=round(1e3 * secs, 3),
                mhyp_per_s=round(c["models_evaluated"] / secs / 1e6, 3),
                gcorr_per_s=round(c["models_evaluated"] * mean_n / secs / 1e9, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    assert cabi.device_count() > 0, "no CUDA device"
    cabi.set_device(0)
    print(json.dumps(card()), flush=True)
    for name, (kind, count, n, s) in WORKLOADS.items():
        host = [problem(kind, n, s, 1000 + i) for i in range(count)]
        dev = to_device(host)
        h = cabi.generate_batch(host)
        d = cabi.generate_batch_device(dev)
        torch.cuda.synchronize()
        hyps = corrs = 0
        for p, x, y in zip(host, h, d):
            nm = x["n_models"]
            assert np.array_equal(nm, y["n_models"].cpu().numpy())
            mask = np.arange(x["scores"].shape[1])[None, :] < nm[:, None]
            assert np.array_equal(x["scores"][mask].view(np.uint64), y["scores"].cpu().numpy()[mask].view(np.uint64))
            assert np.array_equal(x["num_inliers"][mask], y["num_inliers"].cpu().numpy()[mask])
            assert np.array_equal(np.asarray(x["models"])[mask].view(np.uint64),
                                  y["models"].cpu().numpy()[mask].view(np.uint64))
            hyps += int(nm.sum())
            corrs += int(nm.sum()) * len(p["a"])
        del h, d

        def device_call():
            cabi.generate_batch_device(dev)
            torch.cuda.synchronize()

        arr, keep = c_problems(host)
        calls = {"host": lambda: cabi.generate_batch(host), "host_c": lambda: cabi._check(cabi.lib().plb_generate_batch(
            arr, C.c_size_t(len(host)), -1, 8)), "device": device_call}
        times = {k: [] for k in calls}
        for _ in range(args.warmup):
            for f in calls.values():
                f()
        for _ in range(args.reps):
            for k, f in calls.items():
                t0 = time.perf_counter()
                f()
                times[k].append(time.perf_counter() - t0)
        for k, ts in times.items():
            ms = 1e3 * np.array(ts)
            med = float(np.median(ms)) / 1e3
            print(json.dumps(dict(workload=name, form=k, problems=count, n=n, s=s, hypotheses=hyps,
                                  median_ms=round(1e3 * med, 3), min_ms=round(float(ms.min()), 3),
                                  max_ms=round(float(ms.max()), 3), mhyp_per_s=round(hyps / med / 1e6, 3),
                                  gcorr_per_s=round(corrs / med / 1e9, 2))), flush=True)
        print(json.dumps(dict(workload=name, form="ransac_mode0_stage", problems=count, n=n, **ransac_stage(host))),
              flush=True)
        del dev
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
