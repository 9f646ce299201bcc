"""CPU-only: poselib_b200/csrc/solver5_lane.cuh (the thread-per-sample first half of the device relpose_5pt: nullspace,
constraint expansion, elimination, determinant polynomial) compiled for the HOST and compared bit for bit with the
oracle's intermediates on random, noisy-scene and near-degenerate samples."""
import os
import shutil
import subprocess

import numpy as np
import plo_py as P
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(HERE, "_solver5_lane_host_test")


@pytest.fixture(scope="module")
def exe():
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    subprocess.check_call(["nvcc", "-std=c++17", "-O2", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-Xcompiler", "-ffp-contract=off", "-o", EXE, os.path.join(HERE, "solver5_lane_host_test.cu")])
    return EXE


def unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def samples():
    rng = np.random.default_rng(11)
    out = []
    for _ in range(150):  # unrelated bearings (what an outlier-heavy RANSAC sample looks like)
        out.append((unit(rng.normal(size=(5, 3))), unit(rng.normal(size=(5, 3)))))
    for _ in range(150):  # a true two-view scene, image-like bearings, a little noise
        X = np.c_[rng.uniform(-2, 2, (5, 2)), rng.uniform(3, 8, 5)]
        w = rng.normal(size=3) * 0.2
        th = np.linalg.norm(w)
        K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        R = np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th**2 * K @ K
        t = rng.normal(size=3)
        x1 = X[:, :2] / X[:, 2:] + rng.normal(size=(5, 2)) * 1e-3
        Y = X @ R.T + t
        x2 = Y[:, :2] / Y[:, 2:] + rng.normal(size=(5, 2)) * 1e-3
        out.append((unit(np.c_[x1, np.ones(5)]), unit(np.c_[x2, np.ones(5)])))
    for _ in range(40):  # repeated / nearly repeated correspondences: rank-deficient epipolar matrix, zero pivots
        a, b = unit(rng.normal(size=(5, 3))), unit(rng.normal(size=(5, 3)))
        a[4], b[4] = a[0], b[0]
        if rng.uniform() < 0.5:
            a[3], b[3] = unit(a[1] + 1e-9 * rng.normal(size=3)), unit(b[1] + 1e-9 * rng.normal(size=3))
        out.append((a, b))
    return out


def test_lane_first_half_matches_oracle_bitwise(exe):
    S = samples()
    text = [str(len(S))]
    for a, b in S:
        text.append(" ".join(float(v).hex() for v in np.r_[a.reshape(-1), b.reshape(-1)]))
    res = subprocess.run([exe], input="\n".join(text) + "\n", capture_output=True, text=True, check=True).stdout.strip().splitlines()
    assert len(res) == len(S)
    bad = 0
    for (a, b), line in zip(S, res):
        got = np.array([float.fromhex(t) for t in line.split()])
        nb, A, c = P.relpose_5pt_stages(a, b)
        ref = np.r_[nb, A, c]
        if not np.array_equal(got.view(np.uint64), ref.view(np.uint64)):
            fin = np.isfinite(ref) & np.isfinite(got)
            if not (np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(got[fin], ref[fin])):
                bad += 1
    assert bad == 0, f"{bad} of {len(S)} samples differ"
