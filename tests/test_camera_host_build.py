"""CPU-only: poselib_b200/csrc/camera.cuh (the device camera models of the estimate_* pre-step) compiled for the HOST and
compared bit for bit with the oracle's camera models on the reference's example cameras."""
import os
import shutil
import subprocess

import numpy as np
import plo_py as P
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(HERE, "_camera_host_test")
IDS = {"NULL": -1, "SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "RADIAL": 3, "OPENCV": 4}
CAMERAS = [
    ("NULL", 100, 100, []),
    ("SIMPLE_RADIAL", 1936, 1296, [2425.85, 932.383, 628.265, -0.0397695]),
    ("PINHOLE", 6214, 4138, [3425.62, 3426.29, 3118.41, 2069.07]),
    ("SIMPLE_PINHOLE", 6214, 4138, [3425.62, 3118.41, 2069.07]),
    ("RADIAL", 1936, 1296, [2425.85, 932.38, 629.325, -0.04012, 0.00123]),
    ("OPENCV", 3200, 2400, [2575.94, 2608.29, 1599.26, 1257.13, 0.141865, -0.465301, 0, 0]),
    ("OPENCV", 1024, 768, [868.993378, 866.063001, 525.942323, 420.042529, -0.399431, 0.188924, 0.000153, 0.000571]),
]


@pytest.fixture(scope="module")
def exe():
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    subprocess.check_call(["nvcc", "-std=c++17", "-O2", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-ffp-contract=off", "-o", EXE,
                           os.path.join(HERE, "camera_host_test.cu")])
    return EXE


@pytest.mark.parametrize("model,w,h,params", CAMERAS)
def test_device_camera_source_matches_oracle_bitwise(exe, model, w, h, params):
    rng = np.random.default_rng(7)
    if model == "NULL":
        pts = rng.uniform(-0.7, 0.7, (40, 2))
    else:
        pts = np.c_[rng.uniform(0.2 * w, 0.8 * w, 40), rng.uniform(0.2 * h, 0.8 * h, 40)]
    p8 = list(params) + [0.0] * (8 - len(params))
    args = [exe, str(IDS[model])] + [repr(float(v)) for v in p8] + [repr(float(v)) for v in pts.reshape(-1)]
    out = subprocess.check_output(args, text=True).strip().splitlines()
    got = np.array([[float.fromhex(t) for t in line.split()] for line in out])
    cam = None if model == "NULL" else (model, params)
    d, M = P.camera_unproject_with_jac(cam, pts)
    u2 = P.camera_unproject2(cam, pts)
    xp, J, xq = P.camera_project_with_jac(cam, d)
    ref = np.c_[d, M.reshape(len(pts), 6), u2, xp, J.reshape(len(pts), 6), xq]
    assert got.shape == ref.shape
    assert np.array_equal(got, ref), np.abs(got - ref).max()
