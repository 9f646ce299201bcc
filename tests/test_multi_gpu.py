"""GPU tests (-m gpu) of the in-process multi-GPU batch call plb_ransac_batch_multi: a plain C++ client of
include/poselib_b200.h (tests/multi_gpu_client.cc, built by __graft_entry__.build()) and the ctypes binding.  On a
one-GPU box the call degenerates to one device (still through the multi entry point); with `gpurun --gpus N` the same
tests spread the batch over N devices and require results identical to the single-device run."""
import os
import subprocess

import numpy as np
import pytest

from poselib_b200 import problem_generator as G

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cabi():
    from poselib_b200 import cabi as c
    if c.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    c.set_device(0)
    return c


def test_cpp_client_of_the_c_header_drives_every_gpu(cabi):
    exe = os.path.join(ROOT, "tests", "_multi_gpu_client")
    assert os.path.exists(exe), "tests/_multi_gpu_client missing: run __graft_entry__.build()"
    out = subprocess.run([exe, "48"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert f"devices {cabi.device_count()} ok" in out.stdout


def test_batch_multi_equals_batch(cabi):
    probs = []
    for i in range(24):
        if i % 2:
            p = G.relpose_problem(800 + 50 * i, 0.4, config_id=41, problem_idx=i)
            probs.append(dict(kind="relpose", a=p["x1"] / G.FOCAL, b=p["x2"] / G.FOCAL,
                              ransac=cabi.RansacOpt(max_iterations=4000, min_iterations=100, seed=i), max_error=1.0 / G.FOCAL))
        else:
            p = G.abspose_problem(150 + i, 0.5, config_id=42, problem_idx=i)
            probs.append(dict(kind="pnp", a=p["x"] / G.FOCAL, b=p["X"],
                              ransac=cabi.RansacOpt(max_iterations=500, min_iterations=500, seed=i), max_error=12.0 / G.FOCAL))
    one = cabi.ransac_batch(probs, streams=4)
    for n_gpus in (0, 1):
        many = cabi.ransac_batch(probs, streams=3, n_gpus=n_gpus)
        for a, b in zip(one, many):
            assert a["stats"] == b["stats"] and np.array_equal(a["model"], b["model"]) and np.array_equal(a["inliers"], b["inliers"])
    with pytest.raises(cabi.PoseLibB200Error):
        cabi.ransac_batch(probs[:2], n_gpus=cabi.device_count() + 1)


def test_estimate_batch_equals_single_estimate_calls(cabi):
    """plb_estimate_batch: pixels + cameras in; every problem must come out exactly as from its single entry point —
    distorted cameras (device pre-step), the tangent-Sampson estimator, F / H with normalize_points, too few points."""
    F = G.FOCAL
    pin = cabi.Camera("PINHOLE", (F, F, 0.0, 0.0))
    rad = cabi.Camera("SIMPLE_RADIAL", (F, 3.0, -2.0, 0.05))
    bo = cabi.BundleOpt()
    probs = []
    for i in range(4):
        p = G.relpose_problem(900 + 40 * i, 0.5, config_id=43, problem_idx=i)
        probs.append(dict(kind="relpose", a=p["x1"], b=p["x2"], cam1=pin, cam2=rad if i % 2 else pin, max_error=1.0,
                          tangent_sampson=(i >= 2), ransac=cabi.RansacOpt(max_iterations=3000, min_iterations=100, seed=i), bundle=bo))
        p = G.abspose_problem(180 + i, 0.5, config_id=44, problem_idx=i)
        probs.append(dict(kind="pnp", a=p["x"], b=p["X"], cam1=rad if i % 2 else pin, max_error=12.0,
                          ransac=cabi.RansacOpt(max_iterations=400, min_iterations=400, seed=i), bundle=bo))
        p = G.relpose_problem(700, 0.4, config_id=45, problem_idx=i)
        probs.append(dict(kind="fundamental", a=p["x1"], b=p["x2"], max_error=1.0, rfc=bool(i % 2),
                          ransac=cabi.RansacOpt(max_iterations=2000, min_iterations=100, seed=i), bundle=bo))
        p = G.homography_problem(600, 0.6, config_id=46, problem_idx=i)
        probs.append(dict(kind="homography", a=p["x1"], b=p["x2"], max_error=1.0,
                          ransac=cabi.RansacOpt(max_iterations=1500, min_iterations=100, seed=i), bundle=bo))
    probs.append(dict(kind="fundamental", a=np.zeros((5, 2)), b=np.zeros((5, 2)), max_error=1.0, ransac=cabi.RansacOpt(), bundle=bo))
    single = [cabi.estimate(q["kind"], q["a"], q["b"], q["ransac"], q["bundle"], q["max_error"], cam1=q.get("cam1"),
                            cam2=q.get("cam2"), rfc=q.get("rfc", False), tangent_sampson=q.get("tangent_sampson", False))
              for q in probs]
    for n_gpus in (-1, 0):
        batch = cabi.estimate_batch(probs, streams=3, n_gpus=n_gpus)
        for q, a, b in zip(probs, single, batch):
            assert b["status"] == 0
            assert a["stats"] == b["stats"], (q["kind"], a["stats"], b["stats"])
            assert np.array_equal(a["inliers"], b["inliers"]) and np.array_equal(a["model"], b["model"]), q["kind"]
