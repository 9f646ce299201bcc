"""GPU tests (-m gpu) of the device-side round control (csrc/control.cu): the device sampler against the engine's host
sampler — which tests/test_ref_pins.py pins bit for bit to robust/sampling.cc compiled in place — for uniform and PROSAC
sampling, tiny point sets (most samples reject duplicates), state carried across rounds of every size."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cabi():
    from poselib_b200 import cabi as c
    if c.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    c.set_device(0)
    return c


@pytest.mark.parametrize("n,k", [(10000, 5), (200, 3), (5000, 7), (20000, 4), (7, 7), (8, 7), (5, 5), (3, 3), (12, 4),
                                 (37, 5), (1 << 20, 7)])
@pytest.mark.parametrize("seed", [0, 1, 0xdeadbeefcafe])
def test_uniform_sampler_equals_host_sampler(cabi, n, k, seed):
    opt = cabi.RansacOpt(seed=seed)
    iters = 3000
    host = cabi.host_sample_table(n, k, opt, iters)
    for rnd in (1, 31, 32, 33, 1000, 4096):
        dev = cabi.device_sample_table(n, k, opt, iters, round_size=rnd)[0]
        assert np.array_equal(dev, host), (n, k, seed, rnd, np.argwhere((dev != host).any(axis=1))[:3])


def test_many_samplers_in_one_launch(cabi):
    iters, count = 2000, 37
    dev = cabi.device_sample_table(10000, 5, cabi.RansacOpt(seed=100), iters, round_size=512, count=count)
    for j in range(count):
        host = cabi.host_sample_table(10000, 5, cabi.RansacOpt(seed=100 + j), iters)
        assert np.array_equal(dev[j], host), j


@pytest.mark.parametrize("n,k,max_prosac", [(5000, 7, 100000), (500, 7, 3000), (200, 3, 1000), (64, 5, 200), (9, 7, 50),
                                            (7, 7, 10), (2000, 4, 1), (2000, 4, 0), (300, 5, 2)])
@pytest.mark.parametrize("seed", [0, 7])
def test_prosac_sampler_equals_host_sampler(cabi, n, k, max_prosac, seed):
    opt = cabi.RansacOpt(seed=seed, progressive_sampling=1, max_prosac_iterations=max_prosac)
    iters = 6000  # past max_prosac for most cases: the sampler falls back to uniform draws (sampling.cc:86,102)
    host = cabi.host_sample_table(n, k, opt, iters)
    for rnd in (1, 32, 257, 4096):
        dev = cabi.device_sample_table(n, k, opt, iters, round_size=rnd)[0]
        assert np.array_equal(dev, host), (n, k, max_prosac, seed, rnd, np.argwhere((dev != host).any(axis=1))[:3])
    os.environ["PLB_PROSAC_SEQUENTIAL"] = "1"  # the step-by-step subset growth instead of the closed form
    try:
        dev = cabi.device_sample_table(n, k, opt, iters, round_size=300)[0]
    finally:
        del os.environ["PLB_PROSAC_SEQUENTIAL"]
    assert np.array_equal(dev, host)


def test_c3_prosac_full_length(cabi):
    opt = cabi.RansacOpt(seed=0, progressive_sampling=1, max_prosac_iterations=100000)
    host = cabi.host_sample_table(5000, 7, opt, 100000)
    dev = cabi.device_sample_table(5000, 7, opt, 100000, round_size=16384)[0]
    assert np.array_equal(dev, host)


# ---- relpose_8pt / essential_matrix_8pt on the device (solvers/relpose_8pt.cc:52-95, SURVEY §8f row N4) -----------------
def _eight_scene(rng, n, noise):
    """n exact bearing pairs of a random relative pose (|t| = 1), optionally with noise on the image coordinates."""
    w = rng.normal(0, 0.4, 3)
    th = np.linalg.norm(w)
    k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
    t = rng.normal(0, 1, 3)
    t /= np.linalg.norm(t)
    X1 = np.zeros((0, 3))
    while len(X1) < n:  # points in front of both cameras
        c = np.c_[rng.uniform(-0.7, 0.7, (4 * n, 2)), np.ones(4 * n)] * rng.uniform(2.0, 8.0, (4 * n, 1))
        X1 = np.vstack([X1, c[(c @ R.T + t)[:, 2] > 0.5]])
    X1 = X1[:n]
    X2 = X1 @ R.T + t
    a = np.c_[X1[:, :2] / X1[:, 2:3] + rng.normal(0, noise, (n, 2)) if noise else X1[:, :2] / X1[:, 2:3], np.ones(n)]
    b = np.c_[X2[:, :2] / X2[:, 2:3] + rng.normal(0, noise, (n, 2)) if noise else X2[:, :2] / X2[:, 2:3], np.ones(n)]
    return (a / np.linalg.norm(a, axis=1, keepdims=True), b / np.linalg.norm(b, axis=1, keepdims=True),
            {"R_gt": R, "t_gt": t})


@pytest.mark.parametrize("n", [8, 9, 12, 50, 100, 1000])
def test_eight_point_solver_matches_oracle(cabi, n):
    import plo_py as P
    rng = np.random.default_rng(n)
    count = 12
    x1 = np.zeros((count, n, 3))
    x2 = np.zeros((count, n, 3))
    for i in range(count):
        x1[i], x2[i], _ = _eight_scene(rng, n, 0.0 if i % 2 == 0 else 1e-3)
    E = cabi.essential_matrix_8pt_batch(x1, x2)
    poses, npose = cabi.relpose_8pt_batch(x1, x2)
    for i in range(count):
        Eo = P.essential_matrix_8pt(x1[i], x2[i])
        s = np.sign(np.sum(E[i] * Eo)) or 1.0  # the nullspace / eigenvector is defined up to sign
        assert np.allclose(s * E[i], Eo, rtol=0, atol=1e-9 * max(1.0, np.abs(Eo).max())), (n, i, E[i], Eo)
        po = P.relpose_8pt(x1[i], x2[i])
        assert npose[i] == len(po), (n, i, npose[i], len(po))
        for k in range(len(po)):  # same order: motion_from_essential enumerates (R1,t), (R1,-t), (R2,-t), (R2,t)
            d = min(np.abs(poses[i, k] - po[k]).max(), np.abs(np.r_[-poses[i, k, :4], poses[i, k, 4:]] - po[k]).max())
            assert d < 1e-8, (n, i, k, poses[i, k], po[k])


def test_eight_point_pyapi(cabi):
    from poselib_b200 import pyapi
    rng = np.random.default_rng(3)
    x1, x2, p = _eight_scene(rng, 40, 0.0)
    E = pyapi.essential_matrix_8pt(x1, x2)
    res = np.abs(np.einsum("ni,ij,nj->n", x2, E, x1))
    assert res.max() < 1e-9
    poses = pyapi.relpose_8pt(x1, x2)
    assert len(poses) >= 1
    R_gt, t_gt = p["R_gt"], p["t_gt"]
    assert min(np.abs(q.R - R_gt).max() + np.abs(q.t / np.linalg.norm(q.t) - t_gt).max() for q in poses) < 1e-7
