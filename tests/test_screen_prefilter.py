"""CPU tests of the streaming test k_screen runs for the Sampson kinds (relpose, fundamental): |C^| <= K
(scr::sampson_maybe_c, poselib_b200/csrc/screen_math.cuh, compiled for the host by tests/screen_prefilter_host.cc).

It replaces the full prefilter (scr::sampson_maybe: C^2 - alpha'|C^| - beta' <= thr' D^) and must
  * accept every correspondence sampson_maybe accepts, so that the queue pass sees every case it saw before;
  * reject only provable fp64 outliers;
  * add no case that sampson_point would count or flag, so count32 and border stay what they were;
  * keep the share of recorded (correspondence, model) pairs small on the headline data.
Data: C2 and C3 of the bench with the oracle's minimal solvers' models, the same in pixel units and with large offsets,
degenerate models and inputs, residuals within 1e-3 .. 1e-9 of the threshold, and correspondences on the corners of the
coordinate box at the threshold where sampson_maybe starts to accept them (where D^ reaches its box bound)."""
import ctypes as C
import os
import subprocess

import numpy as np
import plo_py as P
import pytest

from poselib_b200 import problem_generator as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "screen_prefilter_host.cc")
_P = C.POINTER(C.c_double)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("prefilter") / "_screen_prefilter_host.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", so])
    return C.CDLL(so)


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_P)


def prefilter(lib, pts, M, sq_thr):
    pts, pp = _d(pts)
    M, mp = _d(np.asarray(M).reshape(-1))
    out = np.zeros(8)
    lib.scr_prefilter(C.c_int(pts.shape[1]), pp, mp, C.c_double(sq_thr), out.ctypes.data_as(_P))
    return dict(lost=int(out[0]), rejected_inliers=int(out[1]), changed=int(out[2]), maybe=int(out[3]),
                maybe_c=int(out[4]), d_over_dmax=out[5], d_over_g=out[6], K=out[7])


def check(lib, pts, M, sq_thr):
    r = prefilter(lib, pts, M, sq_thr)
    assert r["lost"] == 0 and r["rejected_inliers"] == 0 and r["changed"] == 0, r
    assert r["maybe_c"] >= r["maybe"], r
    assert r["d_over_dmax"] <= 1.0, r
    return r


def sample_models(solver, x1, x2, k, n_samples, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_samples):
        idx = rng.choice(len(x1), k, replace=False)
        out.extend(solver(x1[idx], x2[idx]))
    return out


def bearings(x):
    h = np.c_[x, np.ones(len(x))]
    return h / np.linalg.norm(h, axis=1, keepdims=True)


def test_c2_minimal_models(lib):
    """The headline data (C2, normalised coordinates, 1 px) with the 5-point solver's models of random samples: no case
    is lost, and the recorded share stays within a small multiple of that of the full prefilter."""
    p = G.config_c2(0)
    x1, x2 = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
    models = sample_models(lambda a, b: P.relpose_5pt_E(bearings(a), bearings(b)), x1, x2, 5, 400, 11)
    assert len(models) > 1000
    pts = np.vstack([x1.T, x2.T])
    sq_thr = (1.0 / G.FOCAL) ** 2
    maybe = maybe_c = 0
    for E in models:
        r = check(lib, pts, E, sq_thr)
        maybe += r["maybe"]
        maybe_c += r["maybe_c"]
    pairs = len(models) * pts.shape[1]
    # 0.32 % and 0.96 % of the pairs for this seed: a few more cases for the queue pass, against a streaming test of
    # half the instructions
    assert 0.001 < maybe / pairs < 0.005 and maybe_c < 3.5 * maybe, (maybe / pairs, maybe_c / pairs)


def test_c3_minimal_models(lib):
    """C3 (fundamental, pixel coordinates, 1 px) with the 7-point solver's models."""
    p = G.config_c3(0)
    x1, x2 = p["x1"], p["x2"]
    models = sample_models(lambda a, b: P.relpose_7pt(np.c_[a, np.ones(7)], np.c_[b, np.ones(7)]), x1, x2, 7, 150, 12)
    assert len(models) > 150
    pts = np.vstack([x1.T, x2.T])
    for F in models:
        check(lib, pts, F / np.linalg.norm(F), 1.0)


@pytest.mark.parametrize("offset", [0.0, 1e3, 1e5])
def test_pixel_units_and_large_offsets(lib, offset):
    """The C2 scene in pixels (F = K^-T E K^-1), shifted by offset pixels in both images (F' = T^-T F T^-1): the box grows,
    fp32 loses the residual, and the test must still keep every case."""
    rng = np.random.default_rng(int(offset) + 5)
    p = G.relpose_problem(3000, 0.4, config_id=36, problem_idx=0)
    Kinv = np.diag([1 / G.FOCAL, 1 / G.FOCAL, 1.0])
    T = np.array([[1, 0, offset], [0, 1, offset], [0, 0, 1.0]])
    Tinv = np.linalg.inv(T)
    pts = np.vstack([p["x1"].T, p["x2"].T]) + offset
    for s in (0.0, 1e-4, 1e-2, 0.3):
        R = small_rot(rng, s) @ p["R_gt"] if s else p["R_gt"]
        t = p["t_gt"] + rng.normal(0, s, 3)
        F = Tinv.T @ Kinv.T @ essential(R, t / np.linalg.norm(t)) @ Kinv @ Tinv
        for thr in (1.0, 0.1, 12.0):
            check(lib, pts, F / np.linalg.norm(F), thr * thr)


def test_degenerate_models_and_inputs(lib):
    rng = np.random.default_rng(9)
    pts = rng.uniform(-0.8, 0.8, (4, 3000))
    for M in (np.zeros(9), np.r_[np.zeros(8), 1.0], np.r_[1e-30, np.zeros(8)], np.full(9, 1e18), np.full(9, 1e30),
              rng.normal(0, 1e-12, 9), np.r_[np.nan, rng.normal(0, 1, 8)], np.r_[np.inf, rng.normal(0, 1, 8)]):
        for thr in (1e-6, 1e-12, 0.0, 1e6, 1e40):
            r = prefilter(lib, pts, M, thr)
            assert r["lost"] == 0 and r["rejected_inliers"] == 0, (M[:2], thr, r)
    r = prefilter(lib, pts, np.full(9, 1e30), 1e-6)
    assert r["K"] == np.inf and r["maybe_c"] == pts.shape[1]  # K does not fit: every pair goes to sampson_point
    bad = pts.copy()
    bad[1, 5] = np.nan
    bad[2, 9] = np.inf
    E = rng.normal(0, 1, 9)
    r = prefilter(lib, bad, E, 1e-6)
    assert r["lost"] == 0 and r["rejected_inliers"] == 0, r


def test_residuals_on_the_threshold(lib):
    """Thousands of correspondences whose Sampson residual is within 1e-3 ... 1e-9 (relative) of the threshold."""
    rng = np.random.default_rng(7)
    p = G.relpose_problem(2000, 1.0, config_id=34, problem_idx=0)
    E = essential(p["R_gt"], p["t_gt"])
    x1, x2 = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
    thr = 1.0 / G.FOCAL
    n = len(x1)
    l = np.c_[x1, np.ones(n)] @ E.T
    nrm = l[:, :2] / np.linalg.norm(l[:, :2], axis=1, keepdims=True)
    for eps_mag in (1e-3, 1e-5, 1e-7, 1e-9):
        x2p = x2.copy()
        target = thr * (1 + rng.choice([-1, 1], n) * eps_mag * rng.uniform(0.1, 1, n))
        for _ in range(60):  # fixed-point iteration on the signed Sampson distance
            h2 = np.c_[x2p, np.ones(n)]
            Cc = np.einsum("ij,ij->i", h2, l)
            Ex2 = h2 @ E
            den = np.sqrt(l[:, 0] ** 2 + l[:, 1] ** 2 + Ex2[:, 0] ** 2 + Ex2[:, 1] ** 2)
            r = Cc / den
            x2p += ((np.sign(r) * target - r) * (den / np.linalg.norm(l[:, :2], axis=1)))[:, None] * nrm
        check(lib, np.vstack([x1.T, x2p.T]), E, thr * thr)


def test_box_corners_at_the_acceptance_threshold(lib):
    """Models stored exactly in fp32 and correspondences on the corners of the coordinate box, where D reaches its box
    bound G and the fp32 D^ can exceed it: K must cover the rounding of D^ (D^ <= Dmax), and at the smallest threshold
    at which sampson_maybe accepts a corner correspondence, sampson_maybe_c must accept it too."""
    rng = np.random.default_rng(21)
    over_g = 0.0
    closest = 0.0
    for trial in range(40):
        M = rng.normal(0, 1, 9).astype(np.float32).astype(np.float64)
        if trial % 2 == 0:  # every |e_r|, |f_c| reaches its box bound at the corner (+, +, +, +): D = G there
            M = np.abs(M)
        box = rng.uniform(0.2, 2.0, 4).astype(np.float32).astype(np.float64)
        signs = np.array(np.meshgrid(*[[-1.0, 1.0]] * 4)).reshape(4, -1)
        pts = signs * box[:, None]  # all 16 corners
        jit = rng.uniform(0.9, 1.0, (4, 48)).astype(np.float32).astype(np.float64) * rng.choice([-1.0, 1.0], (4, 48))
        pts = np.hstack([pts, jit * box[:, None]])  # and points inside the box
        r = check(lib, pts, M, 1e-3)
        over_g = max(over_g, r["d_over_g"])
        pts_, pp = _d(pts)
        M_, mp = _d(M)
        out = np.zeros(2)
        lib.scr_prefilter_edge(C.c_int(pts_.shape[1]), pp, mp, C.c_double(1e4), out.ctypes.data_as(_P))
        assert out[0] == 0, (trial, out)
        closest = max(closest, out[1])
    # the sets do reach the region the rounding terms are for: some corner D^ is above the exact box bound G, so a K
    # from G alone would not hold, and |C^| comes within 1e-3 of K
    assert over_g > 1.0, over_g
    assert closest > 0.999, closest


# ---- helpers ---------------------------------------------------------------------------------------------------------
def essential(R, t):
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    return tx @ R


def small_rot(rng, s):
    w = rng.normal(0, s, 3)
    th = np.linalg.norm(w)
    k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
