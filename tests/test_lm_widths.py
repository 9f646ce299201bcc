"""The Levenberg-Marquardt kernel (k_lm) at every cluster width, on empty slices and across tile boundaries.

k_lm splits a job over a cluster of 1, 2, 4 or 8 CTAs (lm_cluster_size: correspondences per CTA, PLB_LM_PER_CTA, default
2048; narrowed as the job count of a launch grows), gives CTA r the slice [r*chunk, (r+1)*chunk) with chunk rounded up
to 32 (so the last CTAs of a wide cluster over few points own nothing), sums the CTA partial sums through DSMEM, and in
the camera refiners stages 256 points per pass in a shared-memory tile.  The width of a launch follows the largest
problem of the launch.

  * CPU: the exactly summed cost below restates the per-point robust losses of every refiner (math.fsum, divided by
    max(1, rows)); it is held to the oracle's own initial costs.
  * GPU, natural widths: every refine entry point at sizes around the width boundaries (1 | 2048 | 2049 ... 6144 | 6145
    ... 14336 | 14337) and the tile edges (255, 256, 257), against the oracle (fixed-camera kinds) and, for every call,
    bundle_stats[1] / [2] against the exact sum at the start parameters and at the returned pose and cameras.  The camera
    refiners at 2, 4 and 8 CTAs, and two inliers-first estimates per camera refiner whose polish leaves CTAs 3-7 with
    empty compacted lists, against the reference's own results (tests/golden/reference_lm_widths.json, written by
    tests/golden/make_lm_widths_golden.py; on the CPU the fixture's grid, and where the reference is mounted its
    reproduction bit for bit).
  * GPU, forced widths: the same inputs in child processes with PLB_LM_PER_CTA=1 (every job of 8 or more points on 8
    CTAs, most of them empty at n = 33) and PLB_LM_PER_CTA=1000000 (one CTA, up to 157 tiles), against the in-process
    default: identical iterations, the exact-sum bar in every setting, models and cameras within CROSS_WIDTH_RTOL; RANSAC
    through the LO kernel at every width against the oracle's trajectory.
  * GPU, batches: a batch of PnP problems with camera refinement, whose width follows its largest member, against the
    single calls.
  * GPU, no points: every refine entry point with n = 0 writes what the oracle returns."""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (os.path.join(HERE, "golden"), HERE, ROOT, os.path.join(ROOT, "oracle")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import make_camera_models_golden as MC  # noqa: E402
import make_intrinsics_golden as MG  # noqa: E402
import make_lm_widths_golden as MW  # noqa: E402
import make_relpose_intrinsics_golden as MR  # noqa: E402
import plo_py as P  # noqa: E402
from poselib_b200 import problem_generator as G  # noqa: E402

try:
    from poselib_b200 import cabi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)

# Correspondence counts around the width boundaries of a single call (per_cta 2048: 1 CTA up to 2048, 2 up to 6144, 4 up
# to 14336, 8 above) and the tile edges of the camera refiners (256 points per pass).  40000 gives every CTA of an 8-wide
# cluster 5000 points, 20 tiles.
SIZES = [1, 5, 255, 256, 257, 2048, 2049, 6144, 6145, 14336, 14337, 40000]
CAM_SIZES = MW.CAM_SIZES  # the camera refiners against the reference's results (tests/golden/reference_lm_widths.json)
BOUNDARY_SIZES = [n for n in SIZES if n not in CAM_SIZES]  # ... and at the other sizes against the exact sums only
# Relative bar of bundle_stats[1] / [2] against the exactly summed cost.  A sequential fp64 sum of n non-negative terms
# is within n * 2^-53 of the exact sum (4.4e-12 at 40000); per-term differences of the camera and pose arithmetic are
# far below that.
EXACT_RTOL = 1e-11
# ... or within EXACT_FLOOR of the start cost: with 1 or 5 points a refiner fits the data exactly and its final cost is
# rounding of the residuals themselves (1e-15 px^2 from a start of ~30 px^2), which no summation order explains.  A dropped
# or doubled point of 40000 moves a cost by ~1e-5 of it.
EXACT_FLOOR = 1e-14
# Models and cameras of the same input at two cluster widths (only the order of the cost and normal-equation sums
# differs): the parameter bar of test_camera_models.py against the reference (PAIR_PARAM_RTOL).  Two views leave the
# parameters of fisheye and division cameras weakly constrained, so their stopping point moves with the summation order.
# Measured on an H100 80GB HBM3 (400 W power limit): 1.0e-7, camera parameters of the SIMPLE_RADIAL_FISHEYE +
# SIMPLE_DIVISION pair at 257 points, eight CTAs against one; 1.24e-8 for an OPENCV pair.  The batch of
# test_estimate_batch_width_follows_its_largest_problem: 2.1e-16.
CROSS_WIDTH_RTOL = 1e-6
# Fixed-camera cases whose final cost and model are not held to the oracle's (iterations, the initial cost and both exact
# sums still are): homography with the TRIVIAL loss at 14336 points and more, where gross outliers with residuals of ~1e3
# and 25 unconverged iterations make the oracle's own result move with the order of the points (a permutation moves its
# model by ~10 %), and the fundamental refiner on 5 points, which it fits exactly: both costs are rounding (~1e-22).
NO_ORACLE_RESULT = {("homography", n, "TRIVIAL") for n in (14336, 14337, 40000)} | \
    {("fundamental", 5, loss) for loss in ("TRIVIAL", "CAUCHY")}
FORCED = {"one_cta_per_point": "1", "one_cta": "1000000"}


# ---- exactly summed cost ---------------------------------------------------------------------------------------------
def _loss(loss, scale, r2):
    """robust/robust_loss.h:41-67 (oracle/plo_optim.cc Loss::loss)."""
    sq = scale * scale
    if loss == "TRUNCATED":
        return np.minimum(r2, sq)
    if loss == "HUBER":
        r = np.sqrt(r2)
        return np.where(r <= scale, r2, scale * (2.0 * r - scale))
    if loss == "CAUCHY":
        return sq * np.log1p(r2 * (1.0 / sq))
    return r2


def _total(loss, scale, r2, rows):
    """NormalAccumulator::get_residual (jacobian_accumulator.h:46-58): the loss sum over max(1, residual_count)."""
    return math.fsum(_loss(loss, scale, np.asarray(r2, dtype=np.float64)).tolist()) / max(1.0, float(rows))


def _rot(q):
    return G.quat_to_rotmat(np.asarray(q[:4], dtype=np.float64))


def _essential(pose):
    t = pose[4:7]
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ _rot(pose)


def _project(cam, Z):
    """Camera::project of camera-frame points: the null camera (Z / Z_2), the oracle's camera functions for the models
    it has (0-4), the synthesis projection of make_camera_models_golden.py for the fisheye and division models."""
    if cam is None:
        return Z[:, :2] / Z[:, 2:3]
    model, params = cam
    if MC.MODEL_IDS[model] <= 4:
        return P.camera_project_with_jac((model, list(params)), Z)[2]
    return MC.project(MC.MODEL_IDS[model], np.asarray(params, dtype=np.float64), Z)


def pnp_cost(pose, x, X, loss, scale, cam=None):
    """AbsolutePoseRefiner::compute_residual (optim/absolute.h:49-66): points behind the camera (Z_2 < 0) are skipped and
    not counted."""
    Z = np.asarray(X) @ _rot(pose).T + np.asarray(pose[4:7])
    keep = ~(Z[:, 2] < 0)
    r = _project(cam, Z[keep]) - np.asarray(x)[keep] if keep.any() else np.zeros((0, 2))
    return _total(loss, scale, (r * r).sum(1), int(keep.sum()))


def _sampson_r2(F, x1, x2):
    """Sampson residual of relative.h:98-105 / fundamental.h:53-60 (oracle sampson_resid), squared."""
    h1 = np.c_[x1, np.ones(len(x1))]
    h2 = np.c_[x2, np.ones(len(x2))]
    Ex1 = h1 @ F.T
    Cv = (h2 * Ex1).sum(1)
    n1 = Ex1[:, 0] ** 2 + Ex1[:, 1] ** 2
    Etx2 = h2 @ F
    r = Cv / np.sqrt(n1 + (Etx2[:, 0] ** 2 + Etx2[:, 1] ** 2))
    return r * r


def relpose_cost(pose, x1, x2, loss, scale):
    return _total(loss, scale, _sampson_r2(_essential(pose), x1, x2), len(x1))


def fundamental_cost(F, x1, x2, loss, scale):
    return _total(loss, scale, _sampson_r2(np.asarray(F), x1, x2), len(x1))


def factorised(F):
    """The matrix the fundamental refiner's factorisation reconstructs (optim_utils.h:57-82, fundamental.h:40-51):
    U diag(1, s1 / s0, 0) V^T, up to the sign the cost does not see."""
    U, s, Vt = np.linalg.svd(np.asarray(F, dtype=np.float64))
    return np.outer(U[:, 0], Vt[0]) + (s[1] / s[0]) * np.outer(U[:, 1], Vt[1])


def homography_cost(H, x1, x2, loss, scale):
    """HomographyRefiner (optim/homography.h:60-84): the forward and the backward transfer error, two rows per point."""
    H = np.asarray(H, dtype=np.float64)
    Gm = np.linalg.inv(H) * np.linalg.det(H)  # adj(H); the projection divides the scale out
    h1, h2 = np.c_[x1, np.ones(len(x1))], np.c_[x2, np.ones(len(x2))]
    f = h1 @ H.T
    b = h2 @ Gm.T
    rf = f[:, :2] / f[:, 2:3] - x2
    rb = b[:, :2] / b[:, 2:3] - x1
    return _total(loss, scale, np.r_[(rf * rf).sum(1), (rb * rb).sum(1)], 2 * len(x1))


def tangent_cost(pose, d1, d2, M1, M2, loss, scale):
    """FixCameraRelativePoseRefiner / CameraRelativePoseRefiner residual (optim/relative.h:181-193, 289-330):
    C = d2^T E d1 over the norm of its gradient through the unprojection Jacobians M1, M2 [n, 3, 2]."""
    E = _essential(pose)
    Ed1 = d1 @ E.T
    Cv = (d2 * Ed1).sum(1)
    j1 = np.einsum("nj,jk,nki->ni", d2, E, M1)  # d2^T E M1
    j2 = np.einsum("nj,kj,nki->ni", d1, E, M2)  # d1^T E^T M2
    r = Cv / np.sqrt((j2 ** 2).sum(1) + (j1 ** 2).sum(1))
    return _total(loss, scale, r * r, len(d1))


def pair_cost(pose, x1, x2, cam1, cam2, loss, scale):
    """Tangent Sampson cost of pixels through two cameras of the oracle's models (0-4)."""
    d1, M1 = P.camera_unproject_with_jac((cam1[0], list(cam1[1])), x1)
    d2, M2 = P.camera_unproject_with_jac((cam2[0], list(cam2[1])), x2)
    return tangent_cost(pose, d1, d2, M1, M2, loss, scale)


def _rel(a, b, start):
    """Relative difference of a cost to its exact sum b; 0 within EXACT_FLOOR of the exact start cost."""
    return 0.0 if abs(a - b) <= EXACT_FLOOR * abs(start) else abs(a - b) / max(abs(b), 1e-300)


# ---- problems --------------------------------------------------------------------------------------------------------
def _start(kind, p, seed):
    rng = np.random.default_rng(seed)
    if kind in ("pnp", "relpose"):
        q = p["q_gt"] + rng.normal(0, 0.01, 4)
        t = p["t_gt"] + rng.normal(0, 0.02, 3)
        return np.r_[q / np.linalg.norm(q), t / (np.linalg.norm(t) if kind == "relpose" else 1.0)]
    if kind == "fundamental":
        t = p["t_gt"]
        E = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ p["R_gt"] + rng.normal(0, 0.01, (3, 3))
        return E / np.linalg.norm(E)
    return p["H_gt"] / np.linalg.norm(p["H_gt"]) + rng.normal(0, 0.002, (3, 3))


def fixed_problem(kind, n):
    """Calibrated inputs of the fixed-camera refiners (70 % inliers), a perturbed start model and the loss scale."""
    if kind == "pnp":
        p = G.abspose_problem(n, 0.7, 61, n)
        return p["x"] / G.FOCAL, p["X"], _start(kind, p, n), 12.0 / G.FOCAL
    if kind == "homography":
        p = G.homography_problem(n, 0.7, 64, n)
        return p["x1"] / G.FOCAL, p["x2"] / G.FOCAL, _start(kind, p, n), 2.0 / G.FOCAL
    p = G.relpose_problem(n, 0.7, 62, n)
    return p["x1"] / G.FOCAL, p["x2"] / G.FOCAL, _start(kind, p, n), 2.0 / G.FOCAL


def fixed_cost(kind, model, a, b, loss, scale):
    return {"pnp": pnp_cost, "relpose": relpose_cost, "fundamental": fundamental_cost,
            "homography": homography_cost}[kind](model, a, b, loss, scale)


# PnP cameras and tangent-Sampson pairs (the same camera on both images, and one mixed pair) of the fixture
PNP_CAMERAS, PAIRS = MW.PNP_CAMERAS, MW.PAIRS
_model_name = MW.model_name
pnp_camera_problem, pair_camera_problem = MW.pnp_problem, MW.pair_problem


def exact_camera(cam):
    """The camera functions of the exact cost are the oracle's (models 0-4) for tangent Sampson."""
    return MW.model_id(cam) <= 4


def _bopt(loss, scale, flags=0, max_iterations=100, relative_cost_tol=1e-8):
    return cabi.BundleOpt(max_iterations=max_iterations, loss_type=loss, loss_scale=scale, refine_intrinsics=flags,
                          relative_cost_tol=relative_cost_tol)


# ---- one refine call of each surface, results as plain lists ----------------------------------------------------------
def run_fixed(kind, n, loss, max_iterations=25):
    a, b, m0, scale = fixed_problem(kind, n)
    m, bs = cabi.refine(kind, m0, a, b, cabi.BundleOpt(max_iterations=max_iterations, loss_type=loss, loss_scale=scale))
    return {"bs": list(bs), "model": np.asarray(m).ravel().tolist()}


def check_fixed_exact(kind, n, loss, r):
    a, b, m0, scale = fixed_problem(kind, n)
    start = factorised(m0) if kind == "fundamental" else m0
    model = np.asarray(r["model"]).reshape(3, 3) if kind in ("fundamental", "homography") else np.asarray(r["model"])
    c0, c1 = fixed_cost(kind, start, a, b, loss, scale), fixed_cost(kind, model, a, b, loss, scale)
    assert _rel(r["bs"][1], c0, c0) <= EXACT_RTOL, (kind, n, loss, r["bs"][1], c0)
    assert _rel(r["bs"][2], c1, c0) <= EXACT_RTOL, (kind, n, loss, r["bs"][2], c1)


def ts_fixed_problem(n):
    x1, x2, pose0, c1, c2 = MR.pair_problem(1, 1, n, 500 + n)
    return x1, x2, pose0, ("PINHOLE", c1), ("PINHOLE", c2)


def run_ts_fixed(n, loss, max_iterations=25):
    x1, x2, pose0, c1, c2 = ts_fixed_problem(n)
    pose, bs = cabi.refine_relpose_cameras(pose0, x1, x2, cabi.Camera(*c1), cabi.Camera(*c2),
                                           _bopt(loss, MR.LOSS_SCALE, max_iterations=max_iterations))
    return {"bs": list(bs), "model": list(pose)}


def check_ts_fixed_exact(n, loss, r):
    x1, x2, pose0, c1, c2 = ts_fixed_problem(n)
    c0 = pair_cost(pose0, x1, x2, c1, c2, loss, MR.LOSS_SCALE)
    for cost, pose in ((r["bs"][1], pose0), (r["bs"][2], np.asarray(r["model"]))):
        ref = pair_cost(pose, x1, x2, c1, c2, loss, MR.LOSS_SCALE)
        assert _rel(cost, ref, c0) <= EXACT_RTOL, (n, loss, cost, ref)


def _pnp_seed(cam, n, flags, loss):
    """The fixture's seed on its grid, else one of the size."""
    return MW.bundle_seed(cam, n, flags, loss) if n in CAM_SIZES and flags in MW.FLAGS and loss in MW.LOSSES \
        else 95000 + n


def run_pnp_camera(cam, n, flags, loss, max_iterations=100):
    x, X, pose0, p0 = pnp_camera_problem(cam, n, _pnp_seed(cam, n, flags, loss))
    pose, params, bs = cabi.refine_image(pose0, x, X, cabi.Camera(_model_name(cam), tuple(p0)),
                                         _bopt(loss, MG.LOSS_SCALE, flags, max_iterations))
    return {"bs": list(bs), "model": list(pose), "cams": [list(params)]}


def check_pnp_camera_exact(cam, n, flags, loss, r):
    x, X, pose0, p0 = pnp_camera_problem(cam, n, _pnp_seed(cam, n, flags, loss))
    name = _model_name(cam)
    c0 = pnp_cost(pose0, x, X, loss, MG.LOSS_SCALE, (name, p0))
    for cost, pose, params in ((r["bs"][1], pose0, p0), (r["bs"][2], np.asarray(r["model"]), r["cams"][0])):
        ref = pnp_cost(pose, x, X, loss, MG.LOSS_SCALE, (name, params))
        assert _rel(cost, ref, c0) <= EXACT_RTOL, (cam, n, flags, loss, cost, ref)


def _pair_seed(pair, n, flags, loss):
    return MW.refine_seed(pair, n, flags, loss) if n in CAM_SIZES and flags in MW.FLAGS and loss in MW.LOSSES \
        else 99000 + n


def run_pair_camera(pair, n, flags, loss, max_iterations=100, seed=None):
    seed = _pair_seed(pair, n, flags, loss) if seed is None else seed
    x1, x2, pose0, c1, c2 = pair_camera_problem(pair, n, seed)
    cams = [cabi.Camera(_model_name(c), tuple(p)) for c, p in zip(pair, (c1, c2))]
    pose, p1, p2, bs = cabi.refine_relpose_pair(pose0, x1, x2, cams[0], cams[1],
                                                _bopt(loss, MC.PAIR_LOSS_SCALE, flags, max_iterations))
    return {"bs": list(bs), "model": list(pose), "cams": [list(p1), list(p2)]}


def check_pair_camera_exact(pair, n, flags, loss, r, seed=None):
    if not all(exact_camera(c) for c in pair):
        return
    seed = _pair_seed(pair, n, flags, loss) if seed is None else seed
    x1, x2, pose0, c1, c2 = pair_camera_problem(pair, n, seed)
    names = [_model_name(c) for c in pair]
    c0 = pair_cost(pose0, x1, x2, (names[0], c1), (names[1], c2), loss, MC.PAIR_LOSS_SCALE)
    for cost, pose, p1, p2 in ((r["bs"][1], pose0, c1, c2),
                               (r["bs"][2], np.asarray(r["model"]), r["cams"][0], r["cams"][1])):
        ref = pair_cost(pose, x1, x2, (names[0], p1), (names[1], p2), loss, MC.PAIR_LOSS_SCALE)
        assert _rel(cost, ref, c0) <= EXACT_RTOL, (pair, n, flags, loss, cost, ref)


# ---- CPU: the exact cost is the reference's cost ---------------------------------------------------------------------
@pytest.mark.parametrize("loss", list(MG.LOSSES))
@pytest.mark.parametrize("kind", ["pnp", "relpose", "fundamental", "homography"])
def test_exact_cost_is_the_oracles_initial_cost(kind, loss):
    for n in (1, 257, 3000):
        a, b, m0, scale = fixed_problem(kind, n)
        _, bs = P.refine(kind, m0, a, b, P.BundleOpt(max_iterations=0, loss_type=loss, loss_scale=scale))
        start = factorised(m0) if kind == "fundamental" else m0
        c0 = fixed_cost(kind, start, a, b, loss, scale)
        assert _rel(bs[1], c0, c0) <= 1e-12, (kind, loss, n)


@pytest.mark.parametrize("loss", list(MG.LOSSES))
def test_exact_tangent_cost_is_the_oracles_initial_cost(loss):
    for n in (1, 257, 3000):
        x1, x2, pose0, c1, c2 = ts_fixed_problem(n)
        d1, M1 = P.camera_unproject_with_jac(c1, x1)
        d2, M2 = P.camera_unproject_with_jac(c2, x2)
        _, bs = P.refine_relpose_tangent(pose0, d1, d2, M1, M2,
                                         P.BundleOpt(max_iterations=0, loss_type=loss, loss_scale=MR.LOSS_SCALE))
        c0 = pair_cost(pose0, x1, x2, c1, c2, loss, MR.LOSS_SCALE)
        assert _rel(bs[1], c0, c0) <= 1e-12, (loss, n)


def test_pnp_exact_cost_skips_points_behind_the_camera():
    X = np.array([[0.0, 0.0, 2.0], [0.1, 0.0, -1.0], [0.0, 0.2, 1.0]])
    x = np.array([[0.01, 0.0], [0.0, 0.0], [0.0, 0.19]])
    pose = np.array([1.0, 0, 0, 0, 0, 0, 0])
    _, bs = P.refine("pnp", pose, x, X, P.BundleOpt(max_iterations=0, loss_type="TRIVIAL"))
    assert pnp_cost(pose, x, X, "TRIVIAL", 1.0) == bs[1]
    assert np.isclose(bs[1], (0.01 ** 2 + 0.01 ** 2) / 2, rtol=1e-14, atol=0)  # two rows, not three


def test_fixed_refiner_results_without_a_reference_are_the_listed_ones():
    """NO_ORACLE_RESULT is needed: on each listed case the oracle's model moves with the order of the points
    (homography) or is below 1e-12 of the start cost (an exact fit), and a neighbouring size of each is stable."""
    def run(kind, n, loss, perm=None):
        a, b, m0, scale = fixed_problem(kind, n)
        p = np.arange(n) if perm is None else np.random.default_rng(n).permutation(n)
        return P.refine(kind, m0, a[p], b[p], P.BundleOpt(max_iterations=25, loss_type=loss, loss_scale=scale))
    for kind, n, loss in NO_ORACLE_RESULT:
        om, os_ = run(kind, n, loss)
        if kind == "homography":
            pm = run(kind, n, loss, perm=True)[0]  # moves by more than the model bar of the comparison
            assert min(np.abs(pm - om).max(), np.abs(pm + om).max()) > 1e-6 * np.abs(om).max(), (kind, n, loss)
        else:
            assert os_[2] < 1e-12 * os_[1], (kind, n, loss, os_[:3])
    om, os_ = run("homography", 6145, "TRIVIAL")
    assert np.isclose(run("homography", 6145, "TRIVIAL", perm=True)[1][2], os_[2], rtol=1e-9, atol=0)
    assert not run("fundamental", 255, "TRIVIAL")[1][2] < 1e-12 * run("fundamental", 255, "TRIVIAL")[1][1]


def test_sizes_straddle_every_width_and_tile_edge():
    def width(n, per_cta=2048):
        c = min(8, max(1, -(-n // per_cta)))
        return 4 if 4 < c < 8 else 2 if c == 3 else c
    widths = [width(n) for n in SIZES]
    for w in (1, 2, 4, 8):
        assert w in widths
    for lo, hi in ((2048, 2049), (6144, 6145), (14336, 14337)):
        assert width(lo) < width(hi) and lo in SIZES and hi in SIZES
    assert width(40000) == 8 and -(-40000 // 8) // 256 >= 19  # every CTA walks about 20 tiles
    for n in (33, 257):  # PLB_LM_PER_CTA=1: 8 CTAs, chunk rounded up to 32, the last CTAs own nothing
        chunk = ((-(-n // 8)) + 31) & ~31
        assert sum(1 for r in range(8) if r * chunk >= n) == {33: 6, 257: 3}[n]


# ---- GPU: natural widths --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("loss", ["TRIVIAL", "CAUCHY", "TRUNCATED"])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", ["pnp", "relpose", "fundamental", "homography"])
def test_fixed_refiners_match_oracle_at_every_width(kind, n, loss):
    if loss == "TRUNCATED" and n not in (257, 6145, 40000):
        pytest.skip("TRUNCATED: one size per tile edge and width")
    a, b, m0, scale = fixed_problem(kind, n)
    r = run_fixed(kind, n, loss)
    bo = P.BundleOpt(max_iterations=25, loss_type=loss, loss_scale=scale)
    om, os_ = P.refine(kind, m0, a, b, bo)
    check_fixed_exact(kind, n, loss, r)
    assert int(r["bs"][0]) == int(os_[0]), (r["bs"], os_[:3])
    assert np.isclose(r["bs"][1], os_[1], rtol=1e-10, atol=0), (r["bs"], os_[:3])
    if (kind, n, loss) in NO_ORACLE_RESULT:  # the exact sums above hold the kernel's costs at its start and result
        return
    assert np.isclose(r["bs"][2], os_[2], rtol=1e-7, atol=0), (r["bs"], os_[:3])
    gm = np.asarray(r["model"]).reshape(np.shape(om))
    err = min(np.abs(gm - om).max(), np.abs(gm + om).max()) if gm.ndim == 2 else np.abs(gm - om).max()
    assert err < 1e-6 * max(1.0, np.abs(om).max()), (err, r["bs"], os_[:3])


@pytest.mark.gpu
@pytest.mark.parametrize("loss", ["TRIVIAL", "CAUCHY"])
@pytest.mark.parametrize("n", SIZES)
def test_tangent_sampson_fixed_cameras_match_oracle_at_every_width(n, loss):
    x1, x2, pose0, c1, c2 = ts_fixed_problem(n)
    r = run_ts_fixed(n, loss)
    d1, M1 = P.camera_unproject_with_jac(c1, x1)
    d2, M2 = P.camera_unproject_with_jac(c2, x2)
    om, os_ = P.refine_relpose_tangent(pose0, d1, d2, M1, M2,
                                       P.BundleOpt(max_iterations=25, loss_type=loss, loss_scale=MR.LOSS_SCALE,
                                                   relative_cost_tol=1e-8))
    check_ts_fixed_exact(n, loss, r)
    assert int(r["bs"][0]) == int(os_[0]), (r["bs"], os_[:3])
    assert np.isclose(r["bs"][1], os_[1], rtol=1e-10, atol=0)
    if n != 5:  # 5 points fix the 5 pose parameters exactly: both final costs are rounding (~1e-15 px^2)
        assert np.isclose(r["bs"][2], os_[2], rtol=1e-7, atol=0), (r["bs"], os_[:3])
    assert np.abs(np.asarray(r["model"]) - om).max() < 1e-6, (r["model"], om)


@pytest.mark.gpu
@pytest.mark.parametrize("loss", ["TRIVIAL", "CAUCHY"])
@pytest.mark.parametrize("flags", [1, 7])
@pytest.mark.parametrize("n", BOUNDARY_SIZES)
@pytest.mark.parametrize("cam", PNP_CAMERAS)
def test_pnp_camera_refiner_costs_are_exact_sums(cam, n, flags, loss):
    r = run_pnp_camera(cam, n, flags, loss)
    assert r["bs"][2] <= r["bs"][1], r["bs"]
    check_pnp_camera_exact(cam, n, flags, loss, r)


@pytest.mark.gpu
@pytest.mark.parametrize("loss", ["TRIVIAL", "CAUCHY"])
@pytest.mark.parametrize("flags", [1, 7])
@pytest.mark.parametrize("n", BOUNDARY_SIZES)
@pytest.mark.parametrize("pair", PAIRS)
def test_pair_camera_refiner_costs_are_exact_sums(pair, n, flags, loss):
    r = run_pair_camera(pair, n, flags, loss)
    assert r["bs"][2] <= r["bs"][1], r["bs"]
    assert all(np.all(np.isfinite(c)) for c in r["cams"]) and np.all(np.isfinite(r["model"]))
    check_pair_camera_exact(pair, n, flags, loss, r)


# ---- the fixture of the reference's camera refiners -------------------------------------------------------------------
GOLD = json.load(open(MW.OUT))
needs_reference = pytest.mark.skipif(
    not (MG.reference_available() and os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libplref2.so"))),
    reason="needs the reference checkout and oracle/_ref/libplref2.so")
# Bars against the fixture: those of test_intrinsics_refine.py (iterations exact, initial cost 1e-10, cost 1e-7, pose and
# parameters 1e-6; RANSAC stats and inlier masks exact)
INITIAL_COST_RTOL, COST_RTOL, MODEL_RTOL = 1e-10, 1e-7, 1e-6


def _close(a, b, rtol):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return a.shape == b.shape and np.all(np.abs(a - b) <= rtol * np.maximum(1.0, np.abs(b)))


def _mask(hexbits):
    return np.unpackbits(np.frombuffer(bytes.fromhex(hexbits), dtype=np.uint8))[:MW.ESTIMATE_N]


def test_fixture_covers_the_grid():
    assert sorted((c["camera"], c["n"], c["flags"], c["loss"]) for c in GOLD["bundle"]) == sorted(MW.bundle_cases())
    assert sorted(((c["camera1"], c["camera2"]), c["n"], c["flags"], c["loss"]) for c in GOLD["refine"]) == \
        sorted(MW.refine_cases())
    assert sorted((c["kind"], c["flags"]) for c in GOLD["estimate_cases"]) == sorted(MW.estimate_cases())
    assert all(c["iterations"] > 0 and c["cost"] < c["initial_cost"] for c in GOLD["bundle"] + GOLD["refine"])
    chunk = ((-(-MW.ESTIMATE_N // 8)) + 31) & ~31
    assert 2 * chunk < MW.ESTIMATE_INLIERS < 3 * chunk
    for c in GOLD["estimate_cases"]:  # the polish mask: inliers in CTAs 0-2 of an 8-wide cluster only
        m = _mask(c["inliers"])
        assert m[2 * chunk:MW.ESTIMATE_INLIERS].any() and not m[MW.ESTIMATE_INLIERS:].any(), (c["kind"], c["flags"])


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("ref_lm_widths"))
    return MC.build_client(d)


@needs_reference
def test_reference_reproduces_the_fixture_bitwise(ref):
    for c in GOLD["bundle"]:
        assert MW.ref_bundle_adjust(ref, c["camera"], c["n"], c["flags"], c["loss"]) == c, c
    for c in GOLD["refine"]:
        r = MW.ref_refine(ref, (c["camera1"], c["camera2"]), c["n"], c["flags"], c["loss"], c["seed"])
        assert r == c, c
    for c in GOLD["estimate_cases"]:
        assert MW.ref_estimate(ref, c["kind"], c["flags"], c["seed"]) == c, c


@pytest.mark.gpu
@pytest.mark.parametrize("loss", MW.LOSSES)
@pytest.mark.parametrize("n", CAM_SIZES)
@pytest.mark.parametrize("cam", PNP_CAMERAS)
def test_pnp_camera_refiner_matches_reference_at_every_width(cam, n, loss):
    for c in [c for c in GOLD["bundle"] if (c["camera"], c["n"], c["loss"]) == (cam, n, loss)]:
        r = run_pnp_camera(cam, n, c["flags"], loss)
        tag = (cam, n, c["flags"], loss)
        assert int(r["bs"][0]) == c["iterations"], (tag, r["bs"], c["iterations"])
        assert _close(r["bs"][1], c["initial_cost"], INITIAL_COST_RTOL), (tag, r["bs"], c["initial_cost"])
        assert _close(r["bs"][2], c["cost"], COST_RTOL), (tag, r["bs"], c["cost"])
        assert _close(r["model"], c["pose"], MODEL_RTOL), (tag, r["model"], c["pose"])
        assert _close(r["cams"][0], c["params"], MODEL_RTOL), (tag, r["cams"][0], c["params"])
        check_pnp_camera_exact(cam, n, c["flags"], loss, r)


@pytest.mark.gpu
@pytest.mark.parametrize("loss", MW.LOSSES)
@pytest.mark.parametrize("n", CAM_SIZES)
@pytest.mark.parametrize("pair", PAIRS)
def test_pair_camera_refiner_matches_reference_at_every_width(pair, n, loss):
    for c in [c for c in GOLD["refine"] if ((c["camera1"], c["camera2"]), c["n"], c["loss"]) == (pair, n, loss)]:
        r = run_pair_camera(pair, n, c["flags"], loss, seed=c["seed"])
        tag = (pair, n, c["flags"], loss)
        assert int(r["bs"][0]) == c["iterations"], (tag, r["bs"], c["iterations"])
        assert _close(r["bs"][1], c["initial_cost"], INITIAL_COST_RTOL), (tag, r["bs"], c["initial_cost"])
        assert _close(r["bs"][2], c["cost"], COST_RTOL), (tag, r["bs"], c["cost"])
        assert _close(r["model"], c["pose"], MODEL_RTOL), (tag, r["model"], c["pose"])
        assert _close(r["cams"][0], c["params1"], MODEL_RTOL), (tag, r["cams"][0], c["params1"])
        assert _close(r["cams"][1], c["params2"], MODEL_RTOL), (tag, r["cams"][1], c["params2"])
        check_pair_camera_exact(pair, n, c["flags"], loss, r, seed=c["seed"])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pnp", "pair"])
def test_sorted_estimates_polish_on_empty_ctas_as_the_reference(kind):
    """Inliers first: the final polish of the camera refiners runs 8 CTAs wide, CTAs 3-7 with empty compacted lists."""
    ro = cabi.RansacOpt(**MW.ESTIMATE_RANSAC)
    for c in [c for c in GOLD["estimate_cases"] if c["kind"] == kind]:
        bo = cabi.BundleOpt(refine_intrinsics=c["flags"])
        if kind == "pnp":
            cam = MW.ESTIMATE_CAMERAS["pnp"]
            x, X, p0 = MW.sorted_pnp_problem(cam, c["seed"])
            g = cabi.estimate_image(x, X, cabi.Camera(_model_name(cam), tuple(p0)), ro, bo, MW.ESTIMATE_MAX_ERROR)
            cams = [(g["camera"], c["params"])]
        else:
            pair = MW.ESTIMATE_CAMERAS["pair"]
            x1, x2, c1, c2 = MW.sorted_pair_problem(pair, c["seed"])
            g = cabi.estimate_relative_pose_pair(x1, x2, cabi.Camera(_model_name(pair[0]), tuple(c1)),
                                                 cabi.Camera(_model_name(pair[1]), tuple(c2)), ro, bo, MW.PAIR_MAX_ERROR)
            cams = [(g["camera1"], c["params1"]), (g["camera2"], c["params2"])]
        tag = (kind, c["flags"])
        for key in ("iterations", "refinements", "num_inliers"):
            assert g["stats"][key] == c[key], (tag, key, g["stats"][key], c[key])
        assert np.array_equal(g["inliers"].astype(np.uint8), _mask(c["inliers"])), tag
        assert _close(g["model"], c["pose"], MODEL_RTOL), (tag, g["model"], c["pose"])
        for got, want in cams:
            assert _close(got, want, MODEL_RTOL), (tag, got, want)


# ---- GPU: no points -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refine_entry_points_with_no_points_write_the_oracles_result():
    lib = cabi.lib()
    nan3 = lambda: np.full(3, np.nan)  # noqa: E731
    bo = cabi.BundleOpt()
    pose = np.array([0.9, 0.1, -0.2, 0.3, 0.5, -0.4, 0.7])
    pose /= np.r_[np.linalg.norm(pose[:4]) * np.ones(4), np.ones(3)]
    F = np.array([[0.1, -0.7, 0.2], [0.6, 0.05, -0.3], [-0.25, 0.35, 0.02]])
    empty2, empty3 = np.zeros((0, 2)), np.zeros((0, 3))
    for kind, fn, m0, b in (("pnp", lib.plb_bundle_adjust, pose, empty3), ("relpose", lib.plb_refine_relpose, pose, empty2),
                            ("fundamental", lib.plb_refine_fundamental, F, empty2),
                            ("homography", lib.plb_refine_homography, F, empty2)):
        m = cabi._init_model(kind, m0)
        bs = nan3()
        assert fn(None, None, C.c_size_t(0), m.ctypes.data_as(cabi._P), C.byref(bo), bs.ctypes.data_as(cabi._P)) == 0
        om, os_ = P.refine(kind, m0, empty2, b, P.BundleOpt())
        assert np.array_equal(bs, os_[:3]), (kind, bs, os_[:3])
        gm = cabi._model_out(kind, m)
        if kind == "fundamental":  # the factorisation's reconstruction, up to sign
            assert min(np.abs(gm - om).max(), np.abs(gm + om).max()) < 1e-12, (gm, om)
        else:
            assert np.array_equal(gm, om), (kind, gm, om)
    cam = cabi.Camera("PINHOLE", (800.0, 790.0, 320.0, 240.0))
    d, M = np.zeros((0, 3)), np.zeros((0, 3, 2))
    om, os_ = P.refine_relpose_tangent(pose, d, d, M, M, P.BundleOpt())
    m, bs = pose.copy(), nan3()
    assert lib.plb_refine_relpose_cameras(None, None, C.c_size_t(0), C.byref(cam), C.byref(cam),
                                          m.ctypes.data_as(cabi._P), C.byref(bo), bs.ctypes.data_as(cabi._P)) == 0
    assert np.array_equal(bs, os_[:3]) and np.array_equal(m, om), (bs, os_[:3], m, om)
    # with camera refinement: lm_impl stops before its first step, the cameras stay as given
    for flags in (0, 7):
        b7 = cabi.BundleOpt(refine_intrinsics=flags)
        c, m, bs = cabi.Camera("OPENCV", MG.TRUE_PARAMS[4]), pose.copy(), nan3()
        assert lib.plb_bundle_adjust_image(None, None, C.c_size_t(0), m.ctypes.data_as(cabi._P), C.byref(c), C.byref(b7),
                                           bs.ctypes.data_as(cabi._P)) == 0
        assert np.array_equal(bs, [0.0, 0.0, 0.0]) and np.array_equal(m, pose)
        assert list(c.params[:8]) == MG.TRUE_PARAMS[4]
        c1, c2, m, bs = cabi.Camera("PINHOLE", (800.0, 790.0, 320.0, 240.0)), cabi.Camera("RADIAL_FISHEYE",
                                                                                             MC.CAMERAS["RADIAL_FISHEYE"][1]), pose.copy(), nan3()
        assert lib.plb_refine_relpose_pair(None, None, C.c_size_t(0), C.byref(c1), C.byref(c2), m.ctypes.data_as(cabi._P),
                                           C.byref(b7), bs.ctypes.data_as(cabi._P)) == 0
        assert np.array_equal(bs, [0.0, 0.0, 0.0]) and np.array_equal(m, pose)
        assert list(c1.params[:4]) == [800.0, 790.0, 320.0, 240.0]
        assert list(c2.params[:5]) == MC.CAMERAS["RADIAL_FISHEYE"][1]


# ---- forced widths: one list of cases, run in-process (default width) and in child processes ------------------------
def _ransac_cases():
    """RANSAC problems whose LO refits and final polish go through k_lm: (name, kind, a, b, ropt kwargs, max_error,
    rfc).  The relpose LO subset (subset_mode 1) at 5, 6, 9 and 33 points decides "at most 5 points: untouched" from a
    cluster sum that spans empty CTAs."""
    out = []
    for n in (5, 6, 9, 33, 2049):
        p = G.relpose_problem(n, 0.8, 71, n)
        out.append(("relpose_%d" % n, "relpose", p["x1"] / G.FOCAL, p["x2"] / G.FOCAL,
                    dict(max_iterations=300, min_iterations=50, seed=n), 1.0 / G.FOCAL, False))
    for n in (33, 2049):
        p = G.abspose_problem(n, 0.6, 72, n)
        out.append(("pnp_%d" % n, "pnp", p["x"] / G.FOCAL, p["X"], dict(max_iterations=1000, min_iterations=100, seed=n),
                    12.0 / G.FOCAL, False))
    p = G.relpose_problem(3000, 0.3, 73, 0, prosac_sorted=True)
    out.append(("fundamental_prosac", "fundamental", p["x1"] / 500.0, p["x2"] / 500.0,
                dict(max_iterations=20000, min_iterations=500, seed=3, progressive_sampling=True,
                     max_prosac_iterations=5000), 1.0 / 500.0, True))
    p = G.homography_problem(20000, 0.6, 74, 0)
    out.append(("homography_20000", "homography", p["x1"] / G.FOCAL, p["x2"] / G.FOCAL,
                dict(max_iterations=5000, min_iterations=200, seed=4), 1.0 / G.FOCAL, False))
    return out


def _ts_ransac_case():
    x1, x2, _, c1, c2 = MR.pair_problem(1, 1, 3000, 4242, outliers=0.3)
    return x1, x2, ("PINHOLE", list(c1)), ("PINHOLE", list(c2)), dict(max_iterations=2000, min_iterations=100, seed=5), 1.0


def _batch_problems():
    """24 problems in one ransac_batch: several LO jobs per cluster of the persistent LO grid."""
    out = []
    for i in range(24):
        n = (33, 300, 2049, 7000)[i % 4]
        p = G.relpose_problem(n, 0.6, 75, i)
        out.append(dict(kind="relpose", a=p["x1"] / G.FOCAL, b=p["x2"] / G.FOCAL,
                        ransac=dict(max_iterations=500, min_iterations=100, seed=i), max_error=1.0 / G.FOCAL))
    return out


def width_cases():
    """(name, function) of every case the forced-width comparison runs; each function returns a dict."""
    cases = []
    for kind in ("pnp", "relpose", "fundamental", "homography"):
        for n in (33, 257, 2049, 6145, 40000):
            cases.append(("fixed/%s/%d" % (kind, n), lambda k=kind, n=n: run_fixed(k, n, "CAUCHY")))
        for it in (0, 1):
            for n in (257, 2049, 6145, 40000):
                cases.append(("fixed/%s/%d/it%d" % (kind, n, it), lambda k=kind, n=n, it=it: run_fixed(k, n, "CAUCHY", it)))
    for n in (33, 257, 6145, 40000):
        cases.append(("ts/%d" % n, lambda n=n: run_ts_fixed(n, "CAUCHY")))
        for cam in ("PINHOLE", "OPENCV", "RADIAL_FISHEYE", "DIVISION-"):
            cases.append(("pnpcam/%s/%d" % (cam, n), lambda c=cam, n=n: run_pnp_camera(c, n, 7, "CAUCHY")))
        for pair in PAIRS:
            cases.append(("paircam/%s+%s/%d" % (pair + (n,)), lambda pr=pair, n=n: run_pair_camera(pr, n, 7, "CAUCHY")))
    for it in (0, 1):
        for n in (257, 2049, 6145, 40000):
            cases.append(("pnpcam/OPENCV/%d/it%d" % (n, it), lambda n=n, it=it: run_pnp_camera("OPENCV", n, 7, "TRIVIAL", it)))
            cases.append(("paircam/OPENCV+OPENCV/%d/it%d" % (n, it),
                          lambda n=n, it=it: run_pair_camera(("OPENCV", "OPENCV"), n, 7, "TRIVIAL", it)))
    for name, kind, a, b, kw, me, rfc in _ransac_cases():
        cases.append(("ransac/" + name,
                      lambda kind=kind, a=a, b=b, kw=kw, me=me, rfc=rfc: cabi.ransac(kind, a, b, cabi.RansacOpt(**kw), me,
                                                                                   rfc=rfc)))
    x1, x2, c1, c2, kw, me = _ts_ransac_case()
    cases.append(("ransac/tangent_sampson", lambda: cabi.ransac_relpose_cameras(
        x1, x2, cabi.Camera(*c1), cabi.Camera(*c2), cabi.RansacOpt(**kw), me)))

    def batch():
        probs = [dict(p, ransac=cabi.RansacOpt(**p["ransac"])) for p in _batch_problems()]
        return {"batch": [{k: v for k, v in r.items() if k != "status"} for r in cabi.ransac_batch(probs, streams=2)]}
    cases.append(("ransac/batch24", batch))
    return cases


def _enc(v):
    """JSON with every float in hex (bit for bit across the process boundary) and masks as packed hex."""
    if isinstance(v, dict):
        return {k: _enc(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [_enc(x) for x in v]
    if isinstance(v, np.ndarray):
        if v.dtype == np.int8:
            return {"mask": np.packbits(v.astype(np.uint8)).tobytes().hex(), "n": int(len(v))}
        return [_enc(x) for x in v.tolist()]
    if isinstance(v, (float, np.floating)):
        return {"f": float(v).hex()}
    return int(v)


def _dec(v):
    if isinstance(v, dict):
        if set(v) == {"f"}:
            return float.fromhex(v["f"])
        if set(v) == {"mask", "n"}:
            return np.unpackbits(np.frombuffer(bytes.fromhex(v["mask"]), dtype=np.uint8))[:v["n"]].astype(np.int8)
        return {k: _dec(x) for k, x in v.items()}
    if isinstance(v, list):
        return [_dec(x) for x in v]
    return v


def _run_cases():
    return {name: _dec(_enc(fn())) for name, fn in width_cases()}


def _child(setting):
    env = dict(os.environ, PLB_LM_PER_CTA=FORCED[setting], PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, cwd=ROOT, capture_output=True,
                       text=True, timeout=540)
    assert r.returncode == 0, r.stderr[-4000:]
    return {k: _dec(v) for k, v in json.loads(r.stdout.strip().splitlines()[-1]).items()}


@pytest.fixture(scope="module")
def widths():
    """Results of width_cases() at the default width (in this process) and at the two forced settings (children)."""
    out = {"default": _run_cases()}
    for s in FORCED:
        out[s] = _child(s)
    return out


def _exact_check(name, r):
    parts = name.split("/")
    it = [int(p[2:]) for p in parts if p.startswith("it")]
    if parts[0] == "fixed":
        check_fixed_exact(parts[1], int(parts[2]), "CAUCHY", r)
    elif parts[0] == "ts":
        check_ts_fixed_exact(int(parts[1]), "CAUCHY", r)
    elif parts[0] == "pnpcam":
        check_pnp_camera_exact(parts[1], int(parts[2]), 7, "TRIVIAL" if it else "CAUCHY", r)
    elif parts[0] == "paircam":
        check_pair_camera_exact(tuple(parts[1].split("+")), int(parts[2]), 7, "TRIVIAL" if it else "CAUCHY", r)
    if it:
        assert int(r["bs"][0]) == it[0] or (it[0] == 1 and int(r["bs"][0]) == 0), (name, r["bs"])
        if int(r["bs"][0]) == 0:
            assert r["bs"][2] == r["bs"][1], (name, r["bs"])


def _max_rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b) / np.maximum(1.0, np.abs(b)))) if a.size else 0.0


@pytest.mark.gpu
def test_refiners_agree_across_forced_widths(widths):
    worst = (0.0, ())
    for name, _ in width_cases():
        if name.startswith("ransac/"):
            continue
        base = widths["default"][name]
        for setting in ("default",) + tuple(FORCED):
            r = widths[setting][name]
            _exact_check(name, r)
            assert int(r["bs"][0]) == int(base["bs"][0]), (name, setting, r["bs"], base["bs"])
            for key in ("model", "cams"):
                if key in base:
                    d = _max_rel(np.ravel(r[key]) if key == "model" else np.concatenate([np.ravel(c) for c in r[key]]),
                                 np.ravel(base[key]) if key == "model" else np.concatenate([np.ravel(c) for c in base[key]]))
                    if name.startswith("fixed/fundamental") and key == "model":  # F up to sign
                        d = min(d, _max_rel(-np.ravel(r[key]), np.ravel(base[key])))
                    worst = max(worst, (d, (name, setting, key)))
                    assert d <= CROSS_WIDTH_RTOL, (name, setting, key, d)
    print("largest cross-width relative difference: %.3g at %s" % worst)


@pytest.mark.gpu
def test_ransac_trajectories_hold_at_forced_widths(widths):
    from test_gpu_parity import _same_trajectory
    oracle = {}
    for name, kind, a, b, kw, me, rfc in _ransac_cases():
        oracle["ransac/" + name] = (P.ransac(kind, a, b, P.RansacOpt(**kw), me, rfc=rfc), kind)
    x1, x2, c1, c2, kw, me = _ts_ransac_case()
    oracle["ransac/tangent_sampson"] = (P.ransac_relpose_cameras(x1, x2, c1, c2, P.RansacOpt(**kw), me), "relpose")
    batch = [(P.ransac(p["kind"], p["a"], p["b"], P.RansacOpt(**p["ransac"]), p["max_error"]), p["kind"])
             for p in _batch_problems()]
    for setting in ("default",) + tuple(FORCED):
        for name, (o, kind) in oracle.items():
            _same_trajectory(widths[setting][name], o, relpose=(kind == "relpose"))
        for g, (o, kind) in zip(widths[setting]["ransac/batch24"]["batch"], batch):
            _same_trajectory(g, o, relpose=(kind == "relpose"))


# ---- batches: the width follows the largest problem of the launch ---------------------------------------------------
def _batch_estimate_inputs():
    out = []
    for i, (cam, n) in enumerate((("PINHOLE", 600), ("RADIAL_FISHEYE", 2049), ("OPENCV", 6145), ("PINHOLE", 20000),
                                  ("DIVISION-", 600), ("RADIAL_FISHEYE", 20000))):
        if cam in MC.CAMERAS:
            x, X, _, p0 = MC.problem(cam, n, 97000 + i, outliers=0.3)
        else:
            x, X, _, p0, _ = MG.problem(MG.MODELS[cam], n, 97000 + i, outliers=0.3)
        out.append((cam, x, X, np.asarray(p0, dtype=np.float64), [7, 3, 1, 7, 7, 0][i]))
    return out


@pytest.mark.gpu
def test_estimate_batch_width_follows_its_largest_problem():
    ro = dict(max_iterations=2000, min_iterations=100, seed=11)
    probs, singles = [], []
    for cam, x, X, p0, flags in _batch_estimate_inputs():
        c = cabi.Camera(_model_name(cam), tuple(p0))
        bo = cabi.BundleOpt(refine_intrinsics=flags)
        probs.append(dict(kind="pnp", a=x, b=X, ransac=cabi.RansacOpt(**ro), bundle=bo, max_error=4.0, cam1=c))
        singles.append(cabi.estimate_image(x, X, c, cabi.RansacOpt(**ro), bo, 4.0))
    out = cabi.estimate_batch(probs)
    worst = 0.0
    for i, (o, s) in enumerate(zip(out, singles)):
        assert o["status"] == 0
        for key in ("iterations", "refinements", "num_inliers"):
            assert o["stats"][key] == s["stats"][key], (i, key)
        assert o["stats"]["inlier_ratio"] == s["stats"]["inlier_ratio"], i
        assert np.isclose(o["stats"]["model_score"], s["stats"]["model_score"], rtol=CROSS_WIDTH_RTOL, atol=0), i
        assert np.array_equal(o["inliers"], s["inliers"]), i
        worst = max(worst, _max_rel(o["model"], s["model"]), _max_rel(o["camera1"], s["camera"]))
        assert _max_rel(o["model"], s["model"]) <= CROSS_WIDTH_RTOL, (i, o["model"], s["model"])
        assert _max_rel(o["camera1"], s["camera"]) <= CROSS_WIDTH_RTOL, (i, o["camera1"], s["camera"])
    print("largest batch / single relative difference: %.3g" % worst)


if __name__ == "__main__" and sys.argv[1:] == ["--child"]:
    print(json.dumps({name: _enc(fn()) for name, fn in width_cases()}))
