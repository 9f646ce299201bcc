"""The fisheye and division camera models on the device: SIMPLE_RADIAL_FISHEYE (8), RADIAL_FISHEYE (9), DIVISION (101)
and SIMPLE_DIVISION (102) through every entry point that takes a camera.

Reference: PoseLib's own sources (oracle/_ref/libplref2.so, the reference on mini-Eigen) through
tests/ref_camera_models_client.cc, and their results on seeded problems in tests/golden/reference_camera_models.json
(tests/golden/make_camera_models_golden.py).
  * CPU, where the reference is mounted: the host build of camera.cuh equals the reference's Camera functions bit for
    bit (near-axis points, theta at pi/2, bearings past 90 degrees, division points with disc2 < 0 included), and the
    reference reproduces the fixture bit for bit.
  * CPU, everywhere: the four ids pass argument validation, the reference's other models stay NYI.
  * GPU: every camera function on the device against the host build of the same source (division: bearings,
    calibrated points and projections bit for bit), and the fixture: RANSAC outcomes (inlier masks, stats, iteration
    counts) exactly, costs, poses and cameras to bars chosen from the deviation measured on an H100 (below).  The
    fisheye models use CUDA's atan2 / tan, which are not correctly rounded, so their doubles may differ from glibc's in
    the last bits; on these scenes no decision flips."""
import ctypes as C
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_camera_models_golden as CG  # noqa: E402

try:
    from poselib_b200 import cabi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)

GOLD = json.load(open(CG.OUT))
needs_reference = pytest.mark.skipif(
    not (CG.MG.reference_available() and os.path.exists(os.path.join(CG.ROOT, "oracle", "_ref", "libplref2.so"))),
    reason="needs the reference checkout and oracle/_ref/libplref2.so")
NEW_IDS = (8, 9, 101, 102)
NYI_IDS = (5, 6, 7, 10, 11, 99, 100)

# Relative tolerances against the fixture (|a - b| <= rtol * max(1, |b|)), chosen from the largest deviation
# tools/camera_models_deviation.py measured on one H100 80GB HBM3 (700 W power limit) over every case of the fixture,
# fisheye and division together, with a margin of 2-40x:
#   bundle_adjust_image / estimate_absolute_pose_image: initial cost 1.4e-14, cost 2.7e-14, pose 8.2e-16, params 1.6e-15
#   refine_relpose_pair: initial cost 1.4e-14, cost 8.5e-13, pose 1.8e-9, params 1.4e-7
#   estimate_relative_pose_pair: pose 5.0e-7, params 8.3e-9
# (iteration counts, RANSAC stats and inlier masks: no difference in any case).
IMAGE_RTOL = 1e-12                                    # every value of the single-image calls
PAIR_INITIAL_COST_RTOL, PAIR_COST_RTOL, PAIR_POSE_RTOL, PAIR_PARAM_RTOL = 1e-12, 1e-11, 1e-8, 1e-6
PAIR_ESTIMATE_POSE_RTOL, PAIR_ESTIMATE_PARAM_RTOL = 1e-6, 1e-7


def _cam(name, params):
    return cabi.Camera(CG.CAMERAS[name][0], tuple(params))


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return CG.build_client(str(tmp_path_factory.mktemp("ref_camera_models")))


# ---- CPU ---------------------------------------------------------------------------------------------------
def test_tables_know_the_four_models():
    for name, mid in (("SIMPLE_RADIAL_FISHEYE", 8), ("RADIAL_FISHEYE", 9), ("DIVISION", 101), ("SIMPLE_DIVISION", 102)):
        assert cabi.CAMERA[name] == mid and cabi.CAMERA_NUM_PARAMS[mid] == CG.NUM_PARAMS[mid]
    for mid in (5, 7):
        assert mid not in cabi.CAMERA_NUM_PARAMS


@needs_reference
@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
@pytest.mark.parametrize("cam", list(CG.CAMERAS))
def test_device_camera_source_matches_poselib_bitwise(ref, cam, tmp_path):
    exe = str(tmp_path / "camera_models_host_test")
    subprocess.check_call(["nvcc", "-std=c++17", "-O2", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-Xcompiler", "-ffp-contract=off", "-o", exe, os.path.join(HERE, "camera_models_host_test.cu")])
    model = CG.model_id(cam)
    npar = CG.NUM_PARAMS[model]
    params = CG._p8(cam)
    px, Z = CG.host_points(model, params)
    if model in (101, 102) and params[npar - 1] > 0:
        assert np.any(Z[:, 2] ** 2 - 4.0 * (Z[:, 0] ** 2 + Z[:, 1] ** 2) * params[npar - 1] < 0)  # disc2 < 0 reached
    args = [exe, str(model)] + [repr(float(v)) for v in params] + [repr(1.0 / 1234.5)]
    out = subprocess.check_output(args + ["px"] + [repr(float(v)) for v in px.reshape(-1)], text=True).splitlines()
    outz = subprocess.check_output(args + ["pt"] + [repr(float(v)) for v in Z.reshape(-1)], text=True).splitlines()
    for flags in range(8):
        idx = np.zeros(8, dtype=np.int32)
        m = ref.cm_refine_idx(model, CG._p(params), flags, idx.ctypes.data_as(C.POINTER(C.c_int)))
        assert [int(t) for t in out[flags].split()[1:]] == [m] + idx[:m].tolist(), flags
    assert float.fromhex(out[8].split()[1]) == ref.cm_focal(model, CG._p(params))
    rs = params.copy()
    ref.cm_rescale(model, CG._p(rs), C.c_double(1.0 / 1234.5))
    assert np.array_equal(np.array([float.fromhex(t) for t in out[9].split()[1:]]), rs)
    # pixels: bearing, hnormalized, unproject_with_jac (d, M), unproject_with_jac with params (d, M, dp)
    got = np.array([[float.fromhex(t) for t in line.split()[1:]] for line in out[10:]])
    n = len(px)
    x3, x2, d, M, dp, dq, dpq = (np.zeros(3 * n), np.zeros(2 * n), np.zeros(3 * n), np.zeros(6 * n), np.zeros(24 * n),
                                 np.zeros(3 * n), np.zeros(24 * n))
    pxc = np.ascontiguousarray(px)
    ref.cm_unproject(model, CG._p(params), C.c_int64(n), CG._p(pxc), CG._p(x3), CG._p(x2), CG._p(d), CG._p(M), CG._p(dp),
                     CG._p(dq), CG._p(dpq))
    eq = lambda a, b: np.array_equal(a, b, equal_nan=True)
    assert eq(got[:, 0:3], x3.reshape(n, 3))
    assert eq(got[:, 3:5], x2.reshape(n, 2))
    assert eq(got[:, 5:8], d.reshape(n, 3)) and eq(got[:, 8:14], M.reshape(n, 6))
    assert eq(got[:, 14:17], d.reshape(n, 3)) and eq(got[:, 17:23], M.reshape(n, 6))
    gdp = got[:, 23:].reshape(n, 3, 8)[:, :, :npar]
    assert eq(gdp, dp.reshape(n, 3, 8)[:, :, :npar])
    assert eq(gdp, dpq.reshape(n, 3, 8)[:, :, :npar])  # without a jac_point: the same bits
    assert eq(got[:, 14:17], dq.reshape(n, 3))
    # camera-frame points: project, project_with_jac (xp, J), jac_params
    gz = np.array([[float.fromhex(t) for t in line.split()[1:]] for line in outz[10:]])
    nz = len(Z)
    xp, xq, jac, jp = np.zeros(2 * nz), np.zeros(2 * nz), np.zeros(6 * nz), np.zeros(16 * nz)
    Zc = np.ascontiguousarray(Z)
    ref.cm_project(model, CG._p(params), C.c_int64(nz), CG._p(Zc), CG._p(xp), CG._p(xq), CG._p(jac), CG._p(jp))
    assert eq(gz[:, 0:2], xp.reshape(nz, 2)) and eq(gz[:, 2:4], xq.reshape(nz, 2))
    assert eq(gz[:, 4:10], jac.reshape(nz, 6))
    assert eq(gz[:, 10:].reshape(nz, 2, 8)[:, :, :npar], jp.reshape(nz, 2, 8)[:, :, :npar])


@needs_reference
def test_reference_reproduces_the_fixture_bitwise(ref):
    for case in GOLD["bundle"]:
        assert CG.ref_bundle_adjust(ref, case["camera"], case["flags"], case["loss"]) == case, case
    for case in GOLD["estimate_cases"]:
        assert CG.ref_estimate(ref, case["camera"], case["flags"]) == case, case
    for case in GOLD["refine"]:
        pair = (case["camera1"], case["camera2"])
        assert CG.ref_refine(ref, pair, case["flags"], case["loss"], case["seed"]) == case, case
    for case in GOLD["pair_estimate_cases"]:
        pair = (case["camera1"], case["camera2"])
        assert CG.ref_pair_estimate(ref, pair, case["flags"], case["tangent"], case["seed"]) == case, case


def test_fixture_covers_the_grid():
    assert {(c["camera"], c["flags"], c["loss"]) for c in GOLD["bundle"]} == set(CG.bundle_cases())
    assert {(c["camera"], c["flags"]) for c in GOLD["estimate_cases"]} == set(CG.estimate_cases())
    assert all(c["num_inliers"] > 5 for c in GOLD["estimate_cases"] + GOLD["pair_estimate_cases"])
    assert all(c["cost"] < c["initial_cost"] and c["iterations"] > 0 for c in GOLD["refine"])
    # the refine cases on which no draw is summation-order stable are named, not dropped silently
    kept = {(c["camera1"], c["camera2"], c["flags"], c["loss"]) for c in GOLD["refine"]}
    assert kept == {(*p, f, l) for p, f, l in CG.refine_cases()} - {(*p, f, l) for p, f, l in CG.REFINE_LEFT_OUT}
    assert len(GOLD["refine"]) == len(kept)
    left = {p for p, f, l in CG.REFINE_LEFT_OUT}
    assert all(any(c["flags"] == 7 and (c["camera1"], c["camera2"]) == p for c in GOLD["refine"])
               for p in CG.PAIRS if p not in left)  # every other pair, the mixed fisheye / division one included
    est = {(c["camera1"], c["camera2"], c["flags"], c["tangent"]) for c in GOLD["pair_estimate_cases"]}
    assert est == {(*p, f, t) for p, f, t in CG.pair_estimate_cases()}


def _pts(n=12):
    return np.zeros((n, 2)) + 100.0, np.ones((n, 3))


def test_new_ids_pass_validation_and_the_others_stay_nyi():
    x, X = _pts()
    for mid in NEW_IDS + NYI_IDS:
        cam = cabi.Camera(mid, (500.0, 500.0, 320.0, 240.0, 0.01))
        calls = [lambda: cabi.estimate("pnp", x, X, cabi.RansacOpt(), cabi.BundleOpt(), 1.0, cam1=cam),
                 lambda: cabi.refine_image(np.r_[1.0, np.zeros(6)], x, X, cam, cabi.BundleOpt()),
                 lambda: cabi.estimate("relpose", x, x, cabi.RansacOpt(), cabi.BundleOpt(), 1.0, cam1=cam, cam2=cam,
                                       tangent_sampson=True)]
        for call in calls:
            if mid in NYI_IDS:
                with pytest.raises(cabi.PoseLibB200Error) as e:
                    call()
                assert e.value.code == cabi.PLB_ERR_NYI, mid
            elif cabi.device_count() == 0:  # past validation: the device is what is missing
                with pytest.raises(cabi.PoseLibB200Error) as e:
                    call()
                assert e.value.code == cabi.PLB_ERR_CUDA, mid


def test_pyapi_accepts_the_four_names():
    from poselib_b200 import pyapi
    for name in ("SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE", "DIVISION", "SIMPLE_DIVISION"):
        c = pyapi._camera({"model": name, "params": [500.0, 320.0, 240.0, 0.01, 0.0][:cabi.CAMERA_NUM_PARAMS[cabi.CAMERA[name]]]})
        assert c.model_id == cabi.CAMERA[name]


# ---- GPU ---------------------------------------------------------------------------------------------------
def _close(a, b, rtol):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.all(np.abs(a - b) <= rtol * np.maximum(1.0, np.abs(b)))



def _mask(case, n):
    return np.unpackbits(np.frombuffer(bytes.fromhex(case["inliers"]), dtype=np.uint8))[:n].astype(bool)


def _check_mask(got, case, n):
    want = _mask(case, n)
    diff = np.flatnonzero(got.astype(bool) != want)
    assert len(diff) == 0, ("inlier masks differ", case["camera1"] if "camera1" in case else case["camera"], diff[:10])


@pytest.mark.gpu
@pytest.mark.parametrize("loss", list(CG.LOSSES))
@pytest.mark.parametrize("cam", CG.NEW)
def test_bundle_adjust_image_matches_reference(cam, loss):
    for case in [c for c in GOLD["bundle"] if (c["camera"], c["loss"]) == (cam, loss)]:
        flags = case["flags"]
        x, X, pose0, p0 = CG.problem(cam, CG.BUNDLE_N, CG.bundle_seed(cam, flags, loss))
        b = cabi.BundleOpt(loss_type=loss, loss_scale=GOLD["loss_scale"], relative_cost_tol=GOLD["relative_cost_tol"],
                           refine_intrinsics=flags)
        pose, params, bs = cabi.refine_image(pose0, x, X, _cam(cam, p0), b)
        tag = (cam, loss, flags)
        assert int(bs[0]) == case["iterations"], (tag, bs, case["iterations"])
        assert _close(bs[1], case["initial_cost"], IMAGE_RTOL), (tag, bs, case["initial_cost"])
        assert _close(bs[2], case["cost"], IMAGE_RTOL), (tag, bs, case["cost"])
        assert _close(pose, case["pose"], IMAGE_RTOL), (tag, pose, case["pose"])
        assert _close(params, case["params"], IMAGE_RTOL), (tag, params, case["params"])


@pytest.mark.gpu
@pytest.mark.parametrize("cam", CG.NEW)
def test_estimate_absolute_pose_image_matches_reference(cam):
    x, X, _, p0 = CG.problem(cam, CG.ESTIMATE_N, CG.estimate_seed(cam), outliers=0.3)
    ro = cabi.RansacOpt(**CG.ESTIMATE_RANSAC)
    for case in [c for c in GOLD["estimate_cases"] if c["camera"] == cam]:
        flags = case["flags"]
        g = cabi.estimate_image(x, X, _cam(cam, p0), ro, cabi.BundleOpt(refine_intrinsics=flags), CG.ESTIMATE_MAX_ERROR)
        _check_mask(g["inliers"], case, CG.ESTIMATE_N)
        for key in ("iterations", "refinements", "num_inliers"):
            assert g["stats"][key] == case[key], (cam, flags, key)
        assert _close(g["model"], case["pose"], IMAGE_RTOL), (cam, flags, g["model"], case["pose"])
        assert _close(g["camera"], case["params"], IMAGE_RTOL), (cam, flags, g["camera"], case["params"])


def _pair_id(p):
    return "%s-%s" % p


@pytest.mark.gpu
@pytest.mark.parametrize("pair", CG.PAIRS, ids=[_pair_id(p) for p in CG.PAIRS])
def test_refine_relpose_pair_matches_reference(pair):
    for case in [c for c in GOLD["refine"] if (c["camera1"], c["camera2"]) == pair]:
        x1, x2, pose0, c1, c2 = CG.pair_problem(*pair, CG.PAIR_N, case["seed"])
        b = cabi.BundleOpt(loss_type=case["loss"], loss_scale=GOLD["pair_loss_scale"],
                           relative_cost_tol=GOLD["relative_cost_tol"], refine_intrinsics=case["flags"])
        pose, p1, p2, bs = cabi.refine_relpose_pair(pose0, x1, x2, _cam(pair[0], c1), _cam(pair[1], c2), b)
        tag = (pair, case["loss"], case["flags"])
        assert int(bs[0]) == case["iterations"], (tag, bs, case["iterations"])
        assert _close(bs[1], case["initial_cost"], PAIR_INITIAL_COST_RTOL), (tag, bs, case["initial_cost"])
        assert _close(bs[2], case["cost"], PAIR_COST_RTOL), (tag, bs, case["cost"])
        assert _close(pose, case["pose"], PAIR_POSE_RTOL), (tag, pose, case["pose"])
        assert _close(p1, case["params1"], PAIR_PARAM_RTOL), (tag, p1, case["params1"])
        assert _close(p2, case["params2"], PAIR_PARAM_RTOL), (tag, p2, case["params2"])


@pytest.mark.gpu
@pytest.mark.parametrize("pair", CG.PAIRS, ids=[_pair_id(p) for p in CG.PAIRS])
def test_estimate_relative_pose_matches_reference(pair):
    ro = cabi.RansacOpt(**CG.ESTIMATE_RANSAC)
    for case in [c for c in GOLD["pair_estimate_cases"] if (c["camera1"], c["camera2"]) == pair]:
        flags, tangent = case["flags"], case["tangent"]
        x1, x2, _, c1, c2 = CG.pair_estimate_inputs(pair, case["seed"], tangent)
        cam1, cam2 = _cam(pair[0], c1), _cam(pair[1], c2)
        g = cabi.estimate_relative_pose_pair(x1, x2, cam1, cam2, ro, cabi.BundleOpt(refine_intrinsics=flags),
                                             CG.PAIR_MAX_ERROR, tangent_sampson=tangent)
        tag = (pair, flags, tangent)
        _check_mask(g["inliers"], case, CG.ESTIMATE_N)
        for key in ("iterations", "refinements", "num_inliers"):
            assert g["stats"][key] == case[key], (tag, key)
        assert _close(g["model"], case["pose"], PAIR_ESTIMATE_POSE_RTOL), (tag, g["model"], case["pose"])
        assert _close(g["camera1"], case["params1"], PAIR_ESTIMATE_PARAM_RTOL), (tag, g["camera1"], case["params1"])
        assert _close(g["camera2"], case["params2"], PAIR_ESTIMATE_PARAM_RTOL), (tag, g["camera2"], case["params2"])


@pytest.mark.gpu
def test_mixed_batch_equals_single_calls_and_fast_equals_exact():
    names = ["RADIAL_FISHEYE", "PINHOLE", "DIVISION+", "RADIAL", "SIMPLE_DIVISION-", "SIMPLE_RADIAL_FISHEYE"]
    flags = [7, 3, 1, 0, 7, 3]
    probs, singles = [], []
    ro = cabi.RansacOpt(**CG.ESTIMATE_RANSAC)
    for name, f in zip(names, flags):
        x, X, _, p0 = CG.problem(name, CG.ESTIMATE_N, CG.estimate_seed(name), outliers=0.3)
        cam = _cam(name, p0)
        probs.append(dict(kind="pnp", a=x, b=X, ransac=ro, bundle=cabi.BundleOpt(refine_intrinsics=f),
                          max_error=CG.ESTIMATE_MAX_ERROR, cam1=cam))
        singles.append((cabi.estimate_image(x, X, cam, ro, cabi.BundleOpt(refine_intrinsics=f), CG.ESTIMATE_MAX_ERROR),
                        f, p0))
    out = {}
    try:
        for mode in ("exact", "fast"):
            cabi.set_mode(mode)
            out[mode] = cabi.estimate_batch(probs)
    finally:
        cabi.set_mode("fast")
    for o, e, (s, f, p0) in zip(out["fast"], out["exact"], singles):
        for r in (o, e):
            assert np.array_equal(r["model"], s["model"]) and np.array_equal(r["inliers"], s["inliers"])
            assert r["stats"] == s["stats"]
            assert np.array_equal(r["camera1"], s["camera"] if f else np.asarray(p0))


# Bars of the device camera functions against the host build (which equals the reference bit for bit).  Division:
# bearings, calibrated points and projections use + - * / and sqrt only and must be equal; the rest (pow in the
# division parameter Jacobian, atan2 / tan of the fisheye models) is held to DEVICE_FN_RTOL.  Measured on one H100 80GB
# HBM3 (700 W): fisheye at most 5.5e-14 (RADIAL_FISHEYE projection Jacobians), division 0 in every column.
DEVICE_FN_RTOL = 1e-12


@pytest.mark.gpu
@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
@pytest.mark.parametrize("cam", CG.NEW)
def test_device_camera_functions_match_the_host_build(cam, tmp_path):
    rows = CG.device_camera_rows(cam, str(tmp_path))
    for kind, (dev, host) in rows.items():
        exact = np.arange(dev.shape[1]) < (0 if CG.model_id(cam) in (8, 9) else CG.DIVISION_EXACT_COLUMNS[kind])
        assert np.array_equal(dev[:, exact], host[:, exact], equal_nan=True), (cam, kind)
        dev_r, host_r = dev[:, ~exact], host[:, ~exact]
        ok = np.isfinite(host_r)
        assert np.array_equal(np.isfinite(dev_r), ok), (cam, kind)
        dev_max = np.max(np.abs(dev_r[ok] - host_r[ok]) / np.maximum(1.0, np.abs(host_r[ok])), initial=0.0)
        assert dev_max <= DEVICE_FN_RTOL, (cam, kind, dev_max)
