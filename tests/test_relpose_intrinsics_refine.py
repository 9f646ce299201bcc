"""Camera-parameter refinement in the relative-pose bundle adjustment (CameraRelativePoseRefiner, refine_relpose(x1, x2,
ImagePair*, opt) with BundleOptions::refine_focal_length / refine_principal_point / refine_extra_params):
plb_refine_relpose_pair and plb_estimate_relative_pose_pair.

Reference: PoseLib's own sources (oracle/_ref/libplref2.so, the reference on mini-Eigen) through
tests/ref_relpose_intrinsics_client.cc, and their results on seeded two-view problems in
tests/golden/reference_relpose_intrinsics.json (tests/golden/make_relpose_intrinsics_golden.py).
  * CPU, where the reference is mounted: the host build of camera.cuh's cam_unproject_with_jac_params equals
    Camera::unproject_with_jac's jac_params bit for bit in both of its forms, and the reference reproduces the fixture
    (for the estimate cases: estimate_relative_pose itself and the restatement that keeps the cameras agree bit for
    bit).
  * CPU, everywhere: the C-ABI surface and the argument checks that run before any device call.
  * GPU: the device refiner holds the fixture at the bars of test_bundle_adjust_image_matches_reference, flags that
    select no parameter give the fixed-camera refiner's results, and the estimate entry point keeps RANSAC's outcome
    bit for bit."""
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
import make_relpose_intrinsics_golden as RG  # noqa: E402

try:
    from poselib_b200 import cabi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)

GOLD = json.load(open(RG.OUT))
MODELS = RG.MODELS
needs_reference = pytest.mark.skipif(
    not (RG.MG.reference_available() and os.path.exists(os.path.join(RG.ROOT, "oracle", "_ref", "libplref2.so"))),
    reason="needs the reference checkout and oracle/_ref/libplref2.so")


def _cam(model, params):
    return cabi.Camera(model, tuple(params))


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return RG.build_client(str(tmp_path_factory.mktemp("ref_relpose_intrinsics")))


# ---- CPU ---------------------------------------------------------------------------------------------------
def test_exports():
    lib = cabi.lib()
    for name in ("plb_refine_relpose_pair", "plb_estimate_relative_pose_pair"):
        assert name in cabi.EXPORTS and hasattr(lib, name)


def test_argument_checks_run_before_the_device():
    x = np.zeros((10, 2))
    c = _cam("PINHOLE", (500.0, 500.0, 0.0, 0.0))
    pose = np.r_[1.0, np.zeros(6)]
    bs = np.zeros(3)
    P = C.POINTER(C.c_double)
    xp = x.ctypes.data_as(P)
    lib = cabi.lib()
    b = cabi.BundleOpt(refine_intrinsics=1)
    for c1, c2 in ((None, C.byref(c)), (C.byref(c), None)):
        assert lib.plb_refine_relpose_pair(xp, xp, C.c_size_t(10), c1, c2, pose.ctypes.data_as(P), C.byref(b),
                                           bs.ctypes.data_as(P)) == cabi.PLB_ERR_ARG
    ro = cabi.RansacOpt()
    mask = np.zeros(10, dtype=np.int8)
    for c1, c2 in ((None, C.byref(c)), (C.byref(c), None)):
        assert lib.plb_estimate_relative_pose_pair(xp, xp, C.c_size_t(10), c1, c2, C.byref(ro), C.byref(b),
                                                   C.c_double(1.0), 1, pose.ctypes.data_as(P),
                                                   mask.ctypes.data_as(C.c_char_p), None, None) == cabi.PLB_ERR_ARG
    bad = cabi.Camera("PINHOLE", (500.0, 500.0, 0.0, 0.0))
    bad.model_id = 5  # a model of the reference outside the six on the device path
    with pytest.raises(cabi.PoseLibB200Error) as e:
        cabi.refine_relpose_pair(pose, x, x, bad, c, b)
    assert e.value.code == cabi.PLB_ERR_NYI
    with pytest.raises(cabi.PoseLibB200Error) as e:
        cabi.estimate_relative_pose_pair(x, x, c, bad, ro, b, 1.0)
    assert e.value.code == cabi.PLB_ERR_NYI
    if cabi.device_count() == 0:  # no CPU fallback
        for call in (lambda: cabi.refine_relpose_pair(pose, x, x, c, c, b),
                     lambda: cabi.estimate_relative_pose_pair(x, x, c, c, ro, b, 1.0)):
            with pytest.raises(cabi.PoseLibB200Error) as e:
                call()
            assert e.value.code == cabi.PLB_ERR_CUDA


@needs_reference
@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
@pytest.mark.parametrize("model", [-1, 0, 1, 2, 3, 4])
def test_device_unproject_jac_params_match_poselib_bitwise(ref, model, tmp_path):
    exe = str(tmp_path / "camera_unproject_jac_host_test")
    subprocess.check_call(["nvcc", "-std=c++17", "-O2", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-Xcompiler", "-ffp-contract=off", "-o", exe,
                           os.path.join(HERE, "camera_unproject_jac_host_test.cu")])
    params = np.zeros(8)
    np_model = RG.NUM_PARAMS.get(model, 0)
    if model >= 0:
        params[:np_model] = RG.TRUE_PARAMS[model]
    rng = np.random.RandomState(200 + model)
    xp = rng.uniform(0, 640, (40, 2)) if model >= 0 else rng.uniform(-1, 1, (40, 2))
    # the finite-difference points of CameraRelativePoseRefiner::compute_jacobian (optim/relative.h:392-418)
    xp = np.concatenate([xp, xp + [1e-6, 0.0], xp + [0.0, 1e-6]])
    out = subprocess.check_output([exe, str(model)] + [repr(float(v)) for v in params] +
                                  [repr(float(v)) for v in xp.reshape(-1)], text=True).splitlines()
    got = np.array([[float.fromhex(t) for t in line.split()[1:]] for line in out])
    for with_point in (1, 0):
        d, dp = RG.ref_unproject(ref, model, params, xp, with_point)
        assert np.array_equal(got[:, :3], d), with_point
        assert np.array_equal(got[:, 3:].reshape(-1, 3, 8)[:, :, :np_model], dp[:, :, :np_model]), with_point


@needs_reference
def test_reference_reproduces_the_fixture_bitwise(ref):
    """Every n = 500 case and every fourth n = 6000 case (the n = 6000 runs take seconds each on the CPU)."""
    big = [c for c in GOLD["refine"] if c["n"] == 6000]
    for case in [c for c in GOLD["refine"] if c["n"] == 500] + big[::4]:
        r = RG.ref_refine(ref, (case["camera1"], case["camera2"]), case["n"], case["flags"], case["loss"],
                          case["seed"])
        assert r == case, case
    for case in GOLD["estimate_cases"]:
        pair, flags, seed = (case["camera1"], case["camera2"]), case["flags"], case["seed"]
        assert RG.ref_estimate(ref, pair, flags, seed) == case, case
        plain = RG.ref_estimate(ref, pair, flags, seed, restate=False)  # estimate_relative_pose itself
        for key in ("iterations", "refinements", "num_inliers", "model_score", "pose", "inliers"):
            assert plain[key] == case[key], (case, key)


def test_fixture_covers_every_pair_flag_set_loss_and_size():
    keys = {(c["camera1"], c["camera2"], c["flags"], c["loss"], c["n"]) for c in GOLD["refine"]}
    assert len(keys) == len(RG.PAIRS) * 7 * 4 * 2 and len(GOLD["refine"]) == len(keys)
    assert {(c["camera1"], c["camera2"]) for c in GOLD["refine"]} == set(RG.PAIRS)
    assert any(a != b for a, b in RG.PAIRS)  # m1 != m2: the two cameras' parameter counts differ
    # the problems start inside the basin: every run descends
    assert all(c["cost"] < c["initial_cost"] and c["iterations"] > 0 for c in GOLD["refine"])
    est = {(c["camera1"], c["camera2"], c["flags"]) for c in GOLD["estimate_cases"]}
    assert est == {(*p, f) for p in RG.PAIRS for f in RG.ESTIMATE_FLAGS}
    assert all(c["num_inliers"] > 5 for c in GOLD["estimate_cases"])  # the final bundle adjustment runs


# ---- GPU ---------------------------------------------------------------------------------------------------
def _close(a, b, rtol):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.all(np.abs(a - b) <= rtol * np.maximum(1.0, np.abs(b)))


def _inputs(case):
    m1, m2 = MODELS[case["camera1"]], MODELS[case["camera2"]]
    x1, x2, pose0, c1, c2 = RG.pair_problem(m1, m2, case["n"], case["seed"])
    return x1, x2, pose0, _cam(case["camera1"], c1), _cam(case["camera2"], c2), c1, c2


@pytest.mark.gpu
@pytest.mark.parametrize("n", [500, 6000])
@pytest.mark.parametrize("loss", list(RG.LOSSES))
@pytest.mark.parametrize("pair", RG.PAIRS, ids=["%s-%s" % p for p in RG.PAIRS])
def test_refine_relpose_pair_matches_reference(pair, loss, n):
    for case in [c for c in GOLD["refine"] if (c["camera1"], c["camera2"], c["loss"], c["n"]) == (*pair, loss, n)]:
        flags = case["flags"]
        x1, x2, pose0, cam1, cam2, _, _ = _inputs(case)
        b = cabi.BundleOpt(loss_type=loss, loss_scale=GOLD["loss_scale"], relative_cost_tol=GOLD["relative_cost_tol"],
                           refine_intrinsics=flags)
        pose, p1, p2, bs = cabi.refine_relpose_pair(pose0, x1, x2, cam1, cam2, b)
        tag = (pair, loss, n, flags)
        assert int(bs[0]) == case["iterations"], (tag, bs, case["iterations"])
        assert np.isclose(bs[1], case["initial_cost"], rtol=1e-10, atol=0), tag
        assert np.isclose(bs[2], case["cost"], rtol=1e-7, atol=0), tag
        assert _close(pose, case["pose"], 1e-6), (tag, pose, case["pose"])
        assert _close(p1, case["params1"], 1e-6), (tag, p1, case["params1"])
        assert _close(p2, case["params2"], 1e-6), (tag, p2, case["params2"])


@pytest.mark.gpu
@pytest.mark.parametrize("pair", [("SIMPLE_PINHOLE", "SIMPLE_PINHOLE"), ("PINHOLE", "SIMPLE_PINHOLE"),
                                  ("NULL", "NULL")])
def test_empty_selection_is_the_fixed_camera_refiner(pair):
    """Flags that select no parameter of either camera (extra parameters of pinhole cameras, or NULL cameras) run the
    refiner of plb_refine_relpose_cameras and leave both cameras untouched."""
    m = [MODELS.get(p, 0) for p in pair]
    x1, x2, pose0, c1, c2 = RG.pair_problem(m[0], m[1], 900, 3)
    if pair[0] == "NULL":
        x1, x2 = x1 / 800.0, x2 / 800.0
        c1 = c2 = ()
    cam1, cam2 = _cam(pair[0], c1), _cam(pair[1], c2)
    base_pose, base_bs = cabi.refine_relpose_cameras(pose0, x1, x2, cam1, cam2, cabi.BundleOpt())
    for flags in (4, 7) if pair[0] == "NULL" else (4,):
        pose, p1, p2, bs = cabi.refine_relpose_pair(pose0, x1, x2, cam1, cam2, cabi.BundleOpt(refine_intrinsics=flags))
        assert np.array_equal(pose, base_pose) and np.array_equal(bs, base_bs), flags
        assert np.array_equal(p1, np.asarray(c1, float)) and np.array_equal(p2, np.asarray(c2, float)), flags


@pytest.mark.gpu
def test_refine_relpose_cameras_still_rejects_the_flags():
    case = GOLD["refine"][0]
    x1, x2, pose0, cam1, cam2, _, _ = _inputs(case)
    with pytest.raises(cabi.PoseLibB200Error) as e:
        cabi.refine_relpose_cameras(pose0, x1, x2, cam1, cam2, cabi.BundleOpt(refine_intrinsics=1))
    assert e.value.code == cabi.PLB_ERR_NYI and "plb_refine_relpose_pair" in str(e.value)


def _estimate_inputs(case):
    m1, m2 = MODELS[case["camera1"]], MODELS[case["camera2"]]
    x1, x2, _, c1, c2 = RG.pair_problem(m1, m2, RG.ESTIMATE_N, case["seed"], outliers=0.3)
    return x1, x2, _cam(case["camera1"], c1), _cam(case["camera2"], c2), c1, c2, cabi.RansacOpt(**RG.ESTIMATE_RANSAC)


@pytest.mark.gpu
@pytest.mark.parametrize("pair", RG.PAIRS, ids=["%s-%s" % p for p in RG.PAIRS])
def test_estimate_relative_pose_pair_matches_reference(pair):
    for case in [c for c in GOLD["estimate_cases"] if (c["camera1"], c["camera2"]) == pair]:
        flags = case["flags"]
        x1, x2, cam1, cam2, c1, c2, ro = _estimate_inputs(case)
        g = cabi.estimate_relative_pose_pair(x1, x2, cam1, cam2, ro, cabi.BundleOpt(refine_intrinsics=flags),
                                             RG.ESTIMATE_MAX_ERROR)
        for key in ("iterations", "refinements", "num_inliers"):
            assert g["stats"][key] == case[key], (pair, flags, key)
        mask = np.unpackbits(np.frombuffer(bytes.fromhex(case["inliers"]), dtype=np.uint8))[:RG.ESTIMATE_N]
        assert np.array_equal(g["inliers"].astype(np.uint8), mask), (pair, flags)
        assert _close(g["model"], case["pose"], 1e-6), (pair, flags, g["model"], case["pose"])
        assert _close(g["camera1"], case["params1"], 1e-6), (pair, flags, g["camera1"], case["params1"])
        assert _close(g["camera2"], case["params2"], 1e-6), (pair, flags, g["camera2"], case["params2"])
        # RANSAC (its LO included) keeps the cameras fixed: its outcome is plb_estimate_relative_pose's
        base = cabi.estimate("relpose", x1, x2, ro, cabi.BundleOpt(), RG.ESTIMATE_MAX_ERROR, cam1=cam1, cam2=cam2,
                             tangent_sampson=True)
        assert np.array_equal(g["inliers"], base["inliers"]) and g["stats"] == base["stats"], (pair, flags)
        if flags == 0:  # plb_estimate_relative_pose itself, cameras untouched
            assert np.array_equal(g["model"], base["model"])
            assert np.array_equal(g["camera1"], np.asarray(c1)) and np.array_equal(g["camera2"], np.asarray(c2))


@pytest.mark.gpu
def test_estimate_relative_pose_pair_fast_and_exact_modes_agree():
    case = [c for c in GOLD["estimate_cases"] if c["flags"] == 7][-1]
    x1, x2, cam1, cam2, _, _, ro = _estimate_inputs(case)
    b = cabi.BundleOpt(refine_intrinsics=7)
    out = {}
    try:
        for mode in ("exact", "fast"):
            cabi.set_mode(mode)
            out[mode] = cabi.estimate_relative_pose_pair(x1, x2, cam1, cam2, ro, b, RG.ESTIMATE_MAX_ERROR)
    finally:
        cabi.set_mode("fast")
    for key in ("model", "camera1", "camera2", "inliers"):
        assert np.array_equal(out["exact"][key], out["fast"][key]), key
    assert out["exact"]["stats"] == out["fast"]["stats"]


@pytest.mark.gpu
def test_estimate_relative_pose_pair_without_tangent_sampson_leaves_the_cameras():
    case = GOLD["estimate_cases"][-1]
    x1, x2, cam1, cam2, c1, c2, ro = _estimate_inputs(case)
    g = cabi.estimate_relative_pose_pair(x1, x2, cam1, cam2, ro, cabi.BundleOpt(refine_intrinsics=7),
                                         RG.ESTIMATE_MAX_ERROR, tangent_sampson=False)
    base = cabi.estimate("relpose", x1, x2, ro, cabi.BundleOpt(), RG.ESTIMATE_MAX_ERROR, cam1=cam1, cam2=cam2)
    assert np.array_equal(g["model"], base["model"]) and np.array_equal(g["inliers"], base["inliers"])
    assert np.array_equal(g["camera1"], np.asarray(c1)) and np.array_equal(g["camera2"], np.asarray(c2))


def _build_adapter_client(tmp_path):
    exe = str(tmp_path / "adapter_relpose_intrinsics_test")
    lib_dir = os.path.join(RG.ROOT, "poselib_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(HERE, "adapter_relpose_intrinsics_test.cc"),
                           "-o", exe, "-L" + lib_dir, "-lposelib_b200", "-Wl,-rpath," + lib_dir])
    return exe


def test_adapter_relpose_pair_compiles_and_links(tmp_path):
    out = subprocess.run([_build_adapter_client(tmp_path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "adapter relpose intrinsics link ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_adapter_refines_the_pair_and_estimates_with_the_flags(tmp_path):
    out = subprocess.run([_build_adapter_client(tmp_path), "run"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "adapter relpose intrinsics run ok" in out.stdout, (out.returncode,
                                                                                        out.stdout + out.stderr)
