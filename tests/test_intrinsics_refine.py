"""Camera-parameter refinement in the absolute-pose bundle adjustment (BundleOptions::refine_focal_length /
refine_principal_point / refine_extra_params): plb_bundle_adjust_image, plb_estimate_absolute_pose_image and the batch.

Reference: PoseLib's own sources (oracle/_ref/libplref2.so, the reference on mini-Eigen) through
tests/ref_intrinsics_client.cc, and their results on seeded problems in tests/golden/reference_intrinsics.json
(tests/golden/make_intrinsics_golden.py).
  * CPU, where the reference is mounted: the host build of camera.cuh's cam_jac_params / cam_refine_idx equals
    Camera::project_with_jac's jac_params / Camera::get_param_refinement_idx bit for bit, and the reference reproduces
    the fixture file bit for bit.
  * CPU, everywhere: the C-ABI surface and the argument checks that run before any device call.
  * GPU: the device path holds the fixture at the bars of test_lm_refiners_match_oracle, and the entry points that
    ignore the flags give the results they give without them."""
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
import make_intrinsics_golden as MG  # noqa: E402

try:
    from poselib_b200 import cabi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)

GOLD = json.load(open(MG.OUT))
MODELS = MG.MODELS
needs_reference = pytest.mark.skipif(
    not (MG.reference_available() and os.path.exists(os.path.join(MG.ROOT, "oracle", "_ref", "libplref2.so"))),
    reason="needs the reference checkout and oracle/_ref/libplref2.so")


def _cam(model, params):
    return cabi.Camera(model, tuple(params))


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return MG.build_client(str(tmp_path_factory.mktemp("ref_intrinsics")))


# ---- CPU ---------------------------------------------------------------------------------------------------
def test_exports_and_bundle_opt_layout():
    lib = cabi.lib()
    for name in ("plb_bundle_adjust_image", "plb_estimate_absolute_pose_image"):
        assert name in cabi.EXPORTS and hasattr(lib, name)
    assert C.sizeof(cabi.BundleOpt) == 72
    assert cabi.BundleOpt.refine_intrinsics.offset == 12
    b = cabi.BundleOpt(50, "HUBER", 2.0)  # positional construction keeps its meaning
    assert (b.max_iterations, b.loss_type, b.loss_scale, b.refine_intrinsics) == (50, 2, 2.0, 0)
    assert cabi.BundleOpt(refine_intrinsics=5).refine_intrinsics == 5
    d = cabi.BundleOpt(refine_intrinsics=7)
    lib.plb_bundle_opt_default(C.byref(d))
    assert d.refine_intrinsics == 0


@needs_reference
@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
@pytest.mark.parametrize("model", [-1, 0, 1, 2, 3, 4])
def test_device_camera_refinement_source_matches_poselib_bitwise(ref, model, tmp_path):
    exe = str(tmp_path / "camera_jac_host_test")
    subprocess.check_call(["nvcc", "-std=c++17", "-O2", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-Xcompiler", "-ffp-contract=off", "-o", exe, os.path.join(HERE, "camera_jac_host_test.cu")])
    params = np.zeros(8)
    if model >= 0:
        params[:MG.NUM_PARAMS[model]] = MG.TRUE_PARAMS[model]
    rng = np.random.RandomState(100 + model)
    Z = np.column_stack([rng.uniform(-2, 2, 50), rng.uniform(-2, 2, 50), rng.uniform(0.5, 6, 50)])
    out = subprocess.check_output([exe, str(model)] + [repr(float(v)) for v in params] +
                                  [repr(float(v)) for v in Z.reshape(-1)], text=True).splitlines()
    np_model = MG.NUM_PARAMS.get(model, 0)
    for flags in range(8):
        got = [int(t) for t in out[flags].split()[1:]]
        idx = np.zeros(8, dtype=np.int32)
        m = ref.ri_refine_idx(model, params.ctypes.data_as(C.POINTER(C.c_double)), flags,
                              idx.ctypes.data_as(C.POINTER(C.c_int)))
        assert got == [m] + idx[:m].tolist(), (model, flags)
    got = np.array([[float.fromhex(t) for t in line.split()[1:]] for line in out[8:]]).reshape(50, 2, 8)
    xp, jac, jp = np.zeros(100), np.zeros(300), np.zeros(800)
    Zc = np.ascontiguousarray(Z)
    ref.ri_project_with_jac(model, MG._p(params), C.c_int64(50), MG._p(Zc), MG._p(xp), MG._p(jac), MG._p(jp))
    jp = jp.reshape(50, 2, 8)
    assert np.array_equal(got[:, :, :np_model], jp[:, :, :np_model])


@needs_reference
def test_reference_reproduces_the_fixture_bitwise(ref):
    for case in GOLD["bundle"]:
        r = MG.ref_bundle_adjust(ref, case["model"], case["n"], case["flags"], case["loss"])
        assert r == case, case
    for case in GOLD["estimate_cases"]:
        r = MG.ref_estimate(ref, case["model"], case["flags"])
        assert r == case, case


def test_fixture_covers_every_model_flag_set_and_loss():
    keys = {(c["model"], c["flags"], c["loss"], c["n"]) for c in GOLD["bundle"]}
    assert len(keys) == 5 * 7 * 4 * 2
    # the problems start inside the basin: every run descends
    assert all(c["cost"] < c["initial_cost"] and c["iterations"] > 0 for c in GOLD["bundle"])


def _pts(n=10):
    x = np.zeros((n, 2))
    X = np.ones((n, 3))
    return x, X


def test_estimate_absolute_pose_rejects_refinement_flags():
    x, X = _pts()
    with pytest.raises(cabi.PoseLibB200Error) as e:
        cabi.estimate("pnp", x, X, cabi.RansacOpt(), cabi.BundleOpt(refine_intrinsics=1), 1.0,
                      cam1=_cam("PINHOLE", (500.0, 500.0, 0.0, 0.0)))
    assert e.value.code == cabi.PLB_ERR_ARG and "plb_estimate_absolute_pose_image" in str(e.value)


def test_camera_relative_pose_refinement_is_nyi():
    x, _ = _pts()
    c = _cam("PINHOLE", (500.0, 500.0, 0.0, 0.0))
    r = _cam("RADIAL", (500.0, 0.0, 0.0, 0.0, 0.0))
    with pytest.raises(cabi.PoseLibB200Error) as e:
        cabi.refine_relpose_cameras(None, x, x, c, c, cabi.BundleOpt(refine_intrinsics=2))
    assert e.value.code == cabi.PLB_ERR_NYI
    with pytest.raises(cabi.PoseLibB200Error) as e:
        cabi.estimate("relpose", x, x, cabi.RansacOpt(), cabi.BundleOpt(refine_intrinsics=4), 1.0, cam1=c, cam2=r,
                      tangent_sampson=True)
    assert e.value.code == cabi.PLB_ERR_NYI


# ---- GPU ---------------------------------------------------------------------------------------------------
def _close(a, b, rtol):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.all(np.abs(a - b) <= rtol * np.maximum(1.0, np.abs(b)))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [500, 6000])
@pytest.mark.parametrize("loss", list(MG.LOSSES))
@pytest.mark.parametrize("model", list(MODELS))
def test_bundle_adjust_image_matches_reference(model, loss, n):
    mid = MODELS[model]
    for case in [c for c in GOLD["bundle"] if (c["model"], c["loss"], c["n"]) == (model, loss, n)]:
        flags = case["flags"]
        x, X, pose0, p0, _ = MG.problem(mid, n, MG.bundle_seed(model, n, flags, loss))
        b = cabi.BundleOpt(loss_type=loss, loss_scale=GOLD["loss_scale"], relative_cost_tol=GOLD["relative_cost_tol"],
                           refine_intrinsics=flags)
        pose, params, bs = cabi.refine_image(pose0, x, X, _cam(model, p0), b)
        tag = (model, loss, n, flags)
        assert int(bs[0]) == case["iterations"], (tag, bs, case["iterations"])
        assert np.isclose(bs[1], case["initial_cost"], rtol=1e-10, atol=0), tag
        assert np.isclose(bs[2], case["cost"], rtol=1e-7, atol=0), tag
        assert _close(pose, case["pose"], 1e-6), (tag, pose, case["pose"])
        assert _close(params, case["params"], 1e-6), (tag, params, case["params"])


@pytest.mark.gpu
@pytest.mark.parametrize("model", list(MODELS))
def test_empty_selection_is_the_fixed_camera_refiner(model):
    """Flags that select no parameter of the model (extra parameters of a pinhole camera) change nothing."""
    mid = MODELS[model]
    x, X, pose0, p0, _ = MG.problem(mid, 800, 3)
    base = cabi.refine_image(pose0, x, X, _cam(model, p0), cabi.BundleOpt())
    flags = 4 if model in ("SIMPLE_PINHOLE", "PINHOLE") else 0
    again = cabi.refine_image(pose0, x, X, _cam(model, p0), cabi.BundleOpt(refine_intrinsics=flags))
    for a, b in zip(base, again):
        assert np.array_equal(a, b)
    assert np.array_equal(base[1], p0)


@pytest.mark.gpu
def test_entry_points_that_ignore_the_flags():
    x, X, pose0, _, _ = MG.problem(1, 600, 5)
    xn = x / 800.0
    a = cabi.refine("pnp", pose0, xn, X, cabi.BundleOpt())
    b = cabi.refine("pnp", pose0, xn, X, cabi.BundleOpt(refine_intrinsics=7))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    rng = np.random.RandomState(1)
    x1 = rng.uniform(0, 640, (300, 2))
    x2 = x1 + rng.normal(scale=1.0, size=x1.shape)
    for kind in ("relpose", "homography", "fundamental"):
        a = cabi.refine(kind, None, x1 / 800.0, x2 / 800.0, cabi.BundleOpt())
        b = cabi.refine(kind, None, x1 / 800.0, x2 / 800.0, cabi.BundleOpt(refine_intrinsics=7))
        assert np.array_equal(a[0], b[0], equal_nan=True) and np.array_equal(a[1], b[1], equal_nan=True), kind
    cam = _cam("RADIAL", MG.TRUE_PARAMS[3])
    ro = cabi.RansacOpt(max_iterations=500, min_iterations=50, seed=4)
    for kind, kw in (("relpose", dict(cam1=cam, cam2=cam)), ("homography", {}), ("fundamental", {})):
        a = cabi.estimate(kind, x1, x2, ro, cabi.BundleOpt(), 2.0, **kw)
        b = cabi.estimate(kind, x1, x2, ro, cabi.BundleOpt(refine_intrinsics=7), 2.0, **kw)
        assert np.array_equal(a["model"], b["model"]) and np.array_equal(a["inliers"], b["inliers"]), kind


def _estimate_inputs(model):
    x, X, _, p0, _ = MG.problem(MODELS[model], MG.ESTIMATE_N, MG.estimate_seed(model), outliers=0.3)
    return x, X, p0, cabi.RansacOpt(**MG.ESTIMATE_RANSAC)


@pytest.mark.gpu
@pytest.mark.parametrize("model", list(MODELS))
def test_estimate_absolute_pose_image_matches_reference(model):
    x, X, p0, ro = _estimate_inputs(model)
    base = cabi.estimate("pnp", x, X, ro, cabi.BundleOpt(), MG.ESTIMATE_MAX_ERROR, cam1=_cam(model, p0))
    for case in [c for c in GOLD["estimate_cases"] if c["model"] == model]:
        flags = case["flags"]
        g = cabi.estimate_image(x, X, _cam(model, p0), ro, cabi.BundleOpt(refine_intrinsics=flags), MG.ESTIMATE_MAX_ERROR)
        for key in ("iterations", "refinements", "num_inliers"):
            assert g["stats"][key] == case[key], (flags, key)
        mask = np.unpackbits(np.frombuffer(bytes.fromhex(case["inliers"]), dtype=np.uint8))[:MG.ESTIMATE_N]
        assert np.array_equal(g["inliers"].astype(np.uint8), mask), flags
        assert _close(g["model"], case["pose"], 1e-6), (flags, g["model"], case["pose"])
        assert _close(g["camera"], case["params"], 1e-6), (flags, g["camera"], case["params"])
        if flags == 0:  # the pose of plb_estimate_absolute_pose; the camera of the reference's rescale round trip
            assert np.array_equal(g["model"], base["model"])
            assert np.array_equal(g["camera"], np.array(case["params"]))


@pytest.mark.gpu
def test_estimate_batch_mixes_refined_and_fixed_cameras():
    probs, singles = [], []
    for i, model in enumerate(["PINHOLE", "OPENCV", "SIMPLE_RADIAL", "RADIAL"]):
        x, X, p0, ro = _estimate_inputs(model)
        flags = [3, 0, 7, 0][i]
        cam = _cam(model, p0)
        probs.append(dict(kind="pnp", a=x, b=X, ransac=ro, bundle=cabi.BundleOpt(refine_intrinsics=flags),
                          max_error=MG.ESTIMATE_MAX_ERROR, cam1=cam))
        singles.append((cabi.estimate_image(x, X, cam, ro, cabi.BundleOpt(refine_intrinsics=flags),
                                            MG.ESTIMATE_MAX_ERROR), flags, p0))
    out = cabi.estimate_batch(probs)
    for o, (s, flags, p0) in zip(out, singles):
        assert np.array_equal(o["model"], s["model"]) and np.array_equal(o["inliers"], s["inliers"])
        assert o["stats"] == s["stats"]
        if flags:
            assert np.array_equal(o["camera1"], s["camera"])
        else:
            assert np.array_equal(o["camera1"], np.asarray(p0)), "camera1 of an unflagged problem is left untouched"


@pytest.mark.gpu
def test_estimate_batch_tangent_sampson_camera_refinement_is_nyi():
    x, X, p0, ro = _estimate_inputs("RADIAL")
    cam = _cam("RADIAL", p0)
    prob = dict(kind="relpose", a=x, b=x, ransac=ro, bundle=cabi.BundleOpt(refine_intrinsics=4), max_error=2.0,
                cam1=cam, cam2=cam, tangent_sampson=True)
    with pytest.raises(cabi.PoseLibB200Error) as e:
        cabi.estimate_batch([prob])
    assert e.value.code == cabi.PLB_ERR_NYI
