"""PoseLib's per-residual weights in the LM refiners: plb_bundle_adjust_image_weighted, plb_refine_relpose_weighted,
plb_refine_relpose_cameras_weighted, plb_refine_relpose_pair_weighted, plb_refine_fundamental_weighted,
plb_refine_homography_weighted, the weights= keyword of cabi and the adapter's weights argument.

Reference: PoseLib's own sources (oracle/_ref/libplref2.so, the reference on mini-Eigen) through
tests/ref_weights_client.cc, and their results on seeded problems in tests/golden/reference_weights.json
(tests/golden/make_weights_golden.py).
  * CPU, where the reference is mounted: the reference reproduces the fixture bit for bit.
  * CPU, everywhere: the exports, and the argument checks that run before any device call.
  * GPU: every weighted entry point holds the fixture at the bars of its unweighted counterpart's fixture test; weights
    that are all 1.0 give the unweighted call bit for bit, on one CTA and on a cluster of several; zero weights keep
    their points' rows in the residual count; the adapter routes weights of size n to the weighted entry points."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_weights_golden as WG  # noqa: E402
import reference_cases as RC  # noqa: E402

try:
    from poselib_b200 import cabi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)

GOLD = json.load(open(WG.OUT))
CASES = GOLD["cases"]
WEIGHTED = ("plb_bundle_adjust_image_weighted", "plb_refine_relpose_weighted", "plb_refine_relpose_cameras_weighted",
            "plb_refine_relpose_pair_weighted", "plb_refine_fundamental_weighted", "plb_refine_homography_weighted")
needs_reference = pytest.mark.skipif(
    not (WG.MG.reference_available() and os.path.exists(os.path.join(WG.ROOT, "oracle", "_ref", "libplref2.so"))),
    reason="needs the reference checkout and oracle/_ref/libplref2.so")


def _key(c):
    return (c["kind"], c["camera"], c["flags"], c["loss"], c["n"])


# ---- CPU ---------------------------------------------------------------------------------------------------
def test_exports():
    lib = cabi.lib()
    for name in WEIGHTED:
        assert name in cabi.EXPORTS and hasattr(lib, name), name
    assert not hasattr(lib, "plb_bundle_adjust_weighted")  # the reference's calibrated bundle_adjust drops its weights


def test_argument_checks_run_before_the_device():
    """n > 0 with a null point array is PLB_ERR_ARG; null weights are not an error (uniform weights)."""
    P = C.POINTER(C.c_double)
    x = np.zeros((10, 3))
    w = np.ones(10)
    pose, bs = np.r_[1.0, np.zeros(8)], np.zeros(3)
    xp, wp, mp, bp = (a.ctypes.data_as(P) for a in (x, w, pose, bs))
    b = cabi.BundleOpt()
    c1, c2 = cabi.Camera("PINHOLE", (500.0, 500.0, 0.0, 0.0)), cabi.Camera("PINHOLE", (500.0, 500.0, 0.0, 0.0))
    lib, n = cabi.lib(), C.c_size_t(10)
    calls = {
        "plb_bundle_adjust_image_weighted": lambda a, b_, wt: lib.plb_bundle_adjust_image_weighted(
            a, b_, n, mp, C.byref(c1), C.byref(b), bp, wt),
        "plb_refine_relpose_weighted": lambda a, b_, wt: lib.plb_refine_relpose_weighted(a, b_, n, mp, C.byref(b), bp, wt),
        "plb_refine_relpose_cameras_weighted": lambda a, b_, wt: lib.plb_refine_relpose_cameras_weighted(
            a, b_, n, C.byref(c1), C.byref(c2), mp, C.byref(b), bp, wt),
        "plb_refine_relpose_pair_weighted": lambda a, b_, wt: lib.plb_refine_relpose_pair_weighted(
            a, b_, n, C.byref(c1), C.byref(c2), mp, C.byref(b), bp, wt),
        "plb_refine_fundamental_weighted": lambda a, b_, wt: lib.plb_refine_fundamental_weighted(
            a, b_, n, mp, C.byref(b), bp, wt),
        "plb_refine_homography_weighted": lambda a, b_, wt: lib.plb_refine_homography_weighted(
            a, b_, n, mp, C.byref(b), bp, wt),
    }
    assert set(calls) == set(WEIGHTED)
    for name, call in calls.items():
        for a, b_ in ((None, xp), (xp, None)):
            assert call(a, b_, wp) == cabi.PLB_ERR_ARG, name
            assert call(a, b_, None) == cabi.PLB_ERR_ARG, name
        if cabi.device_count() == 0:  # no CPU fallback; null weights pass the argument checks
            assert call(xp, xp, None) == cabi.PLB_ERR_CUDA, name
            assert call(xp, xp, wp) == cabi.PLB_ERR_CUDA, name
    assert lib.plb_bundle_adjust_image_weighted(xp, xp, n, mp, None, C.byref(b), bp, wp) == cabi.PLB_ERR_ARG
    assert lib.plb_refine_relpose_pair_weighted(xp, xp, n, C.byref(c1), None, mp, C.byref(b), bp, wp) == cabi.PLB_ERR_ARG


def test_fixture_covers_every_refiner_loss_size_and_camera():
    keys = {_key(c) for c in CASES}
    assert keys == set(WG.cases()) and len(keys) == len(CASES)
    assert {c["camera"] for c in CASES if c["kind"] == "image"} == {"NULL", "PINHOLE", "OPENCV", "RADIAL_FISHEYE"}
    for c in CASES:  # zero weights, down-weighted outliers
        w = WG.inputs(c["kind"], c["camera"], c["n"], c["seed"])["weights"]
        assert 0.05 < np.mean(w == 0) < 0.15 and w.max() <= 3.0, _key(c)
        assert np.any((w > 0) & (w < 0.1 * 0.5)), _key(c)
    assert all(c["iterations"] > 0 for c in CASES if c["kind"] in ("image", "pair"))


@needs_reference
def test_reference_reproduces_the_fixture_bitwise(tmp_path):
    lib = WG.build_client(str(tmp_path))
    for c in CASES:
        assert WG.ref_case(lib, _key(c), c["seed"]) == c, _key(c)


# ---- GPU ---------------------------------------------------------------------------------------------------
def _gpu():
    if cabi.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    cabi.set_device(0)


def _bopt(c, I):
    return cabi.BundleOpt(loss_type=c["loss"], loss_scale=I["loss_scale"], relative_cost_tol=GOLD["relative_cost_tol"],
                          max_iterations=GOLD["max_iterations"], refine_intrinsics=c["flags"])


def _cams(I):
    cams = [cabi.Camera(I["model1"], tuple(I["params1"]))]
    if "model2" in I:
        cams.append(cabi.Camera(I["model2"], tuple(I["params2"])))
    return cams


def _run(c, I, weights):
    """The case's refiner on the device: (model, [camera parameters], [iterations, initial_cost, cost])."""
    b = _bopt(c, I)
    if c["kind"] == "image":
        m, p, bs = cabi.refine_image(I["model0"], I["a"], I["b"], _cams(I)[0], b, weights=weights)
        return m, [p], bs
    if c["kind"] == "pair":
        m, p1, p2, bs = cabi.refine_relpose_pair(I["model0"], I["a"], I["b"], *_cams(I), b, weights=weights)
        return m, [p1, p2], bs
    kind = {"calibrated": "pnp", "mismatch": "relpose"}.get(c["kind"], c["kind"])
    m, bs = cabi.refine(kind, I["model0"], I["a"], I["b"], b, weights=weights)
    return m, [], bs


def _close(a, b, rtol):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.all(np.abs(a - b) <= rtol * np.maximum(1.0, np.abs(b)))


def _hex(v):
    return np.array([float.fromhex(t) for t in v])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["image", "pair", "relpose", "fundamental", "homography", "calibrated", "mismatch"])
def test_weighted_refiners_match_the_fixture(kind):
    """Camera cases at the bars of test_bundle_adjust_image_matches_reference (iterations exactly, initial cost 1e-10,
    cost 1e-7, pose and parameters 1e-6); the others at those of the reference-sources refine fixture (initial cost
    1e-10, cost 1e-7, model 1e-6)."""
    _gpu()
    for c in [c for c in CASES if c["kind"] == kind]:
        I = WG.inputs(c["kind"], c["camera"], c["n"], c["seed"])
        m, params, bs = _run(c, I, I["weights"])
        tag = _key(c)
        if kind in ("image", "pair"):
            assert int(bs[0]) == c["iterations"], (tag, bs, c["iterations"])
            assert np.isclose(bs[1], float.fromhex(c["initial_cost"]), rtol=1e-10, atol=0), tag
            assert np.isclose(bs[2], float.fromhex(c["cost"]), rtol=1e-7, atol=0), tag
            assert _close(m, _hex(c["model"]), 1e-6), (tag, m, c["model"])
            for i, p in enumerate(params):
                assert _close(p, _hex(c["params%d" % (i + 1)]), 1e-6), (tag, i, p)
        else:
            gold = dict(model=c["model"], initial_cost=c["initial_cost"], cost=c["cost"])
            RC.check_refine(m, bs, gold, model_tol=1e-6, cost0_rtol=1e-10, cost_rtol=1e-7)


# every weighted entry point, and every instantiation of the weighted kernel: the fixed-camera refiners of the five
# kinds, PnP on a fisheye camera, and the camera-refining PnP and tangent-Sampson refiners with and without one
ONES = [("image", "PINHOLE", 0), ("image", "PINHOLE", 7), ("image", "RADIAL_FISHEYE", 0), ("image", "RADIAL_FISHEYE", 7),
        ("image", "NULL", 0), ("pair", "", 0), ("pair", "", 7), ("fisheye_pair", "", 0), ("fisheye_pair", "", 7),
        ("cameras", "", 0), ("relpose", "", 0), ("fundamental", "", 0), ("homography", "", 0)]


def _ones_case(kind, camera, flags, n):
    """Inputs of a fixture case of the given kind (the fisheye pair and plb_refine_relpose_cameras: problems of
    make_camera_models_golden.py / the pair case); returns (case, inputs)."""
    base = {"fisheye_pair": "pair", "cameras": "pair"}.get(kind, kind)
    c = next(c for c in CASES if c["kind"] == base and c["n"] == n and c["loss"] == "CAUCHY" and c["flags"] == flags and
             (base != "image" or c["camera"] == camera))
    I = WG.inputs(c["kind"], c["camera"], n, c["seed"])
    if kind == "fisheye_pair":
        x1, x2, pose0, p1, p2 = WG.CM.pair_problem("RADIAL_FISHEYE", "RADIAL_FISHEYE", n, c["seed"])
        I.update(a=x1, b=x2, model0=pose0, model1=9, params1=p1, model2=9, params2=p2, loss_scale=2.0)
    return dict(c, kind=base), I


@pytest.mark.gpu
@pytest.mark.parametrize("n", [500, 6000])  # one CTA; a cluster of several
@pytest.mark.parametrize("kind,camera,flags", ONES, ids=["%s-%s-%d" % o for o in ONES])
def test_all_ones_weights_are_the_unweighted_call_bitwise(kind, camera, flags, n):
    _gpu()
    c, I = _ones_case(kind, camera, flags, n)
    ones = np.ones(n)
    if kind == "cameras":
        b = _bopt(dict(c, flags=0), I)
        got = cabi.refine_relpose_cameras(I["model0"], I["a"], I["b"], *_cams(I), b, weights=ones)
        ref = cabi.refine_relpose_cameras(I["model0"], I["a"], I["b"], *_cams(I), b)
        got, ref = (got[0], [], got[1]), (ref[0], [], ref[1])
    else:
        got, ref = _run(c, I, ones), _run(c, I, None)
    assert np.array_equal(got[0], ref[0]), (got[0], ref[0])
    for p, q in zip(got[1], ref[1]):
        assert np.array_equal(p, q), (p, q)
    assert np.array_equal(got[2], ref[2]), (got[2], ref[2])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["relpose", "homography"])
def test_zero_weights_count_their_rows(kind):
    """A zero weight is not a deleted point: its residual still counts in 1 / max(1, count), so the initial cost with
    zero weights is the cost of the kept points scaled by (n - zeros) / n, and the fixture's result is not the result
    of deleting those points."""
    _gpu()
    c = next(c for c in CASES if c["kind"] == kind and c["n"] == 500 and c["loss"] == "CAUCHY")
    I = WG.inputs(c["kind"], c["camera"], c["n"], c["seed"])
    w = I["weights"]
    keep = w != 0
    m_z, _, bs_z = _run(c, I, w)
    gold = dict(model=c["model"], initial_cost=c["initial_cost"], cost=c["cost"])
    RC.check_refine(m_z, bs_z, gold, model_tol=1e-6, cost0_rtol=1e-10, cost_rtol=1e-7)
    J = dict(I, a=I["a"][keep], b=I["b"][keep])
    m_d, _, bs_d = _run(c, J, w[keep])
    n, nk = len(w), int(keep.sum())
    assert nk < n
    assert np.isclose(bs_z[1] * n, bs_d[1] * nk, rtol=1e-12, atol=0), (bs_z, bs_d)
    assert bs_z[1] != bs_d[1] and bs_z[2] != bs_d[2]


def _adapter_build(tmp_path):
    exe = str(tmp_path / "adapter_weights_test")
    root = os.path.dirname(HERE)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(HERE, "adapter_weights_test.cc"), "-o", exe,
                           "-L" + os.path.join(root, "poselib_b200"), "-lposelib_b200",
                           "-Wl,-rpath," + os.path.join(root, "poselib_b200")])
    return exe


def test_adapter_weights_compile_and_link(tmp_path):
    out = subprocess.run([_adapter_build(tmp_path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "adapter weights link ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_adapter_routes_weights_to_the_weighted_entry_points(tmp_path):
    out = subprocess.run([_adapter_build(tmp_path), "run"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "adapter weights run ok" in out.stdout, (out.returncode, out.stdout + out.stderr)
