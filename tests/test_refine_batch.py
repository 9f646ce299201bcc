"""plb_refine_batch / plb_refine_batch_device: the robust/bundle.h refiners over a batch of independent problems, and
the adapter's refine_relpose_batch / bundle_adjust_image_batch.

  * CPU: the ctypes struct against the header (a C program prints sizeof / offsetof), every argument check before any
    device call with every status set and nothing else written, and the adapter templates against stand-in types.
  * GPU: each problem of a mixed batch (every refiner, pinhole / radial / fisheye / division cameras, every
    refine_intrinsics bit, weights and none, every loss, sizes at every cluster width) is its single call bit for bit,
    whatever the batch order, split, streams and n_gpus; the fixtures written by the reference's sources hold through one
    batch; the device form equals the host form (fp64 bit for bit, fp32 on the widened values), leaves its inputs alone,
    reads them after the caller's stream and rejects host, pinned and misaligned pointers."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)
import make_camera_models_golden as CM  # noqa: E402
import make_intrinsics_golden as MG  # noqa: E402
import make_lm_widths_golden as MW  # noqa: E402
import make_relpose_intrinsics_golden as RG  # noqa: E402
import make_weights_golden as WG  # noqa: E402
import reference_cases as RC  # noqa: E402

try:
    from poselib_b200 import cabi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)

REFINERS = list(cabi.REFINER)
LOSSES = ["TRIVIAL", "TRUNCATED", "HUBER", "CAUCHY"]
# 2048 / 2049 / 10000 / 40000: cluster widths 1 / 2 / 4 / 8 at 2048 points per CTA
SIZES = [0, 1, 7, 200, 2048, 2049, 10000, 40000]
IMAGE_CAMERAS = ["PINHOLE", "OPENCV", "RADIAL_FISHEYE", "DIVISION-"]
PAIR_CAMERAS = [("PINHOLE", "RADIAL"), ("RADIAL_FISHEYE", "RADIAL_FISHEYE"), ("DIVISION-", "RADIAL"),
                ("SIMPLE_RADIAL_FISHEYE", "SIMPLE_DIVISION+")]
FLAGS = [1, 2, 4, 7]


# ---- problems ------------------------------------------------------------------------------------------------------
def _slice(d, n):
    return dict(d, a=np.ascontiguousarray(d["a"][:n]), b=np.ascontiguousarray(d["b"][:n]))


def _problem(refiner, n, k):
    """Problem k of a refiner at n points: the loss, the weights, the flags and the cameras rotate with k."""
    m = max(n, 200)  # the scenes need some points; the small sizes are a prefix of a 200-point scene
    seed = 1000 * REFINERS.index(refiner) + k
    bopt = dict(loss_type=LOSSES[k % 4], max_iterations=40, relative_cost_tol=1e-8)
    p = {"refiner": refiner}
    if refiner == "bundle_image":
        cam = IMAGE_CAMERAS[k % 4]
        if cam == "OPENCV":
            I = WG.inputs("image", cam, m, seed)
            x, X, pose0, p0, name = I["a"], I["b"], I["model0"], I["params1"], I["model1"]
        else:
            x, X, pose0, p0 = CM.problem(cam, m, seed, outliers=0.05)
            name = CM.CAMERAS[cam][0]
        p.update(a=x, b=X, model=pose0, cam1=cabi.Camera(name, tuple(p0)))
        bopt.update(loss_scale=2.0, refine_intrinsics=FLAGS[(k // 2) % 4])
    elif refiner in ("relpose_cameras", "relpose_pair"):
        c1, c2 = PAIR_CAMERAS[k % 4]
        x1, x2, pose0, p1, p2 = CM.pair_problem(c1, c2, m, seed, outliers=0.05)
        p.update(a=x1, b=x2, model=pose0, cam1=cabi.Camera(CM.CAMERAS[c1][0], tuple(p1)),
                 cam2=cabi.Camera(CM.CAMERAS[c2][0], tuple(p2)))
        bopt.update(loss_scale=1.0, refine_intrinsics=FLAGS[(k // 2) % 4] if refiner == "relpose_pair" else 0)
    else:
        kind = {"bundle": "calibrated"}.get(refiner, refiner)
        I = WG.inputs(kind, "", m, seed)
        p.update(a=I["a"], b=I["b"], model=I["model0"])
        bopt.update(loss_scale=I["loss_scale"], refine_intrinsics=7)  # ignored by these refiners
    p = _slice(p, n)
    p["bundle"] = cabi.BundleOpt(**bopt)
    if k % 2 == 0:
        w = np.random.default_rng(seed).uniform(0.0, 2.0, n)
        w[::11] = 0.0
        p["weights"] = w
    return p


def mixed_batch():
    return [_problem(r, n, k) for r in REFINERS for k, n in enumerate(SIZES)]


def single(p):
    """The problem's single entry point: dict(model, bundle_stats, camera1, camera2)."""
    r, b, w = p["refiner"], p["bundle"], p.get("weights")
    c1, c2 = p.get("cam1") or cabi.Camera("NULL", ()), p.get("cam2") or cabi.Camera("NULL", ())
    p1, p2 = cabi._camera_params(c1), cabi._camera_params(c2)
    if r == "bundle_image":
        m, p1, bs = cabi.refine_image(p["model"], p["a"], p["b"], c1, b, weights=w)
    elif r == "relpose_pair":
        m, p1, p2, bs = cabi.refine_relpose_pair(p["model"], p["a"], p["b"], c1, c2, b, weights=w)
    elif r == "relpose_cameras":
        m, bs = cabi.refine_relpose_cameras(p["model"], p["a"], p["b"], c1, c2, b, weights=w)
    else:
        m, bs = cabi.refine({"bundle": "pnp"}.get(r, r), p["model"], p["a"], p["b"], b, weights=w)
    return {"model": m, "bundle_stats": bs, "camera1": p1, "camera2": p2}


def _bits(v):
    return np.ascontiguousarray(np.asarray(v, dtype=np.float64)).view(np.uint64)


def assert_same(got, ref, tag):
    for f in ("model", "bundle_stats", "camera1", "camera2"):
        assert np.array_equal(_bits(got[f]), _bits(ref[f])), (tag, f, got[f], ref[f])


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_struct_layout_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    fields = [f for f, _ in cabi.RefineProblem._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "poselib_b200.h"\nint main(void) {\n'
                   '    printf("%zu\\n", sizeof(plb_refine_problem));\n' +
                   "".join('    printf("%%zu\\n", offsetof(plb_refine_problem, %s));\n' % f for f in fields) +
                   '    printf("%d %d %d %d %d %d %d\\n", PLB_REFINER_BUNDLE, PLB_REFINER_BUNDLE_IMAGE, PLB_REFINER_RELPOSE,'
                   ' PLB_REFINER_RELPOSE_CAMERAS, PLB_REFINER_RELPOSE_PAIR, PLB_REFINER_FUNDAMENTAL, PLB_REFINER_HOMOGRAPHY);\n'
                   '    return 0;\n}\n')
    exe = str(tmp_path / "layout")
    subprocess.check_call(["cc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    out = subprocess.check_output([exe], text=True).split("\n")
    assert int(out[0]) == C.sizeof(cabi.RefineProblem)
    for f, line in zip(fields, out[1:]):
        assert int(line) == getattr(cabi.RefineProblem, f).offset, f
    assert [int(v) for v in out[1 + len(fields)].split()] == [cabi.REFINER[r] for r in REFINERS] == list(range(7))
    assert {"plb_refine_batch", "plb_refine_batch_device"} <= set(cabi.EXPORTS)


def _arr(problems):
    """A plb_refine_problem array of host problems (status and model set to sentinels), and what keeps it alive."""
    arr = (cabi.RefineProblem * len(problems))()
    keep = []
    for q, p in zip(arr, problems):
        aa, ap = cabi._d(p["a"])
        ba, bp = cabi._d(p["b"])
        keep.append((aa, ba))
        cabi._fill_refine_problem(q, p, len(aa))
        q.a, q.b = ap, bp
        q.status = 12345
        for k in range(9):
            q.model[k] = 7.0 + k
        for k in range(3):
            q.bundle_stats[k] = -1.0
    return arr, keep


def _untouched(arr, before, code):
    """Every status is `code` and every other byte of the array is as it was (`before`: bytes(arr) before the call)."""
    assert all(q.status == code for q in arr), [q.status for q in arr]
    for q in arr:
        q.status = 12345
    assert bytes(arr) == before


def _cpu_problems():
    rng = np.random.default_rng(5)
    x, X = rng.normal(size=(10, 2)), rng.normal(size=(10, 3)) + [0, 0, 5]
    pin = cabi.Camera("PINHOLE", (500.0, 500.0, 0.0, 0.0))
    out = []
    for r in REFINERS:
        p = {"refiner": r, "a": x, "b": X if r in ("bundle", "bundle_image") else x, "bundle": cabi.BundleOpt()}
        if r in ("bundle_image", "relpose_cameras", "relpose_pair"):
            p.update(cam1=pin, cam2=pin)
        out.append(p)
    return out


def test_argument_checks_run_before_the_device():
    lib = cabi.lib()
    assert lib.plb_refine_batch(None, C.c_size_t(3), -1, 8) == cabi.PLB_ERR_ARG
    assert lib.plb_refine_batch_device(None, C.c_size_t(3), cabi.DTYPE_F64, None, 8) == cabi.PLB_ERR_ARG
    assert lib.plb_refine_batch(None, C.c_size_t(0), -1, 8) == cabi.PLB_OK
    base = _cpu_problems()

    def check(problems, edit, code, form="both", n_gpus=-1, dtype=cabi.DTYPE_F64):
        rcs = []
        for f in ("host", "device"):
            if form not in ("both", f):
                continue
            arr, keep = _arr(problems)
            edit(arr)
            before = bytes(arr)
            if f == "host":
                rcs.append(lib.plb_refine_batch(arr, C.c_size_t(len(problems)), n_gpus, 8))
            else:
                rcs.append(lib.plb_refine_batch_device(arr, C.c_size_t(len(problems)), dtype, None, 8))
            _untouched(arr, before, code)
        assert rcs and all(rc == code for rc in rcs), (rcs, code)

    def set_(i, **kw):
        def edit(arr):
            for k, v in kw.items():
                setattr(arr[i], k, v)
        return edit

    for bad in (-1, 7):
        check(base, set_(3, refiner=bad), cabi.PLB_ERR_ARG)
    for i in range(len(base)):
        check(base, set_(i, a=None), cabi.PLB_ERR_ARG)
        check(base, set_(i, b=None), cabi.PLB_ERR_ARG)
    nyi = cabi.Camera(5, (500.0, 500.0, 0.0, 0.0))  # OPENCV_FISHEYE: not on the path
    for r, field in (("bundle_image", "camera1"), ("relpose_cameras", "camera1"), ("relpose_cameras", "camera2"),
                     ("relpose_pair", "camera2")):
        check(base, set_(REFINERS.index(r), **{field: nyi}), cabi.PLB_ERR_NYI)
    check(base, set_(REFINERS.index("relpose_cameras"), bundle=cabi.BundleOpt(refine_intrinsics=cabi.REFINE_FOCAL_LENGTH)),
          cabi.PLB_ERR_NYI)
    check(base, lambda arr: None, cabi.PLB_ERR_ARG, form="device", dtype=2)
    check(base, lambda arr: None, cabi.PLB_ERR_ARG, form="host", n_gpus=-2)
    # n = 0 needs no points; a camera the refiner does not read is not checked; PLB_REFINER_RELPOSE_CAMERAS without a
    # selection is fine: without a device these reach the device check
    if cabi.device_count() == 0:
        check(base, lambda arr: None, cabi.PLB_ERR_CUDA)
        check(base, set_(2, n=0, a=None, b=None), cabi.PLB_ERR_CUDA)
        check(base, set_(REFINERS.index("relpose"), camera1=nyi), cabi.PLB_ERR_CUDA)
        check(base, set_(REFINERS.index("bundle_image"), camera2=nyi), cabi.PLB_ERR_CUDA)
        check(base, lambda arr: None, cabi.PLB_ERR_CUDA, form="host", n_gpus=5)


def _adapter_build(tmp_path):
    exe = str(tmp_path / "adapter_refine_batch_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(HERE, "adapter_refine_batch_test.cc"),
                           "-o", exe, "-L" + os.path.join(ROOT, "poselib_b200"), "-lposelib_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "poselib_b200")])
    return exe


def test_adapter_batch_templates_compile_and_link(tmp_path):
    out = subprocess.run([_adapter_build(tmp_path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "adapter refine batch link ok" in out.stdout, out.stdout + out.stderr


def test_mixed_batch_covers_the_grid():
    probs = mixed_batch()
    assert {p["refiner"] for p in probs} == set(REFINERS)
    assert {len(p["a"]) for p in probs} == set(SIZES)
    assert {p["bundle"].loss_type for p in probs} == set(range(4))
    img = [p for p in probs if p["refiner"] == "bundle_image"]
    pair = [p for p in probs if p["refiner"] == "relpose_pair"]
    assert {p["cam1"].model_id for p in img} == {1, 4, 9, 101}
    assert {p["cam1"].model_id for p in pair} >= {1, 9, 101, 8}
    for group in (img, pair):
        assert {p["bundle"].refine_intrinsics for p in group} == set(FLAGS)
    assert any("weights" in p for p in probs) and any("weights" not in p for p in probs)


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _gpu():
    if cabi.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    cabi.set_device(0)


@pytest.fixture(scope="module")
def mixed():
    _gpu()
    probs = mixed_batch()
    return probs, [single(p) for p in probs]


@pytest.mark.gpu
def test_mixed_batch_is_the_single_calls_bitwise(mixed):
    probs, ref = mixed
    got = cabi.refine_batch(probs)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g["status"] == cabi.PLB_OK
        assert_same(g, r, (i, probs[i]["refiner"], len(probs[i]["a"])))
    assert any(r["bundle_stats"][0] > 0 for r in ref)
    assert any(not np.array_equal(g["camera1"], cabi._camera_params(p["cam1"]))
               for g, p in zip(got, probs) if p["refiner"] == "bundle_image")


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["reversed", "split", "streams1", "all_gpus"])
def test_batch_composition_does_not_change_the_bits(mixed, how):
    probs, ref = mixed
    idx = list(range(len(probs)))
    if how == "reversed":
        order = idx[::-1]
        got = dict(zip(order, cabi.refine_batch([probs[i] for i in order])))
    elif how == "split":  # sub-batches that mix sizes and refiners differently
        got = {}
        for part in (idx[0::3], idx[1::3], idx[2::3]):
            got.update(zip(part, cabi.refine_batch([probs[i] for i in part], streams=3)))
    elif how == "streams1":
        got = dict(zip(idx, cabi.refine_batch(probs, streams=1)))
    else:
        got = dict(zip(idx, cabi.refine_batch(probs, n_gpus=0, streams=8)))
    for i in idx:
        assert_same(got[i], ref[i], (how, i))


@pytest.mark.gpu
def test_n_gpus_above_the_device_count_is_an_argument_error():
    _gpu()
    probs = [_problem("relpose", 200, 1), _problem("homography", 200, 2)]
    arr, keep = _arr(probs)
    before = bytes(arr)
    assert cabi.lib().plb_refine_batch(arr, C.c_size_t(2), cabi.device_count() + 1, 8) == cabi.PLB_ERR_ARG
    _untouched(arr, before, cabi.PLB_ERR_ARG)


# the fixtures written by the reference's sources, at the bars of their single-call tests
def _close(a, b, rtol):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return a.shape == b.shape and np.all(np.abs(a - b) <= rtol * np.maximum(1.0, np.abs(b)))


def _hex(v):
    return np.array([float.fromhex(t) for t in v])


def _weights_cases():
    gold = json.load(open(WG.OUT))
    out = []
    for c in gold["cases"]:
        I = WG.inputs(c["kind"], c["camera"], c["n"], c["seed"])
        r = {"image": "bundle_image", "pair": "relpose_pair", "calibrated": "bundle", "mismatch": "relpose"}.get(c["kind"],
                                                                                                           c["kind"])
        p = {"refiner": r, "a": I["a"], "b": I["b"], "model": I["model0"], "weights": I["weights"],
             "bundle": cabi.BundleOpt(loss_type=c["loss"], loss_scale=I["loss_scale"],
                                      relative_cost_tol=gold["relative_cost_tol"], max_iterations=gold["max_iterations"],
                                      refine_intrinsics=c["flags"])}
        if c["kind"] in ("image", "pair"):
            p["cam1"] = cabi.Camera(I["model1"], tuple(I["params1"]))
        if c["kind"] == "pair":
            p["cam2"] = cabi.Camera(I["model2"], tuple(I["params2"]))
        out.append((p, c))
    return out


def _check_weights_case(g, c):
    tag = (c["kind"], c["camera"], c["flags"], c["loss"], c["n"])
    bs = g["bundle_stats"]
    if c["kind"] in ("image", "pair"):
        assert int(bs[0]) == c["iterations"], (tag, bs, c["iterations"])
        assert np.isclose(bs[1], float.fromhex(c["initial_cost"]), rtol=1e-10, atol=0), tag
        assert np.isclose(bs[2], float.fromhex(c["cost"]), rtol=1e-7, atol=0), tag
        assert _close(g["model"], _hex(c["model"]), 1e-6), tag
        assert _close(g["camera1"], _hex(c["params1"]), 1e-6), tag
        if c["kind"] == "pair":
            assert _close(g["camera2"], _hex(c["params2"]), 1e-6), tag
    else:
        RC.check_refine(g["model"], bs, dict(model=c["model"], initial_cost=c["initial_cost"], cost=c["cost"]),
                        model_tol=1e-6, cost0_rtol=1e-10, cost_rtol=1e-7)


def _lm_widths_cases():
    import test_lm_widths as LW
    gold = json.load(open(MW.OUT))
    out = []
    for c in gold["bundle"]:
        x, X, pose0, p0 = LW.pnp_camera_problem(c["camera"], c["n"], LW._pnp_seed(c["camera"], c["n"], c["flags"], c["loss"]))
        out.append(({"refiner": "bundle_image", "a": x, "b": X, "model": pose0,
                     "cam1": cabi.Camera(LW._model_name(c["camera"]), tuple(p0)),
                     "bundle": LW._bopt(c["loss"], LW.MG.LOSS_SCALE, c["flags"], 100)}, dict(c, params1=c["params"])))
    for c in gold["refine"]:
        pair = (c["camera1"], c["camera2"])
        x1, x2, pose0, c1, c2 = LW.pair_camera_problem(pair, c["n"], c["seed"])
        out.append(({"refiner": "relpose_pair", "a": x1, "b": x2, "model": pose0,
                     "cam1": cabi.Camera(LW._model_name(pair[0]), tuple(c1)),
                     "cam2": cabi.Camera(LW._model_name(pair[1]), tuple(c2)),
                     "bundle": LW._bopt(c["loss"], LW.MC.PAIR_LOSS_SCALE, c["flags"], 100)}, c))
    return out


def _check_lm_widths_case(g, c):
    tag = (c.get("camera"), c.get("camera1"), c["n"], c["flags"], c["loss"])
    bs = g["bundle_stats"]
    assert int(bs[0]) == c["iterations"], (tag, bs, c["iterations"])
    assert _close(bs[1], c["initial_cost"], 1e-10), tag
    assert _close(bs[2], c["cost"], 1e-7), tag
    assert _close(g["model"], c["pose"], 1e-6), tag
    assert _close(g["camera1"], c["params1"], 1e-6), tag
    if "params2" in c and "camera1" in c:
        assert _close(g["camera2"], c["params2"], 1e-6), tag


def _intrinsics_cases():
    """The bundle cases of reference_intrinsics.json, built as tests/test_intrinsics_refine.py builds them."""
    gold = json.load(open(MG.OUT))
    out = []
    for c in gold["bundle"]:
        x, X, pose0, p0, _ = MG.problem(MG.MODELS[c["model"]], c["n"], MG.bundle_seed(c["model"], c["n"], c["flags"], c["loss"]))
        out.append(({"refiner": "bundle_image", "a": x, "b": X, "model": pose0, "cam1": cabi.Camera(c["model"], tuple(p0)),
                     "bundle": cabi.BundleOpt(loss_type=c["loss"], loss_scale=gold["loss_scale"],
                                              relative_cost_tol=gold["relative_cost_tol"], refine_intrinsics=c["flags"])},
                    dict(c, params1=c["params"])))
    return out


def _relpose_intrinsics_cases():
    """The refine cases of reference_relpose_intrinsics.json, built as tests/test_relpose_intrinsics_refine.py builds
    them."""
    gold = json.load(open(RG.OUT))
    out = []
    for c in gold["refine"]:
        x1, x2, pose0, c1, c2 = RG.pair_problem(RG.MODELS[c["camera1"]], RG.MODELS[c["camera2"]], c["n"], c["seed"])
        out.append(({"refiner": "relpose_pair", "a": x1, "b": x2, "model": pose0,
                     "cam1": cabi.Camera(c["camera1"], tuple(c1)), "cam2": cabi.Camera(c["camera2"], tuple(c2)),
                     "bundle": cabi.BundleOpt(loss_type=c["loss"], loss_scale=gold["loss_scale"],
                                              relative_cost_tol=gold["relative_cost_tol"], refine_intrinsics=c["flags"])},
                    c))
    return out


def _check_intrinsics_case(g, c):
    """The bars of test_bundle_adjust_image_matches_reference / test_refine_relpose_pair_matches_reference: iterations
    exactly, initial cost 1e-10 and cost 1e-7 relative, pose and camera parameters 1e-6."""
    tag = (c.get("model"), c.get("camera1"), c.get("camera2"), c["n"], c["flags"], c["loss"])
    bs = g["bundle_stats"]
    assert int(bs[0]) == c["iterations"], (tag, bs, c["iterations"])
    assert np.isclose(bs[1], c["initial_cost"], rtol=1e-10, atol=0), tag
    assert np.isclose(bs[2], c["cost"], rtol=1e-7, atol=0), tag
    assert _close(g["model"], c["pose"], 1e-6), tag
    assert _close(g["camera1"], c["params1"], 1e-6), tag
    if "params2" in c:
        assert _close(g["camera2"], c["params2"], 1e-6), tag


@pytest.mark.gpu
def test_reference_fixtures_hold_through_one_batch():
    _gpu()
    cases = [(p, c, _check_weights_case) for p, c in _weights_cases()] + \
        [(p, c, _check_lm_widths_case) for p, c in _lm_widths_cases()] + \
        [(p, c, _check_intrinsics_case) for p, c in _intrinsics_cases()] + \
        [(p, c, _check_intrinsics_case) for p, c in _relpose_intrinsics_cases()]
    got = cabi.refine_batch([p for p, _, _ in cases])
    for g, (p, c, check) in zip(got, cases):
        assert g["status"] == cabi.PLB_OK
        check(g, c)


# ---- device form -----------------------------------------------------------------------------------------------------
def _to_device(probs, dtype):
    import torch
    out = []
    for p in probs:
        q = dict(p)
        for k in ("a", "b", "weights"):
            if k in p:
                q[k] = torch.as_tensor(np.asarray(p[k], dtype=np.float64)).to(dtype).cuda()
        out.append(q)
    return out


def _widened(probs):
    out = []
    for p in probs:
        q = dict(p)
        for k in ("a", "b", "weights"):
            if k in p:
                q[k] = np.asarray(p[k], dtype=np.float64).astype(np.float32).astype(np.float64)
        out.append(q)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_device_form_is_the_host_form(mixed, dtype):
    import torch
    probs, ref = mixed
    tdt = getattr(torch, dtype)
    dev = _to_device(probs, tdt)
    before = [{k: v.clone() for k, v in p.items() if isinstance(v, torch.Tensor)} for p in dev]
    got = cabi.refine_batch_device(dev)
    torch.cuda.synchronize()
    want = ref if dtype == "float64" else cabi.refine_batch(_widened(probs))
    for i, (g, r) in enumerate(zip(got, want)):
        assert g["status"] == cabi.PLB_OK
        assert_same(g, r, (dtype, i))
    for p, b in zip(dev, before):  # read only
        for k, v in b.items():
            assert torch.equal(p[k], v), k


@pytest.mark.gpu
def test_device_form_reads_inputs_after_the_callers_stream(mixed):
    import torch
    probs, ref = mixed
    sel = [i for i, p in enumerate(probs) if len(p["a"]) in (200, 10000)]
    dev = _to_device([probs[i] for i in sel], torch.float64)
    side = torch.cuda.Stream()
    garbage = []
    with torch.cuda.stream(side):
        for p in dev:
            g = {k: torch.full_like(p[k], 1e3) for k in ("a", "b")}
            torch.cuda._sleep(20_000_000)  # keep the stream busy: the real values land well after the call is made
            g["a"].copy_(p["a"])
            g["b"].copy_(p["b"])
            garbage.append(g)
    calls = [dict(p, a=g["a"], b=g["b"]) for p, g in zip(dev, garbage)]
    got = cabi.refine_batch_device(calls, stream=side)
    for j, i in enumerate(sel):
        assert_same(got[j], ref[i], ("stream", i))


@pytest.mark.gpu
def test_device_form_rejects_host_pinned_and_misaligned_pointers():
    import torch
    _gpu()
    base = [_problem(r, 50, 1) for r in ("relpose", "bundle_image", "homography")]
    base[0]["weights"] = np.ones(50)
    lib = cabi.lib()

    def call(edit):
        arr, keep = _arr(base)
        dev = _to_device(base, torch.float64)
        for q, p in zip(arr, dev):
            q.a = C.cast(C.c_void_p(p["a"].data_ptr()), cabi._P)
            q.b = C.cast(C.c_void_p(p["b"].data_ptr()), cabi._P)
            if "weights" in p:
                q.weights = C.cast(C.c_void_p(p["weights"].data_ptr()), cabi._P)
        edit(arr, dev)
        before = bytes(arr)
        rc = lib.plb_refine_batch_device(arr, C.c_size_t(len(base)), cabi.DTYPE_F64, None, 8)
        return rc, arr, before

    host = np.zeros((50, 3))
    pinned = torch.zeros(50, 3, dtype=torch.float64).pin_memory()
    for field in ("a", "b", "weights"):
        for name, ptr in (("host", host.ctypes.data), ("pinned", pinned.data_ptr())):
            def edit(arr, dev, field=field, ptr=ptr):
                setattr(arr[0], field, C.cast(C.c_void_p(ptr), cabi._P))
            rc, arr, before = call(edit)
            assert rc == cabi.PLB_ERR_ARG, (field, name)
            _untouched(arr, before, cabi.PLB_ERR_ARG)

        def edit(arr, dev, field=field):
            setattr(arr[0], field, C.cast(C.c_void_p(dev[0][field].data_ptr() + 4), cabi._P))
        rc, arr, before = call(edit)
        assert rc == cabi.PLB_ERR_ARG, (field, "misaligned")
        _untouched(arr, before, cabi.PLB_ERR_ARG)
    rc, arr, _ = call(lambda arr, dev: None)
    assert rc == cabi.PLB_OK and all(q.status == cabi.PLB_OK for q in arr)


@pytest.mark.gpu
def test_adapter_batches_are_the_single_calls(tmp_path):
    out = subprocess.run([_adapter_build(tmp_path), "run"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "adapter refine batch run ok" in out.stdout, (out.returncode, out.stdout + out.stderr)
