"""plb_score_batch / plb_score_batch_device: PoseLib's MSAC scorers and get_inliers over given models.

  * CPU: the ctypes struct against the header, every argument check before any device call (every status set, nothing
    else written), PLB_ERR_NYI for a camera off the path, PLB_ERR_CUDA without a device, and the fixture regenerated bit
    for bit from the reference's sources where the reference checkout exists.
  * GPU: counts and masks equal the fixture and the oracle, scores within the bound of two summation orders; the model
    RANSAC returns gets its recorded count, mask and (unless the final refinement replaced it) score; outputs do not depend on the batch, streams or devices; the device
    form equals the host form; more tiles than a grid dimension holds."""
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
import make_score_golden as SG  # noqa: E402

try:
    from poselib_b200 import cabi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)

U = 2.0 ** -53
with open(os.path.join(HERE, "golden", "reference_scores.json")) as f:
    FIXTURE = json.load(f)["cases"]


def _kind(k):
    return "relpose" if k == "tangent" else k


def fixture_problem(c, want_masks=True):
    """A score_batch problem dict of a fixture case, models as the C-ABI reads them ([m,7] or [r,c] matrices)."""
    I = SG.inputs(c["kind"], c["n"], c["pair"])
    rows = np.array([[float.fromhex(v) for v in mo] for mo in c["models"]])
    models = rows if rows.shape[1] == 7 else rows.reshape(-1, 3, 3).transpose(0, 2, 1)
    p = {"kind": _kind(c["kind"]), "a": I["a"], "b": I["b"], "models": models,
         "sq_threshold": float.fromhex(c["sq_threshold"]), "inliers": want_masks}
    if c["kind"] == "tangent":
        p.update(tangent_sampson=True, cam1=_camera(I["cam1"]), cam2=_camera(I["cam2"]))
    return p


def _camera(c):
    return cabi.Camera(int(c[0]), tuple(c[1]))


def _bits(v):
    return np.ascontiguousarray(np.asarray(v, dtype=np.float64)).view(np.uint64)


def assert_close_scores(got, ref, n, tag):
    """Two summation orders of n nonnegative terms differ by at most 2 n u times the sum."""
    got, ref = np.asarray(got), np.asarray(ref)
    nan = np.isnan(ref)
    assert np.array_equal(nan, np.isnan(got)), (tag, got, ref)
    assert np.all(np.abs(got[~nan] - ref[~nan]) <= 2 * max(n, 1) * U * np.abs(ref[~nan])), (tag, got, ref)


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_struct_layout_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    fields = [f for f, _ in cabi.ScoreProblem._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "poselib_b200.h"\nint main(void) {\n'
                   '    printf("%zu\\n", sizeof(plb_score_problem));\n' +
                   "".join('    printf("%%zu\\n", offsetof(plb_score_problem, %s));\n' % f for f in fields) +
                   '    return 0;\n}\n')
    exe = str(tmp_path / "layout")
    subprocess.check_call(["cc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    out = subprocess.check_output([exe], text=True).split()
    assert int(out[0]) == C.sizeof(cabi.ScoreProblem)
    for f, line in zip(fields, out[1:]):
        assert int(line) == getattr(cabi.ScoreProblem, f).offset, f
    assert {"plb_score_batch", "plb_score_batch_device"} <= set(cabi.EXPORTS)


def test_fixture_regenerates_bit_for_bit():
    if not os.path.isdir("/root/reference/PoseLib") or not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libplref2.so")):
        pytest.skip("needs the reference checkout and oracle/_ref/libplref2.so")
    assert SG.generate()["cases"] == FIXTURE


def test_fixture_covers_the_table():
    assert {c["kind"] for c in FIXTURE} == set(SG.KINDS)
    assert {c["n"] for c in FIXTURE} == set(SG.SIZES)
    assert {c["pair"] for c in FIXTURE if c["kind"] == "tangent"} == {0, 1}


def _cpu_problems():
    rng = np.random.default_rng(5)
    x, X = rng.normal(size=(10, 2)), rng.normal(size=(10, 3)) + [0, 0, 5]
    pose, H = np.array([[1.0, 0, 0, 0, 0, 0, 0]] * 2), np.eye(3)[None].repeat(2, 0)
    pin = cabi.Camera("PINHOLE", (500.0, 500.0, 0.0, 0.0))
    return [{"kind": "pnp", "a": x, "b": X, "models": pose}, {"kind": "relpose", "a": x, "b": x, "models": pose},
            {"kind": "relpose", "a": x, "b": x, "models": pose, "tangent_sampson": True, "cam1": pin, "cam2": pin},
            {"kind": "fundamental", "a": x, "b": x, "models": H}, {"kind": "homography", "a": x, "b": x, "models": H}]


def _arr(problems):
    arr = (cabi.ScoreProblem * len(problems))()
    keep = []
    for q, p in zip(arr, problems):
        aa, ap = cabi._d(p["a"])
        ba, bp = cabi._d(p["b"])
        mo = cabi._score_models(p["kind"], p["models"])
        sc, ct, mk = np.full(len(mo), 7.0), np.full(len(mo), 7, dtype=np.int64), np.full((len(mo), len(aa)), 7, np.int8)
        keep.append((aa, ba, mo, sc, ct, mk))
        cabi._fill_score_problem(q, dict(p, sq_threshold=1e-4), len(aa), len(mo))
        q.a, q.b, q.models = ap, bp, mo.ctypes.data_as(cabi._P)
        q.scores, q.num_inliers = sc.ctypes.data_as(cabi._P), ct.ctypes.data_as(C.POINTER(C.c_int64))
        q.inliers = C.cast(mk.ctypes.data_as(C.POINTER(C.c_char)), C.c_char_p)
        q.status = 12345
    return arr, keep


def test_argument_checks_run_before_the_device():
    lib = cabi.lib()
    assert lib.plb_score_batch(None, C.c_size_t(3), -1, 8) == cabi.PLB_ERR_ARG
    assert lib.plb_score_batch_device(None, C.c_size_t(3), cabi.DTYPE_F64, None, 8) == cabi.PLB_ERR_ARG
    assert lib.plb_score_batch(None, C.c_size_t(0), -1, 8) == cabi.PLB_OK
    base = _cpu_problems()

    def check(edit, code, form="both", n_gpus=-1, dtype=cabi.DTYPE_F64):
        rcs = []
        for f in ("host", "device"):
            if form not in ("both", f):
                continue
            arr, keep = _arr(base)
            edit(arr)
            before, outs = bytes(arr), [bytes(k[3]) + bytes(k[4]) + bytes(k[5]) for k in keep]
            if f == "host":
                rcs.append(lib.plb_score_batch(arr, C.c_size_t(len(base)), n_gpus, 8))
            else:
                rcs.append(lib.plb_score_batch_device(arr, C.c_size_t(len(base)), dtype, None, 8))
            assert all(q.status == code for q in arr), [q.status for q in arr]
            for q in arr:
                q.status = 12345
            assert bytes(arr) == before
            assert [bytes(k[3]) + bytes(k[4]) + bytes(k[5]) for k in keep] == outs
        assert rcs and all(rc == code for rc in rcs), (rcs, code)

    def set_(i, **kw):
        def edit(arr):
            for k, v in kw.items():
                setattr(arr[i], k, v)
        return edit

    for bad in (-1, 4):
        check(set_(1, kind=bad), cabi.PLB_ERR_ARG)
    for i in (0, 3, 4):  # the kinds other than relpose
        check(set_(i, tangent_sampson=1), cabi.PLB_ERR_ARG)
    for i in range(len(base)):
        for field in ("a", "b", "models", "scores", "num_inliers"):
            check(set_(i, **{field: None}), cabi.PLB_ERR_ARG)
    for thr in (float("nan"), float("inf"), -float("inf")):
        check(set_(2, sq_threshold=thr), cabi.PLB_ERR_ARG)
    check(set_(0, m=2 ** 31), cabi.PLB_ERR_ARG)
    check(set_(0, m=2 ** 40, n=2 ** 30), cabi.PLB_ERR_ARG)
    check(set_(0, n=2 ** 62, m=2 ** 30), cabi.PLB_ERR_ARG)  # m * n overflows
    nyi = cabi.Camera(5, (500.0, 500.0, 0.0, 0.0))  # OPENCV_FISHEYE: not on the path
    check(set_(2, camera1=nyi), cabi.PLB_ERR_NYI)
    check(set_(2, camera2=nyi), cabi.PLB_ERR_NYI)
    check(lambda arr: None, cabi.PLB_ERR_ARG, form="device", dtype=2)
    check(lambda arr: None, cabi.PLB_ERR_ARG, form="host", n_gpus=-2)
    if cabi.device_count() == 0:
        # n = 0 or m = 0 need no pointers; cameras are read only with tangent_sampson
        check(lambda arr: None, cabi.PLB_ERR_CUDA)
        check(set_(1, n=0, a=None, b=None), cabi.PLB_ERR_CUDA)
        check(set_(3, m=0, models=None, scores=None, num_inliers=None), cabi.PLB_ERR_CUDA)
        check(set_(1, camera1=nyi), cabi.PLB_ERR_CUDA)
        check(set_(0, inliers=None), cabi.PLB_ERR_CUDA)
        check(lambda arr: None, cabi.PLB_ERR_CUDA, form="host", n_gpus=5)


def _adapter_build(tmp_path):
    exe = str(tmp_path / "adapter_score_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(HERE, "adapter_score_test.cc"), "-o", exe,
                           "-L" + os.path.join(ROOT, "poselib_b200"), "-lposelib_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "poselib_b200")])
    return exe


def test_adapter_score_templates_compile_and_link(tmp_path):
    out = subprocess.run([_adapter_build(tmp_path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "adapter score link ok" in out.stdout, out.stdout + out.stderr


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _gpu():
    if cabi.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    cabi.set_device(0)


def assert_same(got, ref, tag):
    assert np.array_equal(_bits(got["scores"]), _bits(ref["scores"])), (tag, got["scores"], ref["scores"])
    assert np.array_equal(np.asarray(got["num_inliers"]), np.asarray(ref["num_inliers"])), tag
    if ref["inliers"] is None:
        assert got["inliers"] is None, tag
    else:
        assert np.array_equal(np.asarray(got["inliers"]), np.asarray(ref["inliers"])), tag


@pytest.mark.gpu
def test_fixture_counts_masks_and_scores():
    _gpu()
    res = cabi.score_batch([fixture_problem(c) for c in FIXTURE])
    for c, r in zip(FIXTURE, res):
        tag = (c["kind"], c["n"], c["pair"])
        assert r["num_inliers"].tolist() == c["counts"], (tag, r["num_inliers"], c["counts"])
        for j, h in enumerate(c["masks"]):
            assert np.array_equal(r["inliers"][j], SG.unpack(h, c["n"])), (tag, j)
        assert_close_scores(r["scores"], [float.fromhex(s) for s in c["scores"]], c["n"], tag)
        if c["n"] == 0:
            assert np.all(r["scores"] == 0) and np.all(r["num_inliers"] == 0)


def _scene(kind, n, m, seed):
    """n correspondences (30 % outliers) and m models: the truth, perturbed copies and random ones."""
    import make_intrinsics_golden as MG
    rng = np.random.RandomState(seed)
    q = np.concatenate([[1.0], rng.normal(scale=0.2, size=3)])
    q /= np.linalg.norm(q)
    R = MG.quat_to_rot(q)
    X = rng.uniform(-2, 2, size=(n, 3)) + [0, 0, 6]
    t = rng.normal(size=3) if kind == "pnp" else SG._unit(rng.normal(size=3))
    if kind == "homography":
        X[:, 2] = 6.0 + 0.3 * X[:, 0]
    Z = X @ R.T + t
    x2 = Z[:, :2] / Z[:, 2:] + rng.normal(scale=1e-3, size=(n, 2))
    bad = rng.uniform(size=n) < 0.3
    x2[bad] = rng.uniform(-0.5, 0.5, size=(int(bad.sum()), 2))
    if kind == "pnp":
        a, b, truth, sq = x2, X, np.concatenate([q, t]), 0.004 ** 2
    else:
        a, b, sq = X[:, :2] / X[:, 2:], x2, 0.003 ** 2
        truth = (np.concatenate([q, t]) if kind == "relpose" else
                 R + np.outer(t, np.array([-0.3, 0.0, 1.0]) / 6.0))
    msz = 7 if truth.ndim == 1 else 9
    flat = truth.reshape(-1) if msz == 7 else truth.T.reshape(-1)
    rows = flat + rng.normal(scale=1e-3, size=(m, msz)) * (rng.uniform(size=(m, 1)) < 0.7)
    rows[m // 2:] += rng.normal(size=(m - m // 2, msz)) * (rng.uniform(size=(m - m // 2, 1)) < 0.3)
    rows[:1] = flat
    if msz == 7:
        rows[:, :4] /= np.linalg.norm(rows[:, :4], axis=1, keepdims=True)
        models = rows
    else:
        models = rows.reshape(-1, 3, 3).transpose(0, 2, 1)
    return {"kind": kind, "a": np.ascontiguousarray(a), "b": np.ascontiguousarray(b), "models": models,
            "sq_threshold": sq, "inliers": True}


@pytest.mark.gpu
def test_oracle_on_larger_problems():
    import plo_py as P
    _gpu()
    probs = [_scene("relpose", 10000, 1000, 1), _scene("homography", 2000, 300, 2), _scene("pnp", 3000, 200, 3),
             _scene("fundamental", 3000, 100, 4)]
    probs += [_scene(k, 700, m, 10 + m) for m in range(1, 10) for k in ("relpose", "pnp")]
    for p, r in zip(probs, cabi.score_batch(probs)):
        n = len(p["a"])
        for j, mo in enumerate(p["models"]):
            s, cnt = P.score(p["kind"], mo, p["a"], p["b"], p["sq_threshold"])
            mask = P.inliers(p["kind"], mo, p["a"], p["b"], p["sq_threshold"])
            assert r["num_inliers"][j] == cnt, (p["kind"], j)
            assert np.array_equal(r["inliers"][j], np.asarray(mask[:n]) != 0), (p["kind"], j)
            assert_close_scores([r["scores"][j]], [s], n, (p["kind"], j))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_score_of_the_ransac_model_is_its_recorded_score(mode):
    import make_camera_models_golden as CM
    _gpu()
    cabi.set_mode(mode)
    try:
        ropt = cabi.RansacOpt(max_iterations=2000, min_iterations=100, seed=7)
        for kind in ("pnp", "relpose", "fundamental", "homography", "tangent"):
            if kind == "tangent":
                x1, x2, _, _, _ = CM.pair_problem("PINHOLE", "RADIAL", 1500, 17, outliers=0.3)
                c1, c2 = (cabi.Camera(CM.CAMERAS[c][0], tuple(CM.CAMERAS[c][1])) for c in ("PINHOLE", "RADIAL"))
                r = cabi.ransac_relpose_cameras(x1, x2, c1, c2, ropt, 2.0)
                p = {"kind": "relpose", "a": x1, "b": x2, "tangent_sampson": True, "cam1": c1, "cam2": c2}
            else:
                p = _scene(kind, 1500, 1, 40 + len(kind))
                r = cabi.ransac(kind, p["a"], p["b"], ropt, np.sqrt(p["sq_threshold"]))
                p = dict(p)
            max_error = 2.0 if kind == "tangent" else np.sqrt(p["sq_threshold"])
            p.update(models=r["model"][None], sq_threshold=max_error * max_error, inliers=True)
            s = cabi.score_batch([p])[0]
            st = r["stats"]
            assert s["num_inliers"][0] == st["num_inliers"], kind
            assert np.array_equal(s["inliers"][0], r["inliers"] != 0), kind
            # The final refinement replaces the model without recording its (lower) score (ransac_impl.h:190-198)
            assert s["scores"][0] == st["model_score"] or s["scores"][0] < st["model_score"], kind
            if st["refinements"] and s["scores"][0] != st["model_score"]:
                continue
            assert _bits(s["scores"][0]) == _bits(st["model_score"]), (kind, s["scores"][0], st["model_score"])
    finally:
        cabi.set_mode("fast")


def _mixed():
    probs = [fixture_problem(c, want_masks=(i % 3 != 1)) for i, c in enumerate(FIXTURE)]
    return probs + [_scene("relpose", 3000, 37, 5), _scene("pnp", 500, 0, 6)]


@pytest.mark.gpu
def test_outputs_do_not_depend_on_the_batch():
    _gpu()
    probs = _mixed()
    alone = [cabi.score_batch([p])[0] for p in probs]
    for kw in ({}, {"streams": 1}, {"streams": 3}):
        for i, r in enumerate(cabi.score_batch(probs, **kw)):
            assert_same(r, alone[i], (i, kw))
    for i, r in enumerate(cabi.score_batch(probs[::-1])[::-1]):
        assert_same(r, alone[i], ("reversed", i))
    if cabi.device_count() > 1:
        for i, r in enumerate(cabi.score_batch(probs, n_gpus=0)):
            assert_same(r, alone[i], ("all devices", i))
    cabi.set_device(0)


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if cabi.device_count() == 0 or not t.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    return t


def _on_device(torch, probs, dtype, stream=None):
    out = []
    for p in probs:
        q = dict(p)
        with torch.cuda.stream(stream) if stream is not None else _null():
            q["a"] = torch.tensor(p["a"], device="cuda:0").to(dtype)
            q["b"] = torch.tensor(p["b"], device="cuda:0").to(dtype)
            q["models"] = torch.tensor(np.asarray(p["models"], dtype=np.float64), device="cuda:0")
        out.append(q)
    return out


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_device_form_is_the_host_form(torch, dtype):
    _gpu()
    probs = _mixed()
    if dtype == "float32":  # the host form on the widened values
        probs = [dict(p, a=p["a"].astype(np.float32).astype(np.float64), b=p["b"].astype(np.float32).astype(np.float64))
                 for p in probs]
    host = cabi.score_batch(probs)
    side = torch.cuda.Stream()
    dev = _on_device(torch, probs, getattr(torch, dtype), stream=side)  # written on a side stream just before the call
    res = cabi.score_batch_device(dev, stream=side)
    torch.cuda.synchronize()
    for i, (r, h) in enumerate(zip(res, host)):
        got = {"scores": r["scores"].cpu().numpy(), "num_inliers": r["num_inliers"].cpu().numpy(),
               "inliers": None if r["inliers"] is None else r["inliers"].cpu().numpy()}
        assert_same(got, h, (dtype, i))


@pytest.mark.gpu
def test_more_tiles_than_a_grid_dimension(torch):
    _gpu()
    one = _scene("pnp", 40, 300000, 8)  # 75 000 tiles of 4 models
    many = [_scene("homography", 33, 3000, 20 + i) for i in range(100)]  # 750 tiles each, 75 000 in all
    for probs in ([one], many):
        res = cabi.score_batch(probs)
        for p, r in zip(probs[:3] + probs[-2:], res[:3] + res[-2:]):
            import plo_py as P
            for j in (0, 1, len(p["models"]) // 2, len(p["models"]) - 1):
                s, cnt = P.score(p["kind"], p["models"][j], p["a"], p["b"], p["sq_threshold"])
                mask = P.inliers(p["kind"], p["models"][j], p["a"], p["b"], p["sq_threshold"])
                n = len(p["a"])
                assert r["num_inliers"][j] == cnt and np.array_equal(r["inliers"][j], np.asarray(mask[:n]) != 0), j
                assert_close_scores([r["scores"][j]], [s], len(p["a"]), j)
        dev = cabi.score_batch_device(_on_device(torch, probs, torch.float64))
        for r, h in zip(dev, res):
            assert_same({k: None if v is None else v.cpu().numpy() for k, v in r.items() if k != "status"}, h, "device")


@pytest.mark.gpu
def test_adapter_score_templates_match_the_c_abi(tmp_path):
    _gpu()
    out = subprocess.run([_adapter_build(tmp_path), "run"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "adapter score ok" in out.stdout, out.stdout + out.stderr
