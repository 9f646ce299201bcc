"""plb_generate_batch / plb_generate_batch_device: the estimators' generate_models + score_model on caller-drawn samples.

  * CPU: the ctypes struct against the header, every argument check in its documented order (every status set, the
    outputs untouched), PLB_ERR_NYI for a camera off the path, PLB_ERR_CUDA without a device; the fixture written by the
    reference's own estimators (tests/golden/reference_generate.json) covers the table, its samples are
    plb_host_sample_table's, and it is regenerated bit for bit where the reference checkout exists.
  * GPU: model counts exactly and models within the solvers' tolerances against the fixture, and plb_score_batch on the
    fixture's models gives its counts exactly and its scores up to summation order; model counts and models against the
    oracle's solvers, counts exactly and scores within the bound of two
    summation orders against the oracle's scorers; the records equal plb_score_batch on the same models bit for bit; the
    real-focal-check run is the order-preserving subset of the run without it; outputs do not depend on the batch,
    streams, mode, chunking or the form of the call; slots past n_models keep their sentinel; an index out of range in the
    device form is an argument error that leaves every output untouched."""
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
sys.path.insert(0, os.path.join(ROOT, "oracle"))

try:
    from poselib_b200 import cabi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)

U = 2.0 ** -53
K, M = cabi.GENERATE_K, cabi.GENERATE_M


def _bits(v):
    return np.ascontiguousarray(np.asarray(v, dtype=np.float64)).view(np.uint64)


def _quat_rot(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def scene(kind, n, seed, outliers=0.3):
    """n correspondences of a random scene in normalised coordinates (PnP: x, X; else x1, x2), `outliers` of them
    replaced; a plane for the homography."""
    rng = np.random.RandomState(seed)
    q = np.concatenate([[1.0], rng.normal(scale=0.2, size=3)])
    R = _quat_rot(q / np.linalg.norm(q))
    X = rng.uniform(-2, 2, size=(n, 3)) + [0, 0, 6]
    if kind == "homography":
        X[:, 2] = 6.0 + 0.3 * X[:, 0]
    t = rng.normal(size=3)
    Z = X @ R.T + t
    x2 = Z[:, :2] / Z[:, 2:] + rng.normal(scale=1e-3, size=(n, 2))
    bad = rng.uniform(size=n) < outliers
    x2[bad] = rng.uniform(-0.5, 0.5, size=(int(bad.sum()), 2))
    a, b = (x2, X) if kind == "pnp" else (X[:, :2] / X[:, 2:], x2)
    return np.ascontiguousarray(a), np.ascontiguousarray(b)


def samples(kind, n, s, seed, prosac=False):
    """s minimal samples as PoseLib's RandomSampler draws them (plb_host_sample_table)."""
    opt = cabi.RansacOpt(seed=seed, progressive_sampling=prosac)
    return cabi.host_sample_table(n, K[kind], opt, s).astype(np.int32)


def problem(kind, n, s, seed, rfc=False, prosac=False):
    a, b = scene(kind, n, seed)
    thr = 0.004 if kind == "pnp" else 0.003
    return {"kind": kind, "a": a, "b": b, "samples": samples(kind, n, s, seed + 1000, prosac), "sq_threshold": thr * thr,
            "rfc": rfc}


def tangent_problem(cam1, cam2, n, s, seed):
    import make_camera_models_golden as CM
    x1, x2, _, _, _ = CM.pair_problem(cam1, cam2, n, seed, outliers=0.3)
    c1, c2 = (cabi.Camera(CM.CAMERAS[c][0], tuple(CM.CAMERAS[c][1])) for c in (cam1, cam2))
    return {"kind": "relpose", "a": x1, "b": x2, "samples": samples("relpose", n, s, seed + 1000), "sq_threshold": 4.0,
            "tangent_sampson": True, "cam1": c1, "cam2": c2}


with open(os.path.join(HERE, "golden", "reference_generate.json")) as f:
    FIXTURE = json.load(f)["cases"]


def fixture_problem(c):
    """The generate_batch problem of a fixture case: its scene, its recorded samples and max_error squared."""
    import make_generate_golden as GG
    I = GG.inputs(c["kind"], c["n"], c["pair"])
    me = float.fromhex(c["max_error"])
    kind = "relpose" if c["kind"] == "tangent" else c["kind"]
    smp = np.array([s["sample"] for s in c["samples"]], dtype=np.int32).reshape(-1, K[kind])
    p = {"kind": kind, "a": I["a"], "b": I["b"], "samples": smp, "sq_threshold": me * me, "rfc": bool(c["rfc"])}
    if c["kind"] == "tangent":
        p.update(tangent_sampson=True, cam1=cabi.Camera(int(I["cam1"][0]), tuple(I["cam1"][1])),
                 cam2=cabi.Camera(int(I["cam2"][0]), tuple(I["cam2"][1])))
    return p


def fixture_models(c, s):
    """A fixture sample's models as generate_batch returns them: [c,7] poses or [c,3,3] matrices [r,c]."""
    rows = np.array([[float.fromhex(v) for v in mo] for mo in s["models"]]).reshape(len(s["models"]), -1)
    return rows if c["kind"] not in ("fundamental", "homography") else rows.reshape(-1, 3, 3).transpose(0, 2, 1)


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_fixture_covers_the_table():
    import make_generate_golden as GG
    keys = {(c["kind"], c["n"], c["pair"], c["rfc"], c["prosac"]) for c in FIXTURE}
    assert keys == set(GG.cases())
    assert all(len(c["samples"]) >= GG.S // 2 for c in FIXTURE)
    for kind in ("pnp", "relpose", "tangent", "fundamental", "homography"):  # every solver gives models
        assert sum(s["n_models"] for c in FIXTURE if c["kind"] == kind for s in c["samples"]) > 20, kind


def test_fixture_samples_are_the_host_sample_table():
    import make_generate_golden as GG
    for c in FIXTURE:
        kind = "relpose" if c["kind"] == "tangent" else c["kind"]
        n = len(GG.inputs(c["kind"], c["n"], c["pair"])["a"])
        table = cabi.host_sample_table(n, K[kind], cabi.RansacOpt(seed=c["seed"], progressive_sampling=bool(c["prosac"])),
                                       GG.S)
        for s in c["samples"]:
            assert table[s["j"]].tolist() == s["sample"], (c["kind"], c["n"], s["j"])


def test_fixture_regenerates_bit_for_bit():
    if not os.path.isdir("/root/reference/PoseLib") or not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libplref2.so")):
        pytest.skip("needs the reference checkout and oracle/_ref/libplref2.so")
    import make_generate_golden as GG
    assert GG.generate()["cases"] == FIXTURE


def test_struct_layout_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    fields = [f for f, _ in cabi.GenerateProblem._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "poselib_b200.h"\nint main(void) {\n'
                   '    printf("%zu\\n", sizeof(plb_generate_problem));\n' +
                   "".join('    printf("%%zu\\n", offsetof(plb_generate_problem, %s));\n' % f for f in fields) +
                   '    return 0;\n}\n')
    exe = str(tmp_path / "layout")
    subprocess.check_call(["cc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    out = subprocess.check_output([exe], text=True).split()
    assert int(out[0]) == C.sizeof(cabi.GenerateProblem)
    for f, line in zip(fields, out[1:]):
        assert int(line) == getattr(cabi.GenerateProblem, f).offset, f
    assert {"plb_generate_batch", "plb_generate_batch_device"} <= set(cabi.EXPORTS)


def _cpu_problems():
    rng = np.random.default_rng(5)
    x, X = rng.normal(size=(10, 2)), rng.normal(size=(10, 3)) + [0, 0, 5]
    pin = cabi.Camera("PINHOLE", (500.0, 500.0, 0.0, 0.0))
    smp = lambda k: np.arange(2 * k, dtype=np.int32).reshape(2, k) % 10
    return [{"kind": "pnp", "a": x, "b": X, "samples": smp(3)}, {"kind": "relpose", "a": x, "b": x, "samples": smp(5)},
            {"kind": "relpose", "a": x, "b": x, "samples": smp(5), "tangent_sampson": True, "cam1": pin, "cam2": pin},
            {"kind": "fundamental", "a": x, "b": x, "samples": smp(7), "rfc": True},
            {"kind": "homography", "a": x, "b": x, "samples": smp(4)}]


def _arr(problems):
    arr = (cabi.GenerateProblem * len(problems))()
    keep = []
    for q, p in zip(arr, problems):
        aa, ap = cabi._d(p["a"])
        ba, bp = cabi._d(p["b"])
        smp = np.array(p["samples"], dtype=np.int32)  # a copy: the checks below edit it
        s, Mk = len(smp), M[p["kind"]]
        msz = 7 if p["kind"] in ("pnp", "relpose") else 9
        nm, mo = np.full(s, 7, np.int32), np.full(s * Mk * msz, 7.0)
        sc, ct = np.full(s * Mk, 7.0), np.full(s * Mk, 7, np.int64)
        keep.append((aa, ba, smp, nm, mo, sc, ct))
        cabi._fill_generate_problem(q, dict(p, sq_threshold=1e-4), len(aa), s)
        q.a, q.b, q.samples = ap, bp, smp.ctypes.data_as(C.POINTER(C.c_int32))
        q.n_models, q.models = nm.ctypes.data_as(C.POINTER(C.c_int32)), mo.ctypes.data_as(cabi._P)
        q.scores, q.num_inliers = sc.ctypes.data_as(cabi._P), ct.ctypes.data_as(C.POINTER(C.c_int64))
        q.status = 12345
    return arr, keep


def test_argument_checks_in_their_order():
    lib = cabi.lib()
    assert lib.plb_generate_batch(None, C.c_size_t(3), -1, 8) == cabi.PLB_ERR_ARG
    assert lib.plb_generate_batch_device(None, C.c_size_t(3), cabi.DTYPE_F64, None, 8) == cabi.PLB_ERR_ARG
    assert lib.plb_generate_batch(None, C.c_size_t(0), -1, 8) == cabi.PLB_OK
    base = _cpu_problems()
    no_gpu = cabi.device_count() == 0

    def check(edit, code, form="both", n_gpus=-1, dtype=cabi.DTYPE_F64):
        rcs = []
        for f in ("host", "device"):
            if form not in ("both", f):
                continue
            arr, keep = _arr(base)
            edit(arr)
            before, outs = bytes(arr), [b"".join(bytes(x) for x in k[3:]) for k in keep]
            if f == "host":
                rcs.append(lib.plb_generate_batch(arr, C.c_size_t(len(base)), n_gpus, 8))
            else:
                rcs.append(lib.plb_generate_batch_device(arr, C.c_size_t(len(base)), dtype, None, 8))
            assert all(q.status == rcs[-1] for q in arr), [q.status for q in arr]
            for q in arr:
                q.status = 12345
            assert bytes(arr) == before
            assert [b"".join(bytes(x) for x in k[3:]) for k in keep] == outs
        assert rcs and all(rc == code for rc in rcs), (rcs, code)

    def set_(i, **kw):
        def edit(arr):
            for k, v in kw.items():
                setattr(arr[i], k, v)
        return edit

    def both(*edits):
        def edit(arr):
            for e in edits:
                e(arr)
        return edit

    for bad in (-1, 4):
        check(set_(1, kind=bad), cabi.PLB_ERR_ARG)
    for i in (0, 3, 4):  # the kinds other than relpose
        check(set_(i, tangent_sampson=1), cabi.PLB_ERR_ARG)
    for i in (0, 1, 2, 4):  # the kinds other than fundamental
        check(set_(i, real_focal_check=1), cabi.PLB_ERR_ARG)
    for i in range(len(base)):
        for field in ("a", "b", "samples", "n_models", "models", "scores", "num_inliers"):
            check(set_(i, **{field: None}), cabi.PLB_ERR_ARG)
    for thr in (float("nan"), float("inf"), -float("inf")):
        check(set_(2, sq_threshold=thr), cabi.PLB_ERR_ARG)
    check(set_(0, s=2 ** 31), cabi.PLB_ERR_ARG)
    check(set_(4, n=2 ** 26 + 1), cabi.PLB_ERR_ARG)
    nyi = cabi.Camera(5, (500.0, 500.0, 0.0, 0.0))  # OPENCV_FISHEYE: not on the path
    check(set_(2, camera1=nyi), cabi.PLB_ERR_NYI)
    check(set_(2, camera2=nyi), cabi.PLB_ERR_NYI)
    # the order: an argument error of an earlier problem wins; within a problem, NULL before the threshold before s / n,
    # the camera before the indices
    check(both(set_(1, kind=9), set_(2, camera1=nyi)), cabi.PLB_ERR_ARG)
    check(both(set_(2, camera1=nyi), set_(3, kind=9)), cabi.PLB_ERR_NYI)
    check(both(set_(0, a=None), set_(0, sq_threshold=float("nan"))), cabi.PLB_ERR_ARG)
    check(lambda arr: None, cabi.PLB_ERR_ARG, form="device", dtype=2)
    check(lambda arr: None, cabi.PLB_ERR_ARG, form="host", n_gpus=-2)
    # the host form checks every index before any device call; the device form checks them on the device

    def bad_index(i, j, v):
        def edit(arr):
            keep_arr = np.ctypeslib.as_array(arr[i].samples, shape=(int(arr[i].s) * K[base[i]["kind"]],))
            keep_arr[j] = v
        return edit

    for i, v in ((0, 10), (3, -1), (4, 2 ** 31 - 1)):
        check(bad_index(i, 1, v), cabi.PLB_ERR_ARG, form="host")
    check(set_(2, camera1=nyi), cabi.PLB_ERR_NYI, form="host")
    if no_gpu:
        check(lambda arr: None, cabi.PLB_ERR_CUDA)
        check(set_(1, s=0, samples=None, n_models=None, models=None, scores=None, num_inliers=None), cabi.PLB_ERR_CUDA)
        check(set_(0, camera1=nyi), cabi.PLB_ERR_CUDA)  # cameras are read only with tangent_sampson
        check(bad_index(0, 0, -5), cabi.PLB_ERR_CUDA, form="device")
        check(lambda arr: None, cabi.PLB_ERR_CUDA, form="host", n_gpus=5)


def test_bindings_check_their_arguments():
    with pytest.raises(KeyError):
        cabi.generate_batch([{"kind": "nope", "a": np.zeros((4, 2)), "b": np.zeros((4, 2)), "samples": [[0, 1, 2, 3]],
                              "sq_threshold": 1.0}])
    p = _cpu_problems()[4]
    with pytest.raises(cabi.PoseLibB200Error) as e:
        cabi.generate_batch([dict(p, samples=np.array([[0, 1, 2, 10]]), sq_threshold=1.0)])
    assert e.value.code == cabi.PLB_ERR_ARG


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _gpu():
    if cabi.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    cabi.set_device(0)


def _valid(r):
    """(sample, slot) pairs of the written slots."""
    nm = np.asarray(r["n_models"])
    return [(j, m) for j in range(len(nm)) for m in range(int(nm[j]))]


def assert_same(got, ref, tag):
    nm = np.asarray(got["n_models"])
    assert np.array_equal(nm, np.asarray(ref["n_models"])), tag
    mask = np.arange(np.asarray(got["scores"]).shape[1])[None, :] < nm[:, None]
    for f in ("models", "scores"):
        g, r = np.asarray(got[f]), np.asarray(ref[f])
        assert np.array_equal(_bits(g[mask]), _bits(r[mask])), (tag, f)
    assert np.array_equal(np.asarray(got["num_inliers"])[mask], np.asarray(ref["num_inliers"])[mask]), tag


def assert_sentinels(r, tag):
    nm = np.asarray(r["n_models"])
    if nm.size == 0:
        return
    past = np.arange(np.asarray(r["scores"]).shape[1])[None, :] >= nm[:, None]
    assert np.all(np.isnan(np.asarray(r["scores"])[past])), tag
    assert np.all(np.asarray(r["num_inliers"])[past] == -1), tag
    mo = np.asarray(r["models"]).reshape(*past.shape, -1)
    assert np.all(np.isnan(mo[past])), tag


def _bearings(x):
    h = np.c_[x, np.ones(len(x))]
    return h / np.linalg.norm(h, axis=1, keepdims=True)


def oracle_models(P, kind, a, b, idx):
    if kind == "pnp":
        return P.p3p(_bearings(a[idx]), b[idx])
    if kind == "relpose":
        return P.relpose_5pt(_bearings(a[idx]), _bearings(b[idx]))
    if kind == "fundamental":
        return P.relpose_7pt(_bearings(a[idx]), _bearings(b[idx]))
    n, H = P.homography_4pt(_bearings(a[idx]), _bearings(b[idx]), True)
    return H[None] if n else np.zeros((0, 3, 3))


TOL = {"pnp": (1e-9, 1e-9), "relpose": (1e-9, 1e-9), "fundamental": (1e-8, 1e-9), "homography": (1e-10, 1e-12)}


def oracle_cases():
    out = []
    for kind in ("pnp", "relpose", "fundamental", "homography"):
        for n in (K[kind], 257, 2000):
            out.append(problem(kind, n, 64, 100 + n + K[kind]))
    out.append(problem("relpose", 2000, 64, 77, prosac=True))
    out.append(problem("homography", 2000, 64, 78, prosac=True))
    return out


@pytest.mark.gpu
def test_models_and_records_against_the_oracle():
    import plo_py as P
    _gpu()
    probs = oracle_cases()
    for p, r in zip(probs, cabi.generate_batch(probs)):
        kind, n = p["kind"], len(p["a"])
        rtol, atol = TOL[kind]
        for j, idx in enumerate(p["samples"]):
            ref = oracle_models(P, kind, p["a"], p["b"], idx)
            tag = (kind, n, j)
            assert r["n_models"][j] == len(ref), (tag, r["n_models"][j], len(ref))
            got = r["models"][j, :len(ref)]
            assert np.allclose(got, ref, rtol=rtol, atol=atol, equal_nan=True), tag
            for m in range(len(ref)):
                s, cnt = P.score(kind, got[m], p["a"], p["b"], p["sq_threshold"])
                assert r["num_inliers"][j, m] == cnt, tag
                assert abs(r["scores"][j, m] - s) <= 2 * max(n, 1) * U * abs(s), (tag, r["scores"][j, m], s)
        assert_sentinels(r, kind)


@pytest.mark.gpu
def test_fixture_counts_models_and_records():
    _gpu()
    probs = [fixture_problem(c) for c in FIXTURE]
    for c, p, r in zip(FIXTURE, probs, cabi.generate_batch(probs)):
        kind = p["kind"]
        # Tangent Sampson: the bearings come from each side's iterative undistortion (unproject_with_jac), whose last
        # bits differ, and the 5-point solve amplifies that (the oracle's restatement is 7e-9 from the reference on the
        # PINHOLE / RADIAL pair).  Counts stay exact.
        rtol, atol = (1e-6, 1e-6) if c["kind"] == "tangent" else TOL[kind]
        n = len(p["a"])
        for j, s in enumerate(c["samples"]):
            tag = (c["kind"], c["n"], c["pair"], c["rfc"], c["prosac"], s["j"])
            assert r["n_models"][j] == s["n_models"], (tag, r["n_models"][j], s["n_models"])
            if not s["n_models"]:
                continue
            ref = fixture_models(c, s)
            assert np.allclose(r["models"][j, :s["n_models"]], ref, rtol=rtol, atol=atol, equal_nan=True), tag
            # the fixture's own models through plb_score_batch: the reference's counts exactly, its scores up to the
            # summation order
            sp = {k: v for k, v in p.items() if k not in ("samples", "rfc")}
            got = cabi.score_batch([dict(sp, models=ref)])[0]
            assert got["num_inliers"].tolist() == s["counts"], tag
            ref_scores = np.array([float.fromhex(v) for v in s["scores"]])
            assert np.all(np.abs(got["scores"] - ref_scores) <= 2 * max(n, 1) * U * np.abs(ref_scores)), tag
        assert_sentinels(r, c["kind"])


def record_cases():
    probs = [problem(k, 1500, 96, 300 + i) for i, k in enumerate(("pnp", "relpose", "fundamental", "homography"))]
    probs.append(problem("fundamental", 1500, 96, 310, rfc=True))
    probs += [tangent_problem("PINHOLE", "RADIAL", 1200, 96, 311),
              tangent_problem("DIVISION-", "SIMPLE_DIVISION+", 1200, 96, 312)]
    return probs


@pytest.mark.gpu
def test_records_are_score_batch_on_the_same_models():
    _gpu()
    probs = record_cases()
    for p, r in zip(probs, cabi.generate_batch(probs)):
        nm = r["n_models"]
        flat = np.concatenate([r["models"][j, :nm[j]] for j in range(len(nm))])
        sp = {k: v for k, v in p.items() if k not in ("samples", "rfc")}
        s = cabi.score_batch([dict(sp, models=flat)])[0]
        mask = np.arange(M[p["kind"]])[None, :] < nm[:, None]
        assert np.array_equal(_bits(s["scores"]), _bits(r["scores"][mask])), p["kind"]
        assert np.array_equal(s["num_inliers"], r["num_inliers"][mask]), p["kind"]
        assert nm.sum() > len(nm) // 4, (p["kind"], nm.sum())  # the scenes give models
        assert_sentinels(r, p["kind"])


@pytest.mark.gpu
def test_real_focal_check_keeps_the_order_of_the_rest():
    _gpu()
    base = problem("fundamental", 1500, 256, 401)
    off, on = cabi.generate_batch([base, dict(base, rfc=True)])
    dropped = 0
    for j in range(len(base["samples"])):
        a = [tuple(_bits(off["models"][j, m]).tolist()) for m in range(off["n_models"][j])]
        b = [tuple(_bits(on["models"][j, m]).tolist()) for m in range(on["n_models"][j])]
        it = iter(a)
        assert all(x in it for x in b), j  # b is a subsequence of a
        dropped += len(a) - len(b)
        for m, x in enumerate(b):
            k = a.index(x)
            assert _bits(on["scores"][j, m]) == _bits(off["scores"][j, k]) and \
                on["num_inliers"][j, m] == off["num_inliers"][j, k], j
    assert dropped > 0


def mixed_cases():
    """Both kinds of camera, n = 0, s = 0, mixed sizes."""
    probs = record_cases()
    probs.append(tangent_problem("RADIAL", "PINHOLE", 700, 40, 501))
    probs.append({"kind": "pnp", "a": np.zeros((0, 2)), "b": np.zeros((0, 3)), "samples": np.zeros((0, 3), np.int32),
                  "sq_threshold": 1e-4})
    probs.append(dict(problem("homography", 300, 1, 502), samples=np.zeros((0, 4), np.int32)))
    probs += [problem(k, n, 33, 503 + n) for k in ("relpose", "homography") for n in (K[k], 40, 5000)]
    return probs


@pytest.mark.gpu
def test_outputs_do_not_depend_on_the_batch_streams_mode_or_calls():
    _gpu()
    probs = mixed_cases()
    alone = [cabi.generate_batch([p])[0] for p in probs]
    for kw in ({}, {"streams": 1}, {"streams": 8}):
        for i, r in enumerate(cabi.generate_batch(probs, **kw)):
            assert_same(r, alone[i], (i, kw))
    for i, r in enumerate(cabi.generate_batch(probs[::-1])[::-1]):
        assert_same(r, alone[i], ("reversed", i))
    for mode in ("exact", "fast"):
        cabi.set_mode(mode)
        try:
            for i, r in enumerate(cabi.generate_batch(probs)):
                assert_same(r, alone[i], (mode, i))
        finally:
            cabi.set_mode("fast")
    # the same samples over three calls
    for i, p in enumerate(probs):
        s = len(p["samples"])
        cuts = [0, s // 3, 2 * s // 3, s]
        parts = [cabi.generate_batch([dict(p, samples=p["samples"][cuts[c]:cuts[c + 1]])])[0] for c in range(3)]
        joined = {f: np.concatenate([q[f] for q in parts]) for f in ("n_models", "models", "scores", "num_inliers")}
        assert_same(joined, alone[i], ("split", i))
    if cabi.device_count() > 1:
        for i, r in enumerate(cabi.generate_batch(probs, n_gpus=0)):
            assert_same(r, alone[i], ("all devices", i))
    cabi.set_device(0)


@pytest.mark.gpu
def test_one_problem_over_several_chunks():
    _gpu()
    # one problem per call takes at most 65 536 samples per chunk: 200 003 samples are four chunks
    big = problem("homography", 60, 200003, 601)
    r = cabi.generate_batch([big])[0]
    small = cabi.generate_batch([dict(big, samples=big["samples"][j0:j0 + 5000]) for j0 in (0, 65000, 131000, 195003)])
    for j0, q in zip((0, 65000, 131000, 195003), small):
        sub = {f: r[f][j0:j0 + 5000] for f in ("n_models", "models", "scores", "num_inliers")}
        assert_same(sub, q, j0)
    assert_sentinels(r, "big")
    assert r["n_models"].sum() > 50000


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if cabi.device_count() == 0 or not t.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    return t


def _on_device(torch, probs, dtype, stream=None):
    out = []
    with torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream()):
        for p in probs:
            q = dict(p)
            q["a"] = torch.tensor(p["a"], device="cuda:0").to(dtype)
            q["b"] = torch.tensor(p["b"], device="cuda:0").to(dtype)
            q["samples"] = torch.tensor(np.asarray(p["samples"], dtype=np.int32), device="cuda:0")
            out.append(q)
    return out


def _cpu(r):
    return {k: v.cpu().numpy() for k, v in r.items() if k != "status"}


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_device_form_is_the_host_form(torch, dtype):
    _gpu()
    probs = mixed_cases()
    if dtype == "float32":  # the host form on the widened values
        probs = [dict(p, a=p["a"].astype(np.float32).astype(np.float64), b=p["b"].astype(np.float32).astype(np.float64))
                 for p in probs]
    host = cabi.generate_batch(probs)
    side = torch.cuda.Stream()
    dev = _on_device(torch, probs, getattr(torch, dtype), stream=side)  # written on a side stream just before the call
    res = cabi.generate_batch_device(dev, stream=side)
    torch.cuda.synchronize()
    for i, (r, h) in enumerate(zip(res, host)):
        got = _cpu(r)
        assert_same(got, h, (dtype, i))
        assert_sentinels(got, (dtype, i))


@pytest.mark.gpu
def test_device_form_rejects_an_index_out_of_range(torch):
    _gpu()
    probs = mixed_cases()[:4]
    for bad in (-1, 10 ** 6, len(probs[2]["a"])):
        dev = _on_device(torch, probs, torch.float64)
        dev[2]["samples"][7, 1] = bad
        res_shapes = None
        with pytest.raises(cabi.PoseLibB200Error) as e:
            res_shapes = cabi.generate_batch_device(dev)
        assert e.value.code == cabi.PLB_ERR_ARG and res_shapes is None
    # the outputs of a rejected call: run the call by hand to keep them
    dev = _on_device(torch, probs, torch.float64)
    dev[1]["samples"][0, 0] = -3
    arr = (cabi.GenerateProblem * len(dev))()
    outs = []
    for q, p in zip(arr, dev):
        s, Mk = len(p["samples"]), M[p["kind"]]
        msz = 7 if p["kind"] in ("pnp", "relpose") else 9
        o = {"n_models": torch.full((s,), 77, dtype=torch.int32, device="cuda:0"),
             "models": torch.full((s, Mk, msz), float("nan"), dtype=torch.float64, device="cuda:0"),
             "scores": torch.full((s, Mk), float("nan"), dtype=torch.float64, device="cuda:0"),
             "num_inliers": torch.full((s, Mk), -1, dtype=torch.int64, device="cuda:0")}
        outs.append(o)
        cabi._fill_generate_problem(q, p, len(p["a"]), s)
        P = lambda t, ct=cabi._P: C.cast(C.c_void_p(t.data_ptr()), ct)
        q.a, q.b, q.samples = P(p["a"]), P(p["b"]), P(p["samples"], C.POINTER(C.c_int32))
        q.n_models, q.models = P(o["n_models"], C.POINTER(C.c_int32)), P(o["models"])
        q.scores, q.num_inliers = P(o["scores"]), P(o["num_inliers"], C.POINTER(C.c_int64))
    torch.cuda.synchronize()
    rc = cabi.lib().plb_generate_batch_device(arr, C.c_size_t(len(dev)), cabi.DTYPE_F64, None, 8)
    torch.cuda.synchronize()
    assert rc == cabi.PLB_ERR_ARG and all(q.status == cabi.PLB_ERR_ARG for q in arr)
    for o in outs:
        assert bool((o["n_models"] == 77).all()) and bool(o["models"].isnan().all())
        assert bool(o["scores"].isnan().all()) and bool((o["num_inliers"] == -1).all())
