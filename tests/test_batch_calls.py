"""The eight batch entry points check in one order and fail in one way.

plb_ransac_batch[_multi], plb_estimate_batch[_device], plb_refine_batch[_device] and plb_score_batch[_device] run through
one table of cases: an empty batch writes nothing; NULL problems are an argument error; a bad dtype or n_gpus, or one
malformed problem in an otherwise valid batch, sets every status to its code and changes no other byte, in the problem
array or in the caller's masks, scores and counts; without a device a valid batch is a CUDA error, written the same way.
The estimate batches hold the problems that prepare writes into when they run: a tangent-Sampson relative pose whose
start pose is not the identity, and a fundamental matrix with too few points, both with stats and counters prefilled."""
import ctypes as C

import numpy as np
import pytest

try:
    from poselib_b200 import cabi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)

ARG, NYI, CUDA = cabi.PLB_ERR_ARG, cabi.PLB_ERR_NYI, cabi.PLB_ERR_CUDA
SENTINEL = 12345
RNG = np.random.default_rng(11)
X2, X3, X5 = RNG.normal(size=(10, 2)), RNG.normal(size=(10, 3)) + [0, 0, 5], RNG.normal(size=(5, 2))
PIN = cabi.Camera("PINHOLE", (500.0, 500.0, 320.0, 240.0))
FISHEYE = cabi.Camera(5, (500.0, 500.0, 0.0, 0.0))  # OPENCV_FISHEYE: not on the device path
FOCAL = cabi.BundleOpt(refine_intrinsics=cabi.REFINE_FOCAL_LENGTH)


def _prefill(q, *fields):
    for f in fields:
        v = getattr(q, f)
        C.memset(C.addressof(v), 0x5A, C.sizeof(v))


def _mask(n, keep):
    m = np.full(max(n, 1), 7, dtype=np.int8)
    keep.append(m)
    return C.cast(m.ctypes.data_as(C.POINTER(C.c_char)), C.c_char_p)


def _ransac_batch():
    probs = [("pnp", X2, X3), ("relpose", X2, X2), ("fundamental", X2, X2), ("relpose", X2, X2), ("homography", X2, X2)]
    arr, keep, outs = (cabi.Problem * len(probs))(), [], []
    for q, (kind, a, b) in zip(arr, probs):
        aa, ap = cabi._d(a)
        ba, bp = cabi._d(b)
        keep += [aa, ba]
        q.kind, q.n, q.a, q.b = cabi.KIND[kind], len(aa), ap, bp
        q.opt, q.max_error = cabi.RansacOpt(), 1e-2
        for k in range(9):
            q.model[k] = 0.5 + k
        q.inliers = _mask(len(aa), outs)
        _prefill(q, "stats", "counters")
    return arr, keep + outs, outs


def _estimate_batch():
    """Problem 1 (tangent Sampson, start pose not the identity) and problem 2 (F with 5 points) are what an estimate batch
    writes into when it runs; the malformed problem is 3."""
    init = [0.6, 0.8, 0.0, 0.0, 0.1, 0.2, 0.3]
    probs = [dict(kind="pnp", a=X2, b=X3, cam1=PIN),
             dict(kind="relpose", a=X2, b=X2, cam1=PIN, cam2=PIN, tangent_sampson=True, init=init),
             dict(kind="fundamental", a=X5, b=X5),
             dict(kind="relpose", a=X2, b=X2, cam1=PIN, cam2=PIN, init=init),
             dict(kind="homography", a=X2, b=X2)]
    arr, keep, outs = (cabi.EstimateProblem * len(probs))(), [], []
    for q, p in zip(arr, probs):
        aa, ap = cabi._d(p["a"])
        ba, bp = cabi._d(p["b"])
        keep += [aa, ba]
        cabi._fill_estimate_problem(q, dict(p, ransac=cabi.RansacOpt(), bundle=cabi.BundleOpt(), max_error=2.0), len(aa))
        q.a, q.b = ap, bp
        q.inliers = _mask(len(aa), outs)
        _prefill(q, "stats", "counters")
    return arr, keep + outs, outs


def _refine_batch():
    arr, keep = (cabi.RefineProblem * len(cabi.REFINER))(), []
    for q, r in zip(arr, cabi.REFINER):
        aa, ap = cabi._d(X2)
        ba, bp = cabi._d(X3 if r in ("bundle", "bundle_image") else X2)
        wa, wp = cabi._w(np.ones(len(aa)), len(aa))
        keep += [aa, ba, wa]
        cabi._fill_refine_problem(q, dict(refiner=r, bundle=cabi.BundleOpt(), cam1=PIN, cam2=PIN), len(aa))
        q.a, q.b, q.weights = ap, bp, wp
        for k in range(9):
            q.model[k] = 7.0 + k
        for k in range(3):
            q.bundle_stats[k] = -1.0
    return arr, keep, []


def _score_batch():
    pose, H = np.array([[1.0, 0, 0, 0, 0, 0, 0]] * 2), np.eye(3)[None].repeat(2, 0)
    probs = [dict(kind="pnp", a=X2, b=X3, models=pose), dict(kind="relpose", a=X2, b=X2, models=pose),
             dict(kind="relpose", a=X2, b=X2, models=pose, tangent_sampson=True, cam1=PIN, cam2=PIN),
             dict(kind="fundamental", a=X2, b=X2, models=H), dict(kind="homography", a=X2, b=X2, models=H)]
    arr, keep, outs = (cabi.ScoreProblem * len(probs))(), [], []
    for q, p in zip(arr, probs):
        aa, ap = cabi._d(p["a"])
        ba, bp = cabi._d(p["b"])
        mo = cabi._score_models(p["kind"], p["models"])
        sc, ct = np.full(len(mo), 7.0), np.full(len(mo), 7, dtype=np.int64)
        keep += [aa, ba, mo]
        outs += [sc, ct]
        cabi._fill_score_problem(q, dict(p, sq_threshold=1e-4), len(aa), len(mo))
        q.a, q.b, q.models = ap, bp, mo.ctypes.data_as(cabi._P)
        q.scores, q.num_inliers = sc.ctypes.data_as(cabi._P), ct.ctypes.data_as(C.POINTER(C.c_int64))
        q.inliers = _mask(len(aa) * len(mo), outs)
    return arr, keep + outs, outs


def _set(i, **kw):
    def edit(arr):
        for k, v in kw.items():
            setattr(arr[i], k, v)
    return edit


# Per family: the batch, and single malformations of one problem in its middle with the code each must give.
FAMILIES = {
    "ransac": (_ransac_batch, [(_set(3, kind=7), ARG), (_set(3, kind=-1), ARG), (_set(3, a=None), ARG),
                               (_set(3, b=None), ARG), (_set(3, resident=99), ARG)]),
    "estimate": (_estimate_batch, [(_set(3, kind=7), ARG), (_set(3, kind=9), ARG), (_set(3, a=None), ARG),
                                   (_set(3, camera1=FISHEYE), NYI), (_set(3, camera2=FISHEYE), NYI),
                                   (_set(3, tangent_sampson=1, bundle=FOCAL), NYI)]),
    "refine": (_refine_batch, [(_set(3, refiner=7), ARG), (_set(3, a=None), ARG), (_set(3, camera1=FISHEYE), NYI),
                               (_set(3, bundle=FOCAL), NYI)]),
    "score": (_score_batch, [(_set(2, kind=7), ARG), (_set(2, models=None), ARG), (_set(2, camera1=FISHEYE), NYI),
                             (_set(3, tangent_sampson=1), ARG)]),
}

# entry point -> (family, the call on (array, count, n_gpus, dtype), the n_gpus a valid call passes or None)
CALLS = {
    "plb_ransac_batch": ("ransac", lambda L, a, c, g, d: L.plb_ransac_batch(a, c, 8), None),
    "plb_ransac_batch_multi": ("ransac", lambda L, a, c, g, d: L.plb_ransac_batch_multi(a, c, g, 8), 0),
    "plb_estimate_batch": ("estimate", lambda L, a, c, g, d: L.plb_estimate_batch(a, c, g, 8), -1),
    "plb_estimate_batch_device": ("estimate", lambda L, a, c, g, d: L.plb_estimate_batch_device(a, c, d, None, 8), None),
    "plb_refine_batch": ("refine", lambda L, a, c, g, d: L.plb_refine_batch(a, c, g, 8), -1),
    "plb_refine_batch_device": ("refine", lambda L, a, c, g, d: L.plb_refine_batch_device(a, c, d, None, 8), None),
    "plb_score_batch": ("score", lambda L, a, c, g, d: L.plb_score_batch(a, c, g, 8), -1),
    "plb_score_batch_device": ("score", lambda L, a, c, g, d: L.plb_score_batch_device(a, c, d, None, 8), None),
}


@pytest.mark.parametrize("name", list(CALLS))
def test_batch_call_checks_in_one_order_and_fails_in_one_way(name):
    family, call, valid_gpus = CALLS[name]
    build, malformed = FAMILIES[family]
    device = name.endswith("_device")
    lib = cabi.lib()
    no_gpu = cabi.device_count() == 0

    def run(edit, code, n_gpus=valid_gpus, dtype=cabi.DTYPE_F64, count=None):
        arr, keep, outs = build()
        for q in arr:
            q.status = SENTINEL
        edit(arr)
        before, outs_before = bytes(arr), [o.tobytes() for o in outs]
        rc = call(lib, arr, C.c_size_t(len(arr) if count is None else count), n_gpus, dtype)
        assert rc == code, (name, rc, code, lib.plb_last_error())
        want = SENTINEL if count == 0 else code
        assert [q.status for q in arr] == [want] * len(arr), (name, code)
        for q in arr:
            q.status = SENTINEL
        assert bytes(arr) == before, name
        assert [o.tobytes() for o in outs] == outs_before, name

    def valid(arr):
        pass

    assert call(lib, None, C.c_size_t(3), valid_gpus, cabi.DTYPE_F64) == ARG
    run(valid, cabi.PLB_OK, count=0)
    if device:
        run(valid, ARG, dtype=2)
        assert "dtype" in lib.plb_last_error().decode()
    if valid_gpus is not None:
        run(valid, ARG, n_gpus=-2)
        if valid_gpus == 0:  # the multi call takes no "calling thread's device"
            run(valid, ARG, n_gpus=-1)
        run(valid, CUDA if no_gpu else ARG, n_gpus=10 ** 4)
    for edit, code in malformed:
        run(edit, code)
    if no_gpu:
        run(valid, CUDA)
