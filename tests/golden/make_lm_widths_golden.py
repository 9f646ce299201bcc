"""Writes tests/golden/reference_lm_widths.json: PoseLib's own camera-refining bundle adjustments at the sizes where the
device splits a job over 2, 4 or 8 CTAs (tests/test_lm_widths.py).

  * bundle_adjust(x, X, Image*, opt): PNP_CAMERAS x refine flags 1, 7 x TRIVIAL, CAUCHY x CAM_SIZES;
  * refine_relpose(x1, x2, ImagePair*, opt): PAIRS (the same camera on both images, and one mixed pair) x the same grid;
  * estimate_absolute_pose(.., Image*, ..) and estimate_relative_pose with tangent_sampson, refine flags 0 and 7, on
    ESTIMATE_N points whose inliers (30 %) come first, as after a PROSAC quality sort.  The final polish of a 20 000-point
    problem runs on 8 CTAs of 2528 points: CTAs 3-7 hold outliers only, so their compacted polish lists are empty.

The outputs come from the reference's sources compiled on mini-Eigen (oracle/_ref/libplref2.so), called through the
client of make_camera_models_golden.py (tests/ref_camera_models_client.cc), which takes every camera model; the inputs
are regenerated from the seeds by the problem generators of make_intrinsics_golden.py, make_relpose_intrinsics_golden.py
and make_camera_models_golden.py, so the file holds seeds and results only.  As in those generators every two-view case
is also run on oracle/_ref/libplref2_alt.so (mini-Eigen's other summation order) and redrawn until both builds agree, so
the stopping points the file records do not hang on a summation order.

    python tests/golden/make_lm_widths_golden.py          (needs the reference checkout; CPU only)
"""
import ctypes as C
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_camera_models_golden as MC  # noqa: E402
import make_intrinsics_golden as MG  # noqa: E402
import make_relpose_intrinsics_golden as MR  # noqa: E402

OUT = os.path.join(HERE, "reference_lm_widths.json")
# around the width boundaries of a single call (2048 correspondences per CTA: 2, 4, 8 CTAs above 2048, 6144, 14336) and
# one past a 256-point tile; 40000 gives each CTA of an 8-wide cluster 20 tiles
CAM_SIZES = [257, 2049, 6145, 16385, 40000]
PNP_CAMERAS = ["PINHOLE", "OPENCV", "RADIAL_FISHEYE", "DIVISION-"]
PAIRS = [("PINHOLE", "PINHOLE"), ("OPENCV", "OPENCV"), ("RADIAL_FISHEYE", "RADIAL_FISHEYE"), ("DIVISION-", "DIVISION-"),
         ("SIMPLE_RADIAL_FISHEYE", "SIMPLE_DIVISION+")]
FLAGS = (1, 7)
LOSSES = ("TRIVIAL", "CAUCHY")
LOSS_SCALE, PAIR_LOSS_SCALE, RELATIVE_COST_TOL = MG.LOSS_SCALE, MC.PAIR_LOSS_SCALE, 1e-8
ESTIMATE_N, ESTIMATE_INLIERS = 20000, 6000
ESTIMATE_CAMERAS = {"pnp": "RADIAL_FISHEYE", "pair": ("PINHOLE", "PINHOLE")}
ESTIMATE_FLAGS = (0, 7)
ESTIMATE_MAX_ERROR, PAIR_MAX_ERROR = MC.ESTIMATE_MAX_ERROR, MC.PAIR_MAX_ERROR
ESTIMATE_RANSAC = MC.ESTIMATE_RANSAC
MAX_DRAWS = 4


def model_name(cam):
    return MC.CAMERAS[cam][0] if cam in MC.CAMERAS else cam


def model_id(cam):
    return MC.MODEL_IDS[model_name(cam)]


def pnp_problem(cam, n, seed, outliers=0.1):
    """x [n, 2], X [n, 3], start pose, start parameters of camera `cam` (a MC.CAMERAS key or an MG.MODELS name)."""
    if cam in MC.CAMERAS:
        x, X, pose0, p0 = MC.problem(cam, n, seed, outliers)
    else:
        x, X, pose0, p0, _ = MG.problem(MG.MODELS[cam], n, seed, outliers)
    return np.ascontiguousarray(x), np.ascontiguousarray(X), pose0, np.asarray(p0, dtype=np.float64)


def pair_problem(pair, n, seed, outliers=0.0):
    """x1, x2 [n, 2], start pose, start parameters of both cameras."""
    if pair[0] in MR.MODELS and pair[1] in MR.MODELS:
        return MR.pair_problem(MR.MODELS[pair[0]], MR.MODELS[pair[1]], n, seed, outliers)
    return MC.pair_problem(pair[0], pair[1], n, seed, outliers)


def sorted_pnp_problem(cam, seed):
    """ESTIMATE_INLIERS points of pnp_problem without outliers, then ESTIMATE_N - ESTIMATE_INLIERS points whose
    observations are all uniform pixels: the inliers first."""
    x, X, _, p0 = pnp_problem(cam, ESTIMATE_INLIERS, seed, outliers=0.0)
    xo, Xo, _, _ = pnp_problem(cam, ESTIMATE_N - ESTIMATE_INLIERS, seed + 1, outliers=1.0)
    return np.ascontiguousarray(np.r_[x, xo]), np.ascontiguousarray(np.r_[X, Xo]), p0


def sorted_pair_problem(pair, seed):
    """As sorted_pnp_problem for two PINHOLE views.  Uniform pixels near the epipolar line of their partner would pass
    any threshold, so the outliers are those more than 20 px from it at the start pose: every inlier lies in the first
    ESTIMATE_INLIERS points."""
    x1, x2, pose0, c1, c2 = pair_problem(pair, ESTIMATE_INLIERS, seed, outliers=0.0)
    y1, y2, _, _, _ = pair_problem(pair, 2 * (ESTIMATE_N - ESTIMATE_INLIERS), seed + 1, outliers=1.0)
    h1 = np.c_[(y1 - c1[2:4]) / c1[:2], np.ones(len(y1))]
    h2 = np.c_[(y2 - c2[2:4]) / c2[:2], np.ones(len(y2))]
    t = pose0[4:7]
    E = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ MG.quat_to_rot(pose0[:4])
    Ex1, Etx2 = h1 @ E.T, h2 @ E
    d = np.abs((h2 * Ex1).sum(1)) / np.sqrt(Ex1[:, 0] ** 2 + Ex1[:, 1] ** 2 + Etx2[:, 0] ** 2 + Etx2[:, 1] ** 2)
    far = np.flatnonzero(d * c1[0] > 20.0)[:ESTIMATE_N - ESTIMATE_INLIERS]
    assert len(far) == ESTIMATE_N - ESTIMATE_INLIERS
    return np.ascontiguousarray(np.r_[x1, y1[far]]), np.ascontiguousarray(np.r_[x2, y2[far]]), c1, c2


def bundle_seed(cam, n, flags, loss):
    return 110000 + 1000 * PNP_CAMERAS.index(cam) + 100 * LOSSES.index(loss) + 10 * flags + CAM_SIZES.index(n)


def refine_seed(pair, n, flags, loss, draw=0):
    return 120000 + 1000 * PAIRS.index(tuple(pair)) + 100 * LOSSES.index(loss) + 10 * flags + CAM_SIZES.index(n) + \
        100000 * draw


def estimate_seed(kind, flags, draw=0):
    return 130000 + 100 * (kind == "pair") + flags + 100000 * draw


_p = MC._p


def _params(cam, p0):
    p = np.zeros(8)
    p[:len(p0)] = p0
    return p


def ref_bundle_adjust(lib, cam, n, flags, loss):
    x, X, pose0, p0 = pnp_problem(cam, n, bundle_seed(cam, n, flags, loss))
    pose, params, st = pose0.copy(), _params(cam, p0), np.zeros(3)
    lib.cm_bundle_adjust_image(model_id(cam), _p(params), C.c_int64(n), _p(x), _p(X), _p(pose), MG.LOSSES[loss],
                               C.c_double(LOSS_SCALE), 100, C.c_double(RELATIVE_COST_TOL), flags, _p(st))
    return dict(camera=cam, n=n, flags=flags, loss=loss, iterations=int(st[0]), initial_cost=st[1], cost=st[2],
                pose=pose.tolist(), params=params[:len(p0)].tolist())


def ref_refine(lib, pair, n, flags, loss, seed):
    x1, x2, pose0, c1, c2 = pair_problem(pair, n, seed)
    pose, st = pose0.copy(), np.zeros(3)
    p1, p2 = _params(pair[0], c1), _params(pair[1], c2)
    lib.cm_refine_relpose_pair(model_id(pair[0]), _p(p1), model_id(pair[1]), _p(p2), C.c_int64(n), _p(x1), _p(x2),
                               _p(pose), MG.LOSSES[loss], C.c_double(PAIR_LOSS_SCALE), 100,
                               C.c_double(RELATIVE_COST_TOL), flags, _p(st))
    return dict(camera1=pair[0], camera2=pair[1], n=n, flags=flags, loss=loss, seed=seed, iterations=int(st[0]),
                initial_cost=st[1], cost=st[2], pose=pose.tolist(), params1=p1[:len(c1)].tolist(),
                params2=p2[:len(c2)].tolist())


def ref_estimate(lib, kind, flags, seed):
    r = ESTIMATE_RANSAC
    mask, pose, st = np.zeros(ESTIMATE_N, dtype=np.int8), np.zeros(7), np.zeros(4)
    if kind == "pnp":
        cam = ESTIMATE_CAMERAS["pnp"]
        x, X, p0 = sorted_pnp_problem(cam, seed)
        pose[0] = 1.0
        p = _params(cam, p0)
        lib.cm_estimate_absolute_pose(model_id(cam), _p(p), C.c_int64(ESTIMATE_N), _p(x), _p(X),
                                      C.c_double(ESTIMATE_MAX_ERROR), C.c_uint64(r["max_iterations"]),
                                      C.c_uint64(r["min_iterations"]), C.c_uint64(r["seed"]), flags, _p(pose),
                                      mask.ctypes.data_as(C.c_char_p), _p(st))
        params = dict(params=p[:len(p0)].tolist())
    else:
        pair = ESTIMATE_CAMERAS["pair"]
        x1, x2, c1, c2 = sorted_pair_problem(pair, seed)
        p1, p2 = _params(pair[0], c1), _params(pair[1], c2)
        lib.cm_estimate_relative_pose(model_id(pair[0]), _p(p1), model_id(pair[1]), _p(p2), C.c_int64(ESTIMATE_N),
                                      _p(x1), _p(x2), C.c_double(PAIR_MAX_ERROR), C.c_uint64(r["max_iterations"]),
                                      C.c_uint64(r["min_iterations"]), C.c_uint64(r["seed"]), flags, 1, 1, _p(pose),
                                      mask.ctypes.data_as(C.c_char_p), _p(st))
        params = dict(params1=p1[:len(c1)].tolist(), params2=p2[:len(c2)].tolist())
    return dict(kind=kind, flags=flags, seed=seed, iterations=int(st[0]), refinements=int(st[1]), num_inliers=int(st[2]),
                model_score=st[3], pose=pose.tolist(), inliers=np.packbits(mask.astype(np.uint8)).tobytes().hex(),
                **params)


def bundle_cases():
    return [(c, n, f, l) for c in PNP_CAMERAS for l in LOSSES for n in CAM_SIZES for f in FLAGS]


def refine_cases():
    return [(p, n, f, l) for p in PAIRS for l in LOSSES for n in CAM_SIZES for f in FLAGS]


def estimate_cases():
    return [(k, f) for k in ("pnp", "pair") for f in ESTIMATE_FLAGS]


def agree(a, b):
    """Same iteration count (estimates: and RANSAC outcome), pose and parameters within MC.AGREE_TOL."""
    if any(a.get(k) != b.get(k) for k in ("iterations", "refinements", "num_inliers", "inliers")):
        return False
    for key in ("pose", "params", "params1", "params2"):
        if key in a:
            x, y = np.array(a[key]), np.array(b[key])
            if np.any(np.abs(x - y) > MC.AGREE_TOL * np.maximum(1.0, np.abs(y))):
                return False
    return True


_libs = None


def _agreeing_case(c):
    """The first draw of refine or estimate case c on which libplref2 and libplref2_alt agree (its libplref2 result), or
    None."""
    global _libs
    if _libs is None:
        d = tempfile.mkdtemp(prefix="ref_lm_widths_")
        _libs = MC.build_client(d), MC.build_client(d, alt=True)
    for draw in range(MAX_DRAWS):
        if len(c) == 2:
            seed = estimate_seed(*c, draw=draw)
            a, b = (ref_estimate(lib, *c, seed) for lib in _libs)
        else:
            seed = refine_seed(*c, draw=draw)
            a, b = (ref_refine(lib, *c, seed) for lib in _libs)
        if agree(a, b):
            return a
    return None


def main():
    import multiprocessing
    lib = MC.build_client()
    MC.build_client(alt=True)
    two = refine_cases() + estimate_cases()
    with multiprocessing.Pool() as pool:
        res = pool.map(_agreeing_case, two, chunksize=1)
    bad = [c for c, r in zip(two, res) if r is None]
    if bad:
        sys.exit("libplref2 and libplref2_alt disagree on every draw of %s: not written" % (bad,))
    nr = len(refine_cases())
    gold = dict(loss_scale=LOSS_SCALE, pair_loss_scale=PAIR_LOSS_SCALE, relative_cost_tol=RELATIVE_COST_TOL,
                estimate=dict(n=ESTIMATE_N, inliers=ESTIMATE_INLIERS, max_error=ESTIMATE_MAX_ERROR,
                              pair_max_error=PAIR_MAX_ERROR, ransac=ESTIMATE_RANSAC),
                bundle=[ref_bundle_adjust(lib, *c) for c in bundle_cases()], refine=res[:nr], estimate_cases=res[nr:])
    with open(OUT, "w") as f:
        json.dump(gold, f, indent=0)
    print("wrote", OUT, {k: len(v) for k, v in gold.items() if isinstance(v, list)})


if __name__ == "__main__":
    main()
