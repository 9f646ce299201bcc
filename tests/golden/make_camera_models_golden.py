"""Writes tests/golden/reference_camera_models.json: PoseLib's own SIMPLE_RADIAL_FISHEYE, RADIAL_FISHEYE, DIVISION and
SIMPLE_DIVISION cameras through the entry points that take a camera, on synthetic problems.

  * bundle_adjust(x, X, Image*, opt): every test camera x refine flags 0, 1, 3, 7 x 4 losses;
  * estimate_absolute_pose(points2D, points3D, opt, Image*, inliers) with refine flags 0, 1, 3, 7 on every camera;
  * refine_relpose(x1, x2, ImagePair*, opt) and estimate_relative_pose with tangent_sampson (refine flags 0, 1, 3, 7)
    and without it, on camera pairs (the same camera on both images, and mixed pairs with the older models).

Test cameras: the fisheye cameras of the reference's tests/example_cameras.h:40-41 and synthetic division cameras with
k < 0 and k > 0.  Fisheye scenes reach 85 degrees off axis (the two-view ones a few points past 90 degrees); scenes of
the k > 0 division cameras hold points whose projection has disc2 < 0.

The outputs come from the reference's sources compiled on mini-Eigen (oracle/_ref/libplref2.so, `make -C oracle ref2`),
called through tests/ref_camera_models_client.cc; the inputs are regenerated from the seeds by problem() /
pair_problem() (NumPy's legacy RandomState, identical on every machine), so the file holds seeds and results only.  As in
make_relpose_intrinsics_golden.py every two-view case is also run on oracle/_ref/libplref2_alt.so (mini-Eigen's other
summation order) and redrawn until both builds agree, so the stopping decisions the file records do not hang on Eigen's
unpinned summation order; the refine cases on which no draw agrees are named in REFINE_LEFT_OUT and left out of the file.

    python tests/golden/make_camera_models_golden.py          (needs the reference checkout; CPU only)
"""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_intrinsics_golden as MG  # noqa: E402

ROOT = MG.ROOT
REF = MG.REF
OUT = os.path.join(HERE, "reference_camera_models.json")

MODEL_IDS = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "RADIAL": 3, "OPENCV": 4,
             "SIMPLE_RADIAL_FISHEYE": 8, "RADIAL_FISHEYE": 9, "DIVISION": 101, "SIMPLE_DIVISION": 102}
NUM_PARAMS = {-1: 0, 0: 3, 1: 4, 2: 4, 3: 5, 4: 8, 8: 4, 9: 5, 101: 5, 102: 4}
# name -> (model, parameters)
CAMERAS = {
    "SIMPLE_RADIAL_FISHEYE": ("SIMPLE_RADIAL_FISHEYE", [1921.45, 2156.14, 1446.19, -0.0447036]),
    "RADIAL_FISHEYE": ("RADIAL_FISHEYE", [1921.45, 2156.14, 1446.19, -0.0447036, -0.00511989]),
    "DIVISION-": ("DIVISION", [820.0, 790.0, 330.0, 245.0, -0.2]),
    "DIVISION+": ("DIVISION", [820.0, 790.0, 330.0, 245.0, 0.05]),
    "SIMPLE_DIVISION-": ("SIMPLE_DIVISION", [800.0, 320.0, 240.0, -0.15]),
    "SIMPLE_DIVISION+": ("SIMPLE_DIVISION", [800.0, 320.0, 240.0, 0.08]),
    "PINHOLE": ("PINHOLE", MG.TRUE_PARAMS[1]),
    "RADIAL": ("RADIAL", MG.TRUE_PARAMS[3]),
}
NEW = [c for c in CAMERAS if CAMERAS[c][0] not in ("PINHOLE", "RADIAL")]
PAIRS = [(c, c) for c in NEW] + [("RADIAL_FISHEYE", "PINHOLE"), ("DIVISION-", "RADIAL"),
                                 ("SIMPLE_RADIAL_FISHEYE", "SIMPLE_DIVISION+")]
LOSSES = MG.LOSSES
FLAGS = (0, 1, 3, 7)
LOSS_SCALE = 4.0
RELATIVE_COST_TOL = 1e-8  # as in make_intrinsics_golden.py
BUNDLE_N = 600
ESTIMATE_N, ESTIMATE_MAX_ERROR = 1500, 4.0
ESTIMATE_RANSAC = dict(max_iterations=2000, min_iterations=100, seed=11)
PAIR_N, PAIR_LOSS_SCALE, PAIR_MAX_ERROR = 600, 2.0, 1.0
AGREE_TOL = 1e-8
MAX_DRAWS = 12
# Refine cases on which ref2 and ref2alt disagree on all MAX_DRAWS draws: all camera parameters of a fisheye or division
# camera paired with a pinhole / radial one.  Two views leave them nearly unconstrained, and the stopping point depends on
# the summation order.  main() checks that this list is exactly what the draws leave out.
REFINE_LEFT_OUT = [(("RADIAL_FISHEYE", "PINHOLE"), 7, l) for l in MG.LOSSES] + \
    [(("DIVISION-", "RADIAL"), 7, l) for l in MG.LOSSES]


def model_id(cam):
    return MODEL_IDS[CAMERAS[cam][0]]


def project(model, p, Z):
    """<Model>::project of camera-frame points Z [n, 3] -> pixels [n, 2] (data synthesis only; a division point with
    disc2 < 0 projects to (0, 0) as in the reference)."""
    if model in (0, 1, 2, 3, 4):
        return MG.project(model, p, Z)
    rho = np.hypot(Z[:, 0], Z[:, 1])
    if model in (8, 9):
        th = np.arctan2(rho, Z[:, 2])
        rd = th * (1.0 + p[3] * th ** 2 + (p[4] * th ** 4 if model == 9 else 0.0))
        s = rd / np.maximum(rho, 1e-300)
        return np.stack([p[0] * Z[:, 0] * s + p[1], p[0] * Z[:, 1] * s + p[2]], 1)
    fx, fy, cx, cy, k = (p[0], p[1], p[2], p[3], p[4]) if model == 101 else (p[0], p[0], p[1], p[2], p[3])
    disc2 = Z[:, 2] ** 2 - 4.0 * rho ** 2 * k
    r = 2.0 / (Z[:, 2] + np.sqrt(np.maximum(disc2, 0.0)))
    out = np.stack([fx * r * Z[:, 0] + cx, fy * r * Z[:, 1] + cy], 1)
    out[disc2 < 0] = 0.0
    return out


def max_angle(cam):
    """Largest angle off the optical axis of the scene points (degrees)."""
    m = CAMERAS[cam][0]
    return 85.0 if "FISHEYE" in m else 40.0 if "DIVISION" in m else 30.0


def directions(rng, n, deg):
    th = np.radians(deg) * np.sqrt(rng.uniform(size=n))
    ph = rng.uniform(0, 2 * np.pi, n)
    return np.column_stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])


def start_params(cam):
    m, p = CAMERAS[cam]
    p0 = np.array(p, dtype=float)
    nf = 2 if m in ("PINHOLE", "OPENCV", "DIVISION") else 1
    p0[:nf] *= 1.002
    p0[nf:nf + 2] += 1.0
    return p0


def problem(cam, n, seed, outliers=0.1):
    """Points seen by the camera at a random pose (0.5 px noise, `outliers` of them replaced by uniform pixels around
    the principal point), a start pose close to the truth and a start camera with the focal length 0.2 % and the
    principal point 1 px off.  Scenes of k > 0 division cameras also hold 2 % of points at 75 degrees off axis, where
    disc2 < 0 (their observations are uniform pixels).  Returns x [n, 2], X [n, 3], start pose [7], start parameters."""
    m, p = CAMERAS[cam]
    rng = np.random.RandomState(seed)
    ax = rng.normal(size=3)
    ang = 0.3 * rng.uniform()
    q = np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * ax / np.linalg.norm(ax)])
    t = rng.normal(scale=0.3, size=3)
    Zc = directions(rng, n, max_angle(cam)) * rng.uniform(2, 8, n)[:, None]
    beyond = (rng.uniform(size=n) < 0.02) & (CAMERAS[cam][1][-1] > 0) & ("DIVISION" in m)
    Zc[beyond] = np.array([np.sin(np.radians(75.0)), 0.0, np.cos(np.radians(75.0))]) * 4.0
    X = (Zc - t) @ MG.quat_to_rot(q)
    x = project(MODEL_IDS[m], np.array(p), Zc) + rng.normal(scale=0.5, size=(n, 2))
    bad = (rng.uniform(size=n) < outliers) | beyond
    c = np.array(p[1:3] if m not in ("PINHOLE", "DIVISION") else p[2:4])
    x[bad] = c + rng.uniform(-600, 600, size=(int(bad.sum()), 2))
    dq = np.concatenate([[1.0], rng.normal(scale=5e-4, size=3)])
    dq /= np.linalg.norm(dq)
    q0 = np.array([q[0] * dq[0] - q[1:] @ dq[1:], *(q[0] * dq[1:] + dq[0] * q[1:] + np.cross(q[1:], dq[1:]))])
    pose0 = np.concatenate([q0, t + rng.normal(scale=2e-3, size=3)])
    return np.ascontiguousarray(x), np.ascontiguousarray(X), pose0, start_params(cam)


def pair_problem(cam1, cam2, n, seed, outliers=0.0, noise=0.1, past90=False):
    """Points seen by two cameras one unit apart (`noise` px, `outliers` of the second image's points replaced by
    uniform pixels), a start pose close to the truth and start cameras as in problem().  With past90, 2 % of the points
    lie 92-100 degrees off the first camera's axis (fisheye cameras only, for the tangent-Sampson cases).  Returns
    x1 [n, 2], x2 [n, 2], start pose [7], start parameters of both cameras."""
    rng = np.random.RandomState(seed)
    ax = rng.normal(size=3)
    ang = 0.1 + 0.2 * rng.uniform()
    q = np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * ax / np.linalg.norm(ax)])
    t = np.array([1.0, 0.0, 0.0]) + rng.normal(scale=0.2, size=3)
    t /= np.linalg.norm(t)
    deg = min(max_angle(cam1), max_angle(cam2), 70.0)
    Z1 = directions(rng, n, deg) * rng.uniform(3, 8, n)[:, None]
    if past90:
        far = rng.uniform(size=n) < 0.02
        th = np.radians(rng.uniform(92, 100, int(far.sum())))
        ph = rng.uniform(-0.5, 0.5, int(far.sum()))  # on the side of the baseline, so the second camera sees them too
        Z1[far] = np.column_stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)]) * 6.0
    Z2 = Z1 @ MG.quat_to_rot(q).T + t
    x1 = project(model_id(cam1), np.array(CAMERAS[cam1][1]), Z1) + rng.normal(scale=noise, size=(n, 2))
    x2 = project(model_id(cam2), np.array(CAMERAS[cam2][1]), Z2) + rng.normal(scale=noise, size=(n, 2))
    bad = rng.uniform(size=n) < outliers
    x2[bad] = x2[~bad].mean(0) + rng.uniform(-400, 400, size=(int(bad.sum()), 2))
    dq = np.concatenate([[1.0], rng.normal(scale=5e-4, size=3)])
    dq /= np.linalg.norm(dq)
    q0 = np.array([q[0] * dq[0] - q[1:] @ dq[1:], *(q[0] * dq[1:] + dq[0] * q[1:] + np.cross(q[1:], dq[1:]))])
    t0 = t + rng.normal(scale=2e-3, size=3)
    pose0 = np.concatenate([q0, t0 / np.linalg.norm(t0)])
    return np.ascontiguousarray(x1), np.ascontiguousarray(x2), pose0, start_params(cam1), start_params(cam2)


def host_points(model, p):
    """Pixels and camera-frame points that reach every branch of the camera functions: near the axis, theta at pi/2,
    past 90 degrees, disc2 < 0 (k > 0 division cameras), plus a spread of ordinary points."""
    rng = np.random.RandomState(300 + model)
    c = np.array(p[2:4] if model == 101 else p[1:3])
    f = p[0]
    px = c + rng.uniform(-1.5, 1.5, (40, 2)) * f
    px = np.concatenate([px, [c, c + [1e-9 * f, 0.0], c + [3e-9 * f, -2e-9 * f]]])
    if model in (8, 9):  # rd of theta = pi/2 and theta past pi/2
        for th in (np.pi / 2, np.pi / 2 + 1e-9, 1.7, 1.9):
            rd = th * (1.0 + p[3] * th ** 2 + (p[4] * th ** 4 if model == 9 else 0.0))
            px = np.concatenate([px, [c + [f * rd, 0.0], c + [0.0, -f * rd * 0.6], c + [f * rd * 0.8, f * rd * 0.6]]])
    th = np.radians(np.concatenate([rng.uniform(0, 85, 30), [0.0, 1e-9, 89.999, 90.0, 95.0, 120.0]]))
    ph = rng.uniform(0, 2 * np.pi, len(th))
    Z = np.column_stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)]) * rng.uniform(0.5, 5, len(th))[:, None]
    Z = np.concatenate([Z, [[1e-10, -2e-10, 1.0], [0.0, 0.0, 2.0], [3.0, 0.1, 0.2], [2.0, -2.0, 0.1]]])
    return px, Z


# Leading columns of the rows of tests/camera_models_device_test.cu that a division camera computes with + - * / and
# sqrt only (pixels: bearing, hnormalized point, unproject_with_jac's bearing and M; points: every column); the
# remaining pixel columns are the parameter Jacobian, which divides by pow().
DIVISION_EXACT_COLUMNS = {"px": 23, "pt": 26}


def device_camera_rows(cam, out_dir):
    """Builds tests/camera_models_device_test.cu and evaluates the camera functions of `cam` on host_points() on the
    device and with the host build: {"px": (dev, host), "pt": (dev, host)}, rows of doubles."""
    exe = os.path.join(out_dir, "camera_models_device_test")
    subprocess.check_call(["nvcc", "-std=c++17", "-O2", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-Xcompiler", "-ffp-contract=off", "-o", exe,
                           os.path.join(ROOT, "tests", "camera_models_device_test.cu")])
    params = _p8(cam)
    px, Z = host_points(model_id(cam), params)
    rows = {}
    for kind, pts in (("px", px), ("pt", Z)):
        out = subprocess.check_output([exe, str(model_id(cam))] + [repr(float(v)) for v in params] + [kind] +
                                      [repr(float(v)) for v in pts.reshape(-1)], text=True).splitlines()
        vals = {t: np.array([[float.fromhex(v) for v in line.split()[1:]] for line in out if line.split()[0] == t])
                for t in ("dev", "host")}
        rows[kind] = (vals["dev"], vals["host"])
    return rows


def has_past90(pair):
    return "FISHEYE" in CAMERAS[pair[0]][0] and "FISHEYE" in CAMERAS[pair[1]][0]


def build_client(out_dir=None, alt=False):
    """Compiles tests/ref_camera_models_client.cc into a shared library linked with oracle/_ref/libplref2.so (alt:
    libplref2_alt.so, the client itself compiled with the same summation order)."""
    target, lib = ("ref2alt", "plref2_alt") if alt else ("ref2", "plref2")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s", target], stdout=subprocess.DEVNULL,
                          stderr=subprocess.DEVNULL)
    refdir = os.path.join(ROOT, "oracle", "_ref")
    out_dir = out_dir or tempfile.mkdtemp(prefix="ref_camera_models_")
    so = os.path.join(out_dir, "libref_camera_models%s.so" % ("_alt" if alt else ""))
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-w", "-Wno-psabi", "-shared"] +
                          (["-DMINI_EIGEN_ALT_ORDER"] if alt else []) +
                          ["-I" + os.path.join(ROOT, "oracle", "ref", "mini"), "-I" + os.path.join(ROOT, "oracle"),
                           "-I" + REF, os.path.join(ROOT, "tests", "ref_camera_models_client.cc"), "-L" + refdir,
                           "-l" + lib, "-Wl,-rpath," + refdir, "-o", so])
    lib = C.CDLL(so, mode=os.RTLD_LAZY)  # the estimators name out-of-scope solvers that are never called
    lib.cm_refine_idx.restype = C.c_int
    lib.cm_focal.restype = C.c_double
    return lib


_p = MG._p


def _p8(cam, params=None):
    p = np.zeros(8)
    v = CAMERAS[cam][1] if params is None else params
    p[:len(v)] = v
    return p


def bundle_seed(cam, flags, loss):
    return 50000 + 1000 * list(CAMERAS).index(cam) + 100 * list(LOSSES).index(loss) + 10 * flags


def ref_bundle_adjust(lib, cam, flags, loss):
    x, X, pose0, p0 = problem(cam, BUNDLE_N, bundle_seed(cam, flags, loss))
    pose, params, st = pose0.copy(), _p8(cam, p0), np.zeros(3)
    lib.cm_bundle_adjust_image(model_id(cam), _p(params), C.c_int64(BUNDLE_N), _p(x), _p(X), _p(pose), LOSSES[loss],
                               C.c_double(LOSS_SCALE), 100, C.c_double(RELATIVE_COST_TOL), flags, _p(st))
    return dict(camera=cam, flags=flags, loss=loss, iterations=int(st[0]), initial_cost=st[1], cost=st[2],
                pose=pose.tolist(), params=params[:len(p0)].tolist())


def estimate_seed(cam):
    return 60000 + list(CAMERAS).index(cam)


def ref_estimate(lib, cam, flags):
    x, X, _, p0 = problem(cam, ESTIMATE_N, estimate_seed(cam), outliers=0.3)
    pose = np.array([1.0, 0, 0, 0, 0, 0, 0])
    params = _p8(cam, p0)
    mask = np.zeros(ESTIMATE_N, dtype=np.int8)
    st = np.zeros(4)
    r = ESTIMATE_RANSAC
    lib.cm_estimate_absolute_pose(model_id(cam), _p(params), C.c_int64(ESTIMATE_N), _p(x), _p(X),
                                  C.c_double(ESTIMATE_MAX_ERROR), C.c_uint64(r["max_iterations"]),
                                  C.c_uint64(r["min_iterations"]), C.c_uint64(r["seed"]), flags, _p(pose),
                                  mask.ctypes.data_as(C.c_char_p), _p(st))
    return dict(camera=cam, flags=flags, iterations=int(st[0]), refinements=int(st[1]), num_inliers=int(st[2]),
                model_score=st[3], pose=pose.tolist(), params=params[:len(p0)].tolist(),
                inliers=np.packbits(mask.astype(np.uint8)).tobytes().hex())


def refine_seed(pair, flags, loss, draw=0):
    return 70000 + 1000 * PAIRS.index(tuple(pair)) + 100 * list(LOSSES).index(loss) + 10 * flags + 100000 * draw


def ref_refine(lib, pair, flags, loss, seed):
    x1, x2, pose0, c1, c2 = pair_problem(*pair, PAIR_N, seed)
    pose, st = pose0.copy(), np.zeros(3)
    p1, p2 = _p8(pair[0], c1), _p8(pair[1], c2)
    lib.cm_refine_relpose_pair(model_id(pair[0]), _p(p1), model_id(pair[1]), _p(p2), C.c_int64(PAIR_N), _p(x1),
                               _p(x2), _p(pose), LOSSES[loss], C.c_double(PAIR_LOSS_SCALE), 100,
                               C.c_double(RELATIVE_COST_TOL), flags, _p(st))
    return dict(camera1=pair[0], camera2=pair[1], flags=flags, loss=loss, seed=seed, iterations=int(st[0]),
                initial_cost=st[1], cost=st[2], pose=pose.tolist(), params1=p1[:len(c1)].tolist(),
                params2=p2[:len(c2)].tolist())


def pair_estimate_seed(pair, flags, tangent, draw=0):
    return 80000 + 10 * PAIRS.index(tuple(pair)) + flags + 500 * (not tangent) + 100000 * draw


def pair_estimate_inputs(pair, seed, tangent):
    return pair_problem(*pair, ESTIMATE_N, seed, outliers=0.3, past90=tangent and has_past90(pair))


def ref_pair_estimate(lib, pair, flags, tangent, seed, restate=True):
    x1, x2, _, c1, c2 = pair_estimate_inputs(pair, seed, tangent)
    p1, p2 = _p8(pair[0], c1), _p8(pair[1], c2)
    pose, st = np.zeros(7), np.zeros(4)
    mask = np.zeros(ESTIMATE_N, dtype=np.int8)
    r = ESTIMATE_RANSAC
    lib.cm_estimate_relative_pose(model_id(pair[0]), _p(p1), model_id(pair[1]), _p(p2), C.c_int64(ESTIMATE_N), _p(x1),
                                  _p(x2), C.c_double(PAIR_MAX_ERROR), C.c_uint64(r["max_iterations"]),
                                  C.c_uint64(r["min_iterations"]), C.c_uint64(r["seed"]), flags, int(tangent),
                                  int(restate), _p(pose), mask.ctypes.data_as(C.c_char_p), _p(st))
    return dict(camera1=pair[0], camera2=pair[1], flags=flags, tangent=bool(tangent), seed=seed, iterations=int(st[0]),
                refinements=int(st[1]), num_inliers=int(st[2]), model_score=st[3], pose=pose.tolist(),
                params1=p1[:len(c1)].tolist(), params2=p2[:len(c2)].tolist(),
                inliers=np.packbits(mask.astype(np.uint8)).tobytes().hex())


def bundle_cases():
    return [(c, f, l) for c in NEW for l in LOSSES for f in FLAGS]


def estimate_cases():
    return [(c, f) for c in NEW for f in FLAGS]


def refine_cases():
    return [(p, f, l) for p in PAIRS for l in LOSSES for f in (1, 3, 7)]


def pair_estimate_cases():
    return [(p, f, True) for p in PAIRS for f in FLAGS] + [(p, 0, False) for p in PAIRS]


def agree(a, b):
    """ref2 and ref2alt results of one case: same iteration count (estimate: and RANSAC outcome), pose and parameters
    within AGREE_TOL (relative to max(1, |value|))."""
    if any(a.get(k) != b.get(k) for k in ("iterations", "refinements", "num_inliers", "inliers")):
        return False
    for key in ("pose", "params1", "params2"):
        x, y = np.array(a[key]), np.array(b[key])
        if np.any(np.abs(x - y) > AGREE_TOL * np.maximum(1.0, np.abs(y))):
            return False
    return True


_libs = None


def _agreeing_case(c):
    """The first draw of two-view case c on which ref2 and ref2alt agree (its ref2 result), or None."""
    global _libs
    if _libs is None:
        d = tempfile.mkdtemp(prefix="ref_camera_models_")
        _libs = build_client(d), build_client(d, alt=True)
    for draw in range(MAX_DRAWS):
        if len(c) == 3 and isinstance(c[2], bool):
            pair, flags, tangent = c
            seed = pair_estimate_seed(pair, flags, tangent, draw)
            r = ref_pair_estimate(_libs[0], pair, flags, tangent, seed)
            if tangent:
                plain = ref_pair_estimate(_libs[0], pair, flags, tangent, seed, restate=False)
                if {k: v for k, v in plain.items() if k not in ("params1", "params2")} != \
                        {k: v for k, v in r.items() if k not in ("params1", "params2")}:
                    sys.exit("the restatement of estimate_relative_pose differs from it: %s" % (c,))
            if agree(r, ref_pair_estimate(_libs[1], pair, flags, tangent, seed)):
                return r
        else:
            seed = refine_seed(*c, draw=draw)
            r = ref_refine(_libs[0], *c, seed)
            if agree(r, ref_refine(_libs[1], *c, seed)):
                return r
    return None


def main():
    import multiprocessing
    lib = build_client()
    build_client(alt=True)
    two = refine_cases() + pair_estimate_cases()
    with multiprocessing.Pool() as pool:
        res = pool.map(_agreeing_case, two, chunksize=1)
    nr = len(refine_cases())
    bad = [c for c, r in zip(two, res) if r is None]
    if any(r is None for r in res[nr:]):
        sys.exit("ref2 and ref2alt disagree on every draw of an estimate case: not written")
    # Two views of a division camera leave its distortion nearly unconstrained: on some refine cases the stopping point
    # depends on the summation order for every draw.  Those cases are left out of the file.
    if sorted(bad) != sorted(REFINE_LEFT_OUT):
        sys.exit("refine cases without a summation-order stable draw differ from REFINE_LEFT_OUT: %s" % (bad,))
    gold = dict(loss_scale=LOSS_SCALE, pair_loss_scale=PAIR_LOSS_SCALE, relative_cost_tol=RELATIVE_COST_TOL,
                bundle=[ref_bundle_adjust(lib, *c) for c in bundle_cases()],
                estimate_cases=[ref_estimate(lib, *c) for c in estimate_cases()],
                refine=[r for r in res[:nr] if r is not None], pair_estimate_cases=res[nr:])
    with open(OUT, "w") as f:
        json.dump(gold, f, indent=0)
    print("wrote", OUT, {k: len(v) for k, v in gold.items() if isinstance(v, list)})


if __name__ == "__main__":
    main()
