"""Writes tests/golden/reference_intrinsics.json: PoseLib's own camera refinement on synthetic PnP problems.

  * bundle_adjust(x, X, Image*, opt): 5 camera models x 7 refine flag sets x 4 losses, at n = 500 and n = 6000;
  * estimate_absolute_pose(points2D, points3D, opt, Image*, inliers) with refine flags 0, 1, 3, 7 on the 5 models.

The outputs come from the reference's sources compiled on mini-Eigen (oracle/_ref/libplref2.so, `make -C oracle ref2`),
called through tests/ref_intrinsics_client.cc; the inputs are regenerated from the seeds by problem() (NumPy's legacy
RandomState, identical on every machine), so the file holds seeds and results only.

    python tests/golden/make_intrinsics_golden.py          (needs the reference checkout; CPU only)
"""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
OUT = os.path.join(HERE, "reference_intrinsics.json")

MODELS = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "RADIAL": 3, "OPENCV": 4}
NUM_PARAMS = {0: 3, 1: 4, 2: 4, 3: 5, 4: 8}
LOSSES = {"TRIVIAL": 0, "TRUNCATED": 1, "HUBER": 2, "CAUCHY": 3}
LOSS_SCALE = 4.0  # pixels
# relative_cost_tol of the bundle cases.  At the default 1e-10 the stopping test compares cost decreases of ~1e-10 * cost
# with the rounding of a 6000-term cost sum (the truncated outliers alone add ~1e4): a different summation order may
# then stop one iteration earlier or later.  1e-8 keeps the test well above that noise.
RELATIVE_COST_TOL = 1e-8
TRUE_PARAMS = {0: [800.0, 320.0, 240.0], 1: [820.0, 790.0, 330.0, 245.0], 2: [800.0, 320.0, 240.0, -0.05],
               3: [800.0, 320.0, 240.0, -0.05, 0.01], 4: [820.0, 790.0, 330.0, 245.0, -0.05, 0.01, 0.001, -0.0005]}
ESTIMATE_FLAGS = (0, 1, 3, 7)
ESTIMATE_N, ESTIMATE_MAX_ERROR = 2000, 4.0
ESTIMATE_RANSAC = dict(max_iterations=2000, min_iterations=100, seed=11)


def quat_to_rot(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def project(model, p, Z):
    """<Model>::project of camera-frame points Z [n, 3] -> pixels [n, 2] (data synthesis only)."""
    px, py = Z[:, 0] / Z[:, 2], Z[:, 1] / Z[:, 2]
    if model in (0, 1):
        fx, fy, cx, cy = (p[0], p[1], p[2], p[3]) if model == 1 else (p[0], p[0], p[1], p[2])
        return np.stack([fx * px + cx, fy * py + cy], 1)
    r2 = px * px + py * py
    if model in (2, 3):
        a = 1.0 + p[3] * r2 + (p[4] * r2 * r2 if model == 3 else 0.0)
        return np.stack([p[0] * a * px + p[1], p[0] * a * py + p[2]], 1)
    k1, k2, p1, p2 = p[4:8]
    a = 1.0 + k1 * r2 + k2 * r2 * r2
    xd = a * px + 2.0 * p1 * px * py + p2 * (r2 + 2.0 * px * px)
    yd = a * py + 2.0 * p2 * px * py + p1 * (r2 + 2.0 * py * py)
    return np.stack([p[0] * xd + p[2], p[1] * yd + p[3]], 1)


def problem(model, n, seed, outliers=0.1):
    """Points seen by a TRUE_PARAMS[model] camera at a random pose (0.5 px noise, `outliers` of them replaced by uniform
    pixels), a start pose close to the truth and a start camera with the focal length 0.2 % and the principal point
    1 px off.  Returns x [n, 2], X [n, 3], start pose [7], start camera parameters, true parameters."""
    rng = np.random.RandomState(seed)
    ax = rng.normal(size=3)
    ang = 0.3 * rng.uniform()
    q = np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * ax / np.linalg.norm(ax)])
    t = rng.normal(scale=0.3, size=3)
    Zc = np.column_stack([rng.uniform(-1.2, 1.2, n), rng.uniform(-0.9, 0.9, n), np.ones(n)]) * rng.uniform(2, 8, n)[:, None]
    X = (Zc - t) @ quat_to_rot(q)
    p = np.array(TRUE_PARAMS[model])
    x = project(model, p, Zc) + rng.normal(scale=0.5, size=(n, 2))
    bad = rng.uniform(size=n) < outliers
    x[bad] = rng.uniform(0, 640, size=(int(bad.sum()), 2))
    dq = np.concatenate([[1.0], rng.normal(scale=5e-4, size=3)])
    dq /= np.linalg.norm(dq)
    q0 = np.array([q[0] * dq[0] - q[1:] @ dq[1:], *(q[0] * dq[1:] + dq[0] * q[1:] + np.cross(q[1:], dq[1:]))])
    pose0 = np.concatenate([q0, t + rng.normal(scale=2e-3, size=3)])
    p0 = p.copy()
    p0[0] *= 1.002
    nf = 2 if model in (1, 4) else 1
    if nf == 2:
        p0[1] *= 0.998
    p0[nf:nf + 2] += 1.0
    return x, X, pose0, p0, p


def bundle_seed(model, n, flags, loss):
    return 1000 * MODELS[model] + 100 * list(LOSSES).index(loss) + 10 * flags + (n == 6000)


def estimate_seed(model):
    return 7000 + MODELS[model]


def reference_available():
    return os.path.isdir(os.path.join(REF, "PoseLib"))


def build_client(out_dir=None):
    """Compiles tests/ref_intrinsics_client.cc into a shared library linked with oracle/_ref/libplref2.so."""
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "ref2"], stdout=subprocess.DEVNULL,
                          stderr=subprocess.DEVNULL)
    refdir = os.path.join(ROOT, "oracle", "_ref")
    out_dir = out_dir or tempfile.mkdtemp(prefix="ref_intrinsics_")
    so = os.path.join(out_dir, "libref_intrinsics.so")
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-w", "-shared",
                           "-I" + os.path.join(ROOT, "oracle", "ref", "mini"), "-I" + os.path.join(ROOT, "oracle"),
                           "-I" + REF, os.path.join(ROOT, "tests", "ref_intrinsics_client.cc"), "-L" + refdir, "-lplref2",
                           "-Wl,-rpath," + refdir, "-o", so])
    lib = C.CDLL(so, mode=os.RTLD_LAZY)  # the estimators name out-of-scope solvers that are never called
    lib.ri_refine_idx.restype = C.c_int
    return lib


def _p(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def ref_bundle_adjust(lib, model, n, flags, loss):
    mid = MODELS[model]
    x, X, pose0, p0, _ = problem(mid, n, bundle_seed(model, n, flags, loss))
    pose, params, st = pose0.copy(), p0.copy(), np.zeros(3)
    x, X = np.ascontiguousarray(x), np.ascontiguousarray(X)
    lib.ri_bundle_adjust_image(mid, _p(params), C.c_int64(n), _p(x), _p(X), _p(pose), LOSSES[loss],
                               C.c_double(LOSS_SCALE), 100, C.c_double(RELATIVE_COST_TOL), flags, _p(st))
    return dict(model=model, n=n, flags=flags, loss=loss, iterations=int(st[0]), initial_cost=st[1], cost=st[2],
                pose=pose.tolist(), params=params.tolist())


def ref_estimate(lib, model, flags):
    mid = MODELS[model]
    x, X, _, p0, _ = problem(mid, ESTIMATE_N, estimate_seed(model), outliers=0.3)
    pose = np.array([1.0, 0, 0, 0, 0, 0, 0])
    params = p0.copy()
    mask = np.zeros(ESTIMATE_N, dtype=np.int8)
    st = np.zeros(4)
    x, X = np.ascontiguousarray(x), np.ascontiguousarray(X)
    r = ESTIMATE_RANSAC
    lib.ri_estimate_absolute_pose(mid, _p(params), C.c_int64(ESTIMATE_N), _p(x), _p(X), C.c_double(ESTIMATE_MAX_ERROR),
                                  C.c_uint64(r["max_iterations"]), C.c_uint64(r["min_iterations"]), C.c_uint64(r["seed"]),
                                  flags, _p(pose), mask.ctypes.data_as(C.c_char_p), _p(st))
    return dict(model=model, flags=flags, iterations=int(st[0]), refinements=int(st[1]), num_inliers=int(st[2]),
                model_score=st[3], pose=pose.tolist(), params=params.tolist(),
                inliers=np.packbits(mask.astype(np.uint8)).tobytes().hex())


def bundle_cases():
    return [(m, n, f, l) for m in MODELS for l in LOSSES for n in (500, 6000) for f in range(1, 8)]


def estimate_cases():
    return [(m, f) for m in MODELS for f in ESTIMATE_FLAGS]


def main():
    lib = build_client()
    gold = dict(loss_scale=LOSS_SCALE, relative_cost_tol=RELATIVE_COST_TOL, estimate=dict(n=ESTIMATE_N, max_error=ESTIMATE_MAX_ERROR, ransac=ESTIMATE_RANSAC),
                bundle=[ref_bundle_adjust(lib, *c) for c in bundle_cases()],
                estimate_cases=[ref_estimate(lib, *c) for c in estimate_cases()])
    with open(OUT, "w") as f:
        json.dump(gold, f, indent=0)
    print("wrote", OUT, len(gold["bundle"]), "bundle cases,", len(gold["estimate_cases"]), "estimate cases")


if __name__ == "__main__":
    main()
