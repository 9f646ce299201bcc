"""Writes tests/golden/reference_relpose_intrinsics.json: PoseLib's own camera refinement in the relative-pose bundle
adjustment (CameraRelativePoseRefiner) on synthetic two-view problems.

  * refine_relpose(x1, x2, ImagePair*, opt): 7 camera pairs (the five models on both images, PINHOLE/OPENCV and
    SIMPLE_RADIAL/RADIAL) x 7 refine flag sets x 4 losses, at n = 500 and n = 6000;
  * estimate_relative_pose with tangent_sampson and refine flags 0, 1, 3, 7 on the 7 camera pairs, 30 % outliers, and
    the same through a restatement of robust.cc:249-284 from public functions that keeps the refined cameras (its
    pose must equal estimate_relative_pose's bit for bit).

The outputs come from the reference's sources compiled on mini-Eigen (oracle/_ref/libplref2.so, `make -C oracle ref2`),
called through tests/ref_relpose_intrinsics_client.cc; the inputs are regenerated from the seeds by pair_problem()
(NumPy's legacy RandomState, identical on every machine), so the file holds seeds and results only.  Every case is also
run on oracle/_ref/libplref2_alt.so (`make -C oracle ref2alt`, mini-Eigen's other summation order); the file is written
only if both builds agree on the iteration count and to 1e-8 on pose and camera parameters, so the tolerances the GPU
tests use are not summation-order noise.  Two views constrain only two intrinsic parameters, so along the others the
refinement descends a nearly flat valley and stops where relative_cost_tol says; on a few draws that stopping point
depends on the summation order.  Such a draw is redrawn (the next seed of the case, `seed` in the file): every case of
the grid stays, on a draw both orders agree on.

    python tests/golden/make_relpose_intrinsics_golden.py          (needs the reference checkout; CPU only)
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
OUT = os.path.join(HERE, "reference_relpose_intrinsics.json")

MODELS = MG.MODELS
NUM_PARAMS = MG.NUM_PARAMS
LOSSES = MG.LOSSES
TRUE_PARAMS = MG.TRUE_PARAMS
PAIRS = [(m, m) for m in MODELS] + [("PINHOLE", "OPENCV"), ("SIMPLE_RADIAL", "RADIAL")]
LOSS_SCALE = 2.0  # pixels
RELATIVE_COST_TOL = 1e-8  # as in make_intrinsics_golden.py: well above the rounding of a 6000-term cost sum
AGREE_TOL = 1e-8
ESTIMATE_FLAGS = (0, 1, 3, 7)
ESTIMATE_N, ESTIMATE_MAX_ERROR = 2000, 1.0
ESTIMATE_RANSAC = dict(max_iterations=2000, min_iterations=100, seed=11)
NOISE = 0.1  # pixels


def pair_problem(m1, m2, n, seed, outliers=0.0, noise=NOISE):
    """Points seen by a TRUE_PARAMS[m1] camera and a TRUE_PARAMS[m2] camera one unit apart (`noise` px, `outliers` of the
    second image's points replaced by uniform pixels), a start pose close to the truth and start cameras with the focal
    length 0.2 % and the principal point 1 px off.  Points span a wide field of view at depths 2-6 with a general
    motion, so that the distortion and the epipolar geometry constrain focal length and principal point.  Returns
    x1 [n, 2], x2 [n, 2], start pose [7], start parameters of both cameras."""
    rng = np.random.RandomState(seed)
    ax = rng.normal(size=3)
    ang = 0.1 + 0.2 * rng.uniform()
    q = np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * ax / np.linalg.norm(ax)])
    t = np.array([1.0, 0.0, 0.0]) + rng.normal(scale=0.2, size=3)
    t /= np.linalg.norm(t)
    Z1 = np.column_stack([rng.uniform(-1.0, 1.0, n), rng.uniform(-0.75, 0.75, n), np.ones(n)]) * rng.uniform(2, 6, n)[:, None]
    Z2 = Z1 @ MG.quat_to_rot(q).T + t
    p1, p2 = np.array(TRUE_PARAMS[m1]), np.array(TRUE_PARAMS[m2])
    x1 = MG.project(m1, p1, Z1) + rng.normal(scale=noise, size=(n, 2))
    x2 = MG.project(m2, p2, Z2) + rng.normal(scale=noise, size=(n, 2))
    bad = rng.uniform(size=n) < outliers
    x2[bad] = rng.uniform(0, 640, size=(int(bad.sum()), 2))
    dq = np.concatenate([[1.0], rng.normal(scale=5e-4, size=3)])
    dq /= np.linalg.norm(dq)
    q0 = np.array([q[0] * dq[0] - q[1:] @ dq[1:], *(q[0] * dq[1:] + dq[0] * q[1:] + np.cross(q[1:], dq[1:]))])
    t0 = t + rng.normal(scale=2e-3, size=3)
    pose0 = np.concatenate([q0, t0 / np.linalg.norm(t0)])
    starts = []
    for m, p in ((m1, p1), (m2, p2)):
        p0 = p.copy()
        nf = 2 if m in (1, 4) else 1
        p0[:nf] *= 1.002
        p0[nf:nf + 2] += 1.0
        starts.append(p0)
    return np.ascontiguousarray(x1), np.ascontiguousarray(x2), pose0, starts[0], starts[1]


def refine_seed(pair, n, flags, loss, draw=0):
    return 20000 + 1000 * PAIRS.index(tuple(pair)) + 100 * list(LOSSES).index(loss) + 10 * flags + (n == 6000) + \
        100000 * draw


def build_client(out_dir=None, alt=False):
    """Compiles tests/ref_relpose_intrinsics_client.cc into a shared library linked with oracle/_ref/libplref2.so (alt:
    libplref2_alt.so, the client itself compiled with the same summation order)."""
    target, lib = ("ref2alt", "plref2_alt") if alt else ("ref2", "plref2")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s", target], stdout=subprocess.DEVNULL,
                          stderr=subprocess.DEVNULL)
    refdir = os.path.join(ROOT, "oracle", "_ref")
    out_dir = out_dir or tempfile.mkdtemp(prefix="ref_relpose_intrinsics_")
    so = os.path.join(out_dir, "libref_relpose_intrinsics%s.so" % ("_alt" if alt else ""))
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-w", "-Wno-psabi", "-shared"] +
                          (["-DMINI_EIGEN_ALT_ORDER"] if alt else []) +
                          ["-I" + os.path.join(ROOT, "oracle", "ref", "mini"), "-I" + os.path.join(ROOT, "oracle"),
                           "-I" + REF, os.path.join(ROOT, "tests", "ref_relpose_intrinsics_client.cc"), "-L" + refdir,
                           "-l" + lib, "-Wl,-rpath," + refdir, "-o", so])
    return C.CDLL(so, mode=os.RTLD_LAZY)


_p = MG._p


def ref_unproject(lib, model, params, xp, with_point):
    """Camera::unproject_with_jac of pixels xp [n, 2]: bearings [n, 3] and jac_params [n, 3, 8] (unused columns 0)."""
    n = len(xp)
    par = np.zeros(8)
    par[:NUM_PARAMS.get(model, 0)] = params[:NUM_PARAMS.get(model, 0)]
    d, dp = np.zeros(3 * n), np.zeros(24 * n)
    xp = np.ascontiguousarray(xp, dtype=float)
    lib.rr_unproject_with_jac(model, _p(par), C.c_int64(n), _p(xp), int(with_point), _p(d), _p(dp))
    return d.reshape(n, 3), dp.reshape(n, 3, 8)


def ref_refine(lib, pair, n, flags, loss, seed):
    m1, m2 = MODELS[pair[0]], MODELS[pair[1]]
    x1, x2, pose0, c1, c2 = pair_problem(m1, m2, n, seed)
    pose, st = pose0.copy(), np.zeros(3)
    p1, p2 = np.zeros(8), np.zeros(8)
    p1[:len(c1)], p2[:len(c2)] = c1, c2
    lib.rr_refine_relpose_pair(m1, _p(p1), m2, _p(p2), C.c_int64(n), _p(x1), _p(x2), _p(pose), LOSSES[loss],
                               C.c_double(LOSS_SCALE), 100, C.c_double(RELATIVE_COST_TOL), flags, _p(st))
    return dict(camera1=pair[0], camera2=pair[1], n=n, flags=flags, loss=loss, seed=seed, iterations=int(st[0]),
                initial_cost=st[1], cost=st[2], pose=pose.tolist(), params1=p1[:len(c1)].tolist(),
                params2=p2[:len(c2)].tolist())


def estimate_seed(pair, flags, draw=0):
    return 40000 + 10 * PAIRS.index(tuple(pair)) + flags + 100000 * draw


def ref_estimate(lib, pair, flags, seed, restate=True):
    m1, m2 = MODELS[pair[0]], MODELS[pair[1]]
    x1, x2, _, c1, c2 = pair_problem(m1, m2, ESTIMATE_N, seed, outliers=0.3)
    p1, p2 = np.zeros(8), np.zeros(8)
    p1[:len(c1)], p2[:len(c2)] = c1, c2
    pose, st = np.zeros(7), np.zeros(4)
    mask = np.zeros(ESTIMATE_N, dtype=np.int8)
    r = ESTIMATE_RANSAC
    lib.rr_estimate_relative_pose(m1, _p(p1), m2, _p(p2), C.c_int64(ESTIMATE_N), _p(x1), _p(x2),
                                  C.c_double(ESTIMATE_MAX_ERROR), C.c_uint64(r["max_iterations"]),
                                  C.c_uint64(r["min_iterations"]), C.c_uint64(r["seed"]), flags, int(restate),
                                  _p(pose), mask.ctypes.data_as(C.c_char_p), _p(st))
    return dict(camera1=pair[0], camera2=pair[1], flags=flags, seed=seed, iterations=int(st[0]),
                refinements=int(st[1]), num_inliers=int(st[2]), model_score=st[3], pose=pose.tolist(),
                params1=p1[:len(c1)].tolist(), params2=p2[:len(c2)].tolist(),
                inliers=np.packbits(mask.astype(np.uint8)).tobytes().hex())


def estimate_cases():
    return [(p, f) for p in PAIRS for f in ESTIMATE_FLAGS]


def refine_cases():
    return [(p, n, f, l) for p in PAIRS for l in LOSSES for n in (500, 6000) for f in range(1, 8)]


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


MAX_DRAWS = 4
_libs = None


def _agreeing_case(c):
    """The first draw of case c on which ref2 and ref2alt agree (its ref2 result), or None."""
    global _libs
    if _libs is None:
        d = tempfile.mkdtemp(prefix="ref_relpose_intrinsics_")
        _libs = build_client(d), build_client(d, alt=True)
    est = len(c) == 2
    for draw in range(MAX_DRAWS):
        if est:
            seed = estimate_seed(*c, draw=draw)
            r = ref_estimate(_libs[0], *c, seed)
            plain = ref_estimate(_libs[0], *c, seed, restate=False)
            if {k: v for k, v in plain.items() if k not in ("params1", "params2")} != \
                    {k: v for k, v in r.items() if k not in ("params1", "params2")}:
                sys.exit("the restatement of estimate_relative_pose differs from it: %s" % (c,))
            if agree(r, ref_estimate(_libs[1], *c, seed)):
                return r
        else:
            seed = refine_seed(*c, draw=draw)
            r = ref_refine(_libs[0], *c, seed)
            if agree(r, ref_refine(_libs[1], *c, seed)):
                return r
    return None


def main():
    import multiprocessing
    build_client(), build_client(alt=True)  # the reference builds, once, before the workers start
    with multiprocessing.Pool() as pool:
        cases = pool.map(_agreeing_case, refine_cases() + estimate_cases(), chunksize=1)
    bad = [c for c, r in zip(refine_cases() + estimate_cases(), cases) if r is None]
    if bad:
        sys.exit("ref2 and ref2alt disagree on every draw of %d cases, e.g. %s: not written" % (len(bad), bad[:5]))
    nr = len(refine_cases())
    gold = dict(loss_scale=LOSS_SCALE, relative_cost_tol=RELATIVE_COST_TOL, refine=cases[:nr],
                estimate=dict(n=ESTIMATE_N, max_error=ESTIMATE_MAX_ERROR, ransac=ESTIMATE_RANSAC),
                estimate_cases=cases[nr:])
    with open(OUT, "w") as f:
        json.dump(gold, f, indent=0)
    print("wrote", OUT, nr, "refine cases,", len(cases) - nr, "estimate cases")


if __name__ == "__main__":
    main()
