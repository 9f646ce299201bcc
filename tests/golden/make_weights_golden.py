"""Writes tests/golden/reference_weights.json: PoseLib's own refiners with per-residual weights on synthetic problems.

  * bundle_adjust(x, X, Image*, opt, weights) on NULL, PINHOLE, OPENCV and RADIAL_FISHEYE cameras, refine flags 0 and 7;
  * refine_relpose(x1, x2, ImagePair*, opt, weights) on a SIMPLE_RADIAL / RADIAL pair, refine flags 0 (the fixed-camera
    tangent-Sampson refiner) and 7 (CameraRelativePoseRefiner);
  * refine_relpose(x1, x2, CameraPose*, ..), refine_fundamental and refine_homography with weights;
every one with the four losses at n = 500 and n = 6000.  Weights are drawn in [0.1, 3], about 10 % of them are exactly 0
and the outliers' weights are scaled by 0.05.  Two more cases take the reference's uniform-weight branches: weights of the
wrong length (refine_relpose) and the calibrated bundle_adjust(x, X, CameraPose*, opt, weights), which drops its weights.

The outputs come from the reference's sources compiled on mini-Eigen (oracle/_ref/libplref2.so, `make -C oracle ref2`),
called through tests/ref_weights_client.cc; the inputs are regenerated from the seeds by inputs() (NumPy's legacy
RandomState and the seeded generators of poselib_b200/problem_generator.py, identical on every machine), so the file holds
seeds and hex-float results only.  As in make_relpose_intrinsics_golden.py every case is also run on
oracle/_ref/libplref2_alt.so (mini-Eigen's other summation order) and redrawn until both builds agree, so the stopping
decisions the file records do not hang on Eigen's unpinned summation order.

    python tests/golden/make_weights_golden.py          (needs the reference checkout; CPU only)
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
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_camera_models_golden as CM  # noqa: E402
import make_intrinsics_golden as MG  # noqa: E402
import make_relpose_intrinsics_golden as RG  # noqa: E402
import reference_cases as RC  # noqa: E402
from poselib_b200 import problem_generator as G  # noqa: E402

ROOT = MG.ROOT
OUT = os.path.join(HERE, "reference_weights.json")

LOSSES = MG.LOSSES
SIZES = (500, 6000)
FLAGS = (0, 7)
CAMERAS = {"NULL": -1, "PINHOLE": 1, "OPENCV": 4, "RADIAL_FISHEYE": 9}
PAIR = ("SIMPLE_RADIAL", "RADIAL")
MODEL_KINDS = ("relpose", "fundamental", "homography")
MAX_ITERATIONS = 100
# as in make_intrinsics_golden.py: well above the rounding of a 6000-term cost sum
RELATIVE_COST_TOL = 1e-8
AGREE_TOL = 1e-8
MAX_DRAWS = 12
NULL_FOCAL = (820.0, 790.0)  # the NULL camera sees the PINHOLE scene in calibrated coordinates
NULL_PP = (330.0, 245.0)


def weights(n, seed, outliers):
    """Weights in [0.1, 3], ~10 % exactly 0, the outliers' scaled by 0.05."""
    rng = np.random.RandomState(seed + 7)
    w = rng.uniform(0.1, 3.0, n)
    w[rng.uniform(size=n) < 0.1] = 0.0
    w[outliers] *= 0.05
    return w


def _outliers(x, seed, spread):
    """Moves ~10 % of the points x [n, 2] by up to `spread` (in place); returns their mask."""
    rng = np.random.RandomState(seed + 3)
    bad = rng.uniform(size=len(x)) < 0.1
    x[bad] += rng.uniform(-spread, spread, size=(int(bad.sum()), 2))
    return bad


def seed_of(case, draw=0):
    kind, cam, flags, loss, n = case
    base = {"image": 100, "pair": 200, "relpose": 300, "fundamental": 400, "homography": 500, "calibrated": 600,
            "mismatch": 700}[kind]
    ci = list(CAMERAS).index(cam) if kind == "image" else 0
    return 50000 + 1000 * ci + 10 * base + 3 * list(LOSSES).index(loss) + flags + (n == 6000) + 100000 * draw


def cases():
    out = [("image", c, f, l, n) for c in CAMERAS for f in FLAGS for l in LOSSES for n in SIZES]
    out += [("pair", "%s-%s" % PAIR, f, l, n) for f in FLAGS for l in LOSSES for n in SIZES]
    out += [(k, "", 0, l, n) for k in MODEL_KINDS for l in LOSSES for n in SIZES]
    out += [("calibrated", "", 0, "CAUCHY", 500), ("mismatch", "", 0, "CAUCHY", 500)]
    return out


def inputs(kind, camera, n, seed):
    """The problem of a case: dict(a, b, model0, weights, loss_scale) and, for the camera cases, the models and start
    parameters of the cameras (model1 / params1, model2 / params2).  model0: pose [7] or matrix [3, 3]."""
    if kind == "image":
        mid = CAMERAS[camera]
        if mid == 9:
            x, X, pose0, p0 = CM.problem("RADIAL_FISHEYE", n, seed, outliers=0.0)
        else:
            x, X, pose0, p0, _ = MG.problem(max(mid, 1), n, seed, outliers=0.0)
        bad = _outliers(x, seed, 60.0)
        scale = MG.LOSS_SCALE
        if mid == -1:
            x = (x - NULL_PP) / NULL_FOCAL
            p0, scale = np.zeros(0), MG.LOSS_SCALE / NULL_FOCAL[0]
        return dict(a=np.ascontiguousarray(x), b=X, model0=pose0, weights=weights(n, seed, bad), loss_scale=scale,
                    model1=mid, params1=np.asarray(p0, float))
    if kind == "pair":
        m1, m2 = (RG.MODELS[c] for c in PAIR)
        x1, x2, pose0, c1, c2 = RG.pair_problem(m1, m2, n, seed)
        bad = _outliers(x2, seed, 20.0)  # two views hold the cameras loosely: milder outliers keep the TRIVIAL loss stable
        return dict(a=x1, b=x2, model0=pose0, weights=weights(n, seed, bad), loss_scale=RG.LOSS_SCALE, model1=m1,
                    params1=np.asarray(c1, float), model2=m2, params2=np.asarray(c2, float))
    rng = np.random.default_rng(seed)
    if kind == "calibrated":
        p = G.abspose_problem(n, 0.8, 31, seed)
        a, b, scale = p["x"] / G.FOCAL, p["X"], 12.0 / G.FOCAL
        m0 = RC._perturbed("pnp", p, rng)
    else:
        p = G.homography_problem(n, 0.8, 34, seed) if kind == "homography" else G.relpose_problem(n, 0.8, 32, seed)
        a, b, scale = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL, 2.0 / G.FOCAL
        m0 = RC._perturbed("relpose" if kind == "mismatch" else kind, p, rng)
    w = weights(n, seed, ~p["is_inlier"])
    if kind == "mismatch":
        w = w[:-1]  # one weight short: the reference falls back to uniform weights
    return dict(a=np.ascontiguousarray(a), b=np.ascontiguousarray(b), model0=m0, weights=w, loss_scale=scale)


def build_client(out_dir=None, alt=False):
    """Compiles tests/ref_weights_client.cc into a shared library linked with oracle/_ref/libplref2.so (alt:
    libplref2_alt.so, the client itself compiled with the same summation order)."""
    target, lib = ("ref2alt", "plref2_alt") if alt else ("ref2", "plref2")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s", target], stdout=subprocess.DEVNULL,
                          stderr=subprocess.DEVNULL)
    refdir = os.path.join(ROOT, "oracle", "_ref")
    out_dir = out_dir or tempfile.mkdtemp(prefix="ref_weights_")
    so = os.path.join(out_dir, "libref_weights%s.so" % ("_alt" if alt else ""))
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-w", "-Wno-psabi", "-shared"] +
                          (["-DMINI_EIGEN_ALT_ORDER"] if alt else []) +
                          ["-I" + os.path.join(ROOT, "oracle", "ref", "mini"), "-I" + os.path.join(ROOT, "oracle"),
                           "-I" + MG.REF, os.path.join(ROOT, "tests", "ref_weights_client.cc"), "-L" + refdir,
                           "-l" + lib, "-Wl,-rpath," + refdir, "-o", so])
    return C.CDLL(so, mode=os.RTLD_LAZY)


_p = MG._p


def _hex(v):
    return [float(x).hex() for x in np.asarray(v, float).reshape(-1)]


def ref_case(lib, case, seed):
    """Runs one case on the reference; returns its fixture record."""
    kind, camera, flags, loss, n = case
    I = inputs(kind, camera, n, seed)
    a, b, w = I["a"], I["b"], np.ascontiguousarray(I["weights"])
    st = np.zeros(3)
    opt = (LOSSES[loss], C.c_double(I["loss_scale"]), MAX_ITERATIONS, C.c_double(RELATIVE_COST_TOL))
    wargs = (_p(w), C.c_int64(len(w)), _p(st))
    rec = dict(kind=kind, camera=camera, flags=flags, loss=loss, n=n, seed=seed)
    if kind in ("image", "pair"):
        pose = I["model0"].copy()
        p1 = np.zeros(8)
        p1[:len(I["params1"])] = I["params1"]
        if kind == "image":
            lib.rw_bundle_adjust_image(I["model1"], _p(p1), C.c_int64(n), _p(a), _p(b), _p(pose), *opt, flags, *wargs)
        else:
            p2 = np.zeros(8)
            p2[:len(I["params2"])] = I["params2"]
            lib.rw_refine_relpose_pair(I["model1"], _p(p1), I["model2"], _p(p2), C.c_int64(n), _p(a), _p(b), _p(pose),
                                       *opt, flags, *wargs)
            rec["params2"] = _hex(p2[:len(I["params2"])])
        rec["params1"] = _hex(p1[:len(I["params1"])])
        model = pose
    elif kind in ("calibrated", "relpose", "mismatch"):
        model = I["model0"].copy()
        fn = lib.rw_bundle_adjust if kind == "calibrated" else lib.rw_refine_relpose
        fn(C.c_int64(n), _p(a), _p(b), _p(model), *opt, *wargs)
    else:
        m = np.ascontiguousarray(I["model0"].T.reshape(-1))  # column-major
        lib.rw_refine_matrix(int(kind == "homography"), C.c_int64(n), _p(a), _p(b), _p(m), *opt, *wargs)
        model = m.reshape(3, 3).T
    rec.update(iterations=int(st[0]), initial_cost=float(st[1]).hex(), cost=float(st[2]).hex(), model=_hex(model))
    return rec


def agree(r, s):
    """ref2 and ref2alt records of one case: same iteration count, model and parameters within AGREE_TOL."""
    if r["iterations"] != s["iterations"]:
        return False
    for key in ("model", "params1", "params2"):
        x = np.array([float.fromhex(v) for v in r.get(key, [])])
        y = np.array([float.fromhex(v) for v in s.get(key, [])])
        if np.any(np.abs(x - y) > AGREE_TOL * np.maximum(1.0, np.abs(y))):
            return False
    return True


_libs = None


def _agreeing_case(case):
    """The first draw of a case on which ref2 and ref2alt agree (its ref2 record), or None."""
    global _libs
    if _libs is None:
        d = tempfile.mkdtemp(prefix="ref_weights_")
        _libs = build_client(d), build_client(d, alt=True)
    for draw in range(MAX_DRAWS):
        seed = seed_of(case, draw)
        r = ref_case(_libs[0], case, seed)
        if agree(r, ref_case(_libs[1], case, seed)):
            return r
    return None


def main():
    import multiprocessing
    build_client(), build_client(alt=True)  # the reference builds, once, before the workers start
    with multiprocessing.Pool() as pool:
        recs = pool.map(_agreeing_case, cases(), chunksize=1)
    bad = [c for c, r in zip(cases(), recs) if r is None]
    if bad:
        sys.exit("ref2 and ref2alt disagree on every draw of %d cases, e.g. %s: not written" % (len(bad), bad[:5]))
    gold = dict(relative_cost_tol=RELATIVE_COST_TOL, max_iterations=MAX_ITERATIONS, cases=recs)
    with open(OUT, "w") as f:
        json.dump(gold, f, indent=0)
    print("wrote", OUT, len(recs), "cases")


if __name__ == "__main__":
    main()
