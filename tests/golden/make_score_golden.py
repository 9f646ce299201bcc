"""Writes tests/golden/reference_scores.json: PoseLib's own scorers and get_inliers on given models.

Every case is one (kind, n, model set) of the plb_score_batch table:
  * pnp: compute_msac_score / get_inliers(pose, x, X) (robust/utils.cc:36-63,374-383);
  * relpose: compute_sampson_msac_score / get_inliers(pose, x1, x2) (:158-201,434-476);
  * tangent: compute_tangent_sampson_msac_score / get_tangent_sampson_inliers (:269-298,541-569) on the bearings and
    unprojection Jacobians the cameras give the pixels (ransac.cc:155-168), for a PINHOLE / RADIAL pair and a
    DIVISION / SIMPLE_DIVISION pair (the device's division functions equal the host build bit for bit);
  * fundamental: compute_sampson_msac_score / get_inliers(F, x1, x2) (:204-239,479-513);
  * homography: compute_homography_msac_score / get_homography_inliers (:300-329,331-351);
at n in SIZES.  Models: the ground truth, a perturbed one, random ones, the minimal solvers' hypotheses on random
samples, and degenerate ones (a NaN entry, a zero matrix, a PnP pose with the points behind the camera).

The outputs come from the reference's sources compiled on mini-Eigen (oracle/_ref/libplref2.so, `make -C oracle ref2`;
the camera pre-step through tests/ref_camera_models_client.cc); the inputs are regenerated from the seeds by inputs(), so
the file holds seeds, thresholds and results only: counts, scores as hex floats and masks as packed hex bits.

    python tests/golden/make_score_golden.py          (needs the reference checkout; CPU only)
"""
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_camera_models_golden as CM  # noqa: E402
import make_intrinsics_golden as MG  # noqa: E402

ROOT = MG.ROOT
OUT = os.path.join(HERE, "reference_scores.json")
SIZES = (0, 1, 255, 256, 257, 2000)
KINDS = ("pnp", "relpose", "tangent", "fundamental", "homography")
PAIRS = (("PINHOLE", "RADIAL"), ("DIVISION-", "SIMPLE_DIVISION+"))
N_RANDOM, N_SOLVED = 3, 4


def seed_of(kind, n, pair=0):
    return 90000 + 1000 * KINDS.index(kind) + 100 * pair + SIZES.index(n)


def _quat(rng, scale=1.0):
    q = np.concatenate([[1.0], rng.normal(scale=scale, size=3)])
    return q / np.linalg.norm(q)


def _rot(q):
    return MG.quat_to_rot(q)


def _unit(x):
    return x / np.linalg.norm(x, axis=-1, keepdims=True)


def _cm(M):
    return np.asarray(M, dtype=np.float64).T.reshape(-1)


def _skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def inputs(kind, n, pair=0):
    """The correspondences (a, b), the squared threshold, the pixels' cameras (tangent) and the model rows of one case:
    poses [m, 7] or column-major matrices [m, 9].  Everything is drawn from the case's seed with NumPy's legacy
    RandomState, identical on every machine, so the GPU tests rebuild the exact inputs."""
    rng = np.random.RandomState(seed_of(kind, n, pair))
    N = max(n, 8)  # the solvers need samples: the small sizes are a prefix of a larger scene
    q, t = _quat(rng, 0.2), rng.normal(size=3)
    models = []
    out = {"cam1": None, "cam2": None}
    if kind == "tangent":
        c1, c2 = PAIRS[pair]
        x1, x2, pose0, _, _ = CM.pair_problem(c1, c2, N, seed_of(kind, n, pair), outliers=0.3)
        a, b = x1[:n], x2[:n]
        sq = 1.5 ** 2
        models.append(pose0)
        out.update(cam1=(CM.model_id(c1), CM.CAMERAS[c1][1]), cam2=(CM.model_id(c2), CM.CAMERAS[c2][1]))
        gt_pose = None
    elif kind == "pnp":
        X = rng.uniform(-2, 2, size=(N, 3)) + [0, 0, 6]
        Z = X @ _rot(q).T + t
        x = Z[:, :2] / Z[:, 2:] + rng.normal(scale=1e-3, size=(N, 2))
        bad = rng.uniform(size=N) < 0.3
        x[bad] = rng.uniform(-0.5, 0.5, size=(int(bad.sum()), 2))
        a, b, sq = x[:n], X[:n], 0.004 ** 2
        gt_pose = np.concatenate([q, t])
        behind = np.concatenate([q, -t - np.array([0, 0, 20.0])])  # every point behind the camera
        models += [gt_pose, behind]
    else:
        X = rng.uniform(-2, 2, size=(N, 3)) + [0, 0, 6]
        if kind == "homography":
            X[:, 2] = 6.0 + 0.3 * X[:, 0]
        tt = _unit(rng.normal(size=3))
        Z2 = X @ _rot(q).T + tt
        x1 = X[:, :2] / X[:, 2:] + rng.normal(scale=1e-3, size=(N, 2))
        x2 = Z2[:, :2] / Z2[:, 2:] + rng.normal(scale=1e-3, size=(N, 2))
        bad = rng.uniform(size=N) < 0.3
        x2[bad] = rng.uniform(-0.5, 0.5, size=(int(bad.sum()), 2))
        a, b = x1[:n], x2[:n]
        sq = 0.003 ** 2
        gt_pose = np.concatenate([q, tt])
        if kind == "relpose":
            models.append(gt_pose)
        elif kind == "fundamental":
            models += [_cm(_skew(tt) @ _rot(q)), _cm(np.zeros((3, 3)))]
        else:
            nrm, d = np.array([-0.3, 0.0, 1.0]) / 6.0, 1.0  # plane 6 + 0.3 x = z  <=>  n.X = 1
            models += [_cm(_rot(q) + np.outer(tt, nrm / d)), _cm(np.zeros((3, 3)))]
    msz = 7 if kind in ("pnp", "relpose", "tangent") else 9
    base = models[0]
    pert = base + rng.normal(scale=1e-3, size=msz)
    if msz == 7:
        pert[:4] /= np.linalg.norm(pert[:4])
    models.append(pert)
    for _ in range(N_RANDOM):
        r = rng.normal(size=msz)
        if msz == 7:
            r[:4] /= np.linalg.norm(r[:4])
        models.append(r)
    nan = base.copy()
    nan[msz - 1] = np.nan
    models.append(nan)
    out.update(a=np.ascontiguousarray(a, dtype=np.float64), b=np.ascontiguousarray(b, dtype=np.float64), sq=sq,
               models=np.array(models), solver_src=(None if kind == "tangent" else (x1 if kind != "pnp" else x, None if kind == "pnp" else x2, X, rng.randint(0, 2 ** 31, N_SOLVED))))
    return out


def _sample_bearings(x, idx):
    return np.ascontiguousarray(_unit(np.column_stack([x[idx], np.ones(len(idx))])))


def solver_models(lib, kind, I):
    """Hypotheses of the reference's minimal solvers on random samples of the case's scene."""
    if I["solver_src"] is None:
        return []
    xa, xb, X, seeds = I["solver_src"]
    out = []
    P = C.POINTER(C.c_double)
    for s in seeds:
        rng = np.random.RandomState(int(s))
        if kind == "pnp":
            idx = rng.choice(len(X), 3, replace=False)
            xb3, Xs = _sample_bearings(xa, idx), np.ascontiguousarray(X[idx])
            buf = np.zeros(4 * 7)
            k = lib.plr2_p3p(xb3.ctypes.data_as(P), Xs.ctypes.data_as(P), buf.ctypes.data_as(P))
            out += list(buf.reshape(4, 7)[:k])
        elif kind == "relpose":
            idx = rng.choice(len(xa), 5, replace=False)
            b1, b2 = _sample_bearings(xa, idx), _sample_bearings(xb, idx)
            buf = np.zeros(40 * 7)
            k = lib.plr2_relpose_5pt(b1.ctypes.data_as(P), b2.ctypes.data_as(P), buf.ctypes.data_as(P))
            out += list(buf.reshape(40, 7)[:k][:3])
        elif kind == "fundamental":
            idx = rng.choice(len(xa), 7, replace=False)
            b1 = np.ascontiguousarray(np.column_stack([xa[idx], np.ones(7)]))
            b2 = np.ascontiguousarray(np.column_stack([xb[idx], np.ones(7)]))
            buf = np.zeros(3 * 9)
            k = lib.plr2_relpose_7pt(b1.ctypes.data_as(P), b2.ctypes.data_as(P), buf.ctypes.data_as(P))
            out += list(buf.reshape(3, 9)[:k])
        else:
            idx = rng.choice(len(xa), 4, replace=False)
            b1 = np.ascontiguousarray(np.column_stack([xa[idx], np.ones(4)]))
            b2 = np.ascontiguousarray(np.column_stack([xb[idx], np.ones(4)]))
            buf = np.zeros(9)
            k = lib.plr2_homography_4pt(b1.ctypes.data_as(P), b2.ctypes.data_as(P), buf.ctypes.data_as(P), 1)
            if k:
                out.append(buf.copy())
    return out


def all_models(lib, kind, I):
    sol = solver_models(lib, kind, I)
    return np.ascontiguousarray(np.vstack([I["models"]] + ([np.array(sol)] if sol else [])), dtype=np.float64)


def tangent_inputs(cmlib, I):
    """d1, d2 [n, 3] and M1, M2 [n, 6] of the pixels through the reference's Camera::unproject_with_jac."""
    res = []
    for x, (mid, params) in ((I["a"], I["cam1"]), (I["b"], I["cam2"])):
        n = len(x)
        p8 = np.zeros(8)
        p8[:len(params)] = params
        bufs = [np.zeros(max(1, k * n)) for k in (3, 2, 3, 6, 24, 3, 24)]
        P = C.POINTER(C.c_double)
        xp = np.ascontiguousarray(x, dtype=np.float64)
        cmlib.cm_unproject(int(mid), p8.ctypes.data_as(P), C.c_int64(n), xp.ctypes.data_as(P),
                           *[bb.ctypes.data_as(P) for bb in bufs])
        res.append((bufs[2][:3 * n].copy(), bufs[3][:6 * n].copy()))
    return res


def reference(lib, cmlib, kind, I, models):
    """counts, scores, masks of every model (the reference's scorer and get_inliers)."""
    n = len(I["a"])
    P = C.POINTER(C.c_double)
    a, b = I["a"], I["b"]
    counts, scores, masks = [], [], []
    if kind == "tangent":
        (d1, M1), (d2, M2) = tangent_inputs(cmlib, I)
    for mo in models:
        mo = np.ascontiguousarray(mo, dtype=np.float64)
        cnt = C.c_uint64(0)
        mask = np.zeros(max(n, 1), dtype=np.int8)
        mp, mk = mo.ctypes.data_as(P), mask.ctypes.data_as(C.c_char_p)
        if kind == "tangent":
            s = lib.plr2_score_tangent(mp, d1.ctypes.data_as(P), d2.ctypes.data_as(P), M1.ctypes.data_as(P),
                                       M2.ctypes.data_as(P), C.c_uint64(n), C.c_double(I["sq"]), C.byref(cnt), mk)
        else:
            args = (mp, a.ctypes.data_as(P), b.ctypes.data_as(P), C.c_uint64(n), C.c_double(I["sq"]))
            s = getattr(lib, "plr2_score_" + kind)(*args, C.byref(cnt))
            getattr(lib, "plr2_inliers_" + kind)(*args, mk)
        counts.append(int(cnt.value))
        scores.append(float(s).hex())
        masks.append(pack(mask[:n]))
    return counts, scores, masks


def pack(mask):
    return np.packbits(np.asarray(mask, dtype=np.uint8) != 0, bitorder="little").tobytes().hex()


def unpack(h, n):
    return np.unpackbits(np.frombuffer(bytes.fromhex(h), dtype=np.uint8), bitorder="little")[:n].astype(bool)


def load_libs():
    so = os.path.join(ROOT, "oracle", "_ref", "libplref2.so")
    lib = C.CDLL(so, mode=os.RTLD_LAZY)
    for f in ("plr2_score_pnp", "plr2_score_relpose", "plr2_score_fundamental", "plr2_score_homography",
              "plr2_score_tangent"):
        getattr(lib, f).restype = C.c_double
    return lib, CM.build_client()


def cases():
    for kind in KINDS:
        for pair in (range(len(PAIRS)) if kind == "tangent" else (0,)):
            for n in SIZES:
                yield kind, n, pair


def generate():
    lib, cmlib = load_libs()
    out = []
    for kind, n, pair in cases():
        I = inputs(kind, n, pair)
        models = all_models(lib, kind, I)
        counts, scores, masks = reference(lib, cmlib, kind, I, models)
        out.append({"kind": kind, "n": n, "pair": pair, "sq_threshold": I["sq"].hex(),
                    "models": [[float(v).hex() for v in mo] for mo in models], "counts": counts, "scores": scores,
                    "masks": masks})
    return {"cases": out}


if __name__ == "__main__":
    with open(OUT, "w") as f:
        json.dump(generate(), f, indent=0)
        f.write("\n")
    print("wrote", OUT)
