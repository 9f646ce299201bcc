"""Writes tests/golden/reference_generate.json: PoseLib's own estimators' generate_models and score_model on the samples
their RandomSampler draws.

Every case is one (kind, n) of the plb_generate_batch table, S = 20 calls of generate_models in a row:
  * pnp: AbsolutePoseEstimator (robust/estimators/absolute_pose.cc:46-58);
  * relpose: RelativePoseEstimator (relative_pose.cc:48-60);
  * tangent: CameraRelativePoseEstimator (:88-99) on the pixels of a PINHOLE / RADIAL and a DIVISION / SIMPLE_DIVISION
    pair;
  * fundamental: FundamentalEstimator (:384-403) with real_focal_check off and on;
  * homography: HomographyEstimator (homography.cc:36-52);
at n in SIZES (n = k: the first k points of the n = 256 scene), plus a PROSAC case of relpose and of homography.  The
scenes are make_score_golden.inputs(), max_error = sqrt of its squared threshold, the seed seed_of().

The outputs come from the reference's sources compiled on mini-Eigen (oracle/_ref/libplref2.so, `make -C oracle ref2`),
called through tests/ref_generate_client.cc; the inputs are regenerated from the seeds, so the file holds seeds,
thresholds and results only: per sample the indices, the model count, the models as hex floats and score_model's
(score, count) of each, one line per sample.  Every case is also run on oracle/_ref/libplref2_alt.so (mini-Eigen's other summation order);
only the samples whose model count and counts agree between the two builds are kept, so the file does not record
discrete outcomes that hang on Eigen's unpinned summation order.

    python tests/golden/make_generate_golden.py          (needs the reference checkout; CPU only)
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
import make_camera_models_golden as CM  # noqa: E402
import make_score_golden as SG  # noqa: E402

ROOT = SG.ROOT
REF = CM.REF
OUT = os.path.join(HERE, "reference_generate.json")
S = 20
K = {"pnp": 3, "relpose": 5, "tangent": 5, "fundamental": 7, "homography": 4}
M = {"pnp": 4, "relpose": 40, "tangent": 40, "fundamental": 3, "homography": 1}
CLIENT_KIND = {"pnp": 0, "relpose": 1, "tangent": 2, "fundamental": 3, "homography": 4}
SIZES = ("k", 257, 2000)


def cases():
    """(kind, n, pair, rfc, prosac) of every case; n is "k" for the sample size."""
    for kind in ("pnp", "relpose", "tangent", "fundamental", "homography"):
        for pair in ((0, 1) if kind == "tangent" else (0,)):
            for rfc in ((0, 1) if kind == "fundamental" else (0,)):
                for n in SIZES:
                    yield kind, n, pair, rfc, 0
    yield "relpose", 2000, 0, 0, 1
    yield "homography", 2000, 0, 0, 1


def seed_of(kind, n, pair, rfc, prosac):
    return 70000 + 1000 * CLIENT_KIND[kind] + 100 * pair + 10 * (SIZES.index(n)) + 2 * rfc + prosac


def inputs(kind, n, pair):
    """a, b (pixels for tangent), max_error and the cameras (tangent) of a case, from make_score_golden's scenes."""
    I = SG.inputs(kind, 256 if n == "k" else n, pair)
    m = K[kind] if n == "k" else n
    max_error = float(np.sqrt(I["sq"]))
    return {"a": np.ascontiguousarray(I["a"][:m]), "b": np.ascontiguousarray(I["b"][:m]), "max_error": max_error,
            "cam1": I["cam1"], "cam2": I["cam2"]}


def build_client(alt=False):
    target, lib = ("ref2alt", "plref2_alt") if alt else ("ref2", "plref2")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s", target], stdout=subprocess.DEVNULL,
                          stderr=subprocess.DEVNULL)
    refdir = os.path.join(ROOT, "oracle", "_ref")
    so = os.path.join(tempfile.mkdtemp(prefix="ref_generate_"), "libref_generate%s.so" % ("_alt" if alt else ""))
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-w", "-Wno-psabi", "-shared"] +
                          (["-DMINI_EIGEN_ALT_ORDER"] if alt else []) +
                          ["-I" + os.path.join(ROOT, "oracle", "ref", "mini"), "-I" + os.path.join(ROOT, "oracle"),
                           "-I" + REF, os.path.join(ROOT, "tests", "ref_generate_client.cc"), "-L" + refdir,
                           "-l" + lib, "-Wl,-rpath," + refdir, "-o", so])
    return C.CDLL(so, mode=os.RTLD_LAZY)  # the estimators name out-of-scope solvers that are never called


def run(lib, kind, n, pair, rfc, prosac):
    I = inputs(kind, n, pair)
    m, k, Mk = len(I["a"]), K[kind], M[kind]
    msz = 9 if kind in ("fundamental", "homography") else 7
    smp = np.zeros((S, k), dtype=np.int32)
    nm = np.zeros(S, dtype=np.int32)
    models = np.zeros((S, Mk, msz))
    scores = np.zeros((S, Mk))
    counts = np.zeros((S, Mk), dtype=np.uint64)
    P = C.POINTER(C.c_double)
    cams = []
    for c in (I["cam1"], I["cam2"]):
        p8 = np.zeros(8)
        if c is not None:
            p8[:len(c[1])] = c[1]
        cams.append((int(c[0]) if c is not None else -1, p8))
    lib.gen_run(CLIENT_KIND[kind], int(rfc), I["a"].ctypes.data_as(P), I["b"].ctypes.data_as(P), C.c_int64(m),
                cams[0][0], cams[0][1].ctypes.data_as(P), cams[1][0], cams[1][1].ctypes.data_as(P),
                C.c_double(I["max_error"]), C.c_uint64(seed_of(kind, n, pair, rfc, prosac)), int(prosac), C.c_int64(S),
                smp.ctypes.data_as(C.POINTER(C.c_int32)), nm.ctypes.data_as(C.POINTER(C.c_int32)),
                models.ctypes.data_as(P), scores.ctypes.data_as(P), counts.ctypes.data_as(C.POINTER(C.c_uint64)))
    return smp, nm, models, scores, counts


def generate():
    lib, alt = build_client(), build_client(alt=True)
    out = []
    for kind, n, pair, rfc, prosac in cases():
        smp, nm, models, scores, counts = run(lib, kind, n, pair, rfc, prosac)
        _, nm_a, _, _, counts_a = run(alt, kind, n, pair, rfc, prosac)
        samples = []
        for j in range(S):
            c = int(nm[j])
            if nm_a[j] != c or not np.array_equal(counts[j, :c], counts_a[j, :c]):
                continue
            samples.append({"j": j, "sample": smp[j].tolist(), "n_models": c,
                            "models": [[float(v).hex() for v in models[j, i]] for i in range(c)],
                            "scores": [float(scores[j, i]).hex() for i in range(c)],
                            "counts": [int(counts[j, i]) for i in range(c)]})
        out.append({"kind": kind, "n": n, "pair": pair, "rfc": rfc, "prosac": prosac,
                    "seed": seed_of(kind, n, pair, rfc, prosac), "max_error": inputs(kind, n, pair)["max_error"].hex(),
                    "samples": samples})
    return {"cases": out}


def dump(data, f):
    """One line per case header and per sample."""
    cases = data["cases"]
    f.write('{"cases": [\n')
    for ci, c in enumerate(cases):
        head = json.dumps({k: v for k, v in c.items() if k != "samples"})
        f.write(head[:-1] + ', "samples": [\n')
        for si, smp in enumerate(c["samples"]):
            f.write(json.dumps(smp, separators=(",", ":")) + ("," if si + 1 < len(c["samples"]) else "") + "\n")
        f.write("]}" + ("," if ci + 1 < len(cases) else "") + "\n")
    f.write("]}\n")


if __name__ == "__main__":
    with open(OUT, "w") as f:
        dump(generate(), f)
    print("wrote", OUT)
