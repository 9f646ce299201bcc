"""The fp32 screening records of the device (k_screen) against fp64, and the depth of their sums.

GPU (tests/screen_device_test.cu): the library's own steps — launch_transpose, k_screen_ctx, k_screen, launch_score_models
— on problems of every kind, at sizes around the chunk edges of both CTA widths (32 NTHR correspondences), the NaN
padding of the staged arrays and the staging limit, with 1 to ~200 models per problem, good, perturbed, random and
degenerate ones, several grid sizes and batches of problems in one launch.  Every record must bracket the fp64 record
(count64 in [count32 +- border], |score64 - score32| <= err) whenever k_select would use it, the device's fp64 record
must be the oracle's, and count32 / border (every launch) and score32 / err (every launch of one CTA width) must not
depend on the grid or the staging path.

CPU: the warp-compacted queue pass of k_screen restated in Python.  A recorded case lands in the sums of the lane that
picks it from the queue, not of the lane that owns the correspondence, so one lane can add many more than n / NTHR
terms to a model's sum; the error term of the record (scr::record_err, screen_math.cuh) must cover the depth that
adversarial hit patterns reach."""
import ctypes as C
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

from poselib_b200 import problem_generator as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests")
CSRC = os.path.join(ROOT, "poselib_b200", "csrc")

U = 2.0 ** -24
TM = 8         # SCR_TM (kernels.cu)
RQ_TAKE = 8    # SCR_RQ_TAKE (kernels.cu)
STAGE_BYTES = 200 * 1024  # the staging buffer launch_hyp_t allows
PB = 4         # SCR_PB: scr_stage_len pads to multiples of PB * NTHR


# ============================================================================================================
# CPU: restatement of the queue pass
# ============================================================================================================
def queue_pass(hit):
    """One chunk of one warp: the compacted handling of the recorded cases (kernels.cu:1188-1261, k_screen's `for (;;)`
    loop after the streaming steps).  hit[lane][model]: the lane's 32-bit mask of recorded correspondences of the model
    (bit q: correspondence base + tid + q NTHR).  Returns terms[lane][model], the cases each lane adds to its own
    accumulators of the model (cnt / sc / er), and the largest number of entries one lane handled in one pass."""
    hit = [[int(h) for h in row] for row in hit]
    terms = np.zeros((32, TM), dtype=np.int64)
    per_pass = 0
    while True:
        mine = [sum(bin(h).count("1") for h in row) for row in hit]  # mine += __popc(hit[i])
        if not any(mine):                                             # !__any_sync(mine > 0)
            break
        queue = []  # the lanes' entries at their exclusive prefix of take, i.e. in lane order
        for lane in range(32):
            for _ in range(min(mine[lane], RQ_TAKE)):  # take = min(mine, SCR_RQ_TAKE)
                mi = next(i for i in range(TM) if hit[lane][i])  # lowest model with a case left
                hm = hit[lane][mi]
                hit[lane][mi] = hm & (hm - 1)                    # its lowest bit (__ffs)
                queue.append(mi)
        handled = np.zeros(32, dtype=np.int64)
        for e, mi in enumerate(queue):  # for (eidx = lane; eidx < total; eidx += 32): lands in lane eidx & 31's sums
            terms[e % 32, mi] += 1
            handled[e % 32] += 1
        per_pass = max(per_pass, int(handled.max()))
    return terms, per_pass


def masks_from_counts(counts, rng):
    """hit masks with counts[lane][model] recorded cases each (which bits does not change who handles what)"""
    hit = np.zeros((32, TM), dtype=np.int64)
    for lane in range(32):
        for i in range(TM):
            bits = rng.choice(32, int(counts[lane][i]), replace=False)
            hit[lane, i] = int(sum(1 << int(b) for b in bits))
    return hit


# Found by a seeded hill climb over the per-(lane, model) case counts of one warp and chunk: lane 19 ends up adding 78
# terms to model 3's sums (its own cases of that model: 32, one per correspondence of the chunk).
ADVERSARIAL_COUNTS = [
    [13, 3, 7, 21, 7, 12, 10, 0], [18, 23, 32, 13, 8, 26, 10, 2], [0, 22, 13, 28, 28, 12, 24, 32],
    [27, 27, 19, 31, 28, 11, 27, 32], [17, 0, 27, 32, 24, 12, 11, 22], [32, 32, 19, 17, 0, 17, 23, 30],
    [24, 2, 16, 28, 29, 29, 32, 21], [32, 32, 29, 32, 0, 30, 10, 32], [11, 20, 19, 32, 32, 16, 3, 18],
    [32, 32, 1, 29, 10, 8, 29, 24], [28, 24, 3, 13, 10, 0, 15, 11], [6, 32, 32, 32, 28, 11, 18, 7],
    [32, 32, 32, 28, 21, 29, 6, 27], [14, 25, 29, 30, 5, 23, 21, 11], [11, 0, 32, 26, 32, 21, 20, 18],
    [28, 18, 26, 32, 18, 9, 27, 9], [32, 32, 29, 32, 30, 29, 16, 0], [23, 6, 16, 30, 22, 32, 18, 23],
    [7, 11, 12, 31, 14, 18, 0, 12], [28, 19, 26, 32, 2, 27, 8, 12], [24, 13, 0, 11, 19, 13, 23, 32],
    [32, 32, 32, 30, 32, 26, 0, 24], [12, 14, 3, 32, 13, 29, 31, 11], [26, 12, 31, 32, 8, 5, 2, 19],
    [17, 0, 12, 32, 30, 6, 12, 25], [32, 32, 32, 32, 2, 9, 0, 31], [0, 0, 0, 30, 2, 3, 0, 6],
    [11, 8, 18, 32, 11, 0, 0, 28], [26, 24, 19, 32, 22, 23, 4, 28], [14, 6, 30, 24, 31, 24, 17, 1],
    [2, 0, 7, 27, 11, 24, 7, 26], [5, 24, 7, 32, 13, 4, 5, 14]]
# The same search restricted to at most one model per correspondence (what data can realise with the translations of
# the skewed-queue problem below): lane 27 adds 20 terms to model 3's sums while owning 16 of its cases.
SKEW_COUNTS = [
    [1, 3, 3, 5, 2, 4, 2, 0], [3, 4, 1, 2, 5, 2, 4, 2], [5, 0, 4, 0, 0, 0, 6, 11], [0, 1, 0, 3, 0, 0, 0, 1],
    [0, 3, 3, 6, 12, 3, 4, 0], [7, 2, 0, 8, 8, 0, 4, 1], [0, 5, 2, 1, 9, 0, 0, 0], [5, 0, 1, 9, 0, 2, 0, 10],
    [2, 3, 6, 1, 0, 6, 0, 14], [4, 7, 8, 9, 4, 0, 0, 0], [9, 8, 0, 0, 4, 0, 9, 0], [0, 3, 2, 3, 2, 0, 2, 0],
    [5, 0, 0, 12, 1, 0, 5, 6], [0, 14, 2, 9, 0, 0, 4, 3], [1, 0, 1, 0, 2, 5, 0, 0], [0, 6, 0, 1, 0, 4, 0, 0],
    [5, 8, 1, 10, 4, 1, 2, 0], [2, 0, 1, 4, 6, 2, 6, 5], [8, 2, 1, 1, 0, 6, 5, 0], [1, 0, 5, 9, 0, 0, 5, 9],
    [5, 9, 0, 3, 3, 0, 1, 4], [0, 0, 0, 0, 0, 0, 0, 0], [4, 3, 0, 10, 0, 8, 7, 0], [4, 0, 0, 0, 2, 0, 4, 0],
    [3, 2, 1, 8, 6, 9, 0, 0], [5, 5, 1, 0, 6, 9, 4, 2], [3, 1, 13, 0, 4, 3, 0, 0], [1, 4, 9, 16, 0, 0, 0, 2],
    [0, 0, 3, 7, 0, 0, 0, 0], [3, 0, 6, 6, 3, 0, 3, 8], [3, 5, 7, 2, 3, 3, 3, 0], [0, 8, 0, 0, 11, 7, 4, 1]]


def search_counts(seed, steps):
    """Seeded hill climb over the case counts of one warp and chunk, maximising the terms one lane adds to one sum"""
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, 33, (32, TM))

    def value(c):
        return int(queue_pass(masks_from_counts(c, np.random.default_rng(0)))[0].max())

    best = value(counts)
    for _ in range(steps):
        cand = counts.copy()
        for _ in range(rng.integers(1, 4)):
            lane, i = rng.integers(32), rng.integers(TM)
            cand[lane, i] = np.clip(cand[lane, i] + rng.integers(-8, 9), 0, 32)
        v = value(cand)
        if v >= best:
            best, counts = v, cand
    return counts


HOST_SRC = r"""
#include "screen_math.cuh"
using namespace plb::scr;
extern "C" float rec_err(float e_sum, unsigned count, unsigned border, float thr, int n, int nthr) {
    return record_err(e_sum, count, border, thr, n, nthr);
}
// REC_ERR0 of a model as k_screen_ctx sets it (kind as in kernels.cuh; M row-major fp64, 3x4 for pnp)
extern "C" float rec_err0(int kind, const double *M, const float *cmax, double sq_thr) {
    float ctx[CTX_FLOATS] = {0};
    if (kind == 0) transfer_setup<3>(M, cmax + 2, cmax, sq_thr, ctx);
    else if (kind == 3) transfer_setup<2>(M, cmax, cmax + 2, sq_thr, ctx);
    else sampson_setup(M, cmax, sq_thr, ctx);
    return ctx[REC_ERR0];
}
"""


rec_err_lib = [None]


@pytest.fixture(scope="module")
def rec_err(tmp_path_factory):
    d = tmp_path_factory.mktemp("screen_depth")
    src, lib = d / "rec_err.cc", d / "rec_err.so"
    src.write_text(HOST_SRC)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I", CSRC, str(src),
                           "-o", str(lib)])
    rec_err_lib[:] = [str(lib)]
    f = C.CDLL(str(lib)).rec_err
    f.argtypes = [C.c_float, C.c_uint, C.c_uint, C.c_float, C.c_int, C.c_int]
    f.restype = C.c_float
    return f


@pytest.fixture(scope="module")
def rec_err0(rec_err):
    f = C.CDLL(rec_err_lib[0]).rec_err0
    f.argtypes = [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_float), C.c_double]
    f.restype = C.c_float
    return f


def test_overflowing_models_and_non_finite_data_make_no_claim(rec_err0):
    """A model whose fp32 evaluation can overflow, or a problem whose coordinate maxima are NaN (a NaN coordinate) or
    infinite, gets REC_ERR0 = +inf: NaN or inf residuals would otherwise read as certain outliers and leave a finite
    record of count32 = border = 0.  Models on well-scaled data keep REC_ERR0 = 0."""
    rng = np.random.default_rng(11)

    def e0(kind, M, cmax, thr=1e-6):
        M = np.ascontiguousarray(M, dtype=np.float64)
        cm = np.ascontiguousarray(cmax, dtype=np.float32)
        return float(rec_err0(kind, M.ctypes.data_as(C.POINTER(C.c_double)), cm.ctypes.data_as(C.POINTER(C.c_float)), thr))

    for kind, msz in ((0, 12), (1, 9), (2, 9), (3, 9)):
        good = [1.0, 1.0, 1.0, 1.0, 10.0]
        for _ in range(200):
            M = rng.normal(size=msz) * 10.0 ** rng.uniform(-3, 3)
            assert e0(kind, M, good) == 0.0, (kind, M)
            assert e0(kind, M, np.array(good) * 1e3, 1.0) == 0.0, (kind, M)  # pixel units
        M = rng.normal(size=msz)
        for bad in (np.nan, np.inf):
            for j in range(5 if kind == 0 else 4):
                cm = list(good)
                cm[j] = bad
                assert e0(kind, M, cm) == np.inf, (kind, bad, j)
        for Mb in (M * 1e30, M * 1e20, np.where(np.arange(msz) == 0, 1e300, M), np.where(np.arange(msz) == 2, np.inf, M)):
            assert e0(kind, Mb, good) == np.inf, (kind, Mb)
        # a NaN model entry reaches every residual: fp64 and the streaming test both reject everything, 0 +- 0 is exact
        assert e0(kind, np.where(np.arange(msz) == 3, np.nan, M), good) == 0.0, kind


def gamma(d):
    return d * U / (1.0 - d * U)


def check_depth(rec_err, counts_per_chunk, nthr):
    """counts_per_chunk: one warp's case counts of every chunk of a problem of len(...) full chunks.  Every case is
    taken as a plain inlier for the score sum (count32 = the cases of the model: the other warps add nothing), and as
    a plain-or-border case for the error sum (count32 + border = the cases of the model)."""
    rng = np.random.default_rng(len(counts_per_chunk))
    terms = np.zeros((32, TM), dtype=np.int64)
    for counts in counts_per_chunk:
        t, per_pass = queue_pass(masks_from_counts(counts, rng))
        assert per_pass <= RQ_TAKE and t.sum(axis=1).max() <= 32 * TM  # the two facts the bound is built on
        terms += t
    n = len(counts_per_chunk) * 32 * nthr
    red = 5 + nthr // 32 + 1  # warp butterfly (kernels.cu:1267), cross-warp sum and + n thr (write_record, 1066-1075)
    worst = []
    for i in range(TM):
        cases = int(sum(np.asarray(c)[:, i].sum() for c in counts_per_chunk))
        if cases == 0:
            continue
        d = int(terms[:, i].max()) + red
        worst.append(d)
        # score sum: |error| <= gamma_d * count32 * thr + the rounding of n thr and of its addition
        need = gamma(d) * cases + 2.0 * U * n
        got = float(rec_err(0.0, cases, 0, 1.0, n, nthr))
        assert got >= need, (nthr, len(counts_per_chunk), i, d, got, need)
        # error sum over nonnegative terms: the true sum is at most the computed one / (1 - gamma_d); with thr = 0 the
        # record's err is the error sum's share alone (as plain cases and as border cases)
        need = 1.0 / (1.0 - gamma(d))
        for c32, bd in ((cases, 0), (0, cases)):
            got = float(rec_err(1.0, c32, bd, 0.0, n, nthr))
            assert got >= need, (nthr, len(counts_per_chunk), i, d, c32, bd, got, need)
    return max(worst)


@pytest.mark.parametrize("chunks", [1, 2, 3, 5])
@pytest.mark.parametrize("nthr", [128, 512])
def test_record_err_covers_the_queue_depth_of_adversarial_patterns(rec_err, nthr, chunks):
    d = check_depth(rec_err, [ADVERSARIAL_COUNTS] * chunks, nthr)
    # not vacuous: a lane adds far more than its own 32 correspondences per chunk
    assert d - (5 + nthr // 32 + 1) >= 70 * chunks
    check_depth(rec_err, [SKEW_COUNTS] * chunks, nthr)


@pytest.mark.parametrize("seed", [0, 1])
def test_record_err_covers_the_queue_depth_of_searched_patterns(rec_err, seed):
    counts = search_counts(seed, 150)
    rng = np.random.default_rng(100 + seed)
    for nthr in (128, 512):
        for chunks in (1, 2, 3):
            mixed = [counts] + [rng.integers(0, 33, (32, TM)) for _ in range(chunks - 1)]
            check_depth(rec_err, [counts] * chunks, nthr)
            check_depth(rec_err, mixed, nthr)


def test_record_err_depth_is_capped_by_the_count(rec_err):
    """A sum never has more terms than it adds up: on a problem of many chunks the bound follows the count, and it
    grows with the chunks (256 terms per lane each) only up to the count."""
    n = 100 * 32 * 512
    few = float(rec_err(0.0, 10, 0, 1.0, n, 512))
    assert few <= (1.25 * (10 + 22) * U * 10 + 2.2 * U * n) * (1 + 2e-5)
    many = float(rec_err(0.0, 200000, 0, 1.0, n, 512))
    assert many >= gamma(256 * 100 + 22) * 200000
    one_chunk = float(rec_err(0.0, 10000, 0, 1.0, 32 * 512, 512))
    assert one_chunk >= gamma(256 + 22) * 10000 and one_chunk < 2 * gamma(256 + 22) * 10000


# ============================================================================================================
# GPU: the device records against fp64
# ============================================================================================================
KINDS = {"pnp": 0, "relpose": 1, "fundamental": 2, "homography": 3}
NARR = {"pnp": 5, "relpose": 4, "fundamental": 4, "homography": 4}
SIZES = [1, 31, 32, 33, 511, 512, 513, 2047, 2048, 2049, 4096, 4097, 10000, 16384, 16385, 40000]
MODEL_COUNTS = [1, 7, 8, 9, 203]


def stage_len(n, nthr):
    return (n + PB * nthr - 1) // (PB * nthr) * (PB * nthr)


def stage_fits(kind, n_pad_max, nthr):
    return NARR[kind] * stage_len(n_pad_max, nthr) * 4 <= STAGE_BYTES


def staging_limit(kind):
    """largest n whose arrays the library stages in shared memory (launch_hyp_t: 512 threads above 2048)"""
    n = 2048
    while stage_fits(kind, (n + 1 + 31) & ~31, 512):
        n += 1
    return n


def quat(R):
    w = np.sqrt(max(0.0, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    if w > 1e-6:
        return np.array([w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)])
    return np.array([0.0, 1.0, 0.0, 0.0])


def essential(q, t):
    R = G.quat_to_rotmat(q)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    return tx @ R


def gen_problem(kind, n, idx, units="normalised"):
    """(a, b, sq_thr, ground-truth model) of a generator problem; pixel units / offset world frames on request"""
    m = max(n, 64)
    if kind == "pnp":
        p = G.abspose_problem(m, 0.5, 71, idx)
        a, b = p["x"][:n] / G.FOCAL, p["X"][:n].copy()
        gt = np.r_[p["q_gt"], p["t_gt"]]
        thr = 12.0 / G.FOCAL
        if units == "offset":  # the world frame far from the origin: X + o, t - R o
            o = np.array([1e3, -2e3, 5e2])
            b += o
            gt = np.r_[p["q_gt"], p["t_gt"] - p["R_gt"] @ o]
        return a, b, thr * thr, gt
    if kind == "homography":
        p = G.homography_problem(m, 0.5, 74, idx)
        a, b, gt = p["x1"][:n] / G.FOCAL, p["x2"][:n] / G.FOCAL, p["H_gt"] / np.linalg.norm(p["H_gt"])
        thr = 1.0 / G.FOCAL
    else:
        p = G.relpose_problem(m, 0.5, 72 if kind == "relpose" else 73, idx)
        a, b = p["x1"][:n] / G.FOCAL, p["x2"][:n] / G.FOCAL
        gt = np.r_[p["q_gt"], p["t_gt"]] if kind == "relpose" else essential(p["q_gt"], p["t_gt"])
        thr = 1.0 / G.FOCAL
    if units == "pixels" and kind != "relpose":  # F / H in pixel units
        K = np.diag([G.FOCAL, G.FOCAL, 1.0])
        Ki = np.linalg.inv(K)
        gt = (K @ gt @ Ki) if kind == "homography" else (Ki.T @ gt @ Ki)
        gt = gt / np.linalg.norm(gt)
        a, b, thr = a * G.FOCAL, b * G.FOCAL, 1.0
    return np.ascontiguousarray(a), np.ascontiguousarray(b), thr * thr, gt


def models_for(kind, gt, count, rng):
    """count models: ground truth, perturbations 1e-4 .. 1e-1, random, t negated (relpose), degenerate ones"""
    pose = kind in ("pnp", "relpose")
    out = [gt]
    for s in (1e-4, 1e-3, 1e-2, 1e-1):
        if pose:
            q = gt[:4] + rng.normal(0, s, 4)
            out.append(np.r_[q / np.linalg.norm(q), gt[4:] + rng.normal(0, s, 3)])
        else:
            M = gt + rng.normal(0, s * np.abs(gt).max(), (3, 3))
            out.append(M / np.linalg.norm(M))
    if kind == "relpose":
        out.append(np.r_[gt[:4], -gt[4:]])  # the mirrored translation: cheirality decides most points
    nan = np.r_[gt[:6], np.nan] if pose else np.where(np.arange(9).reshape(3, 3) == 4, np.nan, gt)
    out += [np.zeros(7) if pose else np.zeros((3, 3)), nan, gt * 1e30]  # 1e30: fp32 products overflow
    degenerate = set(range(len(out) - 3, len(out)))
    while len(out) < count:
        if pose:
            q = rng.normal(size=4)
            out.append(np.r_[q / np.linalg.norm(q), rng.normal(0, 1, 3)])
        else:
            M = rng.normal(size=(3, 3))
            out.append(M / np.linalg.norm(M))
    out = out[:count]
    return out, [i for i in degenerate if i < count]


def dev_model(kind, M):
    return np.asarray(M, dtype=np.float64).reshape(-1) if kind in ("pnp", "relpose") else np.asarray(M).T.reshape(-1)


def oracle_score(kind, M, a, b, sq_thr):
    import plo_py as P
    return P.score(kind, M, a, b, sq_thr)


def near_threshold_set(n, idx, eps_mag):
    """fundamental / relpose data whose Sampson residuals are within eps_mag (relative) of the threshold
    (the construction of test_screen_bounds.test_residuals_on_the_threshold)"""
    rng = np.random.default_rng(idx)
    p = G.relpose_problem(n, 1.0, 34, idx)
    E = essential(p["q_gt"], p["t_gt"])
    x1, x2 = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
    thr = 1.0 / G.FOCAL
    h1 = np.c_[x1, np.ones(n)]
    l = h1 @ E.T
    nrm = l[:, :2] / np.linalg.norm(l[:, :2], axis=1, keepdims=True)
    x2p = x2.copy()
    target = thr * (1 + rng.choice([-1, 1], n) * eps_mag * rng.uniform(0.1, 1, n))
    for _ in range(60):
        h2 = np.c_[x2p, np.ones(n)]
        Cc = np.einsum("ij,ij->i", h2, l)
        Ex2 = h2 @ E
        den = np.sqrt(l[:, 0] ** 2 + l[:, 1] ** 2 + Ex2[:, 0] ** 2 + Ex2[:, 1] ** 2)
        r = Cc / den
        x2p += ((np.sign(r) * target - r) * (den / np.linalg.norm(l[:, :2], axis=1)))[:, None] * nrm
    return x1, x2p, thr * thr, np.r_[p["q_gt"], p["t_gt"]], E


def skewed_queue_problem(nthr, chunks):
    """homography data whose recorded cases reproduce SKEW_COUNTS in warp 0 of every chunk: model i is the translation
    by (0.05 i, 0); correspondence k sits in warp (k mod NTHR) >> 5, lane (k mod NTHR) & 31, bit
    (k mod 32 NTHR) div NTHR of its chunk; an inlier of model i is x1 + (0.05 i, 0) + noise, everything else is far
    from every model."""
    rng = np.random.default_rng(nthr + chunks)
    n = chunks * 32 * nthr
    a = rng.uniform(-0.5, 0.5, (n, 2))
    b = a + np.array([0.0, 0.3]) + rng.uniform(-0.01, 0.01, (n, 2))  # outliers of every model
    for c in range(chunks):
        for lane in range(32):
            bits = rng.permutation(32)
            pos = 0
            for i in range(TM):
                for _ in range(SKEW_COUNTS[lane][i]):
                    k = c * 32 * nthr + bits[pos] * nthr + lane
                    pos += 1
                    b[k] = a[k] + np.array([0.05 * i, 0.0]) + rng.normal(0, 1e-4, 2)
        # the other warps: a few inliers of their own
        for k in range(c * 32 * nthr, (c + 1) * 32 * nthr):
            if (k % nthr) >= 32 and rng.random() < 0.1:
                b[k] = a[k] + np.array([0.05 * rng.integers(TM), 0.0])
    models = [np.array([[1.0, 0, 0.05 * i], [0, 1.0, 0], [0, 0, 1.0]]) for i in range(TM)]
    return a, b, (2e-3) ** 2, models


class Problem:
    def __init__(self, kind, a, b, sq_thr, models, tag, usable_expected=(), gt_index=None):
        self.kind, self.a, self.b, self.sq_thr, self.models, self.tag = kind, a, b, sq_thr, models, tag
        self.usable_expected = list(usable_expected)  # model indices that must come out usable
        self.gt_index = gt_index


def build_cases(kind):
    """list of (problems, configs): every problem set runs on both CTA widths, on the global-memory path and, where the
    arrays fit, the shared-memory path, each at 1, 7, one-wave and more CTAs than tiles"""
    rng = np.random.default_rng(KINDS[kind])
    lim = staging_limit(kind)
    sizes = SIZES + [lim, lim + 1]
    sets = []
    for j, n in enumerate(sizes):
        a, b, sq, gt = gen_problem(kind, n, j)
        count = MODEL_COUNTS[j % len(MODEL_COUNTS)] if n not in (lim, 16384, 40000) else 203
        models, degen = models_for(kind, gt, count, rng)
        ok = [i for i in range(count) if i not in degen]
        sets.append([Problem(kind, a, b, sq, models, f"generator n={n}", ok, 0)])
    for units in ("pixels", "offset"):
        if (units == "offset") != (kind == "pnp"):
            continue
        a, b, sq, gt = gen_problem(kind, 3000, 50, units)
        models, _ = models_for(kind, gt, 40, rng)
        sets.append([Problem(kind, a, b, sq, models, units)])
    if kind in ("relpose", "fundamental"):
        for eps in (1e-3, 1e-5, 1e-7, 1e-9):
            x1, x2, sq, pose, E = near_threshold_set(2000, 3, eps)
            gtm = pose if kind == "relpose" else E
            models, _ = models_for(kind, gtm, 9, rng)
            sets.append([Problem(kind, x1, x2, sq, models, f"near threshold {eps}")])
    # one NaN coordinate poisons cmax: no record of the problem is usable, the fp64 records still match
    a, b, sq, gt = gen_problem(kind, 3000, 60)
    a = a.copy()
    a[17, 1] = np.nan
    models, _ = models_for(kind, gt, 9, rng)
    sets.append([Problem(kind, a, b, sq, models, "nan coordinate")])
    if kind == "homography":
        for nthr, chunks in ((128, 1), (128, 3), (512, 1), (512, 2)):
            a, b, sq, models = skewed_queue_problem(nthr, chunks)
            sets.append([Problem(kind, a, b, sq, models, f"skewed queue {nthr}x{chunks}", range(TM))])
    # batches: one launch over problems of mixed sizes (a CTA restages several problems, the mbarrier phase wraps)
    for sizes_b in ((40, 2049, 700), (5, 10000, 513, 4097, 33)):
        probs = []
        for i, n in enumerate(sizes_b):
            a, b, sq, gt = gen_problem(kind, n, 80 + i)
            models, degen = models_for(kind, gt, (9, 203, 17, 8, 1)[i], rng)
            probs.append(Problem(kind, a, b, sq, models, f"batch n={n}",
                                 [m for m in range(len(models)) if m not in degen], 0))
        sets.append(probs)
    cases = []
    for probs in sets:
        n_pad_max = max((len(p.a) + 31) & ~31 for p in probs)
        n_tiles = sum((len(p.models) + TM - 1) // TM for p in probs)
        grids = [1, 7, 0, n_tiles + 5]
        cfgs = []
        for nthr in (128, 512):
            cfgs.append((nthr, 0, grids))
            if stage_fits(kind, n_pad_max, nthr):
                cfgs.append((nthr, 1, grids))
        cases.append((probs, cfgs))
    return cases


def write_input(path, kind, cases):
    with open(path, "wb") as f:
        f.write(struct.pack("<i", len(cases)))
        for probs, cfgs in cases:
            f.write(struct.pack("<ii", KINDS[kind], len(probs)))
            for p in probs:
                f.write(struct.pack("<iid", len(p.a), len(p.models), p.sq_thr))
                f.write(np.ascontiguousarray(p.a, dtype="<f8").tobytes())
                f.write(np.ascontiguousarray(p.b, dtype="<f8").tobytes())
                for M in p.models:
                    f.write(dev_model(kind, M).astype("<f8").tobytes())
            f.write(struct.pack("<i", len(cfgs)))
            for nthr, smem, grids in cfgs:
                f.write(struct.pack("<iii", nthr, smem, len(grids)))
                f.write(np.asarray(grids, dtype="<i4").tobytes())


REC = np.dtype([("c32", "<u4"), ("border", "<u4"), ("s32", "<f4"), ("err", "<f4")])
REC64 = np.dtype([("c64", "<u4"), ("s64", "<f8")], align=False)


def read_output(path, cases):
    buf = open(path, "rb").read()
    off, res = 0, []
    for probs, cfgs in cases:
        tm = sum(len(p.models) for p in probs)
        runs = []
        for nthr, smem, grids in cfgs:
            for g in grids:
                used = struct.unpack_from("<i", buf, off)[0]
                off += 4
                runs.append(((nthr, smem, g, used), np.frombuffer(buf, REC, tm, off).copy()))
                off += REC.itemsize * tm
        rec64 = np.frombuffer(buf, REC64, tm, off).copy()
        off += REC64.itemsize * tm
        res.append((runs, rec64))
    assert off == len(buf)
    return res


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("screen_device") / "screen_device_test")
    subprocess.check_call(["nvcc", "-std=c++17", "-O3", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-Xcompiler", "-ffp-contract=off", "-o", exe, os.path.join(HERE, "screen_device_test.cu")])
    return exe


def run_kind(harness, tmp_path, kind):
    cases = build_cases(kind)
    inp, outp = tmp_path / "in.bin", tmp_path / "out.bin"
    write_input(inp, kind, cases)
    subprocess.check_call([harness, str(inp), str(outp)])
    return cases, read_output(outp, cases)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_device_records_bracket_fp64(harness, tmp_path, kind):
    cases, res = run_kind(harness, tmp_path, kind)
    n_checked = 0
    for (probs, cfgs), (runs, rec64) in zip(cases, res):
        base = 0
        for p in probs:
            n = len(p.a)
            sl = slice(base, base + len(p.models))
            base += len(p.models)
            c64, s64 = rec64["c64"][sl].astype(np.int64), rec64["s64"][sl]
            # the device's fp64 record is the oracle's
            for m, M in enumerate(p.models):
                s_or, c_or = oracle_score(kind, M, p.a, p.b, p.sq_thr)
                assert c64[m] == c_or, (p.tag, m, c64[m], c_or)
                assert s64[m] == s_or or abs(s64[m] - s_or) <= 1e-12 * n * p.sq_thr, (p.tag, m, s64[m], s_or)
            first = None
            for cfg, rec in runs:
                r = rec[sl]
                assert not np.any(r["c32"] == 0xFFFFFFFF), (p.tag, cfg)  # every record written
                c32, bd = r["c32"].astype(np.float64), r["border"].astype(np.float64)
                s32, err = r["s32"].astype(np.float64), r["err"].astype(np.float64)
                usable = np.isfinite(s32) & np.isfinite(err)  # control.cu, model_interval
                viol = usable & ((c64 < c32 - bd) | (c64 > c32 + bd) | ~(np.abs(s64 - s32) <= err))
                assert not viol.any(), (p.tag, cfg, np.nonzero(viol)[0], r[viol], c64[viol], s64[viol])
                n_checked += int(usable.sum())
                if p.usable_expected:
                    assert usable[p.usable_expected].all(), (p.tag, cfg, np.nonzero(~usable)[0])
                if p.tag == "nan coordinate":  # no claim, except 0 +- 0 for a NaN model (exact: fp64 rejects everything too)
                    nan_model = np.array([np.isnan(np.asarray(M, dtype=float)).any() for M in p.models])
                    assert not usable[~nan_model].any(), (p.tag, cfg)
                if p.gt_index is not None and c64[p.gt_index] > 0:
                    assert bd[p.gt_index] <= 0.05 * c64[p.gt_index] + 5, (p.tag, cfg, r[p.gt_index], c64[p.gt_index])
                # invariance: count32 / border of every launch; score32 / err of every launch of one CTA width
                if first is None:
                    first = {}
                    ref = r
                assert np.array_equal(r["c32"], ref["c32"]) and np.array_equal(r["border"], ref["border"]), (p.tag, cfg)
                w = first.setdefault(cfg[0], r)
                assert np.array_equal(r["s32"].view("<u4"), w["s32"].view("<u4")), (p.tag, cfg)
                assert np.array_equal(r["err"].view("<u4"), w["err"].view("<u4")), (p.tag, cfg)
    assert n_checked > 1000
