"""The integer streaming test of the Sampson kinds (screen_math.cuh: sampson_qscale / sampson_qrow / sampson_qmodel, the
int8 MMA contraction k_screen runs) against the fp32 test it replaces.

It is only a prefilter: it may record more pairs, never fewer.  Every (model, correspondence) pair that the fp32
streaming test |C^| <= K accepts, and so every pair the full prefilter sampson_maybe accepts, must pass |v| <= K_int, on
relpose (C2) and fundamental (C3) data with eight-point hypotheses from random samples, pixel-unit and large-offset
data, degenerate models, models dominated by E_22, and pairs placed on the fp32 test's own threshold.  The recorded
fraction may rise only modestly over the fp32 test's.  sampson_qword (the word a lane builds itself when the problem is
not staged) must be the same bits as the staged row."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from poselib_b200 import problem_generator as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "poselib_b200", "csrc")

HOST_SRC = r"""
#include "screen_math.cuh"
#include <string.h>
using namespace plb::scr;
// One model (row-major fp64) over n correspondences (fp64 SoA x1.x x1.y x2.x x2.y), cmax and the fp32 copy as
// k_transpose makes them.  out[0]: pairs the fp32 streaming test accepts and the integer test rejects; out[1]: the same
// for the full prefilter; out[2]: pairs the fp32 test accepts; out[3]: pairs the integer test accepts; out[4]: words of
// sampson_qword that differ from sampson_qrow; out[5]: off
extern "C" void qcheck(const double *M, const double *pts, int n, double sq_thr, long long *out) {
    float cmax[4] = {0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < 4; ++c)
        for (int k = 0; k < n; ++k) {
            const float v = f_up(fabs(pts[(size_t)c * n + k]));
            if (!(v <= cmax[c])) cmax[c] = v != v ? v : fmaxf(cmax[c], v);
        }
    float ctx[CTX_FLOATS];
    memset(ctx, 0, sizeof(ctx));
    for (int k = 0; k < 9; ++k) ctx[k] = (float)M[k];
    sampson_setup(M, cmax, sq_thr, ctx);
    uint32_t w[4];
    int c, off;
    sampson_qmodel(M, cmax, ctx[S_CK], w, c, off);
    int e[8];
    sampson_qscale(cmax, e);
    float f[8];
    for (int j = 0; j < 8; ++j) f[j] = ldexpf(1.f, 15 - e[j]);
    for (int k = 0; k < 6; ++k) out[k] = 0;
    out[5] = off;
    for (int k = 0; k < n; ++k) {
        const float a0 = (float)pts[k], a1 = (float)pts[(size_t)n + k], b0 = (float)pts[2 * (size_t)n + k],
                    b1 = (float)pts[3 * (size_t)n + k];
        uint32_t row[4];
        sampson_qrow(a0, a1, b0, b1, f, row);
        for (int t = 0; t < 4; ++t) out[4] += sampson_qword(a0, a1, b0, b1, f, t) != row[t];
        const bool mc = sampson_maybe_c(ctx, ctx[S_CK], a0, a1, b0, b1);
        const bool mb = sampson_maybe(ctx, a0, a1, b0, b1);
        const bool qi = sampson_qtest(w, c, off, row);
        out[0] += mc && !qi;
        out[1] += mb && !qi;
        out[2] += mc;
        out[3] += qi;
    }
}
// C^ of sampson_maybe_c and K, for placing pairs on the threshold
extern "C" void c_and_k(const double *M, const double *pts, int n, double sq_thr, double *C_out, double *K_out) {
    float cmax[4] = {0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < 4; ++c)
        for (int k = 0; k < n; ++k) cmax[c] = fmaxf(cmax[c], f_up(fabs(pts[(size_t)c * n + k])));
    float ctx[CTX_FLOATS];
    memset(ctx, 0, sizeof(ctx));
    for (int k = 0; k < 9; ++k) ctx[k] = (float)M[k];
    sampson_setup(M, cmax, sq_thr, ctx);
    *K_out = ctx[S_CK];
    for (int k = 0; k < n; ++k) {
        const float a0 = (float)pts[k], a1 = (float)pts[(size_t)n + k], b0 = (float)pts[2 * (size_t)n + k],
                    b1 = (float)pts[3 * (size_t)n + k];
        const float e0 = fmaf(ctx[0], a0, fmaf(ctx[1], a1, ctx[2]));
        const float e1 = fmaf(ctx[3], a0, fmaf(ctx[4], a1, ctx[5]));
        const float e2 = fmaf(ctx[6], a0, fmaf(ctx[7], a1, ctx[8]));
        C_out[k] = fmaf(b0, e0, fmaf(b1, e1, e2));
    }
}
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("screen_int")
    src, so = d / "screen_int.cc", d / "screen_int.so"
    src.write_text(HOST_SRC)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I", CSRC, str(src),
                           "-o", str(so)])
    L = C.CDLL(str(so))
    L.qcheck.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, C.c_double, C.POINTER(C.c_longlong)]
    L.c_and_k.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, C.c_double, C.POINTER(C.c_double),
                          C.POINTER(C.c_double)]
    return L


def dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def soa(x1, x2):
    return np.ascontiguousarray(np.r_[x1[:, 0], x1[:, 1], x2[:, 0], x2[:, 1]], dtype=np.float64)


def check(lib, M, pts, sq_thr):
    M = np.ascontiguousarray(np.asarray(M, dtype=np.float64).reshape(9))
    out = np.zeros(6, dtype=np.int64)
    lib.qcheck(dp(M), dp(pts), pts.size // 4, sq_thr, out.ctypes.data_as(C.POINTER(C.c_longlong)))
    assert out[0] == 0 and out[1] == 0, ("pairs the fp32 test records and the integer test loses", out, M)
    assert out[4] == 0, "sampson_qword differs from sampson_qrow"
    return out


def skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def eight_point(x1, x2):
    """the fundamental / essential matrix of 8 correspondences (rank 2, unit Frobenius norm)"""
    A = np.c_[x2[:, :1] * x1, x2[:, :1], x2[:, 1:] * x1, x2[:, 1:], x1, np.ones(len(x1))]
    F = np.linalg.svd(A)[2][-1].reshape(3, 3)
    U, S, Vt = np.linalg.svd(F)
    F = U @ np.diag([S[0], S[1], 0.0]) @ Vt
    return F / np.linalg.norm(F)


def hypotheses(x1, x2, gt, count, rng):
    out = [gt / np.linalg.norm(gt)]
    for s in (1e-4, 1e-3, 1e-2):
        M = gt + rng.normal(0, s * np.abs(gt).max(), (3, 3))
        out.append(M / np.linalg.norm(M))
    while len(out) < count:
        idx = rng.choice(len(x1), 8, replace=False)
        out.append(eight_point(x1[idx], x2[idx]))
    return out


def c2_c3(which, idx):
    p = G.config_c2(idx) if which == "C2" else G.config_c3(idx)
    if which == "C2":  # relpose: calibrated coordinates, 1 px at focal 1000
        x1, x2 = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
        gt = skew(p["t_gt"]) @ p["R_gt"]
        return x1, x2, gt, (1.0 / G.FOCAL) ** 2
    K = np.diag([G.FOCAL, G.FOCAL, 1.0])
    Ki = np.linalg.inv(K)
    gt = Ki.T @ skew(p["t_gt"]) @ p["R_gt"] @ Ki  # fundamental in pixels
    return p["x1"], p["x2"], gt, 1.0


@pytest.mark.parametrize("which", ["C2", "C3"])
def test_integer_test_keeps_every_pair_on_c2_c3(lib, which):
    rng = np.random.default_rng(7)
    acc_f = acc_q = pairs = 0
    for idx in range(2):
        x1, x2, gt, sq = c2_c3(which, idx)
        pts = soa(x1, x2)
        for M in hypotheses(x1, x2, gt, 60, rng):
            out = check(lib, M, pts, sq)
            acc_f += int(out[2])
            acc_q += int(out[3])
            pairs += len(x1)
    frac_f, frac_q = acc_f / pairs, acc_q / pairs
    print(f"{which}: fp32 test records {100 * frac_f:.3f} % of the pairs, the integer test {100 * frac_q:.3f} %")
    assert acc_f > 0
    assert frac_q <= 1.6 * frac_f + 1e-3  # a modest rise: the quantisation is far below the threshold


@pytest.mark.parametrize("units", ["pixels", "offset", "normalised"])
def test_integer_test_keeps_every_pair_on_scaled_data(lib, units):
    rng = np.random.default_rng(11)
    p = G.relpose_problem(3000, 0.5, 72, 1)
    x1, x2 = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
    E = skew(p["t_gt"]) @ p["R_gt"]
    sq = (1.0 / G.FOCAL) ** 2
    if units == "pixels":
        K = np.diag([G.FOCAL, G.FOCAL, 1.0])
        Ki = np.linalg.inv(K)
        E = Ki.T @ E @ Ki
        x1, x2, sq = x1 * G.FOCAL, x2 * G.FOCAL, 1.0
    elif units == "offset":  # coordinates far from the origin: x + o, F = T2^-T E T1^-1
        o = np.array([1e3, -5e2])
        T = np.array([[1, 0, o[0]], [0, 1, o[1]], [0, 0, 1.0]])
        Ti = np.linalg.inv(T)
        E = Ti.T @ E @ Ti
        x1, x2 = x1 + o, x2 + o
    pts = soa(x1, x2)
    for M in hypotheses(x1, x2, E, 40, rng):
        check(lib, M, pts, sq)


def test_integer_test_on_degenerate_models(lib):
    """zero, NaN, E_22-dominated, one-entry, tiny and huge models; the NaN model records nothing (the fp32 test rejects
    every pair), the zero model everything (C = 0 everywhere)"""
    rng = np.random.default_rng(3)
    x1, x2, gt, sq = c2_c3("C2", 0)
    x1, x2 = x1[:3000], x2[:3000]
    pts = soa(x1, x2)
    gt = gt / np.linalg.norm(gt)
    models = [np.zeros((3, 3)), np.where(np.arange(9).reshape(3, 3) == 4, np.nan, gt), gt * 1e-30, gt * 1e30]
    for big in (1e2, 1e4, 1e8):
        M = gt.copy()
        M[2, 2] += big  # E_22 dominates the normalisation
        models.append(M)
    for j in range(9):
        M = np.zeros(9)
        M[j] = 1.0
        models.append(M.reshape(3, 3))
        M = gt.reshape(9).copy()
        M[j] = 0.0
        models.append(M.reshape(3, 3))
    for _ in range(20):
        models.append(rng.normal(size=(3, 3)) * 10.0 ** rng.uniform(-6, 6))
    offs = []
    for M in models:
        offs.append(int(check(lib, M, pts, sq)[5]))
    assert offs[0] == 1 << 26 and offs[1] == -(1 << 26)
    assert sum(o == (1 << 26) for o in offs) < len(offs) // 2  # most models get a real threshold


@pytest.mark.parametrize("eps", [1e-2, 1e-4, 1e-6, 0.0])
def test_integer_test_on_the_fp32_threshold(lib, eps):
    """pairs moved along the epipolar line's normal until C^ sits on +-K (1 - eps): the fp32 test accepts them all, so
    the integer test must too"""
    rng = np.random.default_rng(int(eps * 1e7) + 5)
    x1, x2, gt, sq = c2_c3("C2", 1)
    x1, x2 = x1[:2000].copy(), x2[:2000].copy()
    on = 0
    for M in hypotheses(x1, x2, gt, 12, rng):
        Mf = np.ascontiguousarray(M.reshape(9), dtype=np.float64)
        l = np.c_[x1, np.ones(len(x1))] @ M.T  # E x1: C = x2h . l
        y = x2.copy()
        Cs = np.zeros(len(x1))
        Kv = C.c_double()
        for _ in range(3):
            pts = soa(x1, y)
            lib.c_and_k(dp(Mf), dp(pts), len(x1), sq, dp(Cs), C.byref(Kv))
            K = Kv.value
            if not np.isfinite(K):
                break
            target = rng.choice([-1.0, 1.0], len(x1)) * K * (1 - eps * rng.uniform(0, 1, len(x1)))
            nrm2 = l[:, 0] ** 2 + l[:, 1] ** 2
            y = y + ((target - Cs) / nrm2)[:, None] * l[:, :2]
        pts = soa(x1, y)
        on += int(check(lib, M, pts, sq)[2])
    assert on > 4 * len(x1)  # not vacuous: many pairs sit inside the fp32 threshold
