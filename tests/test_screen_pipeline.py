"""The pipelined fp32 screening pass (k_screen_ctx + k_screen, fast mode).

GPU: fast mode reproduces exact mode bit for bit (stats, model bits, inlier masks) at sizes around the streaming step
of both CTA widths (128 threads up to 2048 correspondences, 512 above), on the shared-memory path and on the
global-memory path (relpose at 12 800 and 20 000 correspondences does not fit the shared-memory stage once padded), and
for a batch of problems of several sizes, so that one CTA restages its arrays across problems.

Host: the NaN padding of the staged arrays is never recorded by the streaming test of any kind, whatever the model
constants, while models with infinite constants still pass every finite correspondence on (and so become candidates
through the non-finite bounds, as before)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from poselib_b200 import problem_generator as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "poselib_b200", "csrc", "screen_math.cuh")

SIZES = [1, 31, 2047, 2048, 2049, 10000, 12800, 20000]


@pytest.fixture(scope="module")
def cabi():
    from poselib_b200 import cabi as c
    if c.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    c.set_device(0)
    return c


def _problem(kind, n, idx):
    """(a, b, max_error); n correspondences are drawn from a larger problem so that tiny n are valid too."""
    m = max(n, 64)
    if kind == "pnp":
        p = G.abspose_problem(m, 0.4, 61, idx)
        a, b, me = p["x"] / G.FOCAL, p["X"], 12.0 / G.FOCAL
    elif kind == "homography":
        p = G.homography_problem(m, 0.5, 64, idx)
        a, b, me = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL, 1.0 / G.FOCAL
    else:
        p = G.relpose_problem(m, 0.3, 62 if kind == "relpose" else 63, idx)
        a, b, me = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL, 1.0 / G.FOCAL
    return np.ascontiguousarray(a[:n]), np.ascontiguousarray(b[:n]), me


def _both_modes(cabi, problems):
    out = {}
    for mode in ("exact", "fast"):
        cabi.set_mode(mode)
        try:
            out[mode] = cabi.Batch(problems).run(streams=2).results()
        finally:
            cabi.set_mode("fast")
    return out["fast"], out["exact"]


def _assert_same(fast, exact):
    assert len(fast) == len(exact)
    for i, (f, e) in enumerate(zip(fast, exact)):
        assert f["stats"] == e["stats"], (i, f["stats"], e["stats"])
        assert np.array_equal(np.asarray(f["model"]), np.asarray(e["model"])), i
        assert np.array_equal(f["inliers"], e["inliers"]), i


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", ["relpose", "fundamental", "homography", "pnp"])
def test_fast_mode_equals_exact_mode(cabi, kind, n):
    a, b, me = _problem(kind, n, 0)
    opt = cabi.RansacOpt(max_iterations=1500, min_iterations=200, seed=5)
    fast, exact = _both_modes(cabi, [dict(kind=kind, a=a, b=b, ransac=opt, max_error=me)])
    _assert_same(fast, exact)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["relpose", "pnp"])
def test_fast_mode_equals_exact_mode_mixed_sizes(cabi, kind):
    problems = []
    for i, n in enumerate([40, 700, 2049, 3000, 6000, 9000, 10000, 5]):
        a, b, me = _problem(kind, n, i)
        problems.append(dict(kind=kind, a=a, b=b, ransac=cabi.RansacOpt(max_iterations=2000, min_iterations=300, seed=i),
                             max_error=me))
    fast, exact = _both_modes(cabi, problems)
    _assert_same(fast, exact)


HOST_SRC = r"""
#include "screen_math.cuh"
using namespace plb::scr;
// For a model M (fp64) and coordinate maxima, fills the context as k_screen_ctx does (model part: M rounded to fp32),
// optionally overrides one constant with +inf, and returns bit 0: maybe() on an all-NaN correspondence,
// bit 1: maybe() on the given finite correspondence p.
extern "C" int nan_probe(int kind, const double *M, const float *cmax, double sq_thr, int inf_at, const float *p) {
    float ctx[CTX_FLOATS] = {0};
    const int msz = kind == 0 ? 12 : 9;
    for (int k = 0; k < msz; ++k) ctx[k] = (float)M[k];
    if (kind == 0) transfer_setup<3>(M, cmax + 2, cmax, sq_thr, ctx);
    else if (kind == 3) transfer_setup<2>(M, cmax, cmax + 2, sq_thr, ctx);
    else sampson_setup(M, cmax, sq_thr, ctx);
    if (inf_at >= 0) ctx[inf_at] = INFINITY;
    const float q = NAN;
    auto maybe = [&](const float *x) {
        if (kind == 0) return transfer_maybe<true>(ctx, pnp_terms(ctx, x[0], x[1], x[2], x[3], x[4]));
        if (kind == 3) return transfer_maybe<false>(ctx, homography_terms(ctx, x[0], x[1], x[2], x[3]));
        return sampson_maybe(ctx, x[0], x[1], x[2], x[3]);
    };
    const float nan5[5] = {q, q, q, q, q};
    return (maybe(nan5) ? 1 : 0) | (maybe(p) ? 2 : 0);
}
"""


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    d = tmp_path_factory.mktemp("screen_nan")
    src, lib = d / "nan_probe.cc", d / "nan_probe.so"
    src.write_text(HOST_SRC)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I",
                           os.path.dirname(HDR), str(src), "-o", str(lib)])
    f = C.CDLL(str(lib)).nan_probe
    f.argtypes = [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_float), C.c_double, C.c_int, C.POINTER(C.c_float)]
    f.restype = C.c_int
    return f


# kind id (as in kernels.cuh): 0 pnp, 1 relpose, 2 fundamental, 3 homography; the streaming test's constants per kind
STREAM_CONSTS = {0: [16, 17], 1: [16, 17, 18], 2: [16, 17, 18], 3: [16, 17]}


@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_nan_padding_is_never_recorded(host, kind):
    rng = np.random.default_rng(kind)
    fp = C.POINTER(C.c_float)
    for _ in range(2000):
        M = rng.normal(size=12) * 10.0 ** rng.uniform(-3, 3)
        cmax = np.abs(rng.normal(size=5)).astype(np.float32) * np.float32(10.0 ** rng.uniform(-2, 2))
        p = (rng.uniform(-1, 1, size=5) * cmax).astype(np.float32)
        sq_thr = 10.0 ** rng.uniform(-8, 0)
        Mp = np.ascontiguousarray(M).ctypes.data_as(C.POINTER(C.c_double))
        r = host(kind, Mp, cmax.ctypes.data_as(fp), sq_thr, -1, p.ctypes.data_as(fp))
        assert r & 1 == 0, (kind, M, cmax, sq_thr)
        for at in STREAM_CONSTS[kind]:
            r = host(kind, Mp, cmax.ctypes.data_as(fp), sq_thr, at, p.ctypes.data_as(fp))
            assert r & 1 == 0, (kind, at)
    # a model whose bound is infinite passes a finite correspondence on (the existing path makes it a candidate)
    M = np.ascontiguousarray(rng.normal(size=12))
    cmax = np.ones(5, dtype=np.float32)
    p = np.full(5, 0.5, dtype=np.float32)
    at = 18 if kind in (1, 2) else 17  # beta' (Sampson) / c' (transfer): +inf widens the test to everything finite
    r = host(kind, M.ctypes.data_as(C.POINTER(C.c_double)), cmax.ctypes.data_as(fp), 1e-6, at, p.ctypes.data_as(fp))
    assert r == 2, (kind, r)
