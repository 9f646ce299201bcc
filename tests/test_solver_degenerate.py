"""The degree-10 Sturm root finder and the minimal solvers on degenerate inputs: rotation-only, tiny-baseline, distant,
planar, collinear and duplicated-correspondence scenes, and adversarial polynomials.

On such inputs the 5-point solver's determinant polynomial loses its leading coefficient, has near-double roots and
clusters, and the interval walk of sturm_bisect10 emits terminal-width intervals and records up to ten of them.  Those
are the branches of the warp-cooperative sturm_bisect10_warp (k5_roots) and of k5_back's root passes that generic data
never reaches.

CPU part: a plain-Python restatement of sturm_bisect10 (Python floats are IEEE doubles without contraction, so the same
operation order gives the same bits), pinned bit for bit to the oracle, classifies the polynomial set and proves it
covers every branch; the oracle's own high-precision residual bars on the scene set.

GPU part: tests/sturm_warp_device_test.cu runs the warp routine (in a kernel that mirrors k5_roots) and the serial
routine on every polynomial in many placements; the batched solvers run on the degenerate scenes; one 5-point instance is
moved through batches of many sizes; LO-RANSAC runs on rotation-dominant data (k5_back), both precision modes."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import plo_py as P

HERE = os.path.dirname(os.path.abspath(__file__))
FOCAL = 1000.0

# ================================================================================ Sturm restatement (solvers.cuh)
TOL = 1e-10


def _div(a, b):
    """IEEE division (Python raises on a zero divisor)."""
    if b == 0.0:
        if a == 0.0 or a != a:
            return math.nan
        return math.copysign(math.inf, a) * math.copysign(1.0, b)
    return a / b


def _sqrt(x):
    return math.sqrt(x) if x >= 0.0 else math.nan  # (NaN compares false: NaN too)


def _fmax(a, b):
    """C fmax: a NaN operand is ignored."""
    if a != a:
        return b
    if b != b:
        return a
    return a if a >= b else b


def _polyval10(f, x):
    fx = x + f[9]
    for i in range(8, -1, -1):
        fx = x * fx + f[i]
    return fx


def _polyval9(f, x):  # f: the derivative part, fvec + 11
    fx = x + f[11 + 8]
    for i in range(7, -1, -1):
        fx = x * fx + f[11 + i]
    return fx


def _build_seq(fvec):
    N = 10
    f1 = list(fvec[:11])
    f2 = list(fvec[11:21]) + [0.0]
    f3 = [0.0] * 11
    svec = [0.0] * 30
    for I in range(N - 1):
        q1 = f1[N - I] * f2[N - 1 - I]
        q0 = f1[N - 1 - I] * f2[N - 1 - I] - f1[N - I] * f2[N - 2 - I]
        f3[0] = f1[0] - q0 * f2[0]
        for j in range(1, N - 1 - I):
            f3[j] = f1[j] - q1 * f2[j - 1] - q0 * f2[j]
        c = -abs(f3[N - 2 - I])
        ci = _div(1.0, c)
        for j in range(N - 1 - I):
            f3[j] = f3[j] * ci
        svec[3 * I], svec[3 * I + 1], svec[3 * I + 2] = q0, q1, c
        if I + 1 < N - 1:
            f1, f2, f3 = f2, f3, f1
        else:
            svec[27], svec[28], svec[29] = f2[0], f2[1], f3[0]
    return svec


def _signchanges(svec, x):
    f2 = svec[29]
    f1 = svec[27] + x * svec[28]
    count = 1 if (f1 < 0) != (f2 < 0) else 0
    for i in range(8, -1, -1):
        f0 = (svec[3 * i] + x * svec[3 * i + 1]) * f1 + svec[3 * i + 2] * f2
        count += 1 if (f0 < 0) != (f1 < 0) else 0
        f2, f1 = f1, f0
    return count


def _ridders_newton(fvec, a, b):
    """sturm_ridders_newton: the refined root, or None where the end values do not bracket a sign change."""
    fa, fb = _polyval10(fvec, a), _polyval10(fvec, b)
    if not ((fa < 0) ^ (fb < 0)):
        return None
    for _ in range(30):
        if abs(a - b) < 1e-3:
            break
        c = (a + b) * 0.5
        fc = _polyval10(fvec, c)
        s = _sqrt(fc * fc - fa * fb)
        if s == 0.0:  # (!s: NaN goes on)
            break
        d = c + _div((a - c) * fc, s) if fa < fb else c + _div((c - a) * fc, s)
        fd = _polyval10(fvec, d)
        if (fc < 0) if fd >= 0 else (fc > 0):
            a, fa, b, fb = c, fc, d, fd
        elif (fa < 0) if fd >= 0 else (fa > 0):
            b, fb = d, fd
        else:
            a, fa = d, fd
    x = (a + b) * 0.5
    for _ in range(10):
        fx = _polyval10(fvec, x)
        if abs(fx) < TOL:
            break
        fpx = 10.0 * _polyval9(fvec, x)
        dx = _div(fx, fpx)
        x = x - dx
        if abs(dx) < TOL:
            break
    return x


def sturm_walk(c):
    """sturm_bisect10 restated.  Returns (roots, info): info["stop"] is "lead0" (c[10] == 0), "s_lo==s_hi" (no walk) or
    None; info["records"] lists the isolated intervals (a, b, terminal_width) in the order sturm_bisect10_warp records
    them; info["max_depth"] / info["max_sp"] bound the walk."""
    c = [float(v) for v in c]
    N = 10
    info = {"stop": None, "records": [], "max_depth": 0, "max_sp": 0}
    if c[N] == 0.0:
        info["stop"] = "lead0"
        return [], info
    c_inv = _div(1.0, c[N])
    fvec = [c[i] * c_inv for i in range(N)] + [1.0]
    fvec += [fvec[i + 1] * ((i + 1) / float(N)) for i in range(N - 1)] + [1.0]
    svec = _build_seq(fvec)
    mx = 0.0
    for i in range(N):
        mx = _fmax(mx, abs(fvec[i]))
    r0 = 1.0 + mx
    s_lo, s_hi = _signchanges(svec, -r0), _signchanges(svec, r0)
    if s_lo - s_hi == 0:
        info["stop"] = "s_lo==s_hi"
        return [], info
    stack = [(-r0, r0, s_lo, s_hi, 0)]
    rec = info["records"]
    while stack:
        a, b, sa, sb, depth = stack.pop()
        while True:
            info["max_depth"] = max(info["max_depth"], depth)
            if depth > 300:
                break
            if b - a < TOL:
                rec.append((a, b, True))
                break
            n_rts = sa - sb
            if n_rts > 1:
                cm = (a + b) * 0.5
                sc = _signchanges(svec, cm)
                if len(stack) < 12 and ((sc - sb) >= 1 or (b - cm) < TOL):
                    stack.append((cm, b, sc, sb, depth + 1))
                    info["max_sp"] = max(info["max_sp"], len(stack))
                b, sb = cm, sc
                depth += 1
            else:
                if n_rts == 1:
                    rec.append((a, b, False))
                break
    roots = []  # phase C / D: refine every record, keep the first ten results
    for a, b, terminal in rec:
        r = b if terminal else _ridders_newton(fvec, a, b)
        if r is not None and len(roots) < 10:
            roots.append(r)
    return roots, info


def _same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.shape != b.shape:
        return False
    both_nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(both_nan | (a.view(np.int64) == b.view(np.int64))))


# ================================================================================ scenes
KINDS = ("generic", "rotation", "baseline1e-6", "baseline1e-9", "planar", "forward", "far", "collinear", "duplicate")
EXACT_WELL_CONDITIONED = ("generic",)  # (forward motion puts the epipole inside the image: up to 7e-4 off)


def _rotation(rng, max_angle=0.6):
    w = rng.normal(size=3)
    w *= rng.uniform(0.05, max_angle) / np.linalg.norm(w)
    th = np.linalg.norm(w)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / th
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def _unit(X):
    return X / np.linalg.norm(X, axis=1, keepdims=True)


def scene_points(kind, rng, n):
    """3D points in camera 1 and the motion (R, t) of camera 2 (X2 = R X1 + t) of one scene of `kind`."""
    R = _rotation(rng)
    t = rng.normal(size=3)
    t /= np.linalg.norm(t)
    if kind == "rotation":
        t = np.zeros(3)
    elif kind == "baseline1e-6":
        t *= 1e-6
    elif kind == "baseline1e-9":
        t *= 1e-9
    elif kind == "forward":
        t = np.array([0.0, 0.0, 1.0]) * rng.choice([-1.0, 1.0])
    uv = rng.uniform(-0.5, 0.5, (n, 2))
    ray = np.c_[uv, np.ones(n)]
    if kind == "planar":
        nrm = np.array([0.0, 0.0, 1.0]) + rng.normal(0, 0.3, 3)
        nrm /= np.linalg.norm(nrm)
        X1 = ray * (rng.uniform(2.0, 6.0) / (ray @ nrm))[:, None]
    elif kind == "collinear":
        p0 = np.r_[rng.uniform(-1, 1, 2), rng.uniform(3, 6)]
        d = rng.normal(size=3)
        X1 = p0 + rng.uniform(-1.5, 1.5, n)[:, None] * (d / np.linalg.norm(d))
    else:
        X1 = ray * rng.uniform(1.0, 10.0, n)[:, None]
    if kind == "far":
        X1 = X1 * 1e8
    if kind == "duplicate":
        X1[-1] = X1[0]
    return X1, R, t


def relpose_scene(kind, idx, npts, noise=0.0):
    """Unit bearing pairs of one scene; `noise` perturbs the bearings (radians, roughly) like real matches."""
    rng = np.random.default_rng([5021, KINDS.index(kind), idx, npts, int(noise > 0)])
    X1, R, t = scene_points(kind, rng, npts)
    x1, x2 = _unit(X1), _unit(X1 @ R.T + t)
    if noise:
        x1, x2 = _unit(x1 + rng.normal(0, noise, x1.shape)), _unit(x2 + rng.normal(0, noise, x2.shape))
        if kind == "duplicate":
            x1[-1], x2[-1] = x1[0], x2[0]
    return x1, x2, R, t


def relpose_set(npts, exact=40, noisy=12):
    out = []
    for kind in KINDS:
        for i in range(exact):
            x1, x2, R, t = relpose_scene(kind, i, npts)
            out.append((kind, x1, x2, R, t))
        for i in range(noisy):
            x1, x2, R, t = relpose_scene(kind, i, npts, noise=1e-3)
            out.append(("noisy-" + kind, x1, x2, R, t))
    return out


PNP_KINDS = ("generic", "collinear-world", "duplicate", "image-collinear", "cheirality-flip", "far")


def pnp_scene(kind, idx):
    """Bearings x (3) and world points X (3) of one P3P instance, with the ground-truth pose (X_cam = R X + t)."""
    rng = np.random.default_rng([5022, PNP_KINDS.index(kind), idx])
    R = _rotation(rng, 1.5)
    t = rng.normal(size=3)
    ray = np.c_[rng.uniform(-0.5, 0.5, (3, 2)), np.ones(3)]
    Xc = ray * rng.uniform(1.0, 10.0, 3)[:, None]
    if kind == "collinear-world":
        p0, d = Xc[0], Xc[1] - Xc[0]
        Xc[2] = p0 + rng.uniform(0.3, 2.0) * d
    elif kind == "duplicate":
        Xc[2] = Xc[0]
    elif kind == "image-collinear":  # the three points on a plane through the camera centre: their images on a line
        Xc[2] = rng.uniform(0.3, 0.7) * Xc[0] + rng.uniform(0.3, 0.7) * Xc[1]
    elif kind == "far":
        Xc = Xc * 1e6
    x = _unit(Xc)
    if kind == "cheirality-flip":
        x[1] = -x[1]
    X = (Xc - t) @ R  # R^T (Xc - t)
    return x, X, R, t


HOMOG_KINDS = ("generic", "rotation", "collinear", "duplicate", "cheirality-flip", "far-plane")


def homography_scene(kind, idx):
    rng = np.random.default_rng([5023, HOMOG_KINDS.index(kind), idx])
    R = _rotation(rng)
    t = np.zeros(3) if kind == "rotation" else rng.normal(size=3) / 3.0
    nrm = np.array([0.0, 0.0, 1.0]) + rng.normal(0, 0.3, 3)
    nrm /= np.linalg.norm(nrm)
    d = rng.uniform(2.0, 6.0) * (1e7 if kind == "far-plane" else 1.0)
    ray = np.c_[rng.uniform(-0.5, 0.5, (4, 2)), np.ones(4)]
    if kind == "collinear":  # three image points on a line
        ray[2, :2] = ray[0, :2] + rng.uniform(0.3, 0.7) * (ray[1, :2] - ray[0, :2])
    elif kind == "duplicate":
        ray[3] = ray[0]
    X1 = ray * (d / (ray @ nrm))[:, None]
    X2 = X1 @ R.T + t
    x1, x2 = _unit(X1), _unit(X2)
    if kind == "cheirality-flip":
        x2[2] = -x2[2]
    H = R + np.outer(t, nrm) / d
    return x1, x2, H


# ================================================================================ polynomial set
def _from_roots(real, complex_pairs, lead):
    """ascending coefficients of lead * prod (x - r) prod ((x - re)^2 + im^2)."""
    p = np.poly1d([lead])
    for r in real:
        p = p * np.poly1d([1.0, -r])
    for re, im in complex_pairs:
        p = p * np.poly1d([1.0, -2.0 * re, re * re + im * im])
    c = np.zeros(11)
    co = p.coeffs[::-1]
    c[:len(co)] = co
    return c


def _scene_polys(kind, count):
    out = []
    for i in range(count):
        x1, x2, _, _ = relpose_scene(kind, 1000 + i, 5)
        out.append(P.relpose_5pt_stages(x1, x2)[2])
    return out


def polynomial_set():
    """(families, polys): the adversarial families and the determinant polynomials of degenerate 5-point scenes."""
    rng = np.random.default_rng(5024)
    fam = {}
    fam["ten separated roots"] = [_from_roots(np.sort(rng.uniform(-5, 5, 10)), [], rng.uniform(0.1, 100))
                                  for _ in range(64)]
    for sep in (1e-3, 1e-6, 1e-9, 1e-11, 0.0):
        polys = []
        for _ in range(24):
            r = rng.uniform(-3, 3)
            others = rng.uniform(-5, 5, 2 * int(rng.integers(0, 5)))
            pairs = [(rng.uniform(-2, 2), rng.uniform(0.1, 2)) for _ in range((8 - len(others)) // 2)]
            polys.append(_from_roots(np.r_[r, r + sep, others], pairs, rng.uniform(0.5, 5)))
        fam["pair at %g" % sep] = polys
    fam["cluster of ten within 1e-12"] = [_from_roots(r + 1e-13 * np.arange(10), [], rng.uniform(0.5, 5))
                                          for r in rng.uniform(-3, 3, 16)]
    fam["no real roots"] = [_from_roots([], [(rng.uniform(-3, 3), rng.uniform(0.05, 3)) for _ in range(5)],
                                        rng.choice([-1.0, 1.0]) * rng.uniform(0.1, 10)) for _ in range(32)]
    fam["roots of size 1e7..1e9"] = [_from_roots(np.r_[10 ** rng.uniform(7, 9, 4) * rng.choice([-1, 1], 4),
                                                       rng.uniform(-2, 2, 2)],
                                                 [(rng.uniform(-1, 1), rng.uniform(0.1, 1)) for _ in range(2)],
                                                 rng.uniform(0.5, 2)) for _ in range(32)]
    lead0 = [_from_roots(np.sort(rng.uniform(-5, 5, 9)), [], 1.0) for _ in range(8)]
    for c in lead0:
        c[10] = 0.0
    fam["leading coefficient 0"] = lead0
    fam["pure rotation scenes"] = _scene_polys("rotation", 400)
    fam["baseline 1e-9 scenes"] = _scene_polys("baseline1e-9", 400)
    fam["far point scenes"] = _scene_polys("far", 400)
    return fam


# Coefficients the device must survive as neighbours: they stop at s_lo == s_hi (or c[10] == 0) before any walk.
def nonfinite_polys():
    base = _from_roots(np.linspace(-2, 2, 10), [], 1.0)
    out = []
    c = base.copy(); c[10] = 5e-324; out.append(c)            # 1 / c[10] = inf
    c = base.copy(); c[10] = 1e-300; c[3] = 1e300; out.append(c)
    c = base.copy(); c[0] = 1e300; c[10] = 1e-300; out.append(c)
    c = base.copy(); c[4] = np.nan; out.append(c)
    c = base.copy(); c[10] = np.nan; out.append(c)
    c = base.copy(); c[2] = np.inf; out.append(c)
    c = base.copy(); c[7] = -np.inf; out.append(c)
    c = base.copy(); c[10] = np.inf; out.append(c)
    out.append(np.full(11, np.nan))
    return out


@pytest.fixture(scope="module")
def polys():
    fam = polynomial_set()
    flat, names = [], []
    for name, ps in fam.items():
        flat += ps
        names += [name] * len(ps)
    return fam, np.array(flat), names


@pytest.fixture(scope="module")
def walks(polys):
    return [sturm_walk(c) for c in polys[1]]


# ================================================================================ CPU
def test_restatement_reproduces_the_oracle_bit_for_bit(polys, walks):
    _, flat, _ = polys
    for i, (c, (roots, _)) in enumerate(zip(flat, walks)):
        ref = P.bisect_sturm10(c)
        assert _same_bits(roots, ref), (i, roots, ref)
    for c in nonfinite_polys():
        assert _same_bits(sturm_walk(c)[0], P.bisect_sturm10(c)), c


def test_polynomial_set_reaches_every_branch(polys, walks):
    """Per-branch counts over the set (printed with -s).  A warp is 32 consecutive polynomials of the set."""
    fam, flat, names = polys
    infos = [w[1] for w in walks]
    lead0 = sum(i["stop"] == "lead0" for i in infos)
    flat_count = sum(i["stop"] == "s_lo==s_hi" for i in infos)
    terminal = sum(any(r[2] for r in i["records"]) for i in infos)
    ten = sum(len(i["records"]) == 10 for i in infos)
    nb = np.array([len(i["records"]) for i in infos])
    warps = nb[:len(nb) // 32 * 32].reshape(-1, 32).sum(axis=1)
    print("\npolynomials %d: leading 0 %d, s_lo == s_hi %d, terminal-width record %d, ten records %d, "
          "warps > 32 records %d, > 64 records %d, max records %d, max depth %d, max stack %d"
          % (len(flat), lead0, flat_count, terminal, ten, (warps > 32).sum(), (warps > 64).sum(), nb.max(),
             max(i["max_depth"] for i in infos), max(i["max_sp"] for i in infos)))
    for name in fam:
        sel = [k for k, n in enumerate(names) if n == name]
        print("  %-28s %4d: leading 0 %3d, s_lo==s_hi %3d, terminal %3d, ten %3d" % (
            name, len(sel), sum(infos[k]["stop"] == "lead0" for k in sel),
            sum(infos[k]["stop"] == "s_lo==s_hi" for k in sel),
            sum(any(r[2] for r in infos[k]["records"]) for k in sel),
            sum(len(infos[k]["records"]) == 10 for k in sel)))
    assert lead0 and flat_count and terminal and ten
    assert (warps > 32).any() and (warps > 64).any()
    # the degenerate scenes reach the degenerate branches on their own, not only the synthetic families
    scene = [k for k, n in enumerate(names) if n.endswith("scenes")]
    assert any(infos[k]["stop"] == "lead0" for k in scene)
    assert any(infos[k]["stop"] == "s_lo==s_hi" for k in scene)
    # every loop of the walk stays inside its bounds; more than ten records (the RT_MAXB = 16 overflow fallback of
    # sturm_bisect10_warp) was never reached with finite coefficients and looks unreachable: a polynomial of degree 10
    # has at most ten isolated intervals, and at most one terminal-width one sits in the stack at a time
    assert max(i["max_depth"] for i in infos) <= 301 and max(i["max_sp"] for i in infos) <= 12
    assert nb.max() <= 10


def test_nonfinite_coefficients_stop_before_the_walk():
    for c in nonfinite_polys():
        roots, info = sturm_walk(c)
        assert info["stop"] in ("s_lo==s_hi", "lead0") and roots == [] and not info["records"], c


# ---- high-precision residuals (mpmath, 50 digits) of solver outputs --------------------------------------------------
def _mp():
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.dps = 50
    return mpmath


def _mpm(M):
    mpmath = _mp()
    return [[mpmath.mpf(float(v)) for v in row] for row in np.asarray(M, dtype=np.float64)]


def _mmul(A, B):
    return [[sum(A[i][k] * B[k][j] for k in range(3)) for j in range(3)] for i in range(3)]


def _mdet(A):
    return (A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0])
            + A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]))


def _fro(A):
    mpmath = _mp()
    return mpmath.sqrt(sum(v * v for row in A for v in row))


def _epipolar(M, x1, x2):
    """max |x2^T M x1| / |M| over the sample."""
    m = _mpm(M)
    nm = _fro(m)
    worst = 0
    for a, b in zip(_mpm(x1), _mpm(x2)):
        v = sum(b[i] * m[i][j] * a[j] for i in range(3) for j in range(3))
        worst = max(worst, abs(v) / nm)
    return float(worst)


def essential_residuals(E, x1, x2):
    """(epipolar, |det E| / |E|^3, |2 E E^T E - tr(E E^T) E| / |E|^3) at 50 digits."""
    m = _mpm(E)
    nm = _fro(m)
    if nm == 0:  # rotation-only samples can give E = 0 (a root where the whole nullspace combination vanishes)
        return 0.0, 0.0, 0.0
    mt =[[m[j][i] for j in range(3)] for i in range(3)]
    eet = _mmul(m, mt)
    tr = eet[0][0] + eet[1][1] + eet[2][2]
    c = _mmul(eet, m)
    cub = [[2 * c[i][j] - tr * m[i][j] for j in range(3)] for i in range(3)]
    return _epipolar(E, x1, x2), float(abs(_mdet(m)) / nm ** 3), float(_fro(cub) / nm ** 3)


def fundamental_residuals(F, x1, x2):
    m = _mpm(F)
    return _epipolar(F, x1, x2), float(abs(_mdet(m)) / _fro(m) ** 3)


def homography_residual(H, x1, x2):
    """max |x2 x (H x1)| / |H x1| (sine of the transfer angle) over the sample."""
    mpmath = _mp()
    m = _mpm(H)
    worst = 0
    for a, b in zip(_mpm(x1), _mpm(x2)):
        y = [sum(m[i][j] * a[j] for j in range(3)) for i in range(3)]
        cr = [b[1] * y[2] - b[2] * y[1], b[2] * y[0] - b[0] * y[2], b[0] * y[1] - b[1] * y[0]]
        worst = max(worst, mpmath.sqrt(sum(v * v for v in cr)) / mpmath.sqrt(sum(v * v for v in y)))
    return float(worst)


def pose_residual(pose, x, X):
    """max |x x (R X + t)| / |R X + t| over the sample, R from the unit quaternion pose[:4] = (w, x, y, z)."""
    mpmath = _mp()
    w, qx, qy, qz = [mpmath.mpf(float(v)) for v in pose[:4]]
    R = [[1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * w), 2 * (qx * qz + qy * w)],
         [2 * (qx * qy + qz * w), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * w)],
         [2 * (qx * qz - qy * w), 2 * (qy * qz + qx * w), 1 - 2 * (qx * qx + qy * qy)]]
    t = [mpmath.mpf(float(v)) for v in pose[4:7]]
    worst = 0
    for a, P_ in zip(_mpm(x), _mpm(X)):
        y = [sum(R[i][j] * P_[j] for j in range(3)) + t[i] for i in range(3)]
        cr = [a[1] * y[2] - a[2] * y[1], a[2] * y[0] - a[0] * y[2], a[0] * y[1] - a[1] * y[0]]
        worst = max(worst, mpmath.sqrt(sum(v * v for v in cr)) / mpmath.sqrt(sum(v * v for v in y)))
    return float(worst)


# Bars: the oracle's worst residual at 50 digits over the first MP_PER_KIND instances of each kind, times 1.5, rounded
# up to a power of ten (floor 1e-15).  They are the oracle's, not targets: on rotation-only, 1e-9-baseline and distant
# scenes the 5-point problem has no well-defined essential matrix, and the roots of the near-degenerate determinant
# polynomial give matrices far from the essential manifold.  The device must meet the same bar on the same instances.
# 5-point: (epipolar, |det E| / |E|^3, |2 E E^T E - tr(E E^T) E| / |E|^3)
BARS_5PT = {
    "generic": (1e-15, 1e-05, 1e-05), "rotation": (1e-15, 0.01, 0.1), "baseline1e-6": (1e-15, 1e-05, 1e-04),
    "baseline1e-9": (1e-15, 1.0, 1.0), "planar": (1e-15, 1e-06, 1e-05), "forward": (1e-15, 1e-06, 1e-04),
    "far": (1e-15, 0.01, 0.1), "collinear": (1e-15, 1e-08, 1e-07), "duplicate": (1e-15, 1e-10, 1e-09),
    "noisy-generic": (1e-15, 1e-09, 1e-08), "noisy-rotation": (1e-15, 1e-08, 1e-07),
    "noisy-baseline1e-6": (1e-15, 1e-05, 1e-05), "noisy-baseline1e-9": (1e-15, 1e-05, 1e-04),
    "noisy-planar": (1e-15, 1e-07, 1e-05), "noisy-forward": (1e-15, 1e-08, 1e-07), "noisy-far": (1e-15, 1e-09, 1e-09),
    "noisy-collinear": (1e-15, 1e-10, 1e-09), "noisy-duplicate": (1e-15, 1e-09, 1e-08),
}
BAR_7PT = (1e-15, 1e-15)  # (epipolar, |det F| / |F|^3): every kind
# homography: max sine of the transfer angle.  Three collinear image points leave H undetermined (the oracle's H
# transfers the fourth point 38 degrees off); duplicated points and flipped cheirality give no H.
BARS_H = {"generic": 1e-14, "rotation": 1e-14, "far-plane": 1e-15, "collinear": 1.0}
# P3P / Lambda Twist: max sine of the reprojection angle.  Collinear world points leave the pose undetermined (no bar).
BARS_P3P = {"generic": 1e-14, "cheirality-flip": 1e-14, "far": 1e-14, "duplicate": 1e-15, "image-collinear": 1e-10}
BARS_LT = {"generic": 1e-13, "cheirality-flip": 1e-13, "far": 1e-14, "duplicate": 1e-15, "image-collinear": 1e-8}
MP_PER_KIND = 6


def _mp_subset(items):
    seen, out = {}, []
    for k, it in enumerate(items):
        seen[it[0]] = seen.get(it[0], 0) + 1
        if seen[it[0]] <= MP_PER_KIND:
            out.append(k)
    return out


def check_5pt_bars(kind, Es, x1, x2):
    # (on rotation-only, tiny-baseline and distant samples some roots give a NaN matrix, on both sides: no residual)
    for E in Es:
        if not np.isfinite(E).all():
            continue
        r = essential_residuals(E, x1, x2)
        assert all(v <= b for v, b in zip(r, BARS_5PT[kind])), (kind, r)


def check_7pt_bars(kind, Fs, x1, x2):
    for F in Fs:
        r = fundamental_residuals(F, x1, x2)
        assert all(v <= b for v, b in zip(r, BAR_7PT)), (kind, r)


def check_h_bar(kind, H, x1, x2):
    assert homography_residual(H, x1, x2) <= BARS_H[kind], kind


def check_pose_bars(bars, kind, poses, x, X):
    if kind in bars:
        for pose in poses:
            assert pose_residual(pose, x, X) <= bars[kind], (kind, pose)


def test_oracle_meets_the_high_precision_bars():
    rel5, rel7 = relpose_set(5), relpose_set(7)
    for k in _mp_subset(rel5):
        kind, x1, x2, _, _ = rel5[k]
        check_5pt_bars(kind, P.relpose_5pt_E(x1, x2), x1, x2)
    for k in _mp_subset(rel7):
        kind, x1, x2, _, _ = rel7[k]
        check_7pt_bars(kind, P.relpose_7pt(x1, x2), x1, x2)
    for kind in HOMOG_KINDS:
        for i in range(MP_PER_KIND):
            x1, x2, _ = homography_scene(kind, i)
            n, H = P.homography_4pt(x1, x2)
            if kind != "collinear":  # (collinear: the degeneracy test decides either way)
                assert n == (kind not in ("duplicate", "cheirality-flip")), (kind, i)
            if n:
                check_h_bar(kind, H, x1, x2)
    for kind in PNP_KINDS:
        for i in range(MP_PER_KIND):
            x, X, _, _ = pnp_scene(kind, i)
            check_pose_bars(BARS_P3P, kind, P.p3p(x, X), x, X)
            check_pose_bars(BARS_LT, kind, P.p3p_lambdatwist(x, X), x, X)


def _E_from(R, t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ R


def recovers(Es, E_gt, tol=1e-6):
    """some returned E equals the ground truth up to scale and sign."""
    g = E_gt / np.linalg.norm(E_gt)
    return any(min(np.abs(E / np.linalg.norm(E) - g).max(), np.abs(E / np.linalg.norm(E) + g).max()) < tol for E in Es)


def test_oracle_recovers_the_ground_truth_on_well_conditioned_scenes():
    for kind, x1, x2, R, t in relpose_set(5, noisy=0):
        if kind in EXACT_WELL_CONDITIONED:
            assert recovers(P.relpose_5pt_E(x1, x2), _E_from(R, t)), kind


# ================================================================================ GPU: Sturm, every placement
@pytest.fixture(scope="module")
def cabi():
    from poselib_b200 import cabi as c
    if c.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    c.set_device(0)
    return c


def _hex(v):
    return float(v).hex()


def _run_sturm_harness(exe, lists):
    """lists: [array [n, 11]] -> per list, [(warp_roots, serial_roots)] per polynomial."""
    text = "\n".join("%d\n" % len(L) + "\n".join(" ".join(_hex(v) for v in c) for c in L) for L in lists)
    out = subprocess.run([exe], input=text, capture_output=True, text=True, check=True).stdout.split("\n")
    res, k = [], 0
    for L in lists:
        assert out[k] == "L %d" % len(L), out[k]
        k += 1
        rows = []
        for _ in range(len(L)):
            w, s = out[k].split(), out[k + 1].split()
            assert w[0] == "w" and s[0] == "s"
            rows.append(([float.fromhex(v) for v in w[2:]], [float.fromhex(v) for v in s[2:]]))
            assert len(rows[-1][0]) == int(w[1]) and len(rows[-1][1]) == int(s[1])
            k += 2
        res.append(rows)
    return res


@pytest.mark.gpu
@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
def test_warp_root_finder_matches_the_oracle_in_every_placement(polys, walks, tmp_path):
    """sturm_bisect10_warp and sturm_bisect10 on the device against the oracle (pinned to the reference's sturm.h), bit
    for bit in count and roots, wherever the polynomial sits: lane 0 and lane 31 of a warp next to lanes with a zero
    leading coefficient, no real roots, ten roots, a cluster or non-finite coefficients; the last, partial warp (lists
    of 32k + 1 and 64k - 1); the whole set in order, reversed and shuffled."""
    exe = str(tmp_path / "sturm_warp_device_test")
    subprocess.check_call(["nvcc", "-std=c++17", "-O2", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-Xcompiler", "-ffp-contract=off", "-o", exe, os.path.join(HERE, "sturm_warp_device_test.cu")])
    fam, flat, _ = polys
    refs = [P.bisect_sturm10(c) for c in flat]
    rng = np.random.default_rng(5025)
    neighbours = [np.array(fam["leading coefficient 0"]), np.array(fam["no real roots"]),
                  np.array(fam["ten separated roots"]), np.array(fam["cluster of ten within 1e-12"]),
                  np.array(nonfinite_polys())]
    lists, index = [], []  # index[l][lane] = position in `flat`, or -1 for a neighbour
    n = len(flat)
    for order in (np.arange(n), np.arange(n)[::-1], rng.permutation(n)):
        lists.append(flat[order])
        index.append(order)
    for k, m in ((5, 1), (3, -1), (0, 1), (1, -1)):  # 32k + 1 and 64k - 1 polynomials: a partial last warp
        L = 32 * k + 1 if m == 1 else 64 * k + m
        sel = rng.choice(n, L, replace=False)
        lists.append(flat[sel])
        index.append(sel)
    # lane 0 / lane 31 next to 30 neighbours of one kind, every polynomial in both places
    order = rng.permutation(n)
    for lane in (0, 31):
        rows, idx = [], []
        for j, p in enumerate(order):
            nb = neighbours[j % len(neighbours)]
            pick = nb[rng.integers(0, len(nb), 31)]
            warp = np.insert(pick, lane if lane == 0 else 31, flat[p], axis=0)
            rows.append(warp)
            idx += [-1] * lane + [p] + [-1] * (31 - lane)
        lists.append(np.concatenate(rows))
        index.append(np.array(idx))
    res = _run_sturm_harness(exe, lists)
    checked = 0
    for L, idx, rows in zip(lists, index, res):
        for lane_pos, (p, (w, s)) in enumerate(zip(idx, rows)):
            if p < 0:  # a neighbour: the warp and the serial routine still agree with each other and the oracle
                ref = P.bisect_sturm10(L[lane_pos])
            else:
                ref = refs[p]
                checked += 1
            assert _same_bits(w, ref), (p, lane_pos, w, ref)
            assert _same_bits(s, ref), (p, lane_pos, s, ref)
    print("\npolynomial placements checked:", checked)


# ================================================================================ GPU: minimal solvers
def _pose_close(a, b, tol):
    """poses equal to tol, the quaternion up to sign."""
    return min(np.abs(a - b).max(), np.abs(np.r_[-a[:4], a[4:]] - b).max()) <= tol


@pytest.mark.gpu
def test_5pt_on_degenerate_scenes_is_bit_identical_to_the_oracle(cabi):
    """relpose_5pt (k5_load -> k5_null -> k5_elim -> k5_roots -> k5_solver_out): counts exact (0 where the leading
    coefficient vanishes), essential matrices bit for bit, poses to 1e-9; the mpmath bars; the ground truth recovered on
    the well-conditioned scenes."""
    items = relpose_set(5)
    x1s, x2s = np.array([it[1] for it in items]), np.array([it[2] for it in items])
    Es, n = cabi.relpose_5pt_batch(x1s, x2s)
    poses, npz = cabi.relpose_5pt_poses_batch(x1s, x2s)
    counts = []
    for i, (kind, x1, x2, R, t) in enumerate(items):
        ref = P.relpose_5pt_E(x1, x2)
        counts.append(len(ref))
        assert n[i] == len(ref), (kind, i, n[i], len(ref))
        assert _same_bits(Es[i, :n[i]], ref), (kind, i)
        refp = P.relpose_5pt(x1, x2)
        assert npz[i] == len(refp), (kind, i)
        assert np.allclose(poses[i, :npz[i]], refp, rtol=1e-9, atol=1e-9, equal_nan=True), (kind, i)
        if kind in EXACT_WELL_CONDITIONED:
            assert recovers(Es[i, :n[i]], _E_from(R, t)), (kind, i)
    for i in _mp_subset(items):
        check_5pt_bars(items[i][0], Es[i, :n[i]], items[i][1], items[i][2])
    counts = np.array(counts)
    warps = counts[:len(counts) // 32 * 32].reshape(-1, 32).sum(axis=1)
    print("\n5pt: %d instances, %d with 0 solutions, %d with >= 8, warps with > 32 roots: %d"
          % (len(items), (counts == 0).sum(), (counts >= 8).sum(), (warps > 32).sum()))


@pytest.mark.gpu
def test_7pt_and_8pt_on_degenerate_scenes_match_the_oracle(cabi):
    """relpose_7pt: counts exact, F to the 1e-8 / 1e-9 bar of the generic tests, det F and epipolar residuals at 50
    digits within the oracle's bars; essential_matrix_8pt / relpose_8pt (8 and 20 points) to the 1e-9 / 1e-8 bars."""
    items = relpose_set(7)
    x1s, x2s = np.array([it[1] for it in items]), np.array([it[2] for it in items])
    Fs, n = cabi.relpose_7pt_batch(x1s, x2s)
    for i, (kind, x1, x2, _, _) in enumerate(items):
        ref = P.relpose_7pt(x1, x2)
        assert n[i] == len(ref), (kind, i, n[i], len(ref))
        assert np.allclose(Fs[i, :n[i]], ref, rtol=1e-8, atol=1e-9, equal_nan=True), (kind, i)
    for i in _mp_subset(items):
        check_7pt_bars(items[i][0], Fs[i, :n[i]], items[i][1], items[i][2])
    bad = []
    for npts in (8, 20):
        items = relpose_set(npts, exact=12, noisy=4)
        x1s, x2s = np.array([it[1] for it in items]), np.array([it[2] for it in items])
        E = cabi.essential_matrix_8pt_batch(x1s, x2s)
        poses, npose = cabi.relpose_8pt_batch(x1s, x2s)
        for i, (kind, x1, x2, _, _) in enumerate(items):
            Eo = P.essential_matrix_8pt(x1, x2)
            s = np.sign(np.sum(E[i] * Eo)) or 1.0
            if not np.allclose(s * E[i], Eo, rtol=0, atol=1e-9 * max(1.0, np.abs(Eo).max())):
                bad.append(("E", npts, kind, i, np.abs(s * E[i] - Eo).max()))
                continue
            po = P.relpose_8pt(x1, x2)
            if npose[i] != len(po) or not all(_pose_close(poses[i, k], po[k], 1e-8) for k in range(len(po))):
                bad.append(("poses", npts, kind, i, npose[i], len(po)))
    assert not bad, bad


def _diff(a, b):
    """max |a - b|, NaN where both are NaN ignored; inf where only one is NaN."""
    if not np.array_equal(np.isnan(a), np.isnan(b)):
        return np.inf
    return np.nanmax(np.abs(a - b), initial=0.0)


def _perturbed(solve, x, X, ref, trials=32):
    """the oracle's solver when every input coordinate moves by at most one ulp: the solution counts it returns, and
    the largest change of its poses where the count stays."""
    rng = np.random.default_rng(5029)
    counts, worst = {len(ref)}, 0.0
    for _ in range(trials):
        xp = x + rng.choice([-1, 0, 1], x.shape) * np.spacing(x)
        Xp = X + rng.choice([-1, 0, 1], X.shape) * np.spacing(X)
        r = solve(xp, Xp)
        counts.add(len(r))
        if len(r) == len(ref):
            worst = max(worst, np.nan_to_num(_diff(r, ref), posinf=0.0))
    return counts, worst


def _within_rounding(solve, x, X, ref, mine):
    """Two P3P configurations are determined only up to rounding.  Three collinear world points fix the pose only up
    to a rotation about their line: the P3P polynomial is then ill-conditioned, and on the oracle alone a 1-ulp change
    of the input moves the poses by up to 1e10 and changes their number (1, 2 or 4 on one instance).  World points
    1e6 away give a translation t = X_cam - R X that cancels terms of size 1e6, whose ulp is 1.2e-10: its last digits
    are rounding, above the absolute 1e-9 bar.  A device result differs from the oracle's by rounding when the
    oracle, on 1-ulp perturbations of its own input, returns the device's count and moves at least a tenth as far."""
    counts, moved = _perturbed(solve, x, X, ref)
    if len(mine) not in counts:
        return False
    return len(mine) != len(ref) or _diff(mine, ref) <= 10 * moved


@pytest.mark.gpu
def test_p3p_and_homography_on_degenerate_configurations_match_the_oracle(cabi):
    """p3p (1e-9), p3p_lambdatwist (1e-9, the count may differ on < 1 % where a threshold sits within rounding) and
    homography_4pt (bit for bit, both cheirality settings) on collinear, duplicated, image-collinear, cheirality-flipped
    and distant configurations; counts exact; residuals at 50 digits within the oracle's bars.  Collinear and distant
    world points: within rounding as _within_rounding defines it."""
    inst = [(k, *pnp_scene(k, i)) for k in PNP_KINDS for i in range(40)]
    xs, Xs = np.array([it[1] for it in inst]), np.array([it[2] for it in inst])
    poses, n = cabi.p3p_batch(xs, Xs)
    lposes, ln = cabi.p3p_lambdatwist_batch(xs, Xs)
    lt_count_diff = ill = 0
    for i, (kind, x, X, _, _) in enumerate(inst):
        ref, lref = P.p3p(x, X), P.p3p_lambdatwist(x, X)
        mine, lmine = poses[i, :n[i]], lposes[i, :ln[i]]
        if kind in ("collinear-world", "far"):
            for solve, a, b in ((P.p3p, mine, ref), (P.p3p_lambdatwist, lmine, lref)):
                if len(a) != len(b) or _diff(a, b) > 1e-9 * max(1.0, np.nanmax(np.abs(b), initial=0.0)):
                    ill += 1
                    assert _within_rounding(solve, x, X, b, a), (kind, i, solve.__name__)
            if i % 40 < MP_PER_KIND:
                check_pose_bars(BARS_P3P, kind, mine, x, X)
                check_pose_bars(BARS_LT, kind, lmine, x, X)
            continue
        assert n[i] == len(ref), (kind, i, n[i], len(ref))
        assert np.allclose(mine, ref, rtol=1e-9, atol=1e-9, equal_nan=True), (kind, i)
        if ln[i] != len(lref):
            lt_count_diff += 1
        else:
            assert _diff(lmine, lref) <= 1e-9 * max(1.0, np.nanmax(np.abs(lref), initial=0.0)), (kind, i)
        if i % 40 < MP_PER_KIND:
            check_pose_bars(BARS_P3P, kind, mine, x, X)
            check_pose_bars(BARS_LT, kind, lmine, x, X)
    print("\ncollinear / distant world points: %d solver outputs differ from the oracle within rounding" % ill)
    assert lt_count_diff <= len(inst) // 100, lt_count_diff
    inst = [(k, *homography_scene(k, i)) for k in HOMOG_KINDS for i in range(40)]
    x1s, x2s = np.array([it[1] for it in inst]), np.array([it[2] for it in inst])
    for cheir in (True, False):
        Hs, n = cabi.homography_4pt_batch(x1s, x2s, check_cheirality=cheir)
        for i, (kind, x1, x2, _) in enumerate(inst):
            nr, ref = P.homography_4pt(x1, x2, check_cheirality=cheir)
            assert n[i] == nr, (kind, i, cheir)
            if nr:
                assert _same_bits(Hs[i], ref), (kind, i, cheir)
                if cheir and i % 40 < MP_PER_KIND:
                    check_h_bar(kind, Hs[i], x1, x2)


@pytest.mark.gpu
def test_5pt_result_does_not_depend_on_batch_position(cabi):
    """One instance at positions 0, 31, 32, 63, 64 and n - 1 of batches of 1 .. 1000 degenerate neighbours (the last
    CTA's idle threads, partial warps, the 64-, 128- and 256-thread CTAs of the phase kernels): identical bits."""
    items = relpose_set(5)
    nref = [len(P.relpose_5pt_E(it[1], it[2])) for it in items]
    targets = [0, int(np.argmax(nref))]  # a generic instance, the instance with the most roots
    pool = [k for k, it in enumerate(items) if it[0] not in ("generic", "noisy-generic")]
    rng = np.random.default_rng(5026)
    for tgt in targets:
        ref = P.relpose_5pt_E(items[tgt][1], items[tgt][2])
        first_pose = None
        for n in (1, 31, 33, 255, 257, 1000):
            fill = rng.choice(pool, n)
            for pos in sorted({p for p in (0, 31, 32, 63, 64, n - 1) if p < n}):
                sel = fill.copy()
                sel[pos] = tgt
                x1s = np.array([items[k][1] for k in sel])
                x2s = np.array([items[k][2] for k in sel])
                Es, cnt = cabi.relpose_5pt_batch(x1s, x2s)
                assert cnt[pos] == len(ref) and _same_bits(Es[pos, :cnt[pos]], ref), (tgt, n, pos)
                poses, npz = cabi.relpose_5pt_poses_batch(x1s, x2s)
                mine = poses[pos, :npz[pos]]
                if first_pose is None:
                    first_pose = mine
                assert _same_bits(mine, first_pose), (tgt, n, pos)


# ================================================================================ GPU: RANSAC on degenerate data (k5_back)
def _same_trajectory(g, o, model_tol=1e-6, relpose=False):
    """the bars of the RANSAC parity tests: iterations, refinements, inlier counts, masks and counters exactly, the
    score to 1e-9, the model to model_tol (F / H up to sign, the relative pose's translation up to scale)."""
    for k in ("iterations", "refinements", "num_inliers"):
        assert g["stats"][k] == o["stats"][k], (k, g["stats"], o["stats"])
    assert np.isclose(g["stats"]["model_score"], o["stats"]["model_score"], rtol=1e-9), (g["stats"], o["stats"])
    assert np.isclose(g["stats"]["inlier_ratio"], o["stats"]["inlier_ratio"], rtol=0, atol=1e-15)
    assert np.array_equal(g["inliers"], o["inliers"]), int((g["inliers"] != o["inliers"]).sum())
    gm, om = np.asarray(g["model"]), np.asarray(o["model"])
    assert np.array_equal(np.isnan(gm), np.isnan(om))
    gm, om = np.nan_to_num(gm), np.nan_to_num(om)
    if gm.ndim == 2:
        err = min(np.abs(gm - om).max(), np.abs(gm + om).max())
    else:
        if relpose:
            gm = np.r_[gm[:4], gm[4:] / max(np.linalg.norm(gm[4:]), 1e-300)]
            om = np.r_[om[:4], om[4:] / max(np.linalg.norm(om[4:]), 1e-300)]
        err = np.abs(gm - om).max()
    assert err <= model_tol * np.abs(om).max(), (err, gm, om)
    for k in ("samples", "hypotheses", "lo_calls"):
        assert g["counters"][k] == o["counters"][k], (k, g["counters"], o["counters"])


def ransac_pair_problem(kind, n, seed, outliers=0.3):
    """calibrated image points (x = X / Z) of two views of a scene of `kind` ("rotation", "baseline1e-6", "far",
    "planar", "duplicate-half"), 0.5 px noise at f = 1000, `outliers` of the second view's points replaced."""
    rng = np.random.default_rng([5027, n, seed, len(kind)])
    base = "generic" if kind == "duplicate-half" else kind
    X1, R, t = scene_points(base, rng, 3 * n)
    X2 = X1 @ R.T + t
    ok = (X2[:, 2] > 0.05 * np.abs(X1[:, 2]).min()) & (np.abs(X2[:, :2] / X2[:, 2:3]) < 0.8).all(axis=1)
    X1, X2 = X1[ok][:n], X2[ok][:n]
    assert len(X1) == n
    u1, u2 = X1[:, :2] / X1[:, 2:3], X2[:, :2] / X2[:, 2:3]
    u1 = u1 + rng.normal(0, 0.5 / FOCAL, u1.shape)
    u2 = u2 + rng.normal(0, 0.5 / FOCAL, u2.shape)
    out = rng.permutation(n)[:int(outliers * n)]
    u2[out] = rng.uniform(-0.5, 0.5, (len(out), 2))
    if kind == "duplicate-half":
        h = n // 2
        u1[h:2 * h], u2[h:2 * h] = u1[:h], u2[:h]
    return u1, u2


def homography_collinear_problem(n, seed, outliers=0.3):
    """a plane seen twice; a third of the image-1 points lie in runs along eight lines."""
    rng = np.random.default_rng([5028, n, seed])
    R = _rotation(rng)
    t = rng.normal(size=3) / 3.0
    nrm = np.array([0.0, 0.0, 1.0]) + rng.normal(0, 0.2, 3)
    nrm /= np.linalg.norm(nrm)
    d = rng.uniform(3.0, 6.0)
    uv = rng.uniform(-0.5, 0.5, (n, 2))
    runs = n // 3
    for j in range(8):
        a, b = rng.uniform(-0.5, 0.5, 2), rng.uniform(-0.5, 0.5, 2)
        sl = slice(j * runs // 8, (j + 1) * runs // 8)
        s = rng.uniform(0, 1, sl.stop - sl.start)
        uv[sl] = a + s[:, None] * (b - a)
    ray = np.c_[uv, np.ones(n)]
    X2 = (ray * (d / (ray @ nrm))[:, None]) @ R.T + t
    u1 = uv + rng.normal(0, 0.5 / FOCAL, uv.shape)
    u2 = X2[:, :2] / X2[:, 2:3] + rng.normal(0, 0.5 / FOCAL, uv.shape)
    out = rng.permutation(n)[:int(outliers * n)]
    u2[out] = rng.uniform(-0.5, 0.5, (len(out), 2))
    return u1, u2


RANSAC_CASES = [("relpose", "rotation", 1000), ("relpose", "rotation", 10000), ("relpose", "baseline1e-6", 3000),
                ("relpose", "far", 2000), ("relpose", "planar", 2000), ("relpose", "duplicate-half", 4000),
                ("fundamental", "rotation", 2000), ("fundamental", "baseline1e-6", 1000), ("fundamental", "far", 2000),
                ("fundamental", "planar", 3000), ("fundamental", "duplicate-half", 2000),
                ("homography", "collinear-runs", 3000), ("homography", "collinear-runs", 10000)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,scene,n", RANSAC_CASES)
def test_ransac_on_degenerate_data_matches_the_oracle_in_both_modes(cabi, kind, scene, n):
    """LO-RANSAC rounds on rotation-dominant, distant, planar and half-duplicated data, where most 5-point samples have
    many roots and k5_back deals out more than 32 roots per warp: the oracle's trajectory, and fast mode equal to
    exact mode bit for bit."""
    if kind == "homography":
        a, b = homography_collinear_problem(n, 0)
        me = 1.0 / FOCAL
    else:
        a, b = ransac_pair_problem(scene, n, 0)
        me = 1.0 / FOCAL
        if kind == "fundamental":  # the uncalibrated-style scaling of the parity tests
            a, b, me = a * 2.0, b * 2.0, 2.0 / FOCAL
    kw = dict(max_iterations=5000, min_iterations=300, seed=7)
    cabi.set_mode("exact")
    e = cabi.ransac(kind, a, b, cabi.RansacOpt(**kw), me)
    cabi.set_mode("fast")
    try:
        f = cabi.ransac(kind, a, b, cabi.RansacOpt(**kw), me)
    finally:
        cabi.set_mode("exact")
    assert f["stats"] == e["stats"], (f["stats"], e["stats"])
    assert np.array_equal(f["inliers"], e["inliers"])
    assert np.array_equal(np.asarray(f["model"]), np.asarray(e["model"]), equal_nan=True)
    assert f["counters"]["hypotheses"] == e["counters"]["hypotheses"]
    o = P.ransac(kind, a, b, P.RansacOpt(**kw), me)
    _same_trajectory(e, o, relpose=(kind == "relpose"))
