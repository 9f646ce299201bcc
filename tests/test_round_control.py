"""The device control of a round: candidate selection (k_select), the best-minimal pass (k_pass1), the LO launch that
follows them, and the rounds the engine redoes when a buffer of the round overflows.

k_select lists the models whose (count, score) record — exact, or an fp32 record with a rigorous error bracket — could
improve the best-minimal state; k_pass1 replays score_models (ransac_impl.h:113-124) over those candidates with their
exact records, in (sample, model) order.  Together they make the fast mode exact: every model that improves the state
must be a candidate, and k_pass1 must read nothing else.

CPU: the serial rule and the candidate rule restated in Python, on unit cases (ties, +-0, NaN) and on the generator of
the device tests; the oracle facts the end-to-end tests rely on.

GPU (tests/round_control_device_test.cu): the control kernels on synthetic rounds against the restatements, with the
exact records of non-candidates poisoned and every buffer between guards; record capacities below demand; the LO
launch of a flagged round; the solve and scoring kernels with model segments below demand.  End to end through the
C-ABI: a relative-pose problem whose every sample gives more poses than the first round reserves, and a PnP group with
more LO triggers than the first round's job list holds."""
import itertools
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

from poselib_b200 import problem_generator as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests")

SEL_CHUNK = 256 * 4  # SEL_THREADS * SEL_SPT (control.cu): samples per pass of k_select
MSZ = 7              # PnP / relpose model size
GUARD = 64           # SEL_GUARD of the harness
CTL_OVERFLOW, CTL_IMP_TOTAL, CTL_JOB_TOTAL, CTL_FLAGS, CTL_WORDS = 2, 5, 6, 7, 8
FLAG_IMP, FLAG_JOB = 1, 2
GB = 0xA5            # guard byte
MAXM = {0: 4, 1: 40}  # kind_max_models: pnp, relpose

RP = np.dtype([("pidx", "<i4"), ("g0", "<i4"), ("B", "<i4"), ("seg_base", "<i4"), ("seg_cap", "<i4"),
               ("reserved", "<i4"), ("lb0", "<f8"), ("ub0", "<f8")])
HDR = np.dtype([("n_models", "<i4"), ("n_cand", "<i4"), ("n_imp", "<i4"), ("imp_base", "<i4"), ("n_trig", "<i4"),
                ("trig_base", "<i4")])
IMP = np.dtype([("sample", "<i4"), ("count", "<u4"), ("score", "<f8"), ("model", "<f8", 9)])
JOB = np.dtype([("pidx", "<i4"), ("slot", "<i4")])
LMOUT = np.dtype([("model", "<f8", 9), ("score", "<f8"), ("count", "<u4"), ("iterations", "<i4"), ("cost", "<f8"),
                  ("initial_cost", "<f8")])
assert RP.itemsize == 40 and HDR.itemsize == 24 and IMP.itemsize == 88 and LMOUT.itemsize == 104


# ============================================================================================================
# restatements
# ============================================================================================================
def serial_improving(recs, lb0, ub0):
    """score_models (ransac_impl.h:113-124) over one round in (sample, model) order from the state (lb0, ub0).
    recs[s] = list of (count, score).  Returns the improving (sample, model) pairs and, per sample with one, its last
    improving model (the LO trigger, :124,139)."""
    bc, bs = lb0, ub0
    imp = []
    for s, models in enumerate(recs):
        for m, (c, sc) in enumerate(models):
            more, better = c > bc, sc < bs
            if more or better:
                imp.append((s, m))
                if more:
                    bc = c
                if better:
                    bs = sc
    last = {}
    for s, m in imp:
        last[s] = m
    return imp, sorted(last.items())


def interval(rec, mode):
    """control.cu model_interval: (c_lo, c_hi, s_lo, s_hi, usable) of a slot's records"""
    if mode == 0:
        c, s = float(rec["c64"]), float(rec["s64"])
        return c, c, s, s, True
    c, b = float(rec["c32"]), float(rec["border"])
    s, e = float(np.float32(rec["s32"])), float(np.float32(rec["err"]))
    return c - b, c + b, s - e, s + e, bool(np.isfinite(s) and np.isfinite(e))


def candidates(recs, lb0, ub0, mode):
    """k_select's rule: a model is a candidate iff it is unusable or its bracket could exceed the running maximum of the
    lower count bounds / fall below the running minimum of the upper score bounds of every usable model before it (C
    fmax / fmin: NaN operands are ignored).  recs[s] = list of slot records.  Returns (sample, model) pairs."""
    LB, UB = lb0, ub0
    out = []
    for s, models in enumerate(recs):
        for m, r in enumerate(models):
            c_lo, c_hi, s_lo, s_hi, usable = interval(r, mode)
            if (not usable) or c_hi > LB or s_lo < UB:
                out.append((s, m))
            if usable:
                LB = float(np.fmax(LB, c_lo))
                UB = float(np.fmin(UB, s_hi))
    return out


# ============================================================================================================
# synthetic rounds
# ============================================================================================================
REC = np.dtype([("c64", "<u4"), ("s64", "<f8"), ("c32", "<u4"), ("border", "<u4"), ("s32", "<f4"), ("err", "<f4")])


def fp32_records(r, rng, exact_err_share=0.3):
    """fp32 records whose brackets contain the exact ones: |c32 - c64| <= border, |s32 - s64| <= err (as doubles);
    a share of the brackets are tight (err = the rounding of s64 itself, border 0)"""
    n = len(r)
    border = rng.integers(0, 4, n).astype(np.int64)
    tight = rng.random(n) < exact_err_share
    border[tight] = 0
    delta = np.array([rng.integers(-b, b + 1) for b in border])
    c32 = np.maximum(r["c64"].astype(np.int64) + delta, 0)
    s64 = r["s64"]
    with np.errstate(invalid="ignore"):
        s32 = (s64 * (1.0 + rng.normal(0, 1e-6, n) * ~tight)).astype(np.float32)
        dev = np.abs(s32.astype(np.float64) - s64)
        err = (dev * (1.0 + rng.uniform(0, 1, n) * ~tight)).astype(np.float32)
        low = err.astype(np.float64) < dev
    err[low] = np.nextafter(err[low], np.float32(np.inf))
    r["c32"], r["border"], r["s32"], r["err"] = c32, border, s32, err
    nan = np.isnan(s64)
    r["s32"][nan] = np.nan  # no finite bracket holds a NaN score: unusable
    return r


def bracket_ok(r):
    c64, c32, b = r["c64"].astype(np.float64), r["c32"].astype(np.float64), r["border"].astype(np.float64)
    s32, e = r["s32"].astype(np.float64), r["err"].astype(np.float64)
    usable = np.isfinite(s32) & np.isfinite(e)
    with np.errstate(invalid="ignore"):
        return ~usable | ((c64 >= c32 - b) & (c64 <= c32 + b) & (np.abs(r["s64"] - s32) <= e))


class Prob:
    """one problem of a synthetic round: per-sample model counts, slot records in (sample, model) order, start state"""

    def __init__(self, nm, recs, lb0, ub0, tail=0):
        self.nm, self.recs, self.lb0, self.ub0, self.tail = list(nm), recs, float(lb0), float(ub0), tail

    def per_sample(self):
        out, k = [], 0
        for n in self.nm:
            out.append(self.recs[k:k + n])
            k += n
        return out


def random_prob(rng, B, shape="mixed", lb0=0.0, ub0=np.finfo(np.float64).max):
    if shape == "empty_runs":
        nm = np.where((np.arange(B) // 37) % 2 == 0, 0, rng.integers(0, 5, B))
    elif shape == "forty":
        nm = np.where(rng.random(B) < 0.3, 40, rng.integers(0, 3, B))
    else:
        nm = rng.choice([0, 0, 1, 1, 2, 3, 4, 10], B)
        if B > 2:
            nm[rng.integers(B)] = 40
    n = int(nm.sum())
    r = np.zeros(n, REC)
    # counts and scores on coarse grids (ties on both), drifting so that improvements keep coming
    drift = np.linspace(0, 1, max(n, 1))[:n]
    r["c64"] = np.clip(rng.integers(0, 30, n) + (drift * 40).astype(int), 0, None)
    r["s64"] = np.round(rng.uniform(0, 200, n) * (1.2 - drift), 0) / 4
    sp = rng.random(n)
    r["s64"][sp < 0.01] = np.nan
    r["s64"][(sp >= 0.01) & (sp < 0.02)] = 0.0
    r["s64"][(sp >= 0.02) & (sp < 0.03)] = -0.0
    fp32_records(r, rng)
    # non-finite fp32 records: unusable models
    k = rng.random(n)
    r["s32"][k < 0.01] = np.inf
    r["err"][(k >= 0.01) & (k < 0.02)] = np.inf
    r["s32"][(k >= 0.02) & (k < 0.025)] = np.nan
    return Prob(nm, r, lb0, ub0, tail=int(rng.integers(0, 5)))


def straddle_prob():
    """improving models at indices 20..59: one sample's run of 40 crosses the 32-entry chunks of k_pass1"""
    nm = [0, 20, 0, 40, 3]
    n = sum(nm)
    r = np.zeros(n, REC)
    r["c64"] = 5
    r["s64"] = 1000.0 - np.arange(n)  # strictly decreasing: every model improves the score
    r["c32"], r["s32"] = r["c64"], r["s64"].astype(np.float32)
    return Prob(nm, r, 0.0, 2000.0)


def edge_prob():
    """brackets touching the running bounds exactly: c_hi == LB and s_lo == UB are not candidates"""
    nm = [3, 2]
    r = np.zeros(5, REC)
    # lb0 = 10, ub0 = 5: model 0 is c 8 +- 2 (c_hi == LB), s 6 +- 1 (s_lo == UB) -> not a candidate, exact (10, 5.5)
    r[0] = (10, 5.5, 8, 2, 6.0, 1.0)
    r[1] = (10, 5.0, 10, 0, 5.0, 0.0)        # exactly the state: no candidate
    r[2] = (11, 7.0, 9, 2, 7.0, 0.0)         # c_hi 11 > 10: candidate, improves on count
    r[3] = (11, 5.0, 10, 1, 5.25, 0.25)      # c_hi 11 == the new LB (c_lo of r[2] is 7 -> LB stays 10): candidate
    r[4] = (3, 4.0, 3, 0, 4.0, 0.0)          # s_lo 4 < UB 5: candidate, improves on score
    return Prob(nm, r, 10.0, 5.0)


def layout(probs, rng):
    """RoundProb array, per-sample n_models / first_slot, flat slot records and models; a problem's samples own slots
    of its segment in a shuffled order (the order of the solve kernels' atomicAdd) and the segment may have an unused
    tail.  Returns (rp, n_models, first_slot, slots, models, slot_of) with slot_of[a][s] = first slot of sample s."""
    rp = np.zeros(len(probs), RP)
    nmodels, firsts, recs, mods, slot_of = [], [], [], [], []
    g0 = seg = 0
    for a, p in enumerate(probs):
        B = len(p.nm)
        cap = int(sum(p.nm)) + p.tail
        rp[a] = (a, g0, B, seg, cap, 0, p.lb0, p.ub0)
        seg_recs = np.zeros(cap, REC)
        seg_mod = rng.normal(size=(cap, MSZ))
        seg_mod[:, :4] /= np.linalg.norm(seg_mod[:, :4], axis=1, keepdims=True)
        if p.tail:  # unused slots: records that would be candidates and improve everything, if they were read
            seg_recs[-p.tail:] = (4000000000, -1e300, 4000000000, 0, -1e30, 0.0)
        order = rng.permutation(B)
        pos, first, ps = 0, np.zeros(B, np.int64), p.per_sample()
        for s in order:
            first[s] = seg + pos
            seg_recs[pos:pos + p.nm[s]] = ps[s]
            pos += p.nm[s]
        nmodels.append(np.asarray(p.nm, np.int32))
        firsts.append(first.astype(np.int32))
        recs.append(seg_recs)
        mods.append(seg_mod)
        slot_of.append(first)
        g0 += B
        seg += cap
    return (rp, np.concatenate(nmodels), np.concatenate(firsts), np.concatenate(recs), np.concatenate(mods), slot_of)


def expected(probs, mode):
    """per problem: candidates, improving models, triggers (lists of (sample, model))"""
    out = []
    for p in probs:
        ps = p.per_sample()
        cand = candidates(ps, p.lb0, p.ub0, mode)
        exact = [[(int(r["c64"]), float(r["s64"])) for r in rr] for rr in ps]
        imp, trig = serial_improving(exact, p.lb0, p.ub0)
        out.append((cand, imp, trig))
    return out


# ============================================================================================================
# CPU tests
# ============================================================================================================
def test_serial_rule_ties_zero_and_nan():
    # ties on count and on score do not improve; a better score with fewer inliers does
    imp, trig = serial_improving([[(5, 3.0), (5, 3.0), (4, 2.0)], [(6, 2.0), (6, 2.0)]], 0.0, np.finfo(float).max)
    assert imp == [(0, 0), (0, 2), (1, 0)] and trig == [(0, 2), (1, 0)]
    # +-0: -0.0 < 0.0 is false
    imp, _ = serial_improving([[(0, 0.0)], [(0, -0.0)], [(0, -1e-300)]], 0.0, 1.0)
    assert imp == [(0, 0), (2, 0)]
    # a NaN score never compares better and leaves the running minimum alone; its count still counts
    imp, _ = serial_improving([[(3, np.nan), (3, 5.0), (4, np.nan)]], 2.0, 10.0)
    assert imp == [(0, 0), (0, 1), (0, 2)]
    # carried state: nothing at or below it improves
    imp, trig = serial_improving([[(7, 4.0), (6, 3.9)], [(8, 9.0)]], 7.0, 4.0)
    assert imp == [(0, 1), (1, 0)] and trig == [(0, 1), (1, 0)]


def test_candidate_rule_edges():
    p = edge_prob()
    assert bracket_ok(p.recs).all()
    cand = candidates(p.per_sample(), p.lb0, p.ub0, 1)
    assert cand == [(0, 2), (1, 0), (1, 1)]
    exact = [[(int(r["c64"]), float(r["s64"])) for r in rr] for rr in p.per_sample()]
    imp, _ = serial_improving(exact, p.lb0, p.ub0)
    assert imp == [(0, 2), (1, 1)] and set(imp) <= set(cand)
    # mode 0: the records are exact; NaN scores are ignored by fmin, equal records are not candidates
    r = np.zeros(4, REC)
    r["c64"] = [3, 3, 2, 4]
    r["s64"] = [np.nan, 1.0, 1.0, 0.5]
    assert candidates([list(r)], 3.0, 2.0, 0) == [(0, 1), (0, 3)]
    # unusable fp32 records are candidates and do not move the bounds
    r["c32"], r["border"], r["s32"], r["err"] = [9, 0, 0, 0], [0, 0, 0, 0], [np.inf, 9, 9, 9], [0, 0, np.inf, 0]
    assert candidates([list(r)], 3.0, 2.0, 1) == [(0, 0), (0, 2)]


@pytest.mark.parametrize("seed", range(6))
def test_generator_brackets_and_candidates_cover_the_improving_models(seed):
    rng = np.random.default_rng(seed)
    for shape in ("mixed", "empty_runs", "forty"):
        p = random_prob(rng, 300, shape)
        assert bracket_ok(p.recs).all()
        (cand, imp, trig), = expected([p], 1)
        assert set(imp) <= set(cand), shape
        assert len(imp) >= 3 and len(cand) < sum(p.nm)
        (cand0, imp0, _), = expected([p], 0)
        assert imp0 == imp and set(imp) <= set(cand0) <= set(cand)


def tiny_baseline_scene():
    """5 points seen from two cameras 1e-6 apart: every ordering of the 5-point sample gives 10 poses"""
    rng = np.random.default_rng(5467)
    w = rng.normal(0, 0.3, 3)
    th = np.linalg.norm(w)
    k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
    t = rng.normal(0, 1, 3) * 1e-6
    X = np.c_[rng.uniform(-1, 1, (5, 2)), np.ones(5)] * rng.uniform(1, 10, (5, 1))
    Y = X @ R.T + t
    return X[:, :2] / X[:, 2:], Y[:, :2] / Y[:, 2:]


def bearings(x):
    h = np.c_[x, np.ones(len(x))]
    return h / np.linalg.norm(h, axis=1, keepdims=True)


def test_tiny_baseline_scene_overflows_the_first_round_reservation():
    """relpose reserves 8 models per sample in its first round; this scene gives more for every sample"""
    import plo_py as P
    x1, x2 = tiny_baseline_scene()
    b1, b2 = bearings(x1), bearings(x2)
    counts = [len(P.relpose_5pt(b1[list(q)], b2[list(q)])) for q in itertools.permutations(range(5))]
    assert len(counts) == 120 and min(counts) >= 9


def pnp_group():
    return [G.abspose_problem(200, 1.0, config_id=7, problem_idx=i) for i in range(256)]


PNP_KW = dict(max_iterations=32)


def test_pnp_group_has_more_lo_triggers_than_the_first_job_list():
    """256 problems x 32 samples: the first round's job list holds max(1024, 8192 / 8) = 1024 LO jobs"""
    import plo_py as P
    total = 0
    for i, p in enumerate(pnp_group()):
        o = P.ransac("pnp", p["x"] / 1000.0, p["X"], P.RansacOpt(seed=i, **PNP_KW), 0.012)
        total += o["stats"]["refinements"] - 1
    assert total > 1024, total


# ============================================================================================================
# GPU: the harness
# ============================================================================================================
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("round_control") / "round_control_device_test")
    subprocess.check_call(["nvcc", "-std=c++17", "-O3", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-Xcompiler", "-ffp-contract=off", "-o", exe,
                           os.path.join(HERE, "round_control_device_test.cu")])
    return exe


class Reader:
    def __init__(self, buf):
        self.buf, self.off = buf, 0

    def arr(self, dtype, n):
        dt = np.dtype(dtype)
        a = np.frombuffer(self.buf, dt, n, self.off).copy()
        self.off += dt.itemsize * n
        return a

    def guarded(self, dtype, n, g):
        """(interior, guards intact)"""
        dt = np.dtype(dtype)
        raw = np.frombuffer(self.buf, np.uint8, dt.itemsize * (n + 2 * g), self.off)
        self.off += raw.size
        gb = dt.itemsize * g
        ok = bool((raw[:gb] == GB).all() and (raw[raw.size - gb:] == GB).all())
        return raw[gb:raw.size - gb].copy().view(dt), ok


def run_select(harness, tmp_path, cases):
    """cases: list of dict(probs, mode, imp_cap, job_cap, lm)"""
    rng = np.random.default_rng(99)
    inp, outp = tmp_path / "sel_in.bin", tmp_path / "sel_out.bin"
    lay = []
    with open(inp, "wb") as f:
        f.write(struct.pack("<i", len(cases)))
        for c in cases:
            L = layout(c["probs"], rng)
            rp, nm, fs, recs, mods, _ = L
            lay.append(L)
            lm_n = 64 if c.get("lm") else 0
            f.write(struct.pack("<8i", c["mode"], c["imp_cap"], c["job_cap"], len(rp), len(nm), len(recs), lm_n,
                                int(len(recs) // 2)))
            f.write(rp.tobytes())
            f.write(nm.astype("<i4").tobytes())
            f.write(fs.astype("<i4").tobytes())
            for fld, dt in (("c64", "<u4"), ("s64", "<f8"), ("c32", "<u4"), ("border", "<u4"), ("s32", "<f4"),
                            ("err", "<f4")):
                f.write(np.ascontiguousarray(recs[fld]).astype(dt).tobytes())
            f.write(mods.astype("<f8").tobytes())
            if lm_n:
                p = G.abspose_problem(lm_n, 1.0, 7, 0)
                f.write((p["x"] / 1000.0).astype("<f8").tobytes())
                f.write(p["X"].astype("<f8").tobytes())
    subprocess.check_call([harness, "select", str(inp), str(outp)])
    R = Reader(open(outp, "rb").read())
    res = []
    for c, (rp, nm, fs, recs, mods, slot_of) in zip(cases, lay):
        na, nt, S = len(rp), len(nm), len(recs)
        d = {}
        guards = []
        for name, dt, n in (("prefix", "<i4", nt), ("cslot", "<i4", S), ("csmp", "<i4", S), ("n_cand", "<i4", na),
                            ("n_models_tot", "<i4", na), ("islot", "<i4", S), ("ismp", "<i4", S),
                            ("ctl", "<i4", CTL_WORDS), ("hdr", HDR, na), ("imp", IMP, c["imp_cap"]),
                            ("job", JOB, c["job_cap"])):
            d[name], ok = R.guarded(dt, n, GUARD)
            guards.append((name, ok))
        if c.get("lm"):
            d["lmout"], ok = R.guarded(LMOUT, c["job_cap"], GUARD)
            guards.append(("lmout", ok))
        d["guards"] = guards
        res.append((d, (rp, nm, fs, recs, mods, slot_of)))
    assert R.off == len(R.buf)
    return res


def check_select(c, d, lay):
    """the harness's dumps against the restatements"""
    rp, nm, fs, recs, mods, slot_of = lay
    probs, mode = c["probs"], c["mode"]
    bad = [n for n, ok in d["guards"] if not ok]
    assert not bad, ("stores outside a buffer", bad)
    exp = expected(probs, mode)
    hdr = d["hdr"]
    tot_imp = sum(len(e[1]) for e in exp)
    tot_trig = sum(len(e[2]) for e in exp)
    assert d["ctl"][CTL_IMP_TOTAL] == tot_imp and d["ctl"][CTL_JOB_TOTAL] == tot_trig
    flags = (FLAG_IMP if tot_imp > c["imp_cap"] else 0) | (FLAG_JOB if tot_trig > c["job_cap"] else 0)
    assert d["ctl"][CTL_FLAGS] == flags, (d["ctl"], tot_imp, tot_trig, c["imp_cap"], c["job_cap"])
    imp_written = np.zeros(c["imp_cap"], bool)
    job_written = np.zeros(c["job_cap"], bool)
    ranges_imp, ranges_trig = [], []
    for a, (p, (cand, imp, trig)) in enumerate(zip(probs, exp)):
        g0, B, seg = int(rp[a]["g0"]), int(rp[a]["B"]), int(rp[a]["seg_base"])
        first = slot_of[a]
        assert np.array_equal(d["prefix"][g0:g0 + B], np.cumsum(p.nm)), a
        assert d["n_models_tot"][a] == sum(p.nm) and d["n_cand"][a] == len(cand), (a, d["n_cand"][a], len(cand))
        got = list(zip(d["csmp"][seg:seg + len(cand)], d["cslot"][seg:seg + len(cand)]))
        assert got == [(s, first[s] + m) for s, m in cand], a
        if mode == 1:
            assert set(imp) <= set(cand), a
        h = hdr[a]
        assert (h["n_models"], h["n_cand"], h["n_imp"], h["n_trig"]) == (sum(p.nm), len(cand), len(imp), len(trig)), a
        if len(imp):
            ranges_imp.append((int(h["imp_base"]), len(imp)))
        if len(trig):
            ranges_trig.append((int(h["trig_base"]), len(trig)))
        fits = h["imp_base"] + len(imp) <= c["imp_cap"] and h["trig_base"] + len(trig) <= c["job_cap"]
        if not fits:
            continue
        # in-place compaction: the improving list at the head of the candidate segment
        assert list(zip(d["ismp"][seg:seg + len(imp)], d["islot"][seg:seg + len(imp)])) == \
            [(s, first[s] + m) for s, m in imp], a
        ps = p.per_sample()
        for i, (s, m) in enumerate(imp):
            r = d["imp"][h["imp_base"] + i]
            slot = first[s] + m
            ex = ps[s][m]
            assert r["sample"] == s and r["count"] == ex["c64"], (a, i, r, ex)
            assert r["score"].tobytes() == np.float64(ex["s64"]).tobytes(), (a, i, r["score"], ex["s64"])
            assert np.array_equal(r["model"][:MSZ].view("<u8"), mods[slot].view("<u8")), (a, i)
            imp_written[h["imp_base"] + i] = True
        for i, (s, m) in enumerate(trig):
            j = d["job"][h["trig_base"] + i]
            assert (j["pidx"], j["slot"]) == (a, first[s] + m), (a, i, j)
            job_written[h["trig_base"] + i] = True
    # the atomicAdd bases tile the totals, in whatever order the problems took them
    for ranges, tot in ((ranges_imp, tot_imp), (ranges_trig, tot_trig)):
        pos = 0
        for base, n in sorted(ranges):
            assert base == pos, (ranges, tot)
            pos += n
        assert pos == tot
    # nothing written but the records of the problems that fit
    imp_raw = d["imp"].view(np.uint8).reshape(len(d["imp"]), -1)
    assert (imp_raw[~imp_written] == GB).all()
    if not c.get("lm"):
        job_raw = d["job"].view(np.uint8).reshape(len(d["job"]), -1)
        assert (job_raw[~job_written] == GB).all()
    return job_written


def mixed_problems(rng, sizes, shape="mixed"):
    out = []
    for i, B in enumerate(sizes):
        lb0 = float(rng.integers(0, 20)) if i % 3 == 1 else 0.0
        ub0 = float(rng.uniform(20, 60)) if i % 3 == 1 else np.finfo(np.float64).max
        out.append(random_prob(rng, B, shape if i % 2 == 0 else "mixed", lb0, ub0))
    return out


def ample_caps(probs):
    """record capacities that always fit: one improving model per slot, one LO job per sample"""
    return dict(imp_cap=sum(sum(p.nm) + p.tail for p in probs), job_cap=sum(len(p.nm) for p in probs))


def select_cases():
    rng = np.random.default_rng(2024)
    sets = {
        "chunk edges": [1, 31, 32, 33, 1023, 1024, 1025, 4097],
        "empty runs": [1, 64, 500, 33],
        "forty": [3, 31, 100, 1025],
        "edges": None,
    }
    cases = []
    for mode in (0, 1):
        for name, sizes in sets.items():
            if sizes is None:
                probs = [edge_prob(), straddle_prob(), straddle_prob(), edge_prob()]
            else:
                shape = {"empty runs": "empty_runs", "forty": "forty"}.get(name, "mixed")
                probs = mixed_problems(rng, sizes, shape)
            cases.append(dict(name=f"{name} mode {mode}", probs=probs, mode=mode, **ample_caps(probs)))
        # ~2000 problems in one launch
        probs = mixed_problems(rng, rng.integers(1, 40, 2000))
        cases.append(dict(name=f"many problems mode {mode}", probs=probs, mode=mode, **ample_caps(probs)))
    return cases


def cap_cases():
    """record capacities below demand: imp only, job only, both (and one that fits exactly)"""
    rng = np.random.default_rng(7)
    probs = mixed_problems(rng, [50] * 60 + [1025, 300])
    exp = expected(probs, 1)
    ti, tt = sum(len(e[1]) for e in exp), sum(len(e[2]) for e in exp)
    assert tt > 100
    out = []
    for name, ic, jc in (("imp", ti // 2, tt + 5), ("job", ti + 5, tt // 2), ("both", ti // 3, tt // 3),
                         ("exact", ti, tt)):
        out.append(dict(name=f"caps {name}", probs=probs, mode=1, imp_cap=ic, job_cap=jc))
    return out


@pytest.mark.gpu
def test_select_and_pass1_match_the_serial_rule(harness, tmp_path):
    cases = select_cases()
    res = run_select(harness, tmp_path, cases)
    n_imp = 0
    for c, (d, lay) in zip(cases, res):
        try:
            check_select(c, d, lay)
        except AssertionError as e:
            raise AssertionError(f"{c['name']}: {e}") from e
        n_imp += int(d["hdr"]["n_imp"].sum())
    assert n_imp > 10000


@pytest.mark.gpu
def test_record_caps_below_demand(harness, tmp_path):
    cases = cap_cases()
    res = run_select(harness, tmp_path, cases)
    for c, (d, lay) in zip(cases, res):
        try:
            check_select(c, d, lay)
        except AssertionError as e:
            raise AssertionError(f"{c['name']}: {e}") from e
    assert [int(d["ctl"][CTL_FLAGS]) for d, _ in res] == [FLAG_IMP, FLAG_JOB, FLAG_IMP | FLAG_JOB, 0]


@pytest.mark.gpu
def test_lo_launch_reads_only_jobs_of_this_round(harness, tmp_path):
    """job_src is pre-filled with a valid job (a dummy template that runs no iteration on a real slot): the LO launch
    after k_pass1 may produce an output only for an entry k_pass1 wrote in this round — none at all when the round is
    flagged, since the host redoes it."""
    cases = [dict(c, lm=True) for c in cap_cases()]
    res = run_select(harness, tmp_path, cases)
    for c, (d, lay) in zip(cases, res):
        written = check_select(c, d, lay)
        raw = d["lmout"].view(np.uint8).reshape(len(d["lmout"]), -1)
        produced = ~(raw == GB).all(axis=1)
        flagged = d["ctl"][CTL_FLAGS] != 0
        assert not (produced & ~written).any(), (c["name"], np.nonzero(produced & ~written)[0][:10])
        if flagged:
            assert not produced.any(), c["name"]
        else:
            assert np.array_equal(produced, written) and written.sum() == d["ctl"][CTL_JOB_TOTAL], c["name"]


# ---- segment overflow in the solve and scoring kernels ----------------------------------------------------------------
def hyp_problems(kind):
    """(n, sq_thr, a, b, samples) per problem: real PnP or relpose data with seeded samples"""
    rng = np.random.default_rng(kind)
    out = []
    if kind == 0:
        for i, B in enumerate((40, 300, 7, 129)):
            p = G.abspose_problem(150 + 50 * i, 0.7, 7, i)
            n = len(p["x"])
            smp = np.array([rng.choice(n, 3, replace=False) for _ in range(B)], dtype=np.uint32)
            out.append((p["x"] / 1000.0, p["X"], (12.0 / 1000) ** 2, smp))
    else:
        x1, x2 = tiny_baseline_scene()
        for i, B in enumerate((50, 20, 64)):
            if i == 1:
                p = G.relpose_problem(300, 0.8, 2, i)
                a, b = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
                smp = np.array([rng.choice(len(a), 5, replace=False) for _ in range(B)], dtype=np.uint32)
            else:
                a, b = x1, x2
                smp = np.array([rng.permutation(5) for _ in range(B)], dtype=np.uint32)
            out.append((a, b, (1.0 / G.FOCAL) ** 2, smp))
    return out


def run_hyp(harness, tmp_path, kind, mode, caps_list):
    probs = hyp_problems(kind)
    msz = MSZ
    inp, outp = tmp_path / "hyp_in.bin", tmp_path / "hyp_out.bin"
    with open(inp, "wb") as f:
        f.write(struct.pack("<5i", 1, kind, mode, len(probs), len(caps_list)))
        for a, b, sq, smp in probs:
            f.write(struct.pack("<id", len(a), sq))
            f.write(np.ascontiguousarray(a, "<f8").tobytes())
            f.write(np.ascontiguousarray(b, "<f8").tobytes())
            f.write(struct.pack("<i", len(smp)))
            f.write(np.ascontiguousarray(smp, "<u4").tobytes())
        for caps in caps_list:
            f.write(np.asarray(caps, "<i4").tobytes())
    subprocess.check_call([harness, "hyp", str(inp), str(outp)])
    buf = open(outp, "rb").read()
    R = Reader(buf)
    na, nt = len(probs), sum(len(p[3]) for p in probs)
    runs = []
    for caps in caps_list:
        r = {"caps": np.asarray(caps)}
        r["overflow"] = int(R.arr("<i4", 1)[0])
        r["seg"], r["pc"] = R.arr("<i4", na), R.arr("<i4", na)
        g, slots = (int(v) for v in R.arr("<i4", 2))
        r["slots"] = slots
        r["nm"], ok1 = R.guarded("<i4", nt, GUARD)
        r["fs"], ok2 = R.guarded("<i4", nt, GUARD)
        r["sample_guards"] = ok1 and ok2
        per = [("counts", "<u4", 1), ("scores", "<f8", 1), ("models", "<f8", msz), ("mp", "<i4", 1)]
        if mode == 1:
            per += [("fcounts", "<u4", 1), ("fscores", "<f4", 1), ("fborder", "<u4", 1), ("ferr", "<f4", 1)]
        for name, dt, k in per:
            raw = np.frombuffer(buf, np.uint8, np.dtype(dt).itemsize * k * (slots + 2 * g), R.off)
            R.off += raw.size
            r[name] = raw.reshape(slots + 2 * g, -1)
        if mode == 1:
            raw = np.frombuffer(buf, np.uint8, 4 * CTX_FLOATS * (slots + 2 * g), R.off)
            R.off += raw.size
            r["fctx"] = raw.reshape(slots + 2 * g, -1)
        r["g"] = g
        runs.append(r)
    assert R.off == len(buf)
    return probs, runs


CTX_FLOATS = 28  # scr::CTX_FLOATS (screen_math.cuh)


def test_ctx_floats_constant():
    src = open(os.path.join(ROOT, "poselib_b200", "csrc", "screen_math.cuh")).read()
    assert f"CTX_FLOATS = {CTX_FLOATS}" in src


def per_sample_models(r, probs, per_fields):
    """per sample: (n_models, the bytes of its models' records)"""
    out = []
    g = r["g"]
    k = 0
    for a, (_, _, _, smp) in enumerate(probs):
        for s in range(len(smp)):
            n, f = int(r["nm"][k]), int(r["fs"][k])
            recs = tuple(r[name][g + f:g + f + n].tobytes() for name in per_fields) if n else ()
            out.append((a, n, recs))
            k += 1
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind,mode", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_overflowing_segments_stay_inside_their_buffers(harness, tmp_path, kind, mode):
    probs = hyp_problems(kind)
    B = [len(p[3]) for p in probs]
    ample = [MAXM[kind] * b for b in B]
    if kind == 0:  # one model per sample reserved: p3p gives up to 4; the third problem keeps ample room
        tight = [b for b in B]
        tight[2] = ample[2]
    else:  # relpose's first-round reservation (8 per sample); the ordinary problem keeps ample room
        tight = [8 * b for b in B]
        tight[1] = ample[1]
    probs, (full, cut) = run_hyp(harness, tmp_path, kind, mode, [ample, tight])
    fields = ["counts", "scores", "models", "mp"] if mode == 0 else \
        ["models", "mp", "fcounts", "fscores", "fborder", "ferr", "fctx"]
    g_off = np.r_[0, np.cumsum(B)]
    demand = full["pc"]
    assert full["overflow"] == 0
    assert [int(full["nm"][g_off[a]:g_off[a + 1]].sum()) for a in range(len(B))] == list(demand)
    over = demand > np.asarray(tight)
    assert over.any() and not over.all()
    assert cut["overflow"] == 1
    for r in (full, cut):
        assert r["sample_guards"]
        g, caps, seg = r["g"], r["caps"], r["seg"]
        inside = np.zeros(r["slots"] + 2 * g, bool)
        for a in range(len(probs)):
            inside[g + seg[a]:g + seg[a] + caps[a]] = True
        for name in fields:
            raw = r[name]
            outside = raw[~inside]
            assert (outside == GB).all(), (name, "stores outside the problems' segments",
                                           np.nonzero(~(raw == GB).all(axis=1) & ~inside)[0][:10] - g)
    A = per_sample_models(full, probs, fields)
    Bc = per_sample_models(cut, probs, fields)
    kept = np.zeros(len(probs), np.int64)
    for (a, n_full, rec_full), (a2, n_cut, rec_cut) in zip(A, Bc):
        assert a == a2
        if not over[a]:
            assert (n_cut, rec_cut) == (n_full, rec_full), a
        else:
            assert n_cut in (0, n_full), (a, n_cut, n_full)  # a dropped sample reports no model
            if n_cut:
                # a kept sample: its models and their records.  score32 / err of k_screen depend on which models
                # share a tile (the queue pass deals a tile's recorded cases out over the lanes), and a segment with
                # dropped samples tiles differently; count32 / border do not
                skip = {"fscores", "ferr"}
                assert [x for x, f in zip(rec_cut, fields) if f not in skip] == \
                    [x for x, f in zip(rec_full, fields) if f not in skip], a
        kept[a] += n_cut
    assert (kept <= np.asarray(tight)).all()
    for a in range(len(probs)):  # kept samples' slots lie inside the segment
        f, n = cut["fs"][g_off[a]:g_off[a + 1]], cut["nm"][g_off[a]:g_off[a + 1]]
        live = n > 0
        assert (f[live] >= cut["seg"][a]).all() and (f[live] + n[live] <= cut["seg"][a] + tight[a]).all(), a


# ============================================================================================================
# GPU: end to end through the C-ABI
# ============================================================================================================
@pytest.fixture(scope="module")
def cabi():
    from poselib_b200 import cabi as c
    if c.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    c.set_device(0)
    return c


def same_result(g, o, model_tol=1e-6, relpose=False):
    from test_gpu_parity import _same_trajectory
    _same_trajectory(g, o, model_tol=model_tol, relpose=relpose)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_relpose_round_redone_after_a_segment_overflow(cabi, mode):
    import plo_py as P
    x1, x2 = tiny_baseline_scene()
    kw = dict(max_iterations=100, seed=3)
    me = 1.0 / G.FOCAL
    others = []
    for i in range(4):
        p = G.relpose_problem(400, 0.6, 2, 10 + i)
        others.append((p["x1"] / G.FOCAL, p["x2"] / G.FOCAL))
    cabi.set_mode(mode)
    try:
        alone = cabi.ransac("relpose", x1, x2, cabi.RansacOpt(**kw), me)
        singles = [cabi.ransac("relpose", a, b, cabi.RansacOpt(**kw), me) for a, b in others]
        items = others[:2] + [(x1, x2)] + others[2:]
        batch = cabi.ransac_batch([dict(kind="relpose", a=a, b=b, ransac=cabi.RansacOpt(**kw), max_error=me)
                                   for a, b in items], streams=1)
    finally:
        cabi.set_mode("exact")
    assert alone["counters"]["rounds"] == 2, alone["counters"]
    o = P.ransac("relpose", x1, x2, P.RansacOpt(**kw), me)
    same_result(alone, o, relpose=True)
    for got, ref in zip(batch, singles[:2] + [alone] + singles[2:]):
        assert got["stats"] == ref["stats"], (got["stats"], ref["stats"])
        assert np.array_equal(got["inliers"], ref["inliers"])
        assert np.array_equal(np.asarray(got["model"]), np.asarray(ref["model"]))


@pytest.mark.gpu
def test_pnp_group_round_redone_after_a_job_list_overflow(cabi):
    import plo_py as P
    probs = pnp_group()
    items = [dict(kind="pnp", a=p["x"] / 1000.0, b=p["X"], ransac=cabi.RansacOpt(seed=i, **PNP_KW), max_error=0.012)
             for i, p in enumerate(probs)]
    batch = cabi.ransac_batch(items, streams=1)
    assert batch[0]["counters"]["rounds"] == 2, batch[0]["counters"]
    for i, (it, got) in enumerate(zip(items, batch)):
        single = cabi.ransac("pnp", it["a"], it["b"], cabi.RansacOpt(seed=i, **PNP_KW), 0.012)
        assert single["counters"]["rounds"] == 1, (i, single["counters"])
        assert got["stats"] == single["stats"], (i, got["stats"], single["stats"])
        assert np.array_equal(got["inliers"], single["inliers"]) and np.array_equal(got["model"], single["model"]), i
        o = P.ransac("pnp", it["a"], it["b"], P.RansacOpt(seed=i, **PNP_KW), 0.012)
        same_result(got, o)
