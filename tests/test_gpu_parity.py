"""GPU parity tests proper (-m gpu): the CUDA path, called through the C-ABI, against the CPU oracle on the
same seeded inputs.  Bars: integer results (sample-driven trajectory: iterations, refinements, inlier counts,
inlier masks) bit-exact; models within 1e-6 relative (north_star), solver outputs within 1e-9."""
import numpy as np
import pytest

import plo_py as P
from poselib_b200 import problem_generator as G

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cabi():
    from poselib_b200 import cabi as c
    if c.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    c.set_device(0)
    return c


def _noisy_samples(npts, count, seed, outliers=True):
    """bearing samples as the estimators build them from noisy/outlier data (not exact minimal instances)."""
    rng = np.random.default_rng(seed)
    x1s, x2s = [], []
    for i in range(count):
        p = G.relpose_problem(64, 0.5 if outliers else 1.0, config_id=20, problem_idx=seed * 1000 + i)
        idx = rng.choice(64, npts, replace=False)
        a = np.c_[p["x1"][idx] / G.FOCAL, np.ones(npts)]
        b = np.c_[p["x2"][idx] / G.FOCAL, np.ones(npts)]
        x1s.append(a / np.linalg.norm(a, axis=1, keepdims=True))
        x2s.append(b / np.linalg.norm(b, axis=1, keepdims=True))
    return np.array(x1s), np.array(x2s)


# ---------------------------------------------------------------------------------------------- solvers
def test_p3p_matches_oracle(cabi):
    xs, Xs = [], []
    for i in range(400):
        x, X, R, t = G.minimal_abspose(i)
        xs.append(x)
        Xs.append(X)
    # plus samples drawn from noisy / outlier data
    for i in range(100):
        p = G.abspose_problem(50, 0.5, config_id=21, problem_idx=i)
        a = np.c_[p["x"][:3] / G.FOCAL, np.ones(3)]
        xs.append(a / np.linalg.norm(a, axis=1, keepdims=True))
        Xs.append(p["X"][:3])
    poses, n = cabi.p3p_batch(np.array(xs), np.array(Xs))
    for i in range(len(xs)):
        ref = P.p3p(xs[i], Xs[i])
        assert n[i] == len(ref), i
        assert np.allclose(poses[i, :n[i]], ref, rtol=1e-9, atol=1e-9, equal_nan=True), i


def test_relpose_5pt_matches_oracle(cabi):
    x1s, x2s = [], []
    for i in range(300):
        x1, x2, R, t = G.minimal_relpose(i, 5)
        x1s.append(x1)
        x2s.append(x2)
    a, b = _noisy_samples(5, 300, 1)
    x1s, x2s = np.concatenate([np.array(x1s), a]), np.concatenate([np.array(x2s), b])
    Es, n = cabi.relpose_5pt_batch(x1s, x2s)
    poses, npz = cabi.relpose_5pt_poses_batch(x1s, x2s)
    exact = 0
    for i in range(len(x1s)):
        ref = P.relpose_5pt_E(x1s[i], x2s[i])
        assert n[i] == len(ref), (i, n[i], len(ref))
        assert np.allclose(Es[i, :n[i]], ref, rtol=1e-9, atol=1e-9, equal_nan=True), i
        exact += np.array_equal(Es[i, :n[i]], ref)
        refp = P.relpose_5pt(x1s[i], x2s[i])
        assert npz[i] == len(refp), i
        assert np.allclose(poses[i, :npz[i]], refp, rtol=1e-9, atol=1e-9, equal_nan=True), i
    print("5pt bit-identical instances:", exact, "/", len(x1s))


def test_relpose_7pt_matches_oracle(cabi):
    x1s, x2s = [], []
    for i in range(300):
        x1, x2, R, t = G.minimal_relpose(i, 7)
        x1s.append(x1)
        x2s.append(x2)
    a, b = _noisy_samples(7, 300, 2)
    x1s, x2s = np.concatenate([np.array(x1s), a]), np.concatenate([np.array(x2s), b])
    Fs, n = cabi.relpose_7pt_batch(x1s, x2s)
    for i in range(len(x1s)):
        ref = P.relpose_7pt(x1s[i], x2s[i])
        assert n[i] == len(ref), i
        assert np.allclose(Fs[i, :n[i]], ref, rtol=1e-8, atol=1e-9, equal_nan=True), i


def test_homography_4pt_matches_oracle(cabi):
    x1s, x2s = [], []
    for i in range(300):
        x1, x2, H = G.minimal_homography(i)
        x1s.append(x1)
        x2s.append(x2)
    a, b = _noisy_samples(4, 300, 3)
    x1s, x2s = np.concatenate([np.array(x1s), a]), np.concatenate([np.array(x2s), b])
    Hs, n = cabi.homography_4pt_batch(x1s, x2s)
    for i in range(len(x1s)):
        nr, ref = P.homography_4pt(x1s[i], x2s[i])
        assert n[i] == nr, i
        if nr:
            assert np.allclose(Hs[i], ref, rtol=1e-10, atol=1e-12, equal_nan=True), i


# ---------------------------------------------------------------------------------------------- RANSAC
def _same_trajectory(g, o, model_tol=1e-6, relpose=False):
    for k in ("iterations", "refinements", "num_inliers"):
        assert g["stats"][k] == o["stats"][k], (k, g["stats"], o["stats"])
    assert np.isclose(g["stats"]["model_score"], o["stats"]["model_score"], rtol=1e-9), (g["stats"], o["stats"])
    assert np.isclose(g["stats"]["inlier_ratio"], o["stats"]["inlier_ratio"], rtol=0, atol=1e-15)
    assert np.array_equal(g["inliers"], o["inliers"]), int((g["inliers"] != o["inliers"]).sum())
    gm, om = np.asarray(g["model"]), np.asarray(o["model"])
    assert np.array_equal(np.isnan(gm), np.isnan(om))
    gm, om = np.nan_to_num(gm), np.nan_to_num(om)  # degenerate inputs give NaN models on both sides
    if gm.ndim == 2:  # F / H are projective entities: defined up to sign (the SVD factorisation of the F refiner
        #               may legitimately return either sign, optim_utils.h:59-73)
        err = min(np.abs(gm - om).max(), np.abs(gm + om).max())
    else:
        if relpose:  # |t| is a gauge freedom of a relative pose (the LM never renormalises it, relative.h:152-157)
            gm = np.r_[gm[:4], gm[4:] / max(np.linalg.norm(gm[4:]), 1e-300)]
            om = np.r_[om[:4], om[4:] / max(np.linalg.norm(om[4:]), 1e-300)]
        err = np.abs(gm - om).max()
    assert err <= model_tol * np.abs(om).max(), (err, gm, om)
    assert g["counters"]["samples"] == o["counters"]["samples"]
    assert g["counters"]["hypotheses"] == o["counters"]["hypotheses"]
    assert g["counters"]["lo_calls"] == o["counters"]["lo_calls"]


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("n,ratio,its", [(200, 0.5, 1000), (1500, 0.35, 3000)])
def test_ransac_pnp_matches_oracle(cabi, n, ratio, its, seed):
    p = G.abspose_problem(n, ratio, 1, seed)
    x = p["x"] / G.FOCAL
    kw = dict(max_iterations=its, min_iterations=min(its, 1000), seed=seed)
    g = cabi.ransac("pnp", x, p["X"], cabi.RansacOpt(**kw), 12.0 / G.FOCAL)
    o = P.ransac("pnp", x, p["X"], P.RansacOpt(**kw), 12.0 / G.FOCAL)
    _same_trajectory(g, o)


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("n,ratio", [(1000, 0.5), (10000, 0.3)])
def test_ransac_relpose_matches_oracle(cabi, n, ratio, seed):
    p = G.relpose_problem(n, ratio, 2, seed)
    x1, x2 = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
    kw = dict(max_iterations=100000, min_iterations=1000, seed=seed)
    g = cabi.ransac("relpose", x1, x2, cabi.RansacOpt(**kw), 1.0 / G.FOCAL)
    o = P.ransac("relpose", x1, x2, P.RansacOpt(**kw), 1.0 / G.FOCAL)
    _same_trajectory(g, o, relpose=True)


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("prosac,rfc", [(False, False), (True, True)])
def test_ransac_fundamental_matches_oracle(cabi, prosac, rfc, seed):
    p = G.relpose_problem(2000, 0.3, 3, seed, prosac_sorted=prosac)
    x1, x2 = p["x1"] / 500.0, p["x2"] / 500.0  # uncalibrated-style scaling, pp at origin for RFC
    kw = dict(max_iterations=20000, min_iterations=1000, seed=seed, progressive_sampling=prosac,
              max_prosac_iterations=5000)
    g = cabi.ransac("fundamental", x1, x2, cabi.RansacOpt(**kw), 1.0 / 500.0, rfc=rfc)
    o = P.ransac("fundamental", x1, x2, P.RansacOpt(**kw), 1.0 / 500.0, rfc=rfc)
    _same_trajectory(g, o)


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("n,ratio", [(2000, 0.6), (20000, 0.6)])
def test_ransac_homography_matches_oracle(cabi, n, ratio, seed):
    p = G.homography_problem(n, ratio, 4, seed)
    x1, x2 = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
    kw = dict(max_iterations=100000, min_iterations=1000, seed=seed)
    g = cabi.ransac("homography", x1, x2, cabi.RansacOpt(**kw), 1.0 / G.FOCAL)
    o = P.ransac("homography", x1, x2, P.RansacOpt(**kw), 1.0 / G.FOCAL)
    _same_trajectory(g, o)


def test_score_initial_model_and_edge_sizes(cabi):
    p = G.relpose_problem(800, 0.5, 2, 11)
    x1, x2 = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
    init = np.r_[p["q_gt"], p["t_gt"]]
    kw = dict(max_iterations=2000, min_iterations=50, seed=5, score_initial_model=True)
    g = cabi.ransac("relpose", x1, x2, cabi.RansacOpt(**kw), 1.0 / G.FOCAL, init=init)
    o = P.ransac("relpose", x1, x2, P.RansacOpt(**kw), 1.0 / G.FOCAL, init=init)
    _same_trajectory(g, o, relpose=True)
    # fewer points than the sample size: default stats, identity model, mask of the identity model
    g = cabi.ransac("relpose", x1[:4], x2[:4], cabi.RansacOpt(), 1.0 / G.FOCAL)
    o = P.ransac("relpose", x1[:4], x2[:4], P.RansacOpt(), 1.0 / G.FOCAL)
    assert g["stats"]["iterations"] == 0 and g["stats"]["model_score"] == o["stats"]["model_score"]
    assert np.array_equal(g["inliers"], o["inliers"]) and np.array_equal(g["model"], o["model"])
    # exactly the sample size; max_iterations smaller than min_iterations
    kw = dict(max_iterations=7, min_iterations=1000, seed=1)
    g = cabi.ransac("relpose", x1[:5], x2[:5], cabi.RansacOpt(**kw), 1.0 / G.FOCAL)
    o = P.ransac("relpose", x1[:5], x2[:5], P.RansacOpt(**kw), 1.0 / G.FOCAL)
    _same_trajectory(g, o, relpose=True)


# ---------------------------------------------------------------------------------------------- estimate_*
def test_estimate_entry_points_match_oracle(cabi):
    cam = cabi.Camera("PINHOLE", (G.FOCAL, G.FOCAL, 0.0, 0.0))
    camt = (G.FOCAL, G.FOCAL, 0.0, 0.0)
    p = G.config_c1(3)
    g = cabi.estimate("pnp", p["x"], p["X"], cabi.RansacOpt(**p["ransac"]), cabi.BundleOpt(), p["max_error"], cam)
    o = P.estimate("pnp", p["x"], p["X"], P.RansacOpt(**p["ransac"]), P.BundleOpt(), p["max_error"], camt)
    _same_trajectory(g, o)
    p = G.relpose_problem(3000, 0.4, 2, 5)
    kw = dict(max_iterations=20000, min_iterations=500, seed=2)
    g = cabi.estimate("relpose", p["x1"], p["x2"], cabi.RansacOpt(**kw), cabi.BundleOpt(), 1.0, cam, cam)
    o = P.estimate("relpose", p["x1"], p["x2"], P.RansacOpt(**kw), P.BundleOpt(), 1.0, camt, camt)
    _same_trajectory(g, o, relpose=True)
    p = G.relpose_problem(2000, 0.4, 3, 6, prosac_sorted=True)
    kw = dict(max_iterations=20000, min_iterations=500, seed=2, progressive_sampling=True)
    g = cabi.estimate("fundamental", p["x1"], p["x2"], cabi.RansacOpt(**kw), cabi.BundleOpt(), 1.0, rfc=True)
    o = P.estimate("fundamental", p["x1"], p["x2"], P.RansacOpt(**kw), P.BundleOpt(), 1.0, rfc=True)
    _same_trajectory(g, o)
    p = G.homography_problem(3000, 0.6, 4, 7)
    kw = dict(max_iterations=20000, min_iterations=500, seed=2)
    g = cabi.estimate("homography", p["x1"], p["x2"], cabi.RansacOpt(**kw), cabi.BundleOpt(), 1.0)
    o = P.estimate("homography", p["x1"], p["x2"], P.RansacOpt(**kw), P.BundleOpt(), 1.0)
    _same_trajectory(g, o)


def test_batch_api_matches_single_calls(cabi):
    probs, singles = [], []
    for i in range(6):
        if i % 2 == 0:
            p = G.abspose_problem(200, 0.5, 5, i)
            a, b, kind, me = p["x"] / G.FOCAL, p["X"], "pnp", 12.0 / G.FOCAL
            kw = dict(max_iterations=1000, min_iterations=1000, seed=i)
        else:
            p = G.relpose_problem(3000, 0.35, 5, i)
            a, b, kind, me = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL, "relpose", 1.0 / G.FOCAL
            kw = dict(max_iterations=50000, min_iterations=1000, seed=i)
        probs.append(dict(kind=kind, a=a, b=b, ransac=cabi.RansacOpt(**kw), max_error=me))
        singles.append(P.ransac(kind, a, b, P.RansacOpt(**kw), me))
    res = cabi.ransac_batch(probs, streams=3)
    for g, o, pr in zip(res, singles, probs):
        assert g["status"] == 0
        _same_trajectory(g, o, relpose=(pr["kind"] == "relpose"))
    # device-resident inputs give the same answers as host inputs
    h = cabi.resident_create("relpose", probs[1]["a"], probs[1]["b"])
    r2 = cabi.ransac_batch([dict(kind="relpose", resident=h, n=len(probs[1]["a"]), ransac=probs[1]["ransac"],
                                 max_error=probs[1]["max_error"])], streams=1)[0]
    cabi.resident_free(h)
    assert r2["stats"] == res[1]["stats"] and np.array_equal(r2["inliers"], res[1]["inliers"])
    assert np.array_equal(r2["model"], res[1]["model"])


# ---------------------------------------------------------------------------------------------- LM refiners
def _perturbed(kind, p, rng):
    if kind == "pnp":
        q = p["q_gt"] + rng.normal(0, 0.01, 4)
        return np.r_[q / np.linalg.norm(q), p["t_gt"] + rng.normal(0, 0.02, 3)]
    if kind == "relpose":
        q = p["q_gt"] + rng.normal(0, 0.01, 4)
        t = p["t_gt"] + rng.normal(0, 0.02, 3)
        return np.r_[q / np.linalg.norm(q), t / np.linalg.norm(t)]
    if kind == "fundamental":
        t = p["t_gt"]
        E = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ p["R_gt"]
        E = E + rng.normal(0, 0.01, (3, 3))
        return E / np.linalg.norm(E)
    H = p["H_gt"] / np.linalg.norm(p["H_gt"])
    return H + rng.normal(0, 0.002, (3, 3))


@pytest.mark.parametrize("loss", ["TRUNCATED", "CAUCHY", "HUBER", "TRIVIAL"])
@pytest.mark.parametrize("kind", ["pnp", "relpose", "fundamental", "homography"])
def test_lm_refiners_match_oracle(cabi, kind, loss):
    rng = np.random.default_rng(7)
    for idx in range(3):
        if kind == "pnp":
            p = G.abspose_problem(500, 0.7, 31, idx)
            a, b = p["x"] / G.FOCAL, p["X"]
            scale = 12.0 / G.FOCAL
        elif kind == "homography":
            p = G.homography_problem(600, 0.7, 34, idx)
            a, b = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
            scale = 2.0 / G.FOCAL
        else:
            p = G.relpose_problem(600, 0.7, 32, idx)
            a, b = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
            scale = 2.0 / G.FOCAL
        m0 = _perturbed(kind, p, rng)
        kw = dict(max_iterations=25, loss_type=loss, loss_scale=scale)
        gm, gs = cabi.refine(kind, m0, a, b, cabi.BundleOpt(**kw))
        om, os_ = P.refine(kind, m0, a, b, P.BundleOpt(**kw))
        # os_ = [iterations, initial_cost, cost, ...]
        assert np.isclose(gs[1], os_[1], rtol=1e-10), (gs, os_)
        assert np.isclose(gs[2], os_[2], rtol=1e-7), (gs, os_)
        if gm.ndim == 2:
            err = min(np.abs(gm - om).max(), np.abs(gm + om).max())
        else:
            err = np.abs(gm - om).max()
        assert err < 1e-6 * max(1.0, np.abs(om).max()), (kind, loss, idx, err, gs, os_[:3])


# ---------------------------------------------------------------------------------------------- fast mode
@pytest.mark.parametrize("kind", ["pnp", "relpose", "fundamental", "homography"])
def test_fast_mode_gives_identical_results(cabi, kind):
    """fp32 screening + fp64 confirmation of candidates must reproduce the exact mode bit for bit (same trajectory,
    same models, same masks), and the oracle trajectory."""
    for seed in range(3):
        if kind == "pnp":
            p = G.abspose_problem(800, 0.4, 41, seed)
            a, b, me = p["x"] / G.FOCAL, p["X"], 12.0 / G.FOCAL
            kw = dict(max_iterations=3000, min_iterations=500, seed=seed)
        elif kind == "homography":
            p = G.homography_problem(4000, 0.5, 44, seed)
            a, b, me = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL, 1.0 / G.FOCAL
            kw = dict(max_iterations=5000, min_iterations=500, seed=seed)
        else:
            p = G.relpose_problem(6000 if kind == "relpose" else 3000, 0.3, 42, seed)
            a, b, me = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL, 1.0 / G.FOCAL
            kw = dict(max_iterations=30000, min_iterations=500, seed=seed)
        cabi.set_mode("exact")
        e = cabi.ransac(kind, a, b, cabi.RansacOpt(**kw), me)
        cabi.set_mode("fast")
        try:
            f = cabi.ransac(kind, a, b, cabi.RansacOpt(**kw), me)
        finally:
            cabi.set_mode("exact")
        assert f["stats"] == e["stats"], (f["stats"], e["stats"])
        assert np.array_equal(f["inliers"], e["inliers"])
        assert np.array_equal(np.asarray(f["model"]), np.asarray(e["model"]))
        assert f["counters"]["hypotheses"] == e["counters"]["hypotheses"]
        assert 0 < f["counters"]["models_confirmed"] < max(64, f["counters"]["models_evaluated"] // 4), f["counters"]
        o = P.ransac(kind, a, b, P.RansacOpt(**kw), me)
        # (the F refiner is run here on un-normalised calibrated coordinates, where its SVD parametrisation is
        #  ill-conditioned: trajectory and masks still agree exactly, the matrix itself to 1e-3)
        _same_trajectory(f, o, model_tol=1e-3 if kind == "fundamental" else 1e-6, relpose=(kind == "relpose"))


# ---------------------------------------------------------------------------------------------- BASELINE configs, full size
@pytest.mark.parametrize("mode", ["exact", "fast"])
def test_baseline_configs_at_full_size(cabi, mode):
    """BASELINE.json configs 1-4 at their full sizes through the estimate_* entry points (pixel coordinates + PINHOLE
    cameras), both precision modes, against the oracle: same trajectory, bit-exact masks, models to 1e-6."""
    cam = cabi.Camera("PINHOLE", (G.FOCAL, G.FOCAL, 0.0, 0.0))
    camt = (G.FOCAL, G.FOCAL, 0.0, 0.0)
    cabi.set_mode(mode)
    try:
        p = G.config_c1(0)
        g = cabi.estimate("pnp", p["x"], p["X"], cabi.RansacOpt(**p["ransac"]), cabi.BundleOpt(), p["max_error"], cam)
        o = P.estimate("pnp", p["x"], p["X"], P.RansacOpt(**p["ransac"]), P.BundleOpt(), p["max_error"], camt)
        _same_trajectory(g, o)
        p = G.config_c2(0)
        g = cabi.estimate("relpose", p["x1"], p["x2"], cabi.RansacOpt(**p["ransac"]), cabi.BundleOpt(), p["max_error"], cam, cam)
        o = P.estimate("relpose", p["x1"], p["x2"], P.RansacOpt(**p["ransac"]), P.BundleOpt(), p["max_error"], camt, camt)
        _same_trajectory(g, o, relpose=True)
        p = G.config_c3(0)
        g = cabi.estimate("fundamental", p["x1"], p["x2"], cabi.RansacOpt(**p["ransac"]), cabi.BundleOpt(), p["max_error"], rfc=True)
        o = P.estimate("fundamental", p["x1"], p["x2"], P.RansacOpt(**p["ransac"]), P.BundleOpt(), p["max_error"], rfc=True)
        _same_trajectory(g, o)
        p = G.config_c4(0)
        g = cabi.estimate("homography", p["x1"], p["x2"], cabi.RansacOpt(**p["ransac"]), cabi.BundleOpt(), p["max_error"])
        o = P.estimate("homography", p["x1"], p["x2"], P.RansacOpt(**p["ransac"]), P.BundleOpt(), p["max_error"])
        _same_trajectory(g, o)
    finally:
        cabi.set_mode("exact")


def test_mixed_batch_config5_style_fast_mode(cabi):
    """BASELINE config 5 in miniature: alternating p3p / 5pt problems with their own seeds through plb_ransac_batch
    (lock-step groups per kind), fast mode, several groups in flight."""
    probs, refs = [], []
    for i in range(16):
        if i % 2 == 0:
            p = G.abspose_problem(200, 0.5, 5, 100 + i)
            a, b, kind, me = p["x"] / G.FOCAL, p["X"], "pnp", 12.0 / G.FOCAL
            kw = dict(max_iterations=1000, min_iterations=1000, seed=i)
        else:
            p = G.relpose_problem(4000, 0.3, 5, 100 + i)
            a, b, kind, me = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL, "relpose", 1.0 / G.FOCAL
            kw = dict(max_iterations=100000, min_iterations=1000, seed=i)
        probs.append(dict(kind=kind, a=a, b=b, ransac=cabi.RansacOpt(**kw), max_error=me))
        refs.append(P.ransac(kind, a, b, P.RansacOpt(**kw), me))
    cabi.set_mode("fast")
    try:
        res = cabi.ransac_batch(probs, streams=3)
    finally:
        cabi.set_mode("exact")
    for g, o, pr in zip(res, refs, probs):
        assert g["status"] == 0
        _same_trajectory(g, o, relpose=(pr["kind"] == "relpose"))


@pytest.mark.parametrize("kind", ["relpose", "fundamental", "homography"])
@pytest.mark.parametrize("big", [False, True])
def test_heterogeneous_group_sizes_both_modes(cabi, kind, big):
    """One lock-step group of problems with very different numbers of correspondences (5 .. 12 000, and up to 20 000
    with `big`, which moves the screening kernel off its shared-memory path): the cost-balanced one-wave partition of
    the screening kernel crosses problem boundaries inside a CTA, the packed solver kernels mix samples of different
    problems in one warp.  Every problem must still follow the oracle's trajectory, in both precision modes."""
    sizes = [5, 9, 40, 333, 1000, 2500, 7001, 12000] + ([20000] if big else [])
    probs, refs = [], []
    for i, n in enumerate(sizes):
        if kind == "homography":
            p = G.homography_problem(n, 0.5, 41, i)
        else:
            p = G.relpose_problem(n, 0.4, 41, i)
        a, b = p["x1"] / G.FOCAL, p["x2"] / G.FOCAL
        kw = dict(max_iterations=3000, min_iterations=200, seed=10 + i)
        probs.append(dict(kind=kind, a=a, b=b, ransac=cabi.RansacOpt(**kw), max_error=1.5 / G.FOCAL))
        refs.append(P.ransac(kind, a, b, P.RansacOpt(**kw), 1.5 / G.FOCAL))
    for mode in ("exact", "fast"):
        cabi.set_mode(mode)
        try:
            res = cabi.ransac_batch(probs, streams=1)
        finally:
            cabi.set_mode("exact")
        for g, o in zip(res, refs):
            assert g["status"] == 0
            _same_trajectory(g, o, relpose=(kind == "relpose"), model_tol=1e-6 if kind != "fundamental" else 1e-3)


# ---------------------------------------------------------------------------------------------- cameras (rows N3 / N1)
DISTORTION_CAMERAS = [  # tests/example_cameras.h:31-38 of the reference, principal point moved to the image centre
    ("SIMPLE_RADIAL", [1100.0, 30.0, -20.0, -0.0397695]),
    ("RADIAL", [1050.0, -15.0, 25.0, -0.04012, 0.00123]),
    ("OPENCV", [1020.0, 990.0, 12.0, -8.0, 0.0141865, -0.0465301, 0.0005, -0.0003]),
    ("OPENCV", [868.993378, 866.063001, 5.9, -4.0, -0.399431, 0.188924, 0.000153, 0.000571]),
    ("SIMPLE_PINHOLE", [950.0, 3.0, 4.0]),
]


def _distort(cam, x_px):
    """pixel observations of the synthetic pinhole camera (f = G.FOCAL, pp = 0) re-imaged by `cam`."""
    X = np.c_[np.asarray(x_px) / G.FOCAL, np.ones(len(x_px))]
    return P.camera_project_with_jac(cam, X)[2]


@pytest.mark.parametrize("model,params", DISTORTION_CAMERAS)
def test_estimate_relative_pose_camera_prestep_on_device(cabi, model, params):
    """robust.cc:287-292: Camera::unproject of every point happens in the layout kernel; the calibrated points must be
    the oracle's doubles, so trajectory and masks are bit-exact."""
    p = G.relpose_problem(2500, 0.45, 31, 2)
    camo = (model, params)
    camg = cabi.Camera(model, params)
    x1, x2 = _distort(camo, p["x1"]), _distort(camo, p["x2"])
    kw = dict(max_iterations=20000, min_iterations=300, seed=4)
    for mode in (0, 1):
        cabi.set_mode(mode)
        g = cabi.estimate("relpose", x1, x2, cabi.RansacOpt(**kw), cabi.BundleOpt(), 1.5, camg, camg)
        cabi.set_mode(0)
        o = P.estimate("relpose", x1, x2, P.RansacOpt(**kw), P.BundleOpt(), 1.5, camo, camo)
        assert o["stats"]["num_inliers"] > 800
        _same_trajectory(g, o, relpose=True)
    # two different cameras
    cam2o = DISTORTION_CAMERAS[1]
    x2b = _distort(cam2o, p["x2"])
    g = cabi.estimate("relpose", x1, x2b, cabi.RansacOpt(**kw), cabi.BundleOpt(), 1.5, camg, cabi.Camera(*cam2o))
    o = P.estimate("relpose", x1, x2b, P.RansacOpt(**kw), P.BundleOpt(), 1.5, camo, cam2o)
    _same_trajectory(g, o, relpose=True)


@pytest.mark.parametrize("model,params", DISTORTION_CAMERAS)
def test_estimate_absolute_pose_distortion_cameras(cabi, model, params):
    """robust.cc:36-126 with a distorted camera: device unprojection + the final bundle adjustment through the
    camera's project_with_jac (optim/absolute.h:80-130)."""
    p = G.abspose_problem(1500, 0.5, 32, 4)
    camo = (model, params)
    x = _distort(camo, p["x"])
    kw = dict(max_iterations=5000, min_iterations=300, seed=1)
    g = cabi.estimate("pnp", x, p["X"], cabi.RansacOpt(**kw), cabi.BundleOpt(), 4.0, cabi.Camera(model, params))
    o = P.estimate("pnp", x, p["X"], P.RansacOpt(**kw), P.BundleOpt(), 4.0, camo)
    assert o["stats"]["num_inliers"] > 600
    _same_trajectory(g, o)


@pytest.mark.parametrize("model,params", DISTORTION_CAMERAS[:4])
def test_tangent_sampson_ransac_matches_oracle(cabi, model, params):
    """ransac.cc:155-168 (CameraRelativePoseEstimator): bearings + unprojection Jacobians computed on the device, 5-point
    solver on the bearings, tangent-Sampson MSAC scoring, LO over all points: same trajectory, bit-exact mask."""
    p = G.relpose_problem(2000, 0.4, 33, 1)
    camo = (model, params)
    camg = cabi.Camera(model, params)
    x1, x2 = _distort(camo, p["x1"]), _distort(camo, p["x2"])
    kw = dict(max_iterations=20000, min_iterations=300, seed=6)
    g = cabi.ransac_relpose_cameras(x1, x2, camg, camg, cabi.RansacOpt(**kw), 1.5)
    o = P.ransac_relpose_cameras(x1, x2, camo, camo, P.RansacOpt(**kw), 1.5)
    assert o["stats"]["num_inliers"] > 600
    _same_trajectory(g, o, relpose=True)
    for mode in (0, 1):  # the precision mode does not apply to this kind; results stay the same
        cabi.set_mode(mode)
        g = cabi.estimate("relpose", x1, x2, cabi.RansacOpt(**kw), cabi.BundleOpt(), 1.5, camg, camg, tangent_sampson=True)
        cabi.set_mode(0)
        o = P.estimate("relpose", x1, x2, P.RansacOpt(**kw), P.BundleOpt(), 1.5, camo, camo, tangent_sampson=True)
        _same_trajectory(g, o, relpose=True)


def test_tangent_sampson_edge_sizes_and_prosac(cabi):
    camo = DISTORTION_CAMERAS[0]
    camg = cabi.Camera(*camo)
    p = G.relpose_problem(400, 0.5, 34, 3, prosac_sorted=True)
    x1, x2 = _distort(camo, p["x1"]), _distort(camo, p["x2"])
    for n in (0, 4, 5, 6, 33, 400):
        kw = dict(max_iterations=300, min_iterations=50, seed=n, progressive_sampling=(n == 400))
        g = cabi.ransac_relpose_cameras(x1[:n], x2[:n], camg, camg, cabi.RansacOpt(**kw), 2.0)
        o = P.ransac_relpose_cameras(x1[:n], x2[:n], camo, camo, P.RansacOpt(**kw), 2.0)
        _same_trajectory(g, o, relpose=True)


@pytest.mark.parametrize("loss", ["TRIVIAL", "TRUNCATED", "HUBER", "CAUCHY"])
def test_refine_relpose_cameras_matches_oracle(cabi, loss):
    camo = DISTORTION_CAMERAS[1]
    camg = cabi.Camera(*camo)
    p = G.relpose_problem(600, 1.0, 35, 2)
    x1, x2 = _distort(camo, p["x1"]), _distort(camo, p["x2"])
    start = np.r_[p["q_gt"], p["t_gt"]] + np.random.default_rng(3).normal(0, 0.003, 7)
    start[:4] /= np.linalg.norm(start[:4])
    d1, M1 = P.camera_unproject_with_jac(camo, x1)
    d2, M2 = P.camera_unproject_with_jac(camo, x2)
    gm, gs = cabi.refine_relpose_cameras(start, x1, x2, camg, camg, cabi.BundleOpt(loss_type=loss, loss_scale=2.0))
    om, os_ = P.refine_relpose_tangent(start, d1, d2, M1, M2, P.BundleOpt(loss_type=loss, loss_scale=2.0))
    assert gs[0] == os_[0], (gs, os_)
    assert np.allclose(gs[1:3], os_[1:3], rtol=1e-9, atol=1e-12)
    assert np.allclose(gm, om, rtol=1e-6, atol=1e-8)


@pytest.mark.gpu
def test_p3p_lambdatwist_matches_oracle(cabi):
    """plb_p3p_lambdatwist_batch (solvers/p3p_lambdatwist.h:44) against the oracle restatement, which is itself bit-identical
    to the reference's own source on mini-Eigen (tests/test_ref_sources.py).  The closed-form cubic root goes through cbrt /
    cos / acos (CUDA's vs glibc's), then one Newton step and the depth refinement: tolerance 1e-9, same solution count
    except where a threshold decision sits within rounding (allowed on < 1 % of the instances)."""
    rng = np.random.default_rng(21)
    xs, Xs = [], []
    while len(xs) < 600:
        X = np.c_[rng.uniform(-2, 2, (3, 2)), rng.uniform(2, 8, 3)]
        w = rng.normal(size=3) * 0.5
        th = np.linalg.norm(w)
        K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        R = np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th**2 * K @ K
        Y = X @ R.T + rng.normal(size=3)
        if (Y[:, 2] < 0.1).any():
            continue
        xs.append(Y / np.linalg.norm(Y, axis=1)[:, None])
        Xs.append(X)
    poses, n = cabi.p3p_lambdatwist_batch(np.array(xs), np.array(Xs))
    count_diff = 0
    for i in range(len(xs)):
        ref = P.p3p_lambdatwist(xs[i], Xs[i])
        if n[i] != len(ref):
            count_diff += 1
            continue
        if len(ref):
            scale = max(1.0, np.abs(ref).max())
            assert np.abs(poses[i, :n[i]] - ref).max() <= 1e-9 * scale, (i, poses[i, :n[i]], ref)
    assert count_diff <= 5, count_diff
    assert n.sum() > 600


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pnp", "homography", "fundamental"])
def test_fast_mode_on_badly_scaled_inputs(cabi, kind):
    """The inputs the fp32 screening copy likes least: 3D points a few thousand units from the origin with a tight
    threshold (PnP), and pixel-unit coordinates of a few thousand with a one-pixel threshold (homography, fundamental
    matrix).  The screening intervals are derived from the data (per-problem coordinate maxima), so the default mode must
    still reproduce the all-fp64 mode bit for bit and follow the oracle's trajectory; what may change is how many models
    need the fp64 confirmation."""
    for seed in range(2):
        if kind == "pnp":
            p = G.abspose_problem(600, 0.45, 51, seed)
            off = np.array([4000.0, -2500.0, 6000.0])
            a, b, me = p["x"] / G.FOCAL, p["X"] + off, 2.0 / G.FOCAL  # (the pose absorbs the offset: t -> t - R off)
            kw = dict(max_iterations=3000, min_iterations=300, seed=seed)
        elif kind == "homography":
            p = G.homography_problem(3000, 0.5, 54, seed)
            # pixels, principal point not removed: coordinates up to ~1100 with a one-pixel threshold (the minimal
            # solver itself is poorly conditioned in these units — few inliers, like the reference — which is beside the
            # point here)
            a, b, me = p["x1"] + 300.0, p["x2"] + 300.0, 1.0
            kw = dict(max_iterations=4000, min_iterations=300, seed=seed)
        else:
            p = G.relpose_problem(2500, 0.4, 52, seed)
            a, b, me = p["x1"] + 1200.0, p["x2"] + 1200.0, 1.0
            kw = dict(max_iterations=8000, min_iterations=300, seed=seed)
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
        for k in ("iterations", "refinements", "num_inliers"):
            assert f["stats"][k] == o["stats"][k], (k, f["stats"], o["stats"])
        assert np.array_equal(f["inliers"], o["inliers"])
