"""GPU half of tests/test_golden_reference.py: the CUDA path, called through the C-ABI, reproduces the committed fixtures
that PoseLib's OWN SOURCES produced (tests/golden/reference_sources.json; generator and provenance:
tests/golden/make_reference_golden.py, DESIGN.md §2) — iterations, refinements, inlier counts and inlier masks exactly, the
MSAC score to 2e-9 and the model to 2e-6 relative (north_star's 1e-6 against the oracle plus the oracle's own, measured,
distance to the fixtures: <= 1e-10).  Every case repeats a case of tests/test_gpu_parity.py input for input.
(The file name sorts last so that `pytest -x` reaches the oracle-parity tests first.)"""
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import reference_cases as RC  # noqa: E402

GOLD = json.load(open(os.path.join(HERE, "golden", "reference_sources.json")))["cases"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(RC.CASES))
def test_cuda_path_reproduces_the_reference_sources_fixtures(name):
    from poselib_b200 import cabi
    if cabi.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    cabi.set_device(0)
    case, gold = RC.CASES[name](), GOLD[name]
    RC.check(RC.run(cabi, case), gold, case["kind"], model_tol=2e-6, score_rtol=2e-9)


REFINE = json.load(open(os.path.join(HERE, "golden", "reference_sources.json")))["refine"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,loss", RC.REFINE_CELLS)
def test_cuda_refiners_reproduce_the_reference_sources_refinements(kind, loss):
    """plb_bundle_adjust / plb_refine_* against the refinements the reference's sources produced — the cases and the
    tolerances of tests/test_gpu_parity.py::test_lm_refiners_match_oracle (initial cost 1e-10, final cost 1e-7, model 1e-6;
    the oracle reproduces these fixtures bit for bit on the CPU)."""
    from poselib_b200 import cabi
    if cabi.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    cabi.set_device(0)
    for (m0, a, b, kw), gold in zip(RC.refine_cases(kind, loss), REFINE[f"{kind}/{loss}"]):
        m, bs = cabi.refine(kind, m0, a, b, cabi.BundleOpt(**kw))
        RC.check_refine(m, bs, gold, model_tol=1e-6, cost0_rtol=1e-10, cost_rtol=1e-7)


SOLVER_GOLD = json.load(open(os.path.join(HERE, "golden", "reference_sources.json")))["solvers"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", RC.SOLVERS)
def test_cuda_solvers_reproduce_the_reference_sources_solver_outputs(name):
    """plb_p3p_batch / plb_p3p_lambdatwist_batch / plb_relpose_7pt_batch / plb_homography_4pt_batch against the solutions the reference's sources
    returned for the first instances of tests/test_gpu_parity.py's solver tests — solution counts exactly, values with
    that file's tolerances (p3p 1e-9, 7pt 1e-8 relative, homography 1e-10 relative)."""
    import numpy as np
    from poselib_b200 import cabi
    if cabi.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    cabi.set_device(0)
    a, b = RC.solver_instances(name)
    fn = {"p3p": cabi.p3p_batch, "p3p_lambdatwist": cabi.p3p_lambdatwist_batch, "relpose_7pt": cabi.relpose_7pt_batch, "homography_4pt": cabi.homography_4pt_batch}[name]
    out, n = fn(a, b)
    like = (7,) if name.startswith("p3p") else (3, 3)
    for i in range(len(a)):
        flat = np.array([float.fromhex(v) for v in SOLVER_GOLD[name][i]])
        g = flat.reshape((-1,) + like)
        assert n[i] == len(g), (name, i, n[i], len(g))
        if name.startswith("p3p"):
            assert np.allclose(out[i, :n[i]], g, rtol=1e-9, atol=1e-9, equal_nan=True), i
        elif name == "relpose_7pt":
            assert np.allclose(out[i, :n[i]], g, rtol=1e-8, atol=1e-9, equal_nan=True), i
        elif n[i]:
            assert np.allclose(out[i], g[0], rtol=1e-10, atol=1e-12, equal_nan=True), i


@pytest.mark.gpu
def test_poselib_client_runs_on_the_b200_backend():
    """tests/dropin_client_test.cc — a client written against PoseLib's own headers only, whose checks pass on PoseLib's own
    CPU implementation (tests/test_dropin_reference_headers.py) — linked with poselib_b200/adapter/poselib_dropin.cc and
    libposelib_b200.so instead: every estimate_*, ransac_relpose, refine_relpose and relpose_5pt call goes through PoseLib's
    declared signatures into the CUDA path.  The binary is built in the CPU container (it needs the reference's headers)."""
    import subprocess
    exe = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "dropin_client")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/dropin_client was not built (build() builds it where the reference's headers are)")
    out = subprocess.run([exe, "run"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "dropin run ok" in out.stdout, out.stdout + out.stderr

