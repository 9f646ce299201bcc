"""GPU test (-m gpu): BASELINE config 5 at FULL size — all 4096 independent problems (2048 p3p C1-type, 2048 5pt C2-type
with 10 000 correspondences each) through ONE plb_ransac_batch call, every single result held to the CPU oracle's:
iterations, refinements, inlier count and the inlier mask (by CRC32) exactly, the model to 1e-6.  The oracle's results are
the committed fixture tests/golden/c5_oracle.npz (written on the CPU by tests/golden/make_c5_golden.py; ≈ 15 CPU-minutes
of oracle time that the GPU box does not have to spend)."""
import os
import zlib

import numpy as np
import pytest

from poselib_b200 import problem_generator as G

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_all_4096_config5_problems_match_the_oracle():
    from poselib_b200 import cabi
    if cabi.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    cabi.set_device(0)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "c5_oracle.npz"))
    count = len(gold["iterations"])
    assert count == 4096
    F = G.FOCAL
    probs = []
    for i in range(count):
        if i % 2 == 0:
            p = G.abspose_problem(200, 0.5, 5, i)
            probs.append(dict(kind="pnp", a=p["x"] / F, b=p["X"], max_error=12.0 / F,
                              ransac=cabi.RansacOpt(max_iterations=1000, min_iterations=1000)))
        else:
            p = G.relpose_problem(10000, 0.3, 5, i)
            probs.append(dict(kind="relpose", a=p["x1"] / F, b=p["x2"] / F, max_error=1.0 / F,
                              ransac=cabi.RansacOpt(max_iterations=100000, min_iterations=1000)))
    res = cabi.ransac_batch(probs, streams=12, n_gpus=0)  # every GPU of the box
    bad = []
    for i, r in enumerate(res):
        st = r["stats"]
        ok = (st["iterations"] == gold["iterations"][i] and st["refinements"] == gold["refinements"][i] and
              st["num_inliers"] == gold["num_inliers"][i] and
              zlib.crc32(np.asarray(r["inliers"], dtype=np.uint8).tobytes()) == gold["mask_crc"][i])
        m, g = np.asarray(r["model"], dtype=np.float64), gold["model"][i]
        if i % 2 == 1:  # |t| of a relative pose is a gauge the refiner never renormalises: compare up to it
            m = np.r_[m[:4], m[4:] / np.linalg.norm(m[4:])]
            g = np.r_[g[:4], g[4:] / np.linalg.norm(g[4:])]
        ok = ok and np.allclose(m, g, rtol=1e-6, atol=1e-8)
        if not ok:
            bad.append((i, st, int(gold["iterations"][i]), int(gold["num_inliers"][i])))
    assert not bad, (len(bad), bad[:5])
