"""Device-vs-reference deviation of the fisheye and division camera models on the GPU: the numbers behind the
tolerances of tests/test_camera_models.py.

  * camera functions: the largest relative deviation |dev - host| / max(1, |host|) of every camera function of
    camera.cuh on the device against its host build (which equals the reference bit for bit), per test camera, and
    whether the division models' arithmetic-only columns are equal;
  * end to end: the largest relative deviation of cost, initial cost, pose and camera parameters of
    plb_bundle_adjust_image, plb_estimate_absolute_pose_image, plb_refine_relpose_pair and
    plb_estimate_relative_pose_pair against tests/golden/reference_camera_models.json, per fisheye / division model, and
    the number of cases whose iteration counts, RANSAC stats or inlier masks differ.
Prints one JSON line per measurement, after one line with the card's name and power limit.

    python tools/camera_models_deviation.py
"""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from poselib_b200 import cabi  # noqa: E402
import make_camera_models_golden as CG  # noqa: E402


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    ok = np.isfinite(b)
    return float(np.max(np.abs(a[ok] - b[ok]) / np.maximum(1.0, np.abs(b[ok])), initial=0.0))


def family(cam):
    return "fisheye" if "FISHEYE" in CG.CAMERAS[cam][0] else "division"


def pair_family(pair):
    """A pair with a fisheye camera counts as fisheye (atan2 / tan), otherwise as division."""
    return "fisheye" if any("FISHEYE" in CG.CAMERAS[c][0] for c in pair) else "division"


def cam_of(name, params):
    return cabi.Camera(CG.CAMERAS[name][0], tuple(params))


def main():
    if cabi.device_count() == 0:
        sys.exit("no CUDA device: nothing is measured")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.splitlines()[0]
    print(json.dumps(dict(card=q.split(",")[0].strip(), power_limit=q.split(",")[1].strip())))
    gold = json.load(open(CG.OUT))
    tmp = tempfile.mkdtemp(prefix="camera_models_deviation_")
    for cam in CG.NEW:
        rows = CG.device_camera_rows(cam, tmp)
        for kind, (dev, host) in rows.items():
            ne = 0 if family(cam) == "fisheye" else CG.DIVISION_EXACT_COLUMNS[kind]
            print(json.dumps(dict(what="camera functions", camera=cam, rows=kind,
                                  exact_columns_equal=bool(np.array_equal(dev[:, :ne], host[:, :ne], equal_nan=True)),
                                  max_rel=rel(dev, host))))
    dev = {}

    def note(fam, call, key, value):
        d = dev.setdefault((fam, call), {})
        d[key] = max(d.get(key, 0.0), value)

    ro = cabi.RansacOpt(**CG.ESTIMATE_RANSAC)
    for c in gold["bundle"]:
        x, X, pose0, p0 = CG.problem(c["camera"], CG.BUNDLE_N, CG.bundle_seed(c["camera"], c["flags"], c["loss"]))
        b = cabi.BundleOpt(loss_type=c["loss"], loss_scale=gold["loss_scale"], relative_cost_tol=gold["relative_cost_tol"],
                           refine_intrinsics=c["flags"])
        pose, params, bs = cabi.refine_image(pose0, x, X, cam_of(c["camera"], p0), b)
        f = family(c["camera"])
        note(f, "bundle_adjust_image", "iteration_mismatches", int(int(bs[0]) != c["iterations"]))
        note(f, "bundle_adjust_image", "initial_cost", rel(bs[1], c["initial_cost"]))
        note(f, "bundle_adjust_image", "cost", rel(bs[2], c["cost"]))
        note(f, "bundle_adjust_image", "pose", rel(pose, c["pose"]))
        note(f, "bundle_adjust_image", "params", rel(params, c["params"]))
    for c in gold["estimate_cases"]:
        x, X, _, p0 = CG.problem(c["camera"], CG.ESTIMATE_N, CG.estimate_seed(c["camera"]), outliers=0.3)
        g = cabi.estimate_image(x, X, cam_of(c["camera"], p0), ro, cabi.BundleOpt(refine_intrinsics=c["flags"]),
                                CG.ESTIMATE_MAX_ERROR)
        mask = np.unpackbits(np.frombuffer(bytes.fromhex(c["inliers"]), dtype=np.uint8))[:CG.ESTIMATE_N].astype(bool)
        f = family(c["camera"])
        note(f, "estimate_absolute_pose_image", "outcome_mismatches",
             int(any(g["stats"][k] != c[k] for k in ("iterations", "refinements", "num_inliers")) or
                 not np.array_equal(g["inliers"].astype(bool), mask)))
        note(f, "estimate_absolute_pose_image", "pose", rel(g["model"], c["pose"]))
        note(f, "estimate_absolute_pose_image", "params", rel(g["camera"], c["params"]))
    for c in gold["refine"]:
        pair = (c["camera1"], c["camera2"])
        x1, x2, pose0, c1, c2 = CG.pair_problem(*pair, CG.PAIR_N, c["seed"])
        b = cabi.BundleOpt(loss_type=c["loss"], loss_scale=gold["pair_loss_scale"],
                           relative_cost_tol=gold["relative_cost_tol"], refine_intrinsics=c["flags"])
        pose, p1, p2, bs = cabi.refine_relpose_pair(pose0, x1, x2, cam_of(pair[0], c1), cam_of(pair[1], c2), b)
        f = pair_family(pair)
        note(f, "refine_relpose_pair", "iteration_mismatches", int(int(bs[0]) != c["iterations"]))
        note(f, "refine_relpose_pair", "initial_cost", rel(bs[1], c["initial_cost"]))
        note(f, "refine_relpose_pair", "cost", rel(bs[2], c["cost"]))
        note(f, "refine_relpose_pair", "pose", rel(pose, c["pose"]))
        note(f, "refine_relpose_pair", "params", max(rel(p1, c["params1"]), rel(p2, c["params2"])))
    for c in gold["pair_estimate_cases"]:
        pair = (c["camera1"], c["camera2"])
        x1, x2, _, c1, c2 = CG.pair_estimate_inputs(pair, c["seed"], c["tangent"])
        g = cabi.estimate_relative_pose_pair(x1, x2, cam_of(pair[0], c1), cam_of(pair[1], c2), ro,
                                             cabi.BundleOpt(refine_intrinsics=c["flags"]), CG.PAIR_MAX_ERROR,
                                             tangent_sampson=c["tangent"])
        mask = np.unpackbits(np.frombuffer(bytes.fromhex(c["inliers"]), dtype=np.uint8))[:CG.ESTIMATE_N].astype(bool)
        f = pair_family(pair)
        note(f, "estimate_relative_pose_pair", "outcome_mismatches",
             int(any(g["stats"][k] != c[k] for k in ("iterations", "refinements", "num_inliers")) or
                 not np.array_equal(g["inliers"].astype(bool), mask)))
        note(f, "estimate_relative_pose_pair", "pose", rel(g["model"], c["pose"]))
        note(f, "estimate_relative_pose_pair", "params", max(rel(g["camera1"], c["params1"]),
                                                             rel(g["camera2"], c["params2"])))
    for (f, call), d in sorted(dev.items()):
        print(json.dumps(dict(what="end to end", family=f, call=call, **d)))


if __name__ == "__main__":
    main()
