"""Writes tests/golden/reference_camera_ops.json: PoseLib's own Camera functions, point by point, for every camera model
on the path, which plb_camera_batch is held to.

Cameras: the seven of tests/test_camera_host_build.py (NULL, SIMPLE_RADIAL, PINHOLE, SIMPLE_PINHOLE, RADIAL and both OPENCV
sets) and the eight of make_camera_models_golden.CAMERAS (both fisheye models, DIVISION and SIMPLE_DIVISION with k < 0
and k > 0, PINHOLE, RADIAL).  Inputs: make_camera_models_golden.host_points of each camera (near the axis, theta at pi/2,
bearings past 90 degrees, division points with disc2 < 0, points behind the camera and at Z = 0), with its spread of
ordinary points cut to the first few, regenerated from their seeds by points(), so the file holds cameras and results
only.

Per camera, from the reference's sources compiled on mini-Eigen (oracle/_ref/libplref2.so) through
tests/ref_camera_models_client.cc:
  pixels  (cm_unproject): x3 = unproject to a bearing, x2 = the 2D unproject wrapper, d / M / dp = unproject_with_jac
          with a jac_point (the jac_point-less call gives the same d and dp bits: checked here, stored once);
  points  (cm_project):   xp = project, xq / jac / jp = project_with_jac.
Matrices are row-major, parameter Jacobians cut to the model's parameter count.  Every array is stored as the base64 of
its zlib-compressed little-endian doubles, so NaN and infinities survive bit for bit.

    python tests/golden/make_camera_ops_golden.py          (needs the reference checkout; CPU only)
"""
import base64
import ctypes as C
import json
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_camera_models_golden as CG  # noqa: E402

OUT = os.path.join(HERE, "reference_camera_ops.json")
IDS = {"NULL": -1, **CG.MODEL_IDS}
# name -> (model, parameters): tests/test_camera_host_build.py's cameras, then make_camera_models_golden.CAMERAS
CAMERAS = {
    "NULL": ("NULL", []),
    "SIMPLE_RADIAL/host": ("SIMPLE_RADIAL", [2425.85, 932.383, 628.265, -0.0397695]),
    "PINHOLE/host": ("PINHOLE", [3425.62, 3426.29, 3118.41, 2069.07]),
    "SIMPLE_PINHOLE/host": ("SIMPLE_PINHOLE", [3425.62, 3118.41, 2069.07]),
    "RADIAL/host": ("RADIAL", [2425.85, 932.38, 629.325, -0.04012, 0.00123]),
    "OPENCV/host": ("OPENCV", [2575.94, 2608.29, 1599.26, 1257.13, 0.141865, -0.465301, 0, 0]),
    "OPENCV/host2": ("OPENCV", [868.993378, 866.063001, 525.942323, 420.042529, -0.399431, 0.188924, 0.000153, 0.000571]),
    **{name: (m, list(p)) for name, (m, p) in CG.CAMERAS.items()},
}
PX_FIELDS = ("x3", "x2", "d", "M", "dp")
# host_points draws 40 ordinary pixels and 30 ordinary points before its branch cases; these many of them are kept
PX_SPREAD, PT_SPREAD = 10, 8
PT_FIELDS = ("xp", "xq", "jac", "jp")


def model_id(name):
    return IDS[CAMERAS[name][0]]


def params8(name):
    p = np.zeros(8)
    v = CAMERAS[name][1]
    p[:len(v)] = v
    return p


def points(name):
    """host_points of the camera: pixels [n, 2] and camera-frame points [n, 3].  The NULL camera's grid is drawn with
    f = 1 and the principal point at the origin, in the normalised coordinates that camera works in.  The first
    PX_SPREAD / PT_SPREAD ordinary pixels / points and every branch case are kept, and three points are added: two at
    Z = 0 (one at the origin) and one behind the camera."""
    p = params8(name)
    if model_id(name) == -1:
        p[0] = 1.0
    px, Z = CG.host_points(model_id(name), p)
    px = np.concatenate([px[:PX_SPREAD], px[40:]])
    Z = np.concatenate([Z[:PT_SPREAD], Z[30:], [[0.3, -0.2, 0.0], [0.0, 0.0, 0.0], [0.5, 0.5, -2.0]]])
    return px, Z


def enc(a):
    return base64.b64encode(zlib.compress(np.ascontiguousarray(a, dtype="<f8").tobytes(), 9)).decode()


def dec(s, shape):
    return np.frombuffer(zlib.decompress(base64.b64decode(s)), dtype="<f8").reshape(shape).copy()


def reference(lib, name):
    """The reference's outputs for camera `name` on points(name): dict of arrays (rows per point)."""
    model, P = model_id(name), CG.NUM_PARAMS[model_id(name)]
    params = params8(name)
    px, Z = points(name)
    n, nz = len(px), len(Z)
    x3, x2, d, M, dp, dq, dpq = (np.zeros(3 * n), np.zeros(2 * n), np.zeros(3 * n), np.zeros(6 * n), np.zeros(24 * n),
                                 np.zeros(3 * n), np.zeros(24 * n))
    pxc = np.ascontiguousarray(px)
    lib.cm_unproject(model, CG._p(params), C.c_int64(n), CG._p(pxc), CG._p(x3), CG._p(x2), CG._p(d), CG._p(M), CG._p(dp),
                     CG._p(dq), CG._p(dpq))
    dp = dp.reshape(n, 3, 8)[:, :, :P]
    if not (np.array_equal(d, dq, equal_nan=True) and np.array_equal(dp, dpq.reshape(n, 3, 8)[:, :, :P], equal_nan=True)):
        sys.exit("unproject_with_jac without a jac_point differs from the call with one: %s" % name)
    xp, xq, jac, jp = np.zeros(2 * nz), np.zeros(2 * nz), np.zeros(6 * nz), np.zeros(16 * nz)
    Zc = np.ascontiguousarray(Z)
    lib.cm_project(model, CG._p(params), C.c_int64(nz), CG._p(Zc), CG._p(xp), CG._p(xq), CG._p(jac), CG._p(jp))
    return dict(x3=x3.reshape(n, 3), x2=x2.reshape(n, 2), d=d.reshape(n, 3), M=M.reshape(n, 3, 2), dp=dp,
                xp=xp.reshape(nz, 2), xq=xq.reshape(nz, 2), jac=jac.reshape(nz, 2, 3), jp=jp.reshape(nz, 2, 8)[:, :, :P])


def case(lib, name):
    r = reference(lib, name)
    return dict(camera=name, model=model_id(name), params=list(CAMERAS[name][1]), n_px=len(r["x3"]),
                n_pt=len(r["xp"]), **{k: enc(r[k]) for k in PX_FIELDS + PT_FIELDS})


def load(path=OUT):
    """The fixture with every array decoded: list of dict(camera, model, params, px, Z, and the fields above)."""
    out = []
    for c in json.load(open(path))["cases"]:
        P = CG.NUM_PARAMS[c["model"]]
        n, nz = c["n_px"], c["n_pt"]
        shapes = dict(x3=(n, 3), x2=(n, 2), d=(n, 3), M=(n, 3, 2), dp=(n, 3, P), xp=(nz, 2), xq=(nz, 2), jac=(nz, 2, 3),
                      jp=(nz, 2, P))
        r = dict(camera=c["camera"], model=c["model"], params=c["params"])
        r["px"], r["Z"] = points(c["camera"])
        r.update({k: dec(c[k], shapes[k]) for k in shapes})
        out.append(r)
    return out


def main():
    lib = CG.build_client()
    gold = dict(cases=[case(lib, name) for name in CAMERAS])
    with open(OUT, "w") as f:
        json.dump(gold, f, indent=0)
    print("wrote", OUT, len(gold["cases"]), "cameras")


if __name__ == "__main__":
    main()
