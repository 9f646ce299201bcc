"""ctypes binding of the C-ABI (include/poselib_b200.h) — the call a Python user (or the parity tests) makes.

Every function goes through `libposelib_b200.so`; there is no Python or CPU compute path here.  If the CUDA
library is missing, import fails loudly; if no GPU is usable, the compute entry points raise PoseLibB200Error.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libposelib_b200.so")

PLB_OK, PLB_ERR_CUDA, PLB_ERR_ARG, PLB_ERR_NYI = 0, -1, -2, -3
KIND = {"pnp": 0, "relpose": 1, "fundamental": 2, "homography": 3}
LOSS = {"TRIVIAL": 0, "TRUNCATED": 1, "HUBER": 2, "CAUCHY": 3}
CAMERA = {"NULL": -1, "SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "RADIAL": 3, "OPENCV": 4,
          "SIMPLE_RADIAL_FISHEYE": 8, "RADIAL_FISHEYE": 9, "DIVISION": 101, "SIMPLE_DIVISION": 102}
CAMERA_NUM_PARAMS = {-1: 0, 0: 3, 1: 4, 2: 4, 3: 5, 4: 8, 8: 4, 9: 5, 101: 5, 102: 4}
# BundleOpt.refine_intrinsics bits (refine_focal_length, refine_principal_point, refine_extra_params)
REFINE_FOCAL_LENGTH, REFINE_PRINCIPAL_POINT, REFINE_EXTRA_PARAMS = 1, 2, 4


class PoseLibB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"poselib_b200 error {code}: {msg}")
        self.code = code


class RansacOpt(C.Structure):
    """PoseLib/types.h:39-50"""
    _fields_ = [("max_iterations", C.c_uint64), ("min_iterations", C.c_uint64),
                ("dyn_num_trials_mult", C.c_double), ("success_prob", C.c_double),
                ("seed", C.c_uint64), ("progressive_sampling", C.c_int32),
                ("score_initial_model", C.c_int32), ("max_prosac_iterations", C.c_uint64)]

    def __init__(self, max_iterations=100000, min_iterations=1000, dyn_num_trials_mult=3.0,
                 success_prob=0.9999, seed=0, progressive_sampling=False, score_initial_model=False,
                 max_prosac_iterations=100000):
        super().__init__(max_iterations, min_iterations, dyn_num_trials_mult, success_prob, seed,
                         int(progressive_sampling), int(score_initial_model), max_prosac_iterations)


class RansacStats(C.Structure):
    """PoseLib/types.h:52-58"""
    _fields_ = [("refinements", C.c_uint64), ("iterations", C.c_uint64), ("num_inliers", C.c_uint64),
                ("inlier_ratio", C.c_double), ("model_score", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class BundleOpt(C.Structure):
    """PoseLib/types.h:60-95"""
    _fields_ = [("max_iterations", C.c_uint64), ("loss_type", C.c_int32), ("refine_intrinsics", C.c_int32),
                ("loss_scale", C.c_double), ("gradient_tol", C.c_double), ("step_tol", C.c_double),
                ("relative_cost_tol", C.c_double), ("initial_lambda", C.c_double),
                ("min_lambda", C.c_double), ("max_lambda", C.c_double)]

    def __init__(self, max_iterations=100, loss_type="CAUCHY", loss_scale=1.0, gradient_tol=1e-12,
                 step_tol=1e-8, relative_cost_tol=1e-10, initial_lambda=1e-3, min_lambda=1e-10,
                 max_lambda=1e10, refine_intrinsics=0):
        lt = LOSS[loss_type] if isinstance(loss_type, str) else int(loss_type)
        super().__init__(max_iterations, lt, int(refine_intrinsics), loss_scale, gradient_tol, step_tol,
                         relative_cost_tol, initial_lambda, min_lambda, max_lambda)


class Counters(C.Structure):
    _fields_ = [("samples", C.c_uint64), ("hypotheses", C.c_uint64), ("scored_corrs", C.c_uint64),
                ("lo_calls", C.c_uint64), ("lo_seconds", C.c_double), ("gpu_launches", C.c_uint64),
                ("samples_evaluated", C.c_uint64), ("gpu_seconds", C.c_double), ("h2d_bytes", C.c_uint64),
                ("d2h_bytes", C.c_uint64), ("models_evaluated", C.c_uint64), ("models_confirmed", C.c_uint64),
                ("gpu_seconds_score", C.c_double), ("gpu_seconds_select", C.c_double), ("gpu_seconds_lo", C.c_double),
                ("rounds", C.c_uint64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class Camera(C.Structure):
    _fields_ = [("model_id", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("reserved", C.c_int32),
                ("params", C.c_double * 8)]

    def __init__(self, model="PINHOLE", params=(1.0, 1.0, 0.0, 0.0), width=0, height=0):
        mid = CAMERA[model] if isinstance(model, str) else int(model)
        p = list(params)[:8] + [0.0] * (8 - len(params))
        super().__init__(mid, width, height, 0, (C.c_double * 8)(*p))


class Problem(C.Structure):
    _fields_ = [("kind", C.c_int32), ("real_focal_check", C.c_int32), ("n", C.c_uint64),
                ("a", C.POINTER(C.c_double)), ("b", C.POINTER(C.c_double)), ("opt", RansacOpt),
                ("max_error", C.c_double), ("model", C.c_double * 9), ("inliers", C.c_char_p),
                ("stats", RansacStats), ("counters", Counters), ("status", C.c_int32), ("resident", C.c_int32)]


EXPORTS = [
    "plb_ransac_opt_default", "plb_bundle_opt_default", "plb_last_error", "plb_device_count", "plb_set_device",
    "plb_set_mode", "plb_host_sample_table", "plb_device_sample_table", "plb_host_dynamic_max_iter", "plb_ransac_pnp", "plb_ransac_relpose", "plb_ransac_relpose_cameras", "plb_ransac_fundamental",
    "plb_ransac_homography",
    "plb_estimate_absolute_pose", "plb_estimate_relative_pose", "plb_estimate_relative_pose_pair", "plb_estimate_fundamental",
    "plb_estimate_homography", "plb_p3p_batch", "plb_p3p_lambdatwist_batch", "plb_relpose_5pt_batch", "plb_relpose_5pt_poses_batch",
    "plb_relpose_7pt_batch", "plb_homography_4pt_batch", "plb_essential_matrix_8pt_batch", "plb_relpose_8pt_batch", "plb_ransac_batch", "plb_ransac_batch_multi", "plb_estimate_batch", "plb_bundle_adjust",
    "plb_bundle_adjust_image", "plb_estimate_absolute_pose_image", "plb_refine_relpose", "plb_refine_relpose_cameras", "plb_refine_relpose_pair", "plb_refine_fundamental", "plb_refine_homography", "plb_resident_create",
    "plb_resident_free", "plb_bundle_adjust_image_weighted", "plb_refine_relpose_weighted",
    "plb_refine_relpose_cameras_weighted", "plb_refine_relpose_pair_weighted", "plb_refine_fundamental_weighted",
    "plb_refine_homography_weighted", "plb_estimate_batch_device", "plb_refine_batch", "plb_refine_batch_device",
    "plb_score_batch", "plb_score_batch_device", "plb_generate_batch", "plb_generate_batch_device",
    "plb_camera_batch", "plb_camera_batch_device",
]
DTYPE_F64, DTYPE_F32 = 0, 1

class EstimateProblem(C.Structure):
    _fields_ = [("kind", C.c_int32), ("real_focal_check", C.c_int32), ("tangent_sampson", C.c_int32), ("reserved", C.c_int32),
                ("n", C.c_uint64), ("a", C.POINTER(C.c_double)), ("b", C.POINTER(C.c_double)),
                ("camera1", Camera), ("camera2", Camera), ("ransac", RansacOpt), ("bundle", BundleOpt),
                ("max_error", C.c_double), ("model", C.c_double * 9), ("inliers", C.c_char_p),
                ("stats", RansacStats), ("counters", Counters), ("status", C.c_int32), ("reserved2", C.c_int32)]


# plb_refine_problem::refiner: the robust/bundle.h refiner of each single entry point
REFINER = {"bundle": 0, "bundle_image": 1, "relpose": 2, "relpose_cameras": 3, "relpose_pair": 4, "fundamental": 5,
           "homography": 6}


class RefineProblem(C.Structure):
    _fields_ = [("refiner", C.c_int32), ("reserved", C.c_int32), ("n", C.c_uint64), ("a", C.POINTER(C.c_double)),
                ("b", C.POINTER(C.c_double)), ("weights", C.POINTER(C.c_double)), ("camera1", Camera),
                ("camera2", Camera), ("bundle", BundleOpt), ("model", C.c_double * 9), ("bundle_stats", C.c_double * 3),
                ("status", C.c_int32), ("reserved2", C.c_int32)]


class ScoreProblem(C.Structure):
    _fields_ = [("kind", C.c_int32), ("tangent_sampson", C.c_int32), ("n", C.c_uint64), ("a", C.POINTER(C.c_double)),
                ("b", C.POINTER(C.c_double)), ("camera1", Camera), ("camera2", Camera), ("m", C.c_uint64),
                ("models", C.POINTER(C.c_double)), ("sq_threshold", C.c_double), ("scores", C.POINTER(C.c_double)),
                ("num_inliers", C.POINTER(C.c_int64)), ("inliers", C.c_char_p), ("status", C.c_int32),
                ("reserved", C.c_int32)]


class GenerateProblem(C.Structure):
    _fields_ = [("kind", C.c_int32), ("tangent_sampson", C.c_int32), ("real_focal_check", C.c_int32),
                ("reserved", C.c_int32), ("n", C.c_uint64), ("a", C.POINTER(C.c_double)), ("b", C.POINTER(C.c_double)),
                ("camera1", Camera), ("camera2", Camera), ("s", C.c_uint64), ("samples", C.POINTER(C.c_int32)),
                ("sq_threshold", C.c_double), ("n_models", C.POINTER(C.c_int32)), ("models", C.POINTER(C.c_double)),
                ("scores", C.POINTER(C.c_double)), ("num_inliers", C.POINTER(C.c_int64)), ("status", C.c_int32),
                ("reserved2", C.c_int32)]


class CameraProblem(C.Structure):
    _fields_ = [("op", C.c_int32), ("reserved", C.c_int32), ("n", C.c_uint64), ("camera", Camera),
                ("in_", C.POINTER(C.c_double)), ("out", C.POINTER(C.c_double)), ("jac", C.POINTER(C.c_double)),
                ("jac_params", C.POINTER(C.c_double)), ("status", C.c_int32), ("reserved2", C.c_int32)]


# plb_camera_problem::op
CAMOP = {"project": 0, "unproject": 1, "unproject_2d": 2}


# plb_generate_problem: indices per sample (k) and model slots per sample (M) of each kind
GENERATE_K = {"pnp": 3, "relpose": 5, "fundamental": 7, "homography": 4}
GENERATE_M = {"pnp": 4, "relpose": 40, "fundamental": 3, "homography": 1}


if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()' "
        "or make -C poselib_b200/csrc).  There is no CPU fallback.")
_lib = C.CDLL(LIB_PATH)
_lib.plb_last_error.restype = C.c_char_p
_P = C.POINTER(C.c_double)


def lib():
    return _lib


def _check(rc):
    if rc != PLB_OK:
        raise PoseLibB200Error(rc, _lib.plb_last_error().decode())


def device_count():
    return _lib.plb_device_count()


def set_device(i):
    _check(_lib.plb_set_device(int(i)))


def set_mode(mode):
    _check(_lib.plb_set_mode({"exact": 0, "fast": 1}.get(mode, mode)))


def host_sample_table(n, k, ropt, iters):
    """First `iters` minimal samples of RandomSampler(n, k, opt) as the engine's host sampler draws them (no device)."""
    out = np.zeros((iters, k), dtype=np.uint32)
    _check(_lib.plb_host_sample_table(C.c_uint64(n), C.c_uint32(k), C.byref(ropt), C.c_uint64(iters),
                                      out.ctypes.data_as(C.POINTER(C.c_uint32))))
    return out


def device_sample_table(n, k, ropt, iters, round_size=4096, count=1):
    """The same table drawn by the engine's DEVICE sampler (k_sample): `count` samplers with seeds seed+j, `round_size`
    samples per launch (state carried across launches).  Returns (count, iters, k)."""
    out = np.zeros((count, iters, k), dtype=np.uint32)
    _check(_lib.plb_device_sample_table(C.c_uint64(n), C.c_uint32(k), C.byref(ropt), C.c_uint64(iters),
                                        C.c_uint64(round_size), C.c_uint32(count),
                                        out.ctypes.data_as(C.POINTER(C.c_uint32))))
    return out


def host_dynamic_max_iter(num_inliers, num_data, sample_sz, success_prob, mult, min_it, max_it):
    _lib.plb_host_dynamic_max_iter.restype = C.c_uint64
    return _lib.plb_host_dynamic_max_iter(C.c_uint64(num_inliers), C.c_uint64(num_data), C.c_uint32(sample_sz),
                                          C.c_double(success_prob), C.c_double(mult), C.c_uint64(min_it),
                                          C.c_uint64(max_it))


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_P)


def _w(weights, n):
    """PoseLib's per-residual weights for n points: used when there is one per point, else uniform (None), as in the
    reference (bundle.cc:107-111 etc.).  Returns (array kept alive by the caller, pointer or None)."""
    if weights is None:
        return None, None
    w = np.ascontiguousarray(weights, dtype=np.float64).reshape(-1)
    return (w, w.ctypes.data_as(_P)) if len(w) == n else (None, None)


def _init_model(kind, init):
    if kind in ("pnp", "relpose"):
        m = np.array([1, 0, 0, 0, 0, 0, 0] if init is None else init, dtype=np.float64)
    else:
        m0 = np.eye(3) if init is None else np.asarray(init, dtype=np.float64)
        m = np.ascontiguousarray(m0.T.reshape(-1)).copy()  # column-major
    return m


def _model_out(kind, m):
    return m if kind in ("pnp", "relpose") else m.reshape(3, 3).T.copy()


def ransac(kind, a, b, ropt, max_error, init=None, rfc=False):
    """ransac_pnp / ransac_relpose / ransac_fundamental / ransac_homography (robust/ransac.h).
    Points are calibrated / normalised; matrices are numpy [r,c].  Returns dict(model, inliers, stats, counters)."""
    n = len(a)
    aa, ap = _d(a)
    ba, bp = _d(b)
    mask = np.zeros(max(n, 1), dtype=np.int8)
    st, cn = RansacStats(), Counters()
    m = _init_model(kind, init)
    mp = m.ctypes.data_as(_P)
    mk = mask.ctypes.data_as(C.c_char_p)
    if kind == "pnp":
        rc = _lib.plb_ransac_pnp(ap, bp, C.c_size_t(n), C.byref(ropt), C.c_double(max_error), mp, mk, C.byref(st),
                                 C.byref(cn))
    elif kind == "relpose":
        rc = _lib.plb_ransac_relpose(ap, bp, C.c_size_t(n), C.byref(ropt), C.c_double(max_error), mp, mk,
                                     C.byref(st), C.byref(cn))
    elif kind == "fundamental":
        rc = _lib.plb_ransac_fundamental(ap, bp, C.c_size_t(n), C.byref(ropt), C.c_double(max_error), int(rfc), mp,
                                         mk, C.byref(st), C.byref(cn))
    else:
        rc = _lib.plb_ransac_homography(ap, bp, C.c_size_t(n), C.byref(ropt), C.c_double(max_error), mp, mk,
                                        C.byref(st), C.byref(cn))
    _check(rc)
    return {"model": _model_out(kind, m), "inliers": mask[:n], "stats": st.as_dict(), "counters": cn.as_dict()}


def ransac_relpose_cameras(x1, x2, cam1, cam2, ropt, max_error):
    """ransac_relpose with camera models (tangent Sampson error, ransac.cc:155-168); points in pixels."""
    n = len(x1)
    aa, ap = _d(x1)
    ba, bp = _d(x2)
    mask = np.zeros(max(n, 1), dtype=np.int8)
    st, cn = RansacStats(), Counters()
    m = _init_model("relpose", None)
    _check(_lib.plb_ransac_relpose_cameras(ap, bp, C.c_size_t(n), C.byref(cam1), C.byref(cam2), C.byref(ropt),
                                           C.c_double(max_error), m.ctypes.data_as(_P),
                                           mask.ctypes.data_as(C.c_char_p), C.byref(st), C.byref(cn)))
    return {"model": _model_out("relpose", m), "inliers": mask[:n], "stats": st.as_dict(), "counters": cn.as_dict()}


def refine_relpose_cameras(pose, x1, x2, cam1, cam2, bopt, weights=None):
    """refine_relpose(x1, x2, ImagePair*, opt) with fixed intrinsics (bundle.cc:237-247); weights: one per point, or
    None (uniform)."""
    n = len(x1)
    aa, ap = _d(x1)
    ba, bp = _d(x2)
    wa, wp = _w(weights, n)
    m = _init_model("relpose", pose)
    bs = np.zeros(3)
    _check(_lib.plb_refine_relpose_cameras_weighted(ap, bp, C.c_size_t(n), C.byref(cam1), C.byref(cam2),
                                                    m.ctypes.data_as(_P), C.byref(bopt), bs.ctypes.data_as(_P), wp))
    return _model_out("relpose", m), bs


def estimate(kind, a, b, ropt, bopt, max_error, cam1=None, cam2=None, init=None, rfc=False, tangent_sampson=False):
    """estimate_absolute_pose / estimate_relative_pose / estimate_fundamental / estimate_homography (robust.h)."""
    n = len(a)
    aa, ap = _d(a)
    ba, bp = _d(b)
    mask = np.zeros(max(n, 1), dtype=np.int8)
    st, cn = RansacStats(), Counters()
    m = _init_model(kind, init)
    mp = m.ctypes.data_as(_P)
    mk = mask.ctypes.data_as(C.c_char_p)
    c1 = cam1 if cam1 is not None else Camera("NULL", ())
    c2 = cam2 if cam2 is not None else Camera("NULL", ())
    if kind == "pnp":
        rc = _lib.plb_estimate_absolute_pose(ap, bp, C.c_size_t(n), C.byref(ropt), C.byref(bopt),
                                             C.c_double(max_error), C.byref(c1), mp, mk, C.byref(st), C.byref(cn))
    elif kind == "relpose":
        rc = _lib.plb_estimate_relative_pose(ap, bp, C.c_size_t(n), C.byref(c1), C.byref(c2), C.byref(ropt),
                                             C.byref(bopt), C.c_double(max_error), int(tangent_sampson), mp, mk,
                                             C.byref(st), C.byref(cn))
    elif kind == "fundamental":
        rc = _lib.plb_estimate_fundamental(ap, bp, C.c_size_t(n), C.byref(ropt), C.byref(bopt),
                                           C.c_double(max_error), int(rfc), mp, mk, C.byref(st), C.byref(cn))
    else:
        rc = _lib.plb_estimate_homography(ap, bp, C.c_size_t(n), C.byref(ropt), C.byref(bopt),
                                          C.c_double(max_error), mp, mk, C.byref(st), C.byref(cn))
    _check(rc)
    return {"model": _model_out(kind, m), "inliers": mask[:n], "stats": st.as_dict(), "counters": cn.as_dict()}


def _copy_camera(cam):
    return Camera(cam.model_id, tuple(cam.params), cam.width, cam.height)


def _camera_params(cam):
    return np.array(cam.params[:CAMERA_NUM_PARAMS[cam.model_id]], dtype=np.float64)


def estimate_image(x, X, cam, ropt, bopt, max_error, init=None):
    """estimate_absolute_pose with an Image* (robust.cc:36-126): bopt.refine_intrinsics selects camera parameters that
    the final bundle adjustment refines with the pose.  Returns dict(model, camera [model's parameters], inliers, stats,
    counters); `cam` is not modified."""
    n = len(x)
    aa, ap = _d(x)
    ba, bp = _d(X)
    mask = np.zeros(max(n, 1), dtype=np.int8)
    st, cn = RansacStats(), Counters()
    m = _init_model("pnp", init)
    c = _copy_camera(cam)
    _check(_lib.plb_estimate_absolute_pose_image(ap, bp, C.c_size_t(n), C.byref(ropt), C.byref(bopt),
                                                 C.c_double(max_error), C.byref(c), m.ctypes.data_as(_P),
                                                 mask.ctypes.data_as(C.c_char_p), C.byref(st), C.byref(cn)))
    return {"model": m, "camera": _camera_params(c), "inliers": mask[:n], "stats": st.as_dict(),
            "counters": cn.as_dict()}


def estimate_relative_pose_pair(x1, x2, cam1, cam2, ropt, bopt, max_error, tangent_sampson=True, init=None):
    """estimate_relative_pose with the cameras in/out: with tangent_sampson, bopt.refine_intrinsics selects camera
    parameters the final bundle adjustment refines with the pose.  Returns dict(model, camera1, camera2 [the models'
    parameters], inliers, stats, counters); cam1 / cam2 are not modified."""
    n = len(x1)
    aa, ap = _d(x1)
    ba, bp = _d(x2)
    mask = np.zeros(max(n, 1), dtype=np.int8)
    st, cn = RansacStats(), Counters()
    m = _init_model("relpose", init)
    c1, c2 = _copy_camera(cam1), _copy_camera(cam2)
    _check(_lib.plb_estimate_relative_pose_pair(ap, bp, C.c_size_t(n), C.byref(c1), C.byref(c2), C.byref(ropt),
                                                C.byref(bopt), C.c_double(max_error), int(tangent_sampson),
                                                m.ctypes.data_as(_P), mask.ctypes.data_as(C.c_char_p), C.byref(st),
                                                C.byref(cn)))
    return {"model": m, "camera1": _camera_params(c1), "camera2": _camera_params(c2), "inliers": mask[:n],
            "stats": st.as_dict(), "counters": cn.as_dict()}


def refine_image(pose, x, X, cam, bopt, weights=None):
    """bundle_adjust(x, X, Image*, opt, weights) (robust/bundle.h:47): points in the camera's pixel units,
    bopt.refine_intrinsics selects the camera parameters refined with the pose; weights: one per point, or None
    (uniform).  Returns (pose, camera parameters, [iterations, initial_cost, cost]); `cam` is not modified."""
    n = len(x)
    aa, ap = _d(x)
    ba, bp = _d(X)
    wa, wp = _w(weights, n)
    m = _init_model("pnp", pose)
    c = _copy_camera(cam)
    bs = np.zeros(3)
    _check(_lib.plb_bundle_adjust_image_weighted(ap, bp, C.c_size_t(n), m.ctypes.data_as(_P), C.byref(c),
                                                 C.byref(bopt), bs.ctypes.data_as(_P), wp))
    return m, _camera_params(c), bs


def refine_relpose_pair(pose, x1, x2, cam1, cam2, bopt, weights=None):
    """refine_relpose(x1, x2, ImagePair*, opt, weights) (bundle.cc:237-256): pixels as given, bopt.refine_intrinsics
    selects the parameters of each camera refined with the pose; weights: one per point, or None (uniform).  Returns
    (pose, camera 1 parameters, camera 2 parameters, [iterations, initial_cost, cost]); cam1 / cam2 are not modified."""
    n = len(x1)
    aa, ap = _d(x1)
    ba, bp = _d(x2)
    wa, wp = _w(weights, n)
    m = _init_model("relpose", pose)
    c1, c2 = _copy_camera(cam1), _copy_camera(cam2)
    bs = np.zeros(3)
    _check(_lib.plb_refine_relpose_pair_weighted(ap, bp, C.c_size_t(n), C.byref(c1), C.byref(c2), m.ctypes.data_as(_P),
                                                 C.byref(bopt), bs.ctypes.data_as(_P), wp))
    return m, _camera_params(c1), _camera_params(c2), bs


def refine(kind, model, a, b, bopt, weights=None):
    """bundle_adjust / refine_relpose / refine_fundamental / refine_homography (robust/bundle.h); weights: one per point,
    or None (uniform).  "pnp" ignores the weights, as the reference's calibrated bundle_adjust does (bundle.cc:84-92).
    Returns (model, [iterations, initial_cost, cost])."""
    n = len(a)
    aa, ap = _d(a)
    ba, bp = _d(b)
    m = _init_model(kind, model)
    bs = np.zeros(3)
    args = [ap, bp, C.c_size_t(n), m.ctypes.data_as(_P), C.byref(bopt), bs.ctypes.data_as(_P)]
    if kind == "pnp":
        _check(_lib.plb_bundle_adjust(*args))
    else:
        wa, wp = _w(weights, n)
        fn = {"relpose": _lib.plb_refine_relpose_weighted, "fundamental": _lib.plb_refine_fundamental_weighted,
              "homography": _lib.plb_refine_homography_weighted}[kind]
        _check(fn(*args, wp))
    return _model_out(kind, m), bs


# ---- solvers (batched; inputs [count, k, 3] unit bearings) -------------------------------------------
def _solver(fn, a, b, per_out, extra=()):
    aa, ap = _d(a)
    ba, bp = _d(b)
    count = aa.shape[0]
    out = np.zeros((count, per_out))
    n_out = np.zeros(count, dtype=np.int32)
    _check(fn(C.c_size_t(count), ap, bp, out.ctypes.data_as(_P), n_out.ctypes.data_as(C.POINTER(C.c_int32)), *extra))
    return out, n_out


def p3p_batch(x, X):
    out, n = _solver(_lib.plb_p3p_batch, x, X, 28)
    return out.reshape(-1, 4, 7), n


def p3p_lambdatwist_batch(x, X):
    out, n = _solver(_lib.plb_p3p_lambdatwist_batch, x, X, 28)
    return out.reshape(-1, 4, 7), n


def relpose_5pt_batch(x1, x2):
    out, n = _solver(_lib.plb_relpose_5pt_batch, x1, x2, 90)
    return out.reshape(-1, 10, 3, 3).transpose(0, 1, 3, 2), n  # column-major -> [r,c]


def relpose_5pt_poses_batch(x1, x2):
    out, n = _solver(_lib.plb_relpose_5pt_poses_batch, x1, x2, 280)
    return out.reshape(-1, 40, 7), n


def relpose_7pt_batch(x1, x2):
    out, n = _solver(_lib.plb_relpose_7pt_batch, x1, x2, 27)
    return out.reshape(-1, 3, 3, 3).transpose(0, 1, 3, 2), n


def homography_4pt_batch(x1, x2, check_cheirality=True):
    out, n = _solver(_lib.plb_homography_4pt_batch, x1, x2, 9, (C.c_int(int(check_cheirality)),))
    return out.reshape(-1, 3, 3).transpose(0, 2, 1), n


def essential_matrix_8pt_batch(x1, x2):
    """solvers/relpose_8pt.h essential_matrix_8pt for [count, n, 3] unit bearings (n >= 8) -> E [count, 3, 3] ([r,c])."""
    aa, ap = _d(x1)
    ba, bp = _d(x2)
    count, n = aa.shape[0], aa.shape[1]
    out = np.zeros((count, 9))
    _check(_lib.plb_essential_matrix_8pt_batch(C.c_size_t(count), C.c_size_t(n), ap, bp, out.ctypes.data_as(_P)))
    return out.reshape(-1, 3, 3).transpose(0, 2, 1)


def relpose_8pt_batch(x1, x2):
    """solvers/relpose_8pt.h relpose_8pt for [count, n, 3] unit bearings -> (poses [count, 4, 7], n_poses [count])."""
    aa, ap = _d(x1)
    ba, bp = _d(x2)
    count, n = aa.shape[0], aa.shape[1]
    out = np.zeros((count, 28))
    n_out = np.zeros(count, dtype=np.int32)
    _check(_lib.plb_relpose_8pt_batch(C.c_size_t(count), C.c_size_t(n), ap, bp, out.ctypes.data_as(_P),
                                      n_out.ctypes.data_as(C.POINTER(C.c_int32))))
    return out.reshape(-1, 4, 7), n_out


def resident_create(kind, a, b):
    """Uploads correspondences once and keeps them in HBM; returns a handle for ransac_batch(resident=...)."""
    aa, ap = _d(a)
    ba, bp = _d(b)
    h = _lib.plb_resident_create(KIND[kind], ap, bp, C.c_size_t(len(aa)))
    if h <= 0:
        _check(h)
    return h


def resident_free(h):
    _check(_lib.plb_resident_free(int(h)))


# ---- batch of problems -------------------------------------------------------------------------------
class Batch:
    """A batch of ransac_* problems marshalled ONCE into the C-ABI's plb_problem array: run() is then just the C call
    (plb_ransac_batch / plb_ransac_batch_multi), the same batch can be run again and again (bench.py, repeated
    estimation on fixed matches) without paying the Python marshalling per call.
    problems: list of dict(kind, a, b, ransac=RansacOpt, max_error, rfc=False, init=None) or dict(kind, resident, n, ...)."""

    def __init__(self, problems):
        self.count = count = len(problems)
        self.kinds = [p["kind"] for p in problems]
        self.arr = (Problem * count)()
        self.keep = []
        self._init = []
        for i, p in enumerate(problems):
            q = self.arr[i]
            if p.get("resident"):
                aa = ba = None
                npts = int(p["n"])
                q.resident = int(p["resident"])
            else:
                aa, ap = _d(p["a"])
                ba, bp = _d(p["b"])
                npts = len(aa)
                q.a, q.b = ap, bp
            mask = np.zeros(max(npts, 1), dtype=np.int8)
            self.keep.append((aa, ba, mask))
            q.kind = KIND[p["kind"]]
            q.real_focal_check = int(p.get("rfc", False))
            q.n = npts
            q.opt = p["ransac"]
            q.max_error = p["max_error"]
            m = _init_model(p["kind"], p.get("init"))
            self._init.append(m)
            for k in range(len(m)):
                q.model[k] = m[k]
            q.inliers = C.cast(mask.ctypes.data_as(C.POINTER(C.c_char)), C.c_char_p)
        self._raw = np.frombuffer(self.arr, dtype=np.uint8).reshape(count, C.sizeof(Problem))

    def run(self, streams=8, n_gpus=None):
        """n_gpus=None: plb_ransac_batch on the current device; an int: plb_ransac_batch_multi (0 = all devices)."""
        for i, m in enumerate(self._init):  # in/out models: restore the start models of a re-run (cheap: <= 9 doubles each)
            if len(m) and self.arr[i].opt.score_initial_model:
                for k in range(len(m)):
                    self.arr[i].model[k] = m[k]
        if n_gpus is None:
            _check(_lib.plb_ransac_batch(self.arr, C.c_size_t(self.count), int(streams)))
        else:
            _check(_lib.plb_ransac_batch_multi(self.arr, C.c_size_t(self.count), int(n_gpus), int(streams)))
        return self

    def _block(self, field, ctype):
        off = getattr(Problem, field).offset
        return self._raw[:, off:off + C.sizeof(ctype)]

    def counter_sums(self):
        """Sum of every plb_counters field over the batch (vectorised over the raw array)."""
        blk = self._block("counters", Counters)
        out = {}
        for name, ct in Counters._fields_:
            o = getattr(Counters, name).offset
            col = np.ascontiguousarray(blk[:, o:o + 8]).view(np.float64 if ct is C.c_double else np.uint64)
            out[name] = float(col.sum()) if ct is C.c_double else int(col.sum())
        return out

    def records(self, indices):
        """Fixed-size result records [index, iterations, refinements, num_inliers, model_score, model(9)] (sharding.pack_results)."""
        st = np.ascontiguousarray(self._block("stats", RansacStats))
        u = st.view(np.uint64).reshape(self.count, -1)
        f = st.view(np.float64).reshape(self.count, -1)
        mo = getattr(Problem, "model").offset
        model = np.ascontiguousarray(self._raw[:, mo:mo + 72]).view(np.float64).reshape(self.count, 9)
        rec = np.zeros((self.count, 14))
        rec[:, 0] = np.asarray(indices, dtype=np.float64)
        rec[:, 1], rec[:, 2], rec[:, 3], rec[:, 4] = u[:, 1], u[:, 0], u[:, 2], f[:, 4]
        rec[:, 5:] = model
        return rec

    def results(self):
        out = []
        for i, kind in enumerate(self.kinds):
            q = self.arr[i]
            m = np.array(q.model[:7] if kind in ("pnp", "relpose") else q.model[:9], dtype=np.float64)
            out.append({"model": _model_out(kind, m), "inliers": self.keep[i][2][:q.n].copy(), "stats": q.stats.as_dict(),
                        "counters": q.counters.as_dict(), "status": q.status})
        return out


def ransac_batch(problems, streams=8, n_gpus=None):
    """problems: list of dict(kind, a, b, ransac=RansacOpt, max_error, rfc=False, init=None).
    n_gpus=None: plb_ransac_batch on the current device; an int: plb_ransac_batch_multi over that many devices of this
    process (0 = all).  Returns list of dict(model, inliers, stats, counters)."""
    return Batch(problems).run(streams, n_gpus).results()


def estimate_batch(problems, streams=8, n_gpus=-1):
    """Batch form of estimate() (plb_estimate_batch).  problems: list of dict(kind, a, b, ransac=RansacOpt, bundle=BundleOpt,
    max_error [pixels], cam1=None, cam2=None, rfc=False, tangent_sampson=False, init=None).  n_gpus: -1 current device,
    0 all devices, k the first k.  Returns list of dict(model, inliers, stats, counters, status)."""
    count = len(problems)
    arr = (EstimateProblem * count)()
    keep = []
    for i, p in enumerate(problems):
        q = arr[i]
        aa, ap = _d(p["a"])
        ba, bp = _d(p["b"])
        npts = len(aa)
        mask = np.zeros(max(npts, 1), dtype=np.int8)
        keep.append((aa, ba, mask))
        _fill_estimate_problem(q, p, npts)
        q.a, q.b = ap, bp
        q.inliers = C.cast(mask.ctypes.data_as(C.POINTER(C.c_char)), C.c_char_p)
    _check(_lib.plb_estimate_batch(arr, C.c_size_t(count), int(n_gpus), int(streams)))
    return _estimate_results(arr, problems, [k[2][:q.n].copy() for k, q in zip(keep, arr)])


def _fill_estimate_problem(q, p, npts):
    """Everything of one plb_estimate_problem but its point and mask pointers."""
    q.kind = KIND[p["kind"]]
    q.real_focal_check = int(p.get("rfc", False))
    q.tangent_sampson = int(p.get("tangent_sampson", False))
    q.n = npts
    q.camera1 = p.get("cam1") or Camera("NULL", ())
    q.camera2 = p.get("cam2") or Camera("NULL", ())
    q.ransac = p["ransac"]
    q.bundle = p["bundle"]
    q.max_error = p["max_error"]
    m = _init_model(p["kind"], p.get("init"))
    for k in range(len(m)):
        q.model[k] = m[k]


def _estimate_results(arr, problems, masks):
    out = []
    for i, p in enumerate(problems):
        q = arr[i]
        kind = p["kind"]
        m = np.array(q.model[:7] if kind in ("pnp", "relpose") else q.model[:9], dtype=np.float64)
        out.append({"model": _model_out(kind, m), "inliers": masks[i], "stats": q.stats.as_dict(),
                    "counters": q.counters.as_dict(), "status": q.status, "camera1": _camera_params(q.camera1)})
    return out


def _device_form(fn, what, points, models=(), stream=None):
    """The checks and set-up of a device form: `points` (a, b and weights, named `what`) must be CUDA torch tensors of
    one device and one dtype, float32 or float64, and `models` CUDA float64 tensors on the same device.  Selects that
    device and returns (device, PLB_DTYPE_*, `stream` as a torch.cuda.Stream [None: the device's current stream]), or
    None when there are no points."""
    import torch
    if not all(isinstance(t, torch.Tensor) and t.is_cuda for t in [*points, *models]):
        raise TypeError(f"{fn}: {what}{' and models' if models else ''} must be CUDA torch tensors")
    if not points:
        return None
    dev, dt = points[0].device, points[0].dtype
    if any(t.device != dev for t in [*points, *models]):
        raise ValueError(f"{fn}: every tensor must be on {dev} (shard the batch by device)")
    dtypes = {torch.float64: DTYPE_F64, torch.float32: DTYPE_F32}
    if dt not in dtypes or any(t.dtype != dt for t in points):
        raise TypeError(f"{fn}: {what} must share one dtype, torch.float32 or torch.float64")
    if any(t.dtype != torch.float64 for t in models):
        raise TypeError(f"{fn}: models must be torch.float64")
    set_device(dev.index)
    if stream is None:
        stream = torch.cuda.current_stream(dev)
    elif not isinstance(stream, torch.cuda.Stream):
        stream = torch.cuda.ExternalStream(int(stream), device=dev)
    return dev, dtypes[dt], stream


def _device_points(fn, i, p, b_dim):
    """Problem i's a [n,2] and b [n,b_dim] as contiguous tensors."""
    a, b = p["a"].contiguous(), p["b"].contiguous()
    n = a.shape[0]
    if tuple(a.shape) != (n, 2) or tuple(b.shape) != (n, b_dim):
        raise ValueError(f"{fn}: problem {i}: a must be [n,2] and b [n,{b_dim}], got {tuple(a.shape)} and "
                         f"{tuple(b.shape)}")
    return a, b


def estimate_batch_device(problems, streams=8, stream=None):
    """estimate_batch (n_gpus=-1) on correspondences that are already on the GPU (plb_estimate_batch_device).
    problems: the dicts estimate_batch takes, with a / b as CUDA torch tensors [n,2] / [n,3] ([n,2] for the 2D-2D kinds),
    all on one device and of one dtype, float32 or float64.  The call runs on that device and reads the inputs after the
    work queued on `stream` (a torch.cuda.Stream or a cudaStream_t handle; default: the device's current stream).
    Returns the dicts of estimate_batch, with `inliers` a CUDA torch.bool tensor of length n (the masks of one call are
    views of one allocation)."""
    import torch
    form = _device_form("estimate_batch_device", "a and b", [t for p in problems for t in (p["a"], p["b"])],
                        stream=stream)
    if form is None:
        return []
    dev, dtype, stream = form
    count = len(problems)
    arr = (EstimateProblem * count)()
    keep = []
    sizes = [p["a"].shape[0] for p in problems]
    with torch.cuda.stream(stream):  # the copies and masks below are ordered before the call's reads and writes
        # one zeroed allocation for the whole batch (one launch, not one per problem); problem i's mask is a view of it
        masks = list(torch.zeros(sum(sizes), dtype=torch.bool, device=dev).split(sizes))
        for i, p in enumerate(problems):
            q = arr[i]
            a, b = _device_points("estimate_batch_device", i, p, 3 if p["kind"] == "pnp" else 2)
            npts = sizes[i]
            keep.append((a, b))
            _fill_estimate_problem(q, p, npts)
            q.a, q.b = C.cast(C.c_void_p(a.data_ptr()), _P), C.cast(C.c_void_p(b.data_ptr()), _P)
            q.inliers = C.cast(C.c_void_p(masks[i].data_ptr() if npts else None), C.c_char_p)
    _check(_lib.plb_estimate_batch_device(arr, C.c_size_t(count), dtype, C.c_void_p(stream.cuda_stream or None),
                                          int(streams)))
    return _estimate_results(arr, problems, masks)


# ---- batch of refiner problems (plb_refine_batch) ------------------------------------------------------------
def _refine_kind(refiner):
    """The model layout of a refiner: a pose, or a 3x3 matrix for "fundamental" / "homography"."""
    return refiner if refiner in ("fundamental", "homography") else "pnp"


def _fill_refine_problem(q, p, npts):
    """Everything of one plb_refine_problem but its point and weight pointers."""
    q.refiner = REFINER[p["refiner"]]
    q.n = npts
    q.camera1 = p.get("cam1") or Camera("NULL", ())
    q.camera2 = p.get("cam2") or Camera("NULL", ())
    q.bundle = p["bundle"]
    m = _init_model(_refine_kind(p["refiner"]), p.get("model"))
    for k in range(len(m)):
        q.model[k] = m[k]


def _refine_results(arr, problems):
    out = []
    for i, p in enumerate(problems):
        q = arr[i]
        kind = _refine_kind(p["refiner"])
        m = np.array(q.model[:7] if kind == "pnp" else q.model[:9], dtype=np.float64)
        out.append({"model": _model_out(kind, m), "bundle_stats": np.array(q.bundle_stats[:3]), "status": q.status,
                    "camera1": _camera_params(q.camera1), "camera2": _camera_params(q.camera2)})
    return out


def refine_batch(problems, n_gpus=-1, streams=8):
    """Batch form of refine / refine_image / refine_relpose_cameras / refine_relpose_pair (plb_refine_batch): each result
    equals its single call bit for bit.  problems: list of dict(refiner [a REFINER key], a, b, bundle=BundleOpt,
    model=None [start pose, or 3x3 matrix [r,c]], weights=None [one per point, else uniform], cam1=None, cam2=None).
    n_gpus: -1 current device, 0 all devices, k the first k.  Returns list of dict(model, bundle_stats [iterations,
    initial_cost, cost], camera1, camera2 [the models' parameters], status); the given cameras are not modified."""
    count = len(problems)
    arr = (RefineProblem * count)()
    keep = []
    for i, p in enumerate(problems):
        q = arr[i]
        aa, ap = _d(p["a"])
        ba, bp = _d(p["b"])
        wa, wp = _w(p.get("weights"), len(aa))
        keep.append((aa, ba, wa))
        _fill_refine_problem(q, p, len(aa))
        q.a, q.b, q.weights = ap, bp, wp
    _check(_lib.plb_refine_batch(arr, C.c_size_t(count), int(n_gpus), int(streams)))
    return _refine_results(arr, problems)


def refine_batch_device(problems, stream=None, streams=8):
    """refine_batch (n_gpus=-1) on points and weights that are already on the GPU (plb_refine_batch_device).
    problems: the dicts refine_batch takes, with a / b / weights as CUDA torch tensors ([n,2] / [n,3] / [n]), all on one
    device and of one dtype, float32 or float64; weights with other than n elements mean uniform weights.  The call runs
    on that device and reads the inputs after the work queued on `stream` (a torch.cuda.Stream or a cudaStream_t handle;
    default: the device's current stream).  Returns the dicts of refine_batch."""
    import torch
    form = _device_form("refine_batch_device", "a, b and weights",
                        [t for p in problems for t in (p["a"], p["b"], p.get("weights")) if t is not None], stream=stream)
    if form is None:
        return []
    _, dtype, stream = form
    count = len(problems)
    arr = (RefineProblem * count)()
    keep = []
    ptr = lambda t: C.cast(C.c_void_p(t.data_ptr() if t is not None else None), _P)
    with torch.cuda.stream(stream):  # any copy .contiguous() makes is ordered before the call's reads
        for i, p in enumerate(problems):
            q = arr[i]
            a, b = _device_points("refine_batch_device", i, p, 3 if p["refiner"] in ("bundle", "bundle_image") else 2)
            npts = a.shape[0]
            w = p.get("weights")
            w = w.contiguous().reshape(-1) if w is not None and w.numel() == npts else None
            keep.append((a, b, w))
            _fill_refine_problem(q, p, npts)
            q.a, q.b, q.weights = ptr(a), ptr(b), ptr(w)
    _check(_lib.plb_refine_batch_device(arr, C.c_size_t(count), dtype, C.c_void_p(stream.cuda_stream or None),
                                        int(streams)))
    return _refine_results(arr, problems)


# ---- scores and inlier masks of given models (plb_score_batch) -------------------------------------------------
def _score_models(kind, models):
    """Models of one problem as the C-ABI reads them: [m,7] poses, or [m,3,3] matrices [r,c] -> column-major rows."""
    m = np.asarray(models, dtype=np.float64)
    if kind in ("pnp", "relpose"):
        return np.ascontiguousarray(m.reshape(-1, 7))
    return np.ascontiguousarray(m.reshape(-1, 3, 3).transpose(0, 2, 1).reshape(-1, 9))


def _fill_score_problem(q, p, npts, m):
    """Everything of one plb_score_problem but its pointers."""
    q.kind = KIND[p["kind"]]
    q.tangent_sampson = int(p.get("tangent_sampson", False))
    q.n = npts
    q.m = m
    q.camera1 = p.get("cam1") or Camera("NULL", ())
    q.camera2 = p.get("cam2") or Camera("NULL", ())
    q.sq_threshold = p["sq_threshold"]


def score_batch(problems, n_gpus=-1, streams=8):
    """MSAC scores, inlier counts and (optionally) inlier masks of given models (plb_score_batch; robust/utils.h).
    problems: list of dict(kind, a, b, models [[m,7] poses or [m,3,3] matrices [r,c]], sq_threshold [squared, in the
    points' units], tangent_sampson=False with cam1 / cam2 [pixels], inliers=False [True: return the masks]).
    n_gpus: -1 current device, 0 all devices, k the first k.  Returns list of dict(scores [m] float64, num_inliers [m]
    int64, inliers [m,n] bool or None, status)."""
    count = len(problems)
    arr = (ScoreProblem * count)()
    out = []
    keep = []
    for i, p in enumerate(problems):
        q = arr[i]
        aa, ap = _d(p["a"])
        ba, bp = _d(p["b"])
        mo = _score_models(p["kind"], p["models"])
        m, npts = len(mo), len(aa)
        r = {"scores": np.zeros(m), "num_inliers": np.zeros(m, dtype=np.int64),
             "inliers": np.zeros((m, npts), dtype=np.bool_) if p.get("inliers") else None}
        keep.append((aa, ba, mo))
        out.append(r)
        _fill_score_problem(q, p, npts, m)
        q.a, q.b, q.models = ap, bp, mo.ctypes.data_as(_P)
        q.scores = r["scores"].ctypes.data_as(_P)
        q.num_inliers = r["num_inliers"].ctypes.data_as(C.POINTER(C.c_int64))
        if r["inliers"] is not None:
            q.inliers = C.cast(r["inliers"].ctypes.data_as(C.POINTER(C.c_char)), C.c_char_p)
    _check(_lib.plb_score_batch(arr, C.c_size_t(count), int(n_gpus), int(streams)))
    for r, q in zip(out, arr):
        r["status"] = q.status
    return out


def score_batch_device(problems, stream=None, streams=8):
    """score_batch (n_gpus=-1) with everything on the GPU (plb_score_batch_device).  problems: the dicts score_batch
    takes, with a / b as CUDA torch tensors ([n,2] / [n,3] or [n,2]) of one device and one dtype, float32 or float64, and
    models a CUDA float64 tensor [m,7] or [m,3,3] ([r,c]).  The call runs on that device and reads the inputs after the
    work queued on `stream` (a torch.cuda.Stream or a cudaStream_t handle; default: the device's current stream).
    Returns the dicts of score_batch with CUDA tensors: scores (float64), num_inliers (int64) and inliers (bool [m,n] or
    None; the masks of one call are views of one zeroed allocation)."""
    import torch
    form = _device_form("score_batch_device", "a and b", [t for p in problems for t in (p["a"], p["b"])],
                        [p["models"] for p in problems], stream)
    if form is None:
        return []
    dev, dtype, stream = form
    count = len(problems)
    arr = (ScoreProblem * count)()
    keep = []
    out = []
    ptr = lambda t: C.cast(C.c_void_p(t.data_ptr() if t is not None and t.numel() else None), _P)
    with torch.cuda.stream(stream):  # the copies and outputs below are ordered before the call's reads and writes
        mods = []
        for i, p in enumerate(problems):
            msz = 7 if p["kind"] in ("pnp", "relpose") else 9
            mo = p["models"].reshape(-1, msz) if msz == 7 else p["models"].reshape(-1, 3, 3).transpose(1, 2).reshape(-1, 9)
            mods.append(mo.contiguous())
        ms = [len(mo) for mo in mods]
        ns = [p["a"].shape[0] for p in problems]
        scores = list(torch.zeros(sum(ms), dtype=torch.float64, device=dev).split(ms))
        counts = list(torch.zeros(sum(ms), dtype=torch.int64, device=dev).split(ms))
        want = [bool(p.get("inliers")) for p in problems]
        sizes = [ms[i] * ns[i] if want[i] else 0 for i in range(count)]
        flat = torch.zeros(sum(sizes), dtype=torch.bool, device=dev).split(sizes)
        for i, p in enumerate(problems):
            q = arr[i]
            a, b = _device_points("score_batch_device", i, p, 3 if p["kind"] == "pnp" else 2)
            npts = ns[i]
            mask = flat[i].view(ms[i], npts) if want[i] else None
            keep.append((a, b))
            _fill_score_problem(q, p, npts, ms[i])
            q.a, q.b, q.models, q.scores = ptr(a), ptr(b), ptr(mods[i]), ptr(scores[i])
            q.num_inliers = C.cast(C.c_void_p(counts[i].data_ptr() if ms[i] else None), C.POINTER(C.c_int64))
            q.inliers = C.cast(C.c_void_p(mask.data_ptr() if mask is not None and mask.numel() else None), C.c_char_p)
            out.append({"scores": scores[i], "num_inliers": counts[i], "inliers": mask})
    _check(_lib.plb_score_batch_device(arr, C.c_size_t(count), dtype, C.c_void_p(stream.cuda_stream or None),
                                       int(streams)))
    for r, q in zip(out, arr):
        r["status"] = q.status
    return out


# ---- hypotheses of caller-drawn minimal samples (plb_generate_batch) ---------------------------------------------
def _fill_generate_problem(q, p, npts, s):
    """Everything of one plb_generate_problem but its pointers."""
    q.kind = KIND[p["kind"]]
    q.tangent_sampson = int(p.get("tangent_sampson", False))
    q.real_focal_check = int(p.get("rfc", False))
    q.n = npts
    q.s = s
    q.camera1 = p.get("cam1") or Camera("NULL", ())
    q.camera2 = p.get("cam2") or Camera("NULL", ())
    q.sq_threshold = p["sq_threshold"]


def _generate_models_out(kind, models):
    """[s, M, 7] poses as they are; [s, M, 9] column-major matrices -> [s, M, 3, 3] [r,c] (a view for torch tensors)."""
    if kind in ("pnp", "relpose"):
        return models
    return models.reshape(*models.shape[:2], 3, 3).swapaxes(-1, -2)


def generate_batch(problems, n_gpus=-1, streams=8):
    """Models and MSAC records of caller-drawn minimal samples (plb_generate_batch): each estimator's generate_models,
    then score_model of every model.  problems: list of dict(kind, a, b, samples [s,k] int indices into [0, n),
    sq_threshold [squared, in the points' units], rfc=False [fundamental], tangent_sampson=False with cam1 / cam2
    [pixels]).  n_gpus: -1 current device, 0 all devices, k the first k.  Returns list of dict(n_models [s] int32,
    models [s,M,7] poses or [s,M,3,3] matrices [r,c], scores [s,M] float64, num_inliers [s,M] int64, status); slots past
    n_models[j] keep the NaN / -1 they start with."""
    count = len(problems)
    arr = (GenerateProblem * count)()
    out = []
    keep = []
    for i, p in enumerate(problems):
        q = arr[i]
        kind, k, M = p["kind"], GENERATE_K[p["kind"]], GENERATE_M[p["kind"]]
        aa, ap = _d(p["a"])
        ba, bp = _d(p["b"])
        smp = np.ascontiguousarray(np.asarray(p["samples"], dtype=np.int32).reshape(-1, k))
        s = len(smp)
        msz = 7 if kind in ("pnp", "relpose") else 9
        r = {"n_models": np.zeros(s, dtype=np.int32), "models": np.full((s, M, msz), np.nan),
             "scores": np.full((s, M), np.nan), "num_inliers": np.full((s, M), -1, dtype=np.int64)}
        keep.append((aa, ba, smp))
        out.append(r)
        _fill_generate_problem(q, p, len(aa), s)
        q.a, q.b, q.samples = ap, bp, smp.ctypes.data_as(C.POINTER(C.c_int32))
        q.n_models = r["n_models"].ctypes.data_as(C.POINTER(C.c_int32))
        q.models, q.scores = r["models"].ctypes.data_as(_P), r["scores"].ctypes.data_as(_P)
        q.num_inliers = r["num_inliers"].ctypes.data_as(C.POINTER(C.c_int64))
    _check(_lib.plb_generate_batch(arr, C.c_size_t(count), int(n_gpus), int(streams)))
    for p, r, q in zip(problems, out, arr):
        r["models"] = _generate_models_out(p["kind"], r["models"])
        r["status"] = q.status
    return out


def generate_batch_device(problems, stream=None, streams=8):
    """generate_batch (n_gpus=-1) with everything on the GPU (plb_generate_batch_device).  problems: the dicts
    generate_batch takes, with a / b as CUDA torch tensors ([n,2] / [n,3] or [n,2]) of one device and one dtype, float32
    or float64, and samples a CUDA torch.int32 tensor [s,k] on the same device.  The call runs on that device and reads
    the inputs after the work queued on `stream` (a torch.cuda.Stream or a cudaStream_t handle; default: the device's
    current stream).  Returns the dicts of generate_batch with CUDA tensors (models a view [s,M,3,3] [r,c] for the
    matrix kinds); the outputs of one call are views of one allocation per field."""
    import torch
    form = _device_form("generate_batch_device", "a and b", [t for p in problems for t in (p["a"], p["b"])],
                        stream=stream)
    if form is None:
        return []
    dev, dtype, stream = form
    for i, p in enumerate(problems):
        smp = p["samples"]
        if not (isinstance(smp, torch.Tensor) and smp.is_cuda and smp.device == dev and smp.dtype == torch.int32):
            raise TypeError(f"generate_batch_device: problem {i}: samples must be a torch.int32 tensor on {dev}")
    count = len(problems)
    arr = (GenerateProblem * count)()
    keep = []
    out = []
    ptr = lambda t, ct=_P: C.cast(C.c_void_p(t.data_ptr() if t.numel() else None), ct)
    with torch.cuda.stream(stream):  # the copies and outputs below are ordered before the call's reads and writes
        smps = [p["samples"].reshape(-1, GENERATE_K[p["kind"]]).contiguous() for p in problems]
        ss = [len(t) for t in smps]
        Ms = [GENERATE_M[p["kind"]] for p in problems]
        mszs = [7 if p["kind"] in ("pnp", "relpose") else 9 for p in problems]
        slots = [s * M for s, M in zip(ss, Ms)]
        n_models = torch.zeros(sum(ss), dtype=torch.int32, device=dev).split(ss)
        models = torch.full((sum(sl * m for sl, m in zip(slots, mszs)),), float("nan"), dtype=torch.float64,
                            device=dev).split([sl * m for sl, m in zip(slots, mszs)])
        scores = torch.full((sum(slots),), float("nan"), dtype=torch.float64, device=dev).split(slots)
        counts = torch.full((sum(slots),), -1, dtype=torch.int64, device=dev).split(slots)
        for i, p in enumerate(problems):
            q = arr[i]
            a, b = _device_points("generate_batch_device", i, p, 3 if p["kind"] == "pnp" else 2)
            keep.append((a, b, smps[i]))
            _fill_generate_problem(q, p, a.shape[0], ss[i])
            q.a, q.b, q.samples = ptr(a), ptr(b), ptr(smps[i], C.POINTER(C.c_int32))
            q.n_models, q.models = ptr(n_models[i], C.POINTER(C.c_int32)), ptr(models[i])
            q.scores, q.num_inliers = ptr(scores[i]), ptr(counts[i], C.POINTER(C.c_int64))
            out.append({"n_models": n_models[i], "models": _generate_models_out(p["kind"], models[i].view(ss[i], Ms[i], mszs[i])),
                        "scores": scores[i].view(ss[i], Ms[i]), "num_inliers": counts[i].view(ss[i], Ms[i])})
    _check(_lib.plb_generate_batch_device(arr, C.c_size_t(count), dtype, C.c_void_p(stream.cuda_stream or None),
                                          int(streams)))
    for r, q in zip(out, arr):
        r["status"] = q.status
    return out


# ---- the camera functions over many points (plb_camera_batch) ----------------------------------------------------
def _camera_shapes(op, cam):
    """Row widths of one camera problem: input, output, and the Jacobians' (rows, columns) as the C-ABI stores them
    column-major per point."""
    P = CAMERA_NUM_PARAMS.get(int(cam.model_id), 0)
    if op == "project":
        return 3, 2, (2, 3), (2, P)
    return 2, 3 if op == "unproject" else 2, (3, 2), (3, P)


def _camera_mats(m, n, rc):
    """n column-major rows x cols matrices -> [n, rows, cols] [r,c] (a view)."""
    return m.reshape(n, rc[1], rc[0]).swapaxes(-1, -2)


def camera_batch(problems, n_gpus=-1, streams=8):
    """PoseLib's Camera functions over many points of many cameras (plb_camera_batch).  problems: list of dict(op [a
    CAMOP key], cam [Camera], x [n,3] camera-frame points (project) or [n,2] pixels (unproject, unproject_2d), jac=False,
    jac_params=False).  project / unproject with jac or jac_params are project_with_jac / unproject_with_jac.
    n_gpus: -1 current device, 0 all devices, k the first k.  Returns list of dict(out [n,2] / [n,3], jac [n,2,3] /
    [n,3,2] or None, jac_params [n,2,P] / [n,3,P] or None, all [r,c], status)."""
    count = len(problems)
    arr = (CameraProblem * count)()
    out = []
    keep = []
    for i, p in enumerate(problems):
        q = arr[i]
        op, cam = p["op"], p["cam"]
        iw, ow, jrc, prc = _camera_shapes(op, cam)
        xa = np.ascontiguousarray(np.asarray(p["x"], dtype=np.float64).reshape(-1, iw))
        n = len(xa)
        r = {"out": np.zeros((n, ow)),
             "jac": np.zeros(n * 6) if p.get("jac") else None,
             "jac_params": np.zeros(n * prc[0] * prc[1]) if p.get("jac_params") else None}
        keep.append(xa)
        out.append(r)
        q.op, q.n, q.camera = CAMOP.get(op, -1) if isinstance(op, str) else int(op), n, cam
        q.in_, q.out = xa.ctypes.data_as(_P), r["out"].ctypes.data_as(_P)
        q.jac = r["jac"].ctypes.data_as(_P) if r["jac"] is not None else None
        q.jac_params = r["jac_params"].ctypes.data_as(_P) if r["jac_params"] is not None else None
    _check(_lib.plb_camera_batch(arr, C.c_size_t(count), int(n_gpus), int(streams)))
    for p, r, q in zip(problems, out, arr):
        _, _, jrc, prc = _camera_shapes(p["op"], p["cam"])
        n = len(r["out"])
        if r["jac"] is not None:
            r["jac"] = _camera_mats(r["jac"], n, jrc)
        if r["jac_params"] is not None:
            r["jac_params"] = _camera_mats(r["jac_params"], n, prc)
        r["status"] = q.status
    return out


def camera_batch_device(problems, stream=None, streams=8):
    """camera_batch (n_gpus=-1) with everything on the GPU (plb_camera_batch_device).  problems: the dicts camera_batch
    takes, with x a CUDA torch tensor, all of one device and one dtype, float32 or float64.  The call runs on that device
    and reads the inputs after the work queued on `stream` (a torch.cuda.Stream or a cudaStream_t handle; default: the
    device's current stream).  Returns the dicts of camera_batch with CUDA float64 tensors (the outputs of one call are
    views of one allocation per field)."""
    import torch
    form = _device_form("camera_batch_device", "x", [p["x"] for p in problems], stream=stream)
    if form is None:
        return []
    dev, dtype, stream = form
    count = len(problems)
    arr = (CameraProblem * count)()
    keep = []
    out = []
    ptr = lambda t: C.cast(C.c_void_p(t.data_ptr() if t is not None and t.numel() else None), _P)
    with torch.cuda.stream(stream):  # the copies and outputs below are ordered before the call's reads and writes
        shapes = [_camera_shapes(p["op"], p["cam"]) for p in problems]
        xs = [p["x"].reshape(-1, sh[0]).contiguous() for p, sh in zip(problems, shapes)]
        ns = [len(x) for x in xs]
        outs = torch.zeros(sum(n * sh[1] for n, sh in zip(ns, shapes)), dtype=torch.float64, device=dev).split(
            [n * sh[1] for n, sh in zip(ns, shapes)])
        jsz = [n * 6 if p.get("jac") else 0 for n, p in zip(ns, problems)]
        psz = [n * sh[3][0] * sh[3][1] if p.get("jac_params") else 0 for n, sh, p in zip(ns, shapes, problems)]
        jacs = torch.zeros(sum(jsz), dtype=torch.float64, device=dev).split(jsz)
        jps = torch.zeros(sum(psz), dtype=torch.float64, device=dev).split(psz)
        for i, p in enumerate(problems):
            q = arr[i]
            op, n, (iw, ow, jrc, prc) = p["op"], ns[i], shapes[i]
            keep.append(xs[i])
            q.op, q.n, q.camera = CAMOP.get(op, -1) if isinstance(op, str) else int(op), n, p["cam"]
            q.in_, q.out = ptr(xs[i]), ptr(outs[i])
            # a requested Jacobian with P = 0 (the NULL camera) still passes a pointer, as the host form does
            q.jac = ptr(jacs[i]) if p.get("jac") else None
            q.jac_params = C.cast(C.c_void_p(jps[i].data_ptr() or None), _P) if p.get("jac_params") else None
            out.append({"out": outs[i].view(n, ow),
                        "jac": _camera_mats(jacs[i], n, jrc) if p.get("jac") else None,
                        "jac_params": _camera_mats(jps[i], n, prc) if p.get("jac_params") else None})
    _check(_lib.plb_camera_batch_device(arr, C.c_size_t(count), dtype, C.c_void_p(stream.cuda_stream or None),
                                        int(streams)))
    for r, q in zip(out, arr):
        r["status"] = q.status
    return out
