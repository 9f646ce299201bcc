"""`poselib`-compatible Python call surface for the CUDA path (SURVEY.md §8f row N4).

Mirrors the signatures, option dictionaries and `(model, info)` returns of the reference's pybind module
(/root/reference/pybind/bindings/estimators/{absolute_pose.cc:317-330, relative_pose.cc:405-463, homography.cc:75-77},
pybind/bindings/solvers.cc:305,341,349 and pybind/helpers.h:31-170,237-253) for the functions on the hot path, so a
script written against `import poselib` runs with `import poselib_b200.pyapi as poselib` for them.  Everything goes
through the C-ABI (`cabi.py`); there is no Python compute path.

    pose, info = estimate_relative_pose(x1, x2, cam1, cam2, {"max_error": 1.0, "ransac": {"seed": 0}})
    info -> {"refinements", "iterations", "num_inliers", "inlier_ratio", "model_score", "inliers": [bool]}
"""
import numpy as np

from . import cabi

__all__ = ["Camera", "CameraPose", "Image", "estimate_absolute_pose", "estimate_relative_pose", "estimate_fundamental",
           "estimate_homography", "p3p", "p3p_lambdatwist", "relpose_5pt", "essential_matrix_5pt", "relpose_7pt", "homography_4pt"]

_CAMERA_IDS = dict(cabi.CAMERA)
# the reference's other models (camera_models.h): a Camera can hold them, its functions raise NYI on them
_OTHER_CAMERA_IDS = {"OPENCV_FISHEYE": 5, "FULL_OPENCV": 6, "FOV": 7, "THIN_PRISM_FISHEYE": 10,
                     "RAD_TAN_THIN_PRISM_FISHEYE": 11, "RADIAL_1D": 99, "SPHERICAL": 100}
_CAMERA_NAMES = {v: k for k, v in {**_CAMERA_IDS, **_OTHER_CAMERA_IDS}.items()}
# focal lengths and principal-point coordinates at the front of each model's parameters (camera.cuh cam_layout)
_CAMERA_FOCALS = {-1: (0, 0), 0: (1, 2), 1: (2, 2), 2: (1, 2), 3: (1, 2), 4: (2, 2), 8: (1, 2), 9: (1, 2), 101: (2, 2),
                  102: (1, 2)}


class CameraPose:
    """camera_pose.h:40-68 — q = (w, x, y, z), t."""

    def __init__(self, q=(1.0, 0.0, 0.0, 0.0), t=(0.0, 0.0, 0.0)):
        self.q = np.asarray(q, dtype=np.float64).copy()
        self.t = np.asarray(t, dtype=np.float64).copy()

    @property
    def R(self):
        w, x, y, z = self.q
        return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                         [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                         [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])

    @property
    def Rt(self):
        return np.c_[self.R, self.t]

    def __repr__(self):
        return f"CameraPose(q={self.q.tolist()}, t={self.t.tolist()})"


class Camera:
    """poselib.Camera (pybind/bindings/types.cc:64-113): Camera(), Camera(model_name, params, width, height) or
    Camera(dict), with model_id, width, height, params, model_name(), todict() and the vector forms of project,
    project_with_jac and unproject, evaluated on the device (cabi.camera_batch)."""

    def __init__(self, *args):
        if len(args) == 1 and isinstance(args[0], dict):  # camera_from_dict (helpers.h:255-264): params as given
            d = args[0]
            self.model_id = Camera._id(str(d["model"]))
            self.width, self.height = int(d.get("width", 0)), int(d.get("height", 0))
            self.params = [float(v) for v in d["params"]]
            return
        if len(args) == 0:
            args = ("NULL", [], 0, 0)
        if len(args) != 4:
            raise TypeError("Camera(), Camera(model_name, params, width, height) or Camera(dict)")
        self.model_id = Camera._id(str(args[0]))
        self.params = [float(v) for v in args[1]]
        self.width, self.height = int(args[2]), int(args[3])
        self._init_params()

    @staticmethod
    def _id(name):
        """Camera::id_from_string (camera_models.cc:123-133): an unknown name is the NULL camera's id, -1."""
        return {**_CAMERA_IDS, **_OTHER_CAMERA_IDS}.get(name, -1)

    def _init_params(self):
        """Camera::init_params (camera_models.cc:75-93) for the ten models on the path."""
        if self.model_id not in _CAMERA_FOCALS:
            return
        fresh = not self.params
        npar = cabi.CAMERA_NUM_PARAMS[self.model_id]
        self.params = (self.params + [0.0] * npar)[:npar]
        nf, npp = _CAMERA_FOCALS[self.model_id]
        if fresh and npar:
            big = self.width > 0 and self.height > 0
            f = max(self.width, self.height) * 1.2 if big else 1.0
            self.params[:nf] = [f] * nf
            self.params[nf:nf + npp] = [self.width / 2.0, self.height / 2.0] if big else [0.0, 0.0]

    def model_name(self):
        return _CAMERA_NAMES.get(self.model_id, "INVALID_MODEL")

    def todict(self):
        return {"model": self.model_name(), "width": self.width, "height": self.height, "params": list(self.params)}

    def _cabi(self):
        return cabi.Camera(self.model_id, tuple(self.params), self.width, self.height)

    def _run(self, op, x, dim, jac=False):
        x = np.asarray(x, dtype=np.float64).reshape(-1, dim)
        return cabi.camera_batch([dict(op=op, cam=self._cabi(), x=x, jac=jac)])[0]

    def project(self, x):
        """Camera::project of a list of 3D points -> list of 2-vectors."""
        return list(self._run("project", x, 3)["out"])

    def project_with_jac(self, x):
        """Camera::project_with_jac -> (list of 2-vectors, list of 2x3 Jacobians)."""
        r = self._run("project", x, 3, jac=True)
        return list(r["out"]), list(r["jac"].copy())

    def unproject(self, xp):
        """Camera::unproject of a list of pixels -> list of unit bearings (3-vectors)."""
        return list(self._run("unproject", xp, 2)["out"])

    def __repr__(self):
        return f"Camera({self.model_name()!r}, {self.params}, {self.width}, {self.height})"


class Image:
    """camera_pose.h `Image`: pose + camera (what estimate_absolute_pose returns)."""

    def __init__(self, pose, camera):
        self.pose = pose
        self.camera = camera


def _camera(cam):
    """camera_from_dict (helpers.h:255-264): {"model", "width", "height", "params"}; a cabi.Camera passes through, a
    Camera is converted."""
    if isinstance(cam, cabi.Camera):
        return cam
    if isinstance(cam, Camera):
        return cam._cabi()
    if cam is None:
        return cabi.Camera("NULL", ())
    name = str(cam["model"]).upper()
    if name not in _CAMERA_IDS:
        # unknown ids raise inside the library exactly like Camera::unproject's "NYI" (camera_models.cc:184-185)
        raise cabi.PoseLibB200Error(cabi.PLB_ERR_NYI, f"NYI: camera model {name} is not on the CUDA path")
    return cabi.Camera(name, tuple(cam["params"]), int(cam.get("width", 0)), int(cam.get("height", 0)))


def _truthy(v):
    return str(v) == "True" or v is True


def _ransac(d):
    """update_ransac_options (helpers.h:31-40) — "score_initial_model" is purposely not settable from Python."""
    kw = {}
    for k in ("max_iterations", "min_iterations", "seed", "max_prosac_iterations"):
        if k in d:
            kw[k] = int(d[k])
    for k in ("dyn_num_trials_mult", "success_prob"):
        if k in d:
            kw[k] = float(d[k])
    if "progressive_sampling" in d:
        kw["progressive_sampling"] = _truthy(d["progressive_sampling"])
    return kw


def _bundle(d):
    """update_bundle_options (helpers.h:42-95); options the CUDA path does not implement are rejected loudly."""
    kw = {}
    if "max_iterations" in d:
        kw["max_iterations"] = int(d["max_iterations"])
    for k in ("loss_scale", "gradient_tol", "step_tol", "relative_cost_tol", "initial_lambda", "min_lambda",
              "max_lambda"):
        if k in d:
            kw[k] = float(d[k])
    if "loss_type" in d:
        lt = str(d["loss_type"]).upper()
        if lt not in cabi.LOSS:
            raise cabi.PoseLibB200Error(cabi.PLB_ERR_NYI, f"NYI: loss_type {lt}")
        kw["loss_type"] = lt
    if str(d.get("lambda_update", "NIELSEN")).upper() != "NIELSEN" or str(d.get("damping", "LEVENBERG")).upper() != "LEVENBERG":
        raise cabi.PoseLibB200Error(cabi.PLB_ERR_NYI, "NYI: only NIELSEN / LEVENBERG are on the CUDA path")
    return kw


def RansacOptions(opt=None):
    """poselib.RansacOptions(opt={}) (pybind/bindings/types.cc:14-20,168): the defaults of PoseLib/types.h:39-50 with the
    given keys overwritten, as a dict with the keys of write_to_dict (helpers.h:175-183)."""
    out = {"max_iterations": 100000, "min_iterations": 1000, "dyn_num_trials_mult": 3.0, "success_prob": 0.9999,
           "seed": 0, "progressive_sampling": False, "max_prosac_iterations": 100000}
    out.update(_ransac(opt or {}))
    return out


def BundleOptions(opt=None):
    """poselib.BundleOptions(opt={}) (types.cc:22-28,169): defaults of PoseLib/types.h:60-95, keys of helpers.h:185-235.
    Values the CUDA path does not implement (FIXED_FACTOR, MARQUARDT, TRUNCATED_CAUCHY / TRUNCATED_LE_ZACH) raise NYI."""
    opt = dict(opt or {})
    out = {"max_iterations": 100, "loss_scale": 1.0, "loss_type": "CAUCHY", "gradient_tol": 1e-12, "step_tol": 1e-8,
           "relative_cost_tol": 1e-10, "initial_lambda": 1e-3, "min_lambda": 1e-10, "max_lambda": 1e10,
           "lambda_factor": 10.0, "verbose": False, "lambda_update": "NIELSEN", "damping": "LEVENBERG"}
    out.update(_bundle(opt))
    if "lambda_factor" in opt:
        out["lambda_factor"] = float(opt["lambda_factor"])
    if "verbose" in opt:
        out["verbose"] = _truthy(opt["verbose"])
    return out


def _info(r):
    """write_to_dict(RansacStats) + inliers as a list of bool (helpers.h:237-253,266-272)."""
    out = dict(r["stats"])
    out["inliers"] = [bool(v) for v in r["inliers"]]
    return out


def _pts(a, dim):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if a.ndim != 2 or a.shape[1] != dim:
        raise ValueError(f"expected an (n, {dim}) array")
    return a


def estimate_absolute_pose(points2D, points3D, camera, opt=None, initial_pose=None):
    """absolute_pose.cc:15-47,317-330.  Returns (Image, info)."""
    opt = opt or {}
    if _truthy(opt.get("estimate_focal_length", False)) or _truthy(opt.get("estimate_extra_params", False)):
        raise cabi.PoseLibB200Error(cabi.PLB_ERR_NYI, "NYI: focal-length estimation (SURVEY §8f N2)")
    rkw = _ransac(opt.get("ransac", {}))
    init = None
    if initial_pose is not None:
        init = np.r_[initial_pose.q, initial_pose.t]
        rkw["score_initial_model"] = True
    cam = _camera(camera)
    r = cabi.estimate("pnp", _pts(points2D, 2), _pts(points3D, 3), cabi.RansacOpt(**rkw),
                      cabi.BundleOpt(**_bundle(opt.get("bundle", {}))), float(opt.get("max_error", 12.0)), cam,
                      init=init)
    return Image(CameraPose(r["model"][:4], r["model"][4:]), camera), _info(r)


def estimate_relative_pose(points2D_1, points2D_2, camera1, camera2, opt=None, initial_pose=None):
    """relative_pose.cc:15-52,405-421.  Returns (CameraPose, info)."""
    opt = opt or {}
    rkw = _ransac(opt.get("ransac", {}))
    init = None
    if initial_pose is not None:
        init = np.r_[initial_pose.q, initial_pose.t]
        rkw["score_initial_model"] = True
    r = cabi.estimate("relpose", _pts(points2D_1, 2), _pts(points2D_2, 2), cabi.RansacOpt(**rkw),
                      cabi.BundleOpt(**_bundle(opt.get("bundle", {}))), float(opt.get("max_error", 1.0)),
                      _camera(camera1), _camera(camera2), init=init,
                      tangent_sampson=_truthy(opt.get("tangent_sampson", False)))
    return CameraPose(r["model"][:4], r["model"][4:]), _info(r)


def estimate_fundamental(points2D_1, points2D_2, opt=None, initial_F=None):
    """relative_pose.cc:460-463.  Returns (F 3x3, info)."""
    opt = opt or {}
    rkw = _ransac(opt.get("ransac", {}))
    if initial_F is not None:
        rkw["score_initial_model"] = True
    r = cabi.estimate("fundamental", _pts(points2D_1, 2), _pts(points2D_2, 2), cabi.RansacOpt(**rkw),
                      cabi.BundleOpt(**_bundle(opt.get("bundle", {}))), float(opt.get("max_error", 1.0)),
                      init=initial_F, rfc=_truthy(opt.get("real_focal_check", False)))
    return r["model"], _info(r)


def estimate_homography(points2D_1, points2D_2, opt=None, initial_H=None):
    """homography.cc:75-77.  Returns (H 3x3, info)."""
    opt = opt or {}
    rkw = _ransac(opt.get("ransac", {}))
    if initial_H is not None:
        rkw["score_initial_model"] = True
    r = cabi.estimate("homography", _pts(points2D_1, 2), _pts(points2D_2, 2), cabi.RansacOpt(**rkw),
                      cabi.BundleOpt(**_bundle(opt.get("bundle", {}))), float(opt.get("max_error", 1.0)),
                      init=initial_H)
    return r["model"], _info(r)


# ---- minimal solvers (pybind/bindings/solvers.cc:305,341,349): lists of solutions, unit bearings in ---------------
def p3p(x, X):
    poses, n = cabi.p3p_batch(_pts(x, 3)[None], _pts(X, 3)[None])
    return [CameraPose(p[:4], p[4:]) for p in poses[0, :n[0]]]


def p3p_lambdatwist(x, X):
    poses, n = cabi.p3p_lambdatwist_batch(_pts(x, 3)[None], _pts(X, 3)[None])
    return [CameraPose(p[:4], p[4:]) for p in poses[0, :n[0]]]


def relpose_5pt(x1, x2):
    poses, n = cabi.relpose_5pt_poses_batch(_pts(x1, 3)[None], _pts(x2, 3)[None])
    return [CameraPose(p[:4], p[4:]) for p in poses[0, :n[0]]]


def essential_matrix_5pt(x1, x2):
    Es, n = cabi.relpose_5pt_batch(_pts(x1, 3)[None], _pts(x2, 3)[None])
    return [E.copy() for E in Es[0, :n[0]]]


def relpose_7pt(x1, x2):
    Fs, n = cabi.relpose_7pt_batch(_pts(x1, 3)[None], _pts(x2, 3)[None])
    return [F.copy() for F in Fs[0, :n[0]]]


def homography_4pt(x1, x2, check_cheirality=True):
    Hs, n = cabi.homography_4pt_batch(_pts(x1, 3)[None], _pts(x2, 3)[None], check_cheirality)
    return [Hs[0].copy()] if n[0] else []


def essential_matrix_8pt(x1, x2):
    """poselib.essential_matrix_8pt (pybind/bindings/solvers.cc): n >= 8 bearing pairs -> E (3x3)."""
    a = np.asarray(x1, dtype=np.float64).reshape(1, -1, 3)
    b = np.asarray(x2, dtype=np.float64).reshape(1, -1, 3)
    return cabi.essential_matrix_8pt_batch(a, b)[0]


def relpose_8pt(x1, x2):
    """poselib.relpose_8pt: n >= 8 bearing pairs -> list of CameraPose (cheirality-consistent motions of E)."""
    a = np.asarray(x1, dtype=np.float64).reshape(1, -1, 3)
    b = np.asarray(x2, dtype=np.float64).reshape(1, -1, 3)
    poses, n = cabi.relpose_8pt_batch(a, b)
    return [CameraPose(poses[0, i, :4], poses[0, i, 4:]) for i in range(int(n[0]))]
