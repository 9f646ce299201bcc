"""plb_camera_batch / plb_camera_batch_device: PoseLib's Camera::project / project_with_jac / unproject /
unproject_with_jac and the 2D unproject over many points of many cameras.

  * CPU: the ctypes struct against the header, every argument check and its order (every status set, outputs
    untouched), PLB_ERR_NYI for the reference's other models, PLB_ERR_CUDA without a device, the fixture regenerated bit
    for bit where the reference exists, the host build of camera.cuh equal to every fixture row, and pyapi.Camera's
    constructors and todict.
  * GPU: every fixture row through both forms and every op, with and without jac / jac_params; the device form equals
    the host form and fp32 inputs give the fp64 call's bits on the widened values; a mixed batch equals the one-problem
    calls for any n_gpus / streams; pyapi.Camera equals cabi; the adapter templates equal the C-ABI."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_camera_ops_golden as OG  # noqa: E402

try:
    from poselib_b200 import cabi, pyapi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)

FIXTURE = OG.load()
NYI_IDS = (5, 6, 7, 10, 11, 99, 100)
# Fisheye models (atan2 / tan on the device, not correctly rounded) in every column, and the division models' parameter
# Jacobians (pow), are held to this relative bar with the fixture's finite / non-finite pattern; every other column is
# bit for bit (+ - * / and sqrt under -fmad=false).
DEVICE_FN_RTOL = 1e-12


def _cam(c):
    return cabi.Camera(int(c["model"]), tuple(c["params"]))


def _eq(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def assert_matches(got, ref, model, exact, tag):
    """Bit for bit where `exact`, else within DEVICE_FN_RTOL with the same finite pattern (see above)."""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, (tag, got.shape, ref.shape)
    if exact and model not in (8, 9):
        assert _eq(got, ref), (tag, np.nanmax(np.abs(got - ref)))
        return
    ok = np.isfinite(ref)
    assert np.array_equal(np.isfinite(got), ok), tag
    dev = np.max(np.abs(got[ok] - ref[ok]) / np.maximum(1.0, np.abs(ref[ok])), initial=0.0)
    assert dev <= DEVICE_FN_RTOL, (tag, dev)


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_struct_layout_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    fields = [f for f, _ in cabi.CameraProblem._fields_]
    cname = {"in_": "in"}
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "poselib_b200.h"\nint main(void) {\n'
                   '    printf("%zu\\n", sizeof(plb_camera_problem));\n' +
                   "".join('    printf("%%zu\\n", offsetof(plb_camera_problem, %s));\n' % cname.get(f, f) for f in fields) +
                   '    printf("%d %d %d\\n", PLB_CAMOP_PROJECT, PLB_CAMOP_UNPROJECT, PLB_CAMOP_UNPROJECT_2D);\n'
                   '    return 0;\n}\n')
    exe = str(tmp_path / "layout")
    subprocess.check_call(["cc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    out = subprocess.check_output([exe], text=True).splitlines()
    assert int(out[0]) == C.sizeof(cabi.CameraProblem)
    for f, line in zip(fields, out[1:]):
        assert int(line) == getattr(cabi.CameraProblem, f).offset, f
    assert out[-1].split() == [str(cabi.CAMOP[k]) for k in ("project", "unproject", "unproject_2d")]
    assert {"plb_camera_batch", "plb_camera_batch_device"} <= set(cabi.EXPORTS)


def test_fixture_covers_every_model_and_branch():
    assert {c["model"] for c in FIXTURE} == {-1, 0, 1, 2, 3, 4, 8, 9, 101, 102}
    assert sum(c["model"] == 4 for c in FIXTURE) == 2
    for m in (101, 102):
        assert {np.sign(c["params"][-1]) for c in FIXTURE if c["model"] == m} == {-1.0, 1.0}
    for c in FIXTURE:
        assert np.any(c["Z"][:, 2] < 0) and np.any(c["Z"][:, 2] == 0)
        if c["model"] in (101, 102) and c["params"][-1] > 0:
            Z = c["Z"]
            assert np.any(Z[:, 2] ** 2 - 4.0 * (Z[:, 0] ** 2 + Z[:, 1] ** 2) * c["params"][-1] < 0)
    assert sum(not np.all(np.isfinite(c["xp"])) for c in FIXTURE) >= 8  # Z = 0 gives non-finite pixels


def test_fixture_regenerates_bit_for_bit(tmp_path):
    if not (os.path.isdir(os.path.join(OG.CG.REF, "PoseLib")) and
            os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libplref2.so"))):
        pytest.skip("needs the reference checkout and oracle/_ref/libplref2.so")
    lib = OG.CG.build_client(str(tmp_path))
    import json
    with open(OG.OUT) as f:
        stored = json.load(f)["cases"]
    assert [OG.case(lib, name) for name in OG.CAMERAS] == stored


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
def test_host_build_reproduces_every_fixture_row(tmp_path):
    exe = str(tmp_path / "camera_models_host_test")
    subprocess.check_call(["nvcc", "-std=c++17", "-O2", "-fmad=false", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-Xcompiler", "-ffp-contract=off", "-o", exe, os.path.join(HERE, "camera_models_host_test.cu")])
    for c in FIXTURE:
        P = OG.CG.NUM_PARAMS[c["model"]]
        args = [exe, str(c["model"])] + [repr(float(v)) for v in OG.params8(c["camera"])] + ["1.0"]
        out = subprocess.check_output(args + ["px"] + [repr(float(v)) for v in c["px"].reshape(-1)], text=True)
        got = np.array([[float.fromhex(t) for t in line.split()[1:]] for line in out.splitlines()[10:]])
        n = len(c["px"])
        assert _eq(got[:, 0:3], c["x3"]) and _eq(got[:, 3:5], c["x2"]), c["camera"]
        assert _eq(got[:, 5:8], c["d"]) and _eq(got[:, 8:14], c["M"].reshape(n, 6)), c["camera"]
        assert _eq(got[:, 14:17], c["d"]) and _eq(got[:, 23:].reshape(n, 3, 8)[:, :, :P], c["dp"]), c["camera"]
        out = subprocess.check_output(args + ["pt"] + [repr(float(v)) for v in c["Z"].reshape(-1)], text=True)
        got = np.array([[float.fromhex(t) for t in line.split()[1:]] for line in out.splitlines()[10:]])
        nz = len(c["Z"])
        assert _eq(got[:, 0:2], c["xp"]) and _eq(got[:, 2:4], c["xq"]), c["camera"]
        assert _eq(got[:, 4:10], c["jac"].reshape(nz, 6)), c["camera"]
        assert _eq(got[:, 10:].reshape(nz, 2, 8)[:, :, :P], c["jp"]), c["camera"]


def _cpu_problems():
    rng = np.random.default_rng(3)
    pin = cabi.Camera("PINHOLE", (500.0, 500.0, 320.0, 240.0))
    opencv = cabi.Camera("OPENCV", (500.0, 500.0, 320.0, 240.0, 0.1, -0.05, 0.001, 0.002))
    return [dict(op=0, cam=pin, x=rng.normal(size=(7, 3)) + [0, 0, 4], jac=True, jac_params=True),
            dict(op=1, cam=opencv, x=rng.uniform(0, 600, size=(9, 2)), jac=True),
            dict(op=2, cam=pin, x=rng.uniform(0, 600, size=(5, 2))),
            dict(op=1, cam=cabi.Camera("NULL", ()), x=rng.normal(size=(4, 2)), jac_params=True)]


def _arr(problems):
    arr = (cabi.CameraProblem * len(problems))()
    keep = []
    for q, p in zip(arr, problems):
        x = np.ascontiguousarray(p["x"], dtype=np.float64)
        n = len(x)
        o, j, jp = np.full(3 * n, 7.0), np.full(6 * n, 7.0), np.full(24 * n, 7.0)
        keep.append((x, o, j, jp))
        q.op, q.n, q.camera = p["op"], n, p["cam"]
        q.in_, q.out = x.ctypes.data_as(cabi._P), o.ctypes.data_as(cabi._P)
        q.jac = j.ctypes.data_as(cabi._P) if p.get("jac") else None
        q.jac_params = jp.ctypes.data_as(cabi._P) if p.get("jac_params") else None
        q.status = 12345
    return arr, keep


def test_argument_checks_run_before_the_device():
    lib = cabi.lib()
    assert lib.plb_camera_batch(None, C.c_size_t(3), -1, 8) == cabi.PLB_ERR_ARG
    assert lib.plb_camera_batch_device(None, C.c_size_t(3), cabi.DTYPE_F64, None, 8) == cabi.PLB_ERR_ARG
    assert lib.plb_camera_batch(None, C.c_size_t(0), -1, 8) == cabi.PLB_OK
    base = _cpu_problems()

    def check(edit, code, form="both", n_gpus=-1, dtype=cabi.DTYPE_F64):
        rcs = []
        for f in ("host", "device"):
            if form not in ("both", f):
                continue
            arr, keep = _arr(base)
            edit(arr)
            before, outs = bytes(arr), [bytes(k[1]) + bytes(k[2]) + bytes(k[3]) for k in keep]
            if f == "host":
                rcs.append(lib.plb_camera_batch(arr, C.c_size_t(len(base)), n_gpus, 8))
            else:
                rcs.append(lib.plb_camera_batch_device(arr, C.c_size_t(len(base)), dtype, None, 8))
            assert all(q.status == code for q in arr), [q.status for q in arr]
            for q in arr:
                q.status = 12345
            assert bytes(arr) == before
            assert [bytes(k[1]) + bytes(k[2]) + bytes(k[3]) for k in keep] == outs
        assert rcs and all(rc == code for rc in rcs), (rcs, code)

    def set_(i, **kw):
        def edit(arr):
            for k, v in kw.items():
                setattr(arr[i], k, v)
        return edit

    def chain(*edits):
        def edit(arr):
            for e in edits:
                e(arr)
        return edit

    for bad in (-1, 3, 1000):
        check(set_(1, op=bad), cabi.PLB_ERR_ARG)
    for i in range(len(base)):
        for field in ("in_", "out"):
            check(set_(i, **{field: None}), cabi.PLB_ERR_ARG)
    j = np.zeros(6)
    check(set_(2, jac=j.ctypes.data_as(cabi._P)), cabi.PLB_ERR_ARG)
    check(set_(2, jac_params=j.ctypes.data_as(cabi._P)), cabi.PLB_ERR_ARG)
    check(set_(0, n=2 ** 61), cabi.PLB_ERR_ARG)  # 2^61 x 6 doubles: n x the widest row overflows
    check(set_(2, n=2 ** 61), cabi.PLB_ERR_ARG)  # 2 doubles x 8 bytes x 2^61 overflows too
    for mid in NYI_IDS:
        check(set_(1, camera=cabi.Camera(mid, (500.0, 500.0, 0.0, 0.0))), cabi.PLB_ERR_NYI)
    # the order: an argument error of a later problem is found after the NYI camera of an earlier one, and an argument
    # error of a problem comes before its own NYI camera
    nyi = cabi.Camera(5, (500.0, 500.0, 0.0, 0.0))
    check(chain(set_(1, camera=nyi), set_(3, op=7)), cabi.PLB_ERR_NYI)
    check(chain(set_(1, camera=nyi, out=None)), cabi.PLB_ERR_ARG)
    check(chain(set_(1, op=9), set_(3, camera=nyi)), cabi.PLB_ERR_ARG)
    check(lambda arr: None, cabi.PLB_ERR_ARG, form="device", dtype=2)
    check(chain(set_(1, camera=nyi)), cabi.PLB_ERR_ARG, form="device", dtype=2)  # dtype before the problems
    check(lambda arr: None, cabi.PLB_ERR_ARG, form="host", n_gpus=-2)
    check(set_(1, camera=nyi), cabi.PLB_ERR_NYI, form="host", n_gpus=-2)  # the problems before n_gpus
    if cabi.device_count() == 0:
        check(lambda arr: None, cabi.PLB_ERR_CUDA)
        check(set_(1, n=0, in_=None, out=None), cabi.PLB_ERR_CUDA)  # n = 0 needs no pointers
        check(lambda arr: None, cabi.PLB_ERR_CUDA, form="host", n_gpus=5)


def test_pyapi_camera_constructors_and_todict():
    c = pyapi.Camera()
    assert (c.model_id, c.width, c.height, c.params, c.model_name()) == (-1, 0, 0, [], "NULL")
    c = pyapi.Camera("PINHOLE", [], 640, 480)  # Camera::init_params: focal = 1.2 max(w, h), principal point = centre
    assert c.params == [768.0, 768.0, 320.0, 240.0] and c.model_id == 1
    c = pyapi.Camera("OPENCV", [], 0, 0)
    assert c.params == [1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]
    c = pyapi.Camera("SIMPLE_RADIAL", [100.0, 1.0], 10, 10)  # params given: resized, not initialised
    assert c.params == [100.0, 1.0, 0.0, 0.0]
    assert pyapi.Camera("NO_SUCH_MODEL", [], 0, 0).model_id == -1  # id_from_string: unknown names are INVALID = -1
    for fx in FIXTURE:
        name = OG.CAMERAS[fx["camera"]][0]
        d = {"model": name, "width": 1920, "height": 1080, "params": list(fx["params"])}
        c = pyapi.Camera(d)
        assert c.todict() == d and c.model_id == fx["model"]
        assert pyapi.Camera(c.todict()).todict() == d
        assert pyapi.Camera(name, fx["params"], 1920, 1080).todict() == d
    assert pyapi.Camera({"model": "FOV", "params": [1.0, 2.0]}).todict() == {"model": "FOV", "width": 0, "height": 0,
                                                                           "params": [1.0, 2.0]}
    cam = pyapi.Camera("RADIAL", [1000.0, 320.0, 240.0, 0.1, 0.01], 640, 480)
    c2 = pyapi._camera(cam)
    assert isinstance(c2, cabi.Camera) and c2.model_id == 3 and list(c2.params)[:5] == cam.params
    with pytest.raises(TypeError):
        pyapi.Camera("PINHOLE", [1.0])


def _adapter_build(tmp_path):
    exe = str(tmp_path / "adapter_camera_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(HERE, "adapter_camera_test.cc"), "-o", exe,
                           "-L" + os.path.join(ROOT, "poselib_b200"), "-lposelib_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "poselib_b200")])
    return exe


def test_adapter_camera_templates_compile_and_link(tmp_path):
    out = subprocess.run([_adapter_build(tmp_path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "adapter camera link ok" in out.stdout, out.stdout + out.stderr


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _gpu():
    if cabi.device_count() == 0:
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    cabi.set_device(0)


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if cabi.device_count() == 0 or not t.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    return t


# (op, jac, jac_params) -> the fixture columns: out, jac, jac_params, and whether the parameter Jacobian is pow-free
CALLS = [("project", False, False), ("project", True, False), ("project", False, True), ("project", True, True),
         ("unproject", False, False), ("unproject", True, False), ("unproject", False, True), ("unproject", True, True),
         ("unproject_2d", False, False)]


def _expected(c, op, jac, jp):
    if op == "project":
        return (c["xq"] if jac or jp else c["xp"]), c["jac"], c["jp"]
    if op == "unproject":
        return (c["d"] if jac or jp else c["x3"]), c["M"], c["dp"]
    return c["x2"], None, None


def _problems(op, jac, jp):
    return [dict(op=op, cam=_cam(c), x=c["Z"] if op == "project" else c["px"], jac=jac, jac_params=jp) for c in FIXTURE]


def _check_fixture(res, op, jac, jp, tag):
    for c, r in zip(FIXTURE, res):
        assert r["status"] == cabi.PLB_OK
        out, J, P = _expected(c, op, jac, jp)
        t = (tag, c["camera"], op, jac, jp)
        assert_matches(r["out"], out, c["model"], True, t + ("out",))
        if jac:
            assert_matches(r["jac"], J, c["model"], True, t + ("jac",))
        else:
            assert r["jac"] is None
        if jp:
            # division: the parameter Jacobian of unproject divides by pow()
            exact = not (op == "unproject" and c["model"] in (101, 102))
            assert_matches(r["jac_params"], P, c["model"], exact, t + ("jac_params",))
        else:
            assert r["jac_params"] is None


@pytest.mark.gpu
@pytest.mark.parametrize("op,jac,jp", CALLS)
def test_fixture_through_the_host_form(op, jac, jp):
    _gpu()
    _check_fixture(cabi.camera_batch(_problems(op, jac, jp)), op, jac, jp, "host")


def _to_host(res):
    return [{k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in r.items()} for r in res]


@pytest.mark.gpu
@pytest.mark.parametrize("op,jac,jp", CALLS)
def test_fixture_through_the_device_form(torch, op, jac, jp):
    probs = _problems(op, jac, jp)
    dev = [dict(p, x=torch.tensor(p["x"], device="cuda:0")) for p in probs]
    got = _to_host(cabi.camera_batch_device(dev))
    _check_fixture(got, op, jac, jp, "device")
    host = cabi.camera_batch(probs)
    for g, h in zip(got, host):
        for k in ("out", "jac", "jac_params"):
            assert (g[k] is None) == (h[k] is None) and (g[k] is None or _eq(g[k], h[k])), k


@pytest.mark.gpu
@pytest.mark.parametrize("op,jac,jp", CALLS)
def test_float_inputs_give_the_double_call_on_the_widened_values(torch, op, jac, jp):
    probs = _problems(op, jac, jp)
    f32 = [dict(p, x=torch.tensor(p["x"], dtype=torch.float32, device="cuda:0")) for p in probs]
    wide = [dict(p, x=p["x"].astype(np.float32).astype(np.float64)) for p in probs]
    got = _to_host(cabi.camera_batch_device(f32))
    ref = cabi.camera_batch(wide)
    for g, h in zip(got, ref):
        for k in ("out", "jac", "jac_params"):
            assert (g[k] is None) == (h[k] is None) and (g[k] is None or _eq(g[k], h[k])), k


def _mixed_batch():
    """About 200 problems: every op (with and without Jacobians) on every fixture camera, n in {0, 1, 255, 256, 257,
    1e5} in turn, points drawn around each camera's fixture grid."""
    rng = np.random.default_rng(11)
    sizes = (0, 1, 255, 256, 257, 100000)
    probs = []
    for i, (c, (op, jac, jp)) in enumerate([(c, k) for k in CALLS for c in FIXTURE][:200]):
        n = sizes[i % len(sizes)]
        src = c["Z"] if op == "project" else c["px"]
        x = src[rng.integers(0, len(src), n)] * (1.0 + 1e-3 * rng.normal(size=(n, 1)))
        probs.append(dict(op=op, cam=_cam(c), x=x, jac=jac, jac_params=jp))
    return probs


@pytest.mark.gpu
def test_mixed_batch_equals_the_single_calls():
    _gpu()
    probs = _mixed_batch()
    singles = [cabi.camera_batch([p])[0] for p in probs]
    runs = [(-1, 1), (-1, 8), (0, 1), (0, 8)]
    for n_gpus, streams in runs:
        got = cabi.camera_batch(probs, n_gpus=n_gpus, streams=streams)
        for g, s in zip(got, singles):
            for k in ("out", "jac", "jac_params"):
                assert (g[k] is None) == (s[k] is None) and (g[k] is None or _eq(g[k], s[k])), (n_gpus, streams, k)


@pytest.mark.gpu
def test_mixed_device_batch_equals_the_host_batch(torch):
    probs = _mixed_batch()
    ref = cabi.camera_batch(probs)
    for streams in (1, 8):
        got = _to_host(cabi.camera_batch_device([dict(p, x=torch.tensor(p["x"], device="cuda:0")) for p in probs],
                                                streams=streams))
        for g, s in zip(got, ref):
            for k in ("out", "jac", "jac_params"):
                assert (g[k] is None) == (s[k] is None) and (g[k] is None or _eq(g[k], s[k])), (streams, k)


@pytest.mark.gpu
def test_device_form_checks_its_pointers(torch):
    _gpu()
    x = torch.zeros((4, 3), dtype=torch.float64, device="cuda:0")
    cam = cabi.Camera("PINHOLE", (500.0, 500.0, 0.0, 0.0))
    arr = (cabi.CameraProblem * 1)()
    host_out = np.zeros(8)
    q = arr[0]
    q.op, q.n, q.camera = 0, 4, cam
    q.in_ = C.cast(C.c_void_p(x.data_ptr()), cabi._P)
    q.out = host_out.ctypes.data_as(cabi._P)  # host memory: step 8
    assert cabi.lib().plb_camera_batch_device(arr, C.c_size_t(1), cabi.DTYPE_F64, None, 1) == cabi.PLB_ERR_ARG
    assert q.status == cabi.PLB_ERR_ARG and not host_out.any()
    out = torch.zeros(9, dtype=torch.float64, device="cuda:0")
    q.out = C.cast(C.c_void_p(out.data_ptr() + 4), cabi._P)  # misaligned
    assert cabi.lib().plb_camera_batch_device(arr, C.c_size_t(1), cabi.DTYPE_F64, None, 1) == cabi.PLB_ERR_ARG
    assert not out.any()


@pytest.mark.gpu
def test_pyapi_camera_methods_equal_cabi():
    _gpu()
    for c in FIXTURE:
        name = OG.CAMERAS[c["camera"]][0]
        cam = pyapi.Camera(name, c["params"], 0, 0) if c["model"] != -1 else pyapi.Camera()
        cc = _cam(c)
        Z, px = list(c["Z"]), list(c["px"])
        ref_p = cabi.camera_batch([dict(op="project", cam=cc, x=c["Z"])])[0]
        ref_pj = cabi.camera_batch([dict(op="project", cam=cc, x=c["Z"], jac=True)])[0]
        ref_u = cabi.camera_batch([dict(op="unproject", cam=cc, x=c["px"])])[0]
        assert _eq(np.array(cam.project(Z)), ref_p["out"])
        xp, J = cam.project_with_jac(Z)
        assert _eq(np.array(xp), ref_pj["out"]) and _eq(np.array(J), ref_pj["jac"])
        assert all(j.shape == (2, 3) for j in J)
        assert _eq(np.array(cam.unproject(px)), ref_u["out"])
    assert pyapi.Camera().project([]) == []
    with pytest.raises(cabi.PoseLibB200Error) as e:
        pyapi.Camera({"model": "FOV", "params": [1.0, 2.0]}).unproject([[1.0, 2.0]])
    assert e.value.code == cabi.PLB_ERR_NYI


@pytest.mark.gpu
def test_adapter_camera_templates_match_the_c_abi(tmp_path):
    _gpu()
    out = subprocess.run([_adapter_build(tmp_path), "run"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "adapter camera ok" in out.stdout, out.stdout + out.stderr
