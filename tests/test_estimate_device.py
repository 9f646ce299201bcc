"""plb_estimate_batch_device / cabi.estimate_batch_device: correspondences already in GPU memory in, inlier masks out in
GPU memory.  Everything else must be plb_estimate_batch on the calling thread's device, bit for bit.
  * CPU: the argument checks that come before the device check, PLB_ERR_CUDA without a device, and the binding's
    rejection of tensors it cannot pass.
  * GPU: parity with plb_estimate_batch on one mixed batch (fp64, and fp32 against the widened values), the caller's
    arrays left untouched, stream order, the PCIe counters, and the rejection of memory that is not on the device."""
import ctypes as C

import numpy as np
import pytest

try:
    from poselib_b200 import cabi
except ImportError:  # the CUDA library is not built on this machine
    pytest.skip("libposelib_b200.so not built", allow_module_level=True)
from poselib_b200 import problem_generator as G

F = G.FOCAL


def _raw_call(probs, a_ptrs, b_ptrs, mask_ptrs, dtype, stream=None, streams=4):
    """plb_estimate_batch_device on raw pointers (the binding only passes CUDA tensors)."""
    arr = (cabi.EstimateProblem * len(probs))()
    for i, p in enumerate(probs):
        cabi._fill_estimate_problem(arr[i], p, p["n"])
        arr[i].a = C.cast(C.c_void_p(a_ptrs[i]), cabi._P)
        arr[i].b = C.cast(C.c_void_p(b_ptrs[i]), cabi._P)
        arr[i].inliers = C.cast(C.c_void_p(mask_ptrs[i]), C.c_char_p)
    rc = cabi.lib().plb_estimate_batch_device(arr, C.c_size_t(len(probs)), int(dtype), C.c_void_p(stream),
                                              int(streams))
    return rc, arr


# ---- CPU ---------------------------------------------------------------------------------------------------
def test_arguments_are_checked_before_the_device():
    lib = cabi.lib()
    assert lib.plb_estimate_batch_device(None, C.c_size_t(0), 0, None, 4) == cabi.PLB_OK
    assert lib.plb_estimate_batch_device(None, C.c_size_t(3), 0, None, 4) == cabi.PLB_ERR_ARG
    arr = (cabi.EstimateProblem * 2)()
    assert lib.plb_estimate_batch_device(arr, C.c_size_t(2), 7, None, 4) == cabi.PLB_ERR_ARG
    assert [q.status for q in arr] == [cabi.PLB_ERR_ARG] * 2
    assert "dtype" in lib.plb_last_error().decode()


def test_no_device_is_a_cuda_error():
    if cabi.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    arr = (cabi.EstimateProblem * 2)()
    assert cabi.lib().plb_estimate_batch_device(arr, C.c_size_t(2), cabi.DTYPE_F32, None, 4) == cabi.PLB_ERR_CUDA
    assert [q.status for q in arr] == [cabi.PLB_ERR_CUDA] * 2


def test_binding_rejects_what_it_cannot_pass():
    torch = pytest.importorskip("torch")
    p = dict(kind="homography", ransac=cabi.RansacOpt(), bundle=cabi.BundleOpt(), max_error=1.0)
    with pytest.raises(TypeError):  # host arrays and host tensors: use estimate_batch
        cabi.estimate_batch_device([dict(p, a=np.zeros((8, 2)), b=np.zeros((8, 2)))])
    with pytest.raises(TypeError):
        cabi.estimate_batch_device([dict(p, a=torch.zeros(8, 2), b=torch.zeros(8, 2))])
    assert cabi.estimate_batch_device([]) == []


# ---- GPU ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch():
    import torch as t
    if cabi.device_count() == 0 or not t.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests need a CUDA device")
    cabi.set_device(0)
    return t


def _cameras():
    return {"NULL": None,
            "PINHOLE": cabi.Camera("PINHOLE", (F, F, 0.0, 0.0)),
            "RADIAL": cabi.Camera("RADIAL", (F, 2.0, -3.0, 0.01, -0.002)),
            "OPENCV": cabi.Camera("OPENCV", (F, 1.01 * F, 1.0, -2.0, 0.01, -0.001, 0.0005, -0.0003)),
            "RADIAL_FISHEYE": cabi.Camera("RADIAL_FISHEYE", (F, -1.0, 2.0, 0.01, 0.001))}


def _mixed_batch():
    """About 64 problems: every kind, five camera models (NULL, PINHOLE, RADIAL, OPENCV, RADIAL_FISHEYE), tangent Sampson
    and real_focal_check both ways, PnP with camera refinement, n = 0 and n below each minimum."""
    cams = _cameras()
    names = list(cams)
    bo = cabi.BundleOpt()
    probs = []
    for i in range(12):
        cname = names[i % len(names)]
        cam = cams[cname]
        unit = F if cam is None else 1.0  # the NULL camera takes calibrated points
        ro = cabi.RansacOpt(max_iterations=1500, min_iterations=50, seed=i)
        p = G.relpose_problem(300 + 37 * i, 0.5, config_id=61, problem_idx=i)
        cam2 = None if cam is None else (cams[names[(i + 2) % len(names)]] or cams["PINHOLE"])
        probs.append(dict(kind="relpose", a=p["x1"] / unit, b=p["x2"] / unit, cam1=cam, cam2=cam2, max_error=1.0 / unit,
                          tangent_sampson=bool(i % 2) and cam is not None, ransac=ro, bundle=bo))
        p = G.abspose_problem(150 + 23 * i, 0.5, config_id=62, problem_idx=i)
        flags = [0, 3, 7, 1][i % 4] if cam is not None else 0
        probs.append(dict(kind="pnp", a=p["x"] / unit, b=p["X"], cam1=cam, max_error=8.0 / unit, ransac=ro,
                          bundle=cabi.BundleOpt(refine_intrinsics=flags)))
        p = G.relpose_problem(250 + 41 * i, 0.45, config_id=63, problem_idx=i)
        probs.append(dict(kind="fundamental", a=p["x1"], b=p["x2"], max_error=1.0, rfc=bool(i % 2), ransac=ro, bundle=bo))
        p = G.homography_problem(200 + 29 * i, 0.6, config_id=64, problem_idx=i)
        probs.append(dict(kind="homography", a=p["x1"], b=p["x2"], max_error=1.0, ransac=ro, bundle=bo))
    rng = np.random.default_rng(65)
    for kind, n in [("pnp", 0), ("relpose", 0), ("fundamental", 0), ("homography", 0), ("pnp", 2), ("relpose", 4),
                    ("fundamental", 6), ("homography", 3), ("relpose", 5), ("fundamental", 7), ("homography", 4)]:
        b_dim = 3 if kind == "pnp" else 2
        probs.append(dict(kind=kind, a=rng.normal(size=(n, 2)) * 100, b=rng.normal(size=(n, b_dim)) * 100,
                          cam1=cams["PINHOLE"] if kind in ("pnp", "relpose") else None,
                          cam2=cams["PINHOLE"] if kind == "relpose" else None, max_error=2.0,
                          ransac=cabi.RansacOpt(max_iterations=200, min_iterations=10, seed=n), bundle=bo))
    return probs


def _same_stats(a, b):
    return all(x == y or (x != x and y != y) for x, y in zip(a.values(), b.values())) and a.keys() == b.keys()


def _assert_same(ref, out, probs, label):
    for i, (r, o) in enumerate(zip(ref, out)):
        tag = (label, i, probs[i]["kind"], len(probs[i]["a"]))
        assert o["status"] == r["status"] == cabi.PLB_OK, tag
        assert _same_stats(r["stats"], o["stats"]), (tag, r["stats"], o["stats"])
        assert np.array_equal(r["model"], o["model"], equal_nan=True), tag
        assert np.array_equal(r["camera1"], o["camera1"], equal_nan=True), tag
        m = o["inliers"]
        if m is not None:
            assert str(m.dtype) == "torch.bool" and m.is_cuda and m.numel() == len(probs[i]["a"]), tag
            assert np.array_equal(m.cpu().numpy().astype(np.int8), r["inliers"]), tag


def _on_device(torch, probs, dtype):
    return [dict(p, a=torch.tensor(p["a"], dtype=dtype, device="cuda:0"),
                 b=torch.tensor(p["b"], dtype=dtype, device="cuda:0")) for p in probs]


@pytest.mark.gpu
def test_fp64_equals_estimate_batch_bit_for_bit(torch):
    probs = _mixed_batch()
    ref = cabi.estimate_batch(probs, streams=4, n_gpus=-1)
    dev = _on_device(torch, probs, torch.float64)
    _assert_same(ref, cabi.estimate_batch_device(dev, streams=4), probs, "fp64")
    # some masks NULL: the rest of every problem is unchanged
    masks = [torch.zeros(len(p["a"]), dtype=torch.uint8, device="cuda:0") if i % 3 else None
             for i, p in enumerate(probs)]
    rc, arr = _raw_call([dict(p, n=len(p["a"])) for p in probs], [d["a"].data_ptr() for d in dev],
                        [d["b"].data_ptr() for d in dev], [m.data_ptr() if m is not None and m.numel() else None
                                                           for m in masks], cabi.DTYPE_F64)
    assert rc == cabi.PLB_OK
    out = cabi._estimate_results(arr, probs, [None] * len(probs))
    _assert_same(ref, out, probs, "null masks")
    torch.cuda.synchronize()
    for m, r in zip(masks, ref):
        if m is not None:
            assert np.array_equal(m.cpu().numpy().astype(np.int8), r["inliers"])


@pytest.mark.gpu
def test_fp32_equals_estimate_batch_on_the_widened_values(torch):
    probs = _mixed_batch()
    dev = _on_device(torch, probs, torch.float32)
    widened = [dict(p, a=d["a"].double().cpu().numpy(), b=d["b"].double().cpu().numpy()) for p, d in zip(probs, dev)]
    ref = cabi.estimate_batch(widened, streams=4, n_gpus=-1)
    _assert_same(ref, cabi.estimate_batch_device(dev, streams=4), probs, "fp32")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_inputs_are_left_untouched(torch, dtype):
    """F / H normalise their points in place; the device call must do that on its own copy."""
    probs = [p for p in _mixed_batch() if p["kind"] in ("fundamental", "homography")]
    dev = _on_device(torch, probs, getattr(torch, dtype))
    before = [(d["a"].clone(), d["b"].clone()) for d in dev]
    cabi.estimate_batch_device(dev)
    for d, (a, b) in zip(dev, before):
        assert torch.equal(d["a"], a) and torch.equal(d["b"], b)


@pytest.mark.gpu
def test_inputs_written_on_the_callers_stream_are_read_after_it(torch):
    """The inputs are produced on a side stream behind a long kernel; the call gets that stream and no host sync."""
    sleep = getattr(torch.cuda, "_sleep", None)
    if sleep is None:
        pytest.skip("torch.cuda._sleep is not available")
    probs = [p for p in _mixed_batch() if len(p["a"]) >= 100][:16]
    ref = cabi.estimate_batch(probs, streams=4, n_gpus=-1)
    src = _on_device(torch, probs, torch.float64)
    side = torch.cuda.Stream(device="cuda:0")
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        sleep(100_000_000)  # ~50 ms of device time ahead of the writes
        dev = [dict(p, a=s["a"] * 1.0, b=s["b"] + 0.0) for p, s in zip(probs, src)]
    _assert_same(ref, cabi.estimate_batch_device(dev, stream=side), probs, "stream")


@pytest.mark.gpu
def test_counters_drop_the_correspondence_and_mask_copies(torch):
    probs = [p for p in _mixed_batch() if len(p["a"]) >= 100]
    ref = cabi.estimate_batch(probs, streams=4, n_gpus=-1)
    out = cabi.estimate_batch_device(_on_device(torch, probs, torch.float64), streams=4)
    corr = sum(8 * len(p["a"]) * (5 if p["kind"] == "pnp" else 4) for p in probs)
    masks = sum(4 * ((len(p["a"]) + 31) // 32) for p in probs)
    h2d = [sum(r["counters"]["h2d_bytes"] for r in res) for res in (ref, out)]
    d2h = [sum(r["counters"]["d2h_bytes"] for r in res) for res in (ref, out)]
    assert h2d[0] - h2d[1] >= corr, (h2d, corr)
    assert d2h[0] - d2h[1] >= masks, (d2h, masks)


@pytest.mark.gpu
def test_memory_off_the_device_is_rejected_before_anything_is_written(torch):
    probs = [dict(p, n=len(p["a"])) for p in _mixed_batch() if p["kind"] == "homography" and len(p["a"]) >= 100][:3]
    dev = _on_device(torch, probs, torch.float64)
    host = [np.ascontiguousarray(p["a"]) for p in probs]
    pinned = [d["a"].cpu().pin_memory() for d in dev]
    host_mask = np.full(probs[0]["n"], 7, dtype=np.int8)

    def run(a_ptrs, mask0=None, dtype=cabi.DTYPE_F64):
        masks = [torch.full((p["n"],), 7, dtype=torch.uint8, device="cuda:0") for p in probs]
        ptrs = [m.data_ptr() for m in masks]
        if mask0 is not None:
            ptrs[0] = mask0
        rc, arr = _raw_call(probs, a_ptrs, [d["b"].data_ptr() for d in dev], ptrs, dtype)
        assert rc == cabi.PLB_ERR_ARG
        assert [q.status for q in arr] == [cabi.PLB_ERR_ARG] * len(probs)
        for q in arr:  # the start model (identity) and the stats are not written
            assert list(q.model) == [1.0, 0, 0, 0, 1.0, 0, 0, 0, 1.0] and q.stats.iterations == 0
        torch.cuda.synchronize()
        assert all(bool((m == 7).all()) for m in masks)

    dptr = [d["a"].data_ptr() for d in dev]
    run([dptr[0], host[1].ctypes.data, dptr[2]])          # pageable host memory (numpy)
    run([dptr[0], dptr[1], pinned[2].data_ptr()])         # page-locked host memory
    run(dptr, mask0=host_mask.ctypes.data)                # inliers on the host
    run([dptr[0] + 4, dptr[1], dptr[2]])                  # misaligned for fp64
    assert np.all(host_mask == 7)
    if torch.cuda.device_count() > 1:                     # memory of another GPU
        other = dev[1]["a"].to("cuda:1")
        run([dptr[0], other.data_ptr(), dptr[2]])
