import os
import sys


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


LIB = os.path.join(ROOT, "poselib_b200", "libposelib_b200.so")
# test modules that load the CUDA C-ABI library (directly or through poselib_b200.pyapi)
NEEDS_LIB = {"test_a_device_control.py", "test_cabi_exports.py", "test_gpu_parity.py", "test_host_logic.py",
             "test_multi_gpu.py", "test_pyapi.py", "test_ref_pins.py", "test_zz_golden_reference_gpu.py", "test_adapter.py",
             "test_dropin_reference_headers.py"}


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")
    # Several test modules import the C-ABI binding at collection time; it refuses to load without the in-tree library.
    # A fresh checkout that runs pytest before __graft_entry__.build() would otherwise fail to collect.
    if not (os.path.exists(LIB) and os.path.exists(os.path.join(ROOT, "oracle", "_build", "libplo.so"))):
        import shutil
        import subprocess
        if shutil.which("nvcc"):
            import __graft_entry__ as ge
            ge.build()
        else:  # no CUDA toolkit on this machine: the oracle, reference-pin and fixture tests still run
            subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s"])


def pytest_ignore_collect(collection_path, config):
    """Without the CUDA library (no nvcc to build it) only the modules that need it are left out."""
    if collection_path.name in NEEDS_LIB and not os.path.exists(LIB):
        return True
    return None
