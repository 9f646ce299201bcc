"""The adapter's camera-refinement surface compiles and links with the refine_* flags set (stand-in Eigen / PoseLib
types, tests/adapter_intrinsics_compile_test.cc); with a GPU the drop-in estimate_absolute_pose refines a focal length."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "poselib_b200", "libposelib_b200.so")

pytestmark = pytest.mark.skipif(not os.path.exists(LIB), reason="libposelib_b200.so not built")


def _build(tmp_path):
    exe = str(tmp_path / "adapter_intrinsics_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "adapter_intrinsics_compile_test.cc"),
                           "-o", exe, "-L" + os.path.join(ROOT, "poselib_b200"), "-lposelib_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "poselib_b200")])
    return exe


def test_adapter_intrinsics_compiles_and_links(tmp_path):
    out = subprocess.run([_build(tmp_path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "adapter intrinsics link ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_adapter_estimate_absolute_pose_refines_the_focal_length(tmp_path):
    out = subprocess.run([_build(tmp_path), "run"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "adapter intrinsics run ok" in out.stdout, (out.returncode, out.stdout + out.stderr)
