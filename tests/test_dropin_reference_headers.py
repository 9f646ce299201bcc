"""The drop-in translation unit (poselib_b200/adapter/poselib_dropin.cc) is compiled against the REFERENCE'S OWN headers
(PoseLib/robust.h, robust/ransac.h, robust/bundle.h, solvers/*.h) and linked, together with libposelib_b200.so, into a
client that includes PoseLib's headers only.  Its 19 definitions must match PoseLib's declarations exactly, otherwise the
client does not link.  Eigen3 is not installed here; the Eigen stand-in of the oracle tree (oracle/ref/mini) is used at
compile time only.  Needs /root/reference (CPU container); the compiled client also has a `run` mode for a GPU box."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
EXE = os.path.join(ROOT, "oracle", "_ref", "dropin_client")

pytestmark = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "PoseLib")), reason="needs the reference's headers")


def test_dropin_defines_poselibs_own_declarations():
    import __graft_entry__ as ge
    ge.build()  # builds the library and, where the reference is mounted, oracle/_ref/dropin_client (build_dropin_client)
    out = subprocess.run([EXE], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "dropin link ok: 19 PoseLib entry points resolved" in out.stdout, out.stdout + out.stderr


def test_the_same_client_passes_on_poselibs_own_cpu_implementation():
    """The client's `run` mode (one PoseLib-style call of every estimate_*, ransac_relpose, refine_relpose, relpose_5pt on
    synthetic scenes with ground truth, with accuracy / inlier-count checks) is first held to PoseLib ITSELF: linked with the
    reference's own sources (the mini-Eigen build, `make -C oracle ref2`) instead of the drop-in, it must pass.  The GPU
    test (tests/test_zz_golden_reference_gpu.py) then runs the identical client on the CUDA backend."""
    import glob
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "ref2"], stdout=subprocess.DEVNULL,
                          stderr=subprocess.DEVNULL)
    objs = [o for o in glob.glob(os.path.join(ROOT, "oracle", "_build", "ref2obj", "**", "*.o"), recursive=True)
            if not o.endswith("ref2_capi.o")]
    exe = os.path.join(ROOT, "tests", "_dropin_client_ref")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-w", "-I" + os.path.join(ROOT, "oracle", "ref", "mini"),
                           "-I" + os.path.join(ROOT, "oracle"), "-I" + REF, os.path.join(ROOT, "tests", "dropin_client_test.cc"),
                           *objs, "-Wl,--unresolved-symbols=ignore-all", "-o", exe])
    out = subprocess.run([exe, "run"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "dropin run ok" in out.stdout, out.stdout + out.stderr

