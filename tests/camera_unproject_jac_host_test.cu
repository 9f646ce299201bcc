// CPU-side check of cam_unproject_with_jac_params (poselib_b200/csrc/camera.cuh), compiled for the host from the same
// source the device runs: bearings and jac_params of pixels, printed as hex doubles for
// tests/test_relpose_intrinsics_refine.py.
#include "../poselib_b200/csrc/camera.cuh"
#include <cstdio>
#include <cstdlib>

using namespace plb;

int main(int argc, char **argv) {
    // argv: model p0..p7 then pairs u v
    if (argc < 10) return 2;
    CamDev c;
    c.model = std::atoi(argv[1]);
    c.reserved = 0;
    for (int i = 0; i < 8; ++i) c.p[i] = std::strtod(argv[2 + i], nullptr);
    for (int a = 10; a + 1 < argc; a += 2) {
        double d[3], M[6], dp[3 * CAM_MAX_PARAMS] = {0};
        cam_unproject_with_jac_params(c, std::strtod(argv[a], nullptr), std::strtod(argv[a + 1], nullptr), d, M, dp);
        std::printf("d");
        for (int i = 0; i < 3; ++i) std::printf(" %a", d[i]);
        for (int i = 0; i < 3 * CAM_MAX_PARAMS; ++i) std::printf(" %a", dp[i]);
        std::printf("\n");
    }
    return 0;
}
