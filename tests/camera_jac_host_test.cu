// CPU-side check of the camera-refinement pieces of poselib_b200/csrc/camera.cuh, compiled for the host from the same
// source the device runs (as tests/camera_host_test.cu does): cam_jac_params of camera-frame points and cam_refine_idx
// for the eight refine flag sets, printed as hex doubles / integers for tests/test_intrinsics_refine.py.
#include "../poselib_b200/csrc/camera.cuh"
#include <cstdio>
#include <cstdlib>

using namespace plb;

int main(int argc, char **argv) {
    // argv: model p0..p7 then triples X Y Z
    if (argc < 10) return 2;
    CamDev c;
    c.model = std::atoi(argv[1]);
    c.reserved = 0;
    for (int i = 0; i < 8; ++i) c.p[i] = std::strtod(argv[2 + i], nullptr);
    for (int flags = 0; flags < 8; ++flags) {
        int idx[CAM_MAX_PARAMS];
        const int m = cam_refine_idx(c.model, flags, idx);
        std::printf("idx %d", m);
        for (int i = 0; i < m; ++i) std::printf(" %d", idx[i]);
        std::printf("\n");
    }
    for (int a = 10; a + 2 < argc; a += 3) {
        const double X = std::strtod(argv[a], nullptr), Y = std::strtod(argv[a + 1], nullptr),
                     Z = std::strtod(argv[a + 2], nullptr);
        double jp[2 * CAM_MAX_PARAMS] = {0};
        cam_jac_params(c, X, Y, Z, jp);
        std::printf("jp");
        for (int i = 0; i < 2 * CAM_MAX_PARAMS; ++i) std::printf(" %a", jp[i]);
        std::printf("\n");
    }
    return 0;
}
