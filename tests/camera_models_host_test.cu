// CPU-side check of every camera function of poselib_b200/csrc/camera.cuh, compiled for the host from the same source
// the device runs (the instantiations with the fisheye and division models, X = true): per pixel the bearing, the hnormalized point and unproject_with_jac with and without parameters; per
// camera-frame point project, project_with_jac and jac_params; refinement indices of the eight flag sets, focal and
// rescale.  Printed as hex doubles / integers for tests/test_camera_models.py.
#include "../poselib_b200/csrc/camera.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>

using namespace plb;

static void put(const double *v, int n) {
    for (int i = 0; i < n; ++i) std::printf(" %a", v[i]);
}

int main(int argc, char **argv) {
    // argv: model p0..p7 scale, then "px" u v pairs or "pt" X Y Z triples until the end
    if (argc < 11) return 2;
    CamDev c;
    c.model = std::atoi(argv[1]);
    c.reserved = 0;
    for (int i = 0; i < 8; ++i) c.p[i] = std::strtod(argv[2 + i], nullptr);
    const double scale = std::strtod(argv[10], nullptr);
    for (int flags = 0; flags < 8; ++flags) {
        int idx[CAM_MAX_PARAMS];
        const int m = cam_refine_idx(c.model, flags, idx);
        std::printf("idx %d", m);
        for (int i = 0; i < m; ++i) std::printf(" %d", idx[i]);
        std::printf("\n");
    }
    CamDev r = c;
    cam_rescale(r, scale);
    const double f = cam_focal(c);
    std::printf("focal");
    put(&f, 1);
    std::printf("\nrescale");
    put(r.p, 8);
    std::printf("\n");
    const bool px = argc > 11 && std::strcmp(argv[11], "px") == 0;
    const int step = px ? 2 : 3;
    for (int a = 12; a + step - 1 < argc; a += step) {
        if (px) {
            const double u = std::strtod(argv[a], nullptr), v = std::strtod(argv[a + 1], nullptr);
            double x[3], ox, oy, d[3], M[6], e[3], N[6], dp[3 * CAM_MAX_PARAMS] = {0};
            cam_unproject<true>(c, u, v, x);
            cam_unproject2<true>(c, u, v, ox, oy);
            cam_unproject_with_jac<true>(c, u, v, d, M);
            cam_unproject_with_jac_params<true>(c, u, v, e, N, dp);
            std::printf("px");
            put(x, 3);
            std::printf(" %a %a", ox, oy);
            put(d, 3);
            put(M, 6);
            put(e, 3);
            put(N, 6);
            put(dp, 3 * CAM_MAX_PARAMS);
        } else {
            const double X = std::strtod(argv[a], nullptr), Y = std::strtod(argv[a + 1], nullptr),
                         Z = std::strtod(argv[a + 2], nullptr);
            double u, v, pu, pv, J[6], jp[2 * CAM_MAX_PARAMS] = {0};
            cam_project<true>(c, X, Y, Z, u, v);
            cam_project_with_jac<true>(c, X, Y, Z, pu, pv, J);
            cam_jac_params<true>(c, X, Y, Z, jp);
            std::printf("pt %a %a %a %a", u, v, pu, pv);
            put(J, 6);
            put(jp, 2 * CAM_MAX_PARAMS);
        }
        std::printf("\n");
    }
    return 0;
}
