// Compile-and-run test of the adapter's relative-pose camera refinement: refine_relpose_pair (ImagePair*) and
// estimate_relative_pose with tangent_sampson and refine_* flags, against stand-ins for the Eigen / PoseLib types as in
// tests/adapter_intrinsics_compile_test.cc.  Built and run by tests/test_relpose_intrinsics_refine.py; `run` (GPU) refines
// perturbed focal lengths of a two-view scene.
#include "../poselib_b200/adapter/poselib_b200.hpp"

#include <cmath>
#include <cstdio>
#include <cstring>

namespace standin {
template <int N> struct Vec {
    double d[N];
    double &operator()(int i) { return d[i]; }
    double operator()(int i) const { return d[i]; }
};
using Vector2d = Vec<2>;
using Vector3d = Vec<3>;
using Vector4d = Vec<4>;
struct Matrix3d { // column-major
    double d[9];
};
struct CameraPose { // camera_pose.h:40-68
    Vector4d q{{1, 0, 0, 0}};
    Vector3d t{{0, 0, 0}};
};
struct Camera { // misc/camera_models.h:59-63
    int model_id = -1, width = 0, height = 0;
    std::vector<double> params;
};
struct ImagePair { // camera_pose.h:124-132
    CameraPose pose;
    Camera camera1, camera2;
};
struct RansacOptions { // types.h:39-50
    size_t max_iterations = 100000, min_iterations = 1000;
    double dyn_num_trials_mult = 3.0, success_prob = 0.9999;
    unsigned long seed = 0;
    bool progressive_sampling = false;
    size_t max_prosac_iterations = 100000;
    bool score_initial_model = false;
};
struct RansacStats { // types.h:52-58
    size_t refinements = 0, iterations = 0, num_inliers = 0;
    double inlier_ratio = 0, model_score = 0;
};
struct BundleOptions { // types.h:60-95
    size_t max_iterations = 100;
    enum LossType { TRIVIAL, TRUNCATED, HUBER, CAUCHY, TRUNCATED_CAUCHY, TRUNCATED_LE_ZACH } loss_type = CAUCHY;
    double loss_scale = 1.0, gradient_tol = 1e-12, step_tol = 1e-8, relative_cost_tol = 1e-10, initial_lambda = 1e-3,
           min_lambda = 1e-10, max_lambda = 1e10;
    bool verbose = false;
    enum LambdaUpdateType { NIELSEN, FIXED_FACTOR } lambda_update = NIELSEN;
    double lambda_factor = 10.0;
    enum DampingType { LEVENBERG, MARQUARDT } damping = LEVENBERG;
    bool refine_focal_length = false, refine_extra_params = false, refine_principal_point = false;
};
struct RelativePoseOptions {
    RansacOptions ransac;
    BundleOptions bundle;
    double max_error = 1.0;
    bool tangent_sampson = false, real_focal_check = false;
};
struct BundleStats { // types.h:97-106, the fields the adapter fills
    size_t iterations = 0;
    double initial_cost = 0, cost = 0;
};
} // namespace standin

int main(int argc, char **argv) {
    using namespace standin;
    // synthetic SIMPLE_PINHOLE pair: focal 800, camera 2 rotated 0.2 rad about y and moved along x
    const int n = 300;
    const double c = std::cos(0.2), s = std::sin(0.2), t[3] = {-0.995, 0.0998, 0.0};
    std::vector<Vector2d> x1(n), x2(n);
    for (int i = 0; i < n; ++i) {
        const double a = 0.37 * i, b = 0.11 * i;
        const double X = 1.5 * std::sin(a), Y = std::cos(1.3 * a), Z = 4.0 + 2.0 * std::sin(b);
        const double X2 = c * X + s * Z + t[0], Y2 = Y + t[1], Z2 = -s * X + c * Z + t[2];
        x1[i] = Vector2d{{800.0 * X / Z + 320.0, 800.0 * Y / Z + 240.0}};
        x2[i] = Vector2d{{800.0 * X2 / Z2 + 320.0, 800.0 * Y2 / Z2 + 240.0}};
    }
    ImagePair pair;
    pair.pose.q = Vector4d{{std::cos(0.1), 0.0, std::sin(0.1), 0.0}};
    pair.pose.t = Vector3d{{t[0], t[1], t[2]}};
    pair.camera1.model_id = pair.camera2.model_id = 0;
    pair.camera1.params = pair.camera2.params = {808.0, 320.0, 240.0};
    RelativePoseOptions opt;
    opt.bundle.refine_focal_length = true;
    opt.tangent_sampson = true;
    opt.max_error = 2.0;
    if (argc > 1 && std::strcmp(argv[1], "run") == 0) {
        BundleStats b = poselib_b200::refine_relpose_pair<BundleStats>(x1, x2, &pair, opt.bundle);
        if (!(b.cost < b.initial_cost) || std::fabs(pair.camera1.params[0] - 800.0) > 4.0 ||
            std::fabs(pair.camera2.params[0] - 800.0) > 4.0)
            return 3;
        const Camera cam1 = pair.camera1, cam2 = pair.camera2;
        CameraPose pose;
        std::vector<char> inliers;
        RansacStats st = poselib_b200::estimate_relative_pose<RansacStats>(x1, x2, cam1, cam2, opt, &pose, &inliers);
        if (st.num_inliers < 290 || std::fabs(pose.q(2) - std::sin(0.1)) > 1e-3) return 4;
        std::printf("adapter relpose intrinsics run ok\n");
        return 0;
    }
    // instantiate without running (link check)
    if (argc > 5) {
        CameraPose pose;
        std::vector<char> inliers;
        poselib_b200::refine_relpose_pair<BundleStats>(x1, x2, &pair, opt.bundle);
        poselib_b200::estimate_relative_pose<RansacStats>(x1, x2, pair.camera1, pair.camera2, opt, &pose, &inliers);
    }
    std::printf("adapter relpose intrinsics link ok\n");
    return 0;
}
