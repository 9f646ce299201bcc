// Compile-and-link test of the adapter's camera-refinement surface (BundleOptions::refine_* mapped onto
// plb_bundle_opt.refine_intrinsics, estimate_absolute_pose writing the camera back, bundle_adjust_image) against the same
// kind of stand-ins for the Eigen / PoseLib types as tests/adapter_compile_test.cc.  Built and run by
// tests/test_adapter_intrinsics.py; `run` (GPU) refines a perturbed focal length.
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
struct Image {
    CameraPose pose;
    Camera camera;
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
struct AbsolutePoseOptions {
    RansacOptions ransac;
    BundleOptions bundle;
    double max_error = 12.0;
    bool estimate_focal_length = false, estimate_extra_params = false;
};
struct RelativePoseOptions {
    RansacOptions ransac;
    BundleOptions bundle;
    double max_error = 1.0;
    bool tangent_sampson = false, real_focal_check = false;
};
struct HomographyOptions {
    RansacOptions ransac;
    BundleOptions bundle;
    double max_error = 1.0;
};
struct BundleStats { // types.h:97-106, the fields the adapter fills
    size_t iterations = 0;
    double initial_cost = 0, cost = 0;
};
} // namespace standin

int main(int argc, char **argv) {
    using namespace standin;
    BundleOptions bo;
    bo.refine_focal_length = true;
    bo.refine_principal_point = true;
    bo.refine_extra_params = true;
    const plb_bundle_opt c = poselib_b200::detail::bundle_to_c(bo);
    if (c.refine_intrinsics != (PLB_REFINE_FOCAL_LENGTH | PLB_REFINE_PRINCIPAL_POINT | PLB_REFINE_EXTRA_PARAMS)) return 1;
    bo.refine_principal_point = bo.refine_extra_params = false;
    if (poselib_b200::detail::bundle_to_c(bo).refine_intrinsics != PLB_REFINE_FOCAL_LENGTH) return 1;
    // synthetic PINHOLE scene: 200 points, focal 800; the camera starts at focal 808
    const int n = 200;
    std::vector<Vector2d> x(n);
    std::vector<Vector3d> X(n);
    for (int i = 0; i < n; ++i) {
        const double a = 0.37 * i, b = 0.11 * i;
        X[i] = Vector3d{{std::sin(a), std::cos(1.3 * a) * 0.7, 4.0 + std::sin(b)}};
        x[i] = Vector2d{{800.0 * X[i](0) / X[i](2) + 320.0, 800.0 * X[i](1) / X[i](2) + 240.0}};
    }
    Image image;
    image.camera.model_id = 1;
    image.camera.params = {808.0, 808.0, 320.0, 240.0};
    AbsolutePoseOptions opt;
    opt.bundle.refine_focal_length = true;
    opt.max_error = 4.0;
    std::vector<char> inliers;
    if (argc > 1 && std::strcmp(argv[1], "run") == 0) {
        RansacStats st = poselib_b200::estimate_absolute_pose<RansacStats>(x, X, opt, &image, &inliers);
        if (image.camera.params.size() != 4 || st.num_inliers < 190 || std::fabs(image.camera.params[0] - 800.0) > 1.0)
            return 3;
        image.camera.params = {808.0, 808.0, 320.0, 240.0};
        poselib_b200::bundle_adjust_image<BundleStats>(x, X, &image, opt.bundle); // link / instantiation
        if (std::fabs(image.camera.params[0] - 800.0) > 1.0) return 4;
        std::printf("adapter intrinsics run ok\n");
        return 0;
    }
    // instantiate without running (link check)
    if (argc > 5) {
        poselib_b200::estimate_absolute_pose<RansacStats>(x, X, opt, &image, &inliers);
        poselib_b200::bundle_adjust_image<BundleStats>(x, X, &image, opt.bundle);
    }
    std::printf("adapter intrinsics link ok\n");
    return 0;
}
