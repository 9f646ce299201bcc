// The adapter's batch refiners, refine_relpose_batch and bundle_adjust_image_batch, against the stand-ins for the Eigen /
// PoseLib types of tests/adapter_weights_test.cc.  Built and run by tests/test_refine_batch.py; `run` (GPU) checks that
// every element of a batch equals the adapter's single call on it bit for bit (pose, camera, stats), with weights of size
// n, of the wrong size (uniform) and missing; without `run`, that batches of mismatched sizes throw.
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
struct BundleStats { // types.h:97-106, the fields the adapter fills
    size_t iterations = 0;
    double initial_cost = 0, cost = 0;
};
} // namespace standin

using namespace standin;

namespace {
int failures = 0;
void expect(bool ok, const char *what, size_t i) {
    if (!ok) {
        std::printf("FAILED: %s (element %zu)\n", what, i);
        ++failures;
    }
}
bool same_pose(const CameraPose &a, const CameraPose &b) {
    return std::memcmp(a.q.d, b.q.d, sizeof(a.q.d)) == 0 && std::memcmp(a.t.d, b.t.d, sizeof(a.t.d)) == 0;
}
bool same_stats(const BundleStats &a, const BundleStats &b) {
    return a.iterations == b.iterations && std::memcmp(&a.initial_cost, &b.initial_cost, sizeof(double)) == 0 &&
           std::memcmp(&a.cost, &b.cost, sizeof(double)) == 0;
}
} // namespace

int main(int argc, char **argv) {
    // problem k: a PINHOLE scene of n_k points seen from two views; every 9th observation is an outlier
    const int sizes[] = {0, 7, 300, 2500};
    const int count = 4;
    std::vector<std::vector<Vector2d>> xs(count), x1s(count), x2s(count);
    std::vector<std::vector<Vector3d>> Xs(count);
    std::vector<std::vector<double>> ws(count);
    for (int k = 0; k < count; ++k) {
        const int n = sizes[k];
        for (int i = 0; i < n; ++i) {
            const double a = 0.37 * i + k, b = 0.11 * i;
            const Vector3d X{{std::sin(a), std::cos(1.3 * a) * 0.7, 4.0 + std::sin(b)}};
            const double Y0 = X(0) - 0.5, Y1 = X(1) + 0.05, Y2 = X(2) + 0.1; // second camera: a translation
            Xs[k].push_back(X);
            xs[k].push_back(Vector2d{{800.0 * X(0) / X(2) + 320.0 + (i % 9 == 4 ? 25.0 : 0.0), 800.0 * X(1) / X(2) + 240.0}});
            x1s[k].push_back(Vector2d{{X(0) / X(2), X(1) / X(2)}});
            x2s[k].push_back(Vector2d{{Y0 / Y2, Y1 / Y2 + (i % 9 == 4 ? 0.03 : 0.0)}});
            ws[k].push_back(i % 9 == 4 ? 0.05 : (i % 10 == 7 ? 0.0 : 0.5 + 0.01 * (i % 50)));
        }
    }
    ws[1].pop_back(); // the wrong size: uniform weights
    ws.pop_back();    // no entry for the last problem: uniform weights
    { // batches of mismatched sizes are refused before any device call
        BundleOptions bo;
        std::vector<CameraPose> short_poses(count - 1);
        std::vector<Image> short_images(count - 1);
        bool thrown = false;
        try {
            poselib_b200::refine_relpose_batch<BundleStats>(x1s, x2s, &short_poses, bo, ws);
        } catch (const std::invalid_argument &) {
            thrown = true;
        }
        expect(thrown, "refine_relpose_batch refuses mismatched sizes", 0);
        thrown = false;
        try {
            poselib_b200::bundle_adjust_image_batch<BundleStats>(xs, Xs, &short_images, bo, ws);
        } catch (const std::invalid_argument &) {
            thrown = true;
        }
        expect(thrown, "bundle_adjust_image_batch refuses mismatched sizes", 0);
        if (failures) return 1;
    }
    if (argc > 1 && std::strcmp(argv[1], "run") == 0) {
        BundleOptions bo;
        bo.loss_scale = 2.0 / 800.0;
        CameraPose p0;
        p0.q = Vector4d{{0.9999, 0.01, -0.005, 0.002}};
        p0.t = Vector3d{{-0.5, 0.05, 0.1}};
        std::vector<CameraPose> poses(count, p0);
        const std::vector<BundleStats> st = poselib_b200::refine_relpose_batch<BundleStats>(x1s, x2s, &poses, bo, ws);
        for (int k = 0; k < count; ++k) {
            CameraPose p = p0;
            const BundleStats s = poselib_b200::refine_relpose<BundleStats>(x1s[k], x2s[k], &p, bo,
                                                                           k < (int)ws.size() ? ws[k] : std::vector<double>());
            expect(same_pose(p, poses[k]), "refine_relpose_batch pose", k);
            expect(same_stats(s, st[k]), "refine_relpose_batch stats", k);
        }
        BundleOptions bi;
        bi.loss_scale = 2.0;
        bi.refine_focal_length = true;
        Image img0;
        img0.pose.q = p0.q;
        img0.pose.t = Vector3d{{0.01, -0.02, 0.01}};
        img0.camera.model_id = 1;
        img0.camera.params = {808.0, 805.0, 321.0, 239.0};
        std::vector<Image> images(count, img0);
        const std::vector<BundleStats> si = poselib_b200::bundle_adjust_image_batch<BundleStats>(xs, Xs, &images, bi, ws);
        for (int k = 0; k < count; ++k) {
            Image img = img0;
            const BundleStats s = poselib_b200::bundle_adjust_image<BundleStats>(xs[k], Xs[k], &img, bi,
                                                                                k < (int)ws.size() ? ws[k] : std::vector<double>());
            expect(same_pose(img.pose, images[k].pose), "bundle_adjust_image_batch pose", k);
            expect(img.camera.params == images[k].camera.params, "bundle_adjust_image_batch camera", k);
            expect(same_stats(s, si[k]), "bundle_adjust_image_batch stats", k);
        }
        expect(si[3].iterations > 0 && images[3].camera.params[0] != 808.0, "the focal length is refined", 3);
        if (failures) return 1;
        std::printf("adapter refine batch run ok\n");
        return 0;
    }
    std::printf("adapter refine batch link ok\n");
    return 0;
}
