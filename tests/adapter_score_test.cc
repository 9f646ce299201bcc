// The adapter's score_* templates against stand-ins for the Eigen / PoseLib types.  Built and run by
// tests/test_score_batch.py; `run` (GPU) checks each template against the C-ABI call it wraps, bit for bit (scores,
// counts, masks), on a small synthetic problem; without `run` it only links.
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
struct Matrix3d { // column-major, as Eigen::Matrix3d
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
} // namespace standin

using namespace standin;

namespace {
int failures = 0;
void expect(bool ok, const char *what) {
    if (!ok) {
        std::printf("FAILED: %s\n", what);
        ++failures;
    }
}
// the C-ABI call the template wraps, on the same rows
poselib_b200::ScoreResult direct(int kind, int ts, const std::vector<double> &a, const std::vector<double> &b, size_t n,
                                 const std::vector<double> &rows, size_t m, double sq, const plb_camera *c1,
                                 const plb_camera *c2) {
    poselib_b200::ScoreResult r;
    r.scores.assign(m, 0.0);
    r.num_inliers.assign(m, 0);
    std::vector<char> flat(m * n);
    plb_score_problem q = plb_score_problem();
    q.kind = kind;
    q.tangent_sampson = ts;
    q.n = n;
    q.a = a.data();
    q.b = b.data();
    q.camera1.model_id = q.camera2.model_id = PLB_CAMERA_NULL;
    if (c1) q.camera1 = *c1;
    if (c2) q.camera2 = *c2;
    q.m = m;
    q.models = rows.data();
    q.sq_threshold = sq;
    q.scores = r.scores.data();
    q.num_inliers = r.num_inliers.data();
    q.inliers = flat.data();
    if (plb_score_batch(&q, 1, -1, 1) != PLB_OK) std::printf("FAILED: plb_score_batch: %s\n", plb_last_error()), ++failures;
    for (size_t i = 0; i < m; ++i) r.inliers.emplace_back(flat.begin() + i * n, flat.begin() + (i + 1) * n);
    return r;
}
bool same(const poselib_b200::ScoreResult &x, const poselib_b200::ScoreResult &y) {
    return x.scores.size() == y.scores.size() &&
           std::memcmp(x.scores.data(), y.scores.data(), sizeof(double) * x.scores.size()) == 0 &&
           x.num_inliers == y.num_inliers && x.inliers == y.inliers;
}
} // namespace

int main(int argc, char **argv) {
    const bool run = argc > 1 && std::strcmp(argv[1], "run") == 0;
    const size_t n = 300;
    std::vector<Vector2d> x1(n), x2(n), x(n);
    std::vector<Vector3d> X(n);
    for (size_t k = 0; k < n; ++k) {
        const double u = std::sin(0.37 * k), v = std::cos(0.23 * k), w = 5.0 + std::sin(0.11 * k);
        X[k] = Vector3d{{u, v, w}};
        x[k] = Vector2d{{u / w + 1e-4 * (k % 7 == 0), v / w}};
        x1[k] = Vector2d{{u / w, v / w}};
        x2[k] = Vector2d{{(u + 0.3) / w + 2e-3 * (k % 5 == 0), v / w}};
    }
    std::vector<CameraPose> poses(3);
    poses[1].t = Vector3d{{-0.3, 0.0, 0.0}};
    poses[2].q = Vector4d{{0.0, 1.0, 0.0, 0.0}};
    std::vector<Matrix3d> mats(2);
    mats[0] = Matrix3d{{1, 0, 0, 0, 1, 0, 0.3 / 5.0, 0, 1}};
    mats[1] = Matrix3d{{0, 0, 0, 0, -0.3, 0, 0, 0.3, 0}};
    Camera cam;
    cam.model_id = 1;
    cam.params = {500.0, 500.0, 0.0, 0.0};
    std::vector<Vector2d> p1(n), p2(n);
    for (size_t k = 0; k < n; ++k) {
        p1[k] = Vector2d{{500.0 * x1[k](0), 500.0 * x1[k](1)}};
        p2[k] = Vector2d{{500.0 * x2[k](0), 500.0 * x2[k](1)}};
    }
    if (!run) {
        // instantiate every template; the library is linked but not called
        auto f0 = &poselib_b200::score_absolute_poses<Vector2d, Vector3d, CameraPose>;
        auto f1 = static_cast<poselib_b200::ScoreResult (*)(const std::vector<Vector2d> &, const std::vector<Vector2d> &,
                                                            const std::vector<CameraPose> &, double, bool)>(
            &poselib_b200::score_relative_poses<Vector2d, CameraPose>);
        auto f2 = static_cast<poselib_b200::ScoreResult (*)(const std::vector<Vector2d> &, const std::vector<Vector2d> &,
                                                            const Camera &, const Camera &,
                                                            const std::vector<CameraPose> &, double, bool)>(
            &poselib_b200::score_relative_poses<Vector2d, Camera, CameraPose>);
        auto f3 = &poselib_b200::score_fundamentals<Vector2d, Matrix3d>;
        auto f4 = &poselib_b200::score_homographies<Vector2d, Matrix3d>;
        expect(f0 && f1 && f2 && f3 && f4, "templates instantiate");
        std::printf("adapter score link ok\n");
        return failures ? 1 : 0;
    }
    auto raw = [](const auto &v) {
        const double *p = reinterpret_cast<const double *>(v.data());
        return std::vector<double>(p, p + sizeof(v[0]) / sizeof(double) * v.size());
    };
    const std::vector<double> prow = raw(poses), mrow = raw(mats);
    const plb_camera c = poselib_b200::detail::camera_to_c(cam);
    expect(same(poselib_b200::score_absolute_poses(x, X, poses, 1e-6, true),
                direct(PLB_KIND_PNP, 0, raw(x), raw(X), n, prow, 3, 1e-6, nullptr, nullptr)), "pnp");
    expect(same(poselib_b200::score_relative_poses(x1, x2, poses, 1e-6, true),
                direct(PLB_KIND_RELPOSE, 0, raw(x1), raw(x2), n, prow, 3, 1e-6, nullptr, nullptr)), "relpose");
    expect(same(poselib_b200::score_relative_poses(p1, p2, cam, cam, poses, 0.25, true),
                direct(PLB_KIND_RELPOSE, 1, raw(p1), raw(p2), n, prow, 3, 0.25, &c, &c)), "tangent Sampson");
    expect(same(poselib_b200::score_fundamentals(x1, x2, mats, 1e-6, true),
                direct(PLB_KIND_FUNDAMENTAL, 0, raw(x1), raw(x2), n, mrow, 2, 1e-6, nullptr, nullptr)), "fundamental");
    expect(same(poselib_b200::score_homographies(x1, x2, mats, 1e-6, true),
                direct(PLB_KIND_HOMOGRAPHY, 0, raw(x1), raw(x2), n, mrow, 2, 1e-6, nullptr, nullptr)), "homography");
    const poselib_b200::ScoreResult no = poselib_b200::score_relative_poses(x1, x2, poses, 1e-6);
    expect(no.inliers.empty() && no.scores.size() == 3, "no masks unless asked for");
    std::printf(failures ? "adapter score FAILED\n" : "adapter score ok\n");
    return failures ? 1 : 0;
}
