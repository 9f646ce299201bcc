// Test client of PoseLib's own camera-refinement code: Camera::project_with_jac with jac_params,
// Camera::get_param_refinement_idx, bundle_adjust(x, X, Image*, opt) and estimate_absolute_pose with the refine_* flags,
// called through a C interface.  It is compiled against the reference's headers and linked with the reference's sources
// built on mini-Eigen (oracle/_ref/libplref2.so, `make -C oracle ref2`); tests/golden/make_intrinsics_golden.py builds it.
#include "PoseLib/misc/camera_models.h"
#include "PoseLib/robust.h"
#include "PoseLib/robust/bundle.h"

#include <cstdint>
#include <vector>

using namespace poselib;

namespace {
const int NP[] = {3, 4, 4, 5, 8};
Camera camera(int model, const double *params) {
    Camera c;
    c.model_id = model;
    c.width = c.height = 0;
    c.params.clear();
    if (model >= 0 && model <= 4) c.params.assign(params, params + NP[model]);
    return c;
}
// loss type, loss scale, max_iterations and the three refine flags; the other fields keep their defaults
BundleOptions bundle(int loss_type, double loss_scale, int max_iterations, int flags) {
    BundleOptions b;
    b.loss_type = (BundleOptions::LossType)loss_type;
    b.loss_scale = loss_scale;
    b.max_iterations = max_iterations;
    b.refine_focal_length = (flags & 1) != 0;
    b.refine_principal_point = (flags & 2) != 0;
    b.refine_extra_params = (flags & 4) != 0;
    return b;
}
std::vector<Point2D> v2(const double *a, int64_t n) {
    std::vector<Point2D> v(n);
    for (int64_t k = 0; k < n; ++k) v[k] = Point2D(a[2 * k], a[2 * k + 1]);
    return v;
}
std::vector<Point3D> v3(const double *a, int64_t n) {
    std::vector<Point3D> v(n);
    for (int64_t k = 0; k < n; ++k) v[k] = Point3D(a[3 * k], a[3 * k + 1], a[3 * k + 2]);
    return v;
}
CameraPose pose_in(const double *p) {
    CameraPose q;
    for (int i = 0; i < 4; ++i) q.q(i) = p[i];
    for (int i = 0; i < 3; ++i) q.t(i) = p[4 + i];
    return q;
}
void pose_out(const CameraPose &q, double *p) {
    for (int i = 0; i < 4; ++i) p[i] = q.q(i);
    for (int i = 0; i < 3; ++i) p[4 + i] = q.t(i);
}
} // namespace

extern "C" {
// Camera::get_param_refinement_idx -> idx (up to 8); returns the count
int ri_refine_idx(int model, const double *params, int flags, int *idx) {
    Camera c = camera(model, params);
    const std::vector<size_t> v = c.get_param_refinement_idx(bundle(0, 1.0, 100, flags));
    for (size_t i = 0; i < v.size(); ++i) idx[i] = (int)v[i];
    return (int)v.size();
}
// Camera::project_with_jac of n points Z (3n): xp (2n), jac (6n, row-major 2x3), jac_params (16n, row-major 2x8, columns
// past the model's parameter count untouched)
void ri_project_with_jac(int model, const double *params, int64_t n, const double *Z, double *xp, double *jac,
                         double *jp) {
    Camera c = camera(model, params);
    for (int64_t k = 0; k < n; ++k) {
        Eigen::Vector2d p;
        Eigen::Matrix<double, 2, 3> J;
        Eigen::Matrix<double, 2, Eigen::Dynamic> Jp;
        c.project_with_jac(Eigen::Vector3d(Z[3 * k], Z[3 * k + 1], Z[3 * k + 2]), &p, &J, &Jp);
        xp[2 * k] = p(0);
        xp[2 * k + 1] = p(1);
        for (int r = 0; r < 2; ++r)
            for (int q = 0; q < 3; ++q) jac[6 * k + 3 * r + q] = J(r, q);
        for (int r = 0; r < 2; ++r)
            for (int q = 0; q < (int)Jp.cols(); ++q) jp[16 * k + 8 * r + q] = Jp(r, q);
    }
}
// bundle_adjust(x, X, Image*, opt) (robust/bundle.h:47); pose (7) and params in/out; stats: iterations, initial, cost
void ri_bundle_adjust_image(int model, double *params, int64_t n, const double *x, const double *X, double *pose,
                            int loss_type, double loss_scale, int max_iterations, double relative_cost_tol, int flags,
                            double *stats) {
    Image image;
    image.camera = camera(model, params);
    image.pose = pose_in(pose);
    BundleOptions o = bundle(loss_type, loss_scale, max_iterations, flags);
    o.relative_cost_tol = relative_cost_tol;
    const BundleStats s = bundle_adjust(v2(x, n), v3(X, n), &image, o);
    pose_out(image.pose, pose);
    for (int i = 0; i < NP[model]; ++i) params[i] = image.camera.params[i];
    stats[0] = (double)s.iterations;
    stats[1] = s.initial_cost;
    stats[2] = s.cost;
}
// estimate_absolute_pose(points2D, points3D, opt, Image*, inliers) (robust.h:45-46) with the default RansacOptions
// except max_iterations / min_iterations / seed; stats: iterations, refinements, num_inliers, model_score
void ri_estimate_absolute_pose(int model, double *params, int64_t n, const double *x, const double *X, double max_error,
                               uint64_t max_iterations, uint64_t min_iterations, uint64_t seed, int flags, double *pose,
                               char *inliers, double *stats) {
    AbsolutePoseOptions o;
    o.ransac.max_iterations = max_iterations;
    o.ransac.min_iterations = min_iterations;
    o.ransac.seed = seed;
    o.bundle = bundle(3, 1.0, 100, flags);
    o.max_error = max_error;
    Image image;
    image.camera = camera(model, params);
    image.pose = pose_in(pose);
    std::vector<char> m(n, 0);
    const RansacStats s = estimate_absolute_pose(v2(x, n), v3(X, n), o, &image, &m);
    pose_out(image.pose, pose);
    for (int i = 0; i < NP[model]; ++i) params[i] = image.camera.params[i];
    for (int64_t k = 0; k < n; ++k) inliers[k] = m[k];
    stats[0] = (double)s.iterations;
    stats[1] = (double)s.refinements;
    stats[2] = (double)s.num_inliers;
    stats[3] = s.model_score;
}
}
