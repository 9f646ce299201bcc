// Test client of PoseLib's own refiners with per-residual weights: bundle_adjust(x, X, Image*, opt, weights),
// bundle_adjust(x, X, CameraPose*, opt, weights), refine_relpose(x1, x2, CameraPose*, opt, weights),
// refine_relpose(x1, x2, ImagePair*, opt, weights), refine_fundamental and refine_homography, called through a C
// interface.  The weights are passed as a vector of nw doubles, so nw != n reaches the reference's uniform-weight branch.
// It is compiled against the reference's headers and linked with the reference's sources built on mini-Eigen
// (oracle/_ref/libplref2.so, or libplref2_alt.so for the other summation order); tests/golden/make_weights_golden.py
// builds it.
#include "PoseLib/misc/camera_models.h"
#include "PoseLib/robust/bundle.h"

#include <cstdint>
#include <vector>

using namespace poselib;

namespace {
int num_params(int model) {
    switch (model) {
    case 0: return 3;
    case 1: case 2: case 8: case 102: return 4;
    case 3: case 9: case 101: return 5;
    case 4: return 8;
    default: return 0;
    }
}
Camera camera(int model, const double *params) {
    Camera c;
    c.model_id = model;
    c.width = c.height = 0;
    c.params.assign(params, params + num_params(model));
    return c;
}
BundleOptions bundle(int loss_type, double loss_scale, int max_iterations, double relative_cost_tol, int flags) {
    BundleOptions b;
    b.loss_type = (BundleOptions::LossType)loss_type;
    b.loss_scale = loss_scale;
    b.max_iterations = max_iterations;
    b.relative_cost_tol = relative_cost_tol;
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
void stats_out(const BundleStats &s, double *stats) {
    stats[0] = (double)s.iterations;
    stats[1] = s.initial_cost;
    stats[2] = s.cost;
}
Eigen::Matrix3d mat_in(const double *m) { // column-major
    Eigen::Matrix3d M;
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) M(r, c) = m[3 * c + r];
    return M;
}
void mat_out(const Eigen::Matrix3d &M, double *m) {
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) m[3 * c + r] = M(r, c);
}
} // namespace

extern "C" {
// bundle_adjust(x, X, Image*, opt, weights) (robust/bundle.h:47); pose (7) and params in/out; model -1: NULL camera
void rw_bundle_adjust_image(int model, double *params, int64_t n, const double *x, const double *X, double *pose,
                            int loss_type, double loss_scale, int max_iterations, double relative_cost_tol, int flags,
                            const double *w, int64_t nw, double *stats) {
    Image image;
    image.camera = camera(model, params);
    image.pose = pose_in(pose);
    const BundleStats s = bundle_adjust(v2(x, n), v3(X, n), &image,
                                        bundle(loss_type, loss_scale, max_iterations, relative_cost_tol, flags),
                                        std::vector<double>(w, w + nw));
    pose_out(image.pose, pose);
    for (int i = 0; i < num_params(model); ++i) params[i] = image.camera.params[i];
    stats_out(s, stats);
}
// bundle_adjust(x, X, CameraPose*, opt, weights) (robust/bundle.h:41-43)
void rw_bundle_adjust(int64_t n, const double *x, const double *X, double *pose, int loss_type, double loss_scale,
                      int max_iterations, double relative_cost_tol, const double *w, int64_t nw, double *stats) {
    CameraPose p = pose_in(pose);
    const BundleStats s = bundle_adjust(v2(x, n), v3(X, n), &p,
                                        bundle(loss_type, loss_scale, max_iterations, relative_cost_tol, 0),
                                        std::vector<double>(w, w + nw));
    pose_out(p, pose);
    stats_out(s, stats);
}
// refine_relpose(x1, x2, CameraPose*, opt, weights) (robust/bundle.h:84-86)
void rw_refine_relpose(int64_t n, const double *x1, const double *x2, double *pose, int loss_type, double loss_scale,
                       int max_iterations, double relative_cost_tol, const double *w, int64_t nw, double *stats) {
    CameraPose p = pose_in(pose);
    const BundleStats s = refine_relpose(v2(x1, n), v2(x2, n), &p,
                                         bundle(loss_type, loss_scale, max_iterations, relative_cost_tol, 0),
                                         std::vector<double>(w, w + nw));
    pose_out(p, pose);
    stats_out(s, stats);
}
// refine_relpose(x1, x2, ImagePair*, opt, weights) (bundle.cc:237-266); pose and both cameras' params in/out
void rw_refine_relpose_pair(int model1, double *params1, int model2, double *params2, int64_t n, const double *x1,
                            const double *x2, double *pose, int loss_type, double loss_scale, int max_iterations,
                            double relative_cost_tol, int flags, const double *w, int64_t nw, double *stats) {
    ImagePair pair;
    pair.camera1 = camera(model1, params1);
    pair.camera2 = camera(model2, params2);
    pair.pose = pose_in(pose);
    const BundleStats s = refine_relpose(v2(x1, n), v2(x2, n), &pair,
                                         bundle(loss_type, loss_scale, max_iterations, relative_cost_tol, flags),
                                         std::vector<double>(w, w + nw));
    pose_out(pair.pose, pose);
    for (int i = 0; i < num_params(model1); ++i) params1[i] = pair.camera1.params[i];
    for (int i = 0; i < num_params(model2); ++i) params2[i] = pair.camera2.params[i];
    stats_out(s, stats);
}
// refine_fundamental / refine_homography(x1, x2, Matrix3d*, opt, weights) (robust/bundle.h:132-134,148-150); M: 9
// doubles column-major in/out
void rw_refine_matrix(int homography, int64_t n, const double *x1, const double *x2, double *m, int loss_type,
                      double loss_scale, int max_iterations, double relative_cost_tol, const double *w, int64_t nw,
                      double *stats) {
    Eigen::Matrix3d M = mat_in(m);
    const BundleOptions o = bundle(loss_type, loss_scale, max_iterations, relative_cost_tol, 0);
    const std::vector<double> weights(w, w + nw);
    const BundleStats s = homography ? refine_homography(v2(x1, n), v2(x2, n), &M, o, weights)
                                     : refine_fundamental(v2(x1, n), v2(x2, n), &M, o, weights);
    mat_out(M, m);
    stats_out(s, stats);
}
}
