// Test client of PoseLib's own camera models SIMPLE_RADIAL_FISHEYE, RADIAL_FISHEYE, DIVISION and SIMPLE_DIVISION (and the
// six models before them): the Camera functions one by one (project, project_with_jac with jac_params, unproject to 3D
// and to 2D, unproject_with_jac with and without a jac_point, get_param_refinement_idx, focal, rescale) and the
// entry points that take a camera — bundle_adjust(x, X, Image*, opt), estimate_absolute_pose(.., Image*, ..),
// refine_relpose(x1, x2, ImagePair*, opt) and estimate_relative_pose with and without tangent_sampson — called through a
// C interface.  It is compiled against the reference's headers and linked with the reference's sources built on
// mini-Eigen (oracle/_ref/libplref2.so, or libplref2_alt.so for the other summation order);
// tests/golden/make_camera_models_golden.py builds it.
#include "PoseLib/misc/camera_models.h"
#include "PoseLib/robust.h"
#include "PoseLib/robust/bundle.h"
#include "PoseLib/robust/ransac.h"

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
void params_out(const Camera &c, double *params) {
    for (int i = 0; i < num_params(c.model_id); ++i) params[i] = c.params[i];
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
void stats_out(const RansacStats &s, double *stats) {
    stats[0] = (double)s.iterations;
    stats[1] = (double)s.refinements;
    stats[2] = (double)s.num_inliers;
    stats[3] = s.model_score;
}
} // namespace

extern "C" {
int cm_num_params(int model) { return num_params(model); }
// Camera::project and project_with_jac of n camera-frame points Z (3n): xp (2n), xq (2n, project_with_jac), jac (6n,
// row-major 2x3), jp (16n, row-major 2x8, columns past the model's parameter count untouched)
void cm_project(int model, const double *params, int64_t n, const double *Z, double *xp, double *xq, double *jac,
                double *jp) {
    const Camera c = camera(model, params);
    for (int64_t k = 0; k < n; ++k) {
        const Eigen::Vector3d z(Z[3 * k], Z[3 * k + 1], Z[3 * k + 2]);
        Eigen::Vector2d p, q;
        Eigen::Matrix<double, 2, 3> J;
        Eigen::Matrix<double, 2, Eigen::Dynamic> Jp;
        c.project(z, &p);
        c.project_with_jac(z, &q, &J, &Jp);
        for (int i = 0; i < 2; ++i) {
            xp[2 * k + i] = p(i);
            xq[2 * k + i] = q(i);
        }
        for (int r = 0; r < 2; ++r)
            for (int s = 0; s < 3; ++s) jac[6 * k + 3 * r + s] = J(r, s);
        for (int r = 0; r < 2; ++r)
            for (int s = 0; s < (int)Jp.cols(); ++s) jp[16 * k + 8 * r + s] = Jp(r, s);
    }
}
// Camera::unproject of n pixels (2n) to bearings x3 (3n) and to hnormalized points x2 (2n); unproject_with_jac with a
// jac_point: d (3n), M (6n, row-major 3x2), dp (24n, row-major 3x8); without a jac_point: dq (3n), dpq (24n)
void cm_unproject(int model, const double *params, int64_t n, const double *xp, double *x3, double *x2, double *d,
                  double *M, double *dp, double *dq, double *dpq) {
    const Camera c = camera(model, params);
    for (int64_t k = 0; k < n; ++k) {
        const Eigen::Vector2d p(xp[2 * k], xp[2 * k + 1]);
        Eigen::Vector3d b, e, f;
        Eigen::Vector2d h;
        Eigen::Matrix<double, 3, 2> J;
        Eigen::Matrix<double, 3, Eigen::Dynamic> Jp, Jq;
        c.unproject(p, &b);
        c.unproject(p, &h);
        c.unproject_with_jac(p, &e, &J, &Jp);
        c.unproject_with_jac(p, &f, nullptr, &Jq);
        for (int i = 0; i < 3; ++i) {
            x3[3 * k + i] = b(i);
            d[3 * k + i] = e(i);
            dq[3 * k + i] = f(i);
        }
        x2[2 * k] = h(0);
        x2[2 * k + 1] = h(1);
        for (int r = 0; r < 3; ++r)
            for (int s = 0; s < 2; ++s) M[6 * k + 2 * r + s] = J(r, s);
        for (int r = 0; r < 3; ++r)
            for (int s = 0; s < (int)Jp.cols(); ++s) dp[24 * k + 8 * r + s] = Jp(r, s);
        for (int r = 0; r < 3; ++r)
            for (int s = 0; s < (int)Jq.cols(); ++s) dpq[24 * k + 8 * r + s] = Jq(r, s);
    }
}
// Camera::get_param_refinement_idx -> idx (up to 8); returns the count
int cm_refine_idx(int model, const double *params, int flags, int *idx) {
    Camera c = camera(model, params);
    const std::vector<size_t> v = c.get_param_refinement_idx(bundle(0, 1.0, 100, 1e-10, flags));
    for (size_t i = 0; i < v.size(); ++i) idx[i] = (int)v[i];
    return (int)v.size();
}
double cm_focal(int model, const double *params) { return camera(model, params).focal(); }
void cm_rescale(int model, double *params, double scale) {
    Camera c = camera(model, params);
    c.rescale(scale);
    params_out(c, params);
}
// bundle_adjust(x, X, Image*, opt) (robust/bundle.h:47); pose (7) and params in/out; stats: iterations, initial, cost
void cm_bundle_adjust_image(int model, double *params, int64_t n, const double *x, const double *X, double *pose,
                            int loss_type, double loss_scale, int max_iterations, double relative_cost_tol, int flags,
                            double *stats) {
    Image image;
    image.camera = camera(model, params);
    image.pose = pose_in(pose);
    const BundleStats s =
        bundle_adjust(v2(x, n), v3(X, n), &image, bundle(loss_type, loss_scale, max_iterations, relative_cost_tol, flags));
    pose_out(image.pose, pose);
    params_out(image.camera, params);
    stats[0] = (double)s.iterations;
    stats[1] = s.initial_cost;
    stats[2] = s.cost;
}
// estimate_absolute_pose(points2D, points3D, opt, Image*, inliers) (robust.h:45-46), default RansacOptions except
// max_iterations / min_iterations / seed, BundleOptions: Cauchy, loss scale 1.0, flags; stats as stats_out
void cm_estimate_absolute_pose(int model, double *params, int64_t n, const double *x, const double *X, double max_error,
                               uint64_t max_iterations, uint64_t min_iterations, uint64_t seed, int flags, double *pose,
                               char *inliers, double *stats) {
    AbsolutePoseOptions o;
    o.ransac.max_iterations = max_iterations;
    o.ransac.min_iterations = min_iterations;
    o.ransac.seed = seed;
    o.bundle = bundle(3, 1.0, 100, 1e-10, flags);
    o.max_error = max_error;
    Image image;
    image.camera = camera(model, params);
    image.pose = pose_in(pose);
    std::vector<char> m(n, 0);
    stats_out(estimate_absolute_pose(v2(x, n), v3(X, n), o, &image, &m), stats);
    pose_out(image.pose, pose);
    params_out(image.camera, params);
    for (int64_t k = 0; k < n; ++k) inliers[k] = m[k];
}
// refine_relpose(x1, x2, ImagePair*, opt) (robust/bundle.h); pose (7) and both cameras' params in/out; stats:
// iterations, initial_cost, cost
void cm_refine_relpose_pair(int model1, double *params1, int model2, double *params2, int64_t n, const double *x1,
                            const double *x2, double *pose, int loss_type, double loss_scale, int max_iterations,
                            double relative_cost_tol, int flags, double *stats) {
    ImagePair pair;
    pair.camera1 = camera(model1, params1);
    pair.camera2 = camera(model2, params2);
    pair.pose = pose_in(pose);
    const BundleStats s =
        refine_relpose(v2(x1, n), v2(x2, n), &pair, bundle(loss_type, loss_scale, max_iterations, relative_cost_tol, flags));
    pose_out(pair.pose, pose);
    params_out(pair.camera1, params1);
    params_out(pair.camera2, params2);
    stats[0] = (double)s.iterations;
    stats[1] = s.initial_cost;
    stats[2] = s.cost;
}
// estimate_relative_pose(x1, x2, camera1, camera2, opt, pose, inliers) (robust.cc:242-314) with the default
// RansacOptions except max_iterations / min_iterations / seed, BundleOptions: Cauchy, loss scale 1.0, flags.
// tangent = 0 runs the unproject pre-step (robust.cc:286-314).  With tangent = 1 and restate = 1 it runs robust.cc:249-284
// from public functions instead (ransac_relpose with the cameras, then refine_relpose on the pair) and also returns the
// pair's cameras, rescaled back by 1 / scale, where the flags select parameters of either camera; otherwise the cameras
// are left as given.  stats as stats_out
void cm_estimate_relative_pose(int model1, double *params1, int model2, double *params2, int64_t n, const double *x1,
                               const double *x2, double max_error, uint64_t max_iterations, uint64_t min_iterations,
                               uint64_t seed, int flags, int tangent, int restate, double *pose, char *inliers,
                               double *stats) {
    RelativePoseOptions o;
    o.ransac.max_iterations = max_iterations;
    o.ransac.min_iterations = min_iterations;
    o.ransac.seed = seed;
    o.bundle = bundle(3, 1.0, 100, 1e-10, flags);
    o.max_error = max_error;
    o.tangent_sampson = tangent != 0;
    const Camera c1 = camera(model1, params1), c2 = camera(model2, params2);
    const std::vector<Point2D> v1 = v2(x1, n), w2 = v2(x2, n);
    CameraPose p;
    std::vector<char> m(n, 0);
    RansacStats s;
    if (!(tangent && restate)) {
        s = estimate_relative_pose(v1, w2, c1, c2, o, &p, &m);
    } else {
        const double scale = 0.5 * (1.0 / c1.focal() + 1.0 / c2.focal());
        RelativePoseOptions os = o;
        os.max_error *= scale;
        os.bundle.loss_scale *= scale;
        std::vector<Point2D> s1(n), s2(n);
        for (int64_t k = 0; k < n; ++k) {
            s1[k] = v1[k] * scale;
            s2[k] = w2[k] * scale;
        }
        Camera k1 = c1, k2 = c2;
        k1.rescale(scale);
        k2.rescale(scale);
        s = ransac_relpose(s1, s2, k1, k2, os, &p, &m);
        if (s.num_inliers > 5) {
            std::vector<Point2D> i1, i2;
            for (int64_t k = 0; k < n; ++k)
                if (m[k]) {
                    i1.push_back(s1[k]);
                    i2.push_back(s2[k]);
                }
            ImagePair pair(p, k1, k2);
            refine_relpose(i1, i2, &pair, os.bundle);
            p = pair.pose;
            if (!k1.get_param_refinement_idx(os.bundle).empty() || !k2.get_param_refinement_idx(os.bundle).empty()) {
                pair.camera1.rescale(1.0 / scale);
                pair.camera2.rescale(1.0 / scale);
                params_out(pair.camera1, params1);
                params_out(pair.camera2, params2);
            }
        }
    }
    pose_out(p, pose);
    for (int64_t k = 0; k < n; ++k) inliers[k] = m[k];
    stats_out(s, stats);
}
}
