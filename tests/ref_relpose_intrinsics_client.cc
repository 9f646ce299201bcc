// Test client of PoseLib's own relative-pose camera refinement: Camera::unproject_with_jac with jac_params (with and
// without a jac_point), refine_relpose(x1, x2, ImagePair*, opt) and estimate_relative_pose with tangent_sampson (plus a
// restatement of its body that keeps the refined cameras), called through a C interface.  It is compiled
// against the reference's headers and linked with the reference's sources built on mini-Eigen (oracle/_ref/libplref2.so,
// or libplref2_alt.so for the other summation order); tests/golden/make_relpose_intrinsics_golden.py builds it.
#include "PoseLib/misc/camera_models.h"
#include "PoseLib/robust.h"
#include "PoseLib/robust/bundle.h"
#include "PoseLib/robust/ransac.h"

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
std::vector<Point2D> v2(const double *a, int64_t n) {
    std::vector<Point2D> v(n);
    for (int64_t k = 0; k < n; ++k) v[k] = Point2D(a[2 * k], a[2 * k + 1]);
    return v;
}
} // namespace

extern "C" {
// Camera::unproject_with_jac of n pixels xp (2n): bearings d (3n) and jac_params dp (24n, row-major 3 x 8, columns past
// the model's parameter count untouched); with_point selects the form with a jac_point (camera_models.cc:480-483) or
// without one (:486-488)
void rr_unproject_with_jac(int model, const double *params, int64_t n, const double *xp, int with_point, double *d,
                           double *dp) {
    Camera c = camera(model, params);
    for (int64_t k = 0; k < n; ++k) {
        Eigen::Vector3d x;
        Eigen::Matrix<double, 3, 2> M;
        Eigen::Matrix<double, 3, Eigen::Dynamic> J;
        c.unproject_with_jac(Eigen::Vector2d(xp[2 * k], xp[2 * k + 1]), &x, with_point ? &M : nullptr, &J);
        for (int i = 0; i < 3; ++i) d[3 * k + i] = x(i);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < (int)J.cols(); ++j) dp[24 * k + 8 * i + j] = J(i, j);
    }
}
// refine_relpose(x1, x2, ImagePair*, opt) (robust/bundle.h); pose (7) and both cameras' params in/out; stats:
// iterations, initial_cost, cost
void rr_refine_relpose_pair(int model1, double *params1, int model2, double *params2, int64_t n, const double *x1,
                            const double *x2, double *pose, int loss_type, double loss_scale, int max_iterations,
                            double relative_cost_tol, int flags, double *stats) {
    ImagePair pair;
    pair.camera1 = camera(model1, params1);
    pair.camera2 = camera(model2, params2);
    for (int i = 0; i < 4; ++i) pair.pose.q(i) = pose[i];
    for (int i = 0; i < 3; ++i) pair.pose.t(i) = pose[4 + i];
    BundleOptions o;
    o.loss_type = (BundleOptions::LossType)loss_type;
    o.loss_scale = loss_scale;
    o.max_iterations = max_iterations;
    o.relative_cost_tol = relative_cost_tol;
    o.refine_focal_length = (flags & 1) != 0;
    o.refine_principal_point = (flags & 2) != 0;
    o.refine_extra_params = (flags & 4) != 0;
    const BundleStats s = refine_relpose(v2(x1, n), v2(x2, n), &pair, o);
    for (int i = 0; i < 4; ++i) pose[i] = pair.pose.q(i);
    for (int i = 0; i < 3; ++i) pose[4 + i] = pair.pose.t(i);
    for (int i = 0; i < NP[model1]; ++i) params1[i] = pair.camera1.params[i];
    for (int i = 0; i < NP[model2]; ++i) params2[i] = pair.camera2.params[i];
    stats[0] = (double)s.iterations;
    stats[1] = s.initial_cost;
    stats[2] = s.cost;
}
// estimate_relative_pose(x1, x2, camera1, camera2, opt, pose, inliers) with tangent_sampson (robust.cc:242-284) and the
// default RansacOptions except max_iterations / min_iterations / seed, BundleOptions: Cauchy, loss scale 1.0, flags.
// restate = 1 runs robust.cc:249-284 from public functions instead (ransac_relpose with the cameras, then
// refine_relpose on the pair) and also returns the pair's cameras, rescaled back by 1 / scale, where the flags select
// parameters of either camera; otherwise the cameras are left as given.  stats: iterations, refinements, num_inliers, model_score
void rr_estimate_relative_pose(int model1, double *params1, int model2, double *params2, int64_t n, const double *x1,
                               const double *x2, double max_error, uint64_t max_iterations, uint64_t min_iterations,
                               uint64_t seed, int flags, int restate, double *pose, char *inliers, double *stats) {
    RelativePoseOptions o;
    o.ransac.max_iterations = max_iterations;
    o.ransac.min_iterations = min_iterations;
    o.ransac.seed = seed;
    o.bundle.refine_focal_length = (flags & 1) != 0;
    o.bundle.refine_principal_point = (flags & 2) != 0;
    o.bundle.refine_extra_params = (flags & 4) != 0;
    o.max_error = max_error;
    o.tangent_sampson = true;
    const Camera c1 = camera(model1, params1), c2 = camera(model2, params2);
    const std::vector<Point2D> v1 = v2(x1, n), w2 = v2(x2, n);
    CameraPose p;
    std::vector<char> m(n, 0);
    RansacStats s;
    if (!restate) {
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
                for (int i = 0; i < NP[model1]; ++i) params1[i] = pair.camera1.params[i];
                for (int i = 0; i < NP[model2]; ++i) params2[i] = pair.camera2.params[i];
            }
        }
    }
    for (int i = 0; i < 4; ++i) pose[i] = p.q(i);
    for (int i = 0; i < 3; ++i) pose[4 + i] = p.t(i);
    for (int64_t k = 0; k < n; ++k) inliers[k] = m[k];
    stats[0] = (double)s.iterations;
    stats[1] = (double)s.refinements;
    stats[2] = (double)s.num_inliers;
    stats[3] = s.model_score;
}
}
