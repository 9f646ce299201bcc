// poselib_b200.hpp — header-only C++ adapter that gives the C-ABI (include/poselib_b200.h) back the call surface of
// PoseLib/robust.h, PoseLib/robust/ransac.h, PoseLib/robust/bundle.h and PoseLib/solvers/*.h for the ONE hot path
// this repository replaces.  Reference signatures (relative to the PoseLib checkout @ a69263d):
//   robust.h:45-46,68-70,112-113,133-134   estimate_absolute_pose / estimate_relative_pose / estimate_fundamental /
//                                          estimate_homography
//   robust/ransac.h:39-40,60-61,85-87,99-101  ransac_pnp / ransac_relpose / ransac_fundamental / ransac_homography
//   solvers/p3p.h:42, p3p_lambdatwist.h:44, relpose_5pt.h:40-43, relpose_7pt.h:39-40, homography_4pt.h:38-39
//
// The adapter is templated on the vector / matrix types so that it compiles both
//   (a) inside PoseLib (or user code) with Eigen:   poselib_b200::estimate_relative_pose(x1, x2, cam1, cam2, opt, &pose, &inl)
//       with Point2D = Eigen::Vector2d, Point3D = Eigen::Vector3d, Eigen::Matrix3d, poselib::CameraPose, and
//   (b) here, where Eigen is not installed, against the 20-line stand-ins of tests/adapter_compile_test.cc.
// Layout facts it relies on (SURVEY.md §8b): std::vector<Eigen::Vector2d/3d>::data() is a dense double[2n]/[3n];
// Eigen::Matrix3d is 9 doubles column-major; CameraPose is q (w,x,y,z) followed by t.
//
// Error convention: PoseLib never reports errors on this path except Camera::unproject throwing
// std::runtime_error("NYI") (misc/camera_models.cc:184-185); every non-zero C-ABI status is thrown the same way.
#pragma once
#include "../../include/poselib_b200.h"

#include <cstdint>
#include <limits>
#include <stdexcept>
#include <string>
#include <vector>

namespace poselib_b200 {

namespace detail {
inline void check(int rc) {
    if (rc != PLB_OK) throw std::runtime_error(std::string("poselib_b200: ") + plb_last_error());
}
// PoseLib/types.h:39-50 -> plb_ransac_opt
template <typename RansacOptions> inline plb_ransac_opt to_c(const RansacOptions &o) {
    plb_ransac_opt c;
    c.max_iterations = o.max_iterations;
    c.min_iterations = o.min_iterations;
    c.dyn_num_trials_mult = o.dyn_num_trials_mult;
    c.success_prob = o.success_prob;
    c.seed = o.seed;
    c.progressive_sampling = o.progressive_sampling ? 1 : 0;
    c.score_initial_model = o.score_initial_model ? 1 : 0;
    c.max_prosac_iterations = o.max_prosac_iterations;
    return c;
}
// PoseLib/types.h:60-95 -> plb_bundle_opt.  Only NIELSEN/LEVENBERG and the TRIVIAL/TRUNCATED/HUBER/CAUCHY losses are
// on the CUDA path; everything else is rejected loudly instead of being silently approximated.
template <typename BundleOptions> inline plb_bundle_opt bundle_to_c(const BundleOptions &o) {
    plb_bundle_opt c;
    c.max_iterations = o.max_iterations;
    switch (static_cast<int>(o.loss_type)) {
    case 0: c.loss_type = PLB_LOSS_TRIVIAL; break;
    case 1: c.loss_type = PLB_LOSS_TRUNCATED; break;
    case 2: c.loss_type = PLB_LOSS_HUBER; break;
    case 3: c.loss_type = PLB_LOSS_CAUCHY; break;
    default: throw std::runtime_error("poselib_b200: NYI loss type (TRUNCATED_CAUCHY / TRUNCATED_LE_ZACH)");
    }
    c.refine_intrinsics = (o.refine_focal_length ? PLB_REFINE_FOCAL_LENGTH : 0) |
                          (o.refine_principal_point ? PLB_REFINE_PRINCIPAL_POINT : 0) |
                          (o.refine_extra_params ? PLB_REFINE_EXTRA_PARAMS : 0);
    c.loss_scale = o.loss_scale;
    c.gradient_tol = o.gradient_tol;
    c.step_tol = o.step_tol;
    c.relative_cost_tol = o.relative_cost_tol;
    c.initial_lambda = o.initial_lambda;
    c.min_lambda = o.min_lambda;
    c.max_lambda = o.max_lambda;
    if (static_cast<int>(o.lambda_update) != 0 || static_cast<int>(o.damping) != 0)
        throw std::runtime_error("poselib_b200: NYI bundle option (FIXED_FACTOR / MARQUARDT)");
    return c;
}
template <typename RansacStats> inline RansacStats from_c(const plb_ransac_stats &s) {
    RansacStats r;
    r.refinements = s.refinements;
    r.iterations = s.iterations;
    r.num_inliers = s.num_inliers;
    r.inlier_ratio = s.inlier_ratio;
    r.model_score = s.model_score;
    return r;
}
// misc/camera_models.h:59-157 -> plb_camera (the ten models of include/poselib_b200.h are on the path; others raise NYI inside the library)
template <typename Camera> inline plb_camera camera_to_c(const Camera &cam) {
    plb_camera c;
    c.model_id = cam.model_id;
    c.width = cam.width;
    c.height = cam.height;
    c.reserved = 0;
    for (int i = 0; i < 8; ++i) c.params[i] = (i < (int)cam.params.size()) ? cam.params[i] : 0.0;
    if (cam.params.empty()) c.model_id = PLB_CAMERA_NULL; // "empty camera assumed to be identity" camera_models.cc:305-307
    return c;
}
// plb_camera -> Camera::params (the model id and the size of the parameter vector are the caller's)
template <typename Camera> inline void camera_from_c(const plb_camera &c, Camera *cam) {
    for (size_t i = 0; i < cam->params.size() && i < 8; ++i) cam->params[i] = c.params[i];
}
template <typename Pose> inline void pose_to(const Pose &p, double out[7]) {
    for (int i = 0; i < 4; ++i) out[i] = p.q(i);
    for (int i = 0; i < 3; ++i) out[4 + i] = p.t(i);
}
template <typename Pose> inline void pose_from(const double in[7], Pose *p) {
    for (int i = 0; i < 4; ++i) p->q(i) = in[i];
    for (int i = 0; i < 3; ++i) p->t(i) = in[4 + i];
}
template <typename Vec> inline const double *raw(const std::vector<Vec> &v) {
    return v.empty() ? nullptr : reinterpret_cast<const double *>(v.data());
}
} // namespace detail

// ---- robust/ransac.h ------------------------------------------------------------------------------------------
template <typename RansacStats, typename P2, typename P3, typename Opt, typename Pose>
RansacStats ransac_pnp(const std::vector<P2> &x, const std::vector<P3> &X, const Opt &opt, Pose *best_model,
                       std::vector<char> *best_inliers) {
    static_assert(sizeof(P2) == 2 * sizeof(double) && sizeof(P3) == 3 * sizeof(double), "dense point layout required");
    double m[7];
    detail::pose_to(*best_model, m);
    plb_ransac_opt ro = detail::to_c(opt.ransac);
    plb_ransac_stats st;
    best_inliers->resize(x.size());
    detail::check(plb_ransac_pnp(detail::raw(x), detail::raw(X), x.size(), &ro, opt.max_error, m,
                                 best_inliers->data(), &st, nullptr));
    detail::pose_from(m, best_model);
    return detail::from_c<RansacStats>(st);
}
template <typename RansacStats, typename P2, typename Opt, typename Pose>
RansacStats ransac_relpose(const std::vector<P2> &x1, const std::vector<P2> &x2, const Opt &opt, Pose *best_model,
                           std::vector<char> *best_inliers) {
    static_assert(sizeof(P2) == 2 * sizeof(double), "dense point layout required");
    double m[7];
    detail::pose_to(*best_model, m);
    plb_ransac_opt ro = detail::to_c(opt.ransac);
    plb_ransac_stats st;
    best_inliers->resize(x1.size());
    detail::check(plb_ransac_relpose(detail::raw(x1), detail::raw(x2), x1.size(), &ro, opt.max_error, m,
                                     best_inliers->data(), &st, nullptr));
    detail::pose_from(m, best_model);
    return detail::from_c<RansacStats>(st);
}
// ransac_relpose(x1, x2, camera1, camera2, RelativePoseOptions, CameraPose*, inliers*)   robust/ransac.h:62-64
template <typename RansacStats, typename P2, typename Camera, typename Opt, typename Pose>
RansacStats ransac_relpose(const std::vector<P2> &x1, const std::vector<P2> &x2, const Camera &camera1,
                           const Camera &camera2, const Opt &opt, Pose *best_model, std::vector<char> *best_inliers) {
    static_assert(sizeof(P2) == 2 * sizeof(double), "dense point layout required");
    double m[7];
    plb_ransac_opt ro = detail::to_c(opt.ransac);
    plb_camera c1 = detail::camera_to_c(camera1), c2 = detail::camera_to_c(camera2);
    plb_ransac_stats st;
    best_inliers->resize(x1.size());
    detail::check(plb_ransac_relpose_cameras(detail::raw(x1), detail::raw(x2), x1.size(), &c1, &c2, &ro, opt.max_error,
                                             m, best_inliers->data(), &st, nullptr));
    detail::pose_from(m, best_model);
    return detail::from_c<RansacStats>(st);
}
template <typename RansacStats, typename P2, typename Opt, typename Mat3>
RansacStats ransac_fundamental(const std::vector<P2> &x1, const std::vector<P2> &x2, const Opt &opt, Mat3 *best_model,
                               std::vector<char> *best_inliers) {
    static_assert(sizeof(Mat3) == 9 * sizeof(double), "column-major 3x3 of doubles required");
    plb_ransac_opt ro = detail::to_c(opt.ransac);
    plb_ransac_stats st;
    best_inliers->resize(x1.size());
    detail::check(plb_ransac_fundamental(detail::raw(x1), detail::raw(x2), x1.size(), &ro, opt.max_error,
                                         opt.real_focal_check ? 1 : 0, reinterpret_cast<double *>(best_model),
                                         best_inliers->data(), &st, nullptr));
    return detail::from_c<RansacStats>(st);
}
template <typename RansacStats, typename P2, typename Opt, typename Mat3>
RansacStats ransac_homography(const std::vector<P2> &x1, const std::vector<P2> &x2, const Opt &opt, Mat3 *best_model,
                              std::vector<char> *best_inliers) {
    static_assert(sizeof(Mat3) == 9 * sizeof(double), "column-major 3x3 of doubles required");
    plb_ransac_opt ro = detail::to_c(opt.ransac);
    plb_ransac_stats st;
    best_inliers->resize(x1.size());
    detail::check(plb_ransac_homography(detail::raw(x1), detail::raw(x2), x1.size(), &ro, opt.max_error,
                                        reinterpret_cast<double *>(best_model), best_inliers->data(), &st, nullptr));
    return detail::from_c<RansacStats>(st);
}

// ---- robust.h ---------------------------------------------------------------------------------------------------
// estimate_absolute_pose(points2D, points3D, AbsolutePoseOptions (by value), Image*, inliers*)   robust.h:45-46
template <typename RansacStats, typename P2, typename P3, typename Opt, typename Image>
RansacStats estimate_absolute_pose(const std::vector<P2> &points2D, const std::vector<P3> &points3D, Opt opt,
                                   Image *image, std::vector<char> *inliers) {
    if (opt.estimate_focal_length || opt.estimate_extra_params)
        throw std::runtime_error("poselib_b200: NYI (focal-length estimation is row N2 of SURVEY.md §8f)");
    double m[7];
    detail::pose_to(image->pose, m);
    plb_ransac_opt ro = detail::to_c(opt.ransac);
    plb_bundle_opt bo = detail::bundle_to_c(opt.bundle);
    plb_camera cam = detail::camera_to_c(image->camera);
    plb_ransac_stats st;
    inliers->resize(points2D.size());
    detail::check(plb_estimate_absolute_pose_image(detail::raw(points2D), detail::raw(points3D), points2D.size(), &ro,
                                                   &bo, opt.max_error, &cam, m, inliers->data(), &st, nullptr));
    detail::pose_from(m, &image->pose);
    detail::camera_from_c(cam, &image->camera); // refined / rescaled intrinsics (robust.cc:103-123)
    return detail::from_c<RansacStats>(st);
}
// estimate_relative_pose(x1, x2, camera1, camera2, RelativePoseOptions, CameraPose*, inliers*)   robust.h:68-70
// With tangent_sampson and refine_* flags the final bundle adjustment refines the cameras too (robust.cc:262-282); like
// the reference, the refined cameras are computed on copies and discarded.
template <typename RansacStats, typename P2, typename Camera, typename Opt, typename Pose>
RansacStats estimate_relative_pose(const std::vector<P2> &x1, const std::vector<P2> &x2, const Camera &camera1,
                                   const Camera &camera2, const Opt &opt, Pose *pose, std::vector<char> *inliers) {
    double m[7];
    detail::pose_to(*pose, m);
    plb_ransac_opt ro = detail::to_c(opt.ransac);
    plb_bundle_opt bo = detail::bundle_to_c(opt.bundle);
    plb_camera c1 = detail::camera_to_c(camera1), c2 = detail::camera_to_c(camera2);
    plb_ransac_stats st;
    inliers->resize(x1.size());
    const bool refine_cameras = opt.tangent_sampson && (bo.refine_intrinsics & (PLB_REFINE_FOCAL_LENGTH |
                                                                                  PLB_REFINE_PRINCIPAL_POINT |
                                                                                  PLB_REFINE_EXTRA_PARAMS)) != 0;
    detail::check(refine_cameras
                      ? plb_estimate_relative_pose_pair(detail::raw(x1), detail::raw(x2), x1.size(), &c1, &c2, &ro, &bo,
                                                        opt.max_error, 1, m, inliers->data(), &st, nullptr)
                      : plb_estimate_relative_pose(detail::raw(x1), detail::raw(x2), x1.size(), &c1, &c2, &ro, &bo,
                                                   opt.max_error, opt.tangent_sampson ? 1 : 0, m, inliers->data(), &st,
                                                   nullptr));
    detail::pose_from(m, pose);
    return detail::from_c<RansacStats>(st);
}
// estimate_fundamental(x1, x2, RelativePoseOptions, Matrix3d*, inliers*)   robust.h:112-113
template <typename RansacStats, typename P2, typename Opt, typename Mat3>
RansacStats estimate_fundamental(const std::vector<P2> &x1, const std::vector<P2> &x2, const Opt &opt, Mat3 *F,
                                 std::vector<char> *inliers) {
    plb_ransac_opt ro = detail::to_c(opt.ransac);
    plb_bundle_opt bo = detail::bundle_to_c(opt.bundle);
    plb_ransac_stats st;
    st.refinements = st.iterations = st.num_inliers = 0;
    st.inlier_ratio = 0;
    st.model_score = std::numeric_limits<double>::max();
    if (x1.size() >= 7) inliers->resize(x1.size()); // robust.cc:548-550 returns before touching `inliers`
    detail::check(plb_estimate_fundamental(detail::raw(x1), detail::raw(x2), x1.size(), &ro, &bo, opt.max_error,
                                           opt.real_focal_check ? 1 : 0, reinterpret_cast<double *>(F),
                                           x1.size() >= 7 ? inliers->data() : nullptr, &st, nullptr));
    return detail::from_c<RansacStats>(st);
}
// estimate_homography(x1, x2, HomographyOptions, Matrix3d*, inliers*)   robust.h:133-134
template <typename RansacStats, typename P2, typename Opt, typename Mat3>
RansacStats estimate_homography(const std::vector<P2> &x1, const std::vector<P2> &x2, const Opt &opt, Mat3 *H,
                                std::vector<char> *inliers) {
    plb_ransac_opt ro = detail::to_c(opt.ransac);
    plb_bundle_opt bo = detail::bundle_to_c(opt.bundle);
    plb_ransac_stats st;
    st.refinements = st.iterations = st.num_inliers = 0;
    st.inlier_ratio = 0;
    st.model_score = std::numeric_limits<double>::max();
    if (x1.size() >= 4) inliers->resize(x1.size()); // robust.cc:716-718
    detail::check(plb_estimate_homography(detail::raw(x1), detail::raw(x2), x1.size(), &ro, &bo, opt.max_error,
                                          reinterpret_cast<double *>(H), x1.size() >= 4 ? inliers->data() : nullptr,
                                          &st, nullptr));
    return detail::from_c<RansacStats>(st);
}

// ---- robust/bundle.h: the LM refiners, with the reference's optional per-residual weights ---------------------------
// BundleStats carries iterations, initial_cost and cost; lambda / step_norm / grad_norm stay at their defaults.
// Weights are used when weights.size() == n and otherwise mean uniform weights, as in the reference (bundle.cc:107-111,
// 217-221, 261-265, 272-276, 328-332, 406-410).
namespace detail {
template <typename BundleStats> inline BundleStats bundle_from_c(const double s[3]) {
    BundleStats b = BundleStats();
    b.iterations = static_cast<size_t>(s[0]);
    b.initial_cost = s[1];
    b.cost = s[2];
    return b;
}
// the weights the *_weighted entry points take: the caller's when there is one per point, else null (uniform)
inline const double *weights_of(const std::vector<double> &weights, size_t n) {
    return weights.size() == n ? weights.data() : nullptr;
}
} // namespace detail
// bundle_adjust(x, X, CameraPose*, BundleOptions, weights)   robust/bundle.h:41-43.  The weights are ignored: the
// reference calls the Image* overload without them (bundle.cc:84-92).
template <typename BundleStats, typename P2, typename P3, typename Pose, typename BOpt>
BundleStats bundle_adjust(const std::vector<P2> &x, const std::vector<P3> &X, Pose *pose, const BOpt &opt,
                          const std::vector<double> &weights = std::vector<double>()) {
    (void)weights;
    double m[7], st[3];
    detail::pose_to(*pose, m);
    plb_bundle_opt bo = detail::bundle_to_c(opt);
    detail::check(plb_bundle_adjust(detail::raw(x), detail::raw(X), x.size(), m, &bo, st));
    detail::pose_from(m, pose);
    return detail::bundle_from_c<BundleStats>(st);
}
// bundle_adjust(x, X, Image*, BundleOptions, weights)   robust/bundle.h:47: the pose and the camera parameters the
// refine_* flags select, points in the camera's pixel units
template <typename BundleStats, typename P2, typename P3, typename Image, typename BOpt>
BundleStats bundle_adjust_image(const std::vector<P2> &x, const std::vector<P3> &X, Image *image, const BOpt &opt,
                                const std::vector<double> &weights = std::vector<double>()) {
    double m[7], st[3];
    detail::pose_to(image->pose, m);
    plb_bundle_opt bo = detail::bundle_to_c(opt);
    plb_camera cam = detail::camera_to_c(image->camera);
    detail::check(plb_bundle_adjust_image_weighted(detail::raw(x), detail::raw(X), x.size(), m, &cam, &bo, st,
                                                   detail::weights_of(weights, x.size())));
    detail::pose_from(m, &image->pose);
    detail::camera_from_c(cam, &image->camera);
    return detail::bundle_from_c<BundleStats>(st);
}
// refine_relpose(x1, x2, CameraPose*, BundleOptions, weights)   robust/bundle.h:84-86
template <typename BundleStats, typename P2, typename Pose, typename BOpt>
BundleStats refine_relpose(const std::vector<P2> &x1, const std::vector<P2> &x2, Pose *pose, const BOpt &opt,
                           const std::vector<double> &weights = std::vector<double>()) {
    double m[7], st[3];
    detail::pose_to(*pose, m);
    plb_bundle_opt bo = detail::bundle_to_c(opt);
    detail::check(plb_refine_relpose_weighted(detail::raw(x1), detail::raw(x2), x1.size(), m, &bo, st,
                                              detail::weights_of(weights, x1.size())));
    detail::pose_from(m, pose);
    return detail::bundle_from_c<BundleStats>(st);
}
// refine_relpose(x1, x2, ImagePair*, BundleOptions, weights)   robust/bundle.cc:237-256: the pose and, in each camera,
// the parameters the refine_* flags select, pixels as given
template <typename BundleStats, typename P2, typename ImagePair, typename BOpt>
BundleStats refine_relpose_pair(const std::vector<P2> &x1, const std::vector<P2> &x2, ImagePair *pair, const BOpt &opt,
                                const std::vector<double> &weights = std::vector<double>()) {
    double m[7], st[3];
    detail::pose_to(pair->pose, m);
    plb_bundle_opt bo = detail::bundle_to_c(opt);
    plb_camera c1 = detail::camera_to_c(pair->camera1), c2 = detail::camera_to_c(pair->camera2);
    detail::check(plb_refine_relpose_pair_weighted(detail::raw(x1), detail::raw(x2), x1.size(), &c1, &c2, m, &bo, st,
                                                   detail::weights_of(weights, x1.size())));
    detail::pose_from(m, &pair->pose);
    detail::camera_from_c(c1, &pair->camera1);
    detail::camera_from_c(c2, &pair->camera2);
    return detail::bundle_from_c<BundleStats>(st);
}
// refine_fundamental(x1, x2, Matrix3d*, BundleOptions, weights)   robust/bundle.h:132-134
template <typename BundleStats, typename P2, typename Mat3, typename BOpt>
BundleStats refine_fundamental(const std::vector<P2> &x1, const std::vector<P2> &x2, Mat3 *F, const BOpt &opt,
                               const std::vector<double> &weights = std::vector<double>()) {
    static_assert(sizeof(Mat3) == 9 * sizeof(double), "column-major 3x3 of doubles required");
    double st[3];
    plb_bundle_opt bo = detail::bundle_to_c(opt);
    detail::check(plb_refine_fundamental_weighted(detail::raw(x1), detail::raw(x2), x1.size(), reinterpret_cast<double *>(F),
                                                  &bo, st, detail::weights_of(weights, x1.size())));
    return detail::bundle_from_c<BundleStats>(st);
}
// refine_homography(x1, x2, Matrix3d*, BundleOptions, weights)   robust/bundle.h:148-150
template <typename BundleStats, typename P2, typename Mat3, typename BOpt>
BundleStats refine_homography(const std::vector<P2> &x1, const std::vector<P2> &x2, Mat3 *H, const BOpt &opt,
                              const std::vector<double> &weights = std::vector<double>()) {
    static_assert(sizeof(Mat3) == 9 * sizeof(double), "column-major 3x3 of doubles required");
    double st[3];
    plb_bundle_opt bo = detail::bundle_to_c(opt);
    detail::check(plb_refine_homography_weighted(detail::raw(x1), detail::raw(x2), x1.size(), reinterpret_cast<double *>(H),
                                                 &bo, st, detail::weights_of(weights, x1.size())));
    return detail::bundle_from_c<BundleStats>(st);
}

// ---- solvers/*.h (one instance; unit bearing vectors).  Return value = number of solutions, like the reference.
template <typename V3, typename Pose> int p3p(const std::vector<V3> &x, const std::vector<V3> &X, std::vector<Pose> *output) {
    if (output == nullptr) return 0; // p3p.cc:41-43
    output->clear();
    double poses[28];
    int32_t n = 0;
    detail::check(plb_p3p_batch(1, detail::raw(x), detail::raw(X), poses, &n));
    for (int i = 0; i < n; ++i) {
        Pose p;
        detail::pose_from(poses + 7 * i, &p);
        output->push_back(p);
    }
    return n;
}
// solvers/p3p_lambdatwist.h:44-45
template <typename V3, typename Pose> int p3p_lambdatwist(const std::vector<V3> &x, const std::vector<V3> &X, std::vector<Pose> *output) {
    output->clear(); // p3p_lambdatwist.cc:137
    double poses[28];
    int32_t n = 0;
    detail::check(plb_p3p_lambdatwist_batch(1, detail::raw(x), detail::raw(X), poses, &n));
    for (int i = 0; i < n; ++i) {
        Pose p;
        detail::pose_from(poses + 7 * i, &p);
        output->push_back(p);
    }
    return n;
}
template <typename V3, typename Mat3> int relpose_5pt(const std::vector<V3> &x1, const std::vector<V3> &x2, std::vector<Mat3> *E) {
    double out[90];
    int32_t n = 0;
    detail::check(plb_relpose_5pt_batch(1, detail::raw(x1), detail::raw(x2), out, &n));
    for (int i = 0; i < n; ++i) { // NB: the reference appends without clearing (relpose_5pt.cc:364,391)
        Mat3 M;
        double *m = reinterpret_cast<double *>(&M);
        for (int k = 0; k < 9; ++k) m[k] = out[9 * i + k];
        E->push_back(M);
    }
    return n;
}
template <typename V3, typename Pose> int relpose_5pt_poses(const std::vector<V3> &x1, const std::vector<V3> &x2, std::vector<Pose> *output) {
    double out[280];
    int32_t n = 0;
    detail::check(plb_relpose_5pt_poses_batch(1, detail::raw(x1), detail::raw(x2), out, &n));
    output->clear(); // relpose_5pt.cc:402
    for (int i = 0; i < n; ++i) {
        Pose p;
        detail::pose_from(out + 7 * i, &p);
        output->push_back(p);
    }
    return n;
}
template <typename V3, typename Mat3> int relpose_7pt(const std::vector<V3> &x1, const std::vector<V3> &x2, std::vector<Mat3> *F) {
    double out[27];
    int32_t n = 0;
    detail::check(plb_relpose_7pt_batch(1, detail::raw(x1), detail::raw(x2), out, &n));
    F->clear(); // relpose_7pt.cc:51
    for (int i = 0; i < n; ++i) {
        Mat3 M;
        double *m = reinterpret_cast<double *>(&M);
        for (int k = 0; k < 9; ++k) m[k] = out[9 * i + k];
        F->push_back(M);
    }
    return n;
}
template <typename V3, typename Mat3>
int homography_4pt(const std::vector<V3> &x1, const std::vector<V3> &x2, Mat3 *H, bool check_cheirality = true) {
    int32_t n = 0;
    detail::check(plb_homography_4pt_batch(1, detail::raw(x1), detail::raw(x2), reinterpret_cast<double *>(H), &n,
                                           check_cheirality ? 1 : 0));
    return n;
}

// essential_matrix_8pt / relpose_8pt (solvers/relpose_8pt.h:45-53): n >= 8 unit bearing pairs
template <typename V3, typename Mat3> void essential_matrix_8pt(const std::vector<V3> &x1, const std::vector<V3> &x2, Mat3 *E) {
    detail::check(plb_essential_matrix_8pt_batch(1, x1.size(), detail::raw(x1), detail::raw(x2), reinterpret_cast<double *>(E)));
}
template <typename V3, typename Pose> int relpose_8pt(const std::vector<V3> &x1, const std::vector<V3> &x2, std::vector<Pose> *output) {
    double out[28];
    int32_t n = 0;
    detail::check(plb_relpose_8pt_batch(1, x1.size(), detail::raw(x1), detail::raw(x2), out, &n));
    output->clear(); // relpose_8pt.cc:91
    for (int i = 0; i < n; ++i) {
        Pose p;
        detail::pose_from(out + 7 * i, &p);
        output->push_back(p);
    }
    return n;
}

// ---- batches of independent image pairs over the GPUs of the process (no reference counterpart: PoseLib callers loop) --
// One estimate_relative_pose per element, all in ONE call: lock-step groups on every device (n_gpus = 0: all devices,
// k: the first k, -1: the calling thread's device), results written back into poses / inliers / the returned stats.
template <typename RansacStats, typename P2, typename Camera, typename Opt, typename Pose>
std::vector<RansacStats> estimate_relative_pose_batch(const std::vector<std::vector<P2>> &x1, const std::vector<std::vector<P2>> &x2,
                                                      const std::vector<Camera> &camera1, const std::vector<Camera> &camera2,
                                                      const Opt &opt, std::vector<Pose> *poses,
                                                      std::vector<std::vector<char>> *inliers, int n_gpus = 0, int streams = 8) {
    const size_t count = x1.size();
    std::vector<plb_estimate_problem> P(count);
    poses->resize(count);
    inliers->resize(count);
    for (size_t i = 0; i < count; ++i) {
        plb_estimate_problem &q = P[i];
        q = plb_estimate_problem();
        q.kind = PLB_KIND_RELPOSE;
        q.tangent_sampson = opt.tangent_sampson ? 1 : 0;
        q.n = x1[i].size();
        q.a = detail::raw(x1[i]);
        q.b = detail::raw(x2[i]);
        q.camera1 = detail::camera_to_c(camera1[i]);
        q.camera2 = detail::camera_to_c(camera2[i]);
        q.ransac = detail::to_c(opt.ransac);
        q.bundle = detail::bundle_to_c(opt.bundle);
        q.max_error = opt.max_error;
        detail::pose_to((*poses)[i], q.model);
        (*inliers)[i].resize(x1[i].size());
        q.inliers = (*inliers)[i].data();
    }
    detail::check(plb_estimate_batch(P.data(), count, n_gpus, streams));
    std::vector<RansacStats> out(count);
    for (size_t i = 0; i < count; ++i) {
        detail::pose_from(P[i].model, &(*poses)[i]);
        out[i] = detail::from_c<RansacStats>(P[i].stats);
    }
    return out;
}
// Many refine_relpose(x1, x2, CameraPose*, opt, weights) (robust/bundle.h:84-86) in one call (plb_refine_batch): element
// i refines (*poses)[i] on x1[i], x2[i] with weights[i], and returns what the single call returns, bit for bit.
// weights[i] is used when it has one weight per point; a missing or wrongly sized entry means uniform weights.
template <typename BundleStats, typename P2, typename Pose, typename BOpt>
std::vector<BundleStats> refine_relpose_batch(const std::vector<std::vector<P2>> &x1, const std::vector<std::vector<P2>> &x2,
                                              std::vector<Pose> *poses, const BOpt &opt,
                                              const std::vector<std::vector<double>> &weights = {}, int n_gpus = 0,
                                              int streams = 8) {
    const size_t count = x1.size();
    if (x2.size() != count || poses->size() != count)
        throw std::invalid_argument("poselib_b200::refine_relpose_batch: x1, x2 and poses differ in size");
    std::vector<plb_refine_problem> P(count);
    for (size_t i = 0; i < count; ++i) {
        plb_refine_problem &q = P[i];
        q = plb_refine_problem();
        q.refiner = PLB_REFINER_RELPOSE;
        q.n = x1[i].size();
        q.a = detail::raw(x1[i]);
        q.b = detail::raw(x2[i]);
        q.weights = i < weights.size() ? detail::weights_of(weights[i], x1[i].size()) : nullptr;
        q.camera1.model_id = q.camera2.model_id = PLB_CAMERA_NULL;
        q.bundle = detail::bundle_to_c(opt);
        detail::pose_to((*poses)[i], q.model);
    }
    detail::check(plb_refine_batch(P.data(), count, n_gpus, streams));
    std::vector<BundleStats> out(count);
    for (size_t i = 0; i < count; ++i) {
        detail::pose_from(P[i].model, &(*poses)[i]);
        out[i] = detail::bundle_from_c<BundleStats>(P[i].bundle_stats);
    }
    return out;
}
// Many bundle_adjust(x, X, Image*, opt, weights) (robust/bundle.h:47) in one call (plb_refine_batch): element i refines
// the pose and the selected camera parameters of (*images)[i], as the single call does, bit for bit.  Weights as in
// refine_relpose_batch.
template <typename BundleStats, typename P2, typename P3, typename Image, typename BOpt>
std::vector<BundleStats> bundle_adjust_image_batch(const std::vector<std::vector<P2>> &x, const std::vector<std::vector<P3>> &X,
                                                   std::vector<Image> *images, const BOpt &opt,
                                                   const std::vector<std::vector<double>> &weights = {}, int n_gpus = 0,
                                                   int streams = 8) {
    const size_t count = x.size();
    if (X.size() != count || images->size() != count)
        throw std::invalid_argument("poselib_b200::bundle_adjust_image_batch: x, X and images differ in size");
    std::vector<plb_refine_problem> P(count);
    for (size_t i = 0; i < count; ++i) {
        plb_refine_problem &q = P[i];
        q = plb_refine_problem();
        q.refiner = PLB_REFINER_BUNDLE_IMAGE;
        q.n = x[i].size();
        q.a = detail::raw(x[i]);
        q.b = detail::raw(X[i]);
        q.weights = i < weights.size() ? detail::weights_of(weights[i], x[i].size()) : nullptr;
        q.camera1 = detail::camera_to_c((*images)[i].camera);
        q.camera2.model_id = PLB_CAMERA_NULL;
        q.bundle = detail::bundle_to_c(opt);
        detail::pose_to((*images)[i].pose, q.model);
    }
    detail::check(plb_refine_batch(P.data(), count, n_gpus, streams));
    std::vector<BundleStats> out(count);
    for (size_t i = 0; i < count; ++i) {
        detail::pose_from(P[i].model, &(*images)[i].pose);
        detail::camera_from_c(P[i].camera1, &(*images)[i].camera);
        out[i] = detail::bundle_from_c<BundleStats>(P[i].bundle_stats);
    }
    return out;
}

// ---- robust/utils.h scorers and get_inliers on given models (plb_score_batch) ----------------------------------------
// compute_msac_score / compute_sampson_msac_score / compute_tangent_sampson_msac_score / compute_homography_msac_score
// with get_inliers / get_tangent_sampson_inliers / get_homography_inliers (robust/utils.h:40-87) for many models of one
// problem in one call: scores[i], num_inliers[i] and, when asked for, inliers[i] (n chars) of model i.  sq_threshold is
// squared, in the points' units (pixels^2 for the tangent-Sampson form).  These are separate names on purpose: the
// drop-in does not redefine utils.h, whose functions PoseLib's own CPU estimators call once per hypothesis.
struct ScoreResult {
    std::vector<double> scores;
    std::vector<int64_t> num_inliers;
    std::vector<std::vector<char>> inliers; // empty unless asked for
};
namespace detail {
inline ScoreResult score_models(plb_score_problem q, const std::vector<double> &rows, bool want_inliers) {
    const size_t m = q.m, n = q.n;
    ScoreResult r;
    r.scores.assign(m, 0.0);
    r.num_inliers.assign(m, 0);
    std::vector<char> flat(want_inliers ? m * n : 0);
    q.models = rows.empty() ? nullptr : rows.data();
    q.scores = r.scores.empty() ? nullptr : r.scores.data();
    q.num_inliers = r.num_inliers.empty() ? nullptr : r.num_inliers.data();
    q.inliers = flat.empty() ? nullptr : flat.data();
    check(plb_score_batch(&q, 1, -1, 1));
    if (want_inliers)
        for (size_t i = 0; i < m; ++i) r.inliers.emplace_back(flat.begin() + i * n, flat.begin() + (i + 1) * n);
    return r;
}
inline plb_score_problem score_problem(int kind, size_t n, const double *a, const double *b, double sq_threshold) {
    plb_score_problem q = plb_score_problem();
    q.kind = kind;
    q.n = n;
    q.a = a;
    q.b = b;
    q.camera1.model_id = q.camera2.model_id = PLB_CAMERA_NULL;
    q.sq_threshold = sq_threshold;
    return q;
}
template <typename Pose> inline std::vector<double> pose_rows(const std::vector<Pose> &poses) {
    std::vector<double> rows(7 * poses.size());
    for (size_t i = 0; i < poses.size(); ++i) pose_to(poses[i], rows.data() + 7 * i);
    return rows;
}
template <typename Mat3> inline std::vector<double> matrix_rows(const std::vector<Mat3> &ms) {
    static_assert(sizeof(Mat3) == 9 * sizeof(double), "column-major 3x3 of doubles required");
    std::vector<double> rows(9 * ms.size());
    for (size_t i = 0; i < ms.size(); ++i)
        for (int k = 0; k < 9; ++k) rows[9 * i + k] = reinterpret_cast<const double *>(&ms[i])[k];
    return rows;
}
} // namespace detail
// compute_msac_score(pose, x, X) (utils.cc:36-63) and get_inliers(pose, x, X) (:374-383)
template <typename P2, typename P3, typename Pose>
ScoreResult score_absolute_poses(const std::vector<P2> &x, const std::vector<P3> &X, const std::vector<Pose> &poses,
                                 double sq_threshold, bool want_inliers = false) {
    static_assert(sizeof(P2) == 2 * sizeof(double) && sizeof(P3) == 3 * sizeof(double), "dense point layout required");
    plb_score_problem q = detail::score_problem(PLB_KIND_PNP, x.size(), detail::raw(x), detail::raw(X), sq_threshold);
    q.m = poses.size();
    return detail::score_models(q, detail::pose_rows(poses), want_inliers);
}
// compute_sampson_msac_score(pose, x1, x2) (utils.cc:158-201) and get_inliers(pose, x1, x2) (:434-476)
template <typename P2, typename Pose>
ScoreResult score_relative_poses(const std::vector<P2> &x1, const std::vector<P2> &x2, const std::vector<Pose> &poses,
                                 double sq_threshold, bool want_inliers = false) {
    static_assert(sizeof(P2) == 2 * sizeof(double), "dense point layout required");
    plb_score_problem q = detail::score_problem(PLB_KIND_RELPOSE, x1.size(), detail::raw(x1), detail::raw(x2), sq_threshold);
    q.m = poses.size();
    return detail::score_models(q, detail::pose_rows(poses), want_inliers);
}
// compute_tangent_sampson_msac_score / get_tangent_sampson_inliers (utils.cc:269-298,541-569) on the pixels x1, x2 of
// camera1, camera2, unprojected as ransac_relpose(x1, x2, camera1, camera2) does (ransac.cc:155-168)
template <typename P2, typename Camera, typename Pose>
ScoreResult score_relative_poses(const std::vector<P2> &x1, const std::vector<P2> &x2, const Camera &camera1,
                                 const Camera &camera2, const std::vector<Pose> &poses, double sq_threshold,
                                 bool want_inliers = false) {
    static_assert(sizeof(P2) == 2 * sizeof(double), "dense point layout required");
    plb_score_problem q = detail::score_problem(PLB_KIND_RELPOSE, x1.size(), detail::raw(x1), detail::raw(x2), sq_threshold);
    q.tangent_sampson = 1;
    q.camera1 = detail::camera_to_c(camera1);
    q.camera2 = detail::camera_to_c(camera2);
    q.m = poses.size();
    return detail::score_models(q, detail::pose_rows(poses), want_inliers);
}
// compute_sampson_msac_score(F, x1, x2) (utils.cc:204-239) and get_inliers(E, x1, x2) (:479-513)
template <typename P2, typename Mat3>
ScoreResult score_fundamentals(const std::vector<P2> &x1, const std::vector<P2> &x2, const std::vector<Mat3> &F,
                               double sq_threshold, bool want_inliers = false) {
    static_assert(sizeof(P2) == 2 * sizeof(double), "dense point layout required");
    plb_score_problem q = detail::score_problem(PLB_KIND_FUNDAMENTAL, x1.size(), detail::raw(x1), detail::raw(x2), sq_threshold);
    q.m = F.size();
    return detail::score_models(q, detail::matrix_rows(F), want_inliers);
}
// compute_homography_msac_score (utils.cc:300-329) and get_homography_inliers (:331-351)
template <typename P2, typename Mat3>
ScoreResult score_homographies(const std::vector<P2> &x1, const std::vector<P2> &x2, const std::vector<Mat3> &H,
                               double sq_threshold, bool want_inliers = false) {
    static_assert(sizeof(P2) == 2 * sizeof(double), "dense point layout required");
    plb_score_problem q = detail::score_problem(PLB_KIND_HOMOGRAPHY, x1.size(), detail::raw(x1), detail::raw(x2), sq_threshold);
    q.m = H.size();
    return detail::score_models(q, detail::matrix_rows(H), want_inliers);
}

// ---- Camera::project / unproject over many cameras (plb_camera_batch) ------------------------------------------------
// The vector forms of Camera::project, project_with_jac (misc/camera_models.cc:205-251), unproject and unproject_with_jac
// (:253-300) for many cameras in one call: camera i's points x[i] -> (*out)[i], with (*jac)[i] and (*jac_params)[i] when
// those are given.  P2 / P3 are dense 2- / 3-vectors of doubles, J a dense column-major 2x3 (project) or 3x2
// (unproject) matrix of doubles (Eigen::Matrix<double, 2, 3> / <3, 2>), JP a matrix with resize(rows, cols) and a
// column-major data() (Eigen::Matrix<double, 2 | 3, Eigen::Dynamic>).  These are separate names on purpose: the drop-in
// does not redefine Camera's members, which PoseLib's own CPU code calls one point at a time.
namespace detail {
struct Mat6 { // the type of an absent point Jacobian argument
    double d[6];
};
struct DynMat { // the type of an absent parameter Jacobian argument
    std::vector<double> v;
    void resize(int r, int c) { v.resize((size_t)r * c); }
    double *data() { return v.data(); }
};
inline int camera_num_params(int model_id) {
    switch (model_id) {
    case PLB_CAMERA_SIMPLE_PINHOLE: return 3;
    case PLB_CAMERA_PINHOLE: case PLB_CAMERA_SIMPLE_RADIAL: case PLB_CAMERA_SIMPLE_RADIAL_FISHEYE:
    case PLB_CAMERA_SIMPLE_DIVISION: return 4;
    case PLB_CAMERA_RADIAL: case PLB_CAMERA_RADIAL_FISHEYE: case PLB_CAMERA_DIVISION: return 5;
    case PLB_CAMERA_OPENCV: return 8;
    default: return 0;
    }
}
template <typename Camera, typename In, typename Out, typename J, typename JP>
void camera_points(int op, const std::vector<Camera> &cameras, const std::vector<std::vector<In>> &x,
                   std::vector<std::vector<Out>> *out, std::vector<std::vector<J>> *jac,
                   std::vector<std::vector<JP>> *jac_params) {
    const int in_w = op == PLB_CAMOP_PROJECT ? 3 : 2, out_w = op == PLB_CAMOP_PROJECT ? 2 : 3, rows = out_w;
    static_assert(sizeof(J) == 6 * sizeof(double), "dense 2x3 / 3x2 Jacobians of doubles required");
    if (sizeof(In) != in_w * sizeof(double) || sizeof(Out) != out_w * sizeof(double))
        throw std::invalid_argument("poselib_b200: dense point layout required");
    if (x.size() != cameras.size()) throw std::invalid_argument("poselib_b200: one point list per camera required");
    const size_t count = cameras.size();
    std::vector<plb_camera_problem> P(count);
    std::vector<std::vector<double>> jp(count);
    out->resize(count);
    if (jac) jac->resize(count);
    if (jac_params) jac_params->resize(count);
    for (size_t i = 0; i < count; ++i) {
        plb_camera_problem &q = P[i] = plb_camera_problem();
        const size_t n = x[i].size();
        q.op = op;
        q.n = n;
        q.camera = camera_to_c(cameras[i]);
        q.in = raw(x[i]);
        (*out)[i].resize(n);
        q.out = n ? reinterpret_cast<double *>((*out)[i].data()) : nullptr;
        if (jac) {
            (*jac)[i].resize(n);
            q.jac = n ? reinterpret_cast<double *>((*jac)[i].data()) : nullptr;
        }
        if (jac_params) {
            jp[i].assign(n * rows * camera_num_params(q.camera.model_id) + 1, 0.0);
            q.jac_params = jp[i].data();
        }
    }
    check(plb_camera_batch(P.data(), count, -1, 1));
    if (!jac_params) return;
    for (size_t i = 0; i < count; ++i) {
        const int np = camera_num_params(P[i].camera.model_id);
        std::vector<JP> &dst = (*jac_params)[i];
        dst.resize(x[i].size());
        for (size_t k = 0; k < dst.size(); ++k) {
            dst[k].resize(rows, np);
            for (int e = 0; e < rows * np; ++e) dst[k].data()[e] = jp[i][k * rows * np + e];
        }
    }
}
} // namespace detail
// Camera::project (jac and jac_params null) or project_with_jac of each camera's points x[i] -> xp[i]
template <typename Camera, typename P3, typename P2, typename J = detail::Mat6, typename JP = detail::DynMat>
void project_points(const std::vector<Camera> &cameras, const std::vector<std::vector<P3>> &x,
                    std::vector<std::vector<P2>> *xp, std::vector<std::vector<J>> *jac = nullptr,
                    std::vector<std::vector<JP>> *jac_params = nullptr) {
    detail::camera_points(PLB_CAMOP_PROJECT, cameras, x, xp, jac, jac_params);
}
// Camera::unproject to bearings (jac and jac_params null) or unproject_with_jac of each camera's pixels xp[i] -> x[i]
template <typename Camera, typename P2, typename P3, typename J = detail::Mat6, typename JP = detail::DynMat>
void unproject_points(const std::vector<Camera> &cameras, const std::vector<std::vector<P2>> &xp,
                      std::vector<std::vector<P3>> *x, std::vector<std::vector<J>> *jac = nullptr,
                      std::vector<std::vector<JP>> *jac_params = nullptr) {
    detail::camera_points(PLB_CAMOP_UNPROJECT, cameras, xp, x, jac, jac_params);
}

} // namespace poselib_b200
