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
    c.reserved = 0;
    c.loss_scale = o.loss_scale;
    c.gradient_tol = o.gradient_tol;
    c.step_tol = o.step_tol;
    c.relative_cost_tol = o.relative_cost_tol;
    c.initial_lambda = o.initial_lambda;
    c.min_lambda = o.min_lambda;
    c.max_lambda = o.max_lambda;
    if (static_cast<int>(o.lambda_update) != 0 || static_cast<int>(o.damping) != 0 || o.refine_focal_length ||
        o.refine_extra_params || o.refine_principal_point)
        throw std::runtime_error("poselib_b200: NYI bundle option (FIXED_FACTOR / MARQUARDT / intrinsics refinement)");
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
// misc/camera_models.h:59-157 -> plb_camera (six models on the path; others raise NYI inside the library)
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
    detail::check(plb_estimate_absolute_pose(detail::raw(points2D), detail::raw(points3D), points2D.size(), &ro, &bo,
                                             opt.max_error, &cam, m, inliers->data(), &st, nullptr));
    detail::pose_from(m, &image->pose);
    return detail::from_c<RansacStats>(st);
}
// estimate_relative_pose(x1, x2, camera1, camera2, RelativePoseOptions, CameraPose*, inliers*)   robust.h:68-70
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
    detail::check(plb_estimate_relative_pose(detail::raw(x1), detail::raw(x2), x1.size(), &c1, &c2, &ro, &bo,
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

// ---- robust/bundle.h: the LM refiners (uniform weights; the reference's optional per-residual weights are NYI) -----
// BundleStats carries iterations, initial_cost and cost; lambda / step_norm / grad_norm stay at their defaults.
namespace detail {
template <typename BundleStats> inline BundleStats bundle_from_c(const double s[3]) {
    BundleStats b = BundleStats();
    b.iterations = static_cast<size_t>(s[0]);
    b.initial_cost = s[1];
    b.cost = s[2];
    return b;
}
inline void no_weights(const std::vector<double> &weights) {
    if (!weights.empty()) throw std::runtime_error("poselib_b200: NYI (per-residual weights in the LM refiners)");
}
} // namespace detail
// bundle_adjust(x, X, CameraPose*, BundleOptions, weights)   robust/bundle.h:41-43
template <typename BundleStats, typename P2, typename P3, typename Pose, typename BOpt>
BundleStats bundle_adjust(const std::vector<P2> &x, const std::vector<P3> &X, Pose *pose, const BOpt &opt,
                          const std::vector<double> &weights = std::vector<double>()) {
    detail::no_weights(weights);
    double m[7], st[3];
    detail::pose_to(*pose, m);
    plb_bundle_opt bo = detail::bundle_to_c(opt);
    detail::check(plb_bundle_adjust(detail::raw(x), detail::raw(X), x.size(), m, &bo, st));
    detail::pose_from(m, pose);
    return detail::bundle_from_c<BundleStats>(st);
}
// refine_relpose(x1, x2, CameraPose*, BundleOptions, weights)   robust/bundle.h:84-86
template <typename BundleStats, typename P2, typename Pose, typename BOpt>
BundleStats refine_relpose(const std::vector<P2> &x1, const std::vector<P2> &x2, Pose *pose, const BOpt &opt,
                           const std::vector<double> &weights = std::vector<double>()) {
    detail::no_weights(weights);
    double m[7], st[3];
    detail::pose_to(*pose, m);
    plb_bundle_opt bo = detail::bundle_to_c(opt);
    detail::check(plb_refine_relpose(detail::raw(x1), detail::raw(x2), x1.size(), m, &bo, st));
    detail::pose_from(m, pose);
    return detail::bundle_from_c<BundleStats>(st);
}
// refine_fundamental(x1, x2, Matrix3d*, BundleOptions, weights)   robust/bundle.h:132-134
template <typename BundleStats, typename P2, typename Mat3, typename BOpt>
BundleStats refine_fundamental(const std::vector<P2> &x1, const std::vector<P2> &x2, Mat3 *F, const BOpt &opt,
                               const std::vector<double> &weights = std::vector<double>()) {
    static_assert(sizeof(Mat3) == 9 * sizeof(double), "column-major 3x3 of doubles required");
    detail::no_weights(weights);
    double st[3];
    plb_bundle_opt bo = detail::bundle_to_c(opt);
    detail::check(plb_refine_fundamental(detail::raw(x1), detail::raw(x2), x1.size(), reinterpret_cast<double *>(F), &bo, st));
    return detail::bundle_from_c<BundleStats>(st);
}
// refine_homography(x1, x2, Matrix3d*, BundleOptions, weights)   robust/bundle.h:148-150
template <typename BundleStats, typename P2, typename Mat3, typename BOpt>
BundleStats refine_homography(const std::vector<P2> &x1, const std::vector<P2> &x2, Mat3 *H, const BOpt &opt,
                              const std::vector<double> &weights = std::vector<double>()) {
    static_assert(sizeof(Mat3) == 9 * sizeof(double), "column-major 3x3 of doubles required");
    detail::no_weights(weights);
    double st[3];
    plb_bundle_opt bo = detail::bundle_to_c(opt);
    detail::check(plb_refine_homography(detail::raw(x1), detail::raw(x2), x1.size(), reinterpret_cast<double *>(H), &bo, st));
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

} // namespace poselib_b200
