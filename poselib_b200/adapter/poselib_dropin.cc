// poselib_dropin.cc — the translation unit a PoseLib maintainer adds to route the ONE hot path to the CUDA library.
//
// It DEFINES, with exactly the signatures PoseLib's own headers DECLARE, the functions of that path, in namespace poselib:
//   PoseLib/robust.h          estimate_absolute_pose :45-46, estimate_relative_pose :68-70, estimate_fundamental :112-113,
//                             estimate_homography :133-134                                   (CPU bodies: robust.cc)
//   PoseLib/robust/ransac.h   ransac_pnp :39-40, ransac_relpose :60-64 (both overloads), ransac_fundamental :85-87,
//                             ransac_homography :99-101                                      (CPU bodies: robust/ransac.cc)
//   PoseLib/robust/bundle.h   bundle_adjust :41-43, refine_relpose :84-86, refine_fundamental :132-134,
//                             refine_homography :148-150                                     (CPU bodies: robust/bundle.cc)
//   PoseLib/solvers/*.h       p3p, p3p_lambdatwist, relpose_5pt (both overloads), relpose_7pt, homography_4pt
//                                                                                        (CPU bodies: solvers/*.cc)
// Build it INSTEAD of the CPU bodies of these symbols (INTEGRATION.md §1) with PoseLib's include path and Eigen, and link
// -lposelib_b200.  Because the declarations come from PoseLib's headers, a signature that drifts from the reference is a
// compile or link error, not a silent overload: tests/test_dropin_reference_headers.py compiles this file against the
// reference's headers and links a client written against PoseLib's headers only.
//
// Entry points of those headers that are NOT on the path (generalized / hybrid / monodepth / focal-estimating variants,
// Image- and ImagePair-based refiners with intrinsics refinement) stay with PoseLib's CPU sources.
#include "PoseLib/robust.h"
#include "PoseLib/robust/bundle.h"
#include "PoseLib/robust/ransac.h"
#include "PoseLib/solvers/homography_4pt.h"
#include "PoseLib/solvers/p3p.h"
#include "PoseLib/solvers/p3p_lambdatwist.h"
#include "PoseLib/solvers/relpose_5pt.h"
#include "PoseLib/solvers/relpose_7pt.h"

#include "poselib_b200.hpp"

namespace poselib {

// ---- PoseLib/robust.h ----------------------------------------------------------------------------------------------
RansacStats estimate_absolute_pose(const std::vector<Point2D> &points2D, const std::vector<Point3D> &points3D,
                                   AbsolutePoseOptions opt, Image *image, std::vector<char> *inliers) {
    return poselib_b200::estimate_absolute_pose<RansacStats>(points2D, points3D, opt, image, inliers);
}
RansacStats estimate_relative_pose(const std::vector<Point2D> &points2D_1, const std::vector<Point2D> &points2D_2,
                                   const Camera &camera1, const Camera &camera2, const RelativePoseOptions &opt,
                                   CameraPose *relative_pose, std::vector<char> *inliers) {
    return poselib_b200::estimate_relative_pose<RansacStats>(points2D_1, points2D_2, camera1, camera2, opt, relative_pose,
                                                             inliers);
}
RansacStats estimate_fundamental(const std::vector<Point2D> &points2D_1, const std::vector<Point2D> &points2D_2,
                                 const RelativePoseOptions &opt, Eigen::Matrix3d *F, std::vector<char> *inliers) {
    return poselib_b200::estimate_fundamental<RansacStats>(points2D_1, points2D_2, opt, F, inliers);
}
RansacStats estimate_homography(const std::vector<Point2D> &points2D_1, const std::vector<Point2D> &points2D_2,
                                const HomographyOptions &opt, Eigen::Matrix3d *H, std::vector<char> *inliers) {
    return poselib_b200::estimate_homography<RansacStats>(points2D_1, points2D_2, opt, H, inliers);
}

// ---- PoseLib/robust/ransac.h ---------------------------------------------------------------------------------------
RansacStats ransac_pnp(const std::vector<Point2D> &x, const std::vector<Point3D> &X, const AbsolutePoseOptions &opt,
                       CameraPose *best_model, std::vector<char> *best_inliers) {
    return poselib_b200::ransac_pnp<RansacStats>(x, X, opt, best_model, best_inliers);
}
RansacStats ransac_relpose(const std::vector<Point2D> &x1, const std::vector<Point2D> &x2,
                           const RelativePoseOptions &opt, CameraPose *best_model, std::vector<char> *best_inliers) {
    return poselib_b200::ransac_relpose<RansacStats>(x1, x2, opt, best_model, best_inliers);
}
RansacStats ransac_relpose(const std::vector<Point2D> &x1, const std::vector<Point2D> &x2, const Camera &camera1,
                           const Camera &camera2, const RelativePoseOptions &opt, CameraPose *best_model,
                           std::vector<char> *best_inliers) {
    return poselib_b200::ransac_relpose<RansacStats>(x1, x2, camera1, camera2, opt, best_model, best_inliers);
}
RansacStats ransac_fundamental(const std::vector<Point2D> &x1, const std::vector<Point2D> &x2,
                               const RelativePoseOptions &opt, Eigen::Matrix3d *best_model,
                               std::vector<char> *best_inliers) {
    return poselib_b200::ransac_fundamental<RansacStats>(x1, x2, opt, best_model, best_inliers);
}
RansacStats ransac_homography(const std::vector<Point2D> &x1, const std::vector<Point2D> &x2,
                              const HomographyOptions &opt, Eigen::Matrix3d *best_model,
                              std::vector<char> *best_inliers) {
    return poselib_b200::ransac_homography<RansacStats>(x1, x2, opt, best_model, best_inliers);
}

// ---- PoseLib/robust/bundle.h ---------------------------------------------------------------------------------------
BundleStats bundle_adjust(const std::vector<Point2D> &x, const std::vector<Point3D> &X, CameraPose *pose,
                          const BundleOptions &opt, const std::vector<double> &weights) {
    return poselib_b200::bundle_adjust<BundleStats>(x, X, pose, opt, weights);
}
BundleStats refine_relpose(const std::vector<Point2D> &x1, const std::vector<Point2D> &x2, CameraPose *pose,
                           const BundleOptions &opt, const std::vector<double> &weights) {
    return poselib_b200::refine_relpose<BundleStats>(x1, x2, pose, opt, weights);
}
BundleStats refine_fundamental(const std::vector<Point2D> &x1, const std::vector<Point2D> &x2, Eigen::Matrix3d *F,
                               const BundleOptions &opt, const std::vector<double> &weights) {
    return poselib_b200::refine_fundamental<BundleStats>(x1, x2, F, opt, weights);
}
BundleStats refine_homography(const std::vector<Point2D> &x1, const std::vector<Point2D> &x2, Eigen::Matrix3d *H,
                              const BundleOptions &opt, const std::vector<double> &weights) {
    return poselib_b200::refine_homography<BundleStats>(x1, x2, H, opt, weights);
}

// ---- PoseLib/solvers/*.h -------------------------------------------------------------------------------------------
int p3p(const std::vector<Eigen::Vector3d> &x, const std::vector<Eigen::Vector3d> &X, std::vector<CameraPose> *output) {
    return poselib_b200::p3p(x, X, output);
}
int p3p_lambdatwist(const std::vector<Eigen::Vector3d> &x, const std::vector<Eigen::Vector3d> &X,
                    std::vector<CameraPose> *output) {
    return poselib_b200::p3p_lambdatwist(x, X, output);
}
int relpose_5pt(const std::vector<Eigen::Vector3d> &x1, const std::vector<Eigen::Vector3d> &x2,
                std::vector<Eigen::Matrix3d> *essential_matrices) {
    return poselib_b200::relpose_5pt(x1, x2, essential_matrices);
}
int relpose_5pt(const std::vector<Eigen::Vector3d> &x1, const std::vector<Eigen::Vector3d> &x2,
                std::vector<CameraPose> *output) {
    return poselib_b200::relpose_5pt_poses(x1, x2, output);
}
int relpose_7pt(const std::vector<Eigen::Vector3d> &x1, const std::vector<Eigen::Vector3d> &x2,
                std::vector<Eigen::Matrix3d> *fundamental_matrices) {
    return poselib_b200::relpose_7pt(x1, x2, fundamental_matrices);
}
int homography_4pt(const std::vector<Eigen::Vector3d> &x1, const std::vector<Eigen::Vector3d> &x2, Eigen::Matrix3d *H,
                   bool check_cheirality) {
    return poselib_b200::homography_4pt(x1, x2, H, check_cheirality);
}

} // namespace poselib
