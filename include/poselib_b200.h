/* poselib_b200 — C-ABI of the H100-native LO-RANSAC / minimal-solver engine.
 *
 * Drop-in boundary for ONE hot path of PoseLib (reference @ a69263d, paths below are relative to the
 * reference checkout): the LO-RANSAC hypothesis pipeline behind PoseLib/robust.h and PoseLib/solvers/.
 * The reference has no FFI/plugin mechanism (plain C++ free functions taking std::vector<Eigen::...>), so
 * every entry point here is the POD restatement of one reference function; the header-only adapter
 * poselib_b200/adapter/poselib_b200.hpp gives them back their PoseLib signatures.
 *
 * Conventions
 *  - plain pointers + sizes, caller-allocated outputs, no exceptions; return 0 = ok, <0 = error
 *    (plb_last_error() holds the message).  The reference never reports errors on this path except
 *    Camera::unproject throwing "NYI" for unknown model ids (misc/camera_models.cc:184-185) -> PLB_ERR_NYI.
 *  - 2D points: double[2n] AoS (std::vector<Eigen::Vector2d>::data()); 3D points: double[3n];
 *    3x3 matrices: 9 doubles COLUMN-major (Eigen::Matrix3d); poses: q (w,x,y,z) then t (CameraPose,
 *    camera_pose.h:40-68).
 *  - `*_inout` models are read as the initial model iff opt->score_initial_model (robust/ransac.cc:47-50).
 *  - inliers: char[n] written by the callee (robust/utils.cc:376), may be NULL.
 *  - too few points: returns 0 with default stats (iterations 0, model_score DBL_MAX)
 *    (robust/ransac_impl.h:161-163, robust.cc:548-550,716-718).
 *  - all compute runs on the current CUDA device (plb_set_device); there is NO CPU fallback:
 *    without a usable device every compute entry point returns PLB_ERR_CUDA.
 */
#ifndef POSELIB_B200_H
#define POSELIB_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PLB_OK 0
#define PLB_ERR_CUDA (-1)
#define PLB_ERR_ARG (-2)
#define PLB_ERR_NYI (-3)

/* PoseLib/types.h:39-50 RansacOptions */
typedef struct plb_ransac_opt {
    uint64_t max_iterations;       /* 100000 */
    uint64_t min_iterations;       /* 1000 */
    double dyn_num_trials_mult;    /* 3.0 */
    double success_prob;           /* 0.9999 */
    uint64_t seed;                 /* 0 */
    int32_t progressive_sampling;  /* 0; PROSAC, assumes data sorted */
    int32_t score_initial_model;   /* 0 */
    uint64_t max_prosac_iterations; /* 100000 */
} plb_ransac_opt;

/* PoseLib/types.h:52-58 RansacStats */
typedef struct plb_ransac_stats {
    uint64_t refinements;
    uint64_t iterations;
    uint64_t num_inliers;
    double inlier_ratio;
    double model_score;
} plb_ransac_stats;

/* PoseLib/types.h:60-95 BundleOptions (fields read by the four in-scope refiners; NIELSEN + LEVENBERG) */
enum { PLB_LOSS_TRIVIAL = 0, PLB_LOSS_TRUNCATED = 1, PLB_LOSS_HUBER = 2, PLB_LOSS_CAUCHY = 3 };
/* refine_intrinsics: BundleOptions::refine_focal_length / refine_principal_point / refine_extra_params (types.h:92-94)
 * as a bit set.  The camera parameters they select (Camera::get_param_refinement_idx, camera_models.cc:545-561: focal
 * lengths, then principal point, then the model's extra parameters — k1..p2 of OPENCV, k / k1, k2 of the radial,
 * fisheye and division models; none for the NULL camera, no extras for the pinhole models) are refined with the pose
 * by plb_bundle_adjust_image and plb_estimate_absolute_pose_image (AbsolutePoseRefiner, optim/absolute.h:40-171), and,
 * for each of the two cameras, by plb_refine_relpose_pair and plb_estimate_relative_pose_pair with tangent_sampson
 * (CameraRelativePoseRefiner, bundle.cc:237-256, optim/relative.h:268-483).
 * Where the selection is non-empty the other entry points behave as follows:
 *   - ignored, as the reference ignores them: plb_bundle_adjust (NULL camera), plb_refine_relpose,
 *     plb_refine_fundamental, plb_refine_homography, plb_estimate_fundamental, plb_estimate_homography and
 *     plb_estimate_relative_pose without tangent_sampson;
 *   - PLB_ERR_NYI, as these cannot return the cameras: plb_refine_relpose_cameras (use plb_refine_relpose_pair), and
 *     plb_estimate_relative_pose / plb_estimate_batch with tangent_sampson when either camera's selection is non-empty;
 *   - PLB_ERR_ARG: plb_estimate_absolute_pose, which cannot return the camera (use plb_estimate_absolute_pose_image);
 *   - plb_estimate_batch refines the camera of PnP problems and writes it into camera1 (camera1 of the other problems
 *     is left untouched).
 * All of this is checked before any device call.  Other bits are ignored. */
enum { PLB_REFINE_FOCAL_LENGTH = 1, PLB_REFINE_PRINCIPAL_POINT = 2, PLB_REFINE_EXTRA_PARAMS = 4 };
typedef struct plb_bundle_opt {
    uint64_t max_iterations;   /* 100 */
    int32_t loss_type;         /* PLB_LOSS_CAUCHY */
    int32_t refine_intrinsics; /* 0; PLB_REFINE_* bits */
    double loss_scale;         /* 1.0 */
    double gradient_tol;       /* 1e-12 */
    double step_tol;           /* 1e-8 */
    double relative_cost_tol;  /* 1e-10 */
    double initial_lambda;     /* 1e-3 */
    double min_lambda;         /* 1e-10 */
    double max_lambda;         /* 1e10 */
} plb_bundle_opt;

/* Counters for the BASELINE metric (SURVEY.md §8d); not part of the reference structs. */
typedef struct plb_counters {
    uint64_t samples;       /* generate_models calls consumed by the loop (== stats.iterations) */
    uint64_t hypotheses;    /* models passed to score_model inside the loop */
    uint64_t scored_corrs;  /* hypotheses * N */
    uint64_t lo_calls;      /* refine_model calls */
    double lo_seconds;      /* host wall time spent waiting on LO kernels */
    uint64_t gpu_launches;  /* kernels launched for this call */
    uint64_t samples_evaluated; /* incl. speculative samples past the serial break point */
    double gpu_seconds;     /* CUDA-event time of the hypothesis kernels (sample + solve + score + select/confirm) */
    uint64_t h2d_bytes;     /* bytes copied host -> device for this call */
    uint64_t d2h_bytes;     /* bytes copied device -> host for this call */
    uint64_t models_evaluated; /* models scored by the hypothesis kernels incl. speculative samples */
    uint64_t models_confirmed; /* fast mode: models rescored in fp64 after the fp32 screening pass */
    double gpu_seconds_score;  /* CUDA-event time of the scoring / screening kernels alone (part of gpu_seconds) */
    double gpu_seconds_select; /* candidate selection + fp64 confirmation of the candidates (part of gpu_seconds) */
    double gpu_seconds_lo;     /* best-minimal pass + LO refinements (k_pass1 + k_lm) of the rounds, CUDA events */
    uint64_t rounds;           /* lock-step rounds (= host synchronisations inside the loop) of the problem's group */
} plb_counters;

/* misc/camera_models.h:39-157 Camera, restricted to the ten models on the path below.  Ids are the reference's
 * CameraModelId values.  The reference's other models -> PLB_ERR_NYI, like the reference's "NYI" throw
 * (camera_models.cc:184-185): OPENCV_FISHEYE (5), FULL_OPENCV (6), FOV (7), THIN_PRISM_FISHEYE (10),
 * RAD_TAN_THIN_PRISM_FISHEYE (11), RADIAL_1D (99) and SPHERICAL (100). */
enum {
    PLB_CAMERA_NULL = -1,
    PLB_CAMERA_SIMPLE_PINHOLE = 0,         /* f, cx, cy */
    PLB_CAMERA_PINHOLE = 1,                /* fx, fy, cx, cy */
    PLB_CAMERA_SIMPLE_RADIAL = 2,          /* f, cx, cy, k */
    PLB_CAMERA_RADIAL = 3,                 /* f, cx, cy, k1, k2 */
    PLB_CAMERA_OPENCV = 4,                 /* fx, fy, cx, cy, k1, k2, p1, p2 */
    PLB_CAMERA_SIMPLE_RADIAL_FISHEYE = 8,  /* f, cx, cy, k */
    PLB_CAMERA_RADIAL_FISHEYE = 9,         /* f, cx, cy, k1, k2 */
    PLB_CAMERA_DIVISION = 101,             /* fx, fy, cx, cy, k */
    PLB_CAMERA_SIMPLE_DIVISION = 102       /* f, cx, cy, k */
};
typedef struct plb_camera {
    int32_t model_id;
    int32_t width, height;
    int32_t reserved;
    double params[8];
} plb_camera;

void plb_ransac_opt_default(plb_ransac_opt *o);
void plb_bundle_opt_default(plb_bundle_opt *o);
const char *plb_last_error(void);
int plb_device_count(void);          /* CUDA devices visible; 0 if none / driver missing */
int plb_set_device(int device);      /* device used by subsequent calls from this thread */
/* precision mode of the calling thread (batch workers inherit it): 1 = fast, the DEFAULT (fp32 SMEM-resident screening
 * of every hypothesis with a rigorous error interval per model + fp64 confirmation of every model whose interval could
 * change the RANSAC state; results identical to mode 0), 0 = exact (fp64 scoring of every hypothesis).  The environment
 * variable PLB_MODE=0 changes the default. */
int plb_set_mode(int mode);

/* ---- host-side pieces of the loop; no device needed (exercised by the CPU test-suite) ---------------------
 * plb_host_sample_table: the first `iters` minimal samples (k indices each) RandomSampler(n, k, opt) draws
 * (robust/sampling.cc:37-61,85-136, incl. PROSAC and the int sign-extension of random_int before `% n`).
 * plb_host_dynamic_max_iter: compute_dynamic_max_iter (robust/ransac_impl.h:58-74). */
int plb_host_sample_table(uint64_t n, uint32_t k, const plb_ransac_opt *opt, uint64_t iters, uint32_t *out);
/* The table the DEVICE sampler of the engine draws (k_sample): `count` samplers with seeds opt->seed + j, `round`
 * samples per launch with the state carried across launches like the engine's rounds.  out: count * iters * k.
 * Test surface: pins the device sampler to plb_host_sample_table (itself pinned to robust/sampling.cc). */
int plb_device_sample_table(uint64_t n, uint32_t k, const plb_ransac_opt *opt, uint64_t iters, uint64_t round,
                            uint32_t count, uint32_t *out);
uint64_t plb_host_dynamic_max_iter(uint64_t num_inliers, uint64_t num_data, uint32_t sample_sz, double success_prob,
                                   double dyn_num_trials_mult, uint64_t min_iterations, uint64_t max_iterations);

/* ---- robust/ransac.h:39-40,60-61,85-87,99-101 (points already calibrated / normalised) ---------- */
int plb_ransac_pnp(const double *x_xy, const double *X_xyz, size_t n, const plb_ransac_opt *opt, double max_error,
                   double pose_inout[7], char *inliers, plb_ransac_stats *stats, plb_counters *counters);
int plb_ransac_relpose(const double *x1_xy, const double *x2_xy, size_t n, const plb_ransac_opt *opt,
                       double max_error, double pose_inout[7], char *inliers, plb_ransac_stats *stats,
                       plb_counters *counters);
int plb_ransac_fundamental(const double *x1_xy, const double *x2_xy, size_t n, const plb_ransac_opt *opt,
                           double max_error, int real_focal_check, double F_inout[9], char *inliers,
                           plb_ransac_stats *stats, plb_counters *counters);
int plb_ransac_homography(const double *x1_xy, const double *x2_xy, size_t n, const plb_ransac_opt *opt,
                          double max_error, double H_inout[9], char *inliers, plb_ransac_stats *stats,
                          plb_counters *counters);
/* robust/ransac.h:62-64, ransac.cc:155-168: relative pose with camera models, scored with the tangent Sampson error
 * on the unprojected bearings (CameraRelativePoseEstimator); x1/x2 and max_error in the pixel units of the cameras.
 * The start pose is reset to identity (ransac.cc:159-160). */
int plb_ransac_relpose_cameras(const double *x1_px, const double *x2_px, size_t n, const plb_camera *camera1,
                               const plb_camera *camera2, const plb_ransac_opt *opt, double max_error,
                               double pose_out[7], char *inliers, plb_ransac_stats *stats, plb_counters *counters);

/* ---- PoseLib/robust.h:45-46,68-70,112-113,133-134 (pixel coordinates + cameras) -------------------
 * The camera pre-step (Camera::unproject / unproject_with_jac of every point, robust.cc:40-43,255-266,287-292) runs
 * on the device.  tangent_sampson = RelativePoseOptions::tangent_sampson (types.h:140). */
int plb_estimate_absolute_pose(const double *points2D, const double *points3D, size_t n,
                               const plb_ransac_opt *ransac, const plb_bundle_opt *bundle, double max_error,
                               const plb_camera *camera, double pose_inout[7], char *inliers,
                               plb_ransac_stats *stats, plb_counters *counters);
/* estimate_absolute_pose with the Image* of the reference (robust.cc:36-126): like plb_estimate_absolute_pose, and the
 * final bundle adjustment also refines the camera parameters bundle->refine_intrinsics selects.  camera_inout is always
 * written back; after a final bundle adjustment (num_inliers > 3) it went through the reference's rescale(scale) /
 * rescale(1 / scale) round trip, which can change the last bits of parameters that were not refined. */
int plb_estimate_absolute_pose_image(const double *points2D, const double *points3D, size_t n,
                                     const plb_ransac_opt *ransac, const plb_bundle_opt *bundle, double max_error,
                                     plb_camera *camera_inout, double pose_inout[7], char *inliers,
                                     plb_ransac_stats *stats, plb_counters *counters);
int plb_estimate_relative_pose(const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                               const plb_camera *camera2, const plb_ransac_opt *ransac,
                               const plb_bundle_opt *bundle, double max_error, int tangent_sampson,
                               double pose_inout[7], char *inliers, plb_ransac_stats *stats,
                               plb_counters *counters);
/* estimate_relative_pose with the cameras in/out (robust.cc:242-314): like plb_estimate_relative_pose, and with
 * tangent_sampson and a non-empty selection of bundle->refine_intrinsics in either camera, the final bundle adjustment
 * (num_inliers > 5) runs CameraRelativePoseRefiner on x * scale with the rescaled cameras.  Pose, inlier mask and stats
 * are the reference's; RANSAC itself (its LO included) keeps the cameras fixed, as the reference does.  The one addition:
 * the refined cameras are written back to camera1_inout / camera2_inout through rescale(1 / scale); the reference
 * computes them and discards them.  Otherwise the cameras are left untouched. */
int plb_estimate_relative_pose_pair(const double *x1, const double *x2, size_t n, plb_camera *camera1_inout,
                                    plb_camera *camera2_inout, const plb_ransac_opt *ransac,
                                    const plb_bundle_opt *bundle, double max_error, int tangent_sampson,
                                    double pose_inout[7], char *inliers, plb_ransac_stats *stats,
                                    plb_counters *counters);
int plb_estimate_fundamental(const double *x1, const double *x2, size_t n, const plb_ransac_opt *ransac,
                             const plb_bundle_opt *bundle, double max_error, int real_focal_check,
                             double F_inout[9], char *inliers, plb_ransac_stats *stats, plb_counters *counters);
int plb_estimate_homography(const double *x1, const double *x2, size_t n, const plb_ransac_opt *ransac,
                            const plb_bundle_opt *bundle, double max_error, double H_inout[9], char *inliers,
                            plb_ransac_stats *stats, plb_counters *counters);

/* ---- PoseLib/solvers/{p3p.h:42, relpose_5pt.h:40-43, relpose_7pt.h:39-40, homography_4pt.h:38-39} ----
 * Inputs are UNIT bearing vectors, `count` independent instances back to back; one warp solves one
 * instance.  n_out[i] receives the number of solutions of instance i (the reference's return value);
 * outputs are padded to the per-solver maximum. */
int plb_p3p_batch(size_t count, const double *x /*count*3*3*/, const double *X /*count*3*3*/,
                  double *poses_out /*count*4*7*/, int32_t *n_out);
/* PoseLib/solvers/p3p_lambdatwist.h:44-45 (the alternative P3P of SURVEY row N2): same layout as plb_p3p_batch.  Its
 * closed-form cubic root goes through cbrt / cos / acos (CUDA's, 1-2 ulp from glibc's) before a Newton step and the
 * depth refinement: solutions agree with the CPU implementation to ~1e-12, not bit for bit. */
int plb_p3p_lambdatwist_batch(size_t count, const double *x /*count*3*3*/, const double *X /*count*3*3*/,
                              double *poses_out /*count*4*7*/, int32_t *n_out);
int plb_relpose_5pt_batch(size_t count, const double *x1 /*count*5*3*/, const double *x2,
                          double *E_out /*count*10*9*/, int32_t *n_out);
int plb_relpose_5pt_poses_batch(size_t count, const double *x1, const double *x2, double *poses_out /*count*40*7*/,
                                int32_t *n_out);
int plb_relpose_7pt_batch(size_t count, const double *x1 /*count*7*3*/, const double *x2,
                          double *F_out /*count*3*9*/, int32_t *n_out);
int plb_homography_4pt_batch(size_t count, const double *x1 /*count*4*3*/, const double *x2,
                             double *H_out /*count*9*/, int32_t *n_out, int check_cheirality);

/* solvers/relpose_8pt.h:45-53 (non-minimal): `count` instances of n >= 8 unit bearing pairs each (x1, x2: count*n*3).
 * essential_matrix_8pt: E_out count*9, column-major (Eigen::Matrix3d).  relpose_8pt: the poses of motion_from_essential
 * that pass the cheirality test on all n correspondences, poses_out count*4*7, n_out[i] = their number.
 * n == 8 takes the Householder nullspace (relpose_8pt.cc:63-67); n > 8 the smallest eigenvector of A^T A (:68-72) — an
 * iterative eigen-solver in the reference as here, so results agree to tolerance, not bit for bit. */
int plb_essential_matrix_8pt_batch(size_t count, size_t n, const double *x1, const double *x2, double *E_out);
int plb_relpose_8pt_batch(size_t count, size_t n, const double *x1, const double *x2, double *poses_out /*count*4*7*/,
                          int32_t *n_out);

/* ---- PoseLib/robust/bundle.h: bundle_adjust (calibrated, :41-43), refine_relpose (:84-86), refine_fundamental
 * (:132-134), refine_homography (:148-150) — the LM refiners the LO step and the final polish are built from.
 * bundle_stats_out (may be NULL): {iterations, initial_cost, cost}.
 * Weights: every refiner below but plb_bundle_adjust has a *_weighted twin that takes PoseLib's per-residual weights,
 * `weights` = n doubles in point order, or NULL for uniform weights (the twin is then the unweighted call).  Point k's
 * residuals enter the cost as weights[k] * loss and the normal equations with weights[k] * loss weight
 * (jacobian_accumulator.h:65-133); a residual with weight 0 still counts in the 1 / max(1, count) scale of the cost, so a
 * zero weight is not the same as dropping the point.  The homography refiner applies a point's weight to both its
 * forward and its backward residual.  Weights are not checked, as in the reference.  The reference uses the weights
 * only when weights.size() == n (bundle.cc:107-111 etc.); the adapter passes NULL otherwise.  There is no weighted
 * plb_bundle_adjust: the reference's calibrated bundle_adjust(x, X, CameraPose*, opt, weights) drops its weights
 * (bundle.cc:84-92). ------------------------------------------------------------------------------------------ */
int plb_bundle_adjust(const double *x_xy, const double *X_xyz, size_t n, double pose_inout[7],
                      const plb_bundle_opt *opt, double bundle_stats_out[3]);
/* bundle.h:47 bundle_adjust(x, X, Image*, opt) (bundle.cc:95-112): the pose and the camera parameters opt->refine_intrinsics
 * selects, points in the camera's pixel units as given (no rescaling).  Only the refined parameters of camera_inout are
 * written. */
int plb_bundle_adjust_image(const double *x_px, const double *X_xyz, size_t n, double pose_inout[7],
                            plb_camera *camera_inout, const plb_bundle_opt *opt, double bundle_stats_out[3]);
int plb_refine_relpose(const double *x1_xy, const double *x2_xy, size_t n, double pose_inout[7],
                       const plb_bundle_opt *opt, double bundle_stats_out[3]);
/* bundle.h refine_relpose(x1, x2, ImagePair*, opt) with fixed intrinsics (bundle.cc:237-247): tangent Sampson refiner */
int plb_refine_relpose_cameras(const double *x1_px, const double *x2_px, size_t n, const plb_camera *camera1,
                               const plb_camera *camera2, double pose_inout[7], const plb_bundle_opt *opt,
                               double bundle_stats_out[3]);
/* bundle.h refine_relpose(x1, x2, ImagePair*, opt) (bundle.cc:237-256): the pose and, in each camera, the parameters
 * opt->refine_intrinsics selects (CameraRelativePoseRefiner, separate intrinsics), pixels as given (no rescaling).  Only
 * the refined parameters of camera1_inout / camera2_inout are written.  Where neither selection is non-empty it is
 * plb_refine_relpose_cameras. */
int plb_refine_relpose_pair(const double *x1_px, const double *x2_px, size_t n, plb_camera *camera1_inout,
                            plb_camera *camera2_inout, double pose_inout[7], const plb_bundle_opt *opt,
                            double bundle_stats_out[3]);
int plb_refine_fundamental(const double *x1_xy, const double *x2_xy, size_t n, double F_inout[9],
                           const plb_bundle_opt *opt, double bundle_stats_out[3]);
int plb_refine_homography(const double *x1_xy, const double *x2_xy, size_t n, double H_inout[9],
                          const plb_bundle_opt *opt, double bundle_stats_out[3]);
int plb_bundle_adjust_image_weighted(const double *x_px, const double *X_xyz, size_t n, double pose_inout[7],
                                     plb_camera *camera_inout, const plb_bundle_opt *opt, double bundle_stats_out[3],
                                     const double *weights);
int plb_refine_relpose_weighted(const double *x1_xy, const double *x2_xy, size_t n, double pose_inout[7],
                                const plb_bundle_opt *opt, double bundle_stats_out[3], const double *weights);
int plb_refine_relpose_cameras_weighted(const double *x1_px, const double *x2_px, size_t n, const plb_camera *camera1,
                                        const plb_camera *camera2, double pose_inout[7], const plb_bundle_opt *opt,
                                        double bundle_stats_out[3], const double *weights);
int plb_refine_relpose_pair_weighted(const double *x1_px, const double *x2_px, size_t n, plb_camera *camera1_inout,
                                     plb_camera *camera2_inout, double pose_inout[7], const plb_bundle_opt *opt,
                                     double bundle_stats_out[3], const double *weights);
int plb_refine_fundamental_weighted(const double *x1_xy, const double *x2_xy, size_t n, double F_inout[9],
                                    const plb_bundle_opt *opt, double bundle_stats_out[3], const double *weights);
int plb_refine_homography_weighted(const double *x1_xy, const double *x2_xy, size_t n, double H_inout[9],
                                   const plb_bundle_opt *opt, double bundle_stats_out[3], const double *weights);

/* ---- batch of independent problems (BASELINE config 5); sharded by the caller across GPUs ---------- */
/* Every batch call below (plb_ransac_batch[_multi], plb_estimate_batch[_device], plb_refine_batch[_device],
 * plb_score_batch[_device], plb_generate_batch[_device], plb_camera_batch[_device]) checks its arguments in one order,
 * before any copy or launch:
 *   1. count 0 -> PLB_OK, nothing written;
 *   2. problems NULL -> PLB_ERR_ARG, nothing written;
 *   3. device forms: a dtype other than PLB_DTYPE_F64 / PLB_DTYPE_F32 -> PLB_ERR_ARG;
 *   4. every problem in order, by the rules its call lists; the first failure's code;
 *   5. n_gpus < -1 -> PLB_ERR_ARG (plb_ransac_batch_multi: n_gpus < 0);
 *   6. no device -> PLB_ERR_CUDA;
 *   7. n_gpus above the device count -> PLB_ERR_ARG;
 *   8. resident correspondences on a device the call does not use -> PLB_ERR_ARG; device forms: a pointer of a problem
 *      that is not device (or managed) memory of the calling thread's device, or is misaligned -> PLB_ERR_ARG;
 *   9. plb_generate_batch_device: a sample index outside [0, n) -> PLB_ERR_ARG, found by one reduction kernel over every
 *      problem's samples and one synchronisation, after the work queued on the caller's stream and before any other
 *      kernel reads a sample.
 * A failure in steps 3-9 writes its code into every status and nothing else: no model, stats, counters, camera, mask,
 * score or count changes.  After the checks, every status receives the call's result. */
enum { PLB_KIND_PNP = 0, PLB_KIND_RELPOSE = 1, PLB_KIND_FUNDAMENTAL = 2, PLB_KIND_HOMOGRAPHY = 3 };
typedef struct plb_problem {
    int32_t kind;             /* PLB_KIND_* */
    int32_t real_focal_check; /* fundamental only */
    uint64_t n;
    const double *a;          /* x (pnp) or x1 : 2n doubles */
    const double *b;          /* X (pnp): 3n doubles ; else x2: 2n doubles */
    plb_ransac_opt opt;
    double max_error;         /* in the units of the points (ransac_* level) */
    double model[9];          /* in/out: pose (7) or matrix (9, column-major) */
    char *inliers;            /* n bytes or NULL */
    plb_ransac_stats stats;   /* out */
    plb_counters counters;    /* out */
    int32_t status;           /* out: PLB_OK / error */
    int32_t resident;         /* > 0: handle from plb_resident_create, a/b are ignored (points already in HBM) */
} plb_problem;
/* Runs ransac_{pnp,relpose,fundamental,homography} on every problem on the calling thread's device; `streams` lock-step
 * groups of problems are in flight at once.  An unknown kind, a / b NULL with n > 0 (and no resident handle), or a
 * resident handle that is not one of plb_resident_create's for the problem's kind -> PLB_ERR_ARG. */
int plb_ransac_batch(plb_problem *problems, size_t count, int streams);
/* The same over the first n_gpus CUDA devices of the process (0 = all of them), in one call from one host thread:
 * problems are partitioned by size x expected iterations, every device runs streams_per_gpu groups at once, results
 * (stats, models, inlier masks) are written straight into the caller's array.  No collective: image pairs are
 * independent (robust/ransac.cc:144-148).  Resident inputs stay on the device that holds them. */
int plb_ransac_batch_multi(plb_problem *problems, size_t count, int n_gpus, int streams_per_gpu);

/* Batch form of estimate_{absolute_pose,relative_pose,fundamental,homography} (robust.h:45-46,68-70,112-113,133-134):
 * every problem takes what the single entry point takes — points in the pixel units of its cameras, RansacOptions,
 * BundleOptions, max_error — so distorted cameras, the tangent-Sampson estimator and the F / H normalisation batch too. */
typedef struct plb_estimate_problem {
    int32_t kind;             /* PLB_KIND_* */
    int32_t real_focal_check; /* fundamental only (RelativePoseOptions::real_focal_check) */
    int32_t tangent_sampson;  /* relative pose only (RelativePoseOptions::tangent_sampson) */
    int32_t reserved;
    uint64_t n;
    const double *a;          /* points2D (pnp) or x1: 2n doubles */
    const double *b;          /* points3D (pnp): 3n doubles; else x2: 2n doubles */
    plb_camera camera1;       /* pnp: the camera; relative pose: camera 1; ignored by fundamental / homography */
    plb_camera camera2;       /* relative pose: camera 2 */
    plb_ransac_opt ransac;
    plb_bundle_opt bundle;
    double max_error;         /* pixels (AbsolutePoseOptions / RelativePoseOptions / HomographyOptions::max_error) */
    double model[9];          /* in/out */
    char *inliers;            /* n bytes or NULL */
    plb_ransac_stats stats;   /* out */
    plb_counters counters;    /* out */
    int32_t status;           /* out */
    int32_t reserved2;
} plb_estimate_problem;
/* n_gpus: 0 = every device of the process, k > 0 = the first k, -1 = the calling thread's device (plb_set_device).
 * Each problem is checked by its single entry point's rules: an unknown kind, or a / b NULL with n > 0 -> PLB_ERR_ARG;
 * a camera the kind reads (camera1 for PnP, both for relative pose) outside the ten models -> PLB_ERR_NYI;
 * tangent_sampson with a non-empty refine_intrinsics selection in either camera -> PLB_ERR_NYI, as the batch returns no
 * relative-pose cameras. */
int plb_estimate_batch(plb_estimate_problem *problems, size_t count, int n_gpus, int streams_per_gpu);
/* plb_estimate_batch(problems, count, -1, streams) with the correspondences and masks in device memory, for callers whose
 * matches are already on the GPU.  Everything else (kinds, cameras, options, model, stats, counters, status, camera1)
 * is as in plb_estimate_batch; only where the data lives differs:
 *  - a, b: device (or managed) memory of the calling thread's device (plb_set_device), contiguous row-major [n,2] /
 *    [n,3] arrays of `dtype`, aligned to it.  With PLB_DTYPE_F32 they are `const float *` cast into the `const double *`
 *    fields.  They are only read: the engine works on its own fp64 copy, and fp32 -> fp64 is exact, so a float call gives
 *    the results of the double call on the widened values.
 *  - inliers: NULL or n bytes of device memory on the same device; receives 0 / 1 as the host call writes them.
 *  - stream: a cudaStream_t of that device (NULL = the legacy default stream).  No input is read before the work queued
 *    on `stream` ahead of the call has finished; when the call returns, every device write it made is complete.
 * Pointers are checked for a problem with n > 0: a / b / inliers that are not device memory of the current device
 * (pageable or page-locked host memory, another GPU), or a / b misaligned for the dtype -> PLB_ERR_ARG.
 * counters.h2d_bytes holds no correspondences and d2h_bytes no masks. */
enum { PLB_DTYPE_F64 = 0, PLB_DTYPE_F32 = 1 };
int plb_estimate_batch_device(plb_estimate_problem *problems, size_t count, int dtype, void *stream, int streams);

/* Batch form of the robust/bundle.h refiners above (bundle.cc:84-112,206-222,237-256,313-333,394-411), for callers that
 * refine many independent problems at once: every two-view geometry of a matching graph, every query of a localisation
 * run.  Each problem carries what its single entry point takes and receives what that call writes; the single entry
 * points are the one-problem case of this call.  Each problem's model, bundle_stats and camera parameters are bit for bit
 * what its single call returns on the same inputs, whatever else is in the batch and for any n_gpus / streams.
 *   refiner                          single entry point                           cameras read / written
 *   PLB_REFINER_BUNDLE               plb_bundle_adjust (weights ignored, as the reference drops them, bundle.cc:84-92)
 *   PLB_REFINER_BUNDLE_IMAGE         plb_bundle_adjust_image[_weighted]           camera1 / its refined parameters
 *   PLB_REFINER_RELPOSE              plb_refine_relpose[_weighted]
 *   PLB_REFINER_RELPOSE_CAMERAS      plb_refine_relpose_cameras[_weighted]        camera1, camera2 / none
 *   PLB_REFINER_RELPOSE_PAIR         plb_refine_relpose_pair[_weighted]           camera1, camera2 / their refined parameters
 *   PLB_REFINER_FUNDAMENTAL          plb_refine_fundamental[_weighted]
 *   PLB_REFINER_HOMOGRAPHY           plb_refine_homography[_weighted]
 * Cameras a refiner does not read are ignored, and parameters the single call leaves alone stay untouched.
 * Every problem is checked by its single entry point's rules: an unknown refiner, or a / b NULL with n > 0 ->
 * PLB_ERR_ARG; a camera the refiner reads outside the ten models -> PLB_ERR_NYI; PLB_REFINER_RELPOSE_CAMERAS with a
 * non-empty refine_intrinsics selection -> PLB_ERR_NYI. */
enum {
    PLB_REFINER_BUNDLE = 0,
    PLB_REFINER_BUNDLE_IMAGE = 1,
    PLB_REFINER_RELPOSE = 2,
    PLB_REFINER_RELPOSE_CAMERAS = 3,
    PLB_REFINER_RELPOSE_PAIR = 4,
    PLB_REFINER_FUNDAMENTAL = 5,
    PLB_REFINER_HOMOGRAPHY = 6
};
typedef struct plb_refine_problem {
    int32_t refiner;          /* PLB_REFINER_* */
    int32_t reserved;
    uint64_t n;
    const double *a;          /* x (2n doubles) or x1 (2n) */
    const double *b;          /* X (3n doubles) or x2 (2n) */
    const double *weights;    /* n per-residual weights, or NULL (uniform) */
    plb_camera camera1;       /* in; the refined parameters written back as the single call writes them */
    plb_camera camera2;
    plb_bundle_opt bundle;
    double model[9];          /* in/out: pose (7) or matrix (9, column-major) */
    double bundle_stats[3];   /* out: iterations, initial_cost, cost */
    int32_t status;           /* out */
    int32_t reserved2;
} plb_refine_problem;
/* n_gpus: 0 = every device of the process, k > 0 = the first k, -1 = the calling thread's device (plb_set_device);
 * streams_per_gpu groups of problems are in flight on each device. */
int plb_refine_batch(plb_refine_problem *problems, size_t count, int n_gpus, int streams_per_gpu);
/* plb_refine_batch(problems, count, -1, streams) with a, b and weights in device memory, as plb_estimate_batch_device
 * takes them: device (or managed) memory of the calling thread's device, contiguous arrays of `dtype` aligned to it
 * (PLB_DTYPE_F32: `const float *` cast into the `const double *` fields).  They are only read, after the work queued on
 * `stream` ahead of the call has finished; fp32 values are widened exactly, so a float call gives the results of the
 * double call on the widened values.  Models, stats and cameras come back in the host array.  A / b / weights of a
 * problem with n > 0 that are not device memory of the current device, or misaligned for the dtype -> PLB_ERR_ARG. */
int plb_refine_batch_device(plb_refine_problem *problems, size_t count, int dtype, void *stream, int streams);

/* Scores and inlier masks of given models (robust/utils.h:40-87), for callers that check matches against models they
 * already have: a pose prior, guided matching against verified F / H, E / F / H inlier counts on the same matches, or
 * hypotheses made outside the library.  One record per (problem, model), at the ransac_* level: points as plb_ransac_*
 * and plb_ransac_relpose_cameras take them, no normalisation, sq_threshold the squared threshold in their units (tangent
 * Sampson: pixels^2).
 *   kind (+ option)                      model       score / num_inliers                   inliers (get_inliers)
 *   PLB_KIND_PNP                         pose (7)    compute_msac_score, utils.cc:36-63    utils.cc:374-383
 *   PLB_KIND_RELPOSE                     pose        compute_sampson_msac_score :158-201   get_inliers :434-476
 *   PLB_KIND_RELPOSE + tangent_sampson   pose        compute_tangent_sampson_msac_score    get_tangent_sampson_inliers
 *     (x1 / x2 pixels of camera1 / camera2, unprojected as ransac.cc:155-168 does)  :269-298   :541-569
 *   PLB_KIND_FUNDAMENTAL (F or E)        3x3 (9)     compute_sampson_msac_score :204-239   get_inliers :479-513
 *   PLB_KIND_HOMOGRAPHY                  3x3         compute_homography_msac_score :300-329  get_homography_inliers :331-351
 * num_inliers and the mask are exactly the reference's; for PnP the count comes from the scorer and the mask from
 * get_inliers, whose formulas can disagree at the last bit, as in the reference.  A score is the fp64 sum of the device's
 * scorer: the same terms as the reference's in a fixed order, the outliers added as one product (n - count) * sq_threshold,
 * so it equals the reference's up to summation order and, bit for bit, the score the RANSAC path records for the same
 * model.  n = 0 gives score 0 and count 0; m = 0 writes nothing.  Camera1 / camera2 are read only with tangent_sampson. */
typedef struct plb_score_problem {
    int32_t kind;             /* PLB_KIND_* */
    int32_t tangent_sampson;  /* relative pose only */
    uint64_t n;
    const double *a;          /* x (pnp) or x1: 2n doubles */
    const double *b;          /* X (pnp): 3n doubles; else x2: 2n doubles */
    plb_camera camera1;
    plb_camera camera2;
    uint64_t m;               /* models */
    const double *models;     /* m x 7 (poses) or m x 9 (column-major matrices) doubles */
    double sq_threshold;
    double *scores;           /* out: m (required when m > 0) */
    int64_t *num_inliers;     /* out: m (required when m > 0) */
    char *inliers;            /* out: NULL, or m x n bytes 0 / 1, model-major */
    int32_t status;           /* out */
    int32_t reserved;
} plb_score_problem;
/* n_gpus: 0 = every device of the process, k > 0 = the first k, -1 = the calling thread's device (plb_set_device);
 * streams_per_gpu groups of problems are in flight on each device.  Every pointer is host memory.  Each problem's
 * outputs are the same bits whatever else is in the batch and for any n_gpus / streams.
 * Each problem is checked: an unknown kind, tangent_sampson on another kind, a / b NULL with n > 0, models / scores /
 * num_inliers NULL with m > 0, a non-finite sq_threshold, m >= 2^31, n > 2^26 or m * n overflowing -> PLB_ERR_ARG; a
 * camera (tangent_sampson) outside the ten models -> PLB_ERR_NYI. */
int plb_score_batch(plb_score_problem *problems, size_t count, int n_gpus, int streams_per_gpu);
/* plb_score_batch(problems, count, -1, streams) with a, b, models, scores, num_inliers and inliers in device (or managed)
 * memory of the calling thread's device: a / b contiguous arrays of `dtype` aligned to it (PLB_DTYPE_F32: `const float *`
 * cast into the `const double *` fields; widened exactly, so a float call gives the double call's results on the widened
 * values), models fp64.  Nothing sized by n or m crosses PCIe.  Inputs are read after the work queued on `stream` ahead of
 * the call; when the call returns, every device write it made is complete.  A pointer of a problem that is not device
 * memory of the current device or is misaligned (a / b: the dtype; models, scores, num_inliers: 8 bytes) ->
 * PLB_ERR_ARG. */
int plb_score_batch_device(plb_score_problem *problems, size_t count, int dtype, void *stream, int streams);

/* Hypotheses of caller-drawn minimal samples: the estimators' generate_models followed by score_model for every model,
 * for callers that draw their own samples (learned or guided sampling, RANSAC variants of their own) or study the
 * hypotheses of a scene.  At the ransac_* level, as plb_score_batch: no normalisation, sq_threshold squared in the points'
 * units (tangent Sampson: pixels^2).
 *   kind (+ option)                      k   M   solver and estimator
 *   PLB_KIND_PNP                         3   4   p3p on x.homogeneous().normalized(), X (estimators/absolute_pose.cc:46-58)
 *   PLB_KIND_RELPOSE                     5  40   relpose_5pt on the normalised homogeneous points (relative_pose.cc:48-60)
 *   PLB_KIND_RELPOSE + tangent_sampson   5  40   relpose_5pt on the bearings of camera1 / camera2 (relative_pose.cc:88-99)
 *   PLB_KIND_FUNDAMENTAL                 7   3   relpose_7pt; with real_focal_check the models failing calculate_RFC are
 *                                                erased, the rest keep their order (relative_pose.cc:384-403)
 *   PLB_KIND_HOMOGRAPHY                  4   1   homography_4pt with check_cheirality (homography.cc:36-52)
 * Sample j (row j of `samples`, k indices into [0, n), duplicates go to the solver as given) gives n_models[j] models in
 * the solver's order in slots [0, n_models[j]) of row j of `models` (M slots of 7 or 9 doubles: poses, or column-major
 * matrices), each with the fp64 score_model record in `scores` / `num_inliers` (fp64 whatever plb_set_mode says).  Slots
 * past n_models[j] are not written.  num_inliers is exactly the reference's count; a score equals, bit for bit, what
 * plb_score_batch returns for the same model; a model is, bit for bit, what the RANSAC path's solver kernels produce for
 * the sample.  None of the outputs depends on the rest of the batch, n_gpus, streams, the mode or the form of the call. */
typedef struct plb_generate_problem {
    int32_t kind;             /* PLB_KIND_* */
    int32_t tangent_sampson;  /* relative pose only: camera1 / camera2 read, a / b in their pixels */
    int32_t real_focal_check; /* fundamental only */
    int32_t reserved;
    uint64_t n;
    const double *a;          /* x (pnp) or x1: 2n doubles */
    const double *b;          /* X (pnp): 3n doubles; else x2: 2n doubles */
    plb_camera camera1;
    plb_camera camera2;
    uint64_t s;               /* samples */
    const int32_t *samples;   /* s x k indices into [0, n), row-major */
    double sq_threshold;
    int32_t *n_models;        /* out: s */
    double *models;           /* out: s x M x (7 | 9) */
    double *scores;           /* out: s x M */
    int64_t *num_inliers;     /* out: s x M */
    int32_t status;           /* out */
    int32_t reserved2;
} plb_generate_problem;
/* n_gpus: 0 = every device of the process, k > 0 = the first k, -1 = the calling thread's device (plb_set_device);
 * streams_per_gpu groups of problems are in flight on each device.  Every pointer is host memory.
 * Each problem is checked: an unknown kind, tangent_sampson on another kind than relative pose, real_focal_check on another
 * kind than fundamental, a / b NULL with n > 0, samples / n_models / models / scores / num_inliers NULL with s > 0, a
 * non-finite sq_threshold, s >= 2^31, s * M * (7 | 9) doubles overflowing, or n > 2^26 -> PLB_ERR_ARG; a camera
 * (tangent_sampson) outside the ten models -> PLB_ERR_NYI; then a sample index outside [0, n) -> PLB_ERR_ARG (every index
 * is checked on the host, before any device call).  s = 0 writes nothing. */
int plb_generate_batch(plb_generate_problem *problems, size_t count, int n_gpus, int streams_per_gpu);
/* plb_generate_batch(problems, count, -1, streams) with a, b, samples and every output in device (or managed) memory of the
 * calling thread's device: a / b contiguous arrays of `dtype` aligned to it (PLB_DTYPE_F32: `const float *` cast into the
 * `const double *` fields; widened exactly, so a float call gives the double call's results on the widened values),
 * samples, n_models aligned to 4 bytes, models, scores, num_inliers to 8.  Nothing sized by n or s crosses PCIe.  Inputs
 * are read after the work queued on `stream` ahead of the call; when the call returns, every device write it made is
 * complete.  A pointer that is not device memory of the current device or is misaligned -> PLB_ERR_ARG (step 8); the
 * sample indices are range-checked on the device (step 9). */
int plb_generate_batch_device(plb_generate_problem *problems, size_t count, int dtype, void *stream, int streams);

/* The Camera functions of misc/camera_models.h over many points of many cameras, for callers who undistort keypoints,
 * need normalised image coordinates or reprojections, or Jacobians for their own optimisers.  Per point:
 *   op                    jac and jac_params NULL                  either given
 *   PLB_CAMOP_PROJECT     Camera::project (camera_models.cc:149-161)  Camera::project_with_jac (:162-175)
 *   PLB_CAMOP_UNPROJECT   Camera::unproject to a bearing (:176-188)  Camera::unproject_with_jac (:190-203)
 *   PLB_CAMOP_UNPROJECT_2D the 2D unproject wrapper, hnormalized (camera_models.h:98-102)   (not allowed)
 * `out` receives the point the function of the row writes (the point of a *_with_jac call is not claimed to equal the
 * plain call's).  jac_params without jac is the reference's call with jac = nullptr.  Matrices are column-major, as
 * Eigen stores them: jac 2x3 (PROJECT) or 3x2 (UNPROJECT) per point, jac_params 2 x P or 3 x P, P the model's parameter
 * count (the NULL camera has P = 0 and writes no parameter Jacobian).  The 2D project wrapper, which normalises through
 * Eigen's unpinned summation order, is not offered.  None of the outputs depends on the rest of the batch, n_gpus,
 * streams, the mode or the form of the call. */
enum { PLB_CAMOP_PROJECT = 0, PLB_CAMOP_UNPROJECT = 1, PLB_CAMOP_UNPROJECT_2D = 2 };
typedef struct plb_camera_problem {
    int32_t op;               /* PLB_CAMOP_* */
    int32_t reserved;
    uint64_t n;
    plb_camera camera;
    const double *in;         /* PROJECT: n x 3 camera-frame points; UNPROJECT[_2D]: n x 2 pixels; row-major */
    double *out;              /* out: PROJECT n x 2 pixels; UNPROJECT n x 3 bearings; UNPROJECT_2D n x 2 */
    double *jac;              /* out: NULL, or n Jacobians w.r.t. the point, 2x3 (PROJECT) / 3x2 (UNPROJECT) */
    double *jac_params;       /* out: NULL, or n Jacobians w.r.t. the parameters, 2 x P / 3 x P */
    int32_t status;           /* out */
    int32_t reserved2;
} plb_camera_problem;
/* n_gpus: 0 = every device of the process, k > 0 = the first k, -1 = the calling thread's device (plb_set_device);
 * streams_per_gpu groups of problems are in flight on each device.  Every pointer is host memory.
 * Each problem is checked: an unknown op, in / out NULL with n > 0, jac or jac_params with PLB_CAMOP_UNPROJECT_2D, or
 * n x (the widest of its rows) doubles overflowing size_t bytes -> PLB_ERR_ARG; a camera outside the ten models ->
 * PLB_ERR_NYI (the reference's "NYI", camera_models.cc:157-158).  n = 0 writes nothing. */
int plb_camera_batch(plb_camera_problem *problems, size_t count, int n_gpus, int streams_per_gpu);
/* plb_camera_batch(problems, count, -1, streams) with in, out, jac and jac_params in device (or managed) memory of the
 * calling thread's device: `in` a contiguous array of `dtype` aligned to it (PLB_DTYPE_F32: `const float *` cast into
 * the `const double *` field; widened exactly, so a float call gives the double call's results on the widened values),
 * out / jac / jac_params fp64, 8-byte aligned.  Nothing sized by n crosses PCIe.  Inputs are read after the work queued
 * on `stream` ahead of the call; when the call returns, every device write it made is complete.  A pointer that is not
 * device memory of the current device or is misaligned -> PLB_ERR_ARG (step 8). */
int plb_camera_batch_device(plb_camera_problem *problems, size_t count, int dtype, void *stream, int streams);

/* Correspondences kept resident in HBM across calls (measurement of the device-resident throughput, and callers
 * that run several estimations on the same matches).  kind: PLB_KIND_*; returns a handle > 0 or an error < 0. */
int plb_resident_create(int kind, const double *a, const double *b, size_t n);
int plb_resident_free(int handle);

#ifdef __cplusplus
}
#endif
#endif /* POSELIB_B200_H */
