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
typedef struct plb_bundle_opt {
    uint64_t max_iterations;   /* 100 */
    int32_t loss_type;         /* PLB_LOSS_CAUCHY */
    int32_t reserved;
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

/* misc/camera_models.h:39-157 Camera, restricted to the six models on the path (others -> PLB_ERR_NYI, like the
 * reference's "NYI" throw, camera_models.cc:184-185).  Ids are the reference's CameraModelId values. */
enum {
    PLB_CAMERA_NULL = -1,
    PLB_CAMERA_SIMPLE_PINHOLE = 0, /* f, cx, cy */
    PLB_CAMERA_PINHOLE = 1,        /* fx, fy, cx, cy */
    PLB_CAMERA_SIMPLE_RADIAL = 2,  /* f, cx, cy, k */
    PLB_CAMERA_RADIAL = 3,         /* f, cx, cy, k1, k2 */
    PLB_CAMERA_OPENCV = 4          /* fx, fy, cx, cy, k1, k2, p1, p2 */
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
int plb_estimate_relative_pose(const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                               const plb_camera *camera2, const plb_ransac_opt *ransac,
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
 * Uniform weights.  bundle_stats_out (may be NULL): {iterations, initial_cost, cost}. ------------------------- */
int plb_bundle_adjust(const double *x_xy, const double *X_xyz, size_t n, double pose_inout[7],
                      const plb_bundle_opt *opt, double bundle_stats_out[3]);
int plb_refine_relpose(const double *x1_xy, const double *x2_xy, size_t n, double pose_inout[7],
                       const plb_bundle_opt *opt, double bundle_stats_out[3]);
/* bundle.h refine_relpose(x1, x2, ImagePair*, opt) with fixed intrinsics (bundle.cc:237-247): tangent Sampson refiner */
int plb_refine_relpose_cameras(const double *x1_px, const double *x2_px, size_t n, const plb_camera *camera1,
                               const plb_camera *camera2, double pose_inout[7], const plb_bundle_opt *opt,
                               double bundle_stats_out[3]);
int plb_refine_fundamental(const double *x1_xy, const double *x2_xy, size_t n, double F_inout[9],
                           const plb_bundle_opt *opt, double bundle_stats_out[3]);
int plb_refine_homography(const double *x1_xy, const double *x2_xy, size_t n, double H_inout[9],
                          const plb_bundle_opt *opt, double bundle_stats_out[3]);

/* ---- batch of independent problems (BASELINE config 5); sharded by the caller across GPUs ---------- */
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
 * groups of problems are in flight at once. */
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
/* n_gpus: 0 = every device of the process, k > 0 = the first k, -1 = the calling thread's device (plb_set_device). */
int plb_estimate_batch(plb_estimate_problem *problems, size_t count, int n_gpus, int streams_per_gpu);

/* Correspondences kept resident in HBM across calls (measurement of the device-resident throughput, and callers
 * that run several estimations on the same matches).  kind: PLB_KIND_*; returns a handle > 0 or an error < 0. */
int plb_resident_create(int kind, const double *a, const double *b, size_t n);
int plb_resident_free(int handle);

#ifdef __cplusplus
}
#endif
#endif /* POSELIB_B200_H */
