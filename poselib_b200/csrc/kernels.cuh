// poselib_b200 — device-side data layout + host-callable launchers (implemented in kernels.cu).
#pragma once
#include "camera.cuh"
#include <cuda_runtime.h>
#include <stdint.h>

namespace plb {

// KIND_RELPOSE_TS: relative pose scored / refined with the tangent Sampson error on unit bearings d1,d2 and the
// unprojection Jacobians M1,M2 of arbitrary camera models (CameraRelativePoseEstimator, ransac.cc:155-168).
enum Kind { KIND_PNP = 0, KIND_RELPOSE = 1, KIND_FUND = 2, KIND_HOMOG = 3, KIND_RELPOSE_TS = 4 };

// Correspondences of ONE problem, resident in HBM as structure-of-arrays fp64 (exactly the caller's doubles):
//   2D-2D kinds : p[0]=x1.x p[1]=x1.y p[2]=x2.x p[3]=x2.y                      (32 B / correspondence)
//   PnP         : p[0]=x.x  p[1]=x.y  p[2]=X.x  p[3]=X.y  p[4]=X.z             (40 B / correspondence)
//   RELPOSE_TS  : ts + j*n_pad, j = 0..2 d1 | 3..5 d2 | 6..11 M1 (3x2 row-major) | 12..17 M2  (144 B / correspondence)
// Lanes read consecutive k -> every warp load is one fully coalesced 256 B request per array.
// f[] is the fp32 copy of the same arrays used by the screening pass (16 B / 20 B per correspondence).
struct ProblemDev {
    const double *p[5];
    const float *f[5];
    int n;
    int kind;
    double sq_thr;  // max_error^2 in the units of the points
    int rfc;        // real focal check (fundamental)
    int n_pad;      // array stride of ts
    const double *ts;
    const float *cmax; // max |coordinate| of every SoA array (fp64 values rounded up): error bounds of the fp32 screening
    // Relpose / fundamental: the integer rows of k_screen's streaming test (screen_math.cuh, 16 B per correspondence, n_pad
    // rows, zero past n), built once per problem by launch_qrows.  Null: k_screen builds them from f[] itself.
    const uint4 *q;
    // The cameras k_lm evaluates, cam[0 .. kind_cam_count(kind)); CAMM_NULL for a problem whose jobs use no camera.
    // Only the polish problem of a task whose final bundle evaluates a camera has them: a copy of the task's problem
    // whose p[0 .. 2 * kind_cam_count(kind)) are the pixels in the units of these cameras (PnP: x.x x.y; RELPOSE_TS:
    // x1.x x1.y x2.x x2.y, stride n_pad; written by k_transpose).
    CamDev cam[2];
};

constexpr __host__ __device__ bool kind_is_relpose(int kind) { return kind == KIND_RELPOSE || kind == KIND_RELPOSE_TS; }
constexpr __host__ __device__ int kind_sample_size(int kind) { return kind == KIND_PNP ? 3 : kind_is_relpose(kind) ? 5 : kind == KIND_FUND ? 7 : 4; }
constexpr __host__ __device__ int kind_max_models(int kind) { return kind == KIND_PNP ? 4 : kind_is_relpose(kind) ? 40 : kind == KIND_FUND ? 3 : 1; }
constexpr __host__ __device__ int kind_model_size(int kind) { return (kind == KIND_PNP || kind_is_relpose(kind)) ? 7 : 9; }
constexpr int TS_ARRAYS = 18;

// One round of hypothesis generation over a GROUP of problems of the same kind.  Global sample index g in
// [0, n_total) belongs to the active problem a with g_off[a] <= g < g_off[a+1]; its ProblemDev is probs[active[a]].
struct RoundDesc {
    const ProblemDev *probs;
    const int *active;   // n_active problem indices
    const int *g_off;    // n_active + 1 offsets into the concatenated sample table
    int n_active;
    const uint32_t *samples; // n_total * K indices
    int n_total;
};

// Per-round output of the hypothesis kernels.  Every active problem a owns the slot segment
// [seg_base[a], seg_base[a] + seg_cap[a]) of models / model_prob / counts / scores and fills it from the front
// (prob_count[a] models); sample g owns slots [first_slot[g], first_slot[g] + n_models[g]) inside its problem's segment.
// Everything stays in HBM: the ordered scans of k_select / k_pass1 reduce it to the few records the host replays.
struct HypOut {
    int *n_models;
    int *first_slot;
    const int *seg_base; // n_active
    const int *seg_cap;  // n_active
    int *prob_count;     // n_active, zeroed before the round
    int max_seg_cap;
    int *overflow;       // set when a segment is full (the engine then redoes the round with worst-case capacity)
    uint32_t *counts;
    double *scores;
    double *models;
    int *model_prob;  // problem index of every model slot
    uint32_t *fcounts; // fast mode: fp32 screening records
    float *fscores;
    uint32_t *fborder; // fast mode: correspondences whose fp32 inlier decision is within the error bound of the test
    float *ferr;       // fast mode: bound of |score32 - score64|
    // relpose_5pt phase buffers (device), sized for the round's n_total samples:
    double *s5_blk;   // 105 x n_total, entry-major (blk[e * n_total + g]): A (39) | Nb (36) | sample bearings x1s,x2s (30)
    double *s5_park;  // 100 x n_total, entry-major: right-hand sides of the elimination, parked by k5_elim
    double *s5_cpoly; // 11 x n_total, coefficient-major (cpoly[c * n_total + g])
    double *s5_roots; // per sample 10 doubles
    int *s5_nroots;   // per sample
};

// ---- device-side control of a round (sampling, candidate selection, best-minimal reduction) -----------------------
// RandomSampler state of one problem (robust/sampling.h:49-83), kept in HBM across the rounds of a group.
struct SamplerDev {
    uint64_t state;        // splitmix64 state (sampling.h:73)
    uint64_t sample_k;     // PROSAC: samples drawn so far + 1 (sampling.cc:91)
    uint64_t max_prosac;   // RansacOptions::max_prosac_iterations
    const uint64_t *growth; // PROSAC growth function, n entries (sampling.cc:105-136), or null
    uint32_t subset_sz;    // PROSAC: current subset size
    uint32_t n, k;         // num_data, sample size
    uint32_t flags;        // bit 0: PROSAC, bit 1: growth[] strictly increasing from k-1 on (closed-form subset size)
};
// One active problem of a round.
struct RoundProb {
    int pidx;     // index into probs[] / sampler states / LO job templates
    int g0, B;    // its samples are g0 .. g0+B-1 of the round's sample table
    int seg_base, seg_cap; // its segment of the model list
    int reserved;
    double lb0;   // best_minimal_inlier_count at the start of the round (ransac_impl.h:99-104)
    double ub0;   // best_minimal_msac_score at the start of the round
};
// Per active problem, written by k_pass1 into mapped pinned host memory: what the host needs to replay score_models().
struct SelHeader {
    int n_models;  // models generated by the round's samples (incl. samples past the serial break point)
    int n_cand;    // fast mode: models the fp32 records could not rule out (rescored in fp64)
    int n_imp;     // models that improve the best-minimal state, in (sample, model) order
    int imp_base;  // first ImpRec of this problem
    int n_trig;    // samples with at least one improving model = LO jobs of this problem
    int trig_base; // first LmJobOut of this problem
};
struct ImpRec {
    int sample;      // sample index inside the round (0-based)
    uint32_t count;  // exact inlier count
    double score;    // exact MSAC score
    double model[9];
};
struct LoJobSrc {
    int pidx;  // LO job template (per problem)
    int slot;  // model slot in the round's model list
};
// round control words in device memory (ints)
enum { CTL_OVERFLOW = 2, CTL_IMP_TOTAL = 5, CTL_JOB_TOTAL = 6, CTL_FLAGS = 7, CTL_WORDS = 8 };
enum { FLAG_IMP_OVERFLOW = 1, FLAG_JOB_OVERFLOW = 2 };

struct SelectArgs {
    const RoundProb *rp;
    int na;
    int mode;                // 0: exact records (counts/scores) for every model; 1: fp32 screening records
    const int *n_models;     // per sample
    const int *first_slot;   // per sample
    const uint32_t *fcounts; // fast mode, per model slot: fp32 inlier count
    const float *fscores;    //   fp32 MSAC score
    const uint32_t *fborder; //   number of correspondences whose fp32 inlier decision is not certain
    const float *ferr;       //   bound of |score32 - score64|
    uint32_t *counts;        // exact records per model slot (mode 0: input; mode 1: filled by k_confirm for candidates)
    double *scores;
    int *prefix;             // out, per sample: inclusive prefix sum of n_models inside its problem
    int *cand_slot;          // out, per problem segment: candidate slots in (sample, model) order
    int *cand_sample;        // out, same layout: their sample index inside the round
    int *n_cand;             // out, per active problem
    int *n_models_tot;       // out, per active problem
};
struct Pass1Args {
    const RoundProb *rp;
    int na;
    int *cand_slot;          // in/out: compacted in place to the improving models
    int *cand_sample;
    const int *n_cand;
    const int *n_models_tot;
    const uint32_t *counts;
    const double *scores;
    const double *models;
    int msz;
    int *ctl;
    int imp_cap, job_cap;
    SelHeader *hdr;          // mapped pinned host memory
    ImpRec *imp;             // mapped pinned host memory
    LoJobSrc *job_src;       // device
};

// LM (local optimisation / final polish) job description — mirrors BundleOptions (types.h:60-95)
struct LmParams {
    int max_iterations;
    int loss_type;   // 0 trivial, 1 truncated, 2 huber, 3 cauchy
    double loss_scale;
    double gradient_tol, step_tol, relative_cost_tol, initial_lambda, min_lambda, max_lambda;
    int subset_mode; // 0: all points; 1: relpose LO subset (Sampson+cheirality inliers at subset_sq_thr of the start pose,
                     //    return untouched if <= 5, estimators/relative_pose.cc:70-76); 2: use given mask
    double subset_sq_thr;
    int score_after; // score the refined model with sq_thr of the problem (count, score)
};
struct LmJob {
    int pidx;               // index into probs[]
    int cam_refine;         // CAM_REFINE_* flags.  A job where some camera of its problem (ProblemDev::cam) has a non-empty
                            // cam_refine_idx(model, cam_refine) refines every such selection with the pose: KIND_PNP
                            // AbsolutePoseRefiner (optim/absolute.h:40-171), KIND_RELPOSE_TS CameraRelativePoseRefiner
                            // (relative.h:268-483)
    long long mask_off;     // offset into the mask buffer (subset_mode 2), else -1
    long long scratch_off;  // offset (ints) into idx_scratch for the active-point list (subset modes 1, 2)
    LmParams prm;
    const double *w;        // per-residual weights of the problem's n points, in point order (device), or null: uniform.
                            // Read only by the W instantiations of k_lm, which launch_lm runs when some job has them
};
struct LmJobOut {
    double model[9];
    double score;
    uint32_t count;
    int iterations;
    double cost, initial_cost;
};
// Pre-step of one problem: caller layout (AoS doubles, device copies) -> resident SoA arrays.
//   mode 0: plain transposition (points already calibrated / normalised)
//   mode 1: Camera::unproject to 2D of a (cam_a) and, for 2D-2D kinds, of b (cam_b)   (robust.cc:40-43,287-292)
//   mode 2: a*scale, b*scale -> unproject_with_jac -> the 18 RELPOSE_TS arrays (robust.cc:255-266,
//           estimators/relative_pose.h:80-81); s32 unused
// px (or null): the pixels of the polish problem (ProblemDev::cam), a*px_scale and, for 2D-2D kinds, b*px_scale, as
// SoA arrays of stride n_pad
struct TransposeDesc {
    const double *a, *b; // 2n and b_dim*n doubles
    double *s64;
    float *s32;
    float *cmax; // 5 floats, zeroed before the launch (or null): per-array max |coordinate| (atomicMax of the bit patterns)
    int n, n_pad, b_dim, mode;
    double scale;
    CamDev cam_a, cam_b;
    double *px;
    double px_scale;
    uint4 *q; // relpose / fundamental: n_pad integer rows of the streaming test (launch_qrows), or null
};
// normalize_points of one problem (robust/utils.cc:584-644, shared scale), in place on the uploaded AoS doubles.
struct NormDesc {
    double *a, *b;  // 2n doubles each
    double *out;    // 5 doubles (mapped pinned host memory): centroid1 (2), centroid2 (2), scale
    int n;
    int centroid;   // normalize_centroid
};
struct MaskDesc {
    int pidx;
    int reserved;
    long long mask_off;
    double model[9];
};
// Correspondences of one problem already in device memory (plb_estimate_batch_device, plb_refine_batch_device): the
// caller's contiguous AoS arrays, read only, gathered into the engine's own input buffer as fp64 (a, b, then w: the
// layout the host path uploads).
struct IngestDesc {
    const void *a, *b; // 2n and b_dim*n values: float (f32) or double
    const void *w;     // n per-residual weights of the same dtype, or null
    double *dst;       // (2 + b_dim + (w ? 1 : 0)) * n doubles
    int n, b_dim, f32;
};
// One final inlier mask for a caller's device buffer: n bytes 0 / 1 from the mask buffer at mask_off.
struct ScatterDesc {
    char *dst;
    long long mask_off;
    int n;
};

// Explicit models of one problem for k_score: m models (stride kind_model_size), records to counts[0..m) / scores[0..m),
// and with masks model i's decision on correspondence k to mask[i * mask_stride + k].  The descriptors of a launch are
// ordered by tile0, the first of their ceil(m / tm_max) tiles in the launch's tile list.
struct ScoreDesc {
    const double *models;
    long long *counts;
    double *scores;
    char *mask;
    long long mask_stride;
    long long tile0;
    long long m;
    int pidx;
    int reserved;
    uint32_t *counts32; // when counts is null: the counts as uint32 (the round's record layout)
};

// Caller-drawn sample indices of one problem (plb_generate_batch_device): `count` int32 indices at src, copied to the
// round's sample table at dst, or (the argument check) tested against [0, n).
struct TakeDesc {
    const int32_t *src;
    uint32_t *dst;
    long long count;
    int n;
    int reserved;
};
// Where the records of one active problem of a generate chunk go.  Direct (the device form): row j of the caller's arrays
// holds sample j's n_models[j] models, maxm slots per row.  Packed (the host form): every problem of the chunk shares
// one staging buffer, models packed problem after problem; n_models[j] and offsets[j] give sample j's count and first
// packed slot.
struct PutDesc {
    int *n_models;
    int *offsets;     // packed only
    double *models;
    double *scores;
    long long *counts;
};
// One camera problem of plb_camera_batch: n points of `cam` at `in` (T of the launch: 3 per point to project, 2 to
// unproject), outputs row-major at out, column-major matrices at jac / jac_params (either may be null).  It owns the
// tiles [tile0, tile0 + ceil(n / CAM_TILE)) of the launch, tile j its points j * CAM_TILE ..; descriptors are ordered by
// tile0.
struct CamOpDesc {
    CamDev cam;
    const void *in;
    double *out, *jac, *jac_params;
    long long n;
    long long tile0;
};
constexpr int CAM_TILE = 256;
enum { CAMOP_PROJECT = 0, CAMOP_UNPROJECT = 1, CAMOP_UNPROJECT_2D = 2 };

// ---- launchers (all asynchronous on `stream`) --------------------------------------------------------------
// normalize_points for n_desc problems (descriptors in device memory), one CTA each.
void launch_normalize(const NormDesc *descs_dev, int n_desc, cudaStream_t stream);
// AoS (caller layout) -> SoA fp64 + fp32 for n_desc problems (descriptors in device memory), camera pre-step fused.
// xcam: some camera of the descriptors is a fisheye or division model (the kernel's instantiation that evaluates them)
void launch_transpose(const TransposeDesc *descs_dev, int n_desc, int max_n_pad, bool xcam, cudaStream_t stream);
// The integer rows of the relpose / fundamental streaming test (TransposeDesc::q, where set) from the fp32 arrays and the
// coordinate maxima that launch_transpose left: after it on the same stream.
void launch_qrows(const TransposeDesc *descs_dev, int n_desc, int max_n_pad, cudaStream_t stream);
// Solve + score kernels of one round (kind = kind of every problem of the group); *out.overflow must be zeroed.
// mode 0: exact fp64 scoring of every model; mode 1: fp32 screening of every model (the candidates k_select lists are
// rescored exactly by launch_confirm).  fctx (mode 1): scratch of scr::CTX_FLOATS floats per model slot for the
// screening constants of the round's models.
void launch_hypotheses(int kind, const RoundDesc &R, const HypOut &out, int mode, int max_n_pad, float *fctx,
                       cudaStream_t stream, cudaEvent_t ev_between = nullptr);
// Exact fp64 scoring of explicit models: the n_tiles tiles of tm_max (score_tile_models(kind) or 1) models of the n_desc
// descriptors (device memory); mask: every descriptor has a mask, written in the same pass.
int score_tile_models(int kind);
void launch_score_models(int kind, bool mask, const ProblemDev *probs, const ScoreDesc *descs_dev, int n_desc,
                         long long n_tiles, int tm_max, cudaStream_t stream);
// The same over a device list of n_models models (stride kind_model_size) with their problem indices, records in the
// round's layout (uint32 counts), in one-model tiles.
void launch_score_models(int kind, const ProblemDev *probs, const double *models, const int *model_prob, int n_models,
                         uint32_t *counts, double *scores, cudaStream_t stream);
// LM refinement: one thread-block cluster per job.  models_in: n_jobs * 9 doubles.  refine_camera (KIND_PNP,
// KIND_RELPOSE_TS): every job refines camera parameters with the pose (LmJob::cam_refine) and writes its
// kind_cam_count(kind) cameras to cam_out[(j * kind_cam_count(kind) + i) * CAM_MAX_PARAMS ..].
constexpr __host__ __device__ int kind_cam_count(int kind) { return kind == KIND_RELPOSE_TS ? 2 : 1; }
// xcam: some camera of the jobs' problems (ProblemDev::cam) is a fisheye or division model.  weighted: some job has
// per-residual weights (LmJob::w); the jobs without them then run with uniform weights in the same launch.
void launch_lm(int kind, bool refine_camera, bool xcam, bool weighted, const ProblemDev *probs, const LmJob *jobs_dev,
               const double *models_in, int n_jobs, int max_n, const char *mask_base, int *idx_scratch,
               int scratch_stride, LmJobOut *out, double *cam_out, cudaStream_t stream);
// The cluster width a launch of one job over n correspondences takes with every SM to itself (lm_set_sm_share(100);
// PLB_LM_PER_CTA and PLB_LM_SM_PCT apply).  The width fixes a job's reduction order, so a job run at this width gives the
// bits of a lone call.
int lm_lone_width(int n);
// launch_lm with the cluster width fixed (lm_lone_width of every job) on a persistent grid of at most sm_count / csize
// clusters, for jobs with subset_mode 0 (no mask, no index scratch).
void launch_lm_width(int kind, bool refine_camera, bool xcam, bool weighted, const ProblemDev *probs,
                     const LmJob *jobs_dev, const double *models_in, int n_jobs, int csize, LmJobOut *out,
                     double *cam_out, cudaStream_t stream);
// LO jobs of a round, listed on the device by k_pass1: job j refines model slot job_src[j].slot of the round's model
// list (stride MSZ) with the template tmpl[job_src[j].pidx]; *n_jobs_dev jobs.  n_jobs_dev is &ctl[CTL_JOB_TOTAL] of the
// round's control words: when the round's CTL_FLAGS word is set no job runs and no job_src entry is read (k_pass1
// left entries unwritten; the round is redone).  A persistent grid of clusters walks the list; est_jobs (host
// estimate) only sizes the clusters / the grid.
void launch_lm_round(int kind, const ProblemDev *probs, const LmJob *tmpl, const LoJobSrc *job_src,
                     const double *models, const int *n_jobs_dev, int job_cap, int est_jobs, int max_n,
                     int *idx_scratch, int scratch_stride, LmJobOut *out, cudaStream_t stream);
int lm_round_max_clusters(int kind, int est_jobs, int max_n);
// Share of the SMs (percent) the LO clusters launched from this host thread may cover (50: batch groups, 100: a lone call).
void lm_set_sm_share(int pct);
// Device-side sampling of a round: one warp per active problem draws its B samples into samples[(g0+s)*K ..] from
// st_in[pidx] and leaves the advanced state in st_out[pidx] (robust/sampling.cc:46-61,85-103).
void launch_sample(const RoundProb *rp, int na, const SamplerDev *st_in, SamplerDev *st_out, uint32_t *samples,
                   cudaStream_t stream);
// Ordered scan over the round's models per problem: which models could improve the best-minimal state.
void launch_select(const SelectArgs &A, cudaStream_t stream);
// fast mode: exact fp64 rescoring of the candidates k_select listed.
void launch_confirm(int kind, const ProblemDev *probs, const SelectArgs &A, const double *models, cudaStream_t stream);
// Exact pass over the candidates: improving models, LO triggers, records for the host replay.
void launch_pass1(const Pass1Args &A, cudaStream_t stream);
// Final inlier masks (robust/utils.cc:331-351,374-383,434-513): one descriptor per mask, sq_thr from the problem.
void launch_inlier_masks(int kind, const ProblemDev *probs, const MaskDesc *descs_dev, int n_desc, int max_n,
                         char *mask_base, cudaStream_t stream);
// Inlier masks as bits (bit k & 31 of word k >> 5) for the device -> host copy; n_bytes is a multiple of 32.
void launch_pack_mask(const char *mask, uint32_t *bits, size_t n_bytes, cudaStream_t stream);
// Device-resident inputs -> fp64 AoS for n_desc problems (descriptors in device memory); max_vals: the largest
// (2 + b_dim + (w ? 1 : 0)) * n of the descriptors.
void launch_ingest(const IngestDesc *descs_dev, int n_desc, size_t max_vals, cudaStream_t stream);
// Final masks straight into the callers' device buffers for n_desc problems; max_n: the largest n of the descriptors.
void launch_scatter_masks(const char *mask, const ScatterDesc *descs_dev, int n_desc, int max_n, cudaStream_t stream);
// Caller-drawn samples for n_desc problems (descriptors in device memory); max_count: the largest count.  bad null: copy
// them into the round's sample table; bad non-null: copy nothing and set *bad to 1 when some index is outside [0, n).
void launch_take_samples(const TakeDesc *descs_dev, int n_desc, long long max_count, int *bad, cudaStream_t stream);
// The records of the round's samples (after launch_hypotheses in mode 0) into the layout of descs_dev[a] for active
// problem a: direct rows of maxm slots, or packed (see PutDesc).
void launch_put_hyps(const RoundDesc &R, const HypOut &out, const PutDesc *descs_dev, int msz, int maxm, bool packed,
                     cudaStream_t stream);
// The camera functions of `op` over the tiles of n_desc descriptors (device memory): jac: some descriptor has a jac or
// jac_params; f32: the inputs are float.
void launch_camera(int op, bool jac, bool f32, const CamOpDesc *descs_dev, int n_desc, long long n_tiles,
                   cudaStream_t stream);
// Batched direct solver calls (solvers/*.h surface): one thread per instance.  kind KIND_RELPOSE also needs the s5_*
// phase buffers of s5 for `count` instances (the other fields are unused).  Returns the number of kernels launched.
int launch_solver_batch(int kind, int variant, size_t count, const double *a, const double *b, double *out, int *n_out,
                        int flags, const HypOut &s5, cudaStream_t stream);
// relpose_8pt / essential_matrix_8pt (solvers/relpose_8pt.cc:52-95): count instances of n >= 8 unit bearing pairs each.
void launch_eightpt(size_t count, int n, const double *x1, const double *x2, int want_poses, double *E_out, double *poses_out,
                    int *n_out, cudaStream_t stream);

} // namespace plb
