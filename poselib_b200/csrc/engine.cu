// poselib_b200 — host engine + C-ABI (include/poselib_b200.h).
//
// The reference runs one serial loop per problem (robust/ransac_impl.h:157-201).  Its sample sequence is a pure
// function of (seed, N, sample size, PROSAC options) and neither scoring nor refinement touch the RNG, so the engine
//   1. generates the sample table for a whole round of iterations on the host (robust/sampling.cc restated below),
//   2. lets the GPU solve + score every sample of the round (one thread per minimal solve, kernels.cu),
//   3. finds, from the per-model (inlier count, MSAC score) records, every model that improves the best-minimal
//      state — that sub-sequence does not depend on LO results — and refines all of them in one batched LM launch,
//   4. replays score_models() (ransac_impl.h:106-154) in iteration order over those records, which reproduces the
//      serial trajectory exactly: LO triggers, stats, dynamic_max_iter and the break test see the same state as the
//      reference loop; samples evaluated past the serial break point are discarded.
// There is no CPU compute path: without a CUDA device every compute entry point fails with PLB_ERR_CUDA.
#include "../../include/poselib_b200.h"
#include "kernels.cuh"
#include "screen_math.cuh"

#include <sched.h>

#include <algorithm>
#include <atomic>
#include <cassert>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <map>
#include <memory>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <mutex>
#include <string>
#include <thread>
#include <tuple>
#include <vector>

namespace plb {

static thread_local std::string g_err;
static thread_local int g_device = 0;
// precision mode of the calling thread (plb_set_mode): 1 = fast (fp32 screening with rigorous error intervals + fp64
// confirmation; same results as 0 = exact, fp64 scoring of every model).  Batch workers inherit the caller's mode.
static int default_mode() {
    static const int m = [] {
        const char *e = std::getenv("PLB_MODE");
        return (e && std::atoi(e) == 0) ? 0 : 1;
    }();
    return m;
}
static thread_local int g_mode = -1; // -1: not set by this thread -> default_mode()
static int current_mode() { return g_mode < 0 ? default_mode() : g_mode; }

#define PLB_CUDA(expr)                                                                                              \
    do {                                                                                                            \
        cudaError_t e_ = (expr);                                                                                    \
        if (e_ != cudaSuccess) {                                                                                    \
            g_err = std::string(#expr) + ": " + cudaGetErrorString(e_);                                             \
            return PLB_ERR_CUDA;                                                                                    \
        }                                                                                                           \
    } while (0)

// ---- robust/sampling.{h,cc}: splitmix64 sampler, restated for the host side of the engine -------------------------
struct Sampler {
    size_t num_data, sample_sz;
    uint64_t state;
    bool use_prosac;
    size_t max_prosac_iterations, sample_k = 0, subset_sz = 0;
    std::vector<size_t> growth;
    Sampler(size_t N, size_t K, const plb_ransac_opt &o)
        : num_data(N), sample_sz(K), state(o.seed), use_prosac(o.progressive_sampling != 0),
          max_prosac_iterations(o.max_prosac_iterations) {
        if (use_prosac) init_prosac();
    }
    // sampling.cc:37-43 — the reference returns `int`; `% N` then sign-extends (sampling.cc:50)
    static inline int next_int(uint64_t &st) {
        st += 0x9e3779b97f4a7c15ULL;
        uint64_t z = st;
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
        return (int)(z ^ (z >> 31));
    }
    inline void draw(size_t k, size_t N, uint32_t *out) { // sampling.cc:46-61
        for (size_t i = 0; i < k; ++i) {
            for (;;) {
                const size_t v = (size_t)(int64_t)next_int(state) % N;
                bool dup = false;
                for (size_t j = 0; j < i; ++j) dup |= (out[j] == (uint32_t)v);
                if (!dup) {
                    out[i] = (uint32_t)v;
                    break;
                }
            }
        }
    }
    void init_prosac() { // sampling.cc:105-136
        growth.assign(std::max(num_data, sample_sz), 0);
        double T_n = (double)max_prosac_iterations;
        for (size_t i = 0; i < sample_sz; ++i) T_n *= static_cast<double>(sample_sz - i) / (num_data - i);
        for (size_t n = 0; n < sample_sz; ++n) growth[n] = 1;
        size_t T_np = 1;
        for (size_t n = sample_sz; n < num_data; ++n) {
            const double T_n_next = T_n * (n + 1.0) / (n + 1.0 - sample_sz);
            T_np += std::ceil(T_n_next - T_n);
            growth[n] = T_np;
            T_n = T_n_next;
        }
        sample_k = 1;
        subset_sz = sample_sz;
    }
    inline void next(uint32_t *out) { // sampling.cc:85-103
        if (use_prosac && sample_k < max_prosac_iterations) {
            draw(sample_sz - 1, subset_sz - 1, out);
            out[sample_sz - 1] = (uint32_t)(subset_sz - 1);
            sample_k++;
            if (sample_k < max_prosac_iterations && sample_k > growth[subset_sz - 1]) {
                if (++subset_sz > num_data) subset_sz = num_data;
            }
        } else {
            draw(sample_sz, num_data, out);
        }
    }
};

// ---- robust/ransac_impl.h:43-74 ----------------------------------------------------------------------------
static double all_inlier_sample_probability(size_t num_inliers, size_t num_data, size_t sample_sz) {
    if (sample_sz == 0) return 1.0;
    if (num_inliers < sample_sz || num_data < sample_sz) return 0.0;
    double p = 1.0;
    for (size_t i = 0; i < sample_sz; ++i) p *= static_cast<double>(num_inliers - i) / static_cast<double>(num_data - i);
    return p;
}
static size_t compute_dynamic_max_iter(size_t num_inliers, size_t num_data, size_t sample_sz, double log_prob_missing,
                                       double mult, size_t min_it, size_t max_it) {
    const double p = all_inlier_sample_probability(num_inliers, num_data, sample_sz);
    if (p >= 0.9999) return min_it;
    if (p <= 0.0001) return max_it;
    const size_t num_iters = static_cast<size_t>(std::ceil(log_prob_missing / std::log(1.0 - p) * mult));
    return std::max(min_it, std::min(max_it, num_iters));
}

// ---- device / pinned buffers with grow-only capacity ---------------------------------------------------------
template <typename T> struct DevBuf {
    T *p = nullptr;
    size_t cap = 0;
    int ensure(size_t n) {
        if (n <= cap) return PLB_OK;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        const size_t want = std::max<size_t>(n + n / 4, 64); // slack: fewer device-synchronising reallocations
        PLB_CUDA(cudaMalloc(&p, want * sizeof(T)));
        cap = want;
        return PLB_OK;
    }
    ~DevBuf() {
        if (p) cudaFree(p);
    }
};
template <typename T> struct PinBuf {
    T *p = nullptr;
    size_t cap = 0;
    int ensure(size_t n) {
        if (n <= cap) return PLB_OK;
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        const size_t want = std::max<size_t>(n + n / 4, 64);
        PLB_CUDA(cudaMallocHost(&p, want * sizeof(T)));
        cap = want;
        return PLB_OK;
    }
    ~PinBuf() {
        if (p) cudaFreeHost(p);
    }
};

// Pinned host memory mapped into the device address space: kernels write small result records straight to it.
template <typename T> struct MapBuf {
    T *p = nullptr;  // host pointer
    T *d = nullptr;  // device alias
    size_t cap = 0;
    int ensure(size_t n) {
        if (n <= cap) return PLB_OK;
        if (p) cudaFreeHost(p);
        p = d = nullptr;
        cap = 0;
        const size_t want = std::max<size_t>(n + n / 4, 64);
        PLB_CUDA(cudaHostAlloc((void **)&p, want * sizeof(T), cudaHostAllocMapped | cudaHostAllocPortable));
        PLB_CUDA(cudaHostGetDevicePointer((void **)&d, p, 0));
        cap = want;
        return PLB_OK;
    }
    ~MapBuf() {
        if (p) cudaFreeHost(p);
    }
};

struct Engine {
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr, ev4 = nullptr;
    cudaEvent_t ev_block = nullptr; // cudaEventBlockingSync: the waiting thread sleeps instead of spinning
    cudaEvent_t ev_in = nullptr;    // plb_estimate_batch_device: recorded in the caller's stream, waited on by every group
    bool ready = false;
    int device = -1;
    DevBuf<double> in, soa64, px64, models, lm_in, s5_blk, s5_park, s5_cpoly, s5_roots;
    DevBuf<int> s5_nroots;
    DevBuf<float> soa32, cmax;
    DevBuf<uint4> qrows; // relpose / fundamental: ProblemDev::q
    DevBuf<uint32_t> samples;
    DevBuf<int> work, subset, act, model_prob, prob_count;
    // round state that stays on the device: sampler states, per-sample / per-model records, candidate lists
    DevBuf<SamplerDev> smp;
    DevBuf<uint64_t> growth;
    DevBuf<RoundProb> rp;
    DevBuf<int> n_models, first_slot, prefix, cand_slot, cand_sample, n_cand, n_models_tot;
    DevBuf<uint32_t> counts, fcounts, fborder;
    DevBuf<double> scores;
    DevBuf<float> fscores, ferr, fctx;
    DevBuf<LmJob> lo_tmpl;
    DevBuf<LoJobSrc> job_src;
    PinBuf<SamplerDev> h_smp;
    PinBuf<uint64_t> h_growth;
    PinBuf<RoundProb> h_rp;
    PinBuf<LmJob> h_lo_tmpl;
    PinBuf<int> h_hypfix;
    DevBuf<char> mask;
    DevBuf<uint32_t> mask_bits;
    PinBuf<uint32_t> h_mask_bits;
    DevBuf<ProblemDev> probs;
    DevBuf<TransposeDesc> tdesc;
    DevBuf<NormDesc> ndesc;
    PinBuf<NormDesc> h_ndesc;
    MapBuf<double> h_norm;
    DevBuf<MaskDesc> mdesc;
    DevBuf<IngestDesc> idesc; // device-resident inputs (plb_estimate_batch_device, plb_refine_batch_device)
    PinBuf<IngestDesc> h_idesc;
    DevBuf<ScatterDesc> sdesc;
    PinBuf<ScatterDesc> h_sdesc;
    DevBuf<ScoreDesc> scdesc; // explicit models (initial models, plb_score_batch)
    PinBuf<ScoreDesc> h_scdesc;
    PinBuf<double> h_models;
    // caller-drawn samples (plb_generate_batch): the callers' sample tables (host form: staged here; device form: taken
    // by k_take_samples), the record descriptors, and the host form's packed records (device staging, per-sample count
    // and offset in mapped memory, the copy the host expands)
    PinBuf<uint32_t> h_samples;
    DevBuf<TakeDesc> tkdesc;
    PinBuf<TakeDesc> h_tkdesc;
    DevBuf<PutDesc> pdesc;
    PinBuf<PutDesc> h_pdesc;
    DevBuf<double> gen_stage;
    PinBuf<double> h_gen_stage;
    MapBuf<int> h_gen;
    // camera functions (plb_camera_batch): the descriptors and the host form's outputs (inputs go up through in / h_in)
    DevBuf<CamOpDesc> cdesc;
    PinBuf<CamOpDesc> h_cdesc;
    DevBuf<double> cam_res;
    PinBuf<double> h_cam_res;
    DevBuf<LmJob> jobs;
    PinBuf<double> h_in, h_lm_in;
    PinBuf<int> h_act, h_work;
    PinBuf<ProblemDev> h_probs;
    PinBuf<TransposeDesc> h_tdesc;
    PinBuf<MaskDesc> h_mdesc;
    PinBuf<LmJob> h_jobs;
    // result records written by the kernels directly into mapped pinned memory (no explicit D2H copies): per round and
    // problem one header, the models that improved the best-minimal state and the LO results
    MapBuf<double> h_scores;
    MapBuf<long long> h_counts;
    MapBuf<SelHeader> h_hdr;
    MapBuf<ImpRec> h_imp;
    MapBuf<LmJobOut> h_lm_out;
    MapBuf<double> h_cam_out; // CAM_MAX_PARAMS per LM job: the camera of a job that refines it
    uint64_t launches = 0;

    int init() {
        int dev = g_device;
        if (ready && device == dev) {
            // the current device is per host thread (worker threads start on device 0): always re-select ours
            PLB_CUDA(cudaSetDevice(dev));
            return PLB_OK;
        }
        int count = 0;
        cudaError_t e = cudaGetDeviceCount(&count);
        if (e != cudaSuccess || count == 0) {
            g_err = std::string("no usable CUDA device: ") + cudaGetErrorString(e);
            return PLB_ERR_CUDA;
        }
        if (dev >= count) {
            g_err = "device index out of range";
            return PLB_ERR_ARG;
        }
        PLB_CUDA(cudaSetDevice(dev));
        if (!stream) PLB_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        if (!ev0) PLB_CUDA(cudaEventCreate(&ev0));
        if (!ev1) PLB_CUDA(cudaEventCreate(&ev1));
        if (!ev2) PLB_CUDA(cudaEventCreate(&ev2));
        if (!ev3) PLB_CUDA(cudaEventCreate(&ev3));
        if (!ev4) PLB_CUDA(cudaEventCreate(&ev4));
        if (!ev_block) PLB_CUDA(cudaEventCreateWithFlags(&ev_block, cudaEventBlockingSync | cudaEventDisableTiming));
        if (!ev_in) PLB_CUDA(cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming));
        {
            int r = h_work.ensure(8);
            if (r) return r;
        }
        device = dev;
        ready = true;
        return PLB_OK;
    }
};
// Is this host pointer page-locked (cudaHostAlloc / cudaHostRegister / torch pin_memory)?  Then the engine copies from it
// directly instead of through its own pinned staging buffer.  Needs a current context (call after Engine::init()).
static bool host_pinned(const void *p) {
    if (!p) return false;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return at.type == cudaMemoryTypeHost;
}
// Is p device or managed memory of `device` (plb_estimate_batch_device)?  Pageable and page-locked host memory are not.
// Needs a current context.
static bool device_memory(const void *p, int device) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) && at.device == device;
}

// Batch workers of an oversubscribed process (more lock-step groups in flight than cores this process may use: several
// ranks sharing a host) wait for their round by sleeping on a blocking event; spinning threads would take the cores from
// the threads that have a round to replay.  Single calls and small batches spin (lowest latency).
static thread_local bool t_blocking_sync = false;
static std::mutex &upload_mutex(int device) {
    static std::mutex m[64];
    return m[(device >= 0 && device < 64) ? device : 0];
}
static thread_local bool t_batch_worker = false; // this thread runs one of several lock-step groups of a batch call

// One engine (stream, events, grow-only buffers) per host thread AND device: a thread that switches devices with
// plb_set_device gets a separate engine for each, so streams and buffers never cross devices.  Engines live as long as
// the process (buffers are reused across calls).
static thread_local std::map<int, Engine *> *g_engines = nullptr;
static Engine *engine() {
    if (!g_engines) g_engines = new std::map<int, Engine *>();
    Engine *&e = (*g_engines)[g_device];
    if (!e) e = new Engine();
    return e;
}

// Persistent worker threads of the batch entry points (created on first use, grown on demand).  Worker w of a dispatch
// always runs job w, so a repeated workload meets the same engine with the same group shapes (no reallocation after the
// first call).  Dispatches are serialised: concurrent callers of plb_ransac_batch queue up instead of sharing engines.
class WorkerPool {
  public:
    void run(int n, const std::function<void(int)> &fn) {
        std::lock_guard<std::mutex> dispatch(dispatch_mtx_);
        if (n <= 0) return;
        {
            std::unique_lock<std::mutex> lk(mtx_);
            while ((int)threads_.size() < n) {
                const int id = (int)threads_.size();
                threads_.emplace_back([this, id] { loop(id); });
            }
            fn_ = &fn;
            n_ = n;
            pending_ = n;
            ++epoch_;
        }
        cv_.notify_all();
        std::unique_lock<std::mutex> lk(mtx_);
        done_.wait(lk, [this] { return pending_ == 0; });
        fn_ = nullptr;
    }

  private:
    void loop(int id) {
        uint64_t seen = 0;
        for (;;) {
            const std::function<void(int)> *fn = nullptr;
            {
                std::unique_lock<std::mutex> lk(mtx_);
                cv_.wait(lk, [&] { return epoch_ != seen; });
                seen = epoch_;
                if (id < n_) fn = fn_;
            }
            if (fn) {
                (*fn)(id);
                std::unique_lock<std::mutex> lk(mtx_);
                if (--pending_ == 0) done_.notify_all();
            }
        }
    }
    std::mutex dispatch_mtx_, mtx_;
    std::condition_variable cv_, done_;
    std::vector<std::thread> threads_;
    const std::function<void(int)> *fn_ = nullptr;
    int n_ = 0, pending_ = 0;
    uint64_t epoch_ = 0;
};
static WorkerPool &worker_pool() {
    static WorkerPool *p = new WorkerPool(); // never destroyed: its threads outlive static destruction
    return *p;
}
// host cores this process may use: affinity mask, capped by the cgroup CPU quota (containers / shared hosts)
static int usable_cpus() {
    static const int cached = [] {
        int n = (int)std::thread::hardware_concurrency();
        cpu_set_t set;
        if (sched_getaffinity(0, sizeof(set), &set) == 0) n = CPU_COUNT(&set);
        if (FILE *f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {
            char q[64];
            long long period = 0;
            if (std::fscanf(f, "%63s %lld", q, &period) == 2 && std::strcmp(q, "max") != 0 && period > 0) {
                const long long quota = std::atoll(q);
                if (quota > 0) n = std::min<long long>(n, std::max<long long>(1, (quota + period - 1) / period));
            }
            std::fclose(f);
        }
        if (const char *e = std::getenv("PLB_HOST_THREADS")) n = std::max(1, std::atoi(e));
        return std::max(1, n);
    }();
    return cached;
}

// correspondences resident in HBM (plb_resident_create)
struct Resident {
    DevBuf<double> soa64;
    DevBuf<float> soa32, cmax;
    DevBuf<uint4> qrows; // relpose / fundamental: ProblemDev::q
    int n = 0, n_pad = 0, kind = 0, device = 0;
};
static std::mutex g_res_mtx;
static std::vector<std::shared_ptr<Resident>> g_resident; // handle = index + 1; calls in flight hold a reference

// LO bundle options of the estimators (estimators/absolute_pose.cc:60-69 etc.): TRUNCATED(max_error), 25 iterations
static LmParams lo_params(int kind, double max_error) {
    LmParams p;
    std::memset(&p, 0, sizeof(p));
    p.max_iterations = 25;
    p.loss_type = PLB_LOSS_TRUNCATED;
    p.loss_scale = max_error;
    p.gradient_tol = 1e-12;
    p.step_tol = 1e-8;
    p.relative_cost_tol = 1e-10;
    p.initial_lambda = 1e-3;
    p.min_lambda = 1e-10;
    p.max_lambda = 1e10;
    p.subset_mode = (kind == KIND_RELPOSE) ? 1 : 0;
    p.subset_sq_thr = 5 * (max_error * max_error); // estimators/relative_pose.cc:70
    p.score_after = 1;
    return p;
}
static LmParams bundle_params(const plb_bundle_opt &b) {
    LmParams p;
    std::memset(&p, 0, sizeof(p));
    p.max_iterations = (int)std::min<uint64_t>(b.max_iterations, 1u << 30);
    p.loss_type = b.loss_type;
    p.loss_scale = b.loss_scale;
    p.gradient_tol = b.gradient_tol;
    p.step_tol = b.step_tol;
    p.relative_cost_tol = b.relative_cost_tol;
    p.initial_lambda = b.initial_lambda;
    p.min_lambda = b.min_lambda;
    p.max_lambda = b.max_lambda;
    p.subset_mode = 2;
    p.score_after = 0;
    return p;
}

struct FinalPolish { // the post-RANSAC refinement of PoseLib/robust.cc (estimate_* entry points)
    bool enabled = false;
    plb_bundle_opt bundle;
    size_t min_inliers = 0; // run iff stats.num_inliers > min_inliers
    // The cameras the bundle evaluates, kind_cam_count(kind) of them, rescaled by `scale`; CAMM_NULL when it evaluates
    // none.  With a camera the bundle runs on the task's polish problem, whose pixels are the caller's times scale: pnp
    // robust.cc:103-123, relpose tangent Sampson with camera refinement :255-282.
    CamDev cam[2] = {{CAMM_NULL, 0, {0, 0, 0, 0, 0, 0, 0, 0}}, {CAMM_NULL, 0, {0, 0, 0, 0, 0, 0, 0, 0}}};
    double scale = 1.0;
    // Image* / ImagePair* forms: CAM_REFINE_* flags of the camera parameters refined with the pose (LmJob::cam_refine),
    // and cam_out[i] (or null) receives cam[i] after the polish, rescaled back by 1 / scale (robust.cc:103-123)
    int cam_refine = 0;
    plb_camera *cam_out[2] = {nullptr, nullptr};
    bool evaluates_camera() const { return cam[0].model != CAMM_NULL || cam[1].model != CAMM_NULL; }
};

// ---- small host-side 3x3 helpers for the estimate_* wrappers (column-major <-> row-major) ---------------------
struct HM3 {
    double m[3][3];
};
static HM3 hm_identity() {
    HM3 r;
    std::memset(&r, 0, sizeof(r));
    r.m[0][0] = r.m[1][1] = r.m[2][2] = 1;
    return r;
}
static HM3 hm_mul(const HM3 &A, const HM3 &B) {
    HM3 C;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C.m[i][j] = A.m[i][0] * B.m[0][j] + A.m[i][1] * B.m[1][j] + A.m[i][2] * B.m[2][j];
    return C;
}
static HM3 hm_T(const HM3 &A) {
    HM3 C;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C.m[i][j] = A.m[j][i];
    return C;
}
static HM3 hm_inv(const HM3 &M) {
    const double(*m)[3] = M.m;
    HM3 c;
    c.m[0][0] = m[1][1] * m[2][2] - m[1][2] * m[2][1];
    c.m[1][0] = m[1][2] * m[2][0] - m[1][0] * m[2][2];
    c.m[2][0] = m[1][0] * m[2][1] - m[1][1] * m[2][0];
    c.m[0][1] = m[0][2] * m[2][1] - m[0][1] * m[2][2];
    c.m[1][1] = m[0][0] * m[2][2] - m[0][2] * m[2][0];
    c.m[2][1] = m[0][1] * m[2][0] - m[0][0] * m[2][1];
    c.m[0][2] = m[0][1] * m[1][2] - m[0][2] * m[1][1];
    c.m[1][2] = m[0][2] * m[1][0] - m[0][0] * m[1][2];
    c.m[2][2] = m[0][0] * m[1][1] - m[0][1] * m[1][0];
    const double det = c.m[0][0] * m[0][0] + c.m[1][0] * m[0][1] + c.m[2][0] * m[0][2];
    const double id = 1.0 / det;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c.m[i][j] *= id;
    return c;
}
static double hm_norm(const HM3 &A) {
    double s = 0;
    for (int j = 0; j < 3; ++j)
        for (int i = 0; i < 3; ++i) s += A.m[i][j] * A.m[i][j];
    return std::sqrt(s);
}
static HM3 hm_from_cm(const double *p) {
    HM3 r;
    for (int k = 0; k < 9; ++k) r.m[k % 3][k / 3] = p[k];
    return r;
}
static void hm_to_cm(const HM3 &A, double *p) {
    for (int k = 0; k < 9; ++k) p[k] = A.m[k % 3][k / 3];
}

// T1, T2 of normalize_points (utils.cc:596-600,622-643) from its centroids and scale: translation by -centroid, then the
// first two rows scaled by 1 / scale
static void norm_transforms(const double *o, HM3 &T1, HM3 &T2) {
    T1 = hm_identity();
    T2 = hm_identity();
    T1.m[0][2] = -o[0];
    T1.m[1][2] = -o[1];
    T2.m[0][2] = -o[2];
    T2.m[1][2] = -o[3];
    const double scale = o[4];
    for (int r = 0; r < 2; ++r)
        for (int c = 0; c < 3; ++c) {
            T1.m[r][c] *= 1.0 / scale;
            T2.m[r][c] *= 1.0 / scale;
        }
}

// One LO-RANSAC problem handed to the group engine (points already calibrated / normalised).
struct Task {
    int kind = 0;
    const double *a = nullptr, *b = nullptr;
    size_t n = 0;
    plb_ransac_opt opt;
    double max_error = 0;
    int rfc = 0;
    double *model = nullptr;   // in/out: 7 or 9 doubles
    char *inliers = nullptr;
    plb_ransac_stats *stats_out = nullptr;
    plb_counters *cnt_out = nullptr;
    FinalPolish polish;
    std::shared_ptr<const Resident> res; // resident correspondences, held for the duration of the call
    // Written by commit_task once the whole call has passed its checks (estimate_* only): `skip`, nothing to run (too
    // few points), gets the default stats and counters; `reset_pose` resets the start pose to the identity (tangent
    // Sampson, ransac.cc:159-160, even when score_initial_model is set).
    bool skip = false, reset_pose = false;
    // normalize_points on the device before anything else (estimate_fundamental / estimate_homography, robust.cc:561,724):
    // 0 none, 1 scale only (real_focal_check keeps the principal point at the origin), 2 centroid + scale.  max_error and
    // the polish loss scale are then given in the units of the raw points and divided by the scale once it is known
    // (robust.cc:562-564,725-727); norm_out receives centroid1, centroid2, scale for the caller's un-normalisation.
    int norm_mode = 0;
    double norm_out[5] = {0, 0, 0, 0, 1};
    // camera pre-step fused into the layout kernel (TransposeDesc modes): 0 none, 1 unproject to 2D, 2 tangent Sampson
    int pre_mode = 0;
    double pre_scale = 1.0;
    CamDev cam_a{CAMM_NULL, 0, {0, 0, 0, 0, 0, 0, 0, 0}}, cam_b{CAMM_NULL, 0, {0, 0, 0, 0, 0, 0, 0, 0}};
    // plb_estimate_batch_device / plb_refine_batch_device: a, b, weights (float when f32) and inliers are device memory
    // of the group's device, read and written only after `ready` (recorded in the caller's stream) has completed
    bool dev_io = false, f32 = false;
    cudaEvent_t ready = nullptr;
    // A robust/bundle.h refiner call instead of LO-RANSAC (run_refine_group): one LM job over all n points with
    // polish.bundle, polish.cam_refine and the cameras polish.cam; the refined model goes to `model`, {iterations,
    // initial_cost, cost} to bstats (or nowhere), the refined parameters of camera i to polish.cam_out[i].
    bool refine = false;
    const void *weights = nullptr; // refine: n per-residual weights in point order (float when f32), or null: uniform
    double *bstats = nullptr;
    // Scoring given models instead of LO-RANSAC (run_score_group): m models (MSZ doubles each; device memory with
    // dev_io), threshold sq_thr; records to scores / counts, and with `inliers` m x n mask bytes, model-major.
    bool score = false;
    size_t m = 0;
    const double *models = nullptr;
    double sq_thr = 0;
    double *scores = nullptr;
    int64_t *counts = nullptr;
    // Hypotheses of caller-drawn samples instead of LO-RANSAC (run_generate_group): s samples of K indices (device memory
    // with dev_io), sample j's n_models[j] models with their records (threshold sq_thr) in row j of gen_models / scores /
    // counts, kind_max_models slots per row.
    bool generate = false;
    size_t s = 0;
    const int32_t *samples = nullptr;
    int32_t *n_models = nullptr;
    double *gen_models = nullptr;
    // Camera functions instead of LO-RANSAC (run_camera_group): op (CAMOP_*) of camera cam_a over the n points at `a`,
    // outputs to cam_out, and the Jacobians to cam_jac / cam_jac_params when they are given.
    bool camop = false;
    int cam_op = 0;
    double *cam_out = nullptr, *cam_jac = nullptr, *cam_jac_params = nullptr;
    // doubles per correspondence the group uploads: the caller layout, then the weight
    size_t in_per_point(int in_arr) const { return (size_t)in_arr + (weights ? 1 : 0); }
};

// per-problem serial state of the reference loop (ransac_impl.h:99-104,157-201)
struct PState {
    Task *t = nullptr;
    int n = 0, n_pad = 0, pidx = 0;
    bool enough = false, active = false;
    bool hyp_pending = false; // hypotheses of the last (broken) round still to be added from Engine::h_hypfix
    size_t it = 0, chunk = 1024;
    size_t best_minimal_inlier_count = 0;
    double best_minimal_msac_score = std::numeric_limits<double>::max();
    size_t dynamic_max_iter = 0;
    double log_prob_missing_model = 0;
    plb_ransac_stats stats;
    plb_counters cnt;
    double best_model[9];
    // per round
    size_t B = 0, g0 = 0;
    long long mask_off = 0;
    long long in_off = -1; // offset of this problem's uploaded AoS input in Engine::in (not resident)
    int polish_pidx = -1;
};

static void update_dynamic(PState &S, int K) { // ransac_impl.h:150-153
    S.stats.inlier_ratio = static_cast<double>(S.stats.num_inliers) / static_cast<double>(S.t->n);
    S.dynamic_max_iter = compute_dynamic_max_iter(S.stats.num_inliers, S.t->n, (size_t)K, S.log_prob_missing_model,
                                                  S.t->opt.dyn_num_trials_mult, S.t->opt.min_iterations,
                                                  S.t->opt.max_iterations);
}

// One LM job staged by the host: its start model (MSZ doubles) and its description.
struct LmTask {
    const double *model;
    LmJob job;
};
// Camera::get_param_refinement_idx of the camera and the refinement flags is non-empty
static bool refines_camera(const CamDev &c, int flags) {
    int idx[CAM_MAX_PARAMS];
    return cam_refine_idx(c.model, flags, idx) > 0;
}
static LmJob lm_job(int pidx, long long mask_off, const LmParams &prm) {
    LmJob J;
    J.pidx = pidx;
    J.cam_refine = 0;
    J.mask_off = mask_off;
    J.scratch_off = 0;
    J.prm = prm;
    J.w = nullptr;
    return J;
}

static bool profiling() {
    static const bool on = std::getenv("PLB_PROFILE") != nullptr;
    return on;
}

// A camera after the final polish: the (refined) parameters of the rescaled camera `c`, rescaled by 1 / scale into `out`
// (robust.cc:121-122; the round trip can change last bits even when nothing was refined).
static void polish_camera_out(CamDev c, double scale, const double *params, plb_camera *out) {
    for (int i = 0; i < CAM_MAX_PARAMS; ++i) c.p[i] = params[i];
    cam_rescale(c, 1.0 / scale);
    const int np = cam_num_params(out->model_id);
    for (int i = 0; i < np; ++i) out->params[i] = c.p[i];
}

// A group of problems of the same kind, run in lock-step rounds: one solve launch, one score launch and one LM launch
// per round for the WHOLE group.  The member functions are the phases of run_group, in the order it calls them.
struct Group {
    Engine &E;
    const int kind, K, MAXM, MSZ;
    // in_arr: doubles per correspondence in the caller layout; n_arr: SoA arrays resident per correspondence
    const int b_dim, in_arr, n_arr, NP;
    std::vector<PState> PS;
    cudaStream_t st = nullptr;
    // device layout of the group (upload)
    size_t in_doubles = 0, soa_elems = 0, mask_bytes = 0, px_elems = 0, q_rows = 0;
    int max_n = 0, max_n_pad = 0, n_up = 0, n_probdev = 0;
    // Round sizes.  A small group leaves the GPU mostly idle, so speculating further ahead costs little time while every
    // round saved is a whole launch chain of latency: the first round and the per-round cap grow as the group shrinks
    // (1 problem: 4096 doubling up to 65536 samples; >= 16 problems: 1024 doubling to 16384).  The first round stays
    // moderate on purpose: a loop that stops right after min_iterations (high inlier ratio) would otherwise pay for
    // thousands of speculative samples and their LO refits (measured: C4 single call 2.0 -> 3.3 ms with 16384).
    const size_t few, CHUNK_MAX, ROUND_MAX;
    static constexpr size_t S_TOT_MAX = 262144;
    // 0 exact, 1 fast (fp32 screen + fp64 confirmation of candidates); the tangent-Sampson kind has no fp32 copy
    const int mode;
    int cap_factor;
    bool big_caps = false;
    size_t gen_rows = 0; // generate(): samples of the largest chunk (the stride of E.h_gen's two per-sample arrays)
    int smp_cur = 0; // sampler states of the current round: E.smp[smp_cur * NP ..]; the advanced ones land in the other half
    std::vector<int> act; // active problems of the current round
    std::vector<uint8_t> first_round;
    // counters of the group
    uint64_t launches0 = 0, h2d = 0, d2h = 0;
    int n_rounds = 0;
    double lo_wait = 0.0;
    float gpu_ms_total = 0.f, gpu_ms_score = 0.f, gpu_ms_confirm = 0.f, gpu_ms_lo = 0.f;
    // host-side phase timer (PLB_PROFILE=1 prints one line per group to stderr)
    enum { PH_SETUP, PH_SAMPLE, PH_LAUNCH, PH_WAIT_HYP, PH_REPLAY, PH_FINAL, PH_N };
    double ph[PH_N] = {0};
    std::chrono::steady_clock::time_point ph_t = std::chrono::steady_clock::now();

    Group(int kind_, std::vector<Task *> &tasks)
        : E(*engine()), kind(kind_), K(kind_sample_size(kind_)), MAXM(kind_max_models(kind_)),
          MSZ(kind_model_size(kind_)), b_dim(kind_ == KIND_PNP ? 3 : 2), in_arr(2 + b_dim),
          n_arr(kind_ == KIND_RELPOSE_TS ? TS_ARRAYS : in_arr), NP((int)tasks.size()), PS(NP),
          few((size_t)std::max(1, std::min(NP, 16))), CHUNK_MAX(std::max<size_t>(16384, 65536 / few)),
          ROUND_MAX(std::max<size_t>(32768, 65536 / few)), mode(kind_ == KIND_RELPOSE_TS ? 0 : current_mode()),
          cap_factor(kind_is_relpose(kind_) ? 8 : MAXM), first_round(NP, 1) {
        for (int i = 0; i < NP; ++i) {
            PState &S = PS[i];
            S.t = tasks[i];
            S.pidx = i;
            S.n = (int)S.t->n;
            S.n_pad = (S.n + 31) & ~31;
        }
    }

    int init() {
        int rc = E.init();
        st = E.stream;
        launches0 = E.launches;
        return rc;
    }
    int sync(double *acc = nullptr) {
        auto t0 = std::chrono::steady_clock::now();
        if (t_blocking_sync) { // more waiting threads than cores: sleep on an event instead of spinning on the stream
            PLB_CUDA(cudaEventRecord(E.ev_block, st));
            PLB_CUDA(cudaEventSynchronize(E.ev_block));
        } else {
            PLB_CUDA(cudaStreamSynchronize(st));
        }
        if (acc) *acc += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        return PLB_OK;
    }
    void mark(int which) {
        if (!profiling()) return;
        const auto now = std::chrono::steady_clock::now();
        ph[which] += std::chrono::duration<double>(now - ph_t).count();
        ph_t = now;
    }

    // ---- state of the serial loop before its first iteration (ransac_impl.h:157-176) --------------------------------
    int init_states() {
        for (PState &S : PS) {
            Task &t = *S.t;
            std::memset(&S.cnt, 0, sizeof(S.cnt));
            S.stats.refinements = S.stats.iterations = S.stats.num_inliers = 0;
            S.stats.inlier_ratio = 0;
            S.stats.model_score = std::numeric_limits<double>::max();
            if (!t.opt.score_initial_model) { // ransac.cc:47-50 etc.: identity unless an initial model is scored
                std::fill(t.model, t.model + MSZ, 0.0);
                if (MSZ == 7) t.model[0] = 1.0;
                else t.model[0] = t.model[4] = t.model[8] = 1.0;
            }
            std::fill(S.best_model, S.best_model + 9, 0.0);
            std::copy(t.model, t.model + MSZ, S.best_model);
            if (t.n > (size_t)(1u << 26)) {
                g_err = "too many correspondences";
                return PLB_ERR_ARG;
            }
            S.enough = t.n >= (size_t)K; // ransac_impl.h:161-163
            S.dynamic_max_iter = t.opt.max_iterations;
            S.log_prob_missing_model = std::log(1.0 - t.opt.success_prob);
        }
        return PLB_OK;
    }

    // ---- device layout of the group: SoA arrays of every non-resident problem, masks, ProblemDev table -------------
    // Stages the caller's arrays and issues their host -> device copies (device-resident arrays: k_ingest); the layout
    // kernel runs in transpose().
    int upload() {
        int rc, n_polish = 0, n_ingest = 0;
        size_t host_doubles = 0, max_ingest = 0; // inputs staged on the host / gathered on the device (k_ingest)
        const int nc = kind_cam_count(kind);
        for (PState &S : PS) {
            if (S.n == 0) continue;
            if (!S.t->res) {
                const size_t vals = S.t->in_per_point(in_arr) * S.n;
                if (S.t->dev_io) {
                    ++n_ingest;
                    max_ingest = std::max(max_ingest, vals);
                } else {
                    host_doubles += vals;
                }
                in_doubles += vals;
                soa_elems += (size_t)n_arr * S.n_pad;
                if (kind == KIND_RELPOSE || kind == KIND_FUND) q_rows += (size_t)S.n_pad;
                ++n_up;
            }
            S.mask_off = (long long)mask_bytes;
            mask_bytes += (size_t)S.n_pad;
            max_n = std::max(max_n, S.n);
            max_n_pad = std::max(max_n_pad, S.n_pad);
            if (S.t->polish.evaluates_camera()) {
                px_elems += 2 * (size_t)nc * S.n_pad;
                ++n_polish;
            }
        }
        n_probdev = NP + n_polish;
        // the staging buffer mirrors E.in's offsets; a group of device-resident inputs needs none
        if ((rc = E.h_in.ensure(host_doubles ? in_doubles : 0)) || (rc = E.in.ensure(in_doubles)) || (rc = E.soa64.ensure(soa_elems)) ||
            (rc = E.soa32.ensure(soa_elems)) || (rc = E.qrows.ensure(q_rows)) || (rc = E.cmax.ensure(5 * (size_t)NP)) || (rc = E.px64.ensure(px_elems)) || (rc = E.mask.ensure(mask_bytes)) ||
            (rc = E.mask_bits.ensure(mask_bytes / 32 + 1)) || (rc = E.h_mask_bits.ensure(mask_bytes / 32 + 1)) ||
            (rc = E.work.ensure(8)) || (rc = E.probs.ensure(n_probdev)) ||
            (rc = E.h_probs.ensure(n_probdev)) || (rc = E.tdesc.ensure(std::max(n_up, 1))) ||
            (rc = E.h_tdesc.ensure(std::max(n_up, 1))) ||
            (n_ingest && ((rc = E.idesc.ensure(n_ingest)) || (rc = E.h_idesc.ensure(n_ingest)))))
            return rc;
        struct DirectCopy {
            double *dst;
            const double *src;
            size_t bytes;
        };
        std::vector<DirectCopy> direct; // page-locked caller arrays: DMA straight from them (issued below, in one turn)
        size_t in_off = 0, soa_off = 0, px_off = 0, q_off = 0;
        std::vector<std::pair<size_t, size_t>> staged; // (offset, doubles) of the inputs that went through the staging buffer
        int iu = 0, ipol = 0, ii = 0;
        cudaEvent_t ready = nullptr; // the one event of the device call the group's tasks come from
        for (int i = 0; i < NP; ++i) {
            PState &S = PS[i];
            ProblemDev &P = E.h_probs.p[i];
            std::memset(&P, 0, sizeof(P));
            P.cam[0].model = P.cam[1].model = CAMM_NULL;
            P.n = S.n;
            P.kind = kind;
            P.sq_thr = (S.t->score || S.t->generate) ? S.t->sq_thr : S.t->max_error * S.t->max_error;
            P.rfc = S.t->rfc;
            P.n_pad = S.n_pad;
            if (S.n == 0) continue;
            P.cmax = E.cmax.p + 5 * (size_t)i;
            if (S.t->res) {
                for (int c = 0; c < n_arr; ++c) {
                    P.p[c] = S.t->res->soa64.p + (size_t)c * S.n_pad;
                    P.f[c] = S.t->res->soa32.p + (size_t)c * S.n_pad;
                }
                P.cmax = S.t->res->cmax.p;
                P.q = S.t->res->qrows.p;
                assert(!S.t->polish.evaluates_camera()); // plb_resident_create takes no camera
            } else {
                S.in_off = (long long)in_off;
                const size_t nw = S.t->weights ? (size_t)S.n : 0; // the weights follow b
                if (S.t->dev_io) { // gathered on the device by k_ingest (below): nothing crosses PCIe
                    IngestDesc &I = E.h_idesc.p[ii++];
                    I.a = S.t->a;
                    I.b = S.t->b;
                    I.w = S.t->weights;
                    I.dst = E.in.p + in_off;
                    I.n = S.n;
                    I.b_dim = b_dim;
                    I.f32 = S.t->f32 ? 1 : 0;
                    ready = S.t->ready;
                } else if (host_pinned(S.t->a) && host_pinned(S.t->b) && (!nw || host_pinned(S.t->weights))) {
                    // the caller's arrays are page-locked: DMA straight from them, no staging copy on the host
                    direct.push_back({E.in.p + in_off, S.t->a, sizeof(double) * 2 * S.n});
                    direct.push_back({E.in.p + in_off + 2 * (size_t)S.n, S.t->b, sizeof(double) * (size_t)b_dim * S.n});
                    if (nw) direct.push_back({E.in.p + in_off + (size_t)in_arr * S.n, (const double *)S.t->weights, sizeof(double) * nw});
                    h2d += sizeof(double) * ((size_t)in_arr * S.n + nw);
                } else {
                    staged.emplace_back(in_off, (size_t)in_arr * S.n + nw);
                    double *ha = E.h_in.p + in_off, *hb = ha + 2 * (size_t)S.n;
                    std::memcpy(ha, S.t->a, sizeof(double) * 2 * S.n);
                    std::memcpy(hb, S.t->b, sizeof(double) * (size_t)b_dim * S.n);
                    if (nw) std::memcpy(hb + (size_t)b_dim * S.n, S.t->weights, sizeof(double) * nw);
                }
                TransposeDesc &D = E.h_tdesc.p[iu++];
                D.a = E.in.p + in_off;
                D.b = D.a + 2 * (size_t)S.n;
                D.s64 = E.soa64.p + soa_off;
                D.s32 = E.soa32.p + soa_off;
                D.cmax = E.cmax.p + 5 * (size_t)i;
                D.n = S.n;
                D.n_pad = S.n_pad;
                D.b_dim = b_dim;
                D.mode = (kind == KIND_RELPOSE_TS) ? 2 : S.t->pre_mode;
                D.scale = S.t->pre_scale;
                D.cam_a = S.t->cam_a;
                D.cam_b = S.t->cam_b;
                D.q = nullptr;
                if (kind == KIND_RELPOSE || kind == KIND_FUND) {
                    D.q = E.qrows.p + q_off;
                    P.q = D.q;
                    q_off += (size_t)S.n_pad;
                }
                if (kind == KIND_RELPOSE_TS) {
                    P.ts = D.s64;
                } else {
                    for (int c = 0; c < n_arr; ++c) {
                        P.p[c] = D.s64 + (size_t)c * S.n_pad;
                        P.f[c] = D.s32 + (size_t)c * S.n_pad;
                    }
                }
                const FinalPolish &fp = S.t->polish;
                D.px = fp.evaluates_camera() ? E.px64.p + px_off : nullptr;
                D.px_scale = fp.scale;
                if (D.px) { // the polish problem: this one with the polish cameras and their pixels
                    S.polish_pidx = NP + ipol++;
                    ProblemDev &PP = E.h_probs.p[S.polish_pidx];
                    PP = P;
                    for (int c = 0; c < 2 * nc; ++c) PP.p[c] = D.px + (size_t)c * S.n_pad;
                    for (int c = 0; c < nc; ++c) PP.cam[c] = fp.cam[c];
                    px_off += 2 * (size_t)nc * S.n_pad;
                }
                in_off += (size_t)in_arr * S.n + nw;
                soa_off += (size_t)n_arr * S.n_pad;
            }
        }
        // The lock-step groups of a batch call start together; left alone, their host->device copies interleave on the
        // one copy engine and every group waits for (nearly) the whole batch to cross PCIe before its first kernel.
        // Issued group by group (the host-side staging above stays parallel), the first group computes while the others'
        // inputs are still in flight.
        std::unique_lock<std::mutex> upload_turn(upload_mutex(E.device), std::defer_lock);
        if (t_batch_worker) upload_turn.lock();
        for (const DirectCopy &c : direct) PLB_CUDA(cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyHostToDevice, st));
        // staged (pageable) inputs: contiguous runs of the pinned staging buffer go up in one copy each
        for (size_t i = 0; i < staged.size();) {
            size_t j = i, off = staged[i].first, len = 0;
            while (j < staged.size() && staged[j].first == off + len) len += staged[j++].second;
            PLB_CUDA(cudaMemcpyAsync(E.in.p + off, E.h_in.p + off, sizeof(double) * len, cudaMemcpyHostToDevice, st));
            h2d += sizeof(double) * len;
            i = j;
        }
        if (n_ingest) {
            PLB_CUDA(cudaMemcpyAsync(E.idesc.p, E.h_idesc.p, sizeof(IngestDesc) * n_ingest, cudaMemcpyHostToDevice, st));
            // the caller's arrays are read after the work it queued on its stream before the call
            PLB_CUDA(cudaStreamWaitEvent(st, ready, 0));
            launch_ingest(E.idesc.p, n_ingest, max_ingest, st);
            E.launches++;
        }
        return PLB_OK;
    }

    // ---- normalize_points on the device (robust/utils.cc:584-644), then the thresholds that depend on its scale ------
    int normalize() {
        std::vector<int> who;
        for (int i = 0; i < NP; ++i)
            if (PS[i].t->norm_mode != 0 && PS[i].in_off >= 0 && PS[i].n > 0) who.push_back(i);
        const int nn = (int)who.size();
        if (!nn) return PLB_OK;
        int rc;
        if ((rc = E.ndesc.ensure(nn)) || (rc = E.h_ndesc.ensure(nn)) || (rc = E.h_norm.ensure(5 * (size_t)nn))) return rc;
        for (int j = 0; j < nn; ++j) {
            const PState &S = PS[who[j]];
            NormDesc &D = E.h_ndesc.p[j];
            D.a = E.in.p + S.in_off;
            D.b = D.a + 2 * (size_t)S.n;
            D.out = E.h_norm.d + 5 * (size_t)j;
            D.n = S.n;
            D.centroid = S.t->norm_mode == 2 ? 1 : 0;
        }
        PLB_CUDA(cudaMemcpyAsync(E.ndesc.p, E.h_ndesc.p, sizeof(NormDesc) * nn, cudaMemcpyHostToDevice, st));
        launch_normalize(E.ndesc.p, nn, st);
        E.launches++;
        if ((rc = sync())) return rc;
        d2h += sizeof(double) * 5 * (size_t)nn;
        for (int j = 0; j < nn; ++j) {
            Task &t = *PS[who[j]].t;
            std::copy(E.h_norm.p + 5 * (size_t)j, E.h_norm.p + 5 * (size_t)j + 5, t.norm_out);
            const double scale = t.norm_out[4];
            t.max_error = t.max_error / scale;                                 // robust.cc:562,725
            t.polish.bundle.loss_scale = t.polish.bundle.loss_scale / scale; // :563,726
            E.h_probs.p[who[j]].sq_thr = t.max_error * t.max_error;
            if (t.opt.score_initial_model) { // robust.cc:566-569 / 729-732: the start model in normalised coordinates
                HM3 T1, T2;
                norm_transforms(t.norm_out, T1, T2);
                HM3 M = (kind == KIND_FUND) ? hm_mul(hm_mul(hm_inv(hm_T(T2)), hm_from_cm(t.model)), hm_inv(T1))
                                            : hm_mul(hm_mul(T2, hm_from_cm(t.model)), hm_inv(T1));
                const double nm = hm_norm(M);
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 3; ++c) M.m[r][c] /= nm;
                hm_to_cm(M, t.model);
                std::copy(t.model, t.model + 9, PS[who[j]].best_model);
            }
        }
        return PLB_OK;
    }

    // ---- ProblemDev table (final thresholds) and the layout kernel: caller AoS -> resident SoA ------------------------
    int transpose() {
        PLB_CUDA(cudaMemcpyAsync(E.probs.p, E.h_probs.p, sizeof(ProblemDev) * n_probdev, cudaMemcpyHostToDevice, st));
        if (n_up) {
            PLB_CUDA(cudaMemsetAsync(E.cmax.p, 0, sizeof(float) * 5 * (size_t)NP, st));
            // Problems with a fisheye or division camera go to the layout kernel's instantiation that evaluates them, the
            // others to the one without: each problem is laid out by the instantiation its lone call uses.
            auto xcam = [](const TransposeDesc &D) { return cam_is_x(D.cam_a.model) || cam_is_x(D.cam_b.model); };
            const int n_plain = (int)(std::stable_partition(E.h_tdesc.p, E.h_tdesc.p + n_up, [&](const TransposeDesc &D) { return !xcam(D); }) -
                                      E.h_tdesc.p);
            PLB_CUDA(cudaMemcpyAsync(E.tdesc.p, E.h_tdesc.p, sizeof(TransposeDesc) * n_up, cudaMemcpyHostToDevice, st));
            for (int x = 0; x < 2; ++x) {
                const int d0 = x ? n_plain : 0, nd = x ? n_up - n_plain : n_plain;
                if (nd == 0) continue;
                launch_transpose(E.tdesc.p + d0, nd, max_n_pad, x == 1, st);
                E.launches++;
            }
            if (kind == KIND_RELPOSE || kind == KIND_FUND) {
                launch_qrows(E.tdesc.p, n_up, max_n_pad, st);
                E.launches++;
            }
        }
        return PLB_OK;
    }

    // Stages a batch of LM jobs (job j: start model batch[j].model, results in E.h_lm_out[j]) and launches one k_lm per
    // refiner: the jobs that refine the camera come last and write their kind_cam_count(kind) cameras to row j of
    // E.h_cam_out.  The caller synchronises.
    // A job refines camera parameters when the flags select some of a camera of its problem (ProblemDev::cam)
    bool refines_camera(const LmJob &J) const {
        for (int i = 0; i < kind_cam_count(kind); ++i)
            if (plb::refines_camera(E.h_probs.p[J.pidx].cam[i], J.cam_refine)) return true;
        return false;
    }
    // A job evaluates a fisheye or division camera
    bool uses_x_camera(const LmJob &J) const {
        for (int i = 0; i < kind_cam_count(kind); ++i)
            if (cam_is_x(E.h_probs.p[J.pidx].cam[i].model)) return true;
        return false;
    }
    // Stages the jobs and their start models and sizes the result rows.  scratch: the jobs select their points
    // (subset modes 1, 2) and need a max_n_pad slice of E.subset each.
    int lm_stage(const std::vector<LmTask> &batch, bool scratch) {
        const int nj = (int)batch.size(), nc = kind_cam_count(kind);
        const bool any_cam = std::any_of(batch.begin(), batch.end(), [&](const LmTask &t) { return refines_camera(t.job); });
        int rc;
        if ((rc = E.h_lm_in.ensure(9 * (size_t)nj)) || (rc = E.h_jobs.ensure(nj)) || (rc = E.jobs.ensure(nj)) ||
            (rc = E.lm_in.ensure(9 * (size_t)nj)) || (rc = E.h_lm_out.ensure(nj)) ||
            (scratch && (rc = E.subset.ensure((size_t)nj * max_n_pad))) ||
            (any_cam && (rc = E.h_cam_out.ensure((size_t)nj * nc * CAM_MAX_PARAMS))))
            return rc;
        for (int j = 0; j < nj; ++j) {
            double *row = E.h_lm_in.p + 9 * (size_t)j;
            std::fill(row, row + 9, 0.0);
            std::copy(batch[j].model, batch[j].model + MSZ, row);
            E.h_jobs.p[j] = batch[j].job;
            E.h_jobs.p[j].scratch_off = scratch ? (long long)j * max_n_pad : 0;
        }
        PLB_CUDA(cudaMemcpyAsync(E.jobs.p, E.h_jobs.p, sizeof(LmJob) * nj, cudaMemcpyHostToDevice, st));
        PLB_CUDA(cudaMemcpyAsync(E.lm_in.p, E.h_lm_in.p, sizeof(double) * 9 * nj, cudaMemcpyHostToDevice, st));
        h2d += (sizeof(LmJob) + sizeof(double) * 9) * nj;
        return PLB_OK;
    }
    int lm_batch(const std::vector<LmTask> &batch) {
        const int nj = (int)batch.size(), nc = kind_cam_count(kind);
        const int n_fixed = (int)(std::partition_point(batch.begin(), batch.end(),
                                                       [&](const LmTask &t) { return !refines_camera(t.job); }) -
                                  batch.begin());
        int rc;
        if ((rc = lm_stage(batch, true))) return rc;
        for (int cam = 0; cam < 2; ++cam) {
            const int j0 = cam ? n_fixed : 0, n = cam ? nj - n_fixed : n_fixed;
            if (n == 0) continue;
            bool xcam = false, weighted = false;
            for (int j = j0; j < j0 + n; ++j) {
                xcam = xcam || uses_x_camera(batch[j].job);
                weighted = weighted || batch[j].job.w;
            }
            launch_lm(kind, cam, xcam, weighted, E.probs.p, E.jobs.p + j0, E.lm_in.p + 9 * (size_t)j0, n, max_n, E.mask.p, E.subset.p,
                      max_n_pad, E.h_lm_out.d + j0, cam ? E.h_cam_out.d + (size_t)j0 * nc * CAM_MAX_PARAMS : nullptr, st);
            E.launches++;
        }
        d2h += sizeof(LmJobOut) * nj + sizeof(double) * nc * CAM_MAX_PARAMS * (nj - n_fixed);
        return PLB_OK;
    }
    // ---- the robust/bundle.h refiners (bundle.cc:84-112,206-222,237-256,313-333,394-411): one LM job per problem over
    // all its points.  A job's bits depend on the k_lm instantiation and on the cluster width, which fixes the order of
    // its reductions, and on nothing else in the launch.  So every job runs at the width a lone call of its size takes
    // (lm_lone_width), in one launch per class of (camera refinement, fisheye / division camera, weights, width): each
    // problem gets the bits of its single call whatever else is in the batch.
    // No points is not special: the job runs with empty slices and reports what lm_impl reports for an empty problem
    // (iterations 0, costs 0; the fundamental refiner returns the matrix its factorisation reconstructs).
    int refine() {
        const int nc = kind_cam_count(kind);
        struct Item {
            int i, cam, xcam, w, width;
            LmJob job;
            bool operator<(const Item &o) const {
                return std::tie(cam, xcam, w, width) < std::tie(o.cam, o.xcam, o.w, o.width);
            }
        };
        std::vector<Item> items(NP);
        for (int i = 0; i < NP; ++i) {
            const PState &S = PS[i];
            LmParams prm = bundle_params(S.t->polish.bundle);
            prm.subset_mode = 0;
            LmJob J = lm_job(S.polish_pidx >= 0 ? S.polish_pidx : i, -1, prm);
            J.cam_refine = S.t->polish.cam_refine;
            // the weights follow the problem's points in E.in (upload)
            if (S.t->weights && S.n > 0) J.w = E.in.p + S.in_off + (size_t)in_arr * S.n;
            items[i] = {i, refines_camera(J), uses_x_camera(J), J.w != nullptr, lm_lone_width(S.n), J};
        }
        std::stable_sort(items.begin(), items.end());
        std::vector<LmTask> batch(NP);
        for (int j = 0; j < NP; ++j) batch[j] = {PS[items[j].i].t->model, items[j].job};
        int rc;
        if ((rc = lm_stage(batch, false))) return rc;
        for (int j0 = 0, j1; j0 < NP; j0 = j1) { // one launch per class: a run of equal keys of the sorted items
            j1 = j0 + 1;
            while (j1 < NP && !(items[j0] < items[j1])) ++j1;
            const Item &c = items[j0];
            launch_lm_width(kind, c.cam, c.xcam, c.w, E.probs.p, E.jobs.p + j0, E.lm_in.p + 9 * (size_t)j0, j1 - j0,
                            c.width, E.h_lm_out.d + j0, c.cam ? E.h_cam_out.d + (size_t)j0 * nc * CAM_MAX_PARAMS : nullptr,
                            st);
            E.launches++;
        }
        if ((rc = sync())) return rc;
        PLB_CUDA(cudaGetLastError());
        for (int j = 0; j < NP; ++j) {
            Task &t = *PS[items[j].i].t;
            const LmJobOut &o = E.h_lm_out.p[j];
            std::copy(o.model, o.model + MSZ, t.model);
            if (items[j].cam) // only the parameters the flags select
                for (int i = 0; i < nc; ++i) {
                    int idx[CAM_MAX_PARAMS];
                    const int m = cam_refine_idx(t.polish.cam[i].model, t.polish.cam_refine, idx);
                    for (int c = 0; c < m; ++c)
                        t.polish.cam_out[i]->params[idx[c]] = E.h_cam_out.p[((size_t)j * nc + i) * CAM_MAX_PARAMS + idx[c]];
                }
            if (t.bstats) {
                t.bstats[0] = o.iterations;
                t.bstats[1] = o.initial_cost;
                t.bstats[2] = o.cost;
            }
        }
        return PLB_OK;
    }
    // ---- given models (plb_score_batch): one k_score pass over the group's (problem, tile) list, one wait --------------
    // The problems that want masks are scored by the mask instantiation, the others by the plain one.  Host tasks: the
    // models go up through a pinned staging buffer, the records come back through mapped memory and the masks as bits
    // (k_pack_mask), from the engine's mask buffer (n_pad bytes per model).  Device tasks: k_score reads the caller's
    // models and writes records and mask bytes (stride n) into the caller's buffers.
    int score() {
        const int TMX = score_tile_models(kind);
        const bool host = !PS[0].t->dev_io; // a call's tasks are all host or all device tasks
        std::vector<int> order;
        for (int pass = 0; pass < 2; ++pass)
            for (int i = 0; i < NP; ++i)
                if (PS[i].t->m > 0 && (PS[i].t->inliers != nullptr) == (pass == 1)) order.push_back(i);
        const int nd = (int)order.size();
        if (!nd) return PLB_OK;
        size_t n_models = 0, mask_total = 0;
        for (int i : order) {
            n_models += PS[i].t->m;
            if (PS[i].t->inliers) mask_total += PS[i].t->m * (size_t)PS[i].n_pad;
        }
        int rc;
        if ((rc = E.scdesc.ensure(nd)) || (rc = E.h_scdesc.ensure(nd))) return rc;
        if (host && ((rc = E.models.ensure(n_models * MSZ)) || (rc = E.h_models.ensure(n_models * MSZ)) ||
                     (rc = E.h_counts.ensure(n_models)) || (rc = E.h_scores.ensure(n_models)) ||
                     (rc = E.mask.ensure(mask_total)) || (rc = E.mask_bits.ensure(mask_total / 32 + 1)) ||
                     (rc = E.h_mask_bits.ensure(mask_total / 32 + 1))))
            return rc;
        size_t moff = 0, maskoff = 0;
        long long tiles = 0, tiles_plain = 0;
        int nd_plain = 0;
        for (int j = 0; j < nd; ++j) {
            const PState &S = PS[order[j]];
            const Task &t = *S.t;
            ScoreDesc &D = E.h_scdesc.p[j];
            D.pidx = S.pidx;
            D.reserved = 0;
            D.counts32 = nullptr;
            D.m = (long long)t.m;
            D.tile0 = tiles;
            if (host) {
                std::memcpy(E.h_models.p + moff * MSZ, t.models, sizeof(double) * MSZ * t.m);
                D.models = E.models.p + moff * MSZ;
                D.counts = E.h_counts.d + moff;
                D.scores = E.h_scores.d + moff;
                D.mask = t.inliers ? E.mask.p + maskoff : nullptr;
                D.mask_stride = S.n_pad;
                if (t.inliers) maskoff += t.m * (size_t)S.n_pad;
            } else {
                D.models = t.models;
                D.counts = reinterpret_cast<long long *>(t.counts);
                D.scores = t.scores;
                D.mask = t.inliers;
                D.mask_stride = S.n;
            }
            moff += t.m;
            tiles += (long long)((t.m + TMX - 1) / TMX);
            if (!t.inliers) {
                tiles_plain = tiles;
                nd_plain = j + 1;
            }
        }
        if (host) {
            PLB_CUDA(cudaMemcpyAsync(E.models.p, E.h_models.p, sizeof(double) * MSZ * n_models, cudaMemcpyHostToDevice, st));
            h2d += sizeof(double) * MSZ * n_models;
        } else { // the caller's models are read after its queued work (a group without points has no k_ingest to wait)
            PLB_CUDA(cudaStreamWaitEvent(st, PS[0].t->ready, 0));
        }
        // the mask descriptors count their tiles from 0 in their own launch
        for (int j = nd_plain; j < nd; ++j) E.h_scdesc.p[j].tile0 -= tiles_plain;
        PLB_CUDA(cudaMemcpyAsync(E.scdesc.p, E.h_scdesc.p, sizeof(ScoreDesc) * nd, cudaMemcpyHostToDevice, st));
        h2d += sizeof(ScoreDesc) * nd;
        launch_score_models(kind, false, E.probs.p, E.scdesc.p, nd_plain, tiles_plain, TMX, st);
        launch_score_models(kind, true, E.probs.p, E.scdesc.p + nd_plain, nd - nd_plain, tiles - tiles_plain, TMX, st);
        E.launches += (nd_plain > 0) + (nd > nd_plain);
        if (host && mask_total) {
            launch_pack_mask(E.mask.p, E.mask_bits.p, mask_total, st);
            E.launches++;
            PLB_CUDA(cudaMemcpyAsync(E.h_mask_bits.p, E.mask_bits.p, mask_total / 8, cudaMemcpyDeviceToHost, st));
            d2h += mask_total / 8;
        }
        if ((rc = sync())) return rc;
        PLB_CUDA(cudaGetLastError());
        if (!host) return PLB_OK;
        moff = maskoff = 0;
        for (int i : order) {
            const PState &S = PS[i];
            const Task &t = *S.t;
            std::copy(E.h_scores.p + moff, E.h_scores.p + moff + t.m, t.scores);
            for (size_t j = 0; j < t.m; ++j) t.counts[j] = (int64_t)E.h_counts.p[moff + j];
            moff += t.m;
            d2h += (sizeof(double) + sizeof(long long)) * t.m;
            if (!t.inliers) continue;
            for (size_t j = 0; j < t.m; ++j) {
                const uint32_t *w = E.h_mask_bits.p + ((maskoff + j * S.n_pad) >> 5); // n_pad is a multiple of 32
                char *dst = t.inliers + j * (size_t)S.n;
                for (int k = 0; k < S.n; ++k) dst[k] = (char)((w[k >> 5] >> (k & 31)) & 1u);
            }
            maskoff += t.m * (size_t)S.n_pad;
        }
        return PLB_OK;
    }
    // ---- camera functions (plb_camera_batch): one k_camera launch over the group's (problem, tile) list, one wait -----
    // Host tasks: every input goes up in one copy from a pinned staging buffer, and every output (per task its points,
    // then the Jacobians it asks for) comes back in one copy that the host spreads over the callers' arrays.  Device
    // tasks: after the caller's stream event, k_camera reads and writes the callers' arrays directly.
    int camera() {
        const Task &t0 = *PS[0].t; // a group's tasks share the op, the form and whether they want Jacobians
        const bool host = !t0.dev_io;
        const int op = t0.cam_op, in_w = op == CAMOP_PROJECT ? 3 : 2, out_w = op == CAMOP_UNPROJECT ? 3 : 2;
        const size_t jp_rows = op == CAMOP_PROJECT ? 2 : 3;
        auto res_w = [&](const Task &t) { // doubles per point of the task's outputs
            return (size_t)out_w + (t.cam_jac ? 6 : 0) + (t.cam_jac_params ? jp_rows * cam_num_params(t.cam_a.model) : 0);
        };
        std::vector<int> order;
        size_t in_total = 0, res_total = 0;
        for (int i = 0; i < NP; ++i)
            if (PS[i].t->n > 0) {
                order.push_back(i);
                in_total += PS[i].t->n * in_w;
                res_total += PS[i].t->n * res_w(*PS[i].t);
            }
        const int nd = (int)order.size();
        if (!nd) return PLB_OK;
        int rc;
        if ((rc = E.cdesc.ensure(nd)) || (rc = E.h_cdesc.ensure(nd))) return rc;
        if (host && ((rc = E.in.ensure(in_total)) || (rc = E.h_in.ensure(in_total)) || (rc = E.cam_res.ensure(res_total)) ||
                     (rc = E.h_cam_res.ensure(res_total))))
            return rc;
        size_t in_off = 0, res_off = 0;
        long long tiles = 0;
        for (int j = 0; j < nd; ++j) {
            const Task &t = *PS[order[j]].t;
            CamOpDesc &D = E.h_cdesc.p[j];
            D.cam = t.cam_a;
            D.n = (long long)t.n;
            D.tile0 = tiles;
            tiles += (D.n + CAM_TILE - 1) / CAM_TILE;
            if (host) {
                std::memcpy(E.h_in.p + in_off, t.a, sizeof(double) * t.n * in_w);
                D.in = E.in.p + in_off;
                double *r = E.cam_res.p + res_off;
                D.out = r;
                r += t.n * out_w;
                D.jac = t.cam_jac ? r : nullptr;
                r += t.cam_jac ? t.n * 6 : 0;
                D.jac_params = t.cam_jac_params ? r : nullptr;
                in_off += t.n * in_w;
                res_off += t.n * res_w(t);
            } else {
                D.in = t.a;
                D.out = t.cam_out;
                D.jac = t.cam_jac;
                D.jac_params = t.cam_jac_params;
            }
        }
        if (host) {
            PLB_CUDA(cudaMemcpyAsync(E.in.p, E.h_in.p, sizeof(double) * in_total, cudaMemcpyHostToDevice, st));
            h2d += sizeof(double) * in_total;
        } else {
            PLB_CUDA(cudaStreamWaitEvent(st, t0.ready, 0));
        }
        PLB_CUDA(cudaMemcpyAsync(E.cdesc.p, E.h_cdesc.p, sizeof(CamOpDesc) * nd, cudaMemcpyHostToDevice, st));
        h2d += sizeof(CamOpDesc) * nd;
        launch_camera(op, t0.cam_jac || t0.cam_jac_params, t0.f32, E.cdesc.p, nd, tiles, st);
        E.launches++;
        if (host) {
            PLB_CUDA(cudaMemcpyAsync(E.h_cam_res.p, E.cam_res.p, sizeof(double) * res_total, cudaMemcpyDeviceToHost, st));
            d2h += sizeof(double) * res_total;
        }
        if ((rc = sync())) return rc;
        PLB_CUDA(cudaGetLastError());
        if (!host) return PLB_OK;
        res_off = 0;
        for (int i : order) {
            const Task &t = *PS[i].t;
            const double *r = E.h_cam_res.p + res_off;
            std::copy(r, r + t.n * out_w, t.cam_out);
            r += t.n * out_w;
            if (t.cam_jac) {
                std::copy(r, r + t.n * 6, t.cam_jac);
                r += t.n * 6;
            }
            if (t.cam_jac_params) std::copy(r, r + t.n * jp_rows * cam_num_params(t.cam_a.model), t.cam_jac_params);
            res_off += t.n * res_w(t);
        }
        return PLB_OK;
    }
    // ---- caller-drawn samples (plb_generate_batch): the round's solve kernels and its exact scoring on given samples ---
    // Chunks of at most ROUND_MAX samples, taken from the problems in order.  A problem's segment holds B x MAXM slots,
    // the worst case, so no chunk overflows or is redone.  Per chunk: the sample table (host form: staged and uploaded;
    // device form: k_take_samples from the callers' tables), launch_hypotheses in mode 0 (fp64 records of every model),
    // then k_put_hyps into the callers' rows (device form) or packed into a staging buffer the host expands (host form),
    // so the padding of the rows does not cross PCIe.  A model's bits depend only on its sample and a record's only on its
    // model and problem, so the chunking changes no output.
    int generate() {
        const bool host = !PS[0].t->dev_io; // a call's tasks are all host or all device tasks
        size_t all = 0;
        for (const PState &S : PS) all += S.t->s;
        if (!all) return PLB_OK;
        const size_t max_total = std::min(all, ROUND_MAX), cap = max_total * (size_t)MAXM;
        gen_rows = max_total;
        int rc;
        // sized once for the largest chunk: a reallocation would synchronise the device
        if ((rc = E.samples.ensure(max_total * K)) || (rc = E.n_models.ensure(max_total)) ||
            (rc = E.first_slot.ensure(max_total)) || (rc = E.counts.ensure(cap)) || (rc = E.scores.ensure(cap)) ||
            (rc = E.models.ensure(cap * MSZ)) || (rc = E.model_prob.ensure(cap)) || (rc = E.h_act.ensure(4 * (size_t)NP + 2)) ||
            (rc = E.act.ensure(4 * (size_t)NP + 2)) || (rc = E.prob_count.ensure(NP)) || (rc = E.work.ensure(CTL_WORDS)) ||
            (rc = E.pdesc.ensure(NP)) || (rc = E.h_pdesc.ensure(NP)))
            return rc;
        if (kind_is_relpose(kind) && ((rc = E.s5_blk.ensure(max_total * 105)) || (rc = E.s5_park.ensure(max_total * 100)) ||
                                      (rc = E.s5_cpoly.ensure(max_total * 11)) || (rc = E.s5_roots.ensure(max_total * 10)) ||
                                      (rc = E.s5_nroots.ensure(max_total))))
            return rc;
        if (host ? ((rc = E.h_samples.ensure(max_total * K)) || (rc = E.h_gen.ensure(2 * max_total)) ||
                    (rc = E.gen_stage.ensure(cap * (MSZ + 2))))
                 : ((rc = E.tkdesc.ensure(NP)) || (rc = E.h_tkdesc.ensure(NP))))
            return rc;
        PLB_CUDA(cudaMemsetAsync(E.work.p, 0, CTL_WORDS * sizeof(int), st));
        if (!host) PLB_CUDA(cudaStreamWaitEvent(st, PS[0].t->ready, 0)); // the callers' tables after their queued work
        std::vector<size_t> done(NP, 0);
        for (;;) {
            act.clear();
            size_t total = 0;
            for (int i = 0; i < NP && total < ROUND_MAX; ++i) {
                PState &S = PS[i];
                if (S.t->s == done[i]) continue;
                S.B = std::min(S.t->s - done[i], ROUND_MAX - total);
                S.g0 = total;
                total += S.B;
                act.push_back(i);
            }
            if (act.empty()) return PLB_OK;
            if ((rc = generate_chunk(total, done, host))) return rc;
            for (int i : act) done[i] += PS[i].B;
        }
    }
    int generate_chunk(size_t total, const std::vector<size_t> &done, bool host) {
        const int na = (int)act.size();
        const size_t cap = total * (size_t)MAXM;
        int rc;
        size_t seg = 0; // h_act layout as in launch_round: active[na] | g_off[na+1] | seg_base[na] | seg_cap[na]
        for (int a = 0; a < na; ++a) {
            const PState &S = PS[act[a]];
            const Task &t = *S.t;
            E.h_act.p[a] = act[a];
            E.h_act.p[na + a] = (int)S.g0;
            E.h_act.p[2 * na + 1 + a] = (int)seg;
            E.h_act.p[3 * na + 1 + a] = (int)(S.B * MAXM);
            seg += S.B * MAXM;
            const int32_t *src = t.samples + done[act[a]] * K;
            PutDesc &D = E.h_pdesc.p[a];
            if (host) {
                std::copy(src, src + S.B * K, E.h_samples.p + S.g0 * K); // int32 -> uint32, all checked to be in [0, n)
                D = {E.h_gen.d + S.g0, E.h_gen.d + gen_rows + S.g0, E.gen_stage.p, E.gen_stage.p + cap * MSZ,
                     reinterpret_cast<long long *>(E.gen_stage.p + cap * (MSZ + 1))};
            } else {
                E.h_tkdesc.p[a] = {src, E.samples.p + S.g0 * K, (long long)(S.B * K), S.n, 0};
                const size_t row = done[act[a]];
                D = {t.n_models + row, nullptr, t.gen_models + row * MAXM * MSZ, t.scores + row * MAXM,
                     reinterpret_cast<long long *>(t.counts) + row * MAXM};
            }
        }
        E.h_act.p[2 * na] = (int)total;
        PLB_CUDA(cudaMemcpyAsync(E.act.p, E.h_act.p, sizeof(int) * (4 * na + 1), cudaMemcpyHostToDevice, st));
        PLB_CUDA(cudaMemcpyAsync(E.pdesc.p, E.h_pdesc.p, sizeof(PutDesc) * na, cudaMemcpyHostToDevice, st));
        if (host) {
            PLB_CUDA(cudaMemcpyAsync(E.samples.p, E.h_samples.p, sizeof(uint32_t) * total * K, cudaMemcpyHostToDevice, st));
            h2d += sizeof(uint32_t) * total * K;
        } else {
            long long max_count = 0;
            for (int a = 0; a < na; ++a) max_count = std::max(max_count, E.h_tkdesc.p[a].count);
            PLB_CUDA(cudaMemcpyAsync(E.tkdesc.p, E.h_tkdesc.p, sizeof(TakeDesc) * na, cudaMemcpyHostToDevice, st));
            launch_take_samples(E.tkdesc.p, na, max_count, nullptr, st);
            E.launches++;
        }
        RoundDesc R;
        R.probs = E.probs.p;
        R.active = E.act.p;
        R.g_off = E.act.p + na;
        R.n_active = na;
        R.samples = E.samples.p;
        R.n_total = (int)total;
        HypOut out{};
        out.n_models = E.n_models.p;
        out.first_slot = E.first_slot.p;
        out.seg_base = E.act.p + 2 * na + 1;
        out.seg_cap = E.act.p + 3 * na + 1;
        out.prob_count = E.prob_count.p;
        out.max_seg_cap = 0;
        for (int a = 0; a < na; ++a) out.max_seg_cap = std::max(out.max_seg_cap, E.h_act.p[3 * na + 1 + a]);
        out.overflow = E.work.p + CTL_OVERFLOW; // cannot be set: every segment has the worst-case capacity
        out.counts = E.counts.p;
        out.scores = E.scores.p;
        out.models = E.models.p;
        out.model_prob = E.model_prob.p;
        if (kind_is_relpose(kind)) {
            out.s5_blk = E.s5_blk.p;
            out.s5_park = E.s5_park.p;
            out.s5_cpoly = E.s5_cpoly.p;
            out.s5_roots = E.s5_roots.p;
            out.s5_nroots = E.s5_nroots.p;
        }
        launch_hypotheses(kind, R, out, 0, max_n_pad, nullptr, st);
        launch_put_hyps(R, out, E.pdesc.p, MSZ, MAXM, host, st);
        E.launches += (kind_is_relpose(kind) ? 6 : 2) + 1;
        // the staging buffers of the next chunk are rewritten once this one's copies and kernels are done
        if ((rc = sync())) return rc;
        PLB_CUDA(cudaGetLastError());
        if (!host) return PLB_OK;
        const int *nm = E.h_gen.p, *off = E.h_gen.p + gen_rows;
        size_t n_out = 0;
        for (size_t g = 0; g < total; ++g) n_out += (size_t)nm[g];
        d2h += sizeof(int) * 2 * total;
        if (n_out) {
            if ((rc = E.h_gen_stage.ensure(n_out * (MSZ + 2)))) return rc;
            double *hm = E.h_gen_stage.p, *hs = hm + n_out * MSZ, *hc = hs + n_out;
            PLB_CUDA(cudaMemcpyAsync(hm, E.gen_stage.p, sizeof(double) * n_out * MSZ, cudaMemcpyDeviceToHost, st));
            PLB_CUDA(cudaMemcpyAsync(hs, E.gen_stage.p + cap * MSZ, sizeof(double) * n_out, cudaMemcpyDeviceToHost, st));
            PLB_CUDA(cudaMemcpyAsync(hc, E.gen_stage.p + cap * (MSZ + 1), sizeof(double) * n_out, cudaMemcpyDeviceToHost, st));
            d2h += sizeof(double) * n_out * (MSZ + 2);
            if ((rc = sync())) return rc;
        }
        const double *hm = E.h_gen_stage.p, *hs = hm + n_out * MSZ;
        const long long *hc = reinterpret_cast<const long long *>(hs + n_out);
        for (int a = 0; a < na; ++a) {
            const PState &S = PS[act[a]];
            const Task &t = *S.t;
            for (size_t j = 0; j < S.B; ++j) {
                const size_t row = done[act[a]] + j, g = S.g0 + j;
                const int c = nm[g];
                const size_t o = (size_t)off[g];
                t.n_models[row] = c;
                std::copy(hm + o * MSZ, hm + (o + c) * MSZ, t.gen_models + row * MAXM * MSZ);
                std::copy(hs + o, hs + o + c, t.scores + row * MAXM);
                for (int m = 0; m < c; ++m) t.counts[row * MAXM + m] = (int64_t)hc[o + m];
            }
        }
        return PLB_OK;
    }
    LmJob lo_job(const PState &S) const { return lm_job(S.pidx, -1, lo_params(kind, S.t->max_error)); }
    // one LO call of the serial loop and its result (ransac_impl.h:135-153)
    void apply_lo(PState &S, const LmJobOut &o) const {
        S.stats.refinements++;
        S.cnt.lo_calls++;
        S.cnt.hypotheses++;
        if (o.score < S.stats.model_score) {
            S.stats.model_score = o.score;
            S.stats.num_inliers = o.count;
            std::copy(o.model, o.model + MSZ, S.best_model);
        }
        update_dynamic(S, K);
    }

    // ---- initial models (ransac_impl.h:173-176) ----------------------------------------------------------------------
    int score_initial_models() {
        std::vector<int> who;
        for (int i = 0; i < NP; ++i)
            if (PS[i].enough && PS[i].t->opt.score_initial_model) who.push_back(i);
        const int nw = (int)who.size();
        if (!nw) return PLB_OK;
        int rc;
        if ((rc = E.h_scdesc.ensure(nw)) || (rc = E.scdesc.ensure(nw)) || (rc = E.h_counts.ensure(nw)) ||
            (rc = E.h_scores.ensure(nw)) || (rc = E.models.ensure((size_t)nw * MSZ)))
            return rc;
        std::vector<double> packed((size_t)nw * MSZ); // the MSZ-strided model list k_score reads
        for (int j = 0; j < nw; ++j) {
            std::copy(PS[who[j]].t->model, PS[who[j]].t->model + MSZ, packed.data() + (size_t)j * MSZ);
            E.h_scdesc.p[j] = {E.models.p + (size_t)j * MSZ, E.h_counts.d + j, E.h_scores.d + j, nullptr, 0, j, 1, who[j], 0};
        }
        PLB_CUDA(cudaMemcpyAsync(E.models.p, packed.data(), sizeof(double) * nw * MSZ, cudaMemcpyHostToDevice, st));
        PLB_CUDA(cudaMemcpyAsync(E.scdesc.p, E.h_scdesc.p, sizeof(ScoreDesc) * nw, cudaMemcpyHostToDevice, st));
        launch_score_models(kind, false, E.probs.p, E.scdesc.p, nw, nw, 1, st); // one-model tiles
        E.launches++;
        if ((rc = sync())) return rc;
        std::vector<LmTask> lo;
        std::vector<PState *> lo_of;
        for (int j = 0; j < nw; ++j) {
            PState &S = PS[who[j]];
            const size_t ic = E.h_counts.p[j];
            const double sc = E.h_scores.p[j];
            S.cnt.hypotheses++;
            const bool more = ic > S.best_minimal_inlier_count, better = sc < S.best_minimal_msac_score;
            if (more || better) {
                if (more) S.best_minimal_inlier_count = ic;
                if (better) S.best_minimal_msac_score = sc;
                if (sc < S.stats.model_score) {
                    S.stats.model_score = sc;
                    S.stats.num_inliers = ic;
                }
                lo.push_back({S.t->model, lo_job(S)});
                lo_of.push_back(&S);
            }
        }
        if (lo.empty()) return PLB_OK;
        if ((rc = lm_batch(lo)) || (rc = sync(&lo_wait))) return rc;
        for (size_t j = 0; j < lo.size(); ++j) apply_lo(*lo_of[j], E.h_lm_out.p[j]);
        return PLB_OK;
    }

    // ---- device sampler states (robust/sampling.h:49-83), PROSAC growth tables (sampling.cc:105-136), LO templates --
    int init_samplers() {
        for (PState &S : PS) {
            S.active = S.enough && S.t->opt.max_iterations > 0;
            S.chunk = std::min<size_t>(4096, std::max<size_t>(1024, 16384 / few));
        }
        size_t growth_total = 0;
        for (PState &S : PS)
            if (S.active && S.t->opt.progressive_sampling) growth_total += std::max<size_t>(S.t->n, (size_t)K);
        int rc;
        if ((rc = E.h_smp.ensure(NP)) || (rc = E.smp.ensure(2 * (size_t)NP)) || (rc = E.h_growth.ensure(growth_total)) ||
            (rc = E.growth.ensure(growth_total)) || (rc = E.h_lo_tmpl.ensure(NP)) || (rc = E.lo_tmpl.ensure(NP)) ||
            (rc = E.h_hypfix.ensure(NP)))
            return rc;
        size_t goff = 0;
        for (int i = 0; i < NP; ++i) {
            PState &S = PS[i];
            SamplerDev &D = E.h_smp.p[i];
            std::memset(&D, 0, sizeof(D));
            E.h_lo_tmpl.p[i] = lo_job(S);
            if (!S.active) continue;
            D.state = S.t->opt.seed;
            D.n = (uint32_t)S.t->n;
            D.k = (uint32_t)K;
            D.max_prosac = S.t->opt.max_prosac_iterations;
            if (S.t->opt.progressive_sampling) {
                Sampler smp(S.t->n, (size_t)K, S.t->opt); // host: the O(N) growth table only
                uint64_t *g = E.h_growth.p + goff;
                bool strict = true;
                for (size_t j = 0; j < smp.growth.size(); ++j) {
                    g[j] = (uint64_t)smp.growth[j];
                    if (j >= (size_t)K && !(smp.growth[j] > smp.growth[j - 1])) strict = false;
                }
                D.growth = E.growth.p + goff;
                D.sample_k = 1;
                D.subset_sz = (uint32_t)K;
                D.flags = 1u | (strict ? 2u : 0u);
                goff += smp.growth.size();
            }
        }
        PLB_CUDA(cudaMemcpyAsync(E.smp.p, E.h_smp.p, sizeof(SamplerDev) * NP, cudaMemcpyHostToDevice, st));
        PLB_CUDA(cudaMemcpyAsync(E.lo_tmpl.p, E.h_lo_tmpl.p, sizeof(LmJob) * NP, cudaMemcpyHostToDevice, st));
        h2d += (sizeof(SamplerDev) + sizeof(LmJob)) * NP;
        if (growth_total) {
            PLB_CUDA(cudaMemcpyAsync(E.growth.p, E.h_growth.p, sizeof(uint64_t) * growth_total, cudaMemcpyHostToDevice, st));
            h2d += sizeof(uint64_t) * growth_total;
        }
        return PLB_OK;
    }

    // break test at the top of iteration `it` (ransac_impl.h:180-184); returns the number of problems still running
    int select_active() {
        act.clear();
        for (int i = 0; i < NP; ++i) {
            PState &S = PS[i];
            if (!S.active) continue;
            if (S.it >= S.t->opt.max_iterations || (S.it > S.t->opt.min_iterations && S.it > S.dynamic_max_iter)) {
                S.active = false;
                continue;
            }
            act.push_back(i);
        }
        return (int)act.size();
    }

    // ---- one lock-step round -----------------------------------------------------------------------------------------
    // Every round is ONE chain of launches with ONE host synchronisation at its end:
    //   k_sample -> solve kernels -> scoring (fp64 of every model, or fp32 screening) -> k_select -> [k_confirm] ->
    //   k_pass1 -> k_lm over the LO triggers it listed.
    // The sampler states, the per-model records and the candidate lists never leave the device; the host receives, per
    // problem, one header, the few models that improved the best-minimal state and the LO results, and replays
    // score_models() (ransac_impl.h:106-154) over those.  A round whose records overflow is redone with larger
    // capacities: nothing was committed, the sampler states of the round are still current.
    int round() {
        const int na = (int)act.size();
        // round sizes: up to the iteration at which the serial loop would stop for the current dynamic_max_iter
        size_t total = 0;
        const size_t per_cap = std::max<size_t>(256, S_TOT_MAX / (size_t)na);
        int est_jobs = 0;
        for (int a = 0; a < na; ++a) {
            PState &S = PS[act[a]];
            const size_t stop_at = std::min<size_t>(S.t->opt.max_iterations, std::max(S.t->opt.min_iterations, S.dynamic_max_iter) + 1);
            // While no model with a usable inlier ratio exists (dyn == max_iterations) the round size doubles from
            // 1024; once dynamic_max_iter has come down, later improvements only lower it a little, so the rest of the
            // loop is evaluated in one go (what is past the final break point is discarded by the replay).
            const bool settled = S.dynamic_max_iter < S.t->opt.max_iterations;
            size_t B = settled ? std::min<size_t>(stop_at - S.it, ROUND_MAX) : std::min(S.chunk, CHUNK_MAX);
            B = std::min(B, per_cap);
            B = std::min(B, stop_at - S.it); // stop_at > it for an active problem
            S.B = B;
            S.g0 = total;
            total += B;
            est_jobs += first_round[act[a]] ? 12 : 2; // LO triggers: a record chain at first, then the odd improvement
        }
        for (;;) {
            int rc;
            if ((rc = launch_round(total, est_jobs)) || (rc = sync())) return rc;
            mark(PH_WAIT_HYP);
            d2h += CTL_WORDS * sizeof(int);
            if (E.h_work.p[CTL_OVERFLOW] != 0) { // model list overflow: redo the round with the worst-case capacity
                if (cap_factor >= MAXM) {
                    g_err = "internal error: model capacity exceeded";
                    return PLB_ERR_CUDA;
                }
                cap_factor = MAXM;
                continue;
            }
            if (E.h_work.p[CTL_FLAGS] != 0) { // more improving models / LO triggers than the record buffers hold
                if (big_caps) {
                    g_err = "internal error: record capacity exceeded";
                    return PLB_ERR_CUDA;
                }
                big_caps = true;
                continue;
            }
            break;
        }
        smp_cur ^= 1;
        float ms = 0.f, ms_sc = 0.f, ms_cf = 0.f, ms_lo = 0.f;
        cudaEventElapsedTime(&ms, E.ev0, E.ev1);
        cudaEventElapsedTime(&ms_sc, E.ev2, E.ev1);
        cudaEventElapsedTime(&ms_cf, E.ev1, E.ev3);
        cudaEventElapsedTime(&ms_lo, E.ev3, E.ev4);
        gpu_ms_total += ms + ms_cf;
        gpu_ms_score += ms_sc;
        gpu_ms_confirm += ms_cf;
        gpu_ms_lo += ms_lo;
        return PLB_OK;
    }

    // the launch chain of one round over the `total` samples sized by round(), ending with the control words' copy
    int launch_round(size_t total, int est_jobs) {
        const int na = (int)act.size();
        const size_t cap_models = total * (size_t)cap_factor;
        // capacity of the host-visible records of the round; exceeded -> the round is redone with the worst case
        const size_t job_cap = big_caps ? total : std::min(total, std::max<size_t>(1024, total / 8));
        const size_t imp_cap = big_caps ? cap_models : std::min(cap_models, 2 * job_cap);
        const int lm_clusters = lm_round_max_clusters(kind, est_jobs, max_n);
        int rc;
        if ((rc = E.samples.ensure(total * K)) || (rc = E.n_models.ensure(total)) || (rc = E.first_slot.ensure(total)) ||
            (rc = E.prefix.ensure(total)) || (rc = E.counts.ensure(cap_models)) || (rc = E.scores.ensure(cap_models)) ||
            (rc = E.models.ensure(cap_models * MSZ)) || (rc = E.model_prob.ensure(cap_models)) ||
            (rc = E.cand_slot.ensure(cap_models)) || (rc = E.cand_sample.ensure(cap_models)) ||
            (rc = E.h_act.ensure(4 * (size_t)na + 2)) || (rc = E.act.ensure(4 * (size_t)na + 2)) ||
            (rc = E.h_rp.ensure(na)) || (rc = E.rp.ensure(na)) || (rc = E.n_cand.ensure(na)) ||
            (rc = E.n_models_tot.ensure(na)) || (rc = E.prob_count.ensure(na)) || (rc = E.h_hdr.ensure(na)) ||
            (rc = E.h_imp.ensure(imp_cap)) || (rc = E.job_src.ensure(job_cap)) || (rc = E.h_lm_out.ensure(job_cap)) ||
            (rc = E.subset.ensure((size_t)lm_clusters * max_n_pad)))
            return rc;
        ++n_rounds;
        // h_act layout: active[na] | g_off[na+1] | seg_base[na] | seg_cap[na]
        int max_seg_cap = 0;
        size_t seg = 0;
        for (int a = 0; a < na; ++a) {
            const PState &S = PS[act[a]];
            E.h_act.p[a] = act[a];
            E.h_act.p[na + a] = (int)S.g0;
            E.h_act.p[2 * na + 1 + a] = (int)seg;
            const int cap = (int)(S.B * (size_t)cap_factor);
            E.h_act.p[3 * na + 1 + a] = cap;
            max_seg_cap = std::max(max_seg_cap, cap);
            RoundProb &Q = E.h_rp.p[a];
            Q.pidx = act[a];
            Q.g0 = (int)S.g0;
            Q.B = (int)S.B;
            Q.seg_base = (int)seg;
            Q.seg_cap = cap;
            Q.reserved = 0;
            Q.lb0 = (double)S.best_minimal_inlier_count;
            Q.ub0 = S.best_minimal_msac_score;
            seg += (size_t)cap;
        }
        E.h_act.p[2 * na] = (int)total;
        PLB_CUDA(cudaMemcpyAsync(E.act.p, E.h_act.p, sizeof(int) * (4 * na + 1), cudaMemcpyHostToDevice, st));
        PLB_CUDA(cudaMemcpyAsync(E.rp.p, E.h_rp.p, sizeof(RoundProb) * na, cudaMemcpyHostToDevice, st));
        h2d += sizeof(int) * (4 * na + 1) + sizeof(RoundProb) * na;
        PLB_CUDA(cudaMemsetAsync(E.work.p, 0, CTL_WORDS * sizeof(int), st));
        RoundDesc R;
        R.probs = E.probs.p;
        R.active = E.act.p;
        R.g_off = E.act.p + na;
        R.n_active = na;
        R.samples = E.samples.p;
        R.n_total = (int)total;
        HypOut out{}; // fast-mode and 5-point buffers stay null unless set below
        out.n_models = E.n_models.p;
        out.first_slot = E.first_slot.p;
        out.seg_base = E.act.p + 2 * na + 1;
        out.seg_cap = E.act.p + 3 * na + 1;
        out.prob_count = E.prob_count.p;
        out.max_seg_cap = max_seg_cap;
        out.overflow = E.work.p + CTL_OVERFLOW;
        out.counts = E.counts.p;
        out.scores = E.scores.p;
        out.models = E.models.p;
        out.model_prob = E.model_prob.p;
        if (mode == 1) {
            if ((rc = E.fcounts.ensure(cap_models)) || (rc = E.fscores.ensure(cap_models)) ||
                (rc = E.fborder.ensure(cap_models)) || (rc = E.ferr.ensure(cap_models)) ||
                (rc = E.fctx.ensure(cap_models * scr::CTX_FLOATS)))
                return rc;
            out.fcounts = E.fcounts.p;
            out.fscores = E.fscores.p;
            out.fborder = E.fborder.p;
            out.ferr = E.ferr.p;
        }
        if (kind_is_relpose(kind)) { // phase buffers of the 3-kernel 5-point solver
            if ((rc = E.s5_blk.ensure(total * 105)) || (rc = E.s5_park.ensure(total * 100)) || (rc = E.s5_cpoly.ensure(total * 11)) ||
                (rc = E.s5_roots.ensure(total * 10)) || (rc = E.s5_nroots.ensure(total)))
                return rc;
            out.s5_blk = E.s5_blk.p;
            out.s5_park = E.s5_park.p;
            out.s5_cpoly = E.s5_cpoly.p;
            out.s5_roots = E.s5_roots.p;
            out.s5_nroots = E.s5_nroots.p;
        }
        // (every buffer of the round is allocated by now: nothing between the events below can stall on cudaMalloc)
        PLB_CUDA(cudaEventRecord(E.ev0, st));
        launch_sample(E.rp.p, na, E.smp.p + (size_t)smp_cur * NP, E.smp.p + (size_t)(smp_cur ^ 1) * NP, E.samples.p, st);
        E.launches++;
        mark(PH_SAMPLE);
        launch_hypotheses(kind, R, out, mode, max_n_pad, E.fctx.p, st, E.ev2);
        PLB_CUDA(cudaEventRecord(E.ev1, st));
        // one solve kernel (5pt: k5_gather, k5_null, k5_elim, k5_roots, k5_back) + scoring (fast mode: k_screen_ctx + k_screen)
        E.launches += (kind_is_relpose(kind) ? 6 : 2) + (mode == 1 && kind != KIND_RELPOSE_TS ? 1 : 0);
        SelectArgs SA;
        SA.rp = E.rp.p;
        SA.na = na;
        SA.mode = mode;
        SA.n_models = E.n_models.p;
        SA.first_slot = E.first_slot.p;
        SA.fcounts = out.fcounts;
        SA.fscores = out.fscores;
        SA.fborder = out.fborder;
        SA.ferr = out.ferr;
        SA.counts = E.counts.p;
        SA.scores = E.scores.p;
        SA.prefix = E.prefix.p;
        SA.cand_slot = E.cand_slot.p;
        SA.cand_sample = E.cand_sample.p;
        SA.n_cand = E.n_cand.p;
        SA.n_models_tot = E.n_models_tot.p;
        launch_select(SA, st);
        E.launches++;
        if (mode == 1) {
            launch_confirm(kind, E.probs.p, SA, E.models.p, st);
            E.launches++;
        }
        PLB_CUDA(cudaEventRecord(E.ev3, st));
        Pass1Args PA;
        PA.rp = E.rp.p;
        PA.na = na;
        PA.cand_slot = E.cand_slot.p;
        PA.cand_sample = E.cand_sample.p;
        PA.n_cand = E.n_cand.p;
        PA.n_models_tot = E.n_models_tot.p;
        PA.counts = E.counts.p;
        PA.scores = E.scores.p;
        PA.models = E.models.p;
        PA.msz = MSZ;
        PA.ctl = E.work.p;
        PA.imp_cap = (int)imp_cap;
        PA.job_cap = (int)job_cap;
        PA.hdr = E.h_hdr.d;
        PA.imp = E.h_imp.d;
        PA.job_src = E.job_src.p;
        launch_pass1(PA, st);
        launch_lm_round(kind, E.probs.p, E.lo_tmpl.p, E.job_src.p, E.models.p, E.work.p + CTL_JOB_TOTAL, (int)job_cap,
                        est_jobs, max_n, E.subset.p, max_n_pad, E.h_lm_out.d, st);
        E.launches += 2;
        PLB_CUDA(cudaEventRecord(E.ev4, st));
        PLB_CUDA(cudaMemcpyAsync(E.h_work.p, E.work.p, CTL_WORDS * sizeof(int), cudaMemcpyDeviceToHost, st));
        mark(PH_LAUNCH);
        return PLB_OK;
    }

    // ---- replay of the serial loop over the round, problem by problem (ransac_impl.h:106-154,180-188) ----------------
    // Only samples with an improving model change the state; between two of them the break test
    // `it > min_iterations && it > dynamic_max_iter` (:182) first holds at max(min_iterations, dyn) + 1.
    int replay() {
        const int na = (int)act.size();
        for (int a = 0; a < na; ++a) {
            PState &S = PS[act[a]];
            first_round[act[a]] = 0;
            const plb_ransac_opt &opt = S.t->opt;
            const SelHeader &H = E.h_hdr.p[a];
            const ImpRec *imp = E.h_imp.p + H.imp_base;
            const LmJobOut *lo = E.h_lm_out.p + H.trig_base;
            d2h += sizeof(SelHeader) + sizeof(ImpRec) * (size_t)H.n_imp + sizeof(LmJobOut) * (size_t)H.n_trig;
            S.cnt.samples_evaluated += S.B;
            S.cnt.models_evaluated += (uint64_t)H.n_models;
            S.cnt.models_confirmed += (mode == 1) ? (uint64_t)H.n_cand : 0;
            S.chunk = std::min(CHUNK_MAX, S.chunk * 2);
            const size_t it0 = S.it, it_end = S.it + S.B;
            int ip = 0, tp = 0;
            size_t cur = it0;
            bool broke = false;
            for (;;) {
                const size_t next_trig = (ip < H.n_imp) ? it0 + (size_t)imp[ip].sample : it_end;
                const size_t brk = std::max(cur, std::max<size_t>(opt.min_iterations, S.dynamic_max_iter) + 1);
                if (brk <= next_trig && brk < it_end) { // the loop leaves at the top of iteration `brk`
                    cur = brk;
                    broke = true;
                    break;
                }
                if (next_trig >= it_end) {
                    cur = it_end;
                    break;
                }
                // iteration next_trig: its improving models in order (ransac_impl.h:113-133), then LO (:135-153)
                const int smp = imp[ip].sample;
                while (ip < H.n_imp && imp[ip].sample == smp) {
                    const size_t ic = imp[ip].count;
                    const double sc = imp[ip].score;
                    if (ic > S.best_minimal_inlier_count) S.best_minimal_inlier_count = ic;
                    if (sc < S.best_minimal_msac_score) S.best_minimal_msac_score = sc;
                    if (sc < S.stats.model_score) { // :127-131
                        S.stats.model_score = sc;
                        std::copy(imp[ip].model, imp[ip].model + MSZ, S.best_model);
                        S.stats.num_inliers = ic;
                    }
                    ++ip;
                }
                apply_lo(S, lo[tp++]);
                cur = next_trig + 1;
            }
            S.cnt.samples += cur - it0;
            S.it = cur;
            if (broke) {
                S.active = false;
                // hypotheses of the samples before the break: one prefix-sum word, fetched behind the round (read at
                // the end of the call; stream order keeps it ahead of the next round's kernels)
                if (cur > it0) {
                    PLB_CUDA(cudaMemcpyAsync(E.h_hypfix.p + S.pidx, E.prefix.p + S.g0 + (cur - it0 - 1), sizeof(int),
                                             cudaMemcpyDeviceToHost, st));
                    S.hyp_pending = true;
                    d2h += sizeof(int);
                }
            } else {
                S.cnt.hypotheses += (uint64_t)H.n_models;
            }
        }
        mark(PH_REPLAY);
        return PLB_OK;
    }

    // ---- final refinement of every problem (ransac_impl.h:190-198), one launch ---------------------------------------
    int final_refine() {
        std::vector<LmTask> jobs;
        std::vector<PState *> of;
        for (PState &S : PS) {
            if (!S.enough) continue;
            S.stats.iterations = S.it;
            jobs.push_back({S.best_model, lo_job(S)});
            of.push_back(&S);
        }
        if (jobs.empty()) return PLB_OK;
        int rc;
        if ((rc = lm_batch(jobs)) || (rc = sync(&lo_wait))) return rc;
        for (size_t j = 0; j < jobs.size(); ++j) {
            PState &S = *of[j];
            const LmJobOut &o = E.h_lm_out.p[j];
            S.stats.refinements++;
            S.cnt.lo_calls++;
            S.cnt.hypotheses++;
            if (o.score < S.stats.model_score) { // NB: model_score itself is not updated by the reference here
                std::copy(o.model, o.model + MSZ, S.best_model);
                S.stats.num_inliers = o.count;
            }
        }
        return PLB_OK;
    }

    // ---- final inlier masks (ransac.cc:54,151,259,311) + optional polish over the inliers (robust.cc) -----------------
    int masks_and_polish() {
        std::vector<int> who;
        for (int i = 0; i < NP; ++i)
            if (PS[i].n > 0) who.push_back(i);
        const int nw = (int)who.size();
        int rc;
        if ((rc = E.h_mdesc.ensure(nw)) || (rc = E.mdesc.ensure(nw))) return rc;
        for (int j = 0; j < nw; ++j) {
            PState &S = PS[who[j]];
            MaskDesc &D = E.h_mdesc.p[j];
            D.pidx = S.pidx;
            D.reserved = 0;
            D.mask_off = S.mask_off;
            std::copy(S.best_model, S.best_model + 9, D.model);
        }
        PLB_CUDA(cudaMemcpyAsync(E.mdesc.p, E.h_mdesc.p, sizeof(MaskDesc) * nw, cudaMemcpyHostToDevice, st));
        h2d += sizeof(MaskDesc) * nw;
        launch_inlier_masks(kind, E.probs.p, E.mdesc.p, nw, max_n, E.mask.p, st);
        E.launches++;
        // robust.cc:103-123,296-311,573-588,736-751: LM over the inliers with the user's BundleOptions
        std::vector<LmTask> pol;
        std::vector<PState *> pol_of;
        for (int cam = 0; cam < 2; ++cam) // the jobs that refine the camera last (lm_batch)
            for (PState &S : PS) {
                if (S.n == 0 || !S.t->polish.enabled || S.stats.num_inliers <= S.t->polish.min_inliers) continue;
                const FinalPolish &fp = S.t->polish;
                LmJob J = lm_job(S.polish_pidx >= 0 ? S.polish_pidx : S.pidx, S.mask_off, bundle_params(fp.bundle));
                J.cam_refine = fp.cam_refine;
                if (refines_camera(J) != (cam == 1)) continue;
                pol.push_back({S.best_model, J});
                pol_of.push_back(&S);
            }
        if (!pol.empty() && (rc = lm_batch(pol))) return rc;
        // host callers: the masks cross PCIe as bits (1/8 of the bytes) and are expanded into the caller's char[n] below;
        // device callers (plb_estimate_batch_device): k_scatter_masks writes them into the caller's buffers
        bool host_out = false;
        int n_scatter = 0, max_scatter = 0;
        for (const PState &S : PS) {
            host_out = host_out || !S.t->dev_io;
            if (S.t->dev_io && S.t->inliers && S.n > 0) {
                ++n_scatter;
                max_scatter = std::max(max_scatter, S.n);
            }
        }
        if (host_out) {
            launch_pack_mask(E.mask.p, E.mask_bits.p, mask_bytes, st);
            E.launches++;
            PLB_CUDA(cudaMemcpyAsync(E.h_mask_bits.p, E.mask_bits.p, sizeof(uint32_t) * (mask_bytes / 32), cudaMemcpyDeviceToHost, st));
        }
        if (n_scatter) {
            if ((rc = E.sdesc.ensure(n_scatter)) || (rc = E.h_sdesc.ensure(n_scatter))) return rc;
            int j = 0;
            for (const PState &S : PS)
                if (S.t->dev_io && S.t->inliers && S.n > 0) E.h_sdesc.p[j++] = {S.t->inliers, S.mask_off, S.n};
            PLB_CUDA(cudaMemcpyAsync(E.sdesc.p, E.h_sdesc.p, sizeof(ScatterDesc) * n_scatter, cudaMemcpyHostToDevice, st));
            launch_scatter_masks(E.mask.p, E.sdesc.p, n_scatter, max_scatter, st);
            E.launches++;
        }
        if ((rc = sync())) return rc;
        for (size_t j = 0; j < pol.size(); ++j) {
            const FinalPolish &fp = pol_of[j]->t->polish;
            std::copy(E.h_lm_out.p[j].model, E.h_lm_out.p[j].model + MSZ, pol_of[j]->best_model);
            const bool refined = refines_camera(pol[j].job);
            for (int i = 0; i < kind_cam_count(kind); ++i)
                if (fp.cam_out[i])
                    polish_camera_out(fp.cam[i], fp.scale,
                                      refined ? E.h_cam_out.p + (j * kind_cam_count(kind) + i) * CAM_MAX_PARAMS : fp.cam[i].p,
                                      fp.cam_out[i]);
        }
        for (PState &S : PS) {
            if (!S.t->dev_io) {
                if (S.t->inliers && S.n > 0) {
                    const uint32_t *w = E.h_mask_bits.p + (S.mask_off >> 5); // mask_off is a multiple of 32
                    char *dst = S.t->inliers;
                    for (int k = 0; k < S.n; ++k) dst[k] = (char)((w[k >> 5] >> (k & 31)) & 1u);
                }
                d2h += (size_t)S.n_pad / 8;
            }
            std::copy(S.best_model, S.best_model + MSZ, S.t->model);
        }
        PLB_CUDA(cudaGetLastError());
        return PLB_OK;
    }

    // ---- the profile line and the counters; group-level counters are attributed to the first problem ----------------
    void report() {
        mark(PH_FINAL);
        if (profiling()) {
            double tot = 0;
            for (int i = 0; i < PH_N; ++i) tot += ph[i];
            std::fprintf(stderr,
                         "[plb profile] kind %d problems %d rounds %d total %.2f ms | setup %.2f sample %.2f launch %.2f "
                         "wait_hyp %.2f replay %.2f final %.2f\n",
                         kind, NP, n_rounds, 1e3 * tot, 1e3 * ph[PH_SETUP], 1e3 * ph[PH_SAMPLE], 1e3 * ph[PH_LAUNCH],
                         1e3 * ph[PH_WAIT_HYP], 1e3 * ph[PH_REPLAY], 1e3 * ph[PH_FINAL]);
        }
        PS[0].cnt.lo_seconds = lo_wait;
        PS[0].cnt.gpu_launches = E.launches - launches0;
        PS[0].cnt.gpu_seconds = gpu_ms_total * 1e-3;
        PS[0].cnt.gpu_seconds_score = gpu_ms_score * 1e-3;
        PS[0].cnt.gpu_seconds_select = gpu_ms_confirm * 1e-3;
        PS[0].cnt.gpu_seconds_lo = gpu_ms_lo * 1e-3;
        PS[0].cnt.rounds = (uint64_t)n_rounds;
        PS[0].cnt.h2d_bytes = h2d;
        PS[0].cnt.d2h_bytes = d2h;
        finish();
    }
    // per-problem outputs: stats and counters
    void finish() {
        for (PState &S : PS) {
            if (S.hyp_pending) S.cnt.hypotheses += (uint64_t)E.h_hypfix.p[S.pidx];
            S.cnt.scored_corrs = S.cnt.hypotheses * S.t->n;
            if (S.t->stats_out) *S.t->stats_out = S.stats;
            if (S.t->cnt_out) *S.t->cnt_out = S.cnt;
        }
    }
};

// Runs a group of problems of the same kind in lock-step rounds (see Group).
static int run_group(int kind, std::vector<Task *> &tasks) {
    Group G(kind, tasks);
    int rc = G.init_states();
    if (rc != PLB_OK) return rc;
    if (std::none_of(G.PS.begin(), G.PS.end(), [](const PState &S) { return S.n > 0; })) {
        G.finish();
        return PLB_OK;
    }
    if ((rc = G.init())) return rc;
    lm_set_sm_share(t_batch_worker ? 50 : 100); // a lone call owns the GPU; batch groups share it
    if ((rc = G.upload()) || (rc = G.normalize()) || (rc = G.transpose()) || (rc = G.score_initial_models()) ||
        (rc = G.init_samplers()))
        return rc;
    G.mark(Group::PH_SETUP);
    while (G.select_active())
        if ((rc = G.round()) || (rc = G.replay())) return rc;
    if ((rc = G.final_refine()) || (rc = G.masks_and_polish())) return rc;
    G.report();
    return PLB_OK;
}

// Single-problem convenience used by the plb_ransac_* / plb_estimate_* entry points.
static int run_ransac(int kind, const double *a, const double *b, size_t n_pts, const plb_ransac_opt &opt,
                      double max_error, int rfc, double *model, char *inliers, plb_ransac_stats *stats_out,
                      plb_counters *cnt_out, const FinalPolish &polish, int pre_mode = 0,
                      const CamDev *cam_a = nullptr, const CamDev *cam_b = nullptr, double pre_scale = 1.0) {
    Task t;
    t.pre_mode = pre_mode;
    t.pre_scale = pre_scale;
    if (cam_a) t.cam_a = *cam_a;
    if (cam_b) t.cam_b = *cam_b;
    t.kind = kind;
    t.a = a;
    t.b = b;
    t.n = n_pts;
    t.opt = opt;
    t.max_error = max_error;
    t.rfc = rfc;
    t.model = model;
    t.inliers = inliers;
    t.stats_out = stats_out;
    t.cnt_out = cnt_out;
    t.polish = polish;
    std::vector<Task *> v{&t};
    return run_group(kind, v);
}

// Runs a group of refiner tasks of the same kind (Task::refine): the upload of the group (sq_thr 0, no normalisation,
// no pre-step beyond the tangent-Sampson one), then one LM job per problem (Group::refine).
static int run_refine_group(int kind, std::vector<Task *> &tasks) {
    Group G(kind, tasks);
    int rc;
    if ((rc = G.init()) || (rc = G.upload()) || (rc = G.transpose()) || (rc = G.refine())) return rc;
    return PLB_OK;
}

// Runs a group of score tasks of the same kind (Task::score): the upload of the group (tangent Sampson: the camera
// pre-step), then one scoring pass over every given model (Group::score).
static int run_score_group(int kind, std::vector<Task *> &tasks) {
    Group G(kind, tasks);
    int rc;
    if ((rc = G.init()) || (rc = G.upload()) || (rc = G.transpose()) || (rc = G.score())) return rc;
    return PLB_OK;
}

// Runs a group of generate tasks of the same kind (Task::generate): the upload of the group (tangent Sampson: the camera
// pre-step), then the solve kernels and exact scoring of every caller-drawn sample (Group::generate).
static int run_generate_group(int kind, std::vector<Task *> &tasks) {
    Group G(kind, tasks);
    int rc;
    if ((rc = G.init()) || (rc = G.upload()) || (rc = G.transpose()) || (rc = G.generate())) return rc;
    return PLB_OK;
}

// Runs a group of camera tasks of one op (Task::camop), all with or all without Jacobians: one k_camera launch
// (Group::camera).  The group's kind is unused.
static int run_camera_group(std::vector<Task *> &tasks) {
    Group G(KIND_PNP, tasks);
    int rc;
    if ((rc = G.init()) || (rc = G.camera())) return rc;
    return PLB_OK;
}

// plb_camera -> CamDev; models outside the ten on the path (cam_layout) are rejected like Camera::unproject's "NYI"
// (misc/camera_models.cc:176-188)
static int camera_dev(const plb_camera *c, CamDev *out) {
    out->model = CAMM_NULL;
    out->reserved = 0;
    for (int i = 0; i < 8; ++i) out->p[i] = 0.0;
    if (!c || c->model_id == PLB_CAMERA_NULL) return PLB_OK;
    CamLayout L;
    if (!cam_layout(c->model_id, L)) {
        g_err = "NYI: camera model not supported by the CUDA path (undistort on the host first)";
        return PLB_ERR_NYI;
    }
    out->model = c->model_id;
    for (int i = 0; i < L.np(); ++i) out->p[i] = c->params[i];
    return PLB_OK;
}

} // namespace plb

using namespace plb;

extern "C" {

void plb_ransac_opt_default(plb_ransac_opt *o) {
    o->max_iterations = 100000;
    o->min_iterations = 1000;
    o->dyn_num_trials_mult = 3.0;
    o->success_prob = 0.9999;
    o->seed = 0;
    o->progressive_sampling = 0;
    o->score_initial_model = 0;
    o->max_prosac_iterations = 100000;
}
void plb_bundle_opt_default(plb_bundle_opt *o) {
    o->max_iterations = 100;
    o->loss_type = PLB_LOSS_CAUCHY;
    o->refine_intrinsics = 0;
    o->loss_scale = 1.0;
    o->gradient_tol = 1e-12;
    o->step_tol = 1e-8;
    o->relative_cost_tol = 1e-10;
    o->initial_lambda = 1e-3;
    o->min_lambda = 1e-10;
    o->max_lambda = 1e10;
}
const char *plb_last_error(void) { return g_err.c_str(); }
int plb_device_count(void) {
    int c = 0;
    if (cudaGetDeviceCount(&c) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return c;
}
int plb_set_device(int device) {
    if (device < 0) {
        g_err = "negative device index";
        return PLB_ERR_ARG;
    }
    g_device = device;
    return PLB_OK;
}
// ---- host-side pieces of the loop, callable without a device (used by the CPU test-suite) --------------------------
// robust/sampling.cc:37-61,85-136: the first `iters` samples (k indices each) of RandomSampler(n, k, opt)
int plb_host_sample_table(uint64_t n, uint32_t k, const plb_ransac_opt *opt, uint64_t iters, uint32_t *out) {
    if (!opt || !out || k == 0 || k > 16 || n < k) {
        g_err = "bad argument";
        return PLB_ERR_ARG;
    }
    Sampler smp((size_t)n, (size_t)k, *opt);
    for (uint64_t i = 0; i < iters; ++i) smp.next(out + i * k);
    return PLB_OK;
}
// robust/ransac_impl.h:51-76 (compute_dynamic_max_iter with log_prob_missing_model = log(1 - success_prob))
uint64_t plb_host_dynamic_max_iter(uint64_t num_inliers, uint64_t num_data, uint32_t sample_sz, double success_prob,
                                   double dyn_num_trials_mult, uint64_t min_iterations, uint64_t max_iterations) {
    return (uint64_t)compute_dynamic_max_iter((size_t)num_inliers, (size_t)num_data, (size_t)sample_sz,
                                              std::log(1.0 - success_prob), dyn_num_trials_mult, (size_t)min_iterations,
                                              (size_t)max_iterations);
}
// The same table drawn by the device sampler (k_sample), `round` samples per launch so that the sampler state is carried
// from launch to launch as in the engine's rounds; `count` independent samplers with seeds opt->seed + j are drawn in the
// same launches (one warp each).  out: count * iters * k indices.
int plb_device_sample_table(uint64_t n, uint32_t k, const plb_ransac_opt *opt, uint64_t iters, uint64_t round,
                            uint32_t count, uint32_t *out) {
    if (!opt || !out || k < 3 || k > 7 || n < k || count == 0 || round == 0 || n > (1u << 26) ||
        iters * (uint64_t)count > (1ull << 28)) {
        g_err = "bad argument";
        return PLB_ERR_ARG;
    }
    Engine &E = *engine();
    int rc = E.init();
    if (rc != PLB_OK) return rc;
    cudaStream_t st = E.stream;
    const int NP = (int)count;
    Sampler host(n, k, *opt);
    const size_t gsz = opt->progressive_sampling ? host.growth.size() : 0;
    if ((rc = E.h_smp.ensure(NP)) || (rc = E.smp.ensure(2 * (size_t)NP)) || (rc = E.h_growth.ensure(gsz)) ||
        (rc = E.growth.ensure(gsz)) || (rc = E.h_rp.ensure(NP)) || (rc = E.rp.ensure(NP)) ||
        (rc = E.samples.ensure((size_t)NP * round * k)))
        return rc;
    bool strict = true;
    for (size_t j = 0; j < gsz; ++j) {
        E.h_growth.p[j] = (uint64_t)host.growth[j];
        if (j >= k && !(host.growth[j] > host.growth[j - 1])) strict = false;
    }
    if (const char *e = std::getenv("PLB_PROSAC_SEQUENTIAL")) strict = strict && std::atoi(e) == 0; // test hook
    for (int i = 0; i < NP; ++i) {
        SamplerDev &D = E.h_smp.p[i];
        std::memset(&D, 0, sizeof(D));
        D.state = opt->seed + (uint64_t)i;
        D.n = (uint32_t)n;
        D.k = k;
        D.max_prosac = opt->max_prosac_iterations;
        if (opt->progressive_sampling) {
            D.growth = E.growth.p;
            D.sample_k = 1;
            D.subset_sz = k;
            D.flags = 1u | (strict ? 2u : 0u);
        }
    }
    PLB_CUDA(cudaMemcpyAsync(E.smp.p, E.h_smp.p, sizeof(SamplerDev) * NP, cudaMemcpyHostToDevice, st));
    if (gsz) PLB_CUDA(cudaMemcpyAsync(E.growth.p, E.h_growth.p, sizeof(uint64_t) * gsz, cudaMemcpyHostToDevice, st));
    int cur = 0;
    for (uint64_t done = 0; done < iters; done += round) {
        const uint64_t B = std::min<uint64_t>(round, iters - done);
        for (int i = 0; i < NP; ++i) {
            RoundProb &Q = E.h_rp.p[i];
            std::memset(&Q, 0, sizeof(Q));
            Q.pidx = i;
            Q.g0 = (int)(i * B);
            Q.B = (int)B;
        }
        PLB_CUDA(cudaMemcpyAsync(E.rp.p, E.h_rp.p, sizeof(RoundProb) * NP, cudaMemcpyHostToDevice, st));
        launch_sample(E.rp.p, NP, E.smp.p + (size_t)cur * NP, E.smp.p + (size_t)(cur ^ 1) * NP, E.samples.p, st);
        E.launches++;
        for (int i = 0; i < NP; ++i)
            PLB_CUDA(cudaMemcpyAsync(out + ((size_t)i * iters + done) * k, E.samples.p + (size_t)i * B * k,
                                     sizeof(uint32_t) * B * k, cudaMemcpyDeviceToHost, st));
        PLB_CUDA(cudaStreamSynchronize(st));
        cur ^= 1;
    }
    PLB_CUDA(cudaGetLastError());
    return PLB_OK;
}
int plb_set_mode(int mode) {
    if (mode != 0 && mode != 1) {
        g_err = "mode must be 0 (exact) or 1 (fast)";
        return PLB_ERR_ARG;
    }
    g_mode = mode;
    return PLB_OK;
}

static int check_ptrs(const void *a, const void *b, const void *opt, const void *model, size_t n) {
    if (!opt || !model || (n > 0 && (!a || !b))) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    return PLB_OK;
}

int plb_ransac_pnp(const double *x, const double *X, size_t n, const plb_ransac_opt *opt, double max_error,
                   double pose[7], char *inliers, plb_ransac_stats *stats, plb_counters *counters) {
    if (int r = check_ptrs(x, X, opt, pose, n)) return r;
    return run_ransac(KIND_PNP, x, X, n, *opt, max_error, 0, pose, inliers, stats, counters, FinalPolish());
}
int plb_ransac_relpose(const double *x1, const double *x2, size_t n, const plb_ransac_opt *opt, double max_error,
                       double pose[7], char *inliers, plb_ransac_stats *stats, plb_counters *counters) {
    if (int r = check_ptrs(x1, x2, opt, pose, n)) return r;
    return run_ransac(KIND_RELPOSE, x1, x2, n, *opt, max_error, 0, pose, inliers, stats, counters, FinalPolish());
}
// robust/ransac.cc:155-168: points in the pixel units of the two cameras, tangent Sampson error
int plb_ransac_relpose_cameras(const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                               const plb_camera *camera2, const plb_ransac_opt *opt, double max_error, double pose[7],
                               char *inliers, plb_ransac_stats *stats, plb_counters *counters) {
    if (int r = check_ptrs(x1, x2, opt, pose, n)) return r;
    CamDev c1, c2;
    if (int r = camera_dev(camera1, &c1)) return r;
    if (int r = camera_dev(camera2, &c2)) return r;
    pose[0] = 1.0; // :159-160
    for (int i = 1; i < 7; ++i) pose[i] = 0.0;
    return run_ransac(KIND_RELPOSE_TS, x1, x2, n, *opt, max_error, 0, pose, inliers, stats, counters, FinalPolish(), 2,
                      &c1, &c2, 1.0);
}
int plb_ransac_fundamental(const double *x1, const double *x2, size_t n, const plb_ransac_opt *opt, double max_error,
                           int real_focal_check, double F[9], char *inliers, plb_ransac_stats *stats,
                           plb_counters *counters) {
    if (int r = check_ptrs(x1, x2, opt, F, n)) return r;
    return run_ransac(KIND_FUND, x1, x2, n, *opt, max_error, real_focal_check, F, inliers, stats, counters,
                      FinalPolish());
}
int plb_ransac_homography(const double *x1, const double *x2, size_t n, const plb_ransac_opt *opt, double max_error,
                          double H[9], char *inliers, plb_ransac_stats *stats, plb_counters *counters) {
    if (int r = check_ptrs(x1, x2, opt, H, n)) return r;
    return run_ransac(KIND_HOMOG, x1, x2, n, *opt, max_error, 0, H, inliers, stats, counters, FinalPolish());
}

// ---- PoseLib/robust.cc estimate_* : pre-step -> Task for the group engine -> post-step -------------------------------
// One estimate_* call is prepared into a Task (points, scaled threshold, camera pre-step mode, final polish), committed,
// run and finished.  Used by the four single entry points and by plb_estimate_batch[_device].
// robust.cc:36-126 (absolute pose, no focal estimation), :242-314 (relative pose; tangent_sampson keeps the scaled pixels
// and runs the tangent-Sampson estimator with the cameras), :544-594 (fundamental), :712-757 (homography).
// The camera pre-step (Camera::unproject / unproject_with_jac of every point) and the scaling of the polish pixels run on
// the device, fused into the layout kernel, and normalize_points (F / H) in k_normalize: nothing here is O(N).
// Camera write-back of estimate_absolute_pose (robust.cc:103-123, Image*): CAM_RET_NONE the caller cannot take the camera
// (refinement flags -> PLB_ERR_ARG), CAM_RET_ALWAYS the Image* form, CAM_RET_REFINED only when parameters are refined.
// BundleOptions::refine_focal_length / refine_principal_point / refine_extra_params as a bit set
static int refine_flags(const plb_bundle_opt *b) { return b->refine_intrinsics & (CAM_REFINE_FOCAL | CAM_REFINE_PP | CAM_REFINE_EXTRA); }
enum { CAM_RET_NONE = 0, CAM_RET_ALWAYS = 1, CAM_RET_REFINED = 2 };
// Checks one call and fills its Task; nothing is written (commit_task writes what the Task asks for).
static int estimate_prepare(int kind, const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                            const plb_camera *camera2, const plb_ransac_opt *ransac, const plb_bundle_opt *bundle,
                            double max_error, int real_focal_check, int tangent_sampson, double *model, char *inliers,
                            plb_ransac_stats *stats, plb_counters *counters, Task &t,
                            plb_camera *camera_out = nullptr, int cam_ret = CAM_RET_NONE,
                            plb_camera *camera2_out = nullptr) {
    if (int r = check_ptrs(x1, x2, ransac, model, n)) return r;
    if (!bundle) {
        g_err = "null bundle options";
        return PLB_ERR_ARG;
    }
    if (kind < 0 || kind > 3) {
        g_err = "unknown problem kind";
        return PLB_ERR_ARG;
    }
    t.a = x1;
    t.b = x2;
    t.n = n;
    t.opt = *ransac;
    t.model = model;
    t.inliers = inliers;
    t.stats_out = stats;
    t.cnt_out = counters;
    FinalPolish &fp = t.polish;
    fp.enabled = true;
    fp.bundle = *bundle;
    if (kind == PLB_KIND_PNP) {
        CamDev cam;
        if (int r = camera_dev(camera1, &cam)) return r;
        fp.cam_refine = refine_flags(bundle);
        const bool refined = refines_camera(cam, fp.cam_refine);
        if (refined && cam_ret == CAM_RET_NONE) {
            g_err = "camera refinement flags need a camera to return: use plb_estimate_absolute_pose_image";
            return PLB_ERR_ARG;
        }
        const double scale = 1.0 / cam_focal(cam);
        fp.bundle.loss_scale = bundle->loss_scale * scale;
        fp.min_inliers = 3;
        if (cam.model != CAMM_NULL) { // the polish runs on pixels*scale with the rescaled camera (robust.cc:103-123)
            fp.cam[0] = cam;
            cam_rescale(fp.cam[0], scale);
            fp.scale = scale;
            if (cam_ret == CAM_RET_ALWAYS || (cam_ret == CAM_RET_REFINED && refined)) fp.cam_out[0] = camera_out;
        }
        t.kind = KIND_PNP;
        t.max_error = max_error * scale;
        t.pre_mode = cam.model != CAMM_NULL ? 1 : 0;
        t.cam_a = cam;
        return PLB_OK;
    }
    if (kind == PLB_KIND_RELPOSE) {
        CamDev c1, c2;
        if (int r = camera_dev(camera1, &c1)) return r;
        if (int r = camera_dev(camera2, &c2)) return r;
        const bool refined = tangent_sampson && (refines_camera(c1, refine_flags(bundle)) || refines_camera(c2, refine_flags(bundle)));
        if (refined && !camera2_out) {
            g_err = "NYI: camera refinement needs cameras to return: use plb_estimate_relative_pose_pair";
            return PLB_ERR_NYI;
        }
        const double scale = 0.5 * (1.0 / cam_focal(c1) + 1.0 / cam_focal(c2));
        fp.bundle.loss_scale = bundle->loss_scale * scale;
        fp.min_inliers = 5;
        t.max_error = max_error * scale;
        if (tangent_sampson) {
            cam_rescale(c1, scale);
            cam_rescale(c2, scale);
            t.reset_pose = true;
            t.kind = KIND_RELPOSE_TS;
            t.pre_mode = 2;
            t.pre_scale = scale;
            if (refined) { // the polish refines the cameras on x * scale with the rescaled cameras (robust.cc:262-282)
                fp.cam[0] = c1;
                fp.cam[1] = c2;
                fp.cam_refine = refine_flags(bundle);
                fp.scale = scale;
                fp.cam_out[0] = camera_out;
                fp.cam_out[1] = camera2_out;
            }
        } else {
            t.kind = KIND_RELPOSE;
            t.pre_mode = (c1.model != CAMM_NULL || c2.model != CAMM_NULL) ? 1 : 0;
        }
        t.cam_a = c1;
        t.cam_b = c2;
        return PLB_OK;
    }
    const size_t min_pts = (kind == PLB_KIND_FUNDAMENTAL) ? 7 : 4; // robust.cc:548-550,716-718
    if (n < min_pts) {
        t.skip = true;
        return PLB_OK;
    }
    // normalize_points(scale = true, centroid = !real_focal_check | true, shared = true) runs on the device (k_normalize);
    // the engine divides max_error and the polish loss scale by the scale it finds (robust.cc:561-564,724-727)
    const bool fund = kind == PLB_KIND_FUNDAMENTAL;
    fp.bundle.loss_scale = bundle->loss_scale;
    fp.min_inliers = min_pts;
    t.kind = fund ? KIND_FUND : KIND_HOMOG;
    t.norm_mode = (fund && real_focal_check) ? 1 : 2;
    t.max_error = max_error;
    t.rfc = fund ? real_focal_check : 0;
    return PLB_OK;
}
// The writes a prepared Task asks for before it runs (Task::skip, Task::reset_pose); none for tasks of other calls.
static void commit_task(Task &t) {
    if (t.skip) {
        if (t.stats_out) {
            plb_ransac_stats &s = *t.stats_out;
            s.refinements = s.iterations = s.num_inliers = 0;
            s.inlier_ratio = 0;
            s.model_score = std::numeric_limits<double>::max();
        }
        if (t.cnt_out) std::memset(t.cnt_out, 0, sizeof(*t.cnt_out));
    }
    if (t.reset_pose) {
        t.model[0] = 1.0;
        for (int i = 1; i < 7; ++i) t.model[i] = 0.0;
    }
}
// The post-step of a normalised F / H task after a successful run; none for other tasks.
// robust.cc:590-591: F = T2^T F T1 ; :753-754: H = T2^-1 H T1 ; both renormalised
static void finish_task(Task &t) {
    if (!t.norm_mode) return;
    HM3 T1, T2;
    norm_transforms(t.norm_out, T1, T2);
    HM3 M = (t.kind == KIND_FUND) ? hm_mul(hm_mul(hm_T(T2), hm_from_cm(t.model)), T1)
                                  : hm_mul(hm_mul(hm_inv(T2), hm_from_cm(t.model)), T1);
    const double nm = hm_norm(M);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) M.m[i][j] /= nm;
    hm_to_cm(M, t.model);
}
static int estimate_single(int kind, const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                           const plb_camera *camera2, const plb_ransac_opt *ransac, const plb_bundle_opt *bundle,
                           double max_error, int real_focal_check, int tangent_sampson, double *model, char *inliers,
                           plb_ransac_stats *stats, plb_counters *counters, plb_camera *camera_out = nullptr,
                           int cam_ret = CAM_RET_NONE, plb_camera *camera2_out = nullptr) {
    Task t;
    if (int r = estimate_prepare(kind, x1, x2, n, camera1, camera2, ransac, bundle, max_error, real_focal_check,
                                 tangent_sampson, model, inliers, stats, counters, t, camera_out, cam_ret, camera2_out))
        return r;
    commit_task(t);
    if (t.skip) return PLB_OK;
    std::vector<Task *> v{&t};
    if (int rc = run_group(t.kind, v)) return rc;
    finish_task(t);
    return PLB_OK;
}
int plb_estimate_absolute_pose(const double *points2D, const double *points3D, size_t n, const plb_ransac_opt *ransac,
                               const plb_bundle_opt *bundle, double max_error, const plb_camera *camera,
                               double pose[7], char *inliers, plb_ransac_stats *stats, plb_counters *counters) {
    return estimate_single(PLB_KIND_PNP, points2D, points3D, n, camera, nullptr, ransac, bundle, max_error, 0, 0, pose,
                           inliers, stats, counters);
}
// robust.cc:36-126 with the Image* of the reference: the camera is read, refined by the final bundle adjustment when
// bundle->refine_intrinsics selects parameters of its model, and written back.
int plb_estimate_absolute_pose_image(const double *points2D, const double *points3D, size_t n,
                                     const plb_ransac_opt *ransac, const plb_bundle_opt *bundle, double max_error,
                                     plb_camera *camera_inout, double pose[7], char *inliers, plb_ransac_stats *stats,
                                     plb_counters *counters) {
    if (!camera_inout) {
        g_err = "null camera";
        return PLB_ERR_ARG;
    }
    return estimate_single(PLB_KIND_PNP, points2D, points3D, n, camera_inout, nullptr, ransac, bundle, max_error, 0, 0,
                           pose, inliers, stats, counters, camera_inout, CAM_RET_ALWAYS);
}
int plb_estimate_relative_pose(const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                               const plb_camera *camera2, const plb_ransac_opt *ransac, const plb_bundle_opt *bundle,
                               double max_error, int tangent_sampson, double pose[7], char *inliers,
                               plb_ransac_stats *stats, plb_counters *counters) {
    return estimate_single(PLB_KIND_RELPOSE, x1, x2, n, camera1, camera2, ransac, bundle, max_error, 0, tangent_sampson,
                           pose, inliers, stats, counters);
}
// robust.cc:242-314 with the ImagePair of the reference: like plb_estimate_relative_pose, and with tangent_sampson the
// final bundle adjustment also refines the parameters bundle->refine_intrinsics selects in either camera, which are then
// written back (the one addition to the reference, which computes them and discards them).
int plb_estimate_relative_pose_pair(const double *x1, const double *x2, size_t n, plb_camera *camera1_inout,
                                    plb_camera *camera2_inout, const plb_ransac_opt *ransac,
                                    const plb_bundle_opt *bundle, double max_error, int tangent_sampson,
                                    double pose[7], char *inliers, plb_ransac_stats *stats, plb_counters *counters) {
    if (!camera1_inout || !camera2_inout) {
        g_err = "null camera";
        return PLB_ERR_ARG;
    }
    return estimate_single(PLB_KIND_RELPOSE, x1, x2, n, camera1_inout, camera2_inout, ransac, bundle, max_error, 0,
                           tangent_sampson, pose, inliers, stats, counters, camera1_inout, CAM_RET_REFINED,
                           camera2_inout);
}
int plb_estimate_fundamental(const double *x1, const double *x2, size_t n, const plb_ransac_opt *ransac,
                             const plb_bundle_opt *bundle, double max_error, int real_focal_check, double F[9],
                             char *inliers, plb_ransac_stats *stats, plb_counters *counters) {
    return estimate_single(PLB_KIND_FUNDAMENTAL, x1, x2, n, nullptr, nullptr, ransac, bundle, max_error,
                           real_focal_check, 0, F, inliers, stats, counters);
}
int plb_estimate_homography(const double *x1, const double *x2, size_t n, const plb_ransac_opt *ransac,
                            const plb_bundle_opt *bundle, double max_error, double H[9], char *inliers,
                            plb_ransac_stats *stats, plb_counters *counters) {
    return estimate_single(PLB_KIND_HOMOGRAPHY, x1, x2, n, nullptr, nullptr, ransac, bundle, max_error, 0, 0, H, inliers,
                           stats, counters);
}

// ---- robust/bundle.h refiners -------------------------------------------------------------------------------
// Every refiner has a _weighted twin that takes PoseLib's per-residual weights (n doubles, null: uniform); the
// unweighted entry point is the twin with null weights.  The weights are not checked, as in the reference: zero and
// negative values enter the sums as they are.  Each entry point is the one-problem case of plb_refine_batch.
// One refiner call, checked and turned into the Task of run_refine_group, by the rules of the single entry points:
// null options, model or camera (where the refiner takes one), or null points with n > 0 -> PLB_ERR_ARG; a camera
// outside the ten models -> PLB_ERR_NYI; PLB_REFINER_RELPOSE_CAMERAS with a non-empty refine_intrinsics selection ->
// PLB_ERR_NYI, as it cannot return the cameras.  cam1 / cam2 are read; out1 / out2 (the Image* / ImagePair* forms)
// receive the refined parameters, and only those.  Nothing is written here.
//   PLB_REFINER_BUNDLE: bundle.cc:84-92, the calibrated AbsolutePoseRefiner; the reference drops the weights.
//   PLB_REFINER_BUNDLE_IMAGE: bundle.cc:95-112, camera_refine_idx from the flags, points in the camera's pixel units.
//   PLB_REFINER_RELPOSE: bundle.cc:206-222.  PLB_REFINER_FUNDAMENTAL: :313-333.  PLB_REFINER_HOMOGRAPHY: :394-411.
//   PLB_REFINER_RELPOSE_CAMERAS: bundle.cc:237-247 with fixed intrinsics, the tangent-Sampson refiner on the
//   unproject_with_jac of both images (the layout kernel's pre-step).
//   PLB_REFINER_RELPOSE_PAIR: bundle.cc:237-256, CameraRelativePoseRefiner with the parameters the flags select in
//   either camera (shared_camera false), pixels as given; without a selection it is PLB_REFINER_RELPOSE_CAMERAS.
static int refine_prepare(int refiner, const double *a, const double *b, size_t n, const double *weights,
                          const plb_camera *cam1, const plb_camera *cam2, plb_camera *out1, plb_camera *out2,
                          const plb_bundle_opt *opt, double *model, double *bstats, Task &t) {
    if (refiner < PLB_REFINER_BUNDLE || refiner > PLB_REFINER_HOMOGRAPHY) {
        g_err = "unknown refiner";
        return PLB_ERR_ARG;
    }
    const bool image = refiner == PLB_REFINER_BUNDLE_IMAGE, pair = refiner == PLB_REFINER_RELPOSE_PAIR;
    if (!opt || !model || (image && !out1) || (pair && (!out1 || !out2)) || (n > 0 && (!a || !b))) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    static const int kinds[] = {KIND_PNP, KIND_PNP, KIND_RELPOSE, KIND_RELPOSE_TS, KIND_RELPOSE_TS, KIND_FUND, KIND_HOMOG};
    t.kind = kinds[refiner];
    t.refine = true;
    t.a = a;
    t.b = b;
    t.n = n;
    t.weights = refiner == PLB_REFINER_BUNDLE ? nullptr : weights;
    t.model = model;
    t.bstats = bstats;
    FinalPolish &fp = t.polish;
    fp.bundle = *opt;
    const int nc = image ? 1 : t.kind == KIND_RELPOSE_TS ? 2 : 0;
    const plb_camera *in[2] = {cam1, cam2};
    CamDev cams[2] = {fp.cam[0], fp.cam[1]};
    for (int i = 0; i < nc; ++i)
        if (int r = camera_dev(in[i], &cams[i])) return r;
    if (!nc) return PLB_OK;
    const int flags = (image || pair) ? refine_flags(opt) : 0;
    const bool refined = refines_camera(cams[0], refine_flags(opt)) || refines_camera(cams[1], refine_flags(opt));
    if (refiner == PLB_REFINER_RELPOSE_CAMERAS && refined) {
        g_err = "NYI: camera refinement needs cameras to return: use plb_refine_relpose_pair";
        return PLB_ERR_NYI;
    }
    if (t.kind == KIND_RELPOSE_TS) { // the cameras of the pre-step
        t.cam_a = cams[0];
        t.cam_b = cams[1];
    }
    // the bundle evaluates the cameras: PnP always, tangent Sampson only to refine them (else ts carries them)
    if (image || refined) std::copy(cams, cams + nc, fp.cam);
    fp.cam_refine = flags;
    fp.cam_out[0] = out1;
    fp.cam_out[1] = out2;
    return PLB_OK;
}
static int refine_single(int refiner, const double *a, const double *b, size_t n, const double *weights,
                         const plb_camera *cam1, const plb_camera *cam2, plb_camera *out1, plb_camera *out2,
                         const plb_bundle_opt *opt, double *model, double *bstats) {
    Task t;
    if (int r = refine_prepare(refiner, a, b, n, weights, cam1, cam2, out1, out2, opt, model, bstats, t)) return r;
    std::vector<Task *> v{&t};
    return run_refine_group(t.kind, v);
}
int plb_bundle_adjust(const double *x, const double *X, size_t n, double pose[7], const plb_bundle_opt *opt,
                      double bs[3]) {
    return refine_single(PLB_REFINER_BUNDLE, x, X, n, nullptr, nullptr, nullptr, nullptr, nullptr, opt, pose, bs);
}
int plb_refine_relpose(const double *x1, const double *x2, size_t n, double pose[7], const plb_bundle_opt *opt,
                       double bs[3]) {
    return plb_refine_relpose_weighted(x1, x2, n, pose, opt, bs, nullptr);
}
int plb_refine_relpose_weighted(const double *x1, const double *x2, size_t n, double pose[7], const plb_bundle_opt *opt,
                                double bs[3], const double *weights) {
    return refine_single(PLB_REFINER_RELPOSE, x1, x2, n, weights, nullptr, nullptr, nullptr, nullptr, opt, pose, bs);
}
int plb_refine_relpose_cameras(const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                               const plb_camera *camera2, double pose[7], const plb_bundle_opt *opt, double bs[3]) {
    return plb_refine_relpose_cameras_weighted(x1, x2, n, camera1, camera2, pose, opt, bs, nullptr);
}
int plb_refine_relpose_cameras_weighted(const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                                        const plb_camera *camera2, double pose[7], const plb_bundle_opt *opt,
                                        double bs[3], const double *weights) {
    return refine_single(PLB_REFINER_RELPOSE_CAMERAS, x1, x2, n, weights, camera1, camera2, nullptr, nullptr, opt, pose, bs);
}
int plb_bundle_adjust_image(const double *x, const double *X, size_t n, double pose[7], plb_camera *camera_inout,
                            const plb_bundle_opt *opt, double bs[3]) {
    return plb_bundle_adjust_image_weighted(x, X, n, pose, camera_inout, opt, bs, nullptr);
}
int plb_bundle_adjust_image_weighted(const double *x, const double *X, size_t n, double pose[7],
                                     plb_camera *camera_inout, const plb_bundle_opt *opt, double bs[3],
                                     const double *weights) {
    return refine_single(PLB_REFINER_BUNDLE_IMAGE, x, X, n, weights, camera_inout, nullptr, camera_inout, nullptr, opt,
                         pose, bs);
}
int plb_refine_relpose_pair(const double *x1, const double *x2, size_t n, plb_camera *camera1_inout,
                            plb_camera *camera2_inout, double pose[7], const plb_bundle_opt *opt, double bs[3]) {
    return plb_refine_relpose_pair_weighted(x1, x2, n, camera1_inout, camera2_inout, pose, opt, bs, nullptr);
}
int plb_refine_relpose_pair_weighted(const double *x1, const double *x2, size_t n, plb_camera *camera1_inout,
                                     plb_camera *camera2_inout, double pose[7], const plb_bundle_opt *opt, double bs[3],
                                     const double *weights) {
    return refine_single(PLB_REFINER_RELPOSE_PAIR, x1, x2, n, weights, camera1_inout, camera2_inout, camera1_inout,
                         camera2_inout, opt, pose, bs);
}
int plb_refine_fundamental(const double *x1, const double *x2, size_t n, double F[9], const plb_bundle_opt *opt,
                           double bs[3]) {
    return plb_refine_fundamental_weighted(x1, x2, n, F, opt, bs, nullptr);
}
int plb_refine_fundamental_weighted(const double *x1, const double *x2, size_t n, double F[9],
                                    const plb_bundle_opt *opt, double bs[3], const double *weights) {
    return refine_single(PLB_REFINER_FUNDAMENTAL, x1, x2, n, weights, nullptr, nullptr, nullptr, nullptr, opt, F, bs);
}
int plb_refine_homography(const double *x1, const double *x2, size_t n, double H[9], const plb_bundle_opt *opt,
                          double bs[3]) {
    return plb_refine_homography_weighted(x1, x2, n, H, opt, bs, nullptr);
}
int plb_refine_homography_weighted(const double *x1, const double *x2, size_t n, double H[9],
                                   const plb_bundle_opt *opt, double bs[3], const double *weights) {
    return refine_single(PLB_REFINER_HOMOGRAPHY, x1, x2, n, weights, nullptr, nullptr, nullptr, nullptr, opt, H, bs);
}

// ---- solvers ------------------------------------------------------------------------------------------------
static int solver_batch(int kind, int variant, size_t count, const double *a, size_t a_sz, const double *b,
                        size_t b_sz, double *out, size_t out_sz, int32_t *n_out, int flags) {
    if (count == 0) return PLB_OK;
    if (!a || !b || !out || !n_out) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    Engine &E = *engine();
    int rc = E.init();
    if (rc != PLB_OK) return rc;
    DevBuf<double> da, db, dout, s5_blk, s5_park, s5_cpoly, s5_roots;
    DevBuf<int> dn, s5_nroots;
    if ((rc = da.ensure(count * a_sz)) || (rc = db.ensure(count * b_sz)) || (rc = dout.ensure(count * out_sz)) ||
        (rc = dn.ensure(count)))
        return rc;
    HypOut s5{};
    if (kind == KIND_RELPOSE) { // phase buffers of the 5-point solver, laid out as in a round of `count` samples
        if ((rc = s5_blk.ensure(count * 105)) || (rc = s5_park.ensure(count * 100)) || (rc = s5_cpoly.ensure(count * 11)) ||
            (rc = s5_roots.ensure(count * 10)) || (rc = s5_nroots.ensure(count)))
            return rc;
        s5.s5_blk = s5_blk.p;
        s5.s5_park = s5_park.p;
        s5.s5_cpoly = s5_cpoly.p;
        s5.s5_roots = s5_roots.p;
        s5.s5_nroots = s5_nroots.p;
    }
    PLB_CUDA(cudaMemcpyAsync(da.p, a, sizeof(double) * count * a_sz, cudaMemcpyHostToDevice, E.stream));
    PLB_CUDA(cudaMemcpyAsync(db.p, b, sizeof(double) * count * b_sz, cudaMemcpyHostToDevice, E.stream));
    E.launches += launch_solver_batch(kind, variant, count, da.p, db.p, dout.p, dn.p, flags, s5, E.stream);
    PLB_CUDA(cudaMemcpyAsync(out, dout.p, sizeof(double) * count * out_sz, cudaMemcpyDeviceToHost, E.stream));
    PLB_CUDA(cudaMemcpyAsync(n_out, dn.p, sizeof(int) * count, cudaMemcpyDeviceToHost, E.stream));
    PLB_CUDA(cudaStreamSynchronize(E.stream));
    PLB_CUDA(cudaGetLastError());
    return PLB_OK;
}
int plb_p3p_batch(size_t count, const double *x, const double *X, double *poses_out, int32_t *n_out) {
    return solver_batch(KIND_PNP, 0, count, x, 9, X, 9, poses_out, 28, n_out, 0);
}
int plb_p3p_lambdatwist_batch(size_t count, const double *x, const double *X, double *poses_out, int32_t *n_out) {
    return solver_batch(KIND_PNP, 1, count, x, 9, X, 9, poses_out, 28, n_out, 0);
}
int plb_relpose_5pt_batch(size_t count, const double *x1, const double *x2, double *E_out, int32_t *n_out) {
    return solver_batch(KIND_RELPOSE, 0, count, x1, 15, x2, 15, E_out, 90, n_out, 0);
}
int plb_relpose_5pt_poses_batch(size_t count, const double *x1, const double *x2, double *poses_out, int32_t *n_out) {
    return solver_batch(KIND_RELPOSE, 1, count, x1, 15, x2, 15, poses_out, 280, n_out, 0);
}
int plb_relpose_7pt_batch(size_t count, const double *x1, const double *x2, double *F_out, int32_t *n_out) {
    return solver_batch(KIND_FUND, 0, count, x1, 21, x2, 21, F_out, 27, n_out, 0);
}
int plb_homography_4pt_batch(size_t count, const double *x1, const double *x2, double *H_out, int32_t *n_out,
                             int check_cheirality) {
    return solver_batch(KIND_HOMOG, 0, count, x1, 12, x2, 12, H_out, 9, n_out, check_cheirality);
}

// solvers/relpose_8pt.h:45-53: `count` instances of n >= 8 unit bearing pairs; E_out count x 9 (column-major) or
// poses_out count x 4 x 7 + n_out
static int eightpt_batch(size_t count, size_t n, const double *x1, const double *x2, int want_poses, double *E_out,
                         double *poses_out, int32_t *n_out) {
    if (count == 0) return PLB_OK;
    if (!x1 || !x2 || n < 8 || n > (1u << 24) || (want_poses ? (!poses_out || !n_out) : !E_out)) {
        g_err = "bad argument";
        return PLB_ERR_ARG;
    }
    Engine &E = *engine();
    int rc = E.init();
    if (rc != PLB_OK) return rc;
    DevBuf<double> da, db, dout;
    DevBuf<int> dn;
    const size_t out_sz = want_poses ? 28 : 9;
    if ((rc = da.ensure(count * n * 3)) || (rc = db.ensure(count * n * 3)) || (rc = dout.ensure(count * out_sz)) ||
        (rc = dn.ensure(count)))
        return rc;
    PLB_CUDA(cudaMemcpyAsync(da.p, x1, sizeof(double) * count * n * 3, cudaMemcpyHostToDevice, E.stream));
    PLB_CUDA(cudaMemcpyAsync(db.p, x2, sizeof(double) * count * n * 3, cudaMemcpyHostToDevice, E.stream));
    PLB_CUDA(cudaMemsetAsync(dout.p, 0, sizeof(double) * count * out_sz, E.stream));
    launch_eightpt(count, (int)n, da.p, db.p, want_poses, dout.p, dout.p, dn.p, E.stream);
    E.launches++;
    PLB_CUDA(cudaMemcpyAsync(want_poses ? poses_out : E_out, dout.p, sizeof(double) * count * out_sz, cudaMemcpyDeviceToHost, E.stream));
    if (want_poses) PLB_CUDA(cudaMemcpyAsync(n_out, dn.p, sizeof(int) * count, cudaMemcpyDeviceToHost, E.stream));
    PLB_CUDA(cudaStreamSynchronize(E.stream));
    PLB_CUDA(cudaGetLastError());
    return PLB_OK;
}
int plb_essential_matrix_8pt_batch(size_t count, size_t n, const double *x1, const double *x2, double *E_out) {
    return eightpt_batch(count, n, x1, x2, 0, E_out, nullptr, nullptr);
}
int plb_relpose_8pt_batch(size_t count, size_t n, const double *x1, const double *x2, double *poses_out, int32_t *n_out) {
    return eightpt_batch(count, n, x1, x2, 1, nullptr, poses_out, n_out);
}

// ---- batch of problems: `streams` lock-step groups in flight per device, each on its own engine / stream ----------
// Problems of the same kind run in lock-step groups (one chain of launches per round for the whole group); the groups of
// a device are spread over `streams` persistent worker threads.  devices[0..n_dev): the CUDA devices to use; problems
// are assigned to devices by longest-processing-time-first on (correspondences x expected iterations), problems whose
// correspondences are resident stay on the device that holds them.
static double task_cost(const Task &t) {
    if (t.refine) return (double)std::max<size_t>(t.n, 1) * (double)std::max<uint64_t>(t.polish.bundle.max_iterations, 1);
    if (t.score) return (double)std::max<size_t>(t.n, 1) * (double)std::max<size_t>(t.m, 1);
    if (t.generate) return (double)std::max<size_t>(t.n, 1) * (double)std::max<size_t>(t.s, 1) * kind_max_models(t.kind);
    if (t.camop) return (double)std::max<size_t>(t.n, 1);
    static const double its[5] = {4.0 * 1000, 0.5 * 14000, 2.0 * 30000, 1.0 * 1000, 0.5 * 14000}; // models x iterations, typical
    const double cap = (double)std::max<uint64_t>(t.opt.max_iterations, 1) * 4.0;
    return (double)std::max<size_t>(t.n, 1) * std::min(its[t.kind], cap);
}
// Runs prepared tasks: dev_of[i] >= 0 pins task i to that device (resident inputs), -1 lets the partition place it.
// Returns the first error; *err_msg receives its text.
static int run_tasks(std::vector<Task> &tasks, std::vector<int> &dev_of, const int *devices, int n_dev, int streams) {
    const size_t count = tasks.size();
    // device assignment: LPT over the tasks that are free to move
    {
        std::vector<double> load(n_dev, 0.0);
        std::vector<size_t> order;
        for (size_t i = 0; i < count; ++i) {
            if (dev_of[i] >= 0) {
                for (int d = 0; d < n_dev; ++d)
                    if (devices[d] == dev_of[i]) load[d] += task_cost(tasks[i]);
            } else {
                order.push_back(i);
            }
        }
        if (n_dev == 1) {
            for (size_t i : order) dev_of[i] = devices[0];
        } else {
            std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) { return task_cost(tasks[x]) > task_cost(tasks[y]); });
            for (size_t i : order) {
                int best = 0;
                for (int d = 1; d < n_dev; ++d)
                    if (load[d] < load[best]) best = d;
                dev_of[i] = devices[best];
                load[best] += task_cost(tasks[i]);
            }
        }
    }
    // groups per device: tasks of the same engine kind run in lock-step (refiner tasks: in one LM phase); camera tasks
    // form groups of one op, with or without Jacobians (one kernel instantiation each)
    auto group_key = [](const Task &t) {
        return t.camop ? KIND_RELPOSE_TS + 1 + 2 * t.cam_op + (t.cam_jac || t.cam_jac_params ? 1 : 0) : t.kind;
    };
    const int nthreads_req = std::max(1, streams);
    struct Job {
        int device;
        std::vector<std::vector<Task *>> groups;
    };
    std::vector<Job> jobs; // one per (device, worker)
    for (int d = 0; d < n_dev; ++d) {
        std::vector<std::vector<Task *>> groups;
        for (int key = 0; key <= KIND_RELPOSE_TS + 2 * CAMOP_UNPROJECT_2D + 2; ++key) {
            std::vector<Task *> of_kind;
            for (size_t i = 0; i < count; ++i)
                if (group_key(tasks[i]) == key && dev_of[i] == devices[d] && !tasks[i].skip) of_kind.push_back(&tasks[i]);
            if (of_kind.empty()) continue;
            const size_t gsz = std::min<size_t>(256, std::max<size_t>(1, (of_kind.size() + nthreads_req - 1) / nthreads_req));
            for (size_t o = 0; o < of_kind.size(); o += gsz)
                groups.emplace_back(of_kind.begin() + o, of_kind.begin() + std::min(of_kind.size(), o + gsz));
        }
        const int nthreads = std::max(1, std::min<int>(nthreads_req, (int)groups.size()));
        for (int t = 0; t < nthreads; ++t) {
            Job j;
            j.device = devices[d];
            for (size_t gi = (size_t)t; gi < groups.size(); gi += (size_t)nthreads) j.groups.push_back(groups[gi]);
            if (!j.groups.empty()) jobs.push_back(std::move(j));
        }
    }
    if (jobs.empty()) return PLB_OK;
    std::atomic<int> first_err(PLB_OK);
    std::string err_msg;
    std::mutex mtx;
    const int mode = current_mode();
    const bool oversubscribed = (int)jobs.size() > usable_cpus();
    auto work = [&](int w) {
        const int saved_dev = g_device, saved_mode = g_mode;
        const bool saved_block = t_blocking_sync, saved_worker = t_batch_worker;
        g_device = jobs[w].device;
        g_mode = mode;
        t_blocking_sync = oversubscribed;
        t_batch_worker = jobs.size() > 1;
        for (auto &grp : jobs[w].groups) {
            const int rc = grp[0]->refine     ? run_refine_group(grp[0]->kind, grp)
                           : grp[0]->score    ? run_score_group(grp[0]->kind, grp)
                           : grp[0]->generate ? run_generate_group(grp[0]->kind, grp)
                           : grp[0]->camop    ? run_camera_group(grp)
                                              : run_group(grp[0]->kind, grp);
            if (rc != PLB_OK) {
                int exp = PLB_OK;
                if (first_err.compare_exchange_strong(exp, rc)) {
                    std::lock_guard<std::mutex> lk(mtx);
                    err_msg = g_err;
                }
            }
        }
        g_device = saved_dev;
        g_mode = saved_mode;
        t_blocking_sync = saved_block;
        t_batch_worker = saved_worker;
    };
    if (jobs.size() == 1) work(0); // the caller's own thread and engine
    else worker_pool().run((int)jobs.size(), work);
    if (first_err.load() != PLB_OK) g_err = err_msg;
    return first_err.load();
}
// ---- the batch entry points -----------------------------------------------------------------------------------------
// Each family turns one problem into its Task with a prepare function that checks the problem by its single call's rules
// and writes nothing; run_batch below does everything else.

// ransac_* of one plb_problem, on its points or on resident correspondences, whose handle the Task holds for the call.
static int ransac_prepare(plb_problem &p, Task &t) {
    if (p.kind < 0 || p.kind > 3) {
        g_err = "unknown problem kind";
        return PLB_ERR_ARG;
    }
    t.kind = p.kind;
    t.a = p.a;
    t.b = p.b;
    t.n = (size_t)p.n;
    t.opt = p.opt;
    t.max_error = p.max_error;
    t.rfc = p.real_focal_check;
    t.model = p.model;
    t.inliers = p.inliers;
    t.stats_out = &p.stats;
    t.cnt_out = &p.counters;
    if (p.resident > 0) {
        {
            std::lock_guard<std::mutex> lk(g_res_mtx);
            if ((size_t)p.resident <= g_resident.size()) t.res = g_resident[p.resident - 1];
        }
        if (!t.res || t.res->kind != p.kind) {
            g_err = "invalid resident handle";
            return PLB_ERR_ARG;
        }
        t.n = (size_t)t.res->n;
    } else if (t.n > 0 && (!p.a || !p.b)) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    return PLB_OK;
}
// estimate_* of one plb_estimate_problem: camera1 receives the refined camera of a PnP problem; relative pose returns
// no cameras, so tangent-Sampson camera refinement is PLB_ERR_NYI.
static int estimate_problem_prepare(plb_estimate_problem &p, Task &t) {
    return estimate_prepare(p.kind, p.a, p.b, (size_t)p.n, &p.camera1, &p.camera2, &p.ransac, &p.bundle, p.max_error,
                            p.real_focal_check, p.tangent_sampson, p.model, p.inliers, &p.stats, &p.counters, t,
                            &p.camera1, CAM_RET_REFINED);
}
static int refine_problem_prepare(plb_refine_problem &p, Task &t) {
    return refine_prepare(p.refiner, p.a, p.b, (size_t)p.n, p.weights, &p.camera1, &p.camera2, &p.camera1, &p.camera2,
                          &p.bundle, p.model, p.bundle_stats, t);
}

// ---- given models: the robust/utils.h scorers and get_inliers (plb_score_batch) ------------------------------------
// One problem checked and turned into the Task of run_score_group: sq_thr is the caller's squared threshold, no
// normalisation and no threshold scaling (the ransac_* level); tangent Sampson unprojects the pixels with the cameras as
// ransac_relpose(x1, x2, camera1, camera2) does (ransac.cc:155-168).  Nothing is written here.
static int score_prepare(const plb_score_problem &p, Task &t) {
    if (p.kind < PLB_KIND_PNP || p.kind > PLB_KIND_HOMOGRAPHY) {
        g_err = "unknown problem kind";
        return PLB_ERR_ARG;
    }
    if (p.tangent_sampson && p.kind != PLB_KIND_RELPOSE) {
        g_err = "tangent_sampson is a relative-pose option";
        return PLB_ERR_ARG;
    }
    if ((p.n > 0 && (!p.a || !p.b)) || (p.m > 0 && (!p.models || !p.scores || !p.num_inliers))) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    if (!std::isfinite(p.sq_threshold)) {
        g_err = "sq_threshold must be finite";
        return PLB_ERR_ARG;
    }
    uint64_t mn = 0;
    if (p.m >= (1ull << 31) || __builtin_mul_overflow(p.m, p.n, &mn) || mn > SIZE_MAX) {
        g_err = "too many models";
        return PLB_ERR_ARG;
    }
    if (p.n > (1u << 26)) {
        g_err = "too many correspondences";
        return PLB_ERR_ARG;
    }
    t.kind = p.kind == PLB_KIND_PNP ? KIND_PNP : p.kind == PLB_KIND_RELPOSE ? KIND_RELPOSE
                                              : p.kind == PLB_KIND_FUNDAMENTAL ? KIND_FUND : KIND_HOMOG;
    if (p.tangent_sampson) {
        if (int r = camera_dev(&p.camera1, &t.cam_a)) return r;
        if (int r = camera_dev(&p.camera2, &t.cam_b)) return r;
        t.kind = KIND_RELPOSE_TS;
        t.pre_mode = 2;
    }
    t.score = true;
    t.a = p.a;
    t.b = p.b;
    t.n = (size_t)p.n;
    t.m = (size_t)p.m;
    t.models = p.models;
    t.sq_thr = p.sq_threshold;
    t.scores = p.scores;
    t.counts = p.num_inliers;
    t.inliers = p.m > 0 && p.n > 0 ? p.inliers : nullptr;
    return PLB_OK;
}

// ---- caller-drawn samples: the estimators' generate_models + score_model (plb_generate_batch) ------------------------
// One problem checked and turned into the Task of run_generate_group, at the ransac_* level as score_prepare; the
// sample indices are left to the caller of this function (host form: generate_host_prepare; device form: the device
// check of run_batch).  Nothing is written here.
static int generate_prepare(const plb_generate_problem &p, Task &t) {
    if (p.kind < PLB_KIND_PNP || p.kind > PLB_KIND_HOMOGRAPHY) {
        g_err = "unknown problem kind";
        return PLB_ERR_ARG;
    }
    if (p.tangent_sampson && p.kind != PLB_KIND_RELPOSE) {
        g_err = "tangent_sampson is a relative-pose option";
        return PLB_ERR_ARG;
    }
    if (p.real_focal_check && p.kind != PLB_KIND_FUNDAMENTAL) {
        g_err = "real_focal_check is a fundamental-matrix option";
        return PLB_ERR_ARG;
    }
    if ((p.n > 0 && (!p.a || !p.b)) ||
        (p.s > 0 && (!p.samples || !p.n_models || !p.models || !p.scores || !p.num_inliers))) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    if (!std::isfinite(p.sq_threshold)) {
        g_err = "sq_threshold must be finite";
        return PLB_ERR_ARG;
    }
    int kind = p.kind == PLB_KIND_PNP ? KIND_PNP : p.kind == PLB_KIND_RELPOSE ? KIND_RELPOSE
                                      : p.kind == PLB_KIND_FUNDAMENTAL ? KIND_FUND : KIND_HOMOG;
    uint64_t sm = 0;
    if (p.s >= (1ull << 31) || __builtin_mul_overflow(p.s, (uint64_t)kind_max_models(kind) * kind_model_size(kind), &sm) ||
        sm > SIZE_MAX / sizeof(double)) {
        g_err = "too many samples";
        return PLB_ERR_ARG;
    }
    if (p.n > (1u << 26)) {
        g_err = "too many correspondences";
        return PLB_ERR_ARG;
    }
    if (p.tangent_sampson) {
        if (int r = camera_dev(&p.camera1, &t.cam_a)) return r;
        if (int r = camera_dev(&p.camera2, &t.cam_b)) return r;
        kind = KIND_RELPOSE_TS;
        t.pre_mode = 2;
    }
    t.kind = kind;
    t.generate = true;
    t.rfc = p.real_focal_check ? 1 : 0;
    t.a = p.a;
    t.b = p.b;
    t.n = (size_t)p.n;
    t.s = (size_t)p.s;
    t.samples = p.samples;
    t.sq_thr = p.sq_threshold;
    t.n_models = p.n_models;
    t.gen_models = p.models;
    t.scores = p.scores;
    t.counts = p.num_inliers;
    return PLB_OK;
}
// The host form: every index of the host table in [0, n), checked before any device call.
static int generate_host_prepare(plb_generate_problem &p, Task &t) {
    if (int r = generate_prepare(p, t)) return r;
    const size_t cnt = t.s * (size_t)kind_sample_size(t.kind);
    for (size_t i = 0; i < cnt; ++i)
        if (t.samples[i] < 0 || (uint64_t)t.samples[i] >= p.n) {
            g_err = "sample index outside [0, n)";
            return PLB_ERR_ARG;
        }
    return PLB_OK;
}
static int generate_device_prepare(plb_generate_problem &p, Task &t) { return generate_prepare(p, t); }

// ---- the camera functions over many points (plb_camera_batch) -----------------------------------------------------
// One problem checked and turned into the Task of run_camera_group: the argument errors first, then the camera (NYI).
// Nothing is written here.
static int camera_prepare(plb_camera_problem &p, Task &t) {
    if (p.op < PLB_CAMOP_PROJECT || p.op > PLB_CAMOP_UNPROJECT_2D) {
        g_err = "unknown camera op";
        return PLB_ERR_ARG;
    }
    if (p.n > 0 && (!p.in || !p.out)) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    if (p.op == PLB_CAMOP_UNPROJECT_2D && (p.jac || p.jac_params)) {
        g_err = "the 2D unproject has no Jacobians";
        return PLB_ERR_ARG;
    }
    const uint64_t rows = p.op == PLB_CAMOP_PROJECT ? 2 : 3;
    uint64_t widest = p.op == PLB_CAMOP_UNPROJECT_2D ? 2 : 3, bytes = 0; // in and out
    if (p.jac) widest = std::max<uint64_t>(widest, 6);
    if (p.jac_params) widest = std::max<uint64_t>(widest, rows * cam_num_params(p.camera.model_id));
    if (__builtin_mul_overflow(p.n, widest * sizeof(double), &bytes) || bytes > SIZE_MAX) {
        g_err = "too many points";
        return PLB_ERR_ARG;
    }
    if (int r = camera_dev(&p.camera, &t.cam_a)) return r;
    t.camop = true;
    t.cam_op = p.op == PLB_CAMOP_PROJECT ? CAMOP_PROJECT : p.op == PLB_CAMOP_UNPROJECT ? CAMOP_UNPROJECT : CAMOP_UNPROJECT_2D;
    t.a = p.in;
    t.n = (size_t)p.n;
    t.cam_out = p.out;
    t.cam_jac = p.jac;
    t.cam_jac_params = p.jac_params;
    return PLB_OK;
}

// Step 9 of the device forms: every sample index of the generate tasks in [0, n), by one reduction kernel over all of
// them, after the work queued on the caller's stream (E.ev_in), and one synchronisation.  The kernels that gather with
// the indices run only after this has passed.
static int check_device_samples(const std::vector<Task> &tasks, Engine &E) {
    int nd = 0;
    for (const Task &t : tasks) nd += t.generate && t.s > 0;
    if (!nd) return PLB_OK;
    int rc;
    if ((rc = E.tkdesc.ensure(nd)) || (rc = E.h_tkdesc.ensure(nd)) || (rc = E.work.ensure(CTL_WORDS))) return rc;
    long long max_count = 0;
    int j = 0;
    for (const Task &t : tasks)
        if (t.generate && t.s > 0) {
            E.h_tkdesc.p[j++] = {t.samples, nullptr, (long long)(t.s * kind_sample_size(t.kind)), (int)t.n, 0};
            max_count = std::max(max_count, E.h_tkdesc.p[j - 1].count);
        }
    PLB_CUDA(cudaMemcpyAsync(E.tkdesc.p, E.h_tkdesc.p, sizeof(TakeDesc) * nd, cudaMemcpyHostToDevice, E.stream));
    PLB_CUDA(cudaMemsetAsync(E.work.p, 0, sizeof(int), E.stream));
    PLB_CUDA(cudaStreamWaitEvent(E.stream, E.ev_in, 0));
    launch_take_samples(E.tkdesc.p, nd, max_count, E.work.p, E.stream);
    PLB_CUDA(cudaMemcpyAsync(E.h_work.p, E.work.p, sizeof(int), cudaMemcpyDeviceToHost, E.stream));
    PLB_CUDA(cudaStreamSynchronize(E.stream));
    PLB_CUDA(cudaGetLastError());
    if (E.h_work.p[0]) {
        g_err = "sample index outside [0, n)";
        return PLB_ERR_ARG;
    }
    return PLB_OK;
}

// What is wrong with the memory of a device-form task, or null.  Sized by n (n > 0): a, b and the weights, when given,
// must be device (or managed) memory of `device` aligned to the dtype's `elem` bytes; sized by m (m > 0): models, scores
// and counts, 8-byte aligned; the inliers the task writes must be device memory; sized by s (s > 0, generate tasks):
// samples and n_models 4-byte, models, scores and counts 8-byte aligned.  Camera tasks (n > 0): in aligned to the dtype,
// out and the Jacobians given 8-byte aligned.
static const char *device_io_error(const Task &t, int device, size_t elem) {
    if (t.camop) {
        if (t.n == 0) return nullptr;
        if (!device_memory(t.a, device)) return "in must be device memory of the current device";
        if ((uintptr_t)t.a % elem) return "in is not aligned to the dtype";
        for (const void *q : {(const void *)t.cam_out, (const void *)t.cam_jac, (const void *)t.cam_jac_params}) {
            if (!q) continue; // only the Jacobians may be null
            if (!device_memory(q, device)) return "out / jac / jac_params must be device memory of the current device";
            if ((uintptr_t)q % sizeof(double)) return "out / jac / jac_params are not 8-byte aligned";
        }
        return nullptr;
    }
    if (t.n > 0)
        for (const void *q : {(const void *)t.a, (const void *)t.b, t.weights}) {
            if (!q) continue; // only the weights may be null
            if (!device_memory(q, device)) return "a / b / weights must be device memory of the current device";
            if ((uintptr_t)q % elem) return "a / b / weights are not aligned to the dtype";
        }
    if (t.m > 0)
        for (const void *q : {(const void *)t.models, (const void *)t.scores, (const void *)t.counts}) {
            if (!device_memory(q, device))
                return "models / scores / num_inliers must be device memory of the current device";
            if ((uintptr_t)q % sizeof(double)) return "models / scores / num_inliers are not 8-byte aligned";
        }
    if (t.n > 0 && t.inliers && !device_memory(t.inliers, device))
        return "inliers must be NULL or device memory of the current device";
    if (t.generate && t.s > 0) {
        for (const void *q : {(const void *)t.samples, (const void *)t.n_models}) {
            if (!device_memory(q, device)) return "samples / n_models must be device memory of the current device";
            if ((uintptr_t)q % sizeof(int32_t)) return "samples / n_models are not 4-byte aligned";
        }
        for (const void *q : {(const void *)t.gen_models, (const void *)t.scores, (const void *)t.counts}) {
            if (!device_memory(q, device)) return "models / scores / num_inliers must be device memory of the current device";
            if ((uintptr_t)q % sizeof(double)) return "models / scores / num_inliers are not 8-byte aligned";
        }
    }
    return nullptr;
}

// Every batch entry point, in the order include/poselib_b200.h states: count 0 -> PLB_OK and problems NULL ->
// PLB_ERR_ARG, writing nothing; then each failure writes its code into every status and nothing else:
//   an unknown dtype (device forms); prepare() of each problem in order, the first failure's code; n_gpus < min_gpus;
//   no device (PLB_ERR_CUDA); n_gpus above the device count; resident correspondences on a device the call does not
//   use; device forms: device_io_error of each task, then the sample indices of the generate tasks on the device.
// Then the caller's stream gets the event the groups wait on (device forms), the tasks' writes are committed, the tasks
// run, every status gets the result, and on success every task gets its post-step.
// n_gpus: -1 the calling thread's device, 0 every device of the process, k the first k.  dtype: PLB_DTYPE_* of a device
// form, whose inputs and outputs are memory of the calling thread's device (n_gpus -1); HOST_IO for the host forms.
enum { HOST_IO = -1 };
} // extern "C": a template has C++ linkage
template <typename P, typename Prepare>
static int run_batch(P *problems, size_t count, Prepare prepare, int n_gpus, int min_gpus, int streams,
                     int dtype = HOST_IO, void *stream = nullptr) {
    if (count == 0) return PLB_OK;
    if (!problems) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    auto fail_all = [&](int rc, const std::string &msg) {
        g_err = msg;
        for (size_t j = 0; j < count; ++j) problems[j].status = rc;
        return rc;
    };
    const bool dev_io = dtype != HOST_IO;
    if (dev_io && dtype != PLB_DTYPE_F64 && dtype != PLB_DTYPE_F32) return fail_all(PLB_ERR_ARG, "unknown dtype");
    std::vector<Task> tasks(count);
    for (size_t i = 0; i < count; ++i)
        if (int r = prepare(problems[i], tasks[i])) return fail_all(r, g_err);
    if (n_gpus < min_gpus) return fail_all(PLB_ERR_ARG, "n_gpus out of range");
    const int have = plb_device_count();
    if (have == 0) return fail_all(PLB_ERR_CUDA, "no usable CUDA device");
    if (n_gpus > have) return fail_all(PLB_ERR_ARG, "n_gpus out of range");
    std::vector<int> devs;
    if (n_gpus == -1) devs.push_back(g_device);
    else
        for (int d = 0; d < (n_gpus == 0 ? have : n_gpus); ++d) devs.push_back(d);
    Engine *E = dev_io ? engine() : nullptr;
    if (E)
        if (int rc = E->init()) return fail_all(rc, g_err);
    const size_t elem = dtype == PLB_DTYPE_F32 ? sizeof(float) : sizeof(double);
    std::vector<int> dev_of(count, -1); // resident inputs stay on the device that holds them
    for (size_t i = 0; i < count; ++i) {
        const Task &t = tasks[i];
        if (t.res) {
            if (std::find(devs.begin(), devs.end(), t.res->device) == devs.end())
                return fail_all(PLB_ERR_ARG, "resident correspondences live on a device this call does not use");
            dev_of[i] = t.res->device;
        }
        if (const char *what = E ? device_io_error(t, E->device, elem) : nullptr)
            return fail_all(PLB_ERR_ARG, "problem " + std::to_string(i) + ": " + what);
    }
    if (E) {
        cudaError_t e = cudaEventRecord(E->ev_in, (cudaStream_t)stream);
        if (e != cudaSuccess)
            return fail_all(PLB_ERR_CUDA, std::string("cudaEventRecord on the caller's stream: ") + cudaGetErrorString(e));
        for (Task &t : tasks) {
            t.dev_io = true;
            t.f32 = dtype == PLB_DTYPE_F32;
            t.ready = E->ev_in;
        }
        if (int rc = check_device_samples(tasks, *E)) return fail_all(rc, g_err);
    }
    for (Task &t : tasks) commit_task(t);
    const int rc = run_tasks(tasks, dev_of, devs.data(), (int)devs.size(), streams);
    for (size_t i = 0; i < count; ++i) {
        problems[i].status = rc;
        if (rc == PLB_OK) finish_task(tasks[i]);
    }
    return rc;
}
extern "C" {

int plb_ransac_batch(plb_problem *problems, size_t count, int streams) {
    return run_batch(problems, count, ransac_prepare, -1, -1, streams);
}
// The same over the first n_gpus CUDA devices of this process (0 = all): in-process multi-GPU, no collective — image
// pairs are independent (robust/ransac.cc:144-148 builds one estimator per call).  Results (stats, models, inlier
// masks) land in the caller's plb_problem array exactly as with plb_ransac_batch.
int plb_ransac_batch_multi(plb_problem *problems, size_t count, int n_gpus, int streams_per_gpu) {
    return run_batch(problems, count, ransac_prepare, n_gpus, 0, streams_per_gpu);
}
// Batch form of the four estimate_* entry points (robust.h:45-46,68-70,112-113,133-134): pixels + cameras in, the
// pre-step of every problem (threshold scaling, camera unprojection and normalize_points on the device), LO-RANSAC in
// lock-step groups per kind (tangent-Sampson problems form their own groups), final bundle and un-normalisation.
int plb_estimate_batch(plb_estimate_problem *problems, size_t count, int n_gpus, int streams_per_gpu) {
    return run_batch(problems, count, estimate_problem_prepare, n_gpus, -1, streams_per_gpu);
}
// The same on the calling thread's device with device-resident inputs and masks: the inputs are gathered into the engine's
// own buffer by k_ingest (F / H normalisation then works in place on that copy, the caller's arrays are only read) and
// the masks are written by k_scatter_masks, so what runs between is the host path's work on the same doubles.
int plb_estimate_batch_device(plb_estimate_problem *problems, size_t count, int dtype, void *stream, int streams) {
    return run_batch(problems, count, estimate_problem_prepare, -1, -1, streams, dtype, stream);
}
int plb_refine_batch(plb_refine_problem *problems, size_t count, int n_gpus, int streams_per_gpu) {
    return run_batch(problems, count, refine_problem_prepare, n_gpus, -1, streams_per_gpu);
}
// The same on the calling thread's device with a / b / weights in its memory: k_ingest gathers them into the engine's
// own input buffer, where the host path's upload puts them, so what runs after is the host path's work on the same doubles.
int plb_refine_batch_device(plb_refine_problem *problems, size_t count, int dtype, void *stream, int streams) {
    return run_batch(problems, count, refine_problem_prepare, -1, -1, streams, dtype, stream);
}
int plb_score_batch(plb_score_problem *problems, size_t count, int n_gpus, int streams_per_gpu) {
    return run_batch(problems, count, score_prepare, n_gpus, -1, streams_per_gpu);
}
// The same on the calling thread's device with everything sized by n or m in its memory: k_ingest gathers a / b into the
// engine's input buffer, k_score reads the caller's models and writes the caller's records and masks.
int plb_score_batch_device(plb_score_problem *problems, size_t count, int dtype, void *stream, int streams) {
    return run_batch(problems, count, score_prepare, -1, -1, streams, dtype, stream);
}

int plb_generate_batch(plb_generate_problem *problems, size_t count, int n_gpus, int streams_per_gpu) {
    return run_batch(problems, count, generate_host_prepare, n_gpus, -1, streams_per_gpu);
}
// The same on the calling thread's device with everything sized by n or s in its memory: the indices are range-checked
// by one kernel before anything gathers with them, k_take_samples copies them into the round's table and k_put_hyps
// writes the records into the caller's rows.
int plb_generate_batch_device(plb_generate_problem *problems, size_t count, int dtype, void *stream, int streams) {
    return run_batch(problems, count, generate_device_prepare, -1, -1, streams, dtype, stream);
}

int plb_camera_batch(plb_camera_problem *problems, size_t count, int n_gpus, int streams_per_gpu) {
    return run_batch(problems, count, camera_prepare, n_gpus, -1, streams_per_gpu);
}
// The same on the calling thread's device with in, out and the Jacobians in its memory: k_camera reads and writes them.
int plb_camera_batch_device(plb_camera_problem *problems, size_t count, int dtype, void *stream, int streams) {
    return run_batch(problems, count, camera_prepare, -1, -1, streams, dtype, stream);
}

int plb_resident_create(int kind, const double *a, const double *b, size_t n_pts) {
    if (kind < 0 || kind > 3 || !a || !b || n_pts == 0 || n_pts > (1u << 26)) {
        g_err = "bad argument";
        return PLB_ERR_ARG;
    }
    Engine &E = *engine();
    int rc = E.init();
    if (rc != PLB_OK) return rc;
    const int n = (int)n_pts, n_pad = (n + 31) & ~31, b_dim = (kind == KIND_PNP) ? 3 : 2, n_arr = 2 + b_dim;
    std::shared_ptr<Resident> R = std::make_shared<Resident>(); // freed on every early return below
    DevBuf<double> da, db;
    const bool qk = kind == KIND_RELPOSE || kind == KIND_FUND;
    if ((rc = R->soa64.ensure((size_t)n_arr * n_pad)) || (rc = R->soa32.ensure((size_t)n_arr * n_pad)) ||
        (rc = R->qrows.ensure(qk ? (size_t)n_pad : 0)) ||
        (rc = R->cmax.ensure(8)) || (rc = da.ensure(2 * (size_t)n)) || (rc = db.ensure((size_t)b_dim * n)) ||
        (rc = E.tdesc.ensure(1)) || (rc = E.h_tdesc.ensure(1)))
        return rc;
    PLB_CUDA(cudaMemcpyAsync(da.p, a, sizeof(double) * 2 * n, cudaMemcpyHostToDevice, E.stream));
    PLB_CUDA(cudaMemcpyAsync(db.p, b, sizeof(double) * b_dim * n, cudaMemcpyHostToDevice, E.stream));
    TransposeDesc &D = E.h_tdesc.p[0];
    std::memset(&D, 0, sizeof(D));
    D.a = da.p;
    D.b = db.p;
    D.s64 = R->soa64.p;
    D.s32 = R->soa32.p;
    D.cmax = R->cmax.p;
    D.q = qk ? R->qrows.p : nullptr;
    D.n = n;
    D.n_pad = n_pad;
    D.b_dim = b_dim;
    D.mode = 0;
    D.scale = 1.0;
    PLB_CUDA(cudaMemsetAsync(R->cmax.p, 0, sizeof(float) * 8, E.stream));
    PLB_CUDA(cudaMemcpyAsync(E.tdesc.p, E.h_tdesc.p, sizeof(TransposeDesc), cudaMemcpyHostToDevice, E.stream));
    launch_transpose(E.tdesc.p, 1, n_pad, false, E.stream);
    launch_qrows(E.tdesc.p, 1, n_pad, E.stream);
    PLB_CUDA(cudaStreamSynchronize(E.stream));
    R->n = n;
    R->n_pad = n_pad;
    R->kind = kind;
    R->device = E.device;
    std::lock_guard<std::mutex> lk(g_res_mtx);
    for (size_t i = 0; i < g_resident.size(); ++i)
        if (!g_resident[i]) {
            g_resident[i] = R;
            return (int)i + 1;
        }
    g_resident.push_back(R);
    return (int)g_resident.size();
}
int plb_resident_free(int handle) {
    std::shared_ptr<Resident> gone; // destroyed (cudaFree) outside the lock; a batch call in flight keeps its own reference
    {
        std::lock_guard<std::mutex> lk(g_res_mtx);
        if (handle <= 0 || (size_t)handle > g_resident.size() || !g_resident[handle - 1]) {
            g_err = "invalid resident handle";
            return PLB_ERR_ARG;
        }
        gone = std::move(g_resident[handle - 1]);
        g_resident[handle - 1] = nullptr;
    }
    return PLB_OK;
}

} // extern "C"
