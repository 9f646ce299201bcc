// poselib_b200 — host engine + C-ABI (include/poselib_b200.h).
//
// The reference runs one serial loop per problem (robust/ransac_impl.h:157-201).  Its sample sequence is a pure
// function of (seed, N, sample size, PROSAC options) and neither scoring nor refinement touch the RNG, so the engine
//   1. generates the sample table for a whole round of iterations on the host (robust/sampling.cc restated below),
//   2. lets the GPU solve + score every sample of the round (one warp per sample, kernels.cu),
//   3. finds, from the per-model (inlier count, MSAC score) records, every model that improves the best-minimal
//      state — that sub-sequence does not depend on LO results — and refines all of them in one batched LM launch,
//   4. replays score_models() (ransac_impl.h:106-154) in iteration order over those records, which reproduces the
//      serial trajectory exactly: LO triggers, stats, dynamic_max_iter and the break test see the same state as the
//      reference loop; samples evaluated past the serial break point are discarded.
// There is no CPU compute path: without a CUDA device every compute entry point fails with PLB_ERR_CUDA.
#include "../../include/poselib_b200.h"
#include "kernels.cuh"

#include <sched.h>

#include <algorithm>
#include <atomic>
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

__global__ void k_gather_models(const double *__restrict__ models, const int *__restrict__ slots, int n, int msz,
                                double *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * 9) return;
    const int j = i / 9, k = i % 9;
    out[i] = (k < msz) ? models[(size_t)slots[j] * msz + k] : 0.0;
}

struct Engine {
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr, ev4 = nullptr;
    cudaEvent_t ev_block = nullptr; // cudaEventBlockingSync: the waiting thread sleeps instead of spinning
    bool ready = false;
    int device = -1;
    DevBuf<double> in, soa64, px64, models, lm_in, s5_blk, s5_park, s5_cpoly, s5_roots;
    DevBuf<int> s5_nroots;
    DevBuf<float> soa32, cmax;
    DevBuf<uint32_t> samples;
    DevBuf<int> work, slots, subset, act, model_prob, prob_count;
    // round state that stays on the device: sampler states, per-sample / per-model records, candidate lists
    DevBuf<SamplerDev> smp;
    DevBuf<uint64_t> growth;
    DevBuf<RoundProb> rp;
    DevBuf<int> n_models, first_slot, prefix, cand_slot, cand_sample, n_cand, n_models_tot;
    DevBuf<uint32_t> counts, fcounts, fborder;
    DevBuf<double> scores;
    DevBuf<float> fscores, ferr;
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
    DevBuf<LmJob> jobs;
    PinBuf<double> h_in, h_lm_in;
    PinBuf<int> h_slots, h_act, h_work;
    PinBuf<ProblemDev> h_probs;
    PinBuf<TransposeDesc> h_tdesc;
    PinBuf<MaskDesc> h_mdesc;
    PinBuf<LmJob> h_jobs;
    // result records written by the kernels directly into mapped pinned memory (no explicit D2H copies): per round and
    // problem one header, the models that improved the best-minimal state and the LO results
    MapBuf<double> h_scores;
    MapBuf<uint32_t> h_counts;
    MapBuf<SelHeader> h_hdr;
    MapBuf<ImpRec> h_imp;
    MapBuf<LmJobOut> h_lm_out;
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
    p.use_camera = 0;
    p.cam.model = CAMM_NULL;
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
    p.cam.model = CAMM_NULL;
    p.score_after = 0;
    return p;
}

struct FinalPolish { // the post-RANSAC refinement of PoseLib/robust.cc (estimate_* entry points)
    bool enabled = false;
    plb_bundle_opt bundle;
    size_t min_inliers = 0; // run iff stats.num_inliers > min_inliers
    // pnp only: refine in pixel*scale coordinates with the rescaled camera (robust.cc:103-123)
    const double *px_scaled = nullptr; // 2n doubles (AoS) or null
    CamDev cam{CAMM_NULL, 0, {0, 0, 0, 0, 0, 0, 0, 0}};
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
    const Resident *res = nullptr;
    bool skip = false; // nothing to run (estimate_* with too few points): the batch runner leaves it alone
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
};

// per-problem serial state of the reference loop (ransac_impl.h:99-104,157-201)
struct PState {
    Task *t = nullptr;
    int n = 0, n_pad = 0, pidx = 0;
    bool enough = false, active = false, broke = false;
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

// Runs a group of problems of the same kind in lock-step rounds: one solve launch, one score launch and (when some
// model improved) one gather + one LM launch per round for the WHOLE group.
static int run_group(int kind, std::vector<Task *> &tasks) {
    Engine &E = *engine();
    const int K = kind_sample_size(kind), MAXM = kind_max_models(kind), MSZ = kind_model_size(kind);
    // in_arr: doubles per correspondence in the caller layout; n_arr: SoA arrays resident per correspondence
    const int b_dim = (kind == KIND_PNP) ? 3 : 2, in_arr = 2 + b_dim, n_arr = (kind == KIND_RELPOSE_TS) ? TS_ARRAYS : in_arr;
    const int NP = (int)tasks.size();
    std::vector<PState> PS(NP);
    bool any_points = false;
    for (int i = 0; i < NP; ++i) {
        Task &t = *tasks[i];
        PState &S = PS[i];
        S.t = &t;
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
        S.n = (int)t.n;
        S.n_pad = (S.n + 31) & ~31;
        S.enough = t.n >= (size_t)K; // ransac_impl.h:161-163
        S.dynamic_max_iter = t.opt.max_iterations;
        S.log_prob_missing_model = std::log(1.0 - t.opt.success_prob);
        any_points |= (t.n > 0);
    }
    auto finish = [&]() {
        for (int i = 0; i < NP; ++i) {
            PState &S = PS[i];
            if (S.hyp_pending) S.cnt.hypotheses += (uint64_t)E.h_hypfix.p[S.pidx];
            S.cnt.scored_corrs = S.cnt.hypotheses * S.t->n;
            if (S.t->stats_out) *S.t->stats_out = S.stats;
            if (S.t->cnt_out) *S.t->cnt_out = S.cnt;
        }
    };
    if (!any_points) {
        finish();
        return PLB_OK;
    }
    int rc = E.init();
    if (rc != PLB_OK) return rc;
    lm_set_sm_share(t_batch_worker ? 50 : 100); // a lone call owns the GPU; batch groups share it
    cudaStream_t st = E.stream;
    const uint64_t launches0 = E.launches;
    uint64_t h2d = 0, d2h = 0;
    double lo_wait = 0.0;
    float gpu_ms_total = 0.f, gpu_ms_score = 0.f, gpu_ms_confirm = 0.f, gpu_ms_lo = 0.f;
    auto sync_timed = [&](double *acc) -> int {
        auto t0 = std::chrono::steady_clock::now();
        if (t_blocking_sync) { // more waiting threads than cores: sleep on an event instead of spinning on the stream
            PLB_CUDA(cudaEventRecord(E.ev_block, st));
            PLB_CUDA(cudaEventSynchronize(E.ev_block));
        } else {
            PLB_CUDA(cudaStreamSynchronize(st));
        }
        if (acc) *acc += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        return PLB_OK;
    };

    // host-side phase timer (PLB_PROFILE=1 prints one line per group to stderr)
    static const bool prof_on = std::getenv("PLB_PROFILE") != nullptr;
    enum { PH_SETUP, PH_SAMPLE, PH_LAUNCH, PH_WAIT_HYP, PH_SELECT, PH_WAIT_CONF, PH_PASS1, PH_WAIT_LM, PH_PASS2, PH_FINAL, PH_N };
    double ph[PH_N] = {0};
    auto ph_t = std::chrono::steady_clock::now();
    auto mark = [&](int which) {
        if (!prof_on) return;
        const auto now = std::chrono::steady_clock::now();
        ph[which] += std::chrono::duration<double>(now - ph_t).count();
        ph_t = now;
    };
    int n_rounds = 0;

    // ---- device layout of the group: SoA arrays of every non-resident problem, masks, ProblemDev table -----------
    size_t in_doubles = 0, soa_elems = 0, mask_bytes = 0, px_elems = 0;
    int max_n = 0, max_n_pad = 0, n_up = 0, n_polish_pnp = 0;
    for (PState &S : PS) {
        if (S.n == 0) continue;
        if (!S.t->res) {
            in_doubles += (size_t)in_arr * S.n;
            soa_elems += (size_t)n_arr * S.n_pad;
            ++n_up;
        }
        S.mask_off = (long long)mask_bytes;
        mask_bytes += (size_t)S.n_pad;
        max_n = std::max(max_n, S.n);
        max_n_pad = std::max(max_n_pad, S.n_pad);
        if (kind == KIND_PNP && S.t->polish.enabled && S.t->polish.px_scaled) {
            px_elems += 2 * (size_t)S.n_pad;
            ++n_polish_pnp;
        }
    }
    const int n_probdev = NP + n_polish_pnp;
    if ((rc = E.h_in.ensure(in_doubles + px_elems)) || (rc = E.in.ensure(in_doubles)) || (rc = E.soa64.ensure(soa_elems)) ||
        (rc = E.soa32.ensure(soa_elems)) || (rc = E.cmax.ensure(5 * (size_t)NP)) || (rc = E.px64.ensure(px_elems)) || (rc = E.mask.ensure(mask_bytes)) ||
        (rc = E.mask_bits.ensure(mask_bytes / 32 + 1)) || (rc = E.h_mask_bits.ensure(mask_bytes / 32 + 1)) ||
        (rc = E.work.ensure(8)) || (rc = E.probs.ensure(n_probdev)) ||
        (rc = E.h_probs.ensure(n_probdev)) || (rc = E.tdesc.ensure(std::max(n_up, 1))) ||
        (rc = E.h_tdesc.ensure(std::max(n_up, 1))))
        return rc;
    {
        struct DirectCopy {
            double *dst;
            const double *src;
            size_t bytes;
        };
        std::vector<DirectCopy> direct; // page-locked caller arrays: DMA straight from them (issued below, in one turn)
        size_t in_off = 0, soa_off = 0, px_off = 0;
        std::vector<std::pair<size_t, size_t>> staged; // (offset, doubles) of the inputs that went through the staging buffer
        int iu = 0, ipol = 0;
        for (int i = 0; i < NP; ++i) {
            PState &S = PS[i];
            S.pidx = i;
            ProblemDev &P = E.h_probs.p[i];
            std::memset(&P, 0, sizeof(P));
            P.n = S.n;
            P.kind = kind;
            P.sq_thr = S.t->max_error * S.t->max_error;
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
            } else {
                S.in_off = (long long)in_off;
                if (host_pinned(S.t->a) && host_pinned(S.t->b)) {
                    // the caller's arrays are page-locked: DMA straight from them, no staging copy on the host
                    direct.push_back({E.in.p + in_off, S.t->a, sizeof(double) * 2 * S.n});
                    direct.push_back({E.in.p + in_off + 2 * (size_t)S.n, S.t->b, sizeof(double) * (size_t)b_dim * S.n});
                    h2d += sizeof(double) * (size_t)in_arr * S.n;
                } else {
                    staged.emplace_back(in_off, (size_t)in_arr * S.n);
                    double *ha = E.h_in.p + in_off, *hb = ha + 2 * (size_t)S.n;
                    std::memcpy(ha, S.t->a, sizeof(double) * 2 * S.n);
                    std::memcpy(hb, S.t->b, sizeof(double) * (size_t)b_dim * S.n);
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
                if (kind == KIND_RELPOSE_TS) {
                    P.ts = D.s64;
                } else {
                    for (int c = 0; c < n_arr; ++c) {
                        P.p[c] = D.s64 + (size_t)c * S.n_pad;
                        P.f[c] = D.s32 + (size_t)c * S.n_pad;
                    }
                }
                in_off += (size_t)in_arr * S.n;
                soa_off += (size_t)n_arr * S.n_pad;
            }
            if (kind == KIND_PNP && S.t->polish.enabled && S.t->polish.px_scaled) {
                // scaled pixels staged as SoA by the host (O(N) once); extra ProblemDev for the polish job
                double *hp = E.h_in.p + in_doubles + px_off;
                for (int k = 0; k < S.n; ++k) {
                    hp[k] = S.t->polish.px_scaled[2 * k];
                    hp[S.n_pad + k] = S.t->polish.px_scaled[2 * k + 1];
                }
                for (int k = S.n; k < S.n_pad; ++k) hp[k] = hp[S.n_pad + k] = 0.0;
                S.polish_pidx = NP + ipol;
                ProblemDev &PP = E.h_probs.p[NP + ipol];
                PP = P;
                PP.p[0] = E.px64.p + px_off;
                PP.p[1] = E.px64.p + px_off + S.n_pad;
                px_off += 2 * (size_t)S.n_pad;
                ++ipol;
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
        if (px_elems) {
            PLB_CUDA(cudaMemcpyAsync(E.px64.p, E.h_in.p + in_doubles, sizeof(double) * px_elems, cudaMemcpyHostToDevice, st));
            h2d += sizeof(double) * px_elems;
        }
        if (upload_turn.owns_lock()) upload_turn.unlock();
        // ---- normalize_points on the device (robust/utils.cc:584-644), then the thresholds that depend on its scale
        {
            std::vector<int> who;
            for (int i = 0; i < NP; ++i)
                if (PS[i].t->norm_mode != 0 && PS[i].in_off >= 0 && PS[i].n > 0) who.push_back(i);
            const int nn = (int)who.size();
            if (nn) {
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
                if ((rc = sync_timed(nullptr))) return rc;
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
            }
        }
        PLB_CUDA(cudaMemcpyAsync(E.probs.p, E.h_probs.p, sizeof(ProblemDev) * n_probdev, cudaMemcpyHostToDevice, st));
        if (n_up) {
            PLB_CUDA(cudaMemsetAsync(E.cmax.p, 0, sizeof(float) * 5 * (size_t)NP, st));
            PLB_CUDA(cudaMemcpyAsync(E.tdesc.p, E.h_tdesc.p, sizeof(TransposeDesc) * n_up, cudaMemcpyHostToDevice, st));
            launch_transpose(E.tdesc.p, n_up, max_n_pad, st);
            E.launches++;
        }
    }

    // LM launch helper: jobs[] + their input models already in E.h_lm_in[0 .. 9*njobs) (or on device, see gathered)
    auto launch_lm_jobs = [&](int njobs, bool models_on_device, size_t dev_model_off) -> int {
        int r;
        if ((r = E.jobs.ensure(njobs)) || (r = E.h_lm_out.ensure(njobs)) || (r = E.lm_in.ensure(9 * (size_t)njobs + dev_model_off)))
            return r;
        PLB_CUDA(cudaMemcpyAsync(E.jobs.p, E.h_jobs.p, sizeof(LmJob) * njobs, cudaMemcpyHostToDevice, st));
        h2d += sizeof(LmJob) * njobs;
        if (!models_on_device) {
            PLB_CUDA(cudaMemcpyAsync(E.lm_in.p + dev_model_off, E.h_lm_in.p, sizeof(double) * 9 * njobs, cudaMemcpyHostToDevice, st));
            h2d += sizeof(double) * 9 * njobs;
        }
        launch_lm(kind, E.probs.p, E.jobs.p, E.lm_in.p + dev_model_off, njobs, max_n, E.mask.p, E.subset.p, max_n_pad,
                  E.h_lm_out.d, st);
        E.launches++;
        d2h += sizeof(LmJobOut) * njobs;
        return PLB_OK;
    };
    auto make_lo_job = [&](LmJob &J, const PState &S, long long scratch_off) {
        J.pidx = S.pidx;
        J.reserved = 0;
        J.mask_off = -1;
        J.scratch_off = scratch_off;
        J.prm = lo_params(kind, S.t->max_error);
    };

    // ---- initial models (ransac_impl.h:173-176) ------------------------------------------------------------------
    {
        std::vector<int> who;
        for (int i = 0; i < NP; ++i)
            if (PS[i].enough && PS[i].t->opt.score_initial_model) who.push_back(i);
        const int nw = (int)who.size();
        if (nw) {
            if ((rc = E.h_lm_in.ensure(9 * (size_t)nw)) || (rc = E.lm_in.ensure(9 * (size_t)nw)) || (rc = E.h_slots.ensure(nw)) ||
                (rc = E.slots.ensure(nw)) || (rc = E.h_counts.ensure(nw)) || (rc = E.h_scores.ensure(nw)) ||
                (rc = E.h_jobs.ensure(nw)) || (rc = E.subset.ensure((size_t)nw * max_n_pad)))
                return rc;
            // the 9-double staging rows double as the MSZ-strided model list expected by k_score
            std::vector<double> packed((size_t)nw * MSZ);
            for (int j = 0; j < nw; ++j) {
                std::fill(E.h_lm_in.p + 9 * j, E.h_lm_in.p + 9 * j + 9, 0.0);
                std::copy(PS[who[j]].t->model, PS[who[j]].t->model + MSZ, E.h_lm_in.p + 9 * j);
                std::copy(PS[who[j]].t->model, PS[who[j]].t->model + MSZ, packed.data() + (size_t)j * MSZ);
                E.h_slots.p[j] = who[j];
            }
            if ((rc = E.models.ensure((size_t)nw * MSZ))) return rc;
            PLB_CUDA(cudaMemcpyAsync(E.models.p, packed.data(), sizeof(double) * nw * MSZ, cudaMemcpyHostToDevice, st));
            PLB_CUDA(cudaMemcpyAsync(E.slots.p, E.h_slots.p, sizeof(int) * nw, cudaMemcpyHostToDevice, st));
            PLB_CUDA(cudaMemcpyAsync(E.work.p + 4, &nw, sizeof(int), cudaMemcpyHostToDevice, st));
            launch_score_models(kind, E.probs.p, E.models.p, E.slots.p, nw, E.work.p + 4, E.h_counts.d, E.h_scores.d, st);
            E.launches++;
            if ((rc = sync_timed(nullptr))) return rc;
            int nj = 0;
            std::vector<int> jw;
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
                    make_lo_job(E.h_jobs.p[nj], S, (long long)nj * max_n_pad);
                    if (nj != j) std::copy(E.h_lm_in.p + 9 * j, E.h_lm_in.p + 9 * j + 9, E.h_lm_in.p + 9 * nj);
                    jw.push_back(who[j]);
                    ++nj;
                }
            }
            if (nj) {
                if ((rc = launch_lm_jobs(nj, false, 0))) return rc;
                if ((rc = sync_timed(&lo_wait))) return rc;
                for (int j = 0; j < nj; ++j) {
                    PState &S = PS[jw[j]];
                    const LmJobOut &o = E.h_lm_out.p[j];
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
            }
        }
    }

    mark(PH_SETUP);
    // ---- main loop in lock-step rounds ------------------------------------------------------------------------------
    // Every round is ONE chain of launches with ONE host synchronisation at its end:
    //   k_sample -> solve kernels -> scoring (fp64 of every model, or fp32 screening) -> k_select -> [k_confirm] ->
    //   k_pass1 -> k_lm over the LO triggers it listed.
    // The sampler state, the per-model records and the candidate lists never leave the device; the host receives, per
    // problem, one header, the few models that improved the best-minimal state and the LO results, and replays
    // score_models() (ransac_impl.h:106-154) over those.
    for (PState &S : PS) S.active = S.enough && S.t->opt.max_iterations > 0;
    {
        // device sampler states (robust/sampling.h:49-83) + PROSAC growth tables (sampling.cc:105-136)
        size_t growth_total = 0;
        for (PState &S : PS)
            if (S.active && S.t->opt.progressive_sampling) growth_total += std::max<size_t>(S.t->n, (size_t)K);
        if ((rc = E.h_smp.ensure(NP)) || (rc = E.smp.ensure(2 * (size_t)NP)) || (rc = E.h_growth.ensure(growth_total)) ||
            (rc = E.growth.ensure(growth_total)) || (rc = E.h_lo_tmpl.ensure(NP)) || (rc = E.lo_tmpl.ensure(NP)) ||
            (rc = E.h_hypfix.ensure(NP)))
            return rc;
        size_t goff = 0;
        for (int i = 0; i < NP; ++i) {
            PState &S = PS[i];
            SamplerDev &D = E.h_smp.p[i];
            std::memset(&D, 0, sizeof(D));
            make_lo_job(E.h_lo_tmpl.p[i], S, 0);
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
    }
    int smp_cur = 0; // sampler states of the current round: E.smp[smp_cur * NP ..]; the advanced ones land in the other half
    // Round sizes.  A small group leaves the GPU mostly idle, so speculating further ahead costs little time while every
    // round saved is a whole launch chain of latency: the first round and the per-round cap grow as the group shrinks
    // (1 problem: 4096 doubling up to 65536 samples; >= 16 problems: 1024 doubling to 16384).  The first round stays
    // moderate on purpose: a loop that stops right after min_iterations (high inlier ratio) would otherwise pay for
    // thousands of speculative samples and their LO refits (measured: C4 single call 2.0 -> 3.3 ms with 16384).
    const size_t few = (size_t)std::max(1, std::min(NP, 16));
    const size_t CHUNK_MAX = std::max<size_t>(16384, 65536 / few), ROUND_MAX = std::max<size_t>(32768, 65536 / few),
                 S_TOT_MAX = 262144;
    for (PState &S : PS) S.chunk = std::min<size_t>(4096, std::max<size_t>(1024, 16384 / few));
    // 0 exact, 1 fast (fp32 screen + fp64 confirmation of candidates); the tangent-Sampson kind has no fp32 copy
    const int mode = (kind == KIND_RELPOSE_TS) ? 0 : current_mode();
    int cap_factor = kind_is_relpose(kind) ? 8 : MAXM;
    bool big_caps = false;
    std::vector<int> act;
    std::vector<uint8_t> first_round(NP, 1);
    for (;;) {
        act.clear();
        for (int i = 0; i < NP; ++i) {
            PState &S = PS[i];
            if (!S.active) continue;
            // break test at the top of iteration `it` (ransac_impl.h:180-184)
            if (S.it >= S.t->opt.max_iterations || (S.it > S.t->opt.min_iterations && S.it > S.dynamic_max_iter)) {
                S.active = false;
                continue;
            }
            act.push_back(i);
        }
        const int na = (int)act.size();
        if (!na) break;
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
        const size_t cap_models = total * (size_t)cap_factor;
        // capacity of the host-visible records of the round; exceeded -> the round is redone with the worst case
        const size_t job_cap = big_caps ? total : std::min(total, std::max<size_t>(1024, total / 8));
        const size_t imp_cap = big_caps ? cap_models : std::min(cap_models, 2 * job_cap);
        const int lm_clusters = lm_round_max_clusters(kind, est_jobs, max_n);
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
        {
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
        }
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
        HypOut out;
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
        out.fcounts = nullptr;
        out.fscores = nullptr;
        out.fborder = nullptr;
        out.ferr = nullptr;
        if (mode == 1) {
            if ((rc = E.fcounts.ensure(cap_models)) || (rc = E.fscores.ensure(cap_models)) ||
                (rc = E.fborder.ensure(cap_models)) || (rc = E.ferr.ensure(cap_models)))
                return rc;
            out.fcounts = E.fcounts.p;
            out.fscores = E.fscores.p;
            out.fborder = E.fborder.p;
            out.ferr = E.ferr.p;
        }
        out.s5_blk = out.s5_park = out.s5_cpoly = out.s5_roots = nullptr;
        out.s5_nroots = nullptr;
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
        launch_hypotheses(kind, R, E.work.p, out, mode, max_n_pad, st, E.ev2);
        PLB_CUDA(cudaEventRecord(E.ev1, st));
        E.launches += kind_is_relpose(kind) ? 5 : 2; // k_solve (or k5_gather + k5_prep_lane + k5_roots + k5_back) + scoring
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
        if ((rc = sync_timed(nullptr))) return rc;
        mark(PH_WAIT_HYP);
        d2h += CTL_WORDS * sizeof(int);
        if (E.h_work.p[CTL_OVERFLOW] != 0) { // model list overflow: redo the round with the worst-case capacity
            if (cap_factor >= MAXM) {        // (nothing was committed: the sampler states of this round are still current)
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
        smp_cur ^= 1;
        float ms = 0.f, ms_sc = 0.f, ms_cf = 0.f;
        cudaEventElapsedTime(&ms, E.ev0, E.ev1);
        cudaEventElapsedTime(&ms_sc, E.ev2, E.ev1);
        cudaEventElapsedTime(&ms_cf, E.ev1, E.ev3);
        gpu_ms_total += ms + ms_cf;
        gpu_ms_score += ms_sc;
        gpu_ms_confirm += ms_cf;
        {
            float ms_lo = 0.f;
            cudaEventElapsedTime(&ms_lo, E.ev3, E.ev4);
            gpu_ms_lo += ms_lo;
        }

        // ---- replay of the serial loop over this round, problem by problem (ransac_impl.h:106-154,180-188) --------
        // Only samples with an improving model change the state; between two of them the break test
        // `it > min_iterations && it > dynamic_max_iter` (:182) first holds at max(min_iterations, dyn) + 1.
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
                const LmJobOut &o = lo[tp++];
                S.stats.refinements++;
                S.cnt.lo_calls++;
                S.cnt.hypotheses++;
                if (o.score < S.stats.model_score) {
                    S.stats.model_score = o.score;
                    S.stats.num_inliers = o.count;
                    std::copy(o.model, o.model + MSZ, S.best_model);
                }
                update_dynamic(S, K);
                cur = next_trig + 1;
            }
            S.cnt.samples += cur - it0;
            S.it = cur;
            if (broke) {
                S.broke = true;
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
        mark(PH_PASS2);
    }
    for (PState &S : PS)
        if (S.enough) S.stats.iterations = S.it;

    // ---- final refinement of every problem (ransac_impl.h:190-198), one launch ---------------------------------------
    {
        std::vector<int> who;
        for (int i = 0; i < NP; ++i)
            if (PS[i].enough) who.push_back(i);
        const int nw = (int)who.size();
        if (nw) {
            if ((rc = E.h_lm_in.ensure(9 * (size_t)nw)) || (rc = E.h_jobs.ensure(nw)) ||
                (rc = E.subset.ensure((size_t)nw * max_n_pad)))
                return rc;
            for (int j = 0; j < nw; ++j) {
                PState &S = PS[who[j]];
                std::fill(E.h_lm_in.p + 9 * j, E.h_lm_in.p + 9 * j + 9, 0.0);
                std::copy(S.best_model, S.best_model + MSZ, E.h_lm_in.p + 9 * j);
                make_lo_job(E.h_jobs.p[j], S, (long long)j * max_n_pad);
            }
            if ((rc = launch_lm_jobs(nw, false, 0))) return rc;
            if ((rc = sync_timed(&lo_wait))) return rc;
            for (int j = 0; j < nw; ++j) {
                PState &S = PS[who[j]];
                const LmJobOut &o = E.h_lm_out.p[j];
                S.stats.refinements++;
                S.cnt.lo_calls++;
                S.cnt.hypotheses++;
                if (o.score < S.stats.model_score) { // NB: model_score itself is not updated by the reference here
                    std::copy(o.model, o.model + MSZ, S.best_model);
                    S.stats.num_inliers = o.count;
                }
            }
        }
    }

    // ---- final inlier masks (ransac.cc:54,151,259,311) + optional polish over the inliers (robust.cc) -----------------
    {
        std::vector<int> who;
        for (int i = 0; i < NP; ++i)
            if (PS[i].n > 0) who.push_back(i);
        const int nw = (int)who.size();
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
        std::vector<int> pol;
        for (int i = 0; i < NP; ++i)
            if (PS[i].n > 0 && PS[i].t->polish.enabled && PS[i].stats.num_inliers > PS[i].t->polish.min_inliers) pol.push_back(i);
        const int npol = (int)pol.size();
        if (npol) {
            // robust.cc:103-123,296-311,573-588,736-751: LM over the inliers with the user's BundleOptions
            if ((rc = E.h_lm_in.ensure(9 * (size_t)npol)) || (rc = E.h_jobs.ensure(npol)) ||
                (rc = E.subset.ensure((size_t)npol * max_n_pad)))
                return rc;
            for (int j = 0; j < npol; ++j) {
                PState &S = PS[pol[j]];
                std::fill(E.h_lm_in.p + 9 * j, E.h_lm_in.p + 9 * j + 9, 0.0);
                std::copy(S.best_model, S.best_model + MSZ, E.h_lm_in.p + 9 * j);
                LmJob &J = E.h_jobs.p[j];
                J.pidx = S.pidx;
                J.reserved = 0;
                J.mask_off = S.mask_off;
                J.scratch_off = (long long)j * max_n_pad;
                J.prm = bundle_params(S.t->polish.bundle);
                if (S.polish_pidx >= 0) {
                    J.pidx = S.polish_pidx;
                    J.prm.use_camera = 1;
                    J.prm.cam = S.t->polish.cam;
                }
            }
            if ((rc = launch_lm_jobs(npol, false, 0))) return rc;
        }
        // the masks cross PCIe as bits (1/8 of the bytes) and are expanded into the caller's char[n] below
        launch_pack_mask(E.mask.p, E.mask_bits.p, mask_bytes, st);
        E.launches++;
        PLB_CUDA(cudaMemcpyAsync(E.h_mask_bits.p, E.mask_bits.p, sizeof(uint32_t) * (mask_bytes / 32), cudaMemcpyDeviceToHost, st));
        if ((rc = sync_timed(nullptr))) return rc;
        for (int j = 0; j < npol; ++j) {
            PState &S = PS[pol[j]];
            std::copy(E.h_lm_out.p[j].model, E.h_lm_out.p[j].model + MSZ, S.best_model);
        }
        for (int i = 0; i < NP; ++i) {
            PState &S = PS[i];
            if (S.t->inliers && S.n > 0) {
                const uint32_t *w = E.h_mask_bits.p + (S.mask_off >> 5); // mask_off is a multiple of 32
                char *dst = S.t->inliers;
                for (int k = 0; k < S.n; ++k) dst[k] = (char)((w[k >> 5] >> (k & 31)) & 1u);
            }
            std::copy(S.best_model, S.best_model + MSZ, S.t->model);
            d2h += (size_t)S.n_pad / 8;
        }
    }
    PLB_CUDA(cudaGetLastError());
    mark(PH_FINAL);
    if (prof_on) {
        double tot = 0;
        for (int i = 0; i < PH_N; ++i) tot += ph[i];
        std::fprintf(stderr,
                     "[plb profile] kind %d problems %d rounds %d total %.2f ms | setup %.2f sample %.2f launch %.2f wait_hyp %.2f "
                     "select %.2f wait_conf %.2f pass1 %.2f wait_lm %.2f pass2 %.2f final %.2f\n",
                     kind, NP, n_rounds, 1e3 * tot, 1e3 * ph[0], 1e3 * ph[1], 1e3 * ph[2], 1e3 * ph[3], 1e3 * ph[4], 1e3 * ph[5],
                     1e3 * ph[6], 1e3 * ph[7], 1e3 * ph[8], 1e3 * ph[9]);
    }
    // group-level counters are attributed to the first problem; per-problem ones are exact
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
    return PLB_OK;
}

// Single-problem convenience used by the plb_ransac_* / plb_estimate_* entry points.
static int run_ransac(int kind, const double *a, const double *b, size_t n_pts, const plb_ransac_opt &opt,
                      double max_error, int rfc, double *model, char *inliers, plb_ransac_stats *stats_out,
                      plb_counters *cnt_out, const FinalPolish &polish, const Resident *res = nullptr,
                      int pre_mode = 0, const CamDev *cam_a = nullptr, const CamDev *cam_b = nullptr,
                      double pre_scale = 1.0) {
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
    t.res = res;
    std::vector<Task *> v{&t};
    return run_group(kind, v);
}

// One LM refinement over all n points (robust/bundle.cc:84-112,206-222,313-333,394-411)
static int run_refine(int kind, const double *a, const double *b, size_t n_pts, double *model,
                      const plb_bundle_opt &bopt, double *bstats, const CamDev *cam_a = nullptr,
                      const CamDev *cam_b = nullptr) {
    if (n_pts == 0) return PLB_OK;
    Engine &E = *engine();
    int rc = E.init();
    if (rc != PLB_OK) return rc;
    cudaStream_t st = E.stream;
    const int n = (int)n_pts, n_pad = (n + 31) & ~31;
    const int b_dim = (kind == KIND_PNP) ? 3 : 2, in_arr = 2 + b_dim, MSZ = kind_model_size(kind);
    const int n_arr = (kind == KIND_RELPOSE_TS) ? TS_ARRAYS : in_arr;
    if ((rc = E.h_in.ensure((size_t)in_arr * n)) || (rc = E.in.ensure((size_t)in_arr * n)) ||
        (rc = E.soa64.ensure((size_t)n_arr * n_pad)) || (rc = E.soa32.ensure((size_t)n_arr * n_pad)) ||
        (rc = E.lm_in.ensure(9)) || (rc = E.h_lm_in.ensure(9)) || (rc = E.h_lm_out.ensure(1)) ||
        (rc = E.probs.ensure(1)) || (rc = E.h_probs.ensure(1)) || (rc = E.tdesc.ensure(1)) || (rc = E.h_tdesc.ensure(1)) ||
        (rc = E.jobs.ensure(1)) || (rc = E.h_jobs.ensure(1)))
        return rc;
    std::memcpy(E.h_in.p, a, sizeof(double) * 2 * n);
    std::memcpy(E.h_in.p + 2 * (size_t)n, b, sizeof(double) * b_dim * n);
    PLB_CUDA(cudaMemcpyAsync(E.in.p, E.h_in.p, sizeof(double) * (size_t)in_arr * n, cudaMemcpyHostToDevice, st));
    TransposeDesc &D = E.h_tdesc.p[0];
    D.a = E.in.p;
    D.b = E.in.p + 2 * (size_t)n;
    D.s64 = E.soa64.p;
    D.s32 = E.soa32.p;
    D.cmax = nullptr;
    D.n = n;
    D.n_pad = n_pad;
    D.b_dim = b_dim;
    D.mode = (kind == KIND_RELPOSE_TS) ? 2 : 0;
    D.scale = 1.0;
    D.cam_a.model = D.cam_b.model = CAMM_NULL;
    if (cam_a) D.cam_a = *cam_a;
    if (cam_b) D.cam_b = *cam_b;
    ProblemDev &P = E.h_probs.p[0];
    std::memset(&P, 0, sizeof(P));
    if (kind == KIND_RELPOSE_TS) {
        P.ts = E.soa64.p;
    } else {
        for (int c = 0; c < n_arr; ++c) {
            P.p[c] = E.soa64.p + (size_t)c * n_pad;
            P.f[c] = E.soa32.p + (size_t)c * n_pad;
        }
    }
    P.n_pad = n_pad;
    P.n = n;
    P.kind = kind;
    P.sq_thr = 0.0;
    LmJob &J = E.h_jobs.p[0];
    J.pidx = 0;
    J.reserved = 0;
    J.mask_off = -1;
    J.scratch_off = 0;
    J.prm = bundle_params(bopt);
    J.prm.subset_mode = 0;
    std::fill(E.h_lm_in.p, E.h_lm_in.p + 9, 0.0);
    std::copy(model, model + MSZ, E.h_lm_in.p);
    PLB_CUDA(cudaMemcpyAsync(E.tdesc.p, E.h_tdesc.p, sizeof(TransposeDesc), cudaMemcpyHostToDevice, st));
    PLB_CUDA(cudaMemcpyAsync(E.probs.p, E.h_probs.p, sizeof(ProblemDev), cudaMemcpyHostToDevice, st));
    PLB_CUDA(cudaMemcpyAsync(E.jobs.p, E.h_jobs.p, sizeof(LmJob), cudaMemcpyHostToDevice, st));
    PLB_CUDA(cudaMemcpyAsync(E.lm_in.p, E.h_lm_in.p, sizeof(double) * 9, cudaMemcpyHostToDevice, st));
    launch_transpose(E.tdesc.p, 1, n_pad, st);
    lm_set_sm_share(100);
    launch_lm(kind, E.probs.p, E.jobs.p, E.lm_in.p, 1, n, nullptr, nullptr, 0, E.h_lm_out.d, st);
    E.launches += 2;
    PLB_CUDA(cudaStreamSynchronize(st));
    PLB_CUDA(cudaGetLastError());
    std::copy(E.h_lm_out.p[0].model, E.h_lm_out.p[0].model + MSZ, model);
    if (bstats) {
        bstats[0] = E.h_lm_out.p[0].iterations;
        bstats[1] = E.h_lm_out.p[0].initial_cost;
        bstats[2] = E.h_lm_out.p[0].cost;
    }
    return PLB_OK;
}

// plb_camera -> CamDev; models outside the six on the path are rejected like Camera::unproject's "NYI"
// (misc/camera_models.cc:176-188)
static int camera_dev(const plb_camera *c, CamDev *out) {
    out->model = CAMM_NULL;
    out->reserved = 0;
    for (int i = 0; i < 8; ++i) out->p[i] = 0.0;
    if (!c || c->model_id == PLB_CAMERA_NULL) return PLB_OK;
    int np = 0;
    switch (c->model_id) {
    case PLB_CAMERA_SIMPLE_PINHOLE: np = 3; break;
    case PLB_CAMERA_PINHOLE: np = 4; break;
    case PLB_CAMERA_SIMPLE_RADIAL: np = 4; break;
    case PLB_CAMERA_RADIAL: np = 5; break;
    case PLB_CAMERA_OPENCV: np = 8; break;
    default: g_err = "NYI: camera model not supported by the CUDA path (undistort on the host first)"; return PLB_ERR_NYI;
    }
    out->model = c->model_id;
    for (int i = 0; i < np; ++i) out->p[i] = c->params[i];
    return PLB_OK;
}
static double camera_focal(const CamDev &c) { // Camera::focal() camera_models.cc:304-324
    switch (c.model) {
    case CAMM_NULL: return 1.0;
    case CAMM_PINHOLE:
    case CAMM_OPENCV: return 0.0 + c.p[0] / 2 + c.p[1] / 2;
    default: return 0.0 + c.p[0] / 1;
    }
}
static void camera_rescale(CamDev &c, double scale) { // Camera::rescale camera_models.cc:432-454
    if (c.model == CAMM_NULL) return;
    const int k = (c.model == CAMM_PINHOLE || c.model == CAMM_OPENCV) ? 4 : 3; // focal_idx then principal_point_idx
    for (int i = 0; i < k; ++i) c.p[i] *= scale;
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
    o->reserved = 0;
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
    return run_ransac(KIND_RELPOSE_TS, x1, x2, n, *opt, max_error, 0, pose, inliers, stats, counters, FinalPolish(),
                      nullptr, 2, &c1, &c2, 1.0);
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
// One estimate_* call, prepared: the Task (points, scaled threshold, camera pre-step mode, final polish) plus what the
// post-step needs (normalising transforms of F / H).  Used by the four single entry points and by plb_estimate_batch.
struct EstimateJob {
    Task t;
    int api_kind = 0; // PLB_KIND_*
    std::vector<double> px;
    HM3 T1, T2;
    bool normalised = false;
    double *model = nullptr;
};
static void default_stats(plb_ransac_stats *stats, plb_counters *counters) {
    if (stats) {
        stats->refinements = stats->iterations = stats->num_inliers = 0;
        stats->inlier_ratio = 0;
        stats->model_score = std::numeric_limits<double>::max();
    }
    if (counters) std::memset(counters, 0, sizeof(*counters));
}
// robust.cc:36-126 (absolute pose, no focal estimation), :242-314 (relative pose; tangent_sampson keeps the scaled pixels
// and runs the tangent-Sampson estimator with the cameras), :544-594 (fundamental), :712-757 (homography).
// The camera pre-step (Camera::unproject / unproject_with_jac of every point) runs on the device, fused into the layout
// kernel; normalize_points (F / H) runs here on the calling (worker) thread.
static int estimate_prepare(int kind, const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                            const plb_camera *camera2, const plb_ransac_opt *ransac, const plb_bundle_opt *bundle,
                            double max_error, int real_focal_check, int tangent_sampson, double *model, char *inliers,
                            plb_ransac_stats *stats, plb_counters *counters, EstimateJob &J) {
    if (int r = check_ptrs(x1, x2, ransac, model, n)) return r;
    if (!bundle) {
        g_err = "null bundle options";
        return PLB_ERR_ARG;
    }
    if (kind < 0 || kind > 3) {
        g_err = "unknown problem kind";
        return PLB_ERR_ARG;
    }
    J.api_kind = kind;
    J.model = model;
    Task &t = J.t;
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
        const double scale = 1.0 / camera_focal(cam);
        fp.bundle.loss_scale = bundle->loss_scale * scale;
        fp.min_inliers = 3;
        if (cam.model != CAMM_NULL) { // the polish runs on pixels*scale with the rescaled camera (robust.cc:103-123)
            J.px.resize(2 * n);
            for (size_t k = 0; k < 2 * n; ++k) J.px[k] = x1[k] * scale;
            fp.px_scaled = J.px.data();
            fp.cam = cam;
            camera_rescale(fp.cam, scale);
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
        const double scale = 0.5 * (1.0 / camera_focal(c1) + 1.0 / camera_focal(c2));
        fp.bundle.loss_scale = bundle->loss_scale * scale;
        fp.min_inliers = 5;
        t.max_error = max_error * scale;
        if (tangent_sampson) {
            camera_rescale(c1, scale);
            camera_rescale(c2, scale);
            model[0] = 1.0; // ransac.cc:159-160: the start pose is reset even when score_initial_model is set
            for (int i = 1; i < 7; ++i) model[i] = 0.0;
            t.kind = KIND_RELPOSE_TS;
            t.pre_mode = 2;
            t.pre_scale = scale;
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
        default_stats(stats, counters);
        t.skip = true;
        return PLB_OK;
    }
    // normalize_points(scale = true, centroid = !real_focal_check | true, shared = true) runs on the device (k_normalize);
    // the engine divides max_error and the polish loss scale by the scale it finds (robust.cc:561-564,724-727)
    const bool fund = kind == PLB_KIND_FUNDAMENTAL;
    J.normalised = true;
    fp.bundle.loss_scale = bundle->loss_scale;
    fp.min_inliers = min_pts;
    t.kind = fund ? KIND_FUND : KIND_HOMOG;
    t.norm_mode = (fund && real_focal_check) ? 1 : 2;
    t.max_error = max_error;
    t.rfc = fund ? real_focal_check : 0;
    return PLB_OK;
}
static void estimate_finish(EstimateJob &J, const Task &t) {
    if (!J.normalised || t.skip) return;
    // robust.cc:590-591: F = T2^T F T1 ; :753-754: H = T2^-1 H T1 ; both renormalised
    norm_transforms(t.norm_out, J.T1, J.T2);
    HM3 M = (J.api_kind == PLB_KIND_FUNDAMENTAL) ? hm_mul(hm_mul(hm_T(J.T2), hm_from_cm(J.model)), J.T1)
                                                 : hm_mul(hm_mul(hm_inv(J.T2), hm_from_cm(J.model)), J.T1);
    const double nm = hm_norm(M);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) M.m[i][j] /= nm;
    hm_to_cm(M, J.model);
}
static int estimate_single(int kind, const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                           const plb_camera *camera2, const plb_ransac_opt *ransac, const plb_bundle_opt *bundle,
                           double max_error, int real_focal_check, int tangent_sampson, double *model, char *inliers,
                           plb_ransac_stats *stats, plb_counters *counters) {
    EstimateJob J;
    if (int r = estimate_prepare(kind, x1, x2, n, camera1, camera2, ransac, bundle, max_error, real_focal_check,
                                 tangent_sampson, model, inliers, stats, counters, J))
        return r;
    if (J.t.skip) return PLB_OK;
    std::vector<Task *> v{&J.t};
    const int rc = run_group(J.t.kind, v);
    if (rc != PLB_OK) return rc;
    estimate_finish(J, J.t);
    return PLB_OK;
}
int plb_estimate_absolute_pose(const double *points2D, const double *points3D, size_t n, const plb_ransac_opt *ransac,
                               const plb_bundle_opt *bundle, double max_error, const plb_camera *camera,
                               double pose[7], char *inliers, plb_ransac_stats *stats, plb_counters *counters) {
    return estimate_single(PLB_KIND_PNP, points2D, points3D, n, camera, nullptr, ransac, bundle, max_error, 0, 0, pose,
                           inliers, stats, counters);
}
int plb_estimate_relative_pose(const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                               const plb_camera *camera2, const plb_ransac_opt *ransac, const plb_bundle_opt *bundle,
                               double max_error, int tangent_sampson, double pose[7], char *inliers,
                               plb_ransac_stats *stats, plb_counters *counters) {
    return estimate_single(PLB_KIND_RELPOSE, x1, x2, n, camera1, camera2, ransac, bundle, max_error, 0, tangent_sampson,
                           pose, inliers, stats, counters);
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
static int refine_entry(int kind, const double *a, const double *b, size_t n, double *model, const plb_bundle_opt *opt,
                        double *bs) {
    if (!opt || !model || (n > 0 && (!a || !b))) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    return run_refine(kind, a, b, n, model, *opt, bs);
}
int plb_bundle_adjust(const double *x, const double *X, size_t n, double pose[7], const plb_bundle_opt *opt,
                      double bs[3]) {
    return refine_entry(KIND_PNP, x, X, n, pose, opt, bs);
}
int plb_refine_relpose(const double *x1, const double *x2, size_t n, double pose[7], const plb_bundle_opt *opt,
                       double bs[3]) {
    return refine_entry(KIND_RELPOSE, x1, x2, n, pose, opt, bs);
}
// robust/bundle.cc:237-266 with fixed intrinsics: unproject_with_jac of both images, then the tangent-Sampson refiner
int plb_refine_relpose_cameras(const double *x1, const double *x2, size_t n, const plb_camera *camera1,
                               const plb_camera *camera2, double pose[7], const plb_bundle_opt *opt, double bs[3]) {
    if (!opt || !pose || (n > 0 && (!x1 || !x2))) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    CamDev c1, c2;
    if (int r = camera_dev(camera1, &c1)) return r;
    if (int r = camera_dev(camera2, &c2)) return r;
    return run_refine(KIND_RELPOSE_TS, x1, x2, n, pose, *opt, bs, &c1, &c2);
}
int plb_refine_fundamental(const double *x1, const double *x2, size_t n, double F[9], const plb_bundle_opt *opt,
                           double bs[3]) {
    return refine_entry(KIND_FUND, x1, x2, n, F, opt, bs);
}
int plb_refine_homography(const double *x1, const double *x2, size_t n, double H[9], const plb_bundle_opt *opt,
                          double bs[3]) {
    return refine_entry(KIND_HOMOG, x1, x2, n, H, opt, bs);
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
    DevBuf<double> da, db, dout;
    DevBuf<int> dn;
    if ((rc = da.ensure(count * a_sz)) || (rc = db.ensure(count * b_sz)) || (rc = dout.ensure(count * out_sz)) ||
        (rc = dn.ensure(count)))
        return rc;
    PLB_CUDA(cudaMemcpyAsync(da.p, a, sizeof(double) * count * a_sz, cudaMemcpyHostToDevice, E.stream));
    PLB_CUDA(cudaMemcpyAsync(db.p, b, sizeof(double) * count * b_sz, cudaMemcpyHostToDevice, E.stream));
    launch_solver_batch(kind, variant, count, da.p, db.p, dout.p, dn.p, flags, E.stream);
    E.launches++;
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
    // groups per device: tasks of the same engine kind run in lock-step
    const int nthreads_req = std::max(1, streams);
    struct Job {
        int device;
        std::vector<std::vector<Task *>> groups;
    };
    std::vector<Job> jobs; // one per (device, worker)
    for (int d = 0; d < n_dev; ++d) {
        std::vector<std::vector<Task *>> groups;
        for (int kind = 0; kind <= KIND_RELPOSE_TS; ++kind) {
            std::vector<Task *> of_kind;
            for (size_t i = 0; i < count; ++i)
                if (tasks[i].kind == kind && dev_of[i] == devices[d] && !tasks[i].skip) of_kind.push_back(&tasks[i]);
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
            const int rc = run_group(grp[0]->kind, grp);
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
static int batch_impl(plb_problem *problems, size_t count, const int *devices, int n_dev, int streams) {
    if (count == 0) return PLB_OK;
    if (!problems) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    if (plb_device_count() == 0) {
        g_err = "no usable CUDA device";
        return PLB_ERR_CUDA;
    }
    for (size_t i = 0; i < count; ++i) {
        problems[i].status = PLB_OK;
        if (problems[i].kind < 0 || problems[i].kind > 3) {
            g_err = "unknown problem kind";
            for (size_t j = 0; j < count; ++j) problems[j].status = PLB_ERR_ARG;
            return PLB_ERR_ARG;
        }
    }
    std::vector<Task> tasks(count);
    std::vector<int> dev_of(count, -1);
    std::vector<std::shared_ptr<Resident>> held; // resident inputs stay alive for the duration of the call
    auto fail_all = [&](int rc, const char *msg) {
        g_err = msg;
        for (size_t j = 0; j < count; ++j) problems[j].status = rc;
        return rc;
    };
    for (size_t i = 0; i < count; ++i) {
        plb_problem &p = problems[i];
        Task &t = tasks[i];
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
            std::shared_ptr<Resident> res;
            {
                std::lock_guard<std::mutex> lk(g_res_mtx);
                if ((size_t)p.resident <= g_resident.size()) res = g_resident[p.resident - 1];
            }
            if (!res || res->kind != p.kind) return fail_all(PLB_ERR_ARG, "invalid resident handle");
            bool ok = false;
            for (int d = 0; d < n_dev; ++d) ok |= (devices[d] == res->device);
            if (!ok) return fail_all(PLB_ERR_ARG, "resident correspondences live on a device this call does not use");
            t.res = res.get();
            t.n = (size_t)res->n;
            dev_of[i] = res->device;
            held.push_back(std::move(res));
        } else if (t.n > 0 && (!p.a || !p.b)) {
            return fail_all(PLB_ERR_ARG, "null argument");
        }
    }
    const int rc = run_tasks(tasks, dev_of, devices, n_dev, streams);
    if (rc != PLB_OK)
        for (size_t i = 0; i < count; ++i) problems[i].status = rc;
    return rc;
}
int plb_ransac_batch(plb_problem *problems, size_t count, int streams) {
    const int dev = g_device;
    return batch_impl(problems, count, &dev, 1, streams);
}
// The same over the first n_gpus CUDA devices of this process (0 = all): in-process multi-GPU, no collective — image
// pairs are independent (robust/ransac.cc:144-148 builds one estimator per call).  Results (stats, models, inlier
// masks) land in the caller's plb_problem array exactly as with plb_ransac_batch.
int plb_ransac_batch_multi(plb_problem *problems, size_t count, int n_gpus, int streams_per_gpu) {
    const int have = plb_device_count();
    if (have == 0) {
        g_err = "no usable CUDA device";
        return PLB_ERR_CUDA;
    }
    if (n_gpus < 0 || n_gpus > have) {
        g_err = "n_gpus out of range";
        return PLB_ERR_ARG;
    }
    if (n_gpus == 0) n_gpus = have;
    std::vector<int> devs(n_gpus);
    for (int d = 0; d < n_gpus; ++d) devs[d] = d;
    return batch_impl(problems, count, devs.data(), n_gpus, streams_per_gpu);
}

// Batch form of the four estimate_* entry points (robust.h:45-46,68-70,112-113,133-134): pixels + cameras in, the
// pre-step of every problem (threshold scaling, camera unprojection on the device, normalize_points on the worker
// threads), LO-RANSAC in lock-step groups per kind (tangent-Sampson problems form their own groups), final bundle and
// un-normalisation.  n_gpus: 0 = all devices of the process, k = the first k, -1 = the calling thread's device only.
int plb_estimate_batch(plb_estimate_problem *problems, size_t count, int n_gpus, int streams_per_gpu) {
    if (count == 0) return PLB_OK;
    if (!problems) {
        g_err = "null argument";
        return PLB_ERR_ARG;
    }
    const int have = plb_device_count();
    if (have == 0) {
        g_err = "no usable CUDA device";
        return PLB_ERR_CUDA;
    }
    if (n_gpus < -1 || n_gpus > have) {
        g_err = "n_gpus out of range";
        return PLB_ERR_ARG;
    }
    std::vector<int> devs;
    if (n_gpus == -1) devs.push_back(g_device);
    else
        for (int d = 0; d < (n_gpus == 0 ? have : n_gpus); ++d) devs.push_back(d);
    std::vector<EstimateJob> jobs(count);
    std::vector<int> rcs(count, PLB_OK);
    std::vector<std::string> msgs(count);
    {
        // the O(N) host part of the pre-step (normalize_points, pixel scaling) in parallel on the worker threads
        const int nt = (int)std::min<size_t>(count, (size_t)std::max(1, usable_cpus()));
        auto prep = [&](int w) {
            for (size_t i = (size_t)w; i < count; i += (size_t)nt) {
                plb_estimate_problem &p = problems[i];
                rcs[i] = estimate_prepare(p.kind, p.a, p.b, (size_t)p.n, &p.camera1, &p.camera2, &p.ransac, &p.bundle,
                                          p.max_error, p.real_focal_check, p.tangent_sampson, p.model, p.inliers, &p.stats,
                                          &p.counters, jobs[i]);
                if (rcs[i] != PLB_OK) msgs[i] = g_err;
            }
        };
        if (nt == 1) prep(0);
        else worker_pool().run(nt, prep);
    }
    for (size_t i = 0; i < count; ++i)
        if (rcs[i] != PLB_OK) {
            g_err = msgs[i];
            for (size_t j = 0; j < count; ++j) problems[j].status = rcs[i];
            return rcs[i];
        }
    // the tasks point into their EstimateJob (normalised copies, scaled pixels), which stays alive until the end of the call
    std::vector<Task> tasks(count);
    std::vector<int> dev_of(count, -1);
    for (size_t i = 0; i < count; ++i) tasks[i] = jobs[i].t;
    const int rc = run_tasks(tasks, dev_of, devs.data(), (int)devs.size(), streams_per_gpu);
    for (size_t i = 0; i < count; ++i) {
        problems[i].status = rc;
        if (rc == PLB_OK) estimate_finish(jobs[i], tasks[i]);
    }
    return rc;
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
    if ((rc = R->soa64.ensure((size_t)n_arr * n_pad)) || (rc = R->soa32.ensure((size_t)n_arr * n_pad)) ||
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
    D.n = n;
    D.n_pad = n_pad;
    D.b_dim = b_dim;
    D.mode = 0;
    D.scale = 1.0;
    PLB_CUDA(cudaMemsetAsync(R->cmax.p, 0, sizeof(float) * 8, E.stream));
    PLB_CUDA(cudaMemcpyAsync(E.tdesc.p, E.h_tdesc.p, sizeof(TransposeDesc), cudaMemcpyHostToDevice, E.stream));
    launch_transpose(E.tdesc.p, 1, n_pad, E.stream);
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
