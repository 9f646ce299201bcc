// poselib_b200 — device-side control of a LO-RANSAC round (sm_90a).
//
// The serial loop of the reference (robust/ransac_impl.h:157-201) draws a sample, scores its models and compares each
// with the running best-minimal state.  Here a whole round of iterations is evaluated at once, and these kernels keep
// the bookkeeping of the round on the device so that the host only replays the handful of models that changed the
// state:
//   k_sample  RandomSampler (robust/sampling.cc:37-61,85-136) for every active problem: splitmix64 is counter based,
//             so lane l of a warp draws sample s+l speculatively from the stream offset it would have if no earlier
//             lane had rejected a duplicate; the prefix up to (and including) the first lane that did reject is final,
//             the rest is redrawn from the corrected offset.  PROSAC subset sizes follow from the growth table.
//   k_select  ordered scan over the round's models of one problem, in (sample, model) order: a model is a CANDIDATE iff
//             its (count, score) record — exact, or an fp32 record with a rigorous error interval — could exceed the
//             running maximum count / fall below the running minimum score of everything before it (two exclusive
//             prefix max/min scans + an ordered compaction).  Also the per-sample prefix sums of the model counts.
//   k_pass1   the same scan over the candidates with their exact fp64 records: the models that improve the
//             best-minimal state (ransac_impl.h:113-124), the last one per sample = an LO trigger (:124,139); writes
//             the records the host replay needs (a few hundred bytes per problem) into mapped pinned memory and the LO
//             job list for k_lm.
#include "kernels.cuh"

namespace plb {

#define CTL_DEV __device__ __forceinline__
constexpr unsigned FULL = 0xffffffffu;
#define D_INF __longlong_as_double(0x7ff0000000000000LL)
#define D_NINF __longlong_as_double((long long)0xfff0000000000000ULL)

// ============================================================================================================
// sampling
// ============================================================================================================
constexpr uint64_t SM_GOLDEN = 0x9e3779b97f4a7c15ULL;
// sampling.cc:37-43: the j-th value (j >= 1) drawn from a generator whose state was `st` is mix(st + j * golden)
CTL_DEV uint64_t splitmix_value(uint64_t st, uint32_t j) {
    uint64_t z = st + (uint64_t)j * SM_GOLDEN;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
    return z ^ (z >> 31);
}
// sampling.cc:50: random_int returns `int`; `% N` happens after the conversion to size_t, i.e. after sign extension:
// a negative v is the 64-bit value 2^64 - |v|.  Both cases reduce to 32-bit remainders, computed without a division
// (Lemire's fastmod: M = floor((2^64 - 1) / n) + 1, a mod n = hi64((M * a mod 2^64) * n), exact for 32-bit a and n).
struct ModN {
    uint64_t M;
    uint32_t n, r64; // r64 = 2^64 mod n
};
CTL_DEV ModN make_mod(uint32_t n) {
    ModN m;
    m.n = n;
    m.M = 0xFFFFFFFFFFFFFFFFull / n + 1ull;
    m.r64 = (uint32_t)((0ull - (uint64_t)n) % (uint64_t)n); // (2^64 - n) mod n
    return m;
}
CTL_DEV uint32_t fastmod(uint32_t a, const ModN &m) { return (uint32_t)__umul64hi(m.M * (uint64_t)a, (uint64_t)m.n); }
CTL_DEV uint32_t draw_mod(uint64_t z, const ModN &m) {
    const int32_t v = (int32_t)(uint32_t)z;
    if (v >= 0) return fastmod((uint32_t)v, m);
    const uint32_t w = fastmod(0u - (uint32_t)v, m); // |v| mod n   (|v| <= 2^31)
    uint32_t r = m.r64 + (m.n - w);                   // (2^64 - |v|) mod n  =  (r64 - w) mod n ;  r < 2n
    if (r >= m.n) r -= m.n;
    if (r >= m.n) r -= m.n;
    return r;
}
// PROSAC subset size after one more sample has been drawn (sampling.cc:97-101); k_pre = sample_k before the draw
CTL_DEV uint32_t prosac_step(const SamplerDev &S, uint32_t sub, uint64_t k_pre) {
    if (k_pre < S.max_prosac) {
        const uint64_t k_post = k_pre + 1;
        if (k_post < S.max_prosac && k_post > S.growth[sub - 1]) {
            if (++sub > S.n) sub = S.n;
        }
    }
    return sub;
}

constexpr int SAMPLE_MAX_K = 7;
__global__ void __launch_bounds__(128) k_sample(const RoundProb *__restrict__ rp, int na, const SamplerDev *__restrict__ st_in,
                                               SamplerDev *__restrict__ st_out, uint32_t *__restrict__ samples) {
    const int w = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (w >= na) return;
    const RoundProb R = rp[w];
    SamplerDev S = st_in[R.pidx];
    const uint32_t K = S.k, N = S.n;
    const bool prosac = (S.flags & 1u) != 0;
    uint64_t state = S.state, sample_k = S.sample_k;
    uint32_t subset = S.subset_sz;
    const ModN modN = make_mod(N);
    int s = 0;
    while (s < R.B) {
        const int my_s = s + lane;
        const bool live = my_s < R.B;
        // which of the window's samples are PROSAC draws (sampling.cc:86): those whose sample_k is below the limit
        uint32_t n_pro_window = 0;
        if (prosac && sample_k < S.max_prosac) {
            const uint64_t r = S.max_prosac - sample_k;
            n_pro_window = r < 32 ? (uint32_t)r : 32u;
        }
        const bool pro = (uint32_t)lane < n_pro_window;
        const uint32_t n_pro_before = (uint32_t)lane < n_pro_window ? (uint32_t)lane : n_pro_window;
        const uint32_t kd = pro ? K - 1 : K; // draws this sample needs when nothing is rejected
        const uint32_t off = n_pro_before * (K - 1) + ((uint32_t)lane - n_pro_before) * K;
        const uint64_t my_k = sample_k + (uint64_t)lane;
        // PROSAC subset size in force when sample_k == my_k (sampling.cc:97-101): the subset grows by at most one per
        // sample, exactly when sample_k passes growth[subset - 1].  With growth[] strictly increasing (flag bit 1) the
        // size at sample_k + l is  subset + #{j >= 0 : growth[subset - 1 + j] < sample_k + l}: lane j looks at entry j,
        // the first lane index l that has passed it is d_j = growth[subset-1+j] - sample_k + 1, one OR-reduction of the
        // bits 1 << d_j and a population count per lane give every lane its subset size.
        uint32_t my_subset = N;
        if (n_pro_window) {
            if (S.flags & 2u) {
                uint32_t bit = 0u;
                const uint64_t gi = (uint64_t)subset - 1ull + (uint64_t)lane;
                if (gi < (uint64_t)N) {
                    const uint64_t g = S.growth[gi];
                    if (g < sample_k) bit = 1u; // already passed (cannot happen for j = 0; kept for safety)
                    else if (g - sample_k + 1ull < 32ull) bit = 1u << (uint32_t)(g - sample_k + 1ull);
                }
                const uint32_t passed = __reduce_or_sync(FULL, bit);
                const uint32_t le = (lane == 31) ? 0xffffffffu : ((2u << lane) - 1u);
                my_subset = subset + (uint32_t)__popc(passed & le);
                if (my_subset > N) my_subset = N;
            } else { // general rule, step by step
                uint32_t sub = subset;
                for (uint64_t kk = sample_k; kk < my_k; ++kk) sub = prosac_step(S, sub, kk);
                my_subset = sub;
            }
        }
        uint32_t idx[SAMPLE_MAX_K];
#pragma unroll
        for (int i = 0; i < SAMPLE_MAX_K; ++i) idx[i] = 0xffffffffu - (uint32_t)i;
        uint32_t c = kd;
        if (live) {
            // sampling.cc:87 draws from the first subset_sz - 1 points
            const ModN mod = pro ? make_mod(my_subset - 1) : modN;
            // fast path: the first kd values of the stream, all computed before any is compared (independent chains)
            bool distinct = true;
#pragma unroll
            for (int i = 0; i < SAMPLE_MAX_K; ++i)
                if ((uint32_t)i < kd) idx[i] = draw_mod(splitmix_value(state, off + 1u + (uint32_t)i), mod);
#pragma unroll
            for (int i = 1; i < SAMPLE_MAX_K; ++i)
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if ((uint32_t)i < kd) distinct &= (idx[i] != idx[j]);
            if (!distinct) {
                // sampling.cc:46-61: redraw while the index is already in the sample
                c = 0;
#pragma unroll
                for (int i = 0; i < SAMPLE_MAX_K; ++i) {
                    if ((uint32_t)i < kd) {
                        for (;;) {
                            ++c;
                            const uint32_t v = draw_mod(splitmix_value(state, off + c), mod);
                            bool dup = false;
#pragma unroll
                            for (int j = 0; j < SAMPLE_MAX_K; ++j)
                                if (j < i) dup |= (idx[j] == v);
                            if (!dup) {
                                idx[i] = v;
                                break;
                            }
                        }
                    }
                }
            }
            if (pro) { // sampling.cc:88: the last point of the subset is forced into the sample
#pragma unroll
                for (int i = 0; i < SAMPLE_MAX_K; ++i)
                    if ((uint32_t)i == K - 1) idx[i] = my_subset - 1;
            }
        }
        const unsigned bad = __ballot_sync(FULL, live && c != kd);
        int f = bad ? (__ffs((int)bad) - 1) : 31; // last lane whose stream offset was right
        if (f > R.B - s - 1) f = R.B - s - 1;
        if (live && lane <= f) {
            uint32_t *dst = samples + ((size_t)R.g0 + (size_t)my_s) * K;
#pragma unroll
            for (int i = 0; i < SAMPLE_MAX_K; ++i)
                if ((uint32_t)i < K) dst[i] = idx[i];
        }
        const uint32_t tot = __shfl_sync(FULL, off + c, f);
        const uint32_t next_sub = (pro && live) ? prosac_step(S, my_subset, my_k) : subset;
        const uint32_t sub_f = __shfl_sync(FULL, next_sub, f);
        state += (uint64_t)tot * SM_GOLDEN;
        if (n_pro_window) {
            const uint32_t adv = (uint32_t)(f + 1) < n_pro_window ? (uint32_t)(f + 1) : n_pro_window;
            sample_k += adv;
            if ((uint32_t)f < n_pro_window) subset = sub_f;
        }
        s += f + 1;
    }
    if (lane == 0) {
        S.state = state;
        S.sample_k = sample_k;
        S.subset_sz = subset;
        st_out[R.pidx] = S;
    }
}
void launch_sample(const RoundProb *rp, int na, const SamplerDev *st_in, SamplerDev *st_out, uint32_t *samples,
                   cudaStream_t stream) {
    if (na <= 0) return;
    k_sample<<<(na + 3) / 4, 128, 0, stream>>>(rp, na, st_in, st_out, samples);
}

// ============================================================================================================
// candidate selection: ordered scan per problem
// ============================================================================================================
constexpr int SEL_THREADS = 256, SEL_WARPS = SEL_THREADS / 32, SEL_SPT = 4;

// Interval [c_lo, c_hi] x [s_lo, s_hi] that contains the exact (fp64) record of model `slot`.
CTL_DEV void model_interval(const SelectArgs &A, int slot, double &c_lo, double &c_hi, double &s_lo, double &s_hi,
                            bool &usable) {
    if (A.mode == 0) {
        const double c = (double)A.counts[slot], s = A.scores[slot];
        c_lo = c_hi = c;
        s_lo = s_hi = s; // NaN scores never compare "better" and are ignored by fmin, exactly as on the host
        usable = true;
        return;
    }
    const double c = (double)A.fcounts[slot], s = (double)A.fscores[slot];
    const double b = (double)A.fborder[slot], e = (double)A.ferr[slot];
    usable = isfinite(s) && isfinite(e);
    c_lo = c - b;
    c_hi = c + b;
    s_lo = s - e;
    s_hi = s + e;
}

struct SelScan {
    double lb[SEL_WARPS], ub[SEL_WARPS];
    int n[SEL_WARPS];
    double tot_lb, tot_ub;
    int tot_n;
};
// exclusive block scan of (max, min, sum); every thread also gets the block totals
CTL_DEV void block_scan3(SelScan *S, double &lb, double &ub, int &n, double &tot_lb, double &tot_ub, int &tot_n) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double ilb = lb, iub = ub;
    int in = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double a = __shfl_up_sync(FULL, ilb, o), b = __shfl_up_sync(FULL, iub, o);
        const int c = __shfl_up_sync(FULL, in, o);
        if (lane >= o) {
            ilb = fmax(ilb, a);
            iub = fmin(iub, b);
            in += c;
        }
    }
    __syncthreads(); // S may still be read by the previous call
    if (lane == 31) {
        S->lb[warp] = ilb;
        S->ub[warp] = iub;
        S->n[warp] = in;
    }
    __syncthreads();
    double plb = D_NINF, pub = D_INF; // -"inf" / +inf
    int pn = 0;
    for (int w2 = 0; w2 < warp; ++w2) {
        plb = fmax(plb, S->lb[w2]);
        pub = fmin(pub, S->ub[w2]);
        pn += S->n[w2];
    }
    double tl = plb, tu = pub;
    int tn = pn;
    for (int w2 = warp; w2 < SEL_WARPS; ++w2) {
        tl = fmax(tl, S->lb[w2]);
        tu = fmin(tu, S->ub[w2]);
        tn += S->n[w2];
    }
    // exclusive value of this thread = prefix of earlier warps combined with earlier lanes of this warp
    double elb = __shfl_up_sync(FULL, ilb, 1), eub = __shfl_up_sync(FULL, iub, 1);
    int en = __shfl_up_sync(FULL, in, 1);
    if (lane == 0) {
        elb = D_NINF;
        eub = D_INF;
        en = 0;
    }
    lb = fmax(plb, elb);
    ub = fmin(pub, eub);
    n = pn + en;
    tot_lb = tl;
    tot_ub = tu;
    tot_n = tn;
}

__global__ void __launch_bounds__(SEL_THREADS) k_select(const SelectArgs A) {
    __shared__ SelScan scan;
    const int a = blockIdx.x;
    const RoundProb R = A.rp[a];
    const int tid = threadIdx.x;
    double carry_lb = R.lb0, carry_ub = R.ub0;
    int carry_nm = 0, carry_nc = 0;
    for (int cb = 0; cb < R.B; cb += SEL_THREADS * SEL_SPT) {
        const int s0 = cb + tid * SEL_SPT;
        int nm[SEL_SPT], fs[SEL_SPT];
#pragma unroll
        for (int q = 0; q < SEL_SPT; ++q) {
            const int s = s0 + q;
            nm[q] = (s < R.B) ? A.n_models[R.g0 + s] : 0;
            fs[q] = (s < R.B) ? A.first_slot[R.g0 + s] : 0;
        }
        // phase 1: what this thread's models contribute to the running bounds
        double lb = D_NINF, ub = D_INF;
        int n = 0;
#pragma unroll
        for (int q = 0; q < SEL_SPT; ++q) {
            for (int m = 0; m < nm[q]; ++m) {
                double c_lo, c_hi, s_lo, s_hi;
                bool usable;
                model_interval(A, fs[q] + m, c_lo, c_hi, s_lo, s_hi, usable);
                if (usable) {
                    lb = fmax(lb, c_lo);
                    ub = fmin(ub, s_hi);
                }
            }
            n += nm[q];
        }
        double tot_lb, tot_ub;
        int tot_n;
        block_scan3(&scan, lb, ub, n, tot_lb, tot_ub, tot_n);
        // phase 2: candidates, with the bounds of everything before each model
        double LB = fmax(carry_lb, lb), UB = fmin(carry_ub, ub);
        int run_n = carry_nm + n;
        unsigned long long cm[SEL_SPT];
        int nc = 0;
#pragma unroll
        for (int q = 0; q < SEL_SPT; ++q) {
            cm[q] = 0ull;
            for (int m = 0; m < nm[q]; ++m) {
                double c_lo, c_hi, s_lo, s_hi;
                bool usable;
                model_interval(A, fs[q] + m, c_lo, c_hi, s_lo, s_hi, usable);
                const bool cand = !usable || (c_hi > LB) || (s_lo < UB);
                if (cand) {
                    cm[q] |= 1ull << m;
                    ++nc;
                }
                if (usable) {
                    LB = fmax(LB, c_lo);
                    UB = fmin(UB, s_hi);
                }
            }
            run_n += nm[q];
            if (s0 + q < R.B) A.prefix[R.g0 + s0 + q] = run_n;
        }
        double d0 = D_NINF, d1 = D_INF, t0, t1;
        int pos = nc, tot_c;
        block_scan3(&scan, d0, d1, pos, t0, t1, tot_c);
        // phase 3: ordered compaction into the problem's candidate segment
        int w = R.seg_base + carry_nc + pos;
#pragma unroll
        for (int q = 0; q < SEL_SPT; ++q) {
            unsigned long long mk = cm[q];
            while (mk) {
                const int m = __ffsll((long long)mk) - 1;
                mk &= mk - 1ull;
                A.cand_slot[w] = fs[q] + m;
                A.cand_sample[w] = s0 + q;
                ++w;
            }
        }
        carry_lb = fmax(carry_lb, tot_lb);
        carry_ub = fmin(carry_ub, tot_ub);
        carry_nm += tot_n;
        carry_nc += tot_c;
    }
    if (tid == 0) {
        A.n_cand[a] = carry_nc;
        A.n_models_tot[a] = carry_nm;
    }
}
void launch_select(const SelectArgs &A, cudaStream_t stream) {
    if (A.na <= 0) return;
    k_select<<<A.na, SEL_THREADS, 0, stream>>>(A);
}

// ============================================================================================================
// exact pass over the candidates: improving models, LO triggers, host records
// ============================================================================================================
CTL_DEV double warp_excl_max(double v, int lane, double &total) {
    double inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double t = __shfl_up_sync(FULL, inc, o);
        if (lane >= o) inc = fmax(inc, t);
    }
    total = __shfl_sync(FULL, inc, 31);
    double e = __shfl_up_sync(FULL, inc, 1);
    if (lane == 0) e = D_NINF;
    return e;
}
CTL_DEV double warp_excl_min(double v, int lane, double &total) {
    double inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double t = __shfl_up_sync(FULL, inc, o);
        if (lane >= o) inc = fmin(inc, t);
    }
    total = __shfl_sync(FULL, inc, 31);
    double e = __shfl_up_sync(FULL, inc, 1);
    if (lane == 0) e = D_INF;
    return e;
}

__global__ void __launch_bounds__(128) k_pass1(const Pass1Args A) {
    const int a = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (a >= A.na) return;
    const RoundProb R = A.rp[a];
    const int nc = A.n_cand[a];
    int *cslot = A.cand_slot + R.seg_base, *csmp = A.cand_sample + R.seg_base;
    // ---- improving models: count > running max or score < running min of everything before (ransac_impl.h:113-124);
    //      models that were not candidates cannot move either running value
    double bc = R.lb0, bs = R.ub0;
    int n_imp = 0;
    for (int c0 = 0; c0 < nc; c0 += 32) {
        const int i = c0 + lane;
        const bool valid = i < nc;
        int slot = 0, smp = 0;
        double c = -1.0, s = D_INF;
        if (valid) {
            slot = cslot[i];
            smp = csmp[i];
            c = (double)A.counts[slot];
            s = A.scores[slot];
        }
        double tc, ts;
        const double ec = fmax(bc, warp_excl_max(c, lane, tc));
        const double es = fmin(bs, warp_excl_min(s, lane, ts));
        const bool imp = valid && ((c > ec) || (s < es));
        const unsigned mk = __ballot_sync(FULL, imp);
        if (imp) {
            const int pos = n_imp + __popc(mk & ((1u << lane) - 1u));
            cslot[pos] = slot; // in place: pos <= i and every read of this chunk is in registers
            csmp[pos] = smp;
        }
        __syncwarp();
        n_imp += __popc(mk);
        bc = fmax(bc, tc);
        bs = fmin(bs, ts);
    }
    // ---- LO triggers: the last improving model of a sample (ransac_impl.h:124,139)
    int n_trig = 0;
    for (int c0 = 0; c0 < n_imp; c0 += 32) {
        const int i = c0 + lane;
        bool trig = false;
        if (i < n_imp) trig = (i + 1 == n_imp) || (csmp[i + 1] != csmp[i]);
        n_trig += __popc(__ballot_sync(FULL, trig));
    }
    int imp_base = 0, trig_base = 0;
    if (lane == 0) {
        imp_base = n_imp ? atomicAdd(A.ctl + CTL_IMP_TOTAL, n_imp) : 0;
        trig_base = n_trig ? atomicAdd(A.ctl + CTL_JOB_TOTAL, n_trig) : 0;
        int fl = 0;
        if (imp_base + n_imp > A.imp_cap) fl |= FLAG_IMP_OVERFLOW;
        if (trig_base + n_trig > A.job_cap) fl |= FLAG_JOB_OVERFLOW;
        if (fl) atomicOr(A.ctl + CTL_FLAGS, fl);
        SelHeader h;
        h.n_models = A.n_models_tot[a];
        h.n_cand = nc;
        h.n_imp = n_imp;
        h.imp_base = imp_base;
        h.n_trig = n_trig;
        h.trig_base = trig_base;
        A.hdr[a] = h;
    }
    imp_base = __shfl_sync(FULL, imp_base, 0);
    trig_base = __shfl_sync(FULL, trig_base, 0);
    if (imp_base + n_imp > A.imp_cap || trig_base + n_trig > A.job_cap) return; // the host redoes the round
    int tp = 0;
    for (int c0 = 0; c0 < n_imp; c0 += 32) {
        const int i = c0 + lane;
        bool trig = false;
        int slot = 0;
        if (i < n_imp) {
            slot = cslot[i];
            trig = (i + 1 == n_imp) || (csmp[i + 1] != csmp[i]);
            ImpRec *r = A.imp + imp_base + i;
            r->sample = csmp[i];
            r->count = A.counts[slot];
            r->score = A.scores[slot];
            const double *m = A.models + (size_t)slot * A.msz;
            for (int k = 0; k < A.msz; ++k) r->model[k] = m[k];
        }
        const unsigned mk = __ballot_sync(FULL, trig);
        if (trig) {
            LoJobSrc j;
            j.pidx = R.pidx;
            j.slot = slot;
            A.job_src[trig_base + tp + __popc(mk & ((1u << lane) - 1u))] = j;
        }
        tp += __popc(mk);
    }
}
void launch_pass1(const Pass1Args &A, cudaStream_t stream) {
    if (A.na <= 0) return;
    k_pass1<<<(A.na + 3) / 4, 128, 0, stream>>>(A);
}

} // namespace plb
