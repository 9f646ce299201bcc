// The device control of a round (control.cu) and the bounds of its buffers, for tests/test_round_control.py.
// Every output buffer sits between guard regions filled with the byte 0xA5 before the launches; every dump includes
// them, so the test sees any store outside a buffer or outside a problem's segment.
//
// Usage: round_control_device_test select <input> <output>
//   launch_select on synthetic records, then the exact record of every slot that is not a candidate is overwritten
//   with a poison value (count 0xFFFFFFFF, score -inf), then launch_pass1, then (lm_n > 0) launch_lm_round over the
//   job list with a dummy template (max_iterations 0) on a small PnP problem.
//   Input: int mode, imp_cap, job_cap, na, n_total, n_slots, lm_n, sentinel_slot;
//          RoundProb[na] (raw structs); int n_models[n_total]; int first_slot[n_total];
//          per slot: uint32 counts[S]; double scores[S]; uint32 fcounts[S], fborder[S]; float fscores[S], ferr[S];
//          double models[S * 7];  lm_n > 0: double x[2 lm_n], X[3 lm_n] (AoS).
//   job_src is pre-filled with the valid job {pidx 0, slot sentinel_slot} when lm_n > 0.
//   Output (guarded dumps, G = SEL_GUARD elements each side): after select: prefix, cand_slot, cand_sample, n_cand,
//          n_models_tot; after pass1: cand_slot, cand_sample, ctl, hdr, imp, job_src; lm_n > 0: LmJobOut[job_cap].
//
// Usage: round_control_device_test hyp <input> <output>
//   launch_hypotheses (solve + exact scoring or fp32 screening) on real problems with given samples, once per
//   segment-capacity configuration.  Problem a's segment starts at seg_base[a] and is followed by a gap of MAXM * B[a]
//   slots; the per-slot buffers have MAXM * n_total guard slots on each side.
//   Input: int kind, mode, na, n_cfg; per problem: int n, double sq_thr, double a[2n], b[b_dim n] (AoS), int B,
//          uint32 samples[B * K]; per config: int seg_cap[na].
//   Output per config: int overflow, int seg_base[na], int prob_count[na], int guard (slots per side), guarded
//          n_models, first_slot (SEL_GUARD), guarded per-slot counts, scores, models (MSZ per slot), model_prob and,
//          mode 1, fcounts, fscores, fborder, ferr, fctx (scr::CTX_FLOATS per slot).
// Little-endian binary, int = int32.
#include "../poselib_b200/csrc/kernels.cu"
#include "../poselib_b200/csrc/control.cu"
#include <cstdio>
#include <cstring>
#include <vector>

using namespace plb;

#define CK(x)                                                                                                          \
    do {                                                                                                               \
        cudaError_t e_ = (x);                                                                                          \
        if (e_ != cudaSuccess) {                                                                                       \
            std::fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));                   \
            std::exit(2);                                                                                              \
        }                                                                                                              \
    } while (0)

constexpr size_t SEL_GUARD = 64;
constexpr int GUARD_BYTE = 0xA5;

static FILE *fin, *fout;
template <class T> static T rd() {
    T v;
    if (std::fread(&v, sizeof(T), 1, fin) != 1) {
        std::fprintf(stderr, "short input\n");
        std::exit(3);
    }
    return v;
}
template <class T> static void rdv(std::vector<T> &v, size_t n) {
    v.resize(n);
    if (n && std::fread(v.data(), sizeof(T), n, fin) != n) {
        std::fprintf(stderr, "short input\n");
        std::exit(3);
    }
}
template <class T> static void wr(const T *p, size_t n) { std::fwrite(p, sizeof(T), n, fout); }

// n elements between two guard regions of g elements, all bytes GUARD_BYTE
template <class T> struct GBuf {
    T *base = nullptr, *p = nullptr;
    size_t n = 0, g = 0;
};
template <class T> static GBuf<T> galloc(size_t n, size_t g) {
    GBuf<T> b;
    b.n = n;
    b.g = g;
    CK(cudaMalloc(&b.base, sizeof(T) * (n + 2 * g)));
    CK(cudaMemset(b.base, GUARD_BYTE, sizeof(T) * (n + 2 * g)));
    b.p = b.base + g;
    return b;
}
template <class T> static GBuf<T> gput(const std::vector<T> &v, size_t g) {
    GBuf<T> b = galloc<T>(v.size(), g);
    if (!v.empty()) CK(cudaMemcpy(b.p, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
    return b;
}
template <class T> static std::vector<T> gget(const GBuf<T> &b) { // interior only
    std::vector<T> v(b.n);
    if (b.n) CK(cudaMemcpy(v.data(), b.p, sizeof(T) * b.n, cudaMemcpyDeviceToHost));
    return v;
}
template <class T> static void gdump(const GBuf<T> &b) { // guards included
    std::vector<T> v(b.n + 2 * b.g);
    CK(cudaMemcpy(v.data(), b.base, sizeof(T) * v.size(), cudaMemcpyDeviceToHost));
    wr(v.data(), v.size());
}
template <class T> static void gfree(GBuf<T> &b) {
    if (b.base) CK(cudaFree(b.base));
    b.base = b.p = nullptr;
}

// ---- caller AoS doubles -> resident SoA arrays of one problem set (launch_transpose, mode 0) ----------------------
struct Problems {
    std::vector<ProblemDev> pd;
    std::vector<void *> allocs;
    int max_n_pad = 0;
};
static Problems upload_problems(int kind, const std::vector<std::vector<double>> &as,
                                const std::vector<std::vector<double>> &bs, const std::vector<double> &thr) {
    const int np = (int)as.size(), b_dim = kind == KIND_PNP ? 3 : 2, narr = 2 + b_dim;
    Problems P;
    std::vector<TransposeDesc> td(np);
    P.pd.resize(np);
    for (int i = 0; i < np; ++i) {
        const int n = (int)(as[i].size() / 2), n_pad = (n + 31) & ~31;
        P.max_n_pad = std::max(P.max_n_pad, n_pad);
        double *a, *b, *s64;
        float *s32, *cmax;
        CK(cudaMalloc(&a, sizeof(double) * (as[i].size() + 1)));
        CK(cudaMalloc(&b, sizeof(double) * (bs[i].size() + 1)));
        CK(cudaMalloc(&s64, sizeof(double) * narr * n_pad));
        CK(cudaMalloc(&s32, sizeof(float) * narr * n_pad));
        CK(cudaMalloc(&cmax, sizeof(float) * 5));
        CK(cudaMemcpy(a, as[i].data(), sizeof(double) * as[i].size(), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(b, bs[i].data(), sizeof(double) * bs[i].size(), cudaMemcpyHostToDevice));
        CK(cudaMemset(cmax, 0, sizeof(float) * 5));
        P.allocs.insert(P.allocs.end(), {(void *)a, (void *)b, (void *)s64, (void *)s32, (void *)cmax});
        TransposeDesc &D = td[i];
        std::memset(&D, 0, sizeof(D));
        D.a = a;
        D.b = b;
        D.s64 = s64;
        D.s32 = s32;
        D.cmax = cmax;
        D.n = n;
        D.n_pad = n_pad;
        D.b_dim = b_dim;
        D.mode = 0;
        D.scale = 1.0;
        D.cam_a.model = D.cam_b.model = CAMM_NULL;
        ProblemDev &Q = P.pd[i];
        std::memset(&Q, 0, sizeof(Q));
        Q.cam[0].model = Q.cam[1].model = CAMM_NULL;
        Q.n = n;
        Q.kind = kind;
        Q.sq_thr = thr[i];
        Q.n_pad = n_pad;
        Q.cmax = cmax;
        for (int c = 0; c < narr; ++c) {
            Q.p[c] = s64 + (size_t)c * n_pad;
            Q.f[c] = s32 + (size_t)c * n_pad;
        }
    }
    TransposeDesc *d_td;
    CK(cudaMalloc(&d_td, sizeof(TransposeDesc) * np));
    CK(cudaMemcpy(d_td, td.data(), sizeof(TransposeDesc) * np, cudaMemcpyHostToDevice));
    launch_transpose(d_td, np, P.max_n_pad, false, 0);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    CK(cudaFree(d_td));
    return P;
}

// ============================================================================================================
// select: k_select, poison, k_pass1 [, k_lm over the job list]
// ============================================================================================================
static void run_select() {
    const int mode = rd<int>(), imp_cap = rd<int>(), job_cap = rd<int>(), na = rd<int>(), n_total = rd<int>();
    const int S = rd<int>(), lm_n = rd<int>(), sentinel_slot = rd<int>();
    constexpr int MSZ = 7;
    std::vector<RoundProb> rp;
    rdv(rp, na);
    std::vector<int> n_models, first_slot;
    rdv(n_models, n_total);
    rdv(first_slot, n_total);
    std::vector<uint32_t> counts, fcounts, fborder;
    std::vector<double> scores, models;
    std::vector<float> fscores, ferr;
    rdv(counts, S);
    rdv(scores, S);
    rdv(fcounts, S);
    rdv(fborder, S);
    rdv(fscores, S);
    rdv(ferr, S);
    rdv(models, (size_t)S * MSZ);
    std::vector<double> lx, lX;
    if (lm_n > 0) {
        rdv(lx, 2 * (size_t)lm_n);
        rdv(lX, 3 * (size_t)lm_n);
    }
    const size_t G = SEL_GUARD;
    auto d_rp = gput(rp, G);
    auto d_nm = gput(n_models, G), d_fs = gput(first_slot, G);
    auto d_counts = gput(counts, G), d_fcounts = gput(fcounts, G), d_fborder = gput(fborder, G);
    auto d_scores = gput(scores, G), d_models = gput(models, G);
    auto d_fscores = gput(fscores, G), d_ferr = gput(ferr, G);
    auto d_prefix = galloc<int>(n_total, G), d_cslot = galloc<int>(S, G), d_csmp = galloc<int>(S, G);
    auto d_ncand = galloc<int>(na, G), d_nmt = galloc<int>(na, G);
    SelectArgs A;
    A.rp = d_rp.p;
    A.na = na;
    A.mode = mode;
    A.n_models = d_nm.p;
    A.first_slot = d_fs.p;
    A.fcounts = d_fcounts.p;
    A.fscores = d_fscores.p;
    A.fborder = d_fborder.p;
    A.ferr = d_ferr.p;
    A.counts = d_counts.p;
    A.scores = d_scores.p;
    A.prefix = d_prefix.p;
    A.cand_slot = d_cslot.p;
    A.cand_sample = d_csmp.p;
    A.n_cand = d_ncand.p;
    A.n_models_tot = d_nmt.p;
    launch_select(A, 0);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    gdump(d_prefix);
    gdump(d_cslot);
    gdump(d_csmp);
    gdump(d_ncand);
    gdump(d_nmt);

    // poison every slot k_pass1 has no business reading: it may only read the exact records of candidates
    {
        const std::vector<int> cs = gget(d_cslot), nc = gget(d_ncand);
        std::vector<char> is_cand(S, 0);
        for (int a = 0; a < na; ++a)
            for (int j = 0; j < nc[a]; ++j) {
                const int s = cs[rp[a].seg_base + j];
                if (s >= 0 && s < S) is_cand[s] = 1;
            }
        std::vector<uint32_t> pc = counts;
        std::vector<double> ps = scores;
        for (int s = 0; s < S; ++s)
            if (!is_cand[s]) {
                pc[s] = 0xFFFFFFFFu;
                ps[s] = -INFINITY;
            }
        CK(cudaMemcpy(d_counts.p, pc.data(), sizeof(uint32_t) * S, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_scores.p, ps.data(), sizeof(double) * S, cudaMemcpyHostToDevice));
    }

    auto d_ctl = galloc<int>(CTL_WORDS, G);
    CK(cudaMemset(d_ctl.p, 0, sizeof(int) * CTL_WORDS));
    auto d_hdr = galloc<SelHeader>(na, G);
    auto d_imp = galloc<ImpRec>(imp_cap, G);
    auto d_job = galloc<LoJobSrc>(job_cap, G);
    if (lm_n > 0) {
        std::vector<LoJobSrc> fill(job_cap);
        for (auto &j : fill) {
            j.pidx = 0;
            j.slot = sentinel_slot;
        }
        CK(cudaMemcpy(d_job.p, fill.data(), sizeof(LoJobSrc) * job_cap, cudaMemcpyHostToDevice));
    }
    Pass1Args B;
    B.rp = d_rp.p;
    B.na = na;
    B.cand_slot = d_cslot.p;
    B.cand_sample = d_csmp.p;
    B.n_cand = d_ncand.p;
    B.n_models_tot = d_nmt.p;
    B.counts = d_counts.p;
    B.scores = d_scores.p;
    B.models = d_models.p;
    B.msz = MSZ;
    B.ctl = d_ctl.p;
    B.imp_cap = imp_cap;
    B.job_cap = job_cap;
    B.hdr = d_hdr.p;
    B.imp = d_imp.p;
    B.job_src = d_job.p;
    launch_pass1(B, 0);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    gdump(d_cslot);
    gdump(d_csmp);
    gdump(d_ctl);
    gdump(d_hdr);
    gdump(d_imp);
    gdump(d_job);

    if (lm_n > 0) {
        // one small PnP problem; every problem's LO template is the same dummy job on it (no iteration)
        Problems P = upload_problems(KIND_PNP, {lx}, {lX}, {1e-4});
        ProblemDev *d_pd;
        CK(cudaMalloc(&d_pd, sizeof(ProblemDev)));
        CK(cudaMemcpy(d_pd, P.pd.data(), sizeof(ProblemDev), cudaMemcpyHostToDevice));
        LmJob t;
        std::memset(&t, 0, sizeof(t));
        t.pidx = 0;
        t.cam_refine = 0;
        t.mask_off = -1;
        t.scratch_off = 0;
        t.prm.max_iterations = 0;
        t.prm.loss_type = 0;
        t.prm.loss_scale = 1.0;
        t.prm.gradient_tol = 1e-12;
        t.prm.step_tol = 1e-8;
        t.prm.relative_cost_tol = 1e-10;
        t.prm.initial_lambda = 1e-3;
        t.prm.min_lambda = 1e-10;
        t.prm.max_lambda = 1e10;
        t.prm.subset_mode = 0;
        t.prm.score_after = 0;
        std::vector<LmJob> tmpl(na, t);
        auto d_tmpl = gput(tmpl, 0);
        auto d_out = galloc<LmJobOut>(job_cap, G);
        int *d_scratch;
        const int est = 64;
        const int nclu = lm_round_max_clusters(KIND_PNP, est, lm_n);
        CK(cudaMalloc(&d_scratch, sizeof(int) * (size_t)nclu * P.max_n_pad + 1));
        launch_lm_round(KIND_PNP, d_pd, d_tmpl.p, d_job.p, d_models.p, d_ctl.p + CTL_JOB_TOTAL, job_cap, est, lm_n, d_scratch,
                        P.max_n_pad, d_out.p, 0);
        CK(cudaGetLastError());
        CK(cudaDeviceSynchronize());
        gdump(d_out);
        gfree(d_out);
        gfree(d_tmpl);
        CK(cudaFree(d_scratch));
        CK(cudaFree(d_pd));
        for (void *p : P.allocs) CK(cudaFree(p));
    }
    for (auto *b : {&d_nm, &d_fs, &d_prefix, &d_cslot, &d_csmp, &d_ncand, &d_nmt, &d_ctl}) gfree(*b);
    gfree(d_rp);
    gfree(d_counts);
    gfree(d_fcounts);
    gfree(d_fborder);
    gfree(d_scores);
    gfree(d_models);
    gfree(d_fscores);
    gfree(d_ferr);
    gfree(d_hdr);
    gfree(d_imp);
    gfree(d_job);
}

// ============================================================================================================
// hyp: launch_hypotheses with given samples and segment capacities
// ============================================================================================================
static void run_hyp() {
    const int kind = rd<int>(), mode = rd<int>(), na = rd<int>(), n_cfg = rd<int>();
    const int K = kind_sample_size(kind), b_dim = kind == KIND_PNP ? 3 : 2;
    const int MAXM = kind_max_models(kind), MSZ = kind_model_size(kind);
    std::vector<std::vector<double>> as(na), bs(na);
    std::vector<double> thr(na);
    std::vector<int> Bs(na), g_off(na + 1, 0);
    std::vector<uint32_t> samples;
    for (int i = 0; i < na; ++i) {
        const int n = rd<int>();
        thr[i] = rd<double>();
        rdv(as[i], 2 * (size_t)n);
        rdv(bs[i], (size_t)b_dim * n);
        Bs[i] = rd<int>();
        std::vector<uint32_t> s;
        rdv(s, (size_t)Bs[i] * K);
        samples.insert(samples.end(), s.begin(), s.end());
        g_off[i + 1] = g_off[i] + Bs[i];
    }
    const int n_total = g_off[na];
    Problems P = upload_problems(kind, as, bs, thr);
    ProblemDev *d_pd;
    CK(cudaMalloc(&d_pd, sizeof(ProblemDev) * na));
    CK(cudaMemcpy(d_pd, P.pd.data(), sizeof(ProblemDev) * na, cudaMemcpyHostToDevice));
    std::vector<int> act(na);
    for (int i = 0; i < na; ++i) act[i] = i;
    auto d_act = gput(act, 0), d_goff = gput(g_off, 0);
    auto d_samples = gput(samples, 0);
    for (int c = 0; c < n_cfg; ++c) {
        std::vector<int> cap;
        rdv(cap, na);
        std::vector<int> seg(na);
        size_t slots = 0;
        int max_cap = 0;
        for (int i = 0; i < na; ++i) {
            seg[i] = (int)slots;
            slots += (size_t)cap[i] + (size_t)MAXM * Bs[i]; // the segment, then a gap that only an overrun reaches
            max_cap = std::max(max_cap, cap[i]);
        }
        const size_t G = (size_t)MAXM * n_total;
        auto d_seg = gput(seg, 0), d_cap = gput(cap, 0);
        auto d_pc = galloc<int>(na, 0);
        auto d_ovf = galloc<int>(1, 0);
        CK(cudaMemset(d_ovf.p, 0, sizeof(int)));
        auto d_nm = galloc<int>(n_total, SEL_GUARD), d_fs = galloc<int>(n_total, SEL_GUARD);
        auto d_counts = galloc<uint32_t>(slots, G), d_fcounts = galloc<uint32_t>(slots, G), d_fborder = galloc<uint32_t>(slots, G);
        auto d_scores = galloc<double>(slots, G);
        auto d_models = galloc<double>(slots * MSZ, G * MSZ);
        auto d_mp = galloc<int>(slots, G);
        auto d_fscores = galloc<float>(slots, G), d_ferr = galloc<float>(slots, G);
        auto d_fctx = galloc<float>(slots * scr::CTX_FLOATS, G * scr::CTX_FLOATS);
        GBuf<double> s5[4];
        GBuf<int> s5n;
        RoundDesc R;
        std::memset(&R, 0, sizeof(R));
        R.probs = d_pd;
        R.active = d_act.p;
        R.g_off = d_goff.p;
        R.n_active = na;
        R.samples = d_samples.p;
        R.n_total = n_total;
        HypOut out;
        std::memset(&out, 0, sizeof(out));
        out.n_models = d_nm.p;
        out.first_slot = d_fs.p;
        out.seg_base = d_seg.p;
        out.seg_cap = d_cap.p;
        out.prob_count = d_pc.p;
        out.max_seg_cap = max_cap;
        out.overflow = d_ovf.p;
        out.counts = d_counts.p;
        out.scores = d_scores.p;
        out.models = d_models.p;
        out.model_prob = d_mp.p;
        if (mode == 1) {
            out.fcounts = d_fcounts.p;
            out.fscores = d_fscores.p;
            out.fborder = d_fborder.p;
            out.ferr = d_ferr.p;
        }
        if (kind_is_relpose(kind)) {
            const size_t per[4] = {105, 100, 11, 10};
            for (int k = 0; k < 4; ++k) s5[k] = galloc<double>(per[k] * n_total, 0);
            s5n = galloc<int>(n_total, 0);
            out.s5_blk = s5[0].p;
            out.s5_park = s5[1].p;
            out.s5_cpoly = s5[2].p;
            out.s5_roots = s5[3].p;
            out.s5_nroots = s5n.p;
        }
        launch_hypotheses(kind, R, out, mode, P.max_n_pad, d_fctx.p, 0);
        CK(cudaGetLastError());
        CK(cudaDeviceSynchronize());
        const std::vector<int> ovf = gget(d_ovf), pc = gget(d_pc);
        const int guard = (int)G;
        wr(ovf.data(), 1);
        wr(seg.data(), na);
        wr(pc.data(), na);
        wr(&guard, 1);
        const int slots_i = (int)slots;
        wr(&slots_i, 1);
        gdump(d_nm);
        gdump(d_fs);
        gdump(d_counts);
        gdump(d_scores);
        gdump(d_models);
        gdump(d_mp);
        if (mode == 1) {
            gdump(d_fcounts);
            gdump(d_fscores);
            gdump(d_fborder);
            gdump(d_ferr);
            gdump(d_fctx);
        }
        for (auto *b : {&d_seg, &d_cap, &d_pc, &d_ovf, &d_nm, &d_fs, &d_mp}) gfree(*b);
        gfree(d_counts);
        gfree(d_fcounts);
        gfree(d_fborder);
        gfree(d_scores);
        gfree(d_models);
        gfree(d_fscores);
        gfree(d_ferr);
        gfree(d_fctx);
        for (auto &b : s5) gfree(b);
        gfree(s5n);
    }
    gfree(d_act);
    gfree(d_goff);
    gfree(d_samples);
    CK(cudaFree(d_pd));
    for (void *p : P.allocs) CK(cudaFree(p));
}

int main(int argc, char **argv) {
    if (argc != 4) {
        std::fprintf(stderr, "usage: %s select|hyp <input> <output>\n", argv[0]);
        return 1;
    }
    fin = std::fopen(argv[2], "rb");
    fout = std::fopen(argv[3], "wb");
    if (!fin || !fout) {
        std::fprintf(stderr, "cannot open the files\n");
        return 1;
    }
    const int n_cases = rd<int>();
    for (int c = 0; c < n_cases; ++c) {
        if (std::strcmp(argv[1], "select") == 0) run_select();
        else if (std::strcmp(argv[1], "hyp") == 0) run_hyp();
        else return 1;
    }
    std::fclose(fout);
    std::fclose(fin);
    return 0;
}
