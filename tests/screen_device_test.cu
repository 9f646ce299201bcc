// Device records of the fp32 screening pass next to the device's own fp64 records, for tests/test_screen_device.py.
// The library's steps run in the engine's order on problems and models read from a file:
//   launch_transpose (mode 0)  caller AoS doubles -> SoA fp64 / fp32 arrays and the coordinate maxima cmax;
//   k_screen_ctx<KIND>         the fp32 constants of every model;
//   k_screen<KIND, NTHR>       once per (NTHR, staging path, grid size) of the case;
//   launch_score_models        the exact fp64 (count, score) of every model.
// Usage: screen_device_test <input> <output>.  Little-endian binary, int = int32.
// Input:  int n_cases; per case:
//           int kind, int n_probs;
//           per problem: int n, int n_models, double sq_thr, double a[2 n], double b[b_dim n] (AoS, b_dim 3 for pnp,
//                        else 2), double models[n_models * 7 (pnp, relpose) or 9 (column-major F / H)];
//           int n_cfg; per config: int nthr (128 | 512), int use_smem, int n_grids, int grids[n_grids]
//                        (grid 0: the library's one-wave size for this launch).
// Output: per case, per config, per grid: int grid_used, then per model (all problems, in order)
//           uint32 count32, uint32 border, float score32, float err;
//         then per model uint32 count64, double score64.
// Records a launch did not write stay 0xffffffff (count32 / border) and NaN.
#include "../poselib_b200/csrc/kernels.cu"
#include <cstdio>
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
template <class T> static T *dalloc(size_t n) {
    T *p = nullptr;
    CK(cudaMalloc(&p, sizeof(T) * (n ? n : 1)));
    return p;
}
template <class T> static T *dput(const std::vector<T> &v) {
    T *p = dalloc<T>(v.size());
    if (!v.empty()) CK(cudaMemcpy(p, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
    return p;
}

template <int KIND, int NTHR>
static int run_screen(const RoundDesc &R, const HypOut &out, const float *fctx, int use_smem, int max_n_pad, int grid) {
    constexpr int NARR = (KIND == KIND_PNP) ? 5 : 4;
    const size_t bytes = use_smem ? (size_t)NARR * (size_t)scr_stage_len<NTHR>(max_n_pad) * 4 : 0;
    if (bytes > 200 * 1024) {
        std::fprintf(stderr, "staging buffer of %zu bytes requested\n", bytes);
        std::exit(4);
    }
    // the library sets the attribute for the 512-thread variant only; this harness runs both on either path
    CK(cudaFuncSetAttribute(k_screen<KIND, NTHR>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    if (grid == 0) { // launch_hyp_t's one wave
        int per_sm = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_screen<KIND, NTHR>, NTHR, bytes));
        if (per_sm < 1) per_sm = 1;
        const long long tiles = ((long long)out.max_seg_cap + SCR_TM - 1) / SCR_TM * (long long)R.n_active;
        grid = per_sm * sm_count();
        if ((long long)grid > tiles) grid = (int)tiles;
        if (grid < 1) grid = 1;
    }
    k_screen<KIND, NTHR><<<grid, NTHR, bytes>>>(R, out, fctx, use_smem);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    return grid;
}

static void run_case() {
    const int kind = rd<int>(), np = rd<int>();
    const int b_dim = kind == KIND_PNP ? 3 : 2, narr = 2 + b_dim, msz = kind_model_size(kind);
    std::vector<int> ns(np), ms(np), seg(np), act(np);
    std::vector<double> thr(np), a_all, b_all, models;
    std::vector<size_t> a_off(np), b_off(np), s_off(np);
    size_t soa = 0;
    int total_m = 0, max_m = 0, max_n_pad = 0;
    for (int i = 0; i < np; ++i) {
        ns[i] = rd<int>();
        ms[i] = rd<int>();
        thr[i] = rd<double>();
        std::vector<double> a, b, m;
        rdv(a, 2 * (size_t)ns[i]);
        rdv(b, (size_t)b_dim * ns[i]);
        rdv(m, (size_t)ms[i] * msz);
        a_off[i] = a_all.size();
        b_off[i] = b_all.size();
        a_all.insert(a_all.end(), a.begin(), a.end());
        b_all.insert(b_all.end(), b.begin(), b.end());
        models.insert(models.end(), m.begin(), m.end());
        seg[i] = total_m;
        act[i] = i;
        total_m += ms[i];
        max_m = std::max(max_m, ms[i]);
        const int n_pad = (ns[i] + 31) & ~31;
        max_n_pad = std::max(max_n_pad, n_pad);
        s_off[i] = soa;
        soa += (size_t)narr * n_pad;
    }
    double *d_a = dput(a_all), *d_b = dput(b_all), *d_models = dput(models);
    double *d_s64 = dalloc<double>(soa);
    float *d_s32 = dalloc<float>(soa), *d_cmax = dalloc<float>(5 * (size_t)np);
    CK(cudaMemset(d_cmax, 0, sizeof(float) * 5 * (size_t)np));
    std::vector<TransposeDesc> td(np);
    std::vector<ProblemDev> pd(np);
    std::vector<int> model_prob(total_m);
    for (int i = 0; i < np; ++i) {
        const int n_pad = (ns[i] + 31) & ~31;
        TransposeDesc &D = td[i];
        std::memset(&D, 0, sizeof(D));
        D.a = d_a + a_off[i];
        D.b = d_b + b_off[i];
        D.s64 = d_s64 + s_off[i];
        D.s32 = d_s32 + s_off[i];
        D.cmax = d_cmax + 5 * (size_t)i;
        D.n = ns[i];
        D.n_pad = n_pad;
        D.b_dim = b_dim;
        D.mode = 0;
        D.scale = 1.0;
        D.cam_a.model = D.cam_b.model = CAMM_NULL;
        ProblemDev &P = pd[i];
        std::memset(&P, 0, sizeof(P));
        P.cam[0].model = P.cam[1].model = CAMM_NULL;
        P.n = ns[i];
        P.kind = kind;
        P.sq_thr = thr[i];
        P.n_pad = n_pad;
        P.cmax = D.cmax;
        for (int c = 0; c < narr; ++c) {
            P.p[c] = D.s64 + (size_t)c * n_pad;
            P.f[c] = D.s32 + (size_t)c * n_pad;
        }
        for (int m = 0; m < ms[i]; ++m) model_prob[seg[i] + m] = i;
    }
    TransposeDesc *d_td = dput(td);
    ProblemDev *d_pd = dput(pd);
    launch_transpose(d_td, np, max_n_pad, false, 0);
    CK(cudaGetLastError());

    int *d_act = dput(act), *d_seg = dput(seg), *d_cnt = dput(ms), *d_mp = dput(model_prob);
    RoundDesc R;
    std::memset(&R, 0, sizeof(R));
    R.probs = d_pd;
    R.active = d_act;
    R.n_active = np;
    HypOut out;
    std::memset(&out, 0, sizeof(out));
    out.seg_base = d_seg;
    out.seg_cap = d_cnt;
    out.prob_count = d_cnt;
    out.max_seg_cap = max_m;
    out.models = d_models;
    out.model_prob = d_mp;
    out.fcounts = dalloc<uint32_t>(total_m);
    out.fscores = dalloc<float>(total_m);
    out.fborder = dalloc<uint32_t>(total_m);
    out.ferr = dalloc<float>(total_m);
    float *d_fctx = dalloc<float>((size_t)total_m * scr::CTX_FLOATS);
    with_kind(kind, [&](auto K) {
        constexpr int KK = decltype(K)::value;
        if constexpr (KK != KIND_RELPOSE_TS)
            k_screen_ctx<KK><<<dim3((max_m + SCR_CTX_THREADS - 1) / SCR_CTX_THREADS, np, 1), SCR_CTX_THREADS>>>(R, out, d_fctx);
    });
    CK(cudaGetLastError());

    std::vector<uint32_t> c32(total_m), bd(total_m);
    std::vector<float> s32(total_m), er(total_m);
    const int n_cfg = rd<int>();
    for (int c = 0; c < n_cfg; ++c) {
        const int nthr = rd<int>(), use_smem = rd<int>(), ng = rd<int>();
        std::vector<int> grids;
        rdv(grids, ng);
        for (int g : grids) {
            CK(cudaMemset(out.fcounts, 0xff, sizeof(uint32_t) * total_m));
            CK(cudaMemset(out.fborder, 0xff, sizeof(uint32_t) * total_m));
            CK(cudaMemset(out.fscores, 0xff, sizeof(float) * total_m));
            CK(cudaMemset(out.ferr, 0xff, sizeof(float) * total_m));
            int used = 0;
            with_kind(kind, [&](auto K) {
                constexpr int KK = decltype(K)::value;
                if constexpr (KK != KIND_RELPOSE_TS) {
                    if (nthr == 128) used = run_screen<KK, 128>(R, out, d_fctx, use_smem, max_n_pad, g);
                    else used = run_screen<KK, 512>(R, out, d_fctx, use_smem, max_n_pad, g);
                }
            });
            CK(cudaMemcpy(c32.data(), out.fcounts, sizeof(uint32_t) * total_m, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(bd.data(), out.fborder, sizeof(uint32_t) * total_m, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(s32.data(), out.fscores, sizeof(float) * total_m, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(er.data(), out.ferr, sizeof(float) * total_m, cudaMemcpyDeviceToHost));
            wr(&used, 1);
            for (int m = 0; m < total_m; ++m) {
                wr(&c32[m], 1);
                wr(&bd[m], 1);
                wr(&s32[m], 1);
                wr(&er[m], 1);
            }
        }
    }
    uint32_t *d_c64 = dalloc<uint32_t>(total_m);
    double *d_s64r = dalloc<double>(total_m);
    launch_score_models(kind, d_pd, d_models, d_mp, total_m, d_c64, d_s64r, 0);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    std::vector<uint32_t> c64(total_m);
    std::vector<double> s64(total_m);
    CK(cudaMemcpy(c64.data(), d_c64, sizeof(uint32_t) * total_m, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(s64.data(), d_s64r, sizeof(double) * total_m, cudaMemcpyDeviceToHost));
    for (int m = 0; m < total_m; ++m) {
        wr(&c64[m], 1);
        wr(&s64[m], 1);
    }
    for (void *p : {(void *)d_a, (void *)d_b, (void *)d_models, (void *)d_s64, (void *)d_s32, (void *)d_cmax, (void *)d_td,
                    (void *)d_pd, (void *)d_act, (void *)d_seg, (void *)d_cnt, (void *)d_mp, (void *)out.fcounts,
                    (void *)out.fscores, (void *)out.fborder, (void *)out.ferr, (void *)d_fctx, (void *)d_c64,
                    (void *)d_s64r})
        CK(cudaFree(p));
}

int main(int argc, char **argv) {
    if (argc != 3) {
        std::fprintf(stderr, "usage: %s <input> <output>\n", argv[0]);
        return 1;
    }
    fin = std::fopen(argv[1], "rb");
    fout = std::fopen(argv[2], "wb");
    if (!fin || !fout) {
        std::fprintf(stderr, "cannot open the files\n");
        return 1;
    }
    const int n_cases = rd<int>();
    for (int c = 0; c < n_cases; ++c) run_case();
    std::fclose(fout);
    std::fclose(fin);
    return 0;
}
