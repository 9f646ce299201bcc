// Host build of csrc/screen_math.cuh for tests/test_screen_prefilter.py: the streaming test of k_screen for the Sampson
// kinds (sampson_maybe_c, |C^| <= K) against the full prefilter it replaces (sampson_maybe), the fp64 Sampson test and
// the queue pass's evaluation (sampson_point), one model over n correspondences.
#include "../poselib_b200/csrc/screen_math.cuh"
#include <cmath>
#include <vector>
using namespace plb::scr;

namespace {
double sampson_r2_64(const double *E, double x1_0, double x1_1, double x2_0, double x2_1) {
    const double Ex1_0 = E[0] * x1_0 + E[1] * x1_1 + E[2];
    const double Ex1_1 = E[3] * x1_0 + E[4] * x1_1 + E[5];
    const double Ex1_2 = E[6] * x1_0 + E[7] * x1_1 + E[8];
    const double Ex2_0 = E[0] * x2_0 + E[3] * x2_1 + E[6];
    const double Ex2_1 = E[1] * x2_0 + E[4] * x2_1 + E[7];
    const double C = x2_0 * Ex1_0 + x2_1 * Ex1_1 + Ex1_2;
    const double Cx = Ex1_0 * Ex1_0 + Ex1_1 * Ex1_1;
    const double Cy = Ex2_0 * Ex2_0 + Ex2_1 * Ex2_1;
    return C * C / (Cx + Cy);
}
struct Setup {
    std::vector<float> f;
    float cmax[4] = {0, 0, 0, 0};
    float ctx[CTX_FLOATS];
};
void setup(Setup &S, int n, const double *pts, const double *M, double sq_thr) {
    S.f.resize(4 * (size_t)n);
    for (int c = 0; c < 4; ++c)
        for (int k = 0; k < n; ++k) {
            S.f[(size_t)c * n + k] = (float)pts[(size_t)c * n + k];
            S.cmax[c] = std::fmax(S.cmax[c], f_up(std::fabs(pts[(size_t)c * n + k])));
        }
    for (int k = 0; k < CTX_FLOATS; ++k) S.ctx[k] = 0.f;
    for (int k = 0; k < 9; ++k) S.ctx[k] = (float)M[k];
    sampson_setup(M, S.cmax, sq_thr, S.ctx);
}
} // namespace

extern "C" {
// pts: 4 arrays of n doubles (x1.x x1.y x2.x x2.y), cmax from them as k_transpose computes it; M: 3x3 row-major fp64.
// out[0] pairs sampson_maybe accepts and sampson_maybe_c rejects (cases the streaming pass would lose)
// out[1] pairs sampson_maybe_c rejects whose fp64 Sampson residual is under the threshold
// out[2] pairs sampson_maybe_c accepts that sampson_maybe rejects and sampson_point counts (plain) or flags (border):
//        such a pair would change count32 or border
// out[3] pairs sampson_maybe accepts, out[4] pairs sampson_maybe_c accepts
// out[5] max D^ / Dmax (Dmax = sampson_dmax), out[6] max D^ / G (G = A_0^2 + A_1^2 + B_0^2 + B_1^2, the box bound of
//        the exact D without the rounding of D^), out[7] K
void scr_prefilter(int n, const double *pts, const double *M, double sq_thr, double *out) {
    Setup S;
    setup(S, n, pts, M, sq_thr);
    double A[3], B[2];
    sampson_rows(M, S.cmax, A, B);
    const double G = A[0] * A[0] + A[1] * A[1] + B[0] * B[0] + B[1] * B[1];
    const double Dmax = sampson_dmax(M, S.cmax);
    const float K = S.ctx[S_CK];
    for (int i = 0; i < 8; ++i) out[i] = 0.0;
    for (int k = 0; k < n; ++k) {
        const float a0 = S.f[k], a1 = S.f[(size_t)n + k], b0 = S.f[2 * (size_t)n + k], b1 = S.f[3 * (size_t)n + k];
        const bool mb = sampson_maybe(S.ctx, a0, a1, b0, b1);
        const bool mc = sampson_maybe_c(S.ctx, K, a0, a1, b0, b1);
        if (mb && !mc) out[0] += 1;
        if (!mc && sampson_r2_64(M, pts[k], pts[(size_t)n + k], pts[2 * (size_t)n + k], pts[3 * (size_t)n + k]) < sq_thr)
            out[1] += 1;
        if (mc && !mb) {
            bool plain, border;
            float v, e;
            sampson_point(S.ctx, a0, a1, b0, b1, plain, border, v, e);
            if (plain || border) out[2] += 1;
        }
        out[3] += mb;
        out[4] += mc;
        const float D = sampson_terms(S.ctx, a0, a1, b0, b1).D;
        if (std::isfinite(D)) {
            out[5] = std::fmax(out[5], (double)D / Dmax);
            out[6] = std::fmax(out[6], (double)D / G);
        }
    }
    out[7] = K;
}
// For every correspondence k: the smallest threshold (bisected in fp64 over [0, hi]) at which sampson_maybe accepts it,
// and whether sampson_maybe_c accepts it there.  out[0]: correspondences it rejects there; out[1]: max |C^| / K there
// (how close the adversarial set brings |C^| to K).
void scr_prefilter_edge(int n, const double *pts, const double *M, double hi, double *out) {
    out[0] = out[1] = 0.0;
    Setup S;
    for (int k = 0; k < n; ++k) {
        double lo = 0.0, up = hi;
        setup(S, n, pts, M, up);
        const float a0 = S.f[k], a1 = S.f[(size_t)n + k], b0 = S.f[2 * (size_t)n + k], b1 = S.f[3 * (size_t)n + k];
        if (!sampson_maybe(S.ctx, a0, a1, b0, b1)) continue;
        for (int it = 0; it < 80; ++it) {
            const double mid = 0.5 * (lo + up);
            setup(S, n, pts, M, mid);
            if (sampson_maybe(S.ctx, a0, a1, b0, b1)) up = mid;
            else lo = mid;
        }
        setup(S, n, pts, M, up);
        if (!sampson_maybe_c(S.ctx, S.ctx[S_CK], a0, a1, b0, b1)) out[0] += 1;
        const float C = sampson_terms(S.ctx, a0, a1, b0, b1).C;
        out[1] = std::fmax(out[1], (double)std::fabs(C) / (double)S.ctx[S_CK]);
    }
}
}
