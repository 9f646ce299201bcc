// Host build of csrc/screen_math.cuh (the arithmetic of the fp32 screening pass) for tests/test_screen_bounds.py:
// evaluates one model over n correspondences exactly as k_screen does (same functions, fmaf from libm) next to the fp64
// formulas of the exact kernels (kernels.cu: sampson_r2 / homography_r2 / reprojection with the z2 <= 0 skip,
// device_math.cuh: cheirality_ok) and checks, correspondence by correspondence and for the totals, that the fp32
// record brackets the fp64 one:  streaming test false => fp64 outlier;  !border => same decision;
// |count64 - count32| <= border;  |score64 - score32| <= err.
#include "../poselib_b200/csrc/screen_math.cuh"
#include <cmath>
#include <cstdio>
#include <cstdlib>
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
double homography_r2_64(const double *H, double x1_0, double x1_1, double x2_0, double x2_1) {
    const double Hx1_0 = H[0] * x1_0 + H[1] * x1_1 + H[2];
    const double Hx1_1 = H[3] * x1_0 + H[4] * x1_1 + H[5];
    const double inv = 1.0 / (H[6] * x1_0 + H[7] * x1_1 + H[8]);
    const double r0 = Hx1_0 * inv - x2_0, r1 = Hx1_1 * inv - x2_1;
    return r0 * r0 + r1 * r1;
}
struct V3 {
    double x, y, z;
};
V3 bearing64(double u, double v) {
    const double n = std::sqrt(u * u + v * v + 1.0);
    return V3{u / n, v / n, 1.0 / n};
}
V3 quat_rotate64(const double *q, V3 p) { // misc/quaternion.h:61-70
    const double q1 = q[0], q2 = q[1], q3 = q[2], q4 = q[3];
    const double p1 = p.x, p2 = p.y, p3 = p.z;
    const double px1 = -p1 * q2 - p2 * q3 - p3 * q4;
    const double px2 = p1 * q1 - p2 * q4 + p3 * q3;
    const double px3 = p2 * q1 + p1 * q4 - p3 * q2;
    const double px4 = p2 * q2 - p1 * q3 + p3 * q1;
    return V3{px2 * q1 - px1 * q2 - px3 * q4 + px4 * q3, px3 * q1 - px1 * q3 + px2 * q4 - px4 * q2,
              px3 * q2 - px2 * q3 - px1 * q4 + px4 * q1};
}
bool cheirality64(const double *q, const double *t, V3 x1, V3 x2) {
    const V3 R = quat_rotate64(q, x1);
    const double a = -(R.x * x2.x + R.y * x2.y + R.z * x2.z);
    const double b1 = -(R.x * t[0] + R.y * t[1] + R.z * t[2]);
    const double b2 = x2.x * t[0] + x2.y * t[1] + x2.z * t[2];
    const double l1 = b1 - a * b2, l2 = -a * b1 + b2, md = 0.01 * (1 - a * a);
    return l1 > md && l2 > md;
}
struct Tot {
    long long c64 = 0, c32 = 0, border = 0, viol_point = 0, maybe = 0;
    double s64 = 0;
    float s32 = 0.f, err = 0.f;
};
void finish(const Tot &T, int n, double sq_thr, float thr, double *out) {
    const double score64 = T.s64 + (double)(n - T.c64) * sq_thr;
    const float score32 = T.s32 + (float)n * thr;
    const float depth = (float)(T.c32 + 24);
    float et = T.err * (1.f + 1e-5f) + U * thr * (depth * (float)T.c32 + 2.2f * (float)n);
    et *= (1.f + 1e-5f);
    long long viol = T.viol_point;
    if (::llabs(T.c64 - T.c32) > T.border) ++viol;
    // a non-finite err makes no claim about the score (k_select then always rescores the model)
    if (std::isfinite(et) && !(std::fabs(score64 - (double)score32) <= (double)et)) ++viol;
    out[0] = (double)viol;
    out[1] = (double)T.c64;
    out[2] = (double)T.c32;
    out[3] = (double)T.border;
    out[4] = score64;
    out[5] = (double)score32;
    out[6] = (double)et;
    out[7] = (double)T.maybe;
}
} // namespace

extern "C" {
// kind: 1 relpose (Sampson + cheirality), 2 fundamental (Sampson).  pts: 4 arrays of n doubles (x1.x x1.y x2.x x2.y);
// M: 3x3 row-major fp64; qt: q(4) t(3) for kind 1.
void scr_check_sampson(int kind, int n, const double *pts, const double *M, const double *qt, double sq_thr, double *out) {
    std::vector<float> f(4 * (size_t)n);
    float cmax[4] = {0, 0, 0, 0};
    for (int c = 0; c < 4; ++c)
        for (int k = 0; k < n; ++k) {
            f[(size_t)c * n + k] = (float)pts[(size_t)c * n + k];
            cmax[c] = std::fmax(cmax[c], f_up(std::fabs(pts[(size_t)c * n + k])));
        }
    float ctx[CTX_FLOATS];
    for (int k = 0; k < 9; ++k) ctx[k] = (float)M[k];
    if (kind == 1)
        for (int k = 0; k < 7; ++k) ctx[9 + k] = (float)qt[k];
    sampson_setup(M, cmax, sq_thr, ctx);
    if (kind == 1) cheirality_setup(qt, qt + 4, ctx);
    const float thr = (float)sq_thr;
    Tot T;
    for (int k = 0; k < n; ++k) {
        const double a0 = pts[k], a1 = pts[(size_t)n + k], b0 = pts[2 * (size_t)n + k], b1 = pts[3 * (size_t)n + k];
        const double r2 = sampson_r2_64(M, a0, a1, b0, b1);
        bool in64 = r2 < sq_thr;
        if (in64 && kind == 1) in64 = cheirality64(qt, qt + 4, bearing64(a0, a1), bearing64(b0, b1));
        if (in64) {
            ++T.c64;
            T.s64 += r2;
        }
        const float fa0 = f[k], fa1 = f[(size_t)n + k], fb0 = f[2 * (size_t)n + k], fb1 = f[3 * (size_t)n + k];
        const bool mb = sampson_maybe(ctx, fa0, fa1, fb0, fb1);
        if (!mb && r2 < sq_thr) ++T.viol_point; // ruled out although the fp64 residual is under the threshold
        if (!mb) continue;
        ++T.maybe;
        bool plain, border;
        float v, e;
        sampson_point(ctx, fa0, fa1, fb0, fb1, plain, border, v, e);
        if (kind == 1 && (plain || border)) {
            bool ok, cb;
            cheirality_point(ctx + 9, ctx[S_EH], fa0, fa1, fb0, fb1, ok, cb);
            if (cb) {
                border = true;
                e += thr;
            } else if (!ok) {
                border = false;
            }
            plain = plain && ok;
        }
        if (!border && plain != in64) ++T.viol_point;
        if (border) ++T.border;
        if (plain) {
            ++T.c32;
            T.s32 += v;
        }
        if (plain || border) T.err += e;
    }
    finish(T, n, sq_thr, thr, out);
}
// kind: 3 homography (pts: x1.x x1.y x2.x x2.y, M 3x3), 0 pnp (pts: x.x x.y X.x X.y X.z, M = [R t] 3x4 row-major)
void scr_check_transfer(int kind, int n, const double *pts, const double *M, double sq_thr, double *out) {
    const int narr = kind == 0 ? 5 : 4;
    std::vector<float> f((size_t)narr * n);
    float cmax[5] = {0, 0, 0, 0, 0};
    for (int c = 0; c < narr; ++c)
        for (int k = 0; k < n; ++k) {
            f[(size_t)c * n + k] = (float)pts[(size_t)c * n + k];
            cmax[c] = std::fmax(cmax[c], f_up(std::fabs(pts[(size_t)c * n + k])));
        }
    float ctx[CTX_FLOATS];
    for (int k = 0; k < (kind == 0 ? 12 : 9); ++k) ctx[k] = (float)M[k];
    if (kind == 0) transfer_setup<3>(M, cmax + 2, cmax, sq_thr, ctx);
    else transfer_setup<2>(M, cmax, cmax + 2, sq_thr, ctx);
    const float thr = (float)sq_thr;
    Tot T;
    for (int k = 0; k < n; ++k) {
        double r2;
        bool in64;
        TransferTerms tt;
        if (kind == 0) {
            const double x0 = pts[k], x1 = pts[(size_t)n + k], X0 = pts[2 * (size_t)n + k], X1 = pts[3 * (size_t)n + k],
                         X2 = pts[4 * (size_t)n + k];
            const double z0 = M[0] * X0 + M[1] * X1 + M[2] * X2 + M[3];
            const double z1 = M[4] * X0 + M[5] * X1 + M[6] * X2 + M[7];
            const double z2 = M[8] * X0 + M[9] * X1 + M[10] * X2 + M[11];
            in64 = false;
            r2 = INFINITY;
            if (!(z2 <= 0.0)) {
                const double inv = 1.0 / z2;
                const double r0 = z0 * inv - x0, r1 = z1 * inv - x1;
                r2 = r0 * r0 + r1 * r1;
                in64 = r2 < sq_thr;
            }
            tt = pnp_terms(ctx, f[k], f[(size_t)n + k], f[2 * (size_t)n + k], f[3 * (size_t)n + k], f[4 * (size_t)n + k]);
        } else {
            const double a0 = pts[k], a1 = pts[(size_t)n + k], b0 = pts[2 * (size_t)n + k], b1 = pts[3 * (size_t)n + k];
            r2 = homography_r2_64(M, a0, a1, b0, b1);
            in64 = r2 < sq_thr;
            tt = homography_terms(ctx, f[k], f[(size_t)n + k], f[2 * (size_t)n + k], f[3 * (size_t)n + k]);
        }
        if (in64) {
            ++T.c64;
            T.s64 += r2;
        }
        const bool mb = kind == 0 ? transfer_maybe<true>(ctx, tt) : transfer_maybe<false>(ctx, tt);
        if (!mb) {
            if (in64) ++T.viol_point;
            continue;
        }
        ++T.maybe;
        bool plain, border;
        float v, e;
        if (kind == 0) transfer_point<true>(ctx, tt, plain, border, v, e);
        else transfer_point<false>(ctx, tt, plain, border, v, e);
        if (!border && plain != in64) ++T.viol_point;
        if (border) ++T.border;
        if (plain) {
            ++T.c32;
            T.s32 += v;
        }
        if (plain || border) T.err += e;
    }
    finish(T, n, sq_thr, thr, out);
}
}
