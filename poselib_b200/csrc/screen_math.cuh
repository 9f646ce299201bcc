// poselib_b200 — arithmetic of the fp32 screening pass (fast mode) with a RIGOROUS bracket of the fp64 result.
//
// k_screen scores every model of a round in fp32.  Its records only decide which models are rescored in fp64, so they
// must never rule out a model whose exact record would have changed the RANSAC state.  For every model the kernel
// therefore produces, besides (count32, score32):
//   border : the number of correspondences whose inlier decision in fp32 is not PROVABLY the fp64 decision, so that
//            count64 is in [count32 - border, count32 + border];
//   err    : a bound of |score64 - score32|.
// k_select turns these into intervals and keeps every model whose interval could beat the running best (control.cu).
//
// Error model (u = 2^-24, gamma_k = k u / (1 - k u)).  The fp32 inputs are roundings of the fp64 data: coordinates
// x^ = x (1 + d), |d| <= u, model constants likewise.  A nested-FMA sum of products of those accumulates at most k
// factors (1 + d) per elementary term, so |computed - exact| <= gamma_k * (sum of |elementary terms|); the sums of
// absolute terms are bounded per MODEL from the per-problem coordinate maxima cmax[] (computed by k_transpose from the
// fp64 data), which turns every bound into a handful of per-model constants (ctx[16..]).  "exact" means real arithmetic
// on the fp64 data; the fp64 kernels differ from it by the same structure with u64 = 2^-53, i.e. 2^-29 of these bounds —
// covered by rounding every k up (7 -> 8, ...).  The derivation of each constant is next to its definition.
//
// All functions are __host__ __device__: tests/test_screen_bounds.py compiles this header for the CPU (with fmaf) and
// checks the bracket against fp64 on millions of random and adversarial points (values on the threshold, large
// offsets, pixel units, near-degenerate models).
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define SCR_HD __host__ __device__ __forceinline__
#else
#define SCR_HD inline
#endif

namespace plb {
namespace scr {

constexpr float U = 5.9604644775390625e-8f; // 2^-24
constexpr double Ud = 5.9604644775390625e-8;

// smallest float >= x (x finite or not)
SCR_HD float f_up(double x) {
    float f = (float)x;
    if ((double)f < x) f = nextafterf(f, INFINITY);
    return f;
}
SCR_HD float f_down(double x) {
    float f = (float)x;
    if ((double)f > x) f = nextafterf(f, -INFINITY);
    return f;
}
SCR_HD float fast_rcp(float x) {
#if defined(__CUDA_ARCH__)
    return __fdividef(1.f, x); // <= 2 ulp
#else
    return 1.f / x;
#endif
}
SCR_HD float fast_rsqrt(float x) {
#if defined(__CUDA_ARCH__)
    return rsqrtf(x); // <= 2 ulp
#else
    return 1.f / sqrtf(x);
#endif
}

// ---- layout of one model's constants in shared memory (floats) -----------------------------------------------
constexpr int CTX_FLOATS = 28;
// [0..15]  the model: 3x3 row-major (E / F / H) [+ q(4), t(3) for relpose]  |  3x4 row-major [R t] for pnp
enum {
    // Sampson kinds (relpose, fundamental)
    S_THR_P = 16,   // prefilter: thr^ (1 + 128u)
    S_ALPHA_P = 17, //            alpha (1 + 64u)
    S_BETA_P = 18,  //            beta (1 + 64u)
    S_THR = 19,     // thr^ = fl32(sq_thr)
    S_ALPHA = 20,   // 2 eC
    S_BETA = 21,    // eC^2 + thr beta_D
    S_ERR_K = 22,   // 4 beta + 2 thr beta_D   (constant part of the per-point score error numerator)
    S_DMIN = 23,    // 4 beta_D: below this denominator nothing can be said about the residual
    S_EH = 24,      // relpose: bound of the fp32 error of lambda - min_depth (cheirality test)
    // transfer kinds (homography, pnp): | d | < thr_s * w
    T_THRS_P = 16,  // prefilter: sqrt(thr) rounded up (1 + 8u)
    T_C_P = 17,     //            c (1 + 8u),  c = e_d + thr_s e_w
    T_THR = 19,     // thr^
    T_THRS_LO = 20, // sqrt(thr) rounded down
    T_THRS_HI = 21, // sqrt(thr) rounded up
    T_ED = 22,      // e_d
    T_EW = 23,      // e_w
    T_ERR_K = 24    // 9 thr_s c
};

// ============================================================================================================
// Sampson error (robust/utils.cc:158-239):  C = x2^T E x1,  D = (E x1)_0^2 + (E x1)_1^2 + (E^T x2)_0^2 + (E^T x2)_1^2,
// inlier iff C^2 < thr D.
//
//   e^_r = fma(m_r0, a0, fma(m_r1, a1, m_r2))           <= 4 factors/term :  |e^_r - e_r| <= gamma_4 A_r,
//                                                        A_r = |E_r0| a0max + |E_r1| a1max + |E_r2|   (f^_c: B_c alike)
//   C^   = fma(b0, e^_0, fma(b1, e^_1, e^_2))           <= 7 factors/term :  |C^ - C| <= gamma_7 S =: eC  (8u S used)
//                                                        S = b0max A_0 + b1max A_1 + A_2
//   D^   = fma(e0,e0,fma(e1,e1,fma(f0,f0,f1 f1)))        |D^ - G^| <= gamma_4 G^  with G^ = sum of the computed squares,
//          |G^ - D| <= sum eta (2|g^| + eta) <= 4 eta sqrt(G^) + 4 eta^2 <= 8u G^ + eta^2 (4 + 1/(2u)),
//          eta = gamma_4 max(A_0, A_1, B_0, B_1)         =>  |D^ - D| <= 13u D^ + beta_D,  beta_D = 9u Amax^2 >= eta^2 (4 + 1/(2u))
//   num = fl(C^ C^),  t = fl(thr^ D^)                    |num - C^2| <= u num + eC (2|C^| + eC)
//                                                        |t - thr D| <= 19u t + thr beta_D
//   => | (num - t) - (C^2 - thr D) | <= E_f = alpha |C^| + kappa (num + t) + beta,
//      alpha = 2 eC, kappa = 20u (24u used: covers the fp32 evaluation of E_f itself), beta = eC^2 + thr beta_D (1 + 4u).
// ============================================================================================================
// M: row-major 3x3 in fp64 (the exact model the fp64 kernels use); cmax: a0max a1max b0max b1max.
SCR_HD void sampson_setup(const double *M, const float *cmax, double sq_thr, float *ctx) {
    const double a0 = cmax[0], a1 = cmax[1], b0 = cmax[2], b1 = cmax[3];
    double A[3], B[2];
    for (int r = 0; r < 3; ++r) A[r] = fabs(M[3 * r]) * a0 + fabs(M[3 * r + 1]) * a1 + fabs(M[3 * r + 2]);
    for (int c = 0; c < 2; ++c) B[c] = fabs(M[c]) * b0 + fabs(M[3 + c]) * b1 + fabs(M[6 + c]);
    const double S = b0 * A[0] + b1 * A[1] + A[2];
    const double Amax = fmax(fmax(A[0], A[1]), fmax(B[0], B[1]));
    const double eC = 8.0 * Ud * S;
    const double betaD = 9.0 * Ud * Amax * Amax;
    const float thr = (float)sq_thr;
    const double thr_hi = (double)thr * (1.0 + 2.0 * Ud) + 1e-300; // >= sq_thr and >= thr^
    const double alpha = 2.0 * eC, beta = eC * eC + thr_hi * betaD * (1.0 + 4.0 * Ud);
    ctx[S_THR] = thr;
    ctx[S_ALPHA] = f_up(alpha * (1.0 + 8.0 * Ud));
    ctx[S_BETA] = f_up(beta * (1.0 + 8.0 * Ud));
    ctx[S_THR_P] = f_up((double)thr * (1.0 + 128.0 * Ud));
    ctx[S_ALPHA_P] = f_up(alpha * (1.0 + 64.0 * Ud));
    ctx[S_BETA_P] = f_up(beta * (1.0 + 64.0 * Ud));
    ctx[S_ERR_K] = f_up((4.0 * beta + 2.0 * thr_hi * betaD) * (1.0 + 8.0 * Ud));
    ctx[S_DMIN] = f_up(4.0 * betaD);
}
struct SampsonTerms {
    float C, D;
};
SCR_HD SampsonTerms sampson_terms(const float *M, float a0, float a1, float b0, float b1) {
    const float e0 = fmaf(M[0], a0, fmaf(M[1], a1, M[2]));
    const float e1 = fmaf(M[3], a0, fmaf(M[4], a1, M[5]));
    const float e2 = fmaf(M[6], a0, fmaf(M[7], a1, M[8]));
    const float f0 = fmaf(M[0], b0, fmaf(M[3], b1, M[6]));
    const float f1 = fmaf(M[1], b0, fmaf(M[4], b1, M[7]));
    SampsonTerms T;
    T.C = fmaf(b0, e0, fmaf(b1, e1, e2));
    T.D = fmaf(e0, e0, fmaf(e1, e1, fmaf(f0, f0, f1 * f1)));
    return T;
}
// Streaming-pass test: false only if the correspondence is PROVABLY an outlier in fp64 (num - t > E_f):
//   num (1 - kappa) - alpha |C| - beta <= t (1 + kappa)   evaluated as   C C - beta' - alpha' |C| <= thr' D
// (thr' / alpha' / beta' carry the (1 +- kappa) factors and the three roundings of this expression).
SCR_HD bool sampson_maybe(const float *ctx, float a0, float a1, float b0, float b1) {
    const SampsonTerms T = sampson_terms(ctx, a0, a1, b0, b1);
    const float g = fmaf(-ctx[S_ALPHA_P], fabsf(T.C), fmaf(T.C, T.C, -ctx[S_BETA_P]));
    return g <= ctx[S_THR_P] * T.D;
}
// Full evaluation of one correspondence the streaming pass could not rule out.
//   plain  : the fp32 decision num < t (what count32 / score32 use)
//   border : the fp64 decision is not provably the same
//   v      : r^2 - thr in fp32 (valid if plain)
//   e      : bound of the error this correspondence can contribute to |score64 - score32| (valid if plain || border):
//            (r^2 - thr) = f / D;  | f/D - f~/D^ | <= 2 E_f / D^ + 2 thr (16u + beta_D / D^)  for D^ > 4 beta_D; a
//            misclassified borderline point contributes at most |f| / D <= 4 E_f / D^.  Rounding of the division and of
//            the subtraction: 4u (num/D^ + thr) <= 8u thr.   =>  e = rD (4 E_f + 2 thr beta_D) + 40u thr
SCR_HD void sampson_point(const float *ctx, float a0, float a1, float b0, float b1, bool &plain, bool &border, float &v,
                          float &e) {
    const SampsonTerms T = sampson_terms(ctx, a0, a1, b0, b1);
    const float thr = ctx[S_THR];
    const float num = T.C * T.C, t = thr * T.D;
    plain = num < t;
    const float Ef = fmaf(ctx[S_ALPHA], fabsf(T.C), fmaf(24.f * U, num + t, ctx[S_BETA]));
    border = !(fabsf(num - t) > Ef);
    const float rD = fast_rcp(T.D);
    v = fmaf(num, rD, -thr);
    e = fmaf(rD, fmaf(4.f, Ef, ctx[S_ERR_K]), 40.f * U * thr);
    if (!(T.D > ctx[S_DMIN])) e = INFINITY;
}

// ============================================================================================================
// Cheirality of a relative pose on one correspondence (misc/essential.cc:40-57 via robust/utils.cc:187-197):
//   u1 = (a0,a1,1)/|.|, u2 alike;  w = R(q) u1;  a = -w.u2, b1 = -w.t, b2 = u2.t;
//   lambda1 = b1 - a b2, lambda2 = -a b1 + b2, md = 0.01 (1 - a^2);  ok iff lambda1 > md && lambda2 > md.
// fp32 error of h_i = lambda_i - md, with Qn = |q|_2^2, qm = max |q_i| (qm^2 <= Qn), T1 = |t|_1, all bearings of norm
// <= 1 + 8u (rsqrt: 2 ulp + 3 roundings):
//   w_j   : 12 elementary terms u q q, <= 16 factors each, sum of |terms| <= 4 sqrt(3) qm^2   -> <= 128u Qn
//   a     : sum of |terms| <= 12 qm^2, <= 27 factors                                           -> ea  <= 400u Qn
//   b1    : sum of |terms| <= 4 sqrt(3) qm^2 T1, <= 20 factors                                 -> eb1 <= 160u Qn T1
//   b2    : sum of |terms| <= sqrt(3) T1, <= 12 factors                                        -> eb2 <= 24u T1
//   |a| <= Qn(1+..), |b1| <= Qn T1, |b2| <= T1:
//   lambda1: eb1 + |a| eb2 + |b2| ea + 4u Qn T1        <= u T1 (160 Qn + 24 Qn + 400 Qn + 4 Qn) = 588u Qn T1
//   lambda2: |a| eb1 + |b1| ea + eb2 + 4u (Qn^2 + 1)T1 <= u T1 (560 Qn^2 + 28 + 4 Qn^2)
//   md     : 0.01 (2 |a| ea + ea^2 + 2u (1 + a^2))     <= u (8 Qn^2 + 1)
//   E_h = 1024u (1 + Qn)^2 (1 + T1)   dominates all three sums.
// ============================================================================================================
SCR_HD void cheirality_setup(const double *q, const double *t, float *ctx) {
    const double Qn = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    const double T1 = fabs(t[0]) + fabs(t[1]) + fabs(t[2]);
    ctx[S_EH] = f_up(1024.0 * Ud * (1.0 + Qn) * (1.0 + Qn) * (1.0 + T1));
}
SCR_HD void cheirality_point(const float *qt, float Eh, float a0, float a1, float b0, float b1, bool &ok, bool &border) {
    const float in1 = fast_rsqrt(fmaf(a0, a0, fmaf(a1, a1, 1.f)));
    const float in2 = fast_rsqrt(fmaf(b0, b0, fmaf(b1, b1, 1.f)));
    const float u0 = a0 * in1, u1 = a1 * in1, u2 = in1;
    const float v0 = b0 * in2, v1 = b1 * in2, v2 = in2;
    const float *q = qt, *t = qt + 4;
    const float px1 = -u0 * q[1] - u1 * q[2] - u2 * q[3];
    const float px2 = u0 * q[0] - u1 * q[3] + u2 * q[2];
    const float px3 = u1 * q[0] + u0 * q[3] - u2 * q[1];
    const float px4 = u1 * q[1] - u0 * q[2] + u2 * q[0];
    const float w0 = px2 * q[0] - px1 * q[1] - px3 * q[3] + px4 * q[2];
    const float w1 = px3 * q[0] - px1 * q[2] + px2 * q[3] - px4 * q[1];
    const float w2 = px3 * q[1] - px2 * q[2] - px1 * q[3] + px4 * q[0];
    const float aa = -(w0 * v0 + w1 * v1 + w2 * v2);
    const float bb1 = -(w0 * t[0] + w1 * t[1] + w2 * t[2]);
    const float bb2 = v0 * t[0] + v1 * t[1] + v2 * t[2];
    const float l1 = bb1 - aa * bb2, l2 = -aa * bb1 + bb2;
    const float md = 0.01f * (1.f - aa * aa);
    const float h1 = l1 - md, h2 = l2 - md;
    ok = (l1 > md) && (l2 > md);
    // certain iff one of the two tests fails by more than the bound, or both hold by more than the bound
    const bool sure_no = (h1 < -Eh) || (h2 < -Eh);
    const bool sure_yes = (h1 > Eh) && (h2 > Eh);
    border = !(sure_no || sure_yes);
}

// ============================================================================================================
// Transfer errors:  homography  r = (H x1)_{01} / (H x1)_2 - x2     (robust/utils.cc:300-329)
//                   pnp         r = (R X + t)_{01} / (R X + t)_2 - x, skipped when the depth is <= 0 (utils.cc:36-63)
// Both are  |d| < thr_s |w|  with  d_r = h_r - w y_r  (y = the observed 2D point), thr_s = sqrt(thr); pnp additionally
// needs w > 0.  With J terms per row (2 + constant for H, 3 + constant for pnp):
//   |h^_r - h_r| <= gamma_{J+2} R_r,  R_r = sum |M_rj| xmax_j (+ |M_r,last|);     e_w = gamma_{J+2} R_2
//   d^_r = fma(-w^, y_r, h^_r):  |d^_r - d_r| <= gamma_{J+5} (R_r + ymax_r R_2) =: eta_r;     e_d = eta_0 + eta_1
//   N^ = |d^| (Euclidean):  | N^ - N | <= e_d;   num = fma(d0,d0,d1 d1) = N^2 (1 + 2u)
//   certain inlier  :  N^ + e_d <  thr_s (|w^| - e_w)
//   certain outlier :  N^ - e_d >= thr_s (|w^| + e_w)
//   streaming test (not a certain outlier):  N^ < thr_s |w^| + c,  c = e_d + thr_s e_w,  squared:
//        num <= (fma(thr_s', |w^|, c'))^2   with thr_s' = thr_s (1 + 8u), c' = c (1 + 8u)   (three roundings on the right)
//   score: rho = N / |w|;  |rho - rho^| <= (e_d + rho^ e_w) / (|w^| - e_w);  for |w^| > 2 e_w and rho, rho^ <= 1.1 thr_s
//        |rho^2 - rho^^2| <= 4.4 thr_s c / |w^|;  misclassified borderline points twice that  ->  e = 9 thr_s c / |w^| + 16u thr
// ============================================================================================================
// M: row-major 3 x (J+1) in fp64; xmax: maxima of the J coordinates M is applied to; ymax: maxima of the observed 2D point.
template <int J> SCR_HD void transfer_setup(const double *M, const float *xmax, const float *ymax, double sq_thr, float *ctx) {
    double R[3];
    for (int r = 0; r < 3; ++r) {
        double s = fabs(M[(J + 1) * r + J]);
        for (int j = 0; j < J; ++j) s += fabs(M[(J + 1) * r + j]) * (double)xmax[j];
        R[r] = s;
    }
    const double g_h = (double)(J + 3) * Ud, g_d = (double)(J + 6) * Ud; // gamma_{J+2}, gamma_{J+5} rounded up
    const double e_w = g_h * R[2];
    const double e_d = g_d * (R[0] + (double)ymax[0] * R[2]) + g_d * (R[1] + (double)ymax[1] * R[2]);
    const float thr = (float)sq_thr;
    const double thr_s = sqrt(fmax((double)thr, sq_thr));
    const double c = e_d + thr_s * (1.0 + 2.0 * Ud) * e_w;
    ctx[T_THR] = thr;
    ctx[T_THRS_LO] = f_down(sqrt(fmin((double)thr, sq_thr)) * (1.0 - 2.0 * Ud));
    ctx[T_THRS_HI] = f_up(thr_s * (1.0 + 2.0 * Ud));
    ctx[T_ED] = f_up(e_d * (1.0 + 4.0 * Ud));
    ctx[T_EW] = f_up(e_w * (1.0 + 4.0 * Ud));
    ctx[T_THRS_P] = f_up(thr_s * (1.0 + 8.0 * Ud));
    ctx[T_C_P] = f_up(c * (1.0 + 8.0 * Ud));
    ctx[T_ERR_K] = f_up(9.0 * thr_s * c * (1.0 + 8.0 * Ud));
}
struct TransferTerms {
    float num, w;
};
SCR_HD TransferTerms homography_terms(const float *M, float a0, float a1, float b0, float b1) {
    const float h0 = fmaf(M[0], a0, fmaf(M[1], a1, M[2]));
    const float h1 = fmaf(M[3], a0, fmaf(M[4], a1, M[5]));
    const float w = fmaf(M[6], a0, fmaf(M[7], a1, M[8]));
    const float d0 = fmaf(-w, b0, h0), d1 = fmaf(-w, b1, h1);
    TransferTerms T;
    T.num = fmaf(d0, d0, d1 * d1);
    T.w = w;
    return T;
}
SCR_HD TransferTerms pnp_terms(const float *P, float x0, float x1, float X0, float X1, float X2) {
    const float z0 = fmaf(P[0], X0, fmaf(P[1], X1, fmaf(P[2], X2, P[3])));
    const float z1 = fmaf(P[4], X0, fmaf(P[5], X1, fmaf(P[6], X2, P[7])));
    const float z2 = fmaf(P[8], X0, fmaf(P[9], X1, fmaf(P[10], X2, P[11])));
    const float d0 = fmaf(-z2, x0, z0), d1 = fmaf(-z2, x1, z1);
    TransferTerms T;
    T.num = fmaf(d0, d0, d1 * d1);
    T.w = z2;
    return T;
}
// SIGNED: pnp (w must be positive); homography uses |w|.
template <bool SIGNED> SCR_HD bool transfer_maybe(const float *ctx, TransferTerms T) {
    const float z = fmaf(ctx[T_THRS_P], SIGNED ? T.w : fabsf(T.w), ctx[T_C_P]);
    return (z > 0.f) && (T.num <= z * z);
}
template <bool SIGNED>
SCR_HD void transfer_point(const float *ctx, TransferTerms T, bool &plain, bool &border, float &v, float &e) {
    const float thr = ctx[T_THR], e_d = ctx[T_ED], e_w = ctx[T_EW];
    const float den = T.w * T.w;
    const bool valid = SIGNED ? (T.w > 0.f) : true;
    plain = valid && (T.num < thr * den);
    const float wa = fabsf(T.w);
    const float Nn = sqrtf(T.num);
    const bool sure_in = fmaf(Nn, 1.f + 4.f * U, e_d) < ctx[T_THRS_LO] * (wa - e_w) * (1.f - 4.f * U);
    const bool sure_out = fmaf(Nn, 1.f - 4.f * U, -e_d) >= ctx[T_THRS_HI] * (wa + e_w) * (1.f + 4.f * U);
    if (SIGNED) {
        // depth sign: certain only outside [-e_w, e_w]; a certainly negative depth is a certain outlier
        const bool sure_neg = T.w < -e_w, sure_pos = T.w > e_w;
        border = !(sure_neg || (sure_pos && (sure_in || sure_out)));
    } else {
        border = !(sure_in || sure_out);
    }
    const float rw = fast_rcp(wa);
    v = fmaf(T.num, rw * rw, -thr);
    e = fmaf(ctx[T_ERR_K], rw, 16.f * U * thr);
    if (!(wa > 2.f * e_w)) e = INFINITY;
}

} // namespace scr
} // namespace plb
