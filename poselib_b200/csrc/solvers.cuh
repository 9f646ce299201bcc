// poselib_b200 — minimal solvers as scalar device functions (one thread = one minimal sample).
//
// p3p, p3p_lambdatwist and homography_4pt are closed forms.  relpose_7pt runs the scalar nullspace routine of
// solver5_lane.cuh on the calling thread's slice of shared memory.  relpose_5pt is split into phase kernels
// (kernels.cu): its first half is solver5_lane.cuh, the Sturm root isolation, back-substitution and motion
// decomposition are below.  Every individual dot product / accumulation keeps the left-to-right order of the
// reference so results agree with the CPU path to the last bits wherever libm is not involved.
//
// Reference (relative to /root/reference): solvers/p3p.cc:39-202 + p3p_common.h; solvers/relpose_5pt.cc:101-409;
// solvers/relpose_7pt.cc:10-60; solvers/homography_4pt.cc:36-128; misc/sturm.h:47-274; misc/univariate.cc:48-126;
// misc/essential.cc:103-169.
#pragma once
#include "device_math.cuh"
#include "solver5_lane.cuh"

namespace plb {

// ================================ scalar helpers ==========================================================
// misc/univariate.cc:74-92
PLB_DEV bool cubic_single_real(double c2, double c1, double c0, double &root) {
    double a = c1 - c2 * c2 / 3.0;
    double b = (2.0 * c2 * c2 * c2 - 9.0 * c2 * c1) / 27.0 + c0;
    double c = b * b / 4.0 + a * a * a / 27.0;
    if (c != 0) {
        if (c > 0) {
            c = sqrt(c);
            b *= -0.5;
            root = cbrt(b + c) + cbrt(b - c) - c2 / 3.0;
            return true;
        }
        c = 3.0 * b / (2.0 * a) * sqrt(-3.0 / a);
        root = 2.0 * sqrt(-a / 3.0) * cos(acos(c) / 3.0) - c2 / 3.0;
    } else {
        root = -c2 / 3.0 + (a != 0 ? (3.0 * b / a) : 0);
    }
    return false;
}
// misc/univariate.cc:94-126
PLB_DEV int cubic_real(double c2, double c1, double c0, double *roots) {
    double a = c1 - c2 * c2 / 3.0;
    double b = (2.0 * c2 * c2 * c2 - 9.0 * c2 * c1) / 27.0 + c0;
    double c = b * b / 4.0 + a * a * a / 27.0;
    int n;
    if (a == 0.0 && b == 0.0) {
        roots[0] = roots[1] = roots[2] = -c2 / 3.0;
        n = 3;
    } else if (c > 0) {
        c = sqrt(c);
        b *= -0.5;
        roots[0] = cbrt(b + c) + cbrt(b - c) - c2 / 3.0;
        n = 1;
    } else {
        c = 3.0 * b / (2.0 * a) * sqrt(-3.0 / a);
        const double d = 2.0 * sqrt(-a / 3.0);
        const double third = acos(c) / 3.0;
        roots[0] = d * cos(third) - c2 / 3.0;
        roots[1] = d * cos(third - 2.09439510239319526263557236234192) - c2 / 3.0;
        roots[2] = d * cos(third - 4.18879020478639052527114472468384) - c2 / 3.0;
        n = 3;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (i < n) {
            const double x = roots[i], x2 = x * x, x3 = x * x2;
            roots[i] += -(x3 + c2 * x2 + c1 * x + c0) / (3 * x2 + 2 * c2 * x + c1);
        }
    }
    return n;
}
// misc/univariate.cc:48-61
PLB_DEV int quadratic_real(double a, double b, double c, double *roots) {
    const double disc = b * b - 4 * a * c;
    if (disc < 0) return 0;
    const double sq = sqrt(disc);
    roots[0] = (b > 0) ? (2 * c) / (-b - sq) : (2 * c) / (-b + sq);
    roots[1] = c / (a * roots[0]);
    return 2;
}

// ================================ p3p (Ding et al. CVPR'23) ================================================
// p3p_common.h:7-29
PLB_DEV bool p3p_root2real(double b, double c, double &r1, double &r2) {
    const double v = b * b - 4.0 * c;
    if (v < -1.0e-12) {
        r1 = r2 = -0.5 * b;
        return false;
    }
    if (v < 0.0) {
        r1 = -0.5 * b;
        r2 = -2;
        return true;
    }
    const double y = sqrt(v);
    if (b < 0) {
        r1 = 0.5 * (-b + y);
        r2 = 0.5 * (-b - y);
    } else {
        r1 = 2.0 * c / (-b + y);
        r2 = 2.0 * c / (-b - y);
    }
    return true;
}
// p3p_common.h:72-94
PLB_DEV void p3p_refine_lambda(double &l1, double &l2, double &l3, double a12, double a13, double a23, double b12,
                               double b13, double b23) {
    for (int it = 0; it < 5; ++it) {
        const double r1 = (l1 * l1 - 2.0 * l1 * l2 * b12 + l2 * l2 - a12);
        const double r2 = (l1 * l1 - 2.0 * l1 * l3 * b13 + l3 * l3 - a13);
        const double r3 = (l2 * l2 - 2.0 * l2 * l3 * b23 + l3 * l3 - a23);
        if (fabs(r1) + fabs(r2) + fabs(r3) < 1e-10) return;
        const double x11 = l1 - l2 * b12, x12 = l2 - l1 * b12;
        const double x21 = l1 - l3 * b13, x23 = l3 - l1 * b13;
        const double x32 = l2 - l3 * b23, x33 = l3 - l2 * b23;
        const double detJ = 0.5 / (x11 * x23 * x32 + x12 * x21 * x33);
        l1 += (-x23 * x32 * r1 - x12 * x33 * r2 + x12 * x23 * r3) * detJ;
        l2 += (-x21 * x33 * r1 + x11 * x33 * r2 - x11 * x23 * r3) * detJ;
        l3 += (x21 * x32 * r1 - x11 * x32 * r2 - x12 * x21 * r3) * detJ;
    }
}

// Solves one P3P instance.  xs: 3 unit bearings, Xs: 3 world points.  Writes up to 4 poses (7 doubles each) to
// `out` and returns the count.   p3p.cc:39-202
PLB_DEV int solve_p3p(const d3 *xs, const d3 *Xs, double *out) {
    d3 x0 = xs[0], x1 = xs[1], x2 = xs[2];
    d3 P0 = Xs[0], P1 = Xs[1], P2 = Xs[2];
    d3 X01 = P0 - P1, X02 = P0 - P2, X12 = P1 - P2;
    double a01 = dot(X01, X01), a02 = dot(X02, X02), a12 = dot(X12, X12);
    // make |P1-P2| the largest side (p3p.cc:58-73)
    if (a01 > a02) {
        if (a01 > a12) {
            d3 t = x0; x0 = x2; x2 = t;
            t = P0; P0 = P2; P2 = t;
            double s = a01; a01 = a12; a12 = s;
            X01 = -X12;
            X02 = -X02;
        }
    } else if (a02 > a12) {
        d3 t = x0; x0 = x1; x1 = t;
        t = P0; P0 = P1; P1 = t;
        double s = a02; a02 = a12; a12 = s;
        X01 = -X01;
        X02 = X12;
    }
    const double a12d = 1.0 / a12;
    const double a = a01 * a12d, b = a02 * a12d;
    const double m01 = dot(x0, x1), m02 = dot(x0, x2), m12 = dot(x1, x2);
    const double m12sq = -m12 * m12 + 1.0;
    const double m02sq = -1.0 + m02 * m02;
    const double m01sq = -1.0 + m01 * m01;
    const double ab = a * b, bsq = b * b, asq = a * a;
    const double m013 = -2.0 + 2.0 * m01 * m02 * m12;
    const double bsqm12sq = bsq * m12sq, asqm12sq = asq * m12sq, abm12sq = 2.0 * ab * m12sq;
    const double k3_inv = 1.0 / (bsqm12sq + b * m02sq);
    const double k2 = k3_inv * ((-1.0 + a) * m02sq + abm12sq + bsqm12sq + b * m013);
    const double k1 = k3_inv * (asqm12sq + abm12sq + a * m013 + (-1.0 + b) * m01sq);
    const double k0 = k3_inv * (asqm12sq + a * m01sq);
    double s;
    const bool G = cubic_single_real(k2, k1, k0, s);
    // degenerate conic C = C0 + s*C1 (p3p.cc:103-112), symmetric
    const double C00 = -a + s * (1 - b), C01 = -m02 * s, C02 = a * m12 + b * m12 * s;
    const double C11 = s + 1, C12 = -m01, C22 = -a - b * s + 1;
    // split into two lines (p3p_common.h:31-70)
    d3 pl, ql;
    {
        const double A00 = C12 * C12 - C11 * C22, A11 = C02 * C02 - C00 * C22, A22 = C01 * C01 - C00 * C11;
        const double A01 = C01 * C22 - C02 * C12, A02 = C02 * C11 - C01 * C12, A12 = C00 * C12 - C02 * C01;
        d3 v;
        if (A00 > A11) {
            if (A00 > A22) v = mk(A00, A01, A02) / sqrt(A00);
            else v = mk(A02, A12, A22) / sqrt(A22);
        } else if (A11 > A22) {
            v = mk(A01, A11, A12) / sqrt(A11);
        } else {
            v = mk(A02, A12, A22) / sqrt(A22);
        }
        // C + [v]x : first column -> p, first row -> q
        pl = mk(C00, C01 + v.z, C02 - v.y);
        ql = mk(C00, C01 - v.z, C02 + v.y);
    }
    m3 XX;
    set_col(XX, 0, X01);
    set_col(XX, 1, X02);
    set_col(XX, 2, cross(X01, X02));
    XX = inv3(XX);

    int n_sols = 0;
#pragma unroll 1
    for (int i = 0; i < 2; ++i) {
        const d3 L = (i == 0) ? pl : ql;
        const double p0 = L.x, p1 = L.y, p2 = L.z;
        const bool switch_12 = fabs(p0) <= fabs(p1);
        double w0, w1, cb, cc;
        if (switch_12) {
            w0 = -p0 / p1;
            w1 = -p2 / p1;
            const double ca = 1.0 / (w1 * w1 - b);
            cb = 2.0 * (b * m12 - m02 * w1 + w0 * w1) * ca;
            cc = (w0 * w0 - 2 * m02 * w0 - b + 1.0) * ca;
        } else {
            w0 = -p1 / p0;
            w1 = -p2 / p0;
            const double ca = 1.0 / (-a * w1 * w1 + 2 * a * m12 * w1 - a + 1);
            cb = 2 * (a * m12 * w0 - m01 - a * w0 * w1) * ca;
            cc = (1 - a * w0 * w0) * ca;
        }
        double taus[2];
        if (p3p_root2real(cb, cc, taus[0], taus[1])) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const double tau = taus[j];
                if (tau <= 0) continue;
                double d0, d1, d2;
                if (switch_12) {
                    d2 = sqrt(a12 / (tau * (tau - 2.0 * m12) + 1.0));
                    d1 = tau * d2;
                    d0 = (w0 * d2 + w1 * d1);
                    if (d0 < 0) continue;
                } else {
                    d0 = sqrt(a01 / (tau * (tau - 2.0 * m01) + 1.0));
                    d1 = tau * d0;
                    d2 = w0 * d0 + w1 * d1;
                    if (d2 < 0) continue;
                }
                p3p_refine_lambda(d0, d1, d2, a01, a02, a12, m01, m02, m12);
                const d3 v1 = d0 * x0 - d1 * x1;
                const d3 v2 = d0 * x0 - d2 * x2;
                m3 YY;
                set_col(YY, 0, v1);
                set_col(YY, 1, v2);
                set_col(YY, 2, cross(v1, v2));
                const m3 R = mmul(YY, XX);
                const d3 t = d0 * x0 - mvec(R, P0);
                double q[4];
                rot_to_quat(R, q);
                double *o = out + 7 * n_sols;
                o[0] = q[0]; o[1] = q[1]; o[2] = q[2]; o[3] = q[3];
                o[4] = t.x; o[5] = t.y; o[6] = t.z;
                ++n_sols;
            }
        }
        if (n_sols > 0 && G) break;
    }
    return n_sols;
}

// ---- p3p_lambdatwist (solvers/p3p_lambdatwist.cc:36-244): Persson & Nordberg's Lambda Twist, PoseLib's alternative P3P.
// Same calling convention as solve_p3p.  cbrt / cos / acos are CUDA's (1-2 ulp from glibc's): the closed-form root only
// seeds one Newton step on the cubic and the depths are polished by p3p_refine_lambda, so the poses agree with the CPU
// restatement to ~1e-13, not bit for bit.
PLB_DEV d3 lt_eigvec_known0(const m3 &M, double sig) {
    const double c = sig * sig + M(0, 0) * M(1, 1) - sig * (M(0, 0) + M(1, 1)) - M(0, 1) * M(0, 1);
    const double a1 = (sig * M(0, 2) + M(0, 1) * M(1, 2) - M(0, 2) * M(1, 1)) / c;
    const double a2 = (sig * M(1, 2) + M(0, 1) * M(0, 2) - M(0, 0) * M(1, 2)) / c;
    const double n = 1.0 / sqrt(1 + a1 * a1 + a2 * a2);
    return mk(a1 * n, a2 * n, n);
}
PLB_DEV m3 lt_cross_columns(const m3 &D) {
    m3 R;
    set_col(R, 0, cross(mcol(D, 1), mcol(D, 2)));
    set_col(R, 1, cross(mcol(D, 2), mcol(D, 0)));
    set_col(R, 2, cross(mcol(D, 0), mcol(D, 1)));
    return R;
}
// sum over the entries (column-major) of the element-wise product
PLB_DEV double lt_array_prod_sum(const m3 &A, const m3 &B) {
    double s = A(0, 0) * B(0, 0);
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int r = 0; r < 3; ++r)
            if (c + r > 0) s = s + A(r, c) * B(r, c);
    return s;
}
PLB_DEV int solve_p3p_lambdatwist(const d3 *xs, const d3 *Xs, double *out) {
    const d3 x0 = xs[0], x1 = xs[1], x2 = xs[2];
    const d3 dX12 = Xs[0] - Xs[1], dX13 = Xs[0] - Xs[2], dX23 = Xs[1] - Xs[2];
    const double a12 = dot(dX12, dX12), b12 = dot(x0, x1);
    const double a13 = dot(dX13, dX13), b13 = dot(x0, x2);
    const double a23 = dot(dX23, dX23), b23 = dot(x1, x2);
    const double a23b12 = a23 * b12, a12b23 = a12 * b23, a23b13 = a23 * b13, a13b23 = a13 * b23;
    m3 D1, D2; // :89-92
    D1(0, 0) = a23;     D1(0, 1) = -a23b12;   D1(0, 2) = 0.0;
    D1(1, 0) = -a23b12; D1(1, 1) = a23 - a12; D1(1, 2) = a12b23;
    D1(2, 0) = 0.0;     D1(2, 1) = a12b23;    D1(2, 2) = -a12;
    D2(0, 0) = a23;     D2(0, 1) = 0.0;       D2(0, 2) = -a23b13;
    D2(1, 0) = 0.0;     D2(1, 1) = -a13;      D2(1, 2) = a13b23;
    D2(2, 0) = -a23b13; D2(2, 1) = a13b23;    D2(2, 2) = a23 - a13;
    const m3 DX1 = lt_cross_columns(D1), DX2 = lt_cross_columns(D2);
    // p(gamma) = det(D1 + gamma D2)  (:98-103), monic, one real root in closed form (:110-121) + one Newton step (:123-126)
    const double c3 = dot(mcol(D2, 0), mcol(DX2, 0));
    double c2 = lt_array_prod_sum(D1, DX2);
    double c1 = lt_array_prod_sum(D2, DX1);
    double c0 = dot(mcol(D1, 0), mcol(DX1, 0));
    const double c3inv = 1.0 / c3;
    c2 *= c3inv;
    c1 *= c3inv;
    c0 *= c3inv;
    double a = c1 - c2 * c2 / 3.0;
    double b = (2.0 * c2 * c2 * c2 - 9.0 * c2 * c1) / 27.0 + c0;
    double c = b * b / 4.0 + a * a * a / 27.0;
    double gamma;
    if (c > 0) {
        c = sqrt(c);
        b *= -0.5;
        gamma = cbrt(b + c) + cbrt(b - c) - c2 / 3.0;
    } else {
        c = 3.0 * b / (2.0 * a) * sqrt(-3.0 / a);
        gamma = 2.0 * sqrt(-a / 3.0) * cos(acos(c) / 3.0) - c2 / 3.0;
    }
    const double f = gamma * gamma * gamma + c2 * gamma * gamma + c1 * gamma + c0;
    const double df = 3.0 * gamma * gamma + 2.0 * c2 * gamma + c1;
    gamma = gamma - f / df;

    m3 D0;
#pragma unroll
    for (int k = 0; k < 9; ++k) D0.a[k] = D1.a[k] + gamma * D2.a[k];
    double sig1, sig2;
    { // compute_eig3x3known0 (:36-65)
        const double p1 = -D0(0, 0) - D0(1, 1) - D0(2, 2);
        const double p0 = -D0(0, 1) * D0(0, 1) - D0(0, 2) * D0(0, 2) - D0(1, 2) * D0(1, 2) + D0(0, 0) * (D0(1, 1) + D0(2, 2)) +
                          D0(1, 1) * D0(2, 2);
        const double disc = sqrt(p1 * p1 / 4.0 - p0);
        const double tmp = -p1 / 2.0;
        sig1 = tmp + disc;
        sig2 = tmp - disc;
        if (fabs(sig1) < fabs(sig2)) {
            const double t = sig1;
            sig1 = sig2;
            sig2 = t;
        }
    }
    const d3 e1 = lt_eigvec_known0(D0, sig1), e2 = lt_eigvec_known0(D0, sig2);
    double s = sqrt(-sig2 / sig1);

    m3 XX;
    set_col(XX, 0, dX12);
    set_col(XX, 1, dX13);
    set_col(XX, 2, cross(dX12, dX13));
    XX = inv3(XX);
    const double TOL_DOUBLE_ROOT = 1e-12;
    int n_sols = 0;
#pragma unroll 1
    for (int s_flip = 0; s_flip < 2; ++s_flip, s = -s) {
        const double u1 = e1.x - s * e2.x, u2 = e1.y - s * e2.y, u3 = e1.z - s * e2.z;
        const bool switch_12 = fabs(u1) < fabs(u2);
        double qa, qb, qc, w0, w1;
        if (switch_12) { // solve for lambda2 (:164-205)
            w0 = -u1 / u2;
            w1 = -u3 / u2;
            qa = -a13 * w1 * w1 + 2 * a13b23 * w1 - a13 + a23;
            qb = 2 * a13b23 * w0 - 2 * a23b13 - 2 * a13 * w0 * w1;
            qc = -a13 * w0 * w0 + a23;
        } else { // lambda1 as a combination of lambda2 and lambda3 (:207-236)
            w0 = -u2 / u1;
            w1 = -u3 / u1;
            qa = (a13 - a12) * w1 * w1 + 2.0 * a12 * b13 * w1 - a12;
            qb = -2.0 * a13 * b12 * w1 + 2.0 * a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13);
            qc = (a13 - a12) * w0 * w0 - 2.0 * a13 * b12 * w0 + a13;
        }
        const double b2m4ac = qb * qb - 4.0 * qa * qc;
        if (b2m4ac < -TOL_DOUBLE_ROOT) continue;
        const double sq = sqrt(fmax(0.0, b2m4ac));
        double tau = (qb > 0) ? (2.0 * qc) / (-qb - sq) : (2.0 * qc) / (-qb + sq);
#pragma unroll 1
        for (int tau_flip = 0; tau_flip < 2; ++tau_flip, tau = qc / (qa * tau)) {
            if (tau > 0) {
                double l1, l2, l3;
                if (switch_12) {
                    l1 = sqrt(a13 / (tau * (tau - 2.0 * b13) + 1.0));
                    l3 = tau * l1;
                    l2 = w0 * l1 + w1 * l3;
                    if (l2 < 0) continue;
                } else {
                    l2 = sqrt(a23 / (tau * (tau - 2.0 * b23) + 1.0));
                    l3 = tau * l2;
                    l1 = w0 * l2 + w1 * l3;
                    if (l1 < 0) continue;
                }
                p3p_refine_lambda(l1, l2, l3, a12, a13, a23, b12, b13, b23);
                const d3 v1 = l1 * x0 - l2 * x1;
                const d3 v2 = l1 * x0 - l3 * x2;
                m3 YY;
                set_col(YY, 0, v1);
                set_col(YY, 1, v2);
                set_col(YY, 2, cross(v1, v2));
                const m3 R = mmul(YY, XX);
                const d3 t = l1 * x0 - mvec(R, Xs[0]);
                double q[4];
                rot_to_quat(R, q);
                double *o = out + 7 * n_sols;
                o[0] = q[0]; o[1] = q[1]; o[2] = q[2]; o[3] = q[3];
                o[4] = t.x; o[5] = t.y; o[6] = t.z;
                ++n_sols;
            }
            if (b2m4ac < TOL_DOUBLE_ROOT) break;
        }
    }
    return n_sols;
}

// ================================ homography_4pt (SKS / ACA closed form) ===================================
// homography_4pt.cc:36-128.  Writes H (9 doubles COLUMN-major) to out; returns 0/1.
PLB_DEV int solve_h4(const d3 *x1, const d3 *x2, double *out, bool check_cheirality) {
    if (check_cheirality) {
        d3 p = cross(x1[0], x1[1]), q = cross(x2[0], x2[1]);
        if (dot(p, x1[2]) * dot(q, x2[2]) < 0) return 0;
        if (dot(p, x1[3]) * dot(q, x2[3]) < 0) return 0;
        p = cross(x1[2], x1[3]);
        q = cross(x2[2], x2[3]);
        if (dot(p, x1[0]) * dot(q, x2[0]) < 0) return 0;
        if (dot(p, x1[1]) * dot(q, x2[1]) < 0) return 0;
    }
    double ax[4], ay[4], bx[4], by[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        ax[i] = x1[i].x / x1[i].z;
        ay[i] = x1[i].y / x1[i].z;
        bx[i] = x2[i].x / x2[i].z;
        by[i] = x2[i].y / x2[i].z;
    }
    const double sNx = ax[1] - ax[0], sPx = ax[2] - ax[0], sQx = ax[3] - ax[0];
    const double sNy = ay[1] - ay[0], sPy = ay[2] - ay[0], sQy = ay[3] - ay[0];
    const double fA1 = sNx * sPy - sNy * sPx;
    const double Q3x = sPy * sQx - sPx * sQy;
    const double Q3y = sNx * sQy - sNy * sQx;
    const double tNx = bx[1] - bx[0], tPx = bx[2] - bx[0], tQx = bx[3] - bx[0];
    const double tNy = by[1] - by[0], tPy = by[2] - by[0], tQy = by[3] - by[0];
    const double fA2 = tNx * tPy - tNy * tPx;
    const double Q4x = tPy * tQx - tPx * tQy;
    const double Q4y = tNx * tQy - tNy * tQx;
    const double tt1 = fA1 - Q3x - Q3y;
    const double C11 = Q3y * Q4x * tt1;
    const double C22 = Q3x * Q4y * tt1;
    const double C33 = Q3x * Q3y * (fA2 - Q4x - Q4y);
    const double C31 = C11 - C33, C32 = C22 - C33;
    const double tt3 = bx[0] * C33, tt4 = by[0] * C33;
    const double H1_11 = bx[1] * C11 - tt3, H1_12 = bx[2] * C22 - tt3;
    const double H1_21 = by[1] * C11 - tt4, H1_22 = by[2] * C22 - tt4;
    m3 H;
    H.a[0] = H1_11 * sPy - H1_12 * sNy;
    H.a[1] = H1_12 * sNx - H1_11 * sPx;
    H.a[3] = H1_21 * sPy - H1_22 * sNy;
    H.a[4] = H1_22 * sNx - H1_21 * sPx;
    H.a[6] = C31 * sPy - C32 * sNy;
    H.a[7] = C32 * sNx - C31 * sPx;
    H.a[2] = tt3 * fA1 - H.a[0] * ax[0] - H.a[1] * ay[0];
    H.a[5] = tt4 * fA1 - H.a[3] * ax[0] - H.a[4] * ay[0];
    H.a[8] = C33 * fA1 - H.a[6] * ax[0] - H.a[7] * ay[0];
    double n2 = 0; // Frobenius norm, column-major accumulation like Eigen's squaredNorm
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int r = 0; r < 3; ++r) n2 += H(r, c) * H(r, c);
    if (n2 > 0) {
        const double n = sqrt(n2);
#pragma unroll
        for (int k = 0; k < 9; ++k) H.a[k] /= n;
    }
    if (fabs(det3(H)) < 1e-8) return 0;
#pragma unroll
    for (int k = 0; k < 9; ++k) out[k] = H(k % 3, k / 3);
    return 1;
}

// ================================ Sturm root isolation, degree 10 ==========================================
// Scalar (single-lane) restatement of misc/sturm.h:47-274.  The recursion of isolate_roots is unrolled into an
// explicit interval stack that visits intervals in the same left-to-right depth-first order.
struct SturmWork {
    double fvec[21]; // monic polynomial (11) + monic-normalised derivative (10)
    double svec[30];
};
PLB_DEV double sturm_polyval10(const double *f, double x) {
    double fx = x + f[9];
#pragma unroll
    for (int i = 8; i >= 0; --i) fx = x * fx + f[i];
    return fx;
}
PLB_DEV double sturm_polyval9(const double *f, double x) {
    double fx = x + f[8];
#pragma unroll
    for (int i = 7; i >= 0; --i) fx = x * fx + f[i];
    return fx;
}
PLB_DEV int sturm_signchanges(const double *svec, double x) {
    double f2 = svec[29];
    double f1 = svec[27] + x * svec[28];
    int count = ((f1 < 0) != (f2 < 0)) ? 1 : 0;
#pragma unroll
    for (int i = 8; i >= 0; --i) {
        const double f0 = (svec[3 * i] + x * svec[3 * i + 1]) * f1 + svec[3 * i + 2] * f2;
        count += ((f0 < 0) != (f1 < 0)) ? 1 : 0;
        f2 = f1;
        f1 = f0;
    }
    return count;
}
// One step of the Sturm-sequence construction (sturm.h:56-79) with compile-time indices; the three work buffers rotate
// roles (f1,f2,f3) -> (f2,f3,f1) from step to step exactly like the reference's pointer juggling, so after inlining
// every array element lives in a register.
template <int I> PLB_DEV void sturm_step(double (&f1)[11], double (&f2)[11], double (&f3)[11], double *svec) {
    constexpr int N = 10;
    const double q1 = f1[N - I] * f2[N - 1 - I];
    const double q0 = f1[N - 1 - I] * f2[N - 1 - I] - f1[N - I] * f2[N - 2 - I];
    f3[0] = f1[0] - q0 * f2[0];
#pragma unroll
    for (int j = 1; j < N - 1 - I; ++j) f3[j] = f1[j] - q1 * f2[j - 1] - q0 * f2[j];
    const double c = -fabs(f3[N - 2 - I]);
    const double ci = 1.0 / c;
#pragma unroll
    for (int j = 0; j < N - 1 - I; ++j) f3[j] = f3[j] * ci;
    svec[3 * I] = q0;
    svec[3 * I + 1] = q1;
    svec[3 * I + 2] = c;
    if constexpr (I + 1 < N - 1) {
        sturm_step<I + 1>(f2, f3, f1, svec);
    } else {
        svec[3 * N - 3] = f2[0];
        svec[3 * N - 2] = f2[1];
        svec[3 * N - 1] = f3[0];
    }
}
PLB_DEV void sturm_build_seq(const double *fvec, double *svec) {
    constexpr int N = 10;
    double f1[11], f2[11], f3[11];
#pragma unroll
    for (int i = 0; i < N + 1; ++i) f1[i] = fvec[i];
#pragma unroll
    for (int i = 0; i < N; ++i) f2[i] = fvec[N + 1 + i];
    f2[N] = 0.0;
#pragma unroll
    for (int i = 0; i < N + 1; ++i) f3[i] = 0.0;
    sturm_step<0>(f1, f2, f3, svec);
}
PLB_DEV void sturm_ridders_newton(const double *fvec, double a, double b, double *roots, int &n_roots, double tol) {
    double fa = sturm_polyval10(fvec, a);
    double fb = sturm_polyval10(fvec, b);
    if (!((fa < 0) ^ (fb < 0))) return;
    for (int iter = 0; iter < 30; ++iter) {
        if (fabs(a - b) < 1e-3) break;
        const double c = (a + b) * 0.5;
        const double fc = sturm_polyval10(fvec, c);
        const double s = sqrt(fc * fc - fa * fb);
        if (!s) break;
        const double d = (fa < fb) ? c + (a - c) * fc / s : c + (c - a) * fc / s;
        const double fd = sturm_polyval10(fvec, d);
        if (fd >= 0 ? (fc < 0) : (fc > 0)) {
            a = c; fa = fc; b = d; fb = fd;
        } else if (fd >= 0 ? (fa < 0) : (fa > 0)) {
            b = d; fb = fd;
        } else {
            a = d; fa = fd;
        }
    }
    double x = (a + b) * 0.5;
    for (int iter = 0; iter < 10; ++iter) {
        const double fx = sturm_polyval10(fvec, x);
        if (fabs(fx) < tol) break;
        const double fpx = 10.0 * sturm_polyval9(fvec + 11, x);
        const double dx = fx / fpx;
        x = x - dx;
        if (fabs(dx) < tol) break;
    }
    roots[n_roots++] = x;
}
// coeffs: 11 ascending coefficients; roots: up to 10, ascending.  w: scratch (shared or local).
PLB_DEV int sturm_bisect10(const double *coeffs, double *roots, SturmWork *w) {
    constexpr int N = 10;
    const double tol = 1e-10;
    if (coeffs[N] == 0.0) return 0;
    double *fvec = w->fvec, *svec = w->svec;
    const double c_inv = 1.0 / coeffs[N];
#pragma unroll
    for (int i = 0; i < N; ++i) fvec[i] = coeffs[i] * c_inv;
    fvec[N] = 1.0;
#pragma unroll
    for (int i = 0; i < N - 1; ++i) fvec[N + 1 + i] = fvec[i + 1] * ((i + 1) / double(N));
    fvec[2 * N] = 1.0;
    sturm_build_seq(fvec, svec);
    double mx = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) mx = fmax(mx, fabs(fvec[i]));
    const double r0 = 1.0 + mx;
    const int s_lo = sturm_signchanges(svec, -r0), s_hi = sturm_signchanges(svec, r0);
    if (s_lo - s_hi == 0) return 0;
    int n_roots = 0;
    // explicit stack of pending right halves.  A right half is only worth visiting if it holds a root (sc-sb >= 1)
    // or is already narrower than tol (the reference then emits its upper end whatever the count, sturm.h:216-219);
    // pending intervals are disjoint and each holds >= 1 root, plus at most one terminal-width one: 12 suffice.
    double st_a[12], st_b[12];
    int st_sa[12], st_sb[12], st_depth[12];
    int sp = 0;
    st_a[0] = -r0; st_b[0] = r0; st_sa[0] = s_lo; st_sb[0] = s_hi; st_depth[0] = 0;
    sp = 1;
    while (sp > 0) {
        --sp;
        double a = st_a[sp], b = st_b[sp];
        int sa = st_sa[sp], sb = st_sb[sp], depth = st_depth[sp];
        // walk down the left spine, pushing right halves
        for (;;) {
            if (depth > 300) break;
            if (b - a < tol) {
                if (n_roots < 10) roots[n_roots++] = b;
                break;
            }
            const int n_rts = sa - sb;
            if (n_rts > 1) {
                const double c = (a + b) * 0.5;
                const int sc = sturm_signchanges(svec, c);
                if (sp < 12 && ((sc - sb) >= 1 || (b - c) < tol)) {
                    st_a[sp] = c; st_b[sp] = b; st_sa[sp] = sc; st_sb[sp] = sb; st_depth[sp] = depth + 1;
                    ++sp;
                }
                b = c;
                sb = sc;
                ++depth;
            } else {
                if (n_rts == 1 && n_roots < 10) sturm_ridders_newton(fvec, a, b, roots, n_roots, tol);
                break;
            }
        }
    }
    return n_roots;
}

// ---- warp-cooperative variant used by k5_roots: lane = sample, 32 samples per warp ------------------------------------
// sturm_bisect10 run by 32 lanes on 32 different polynomials diverges badly: every lane is at a different point of the
// interval walk or inside a Ridders/Newton
// refinement.  The same computation is regrouped into phases that keep the warp converged:
//   A  Sturm sequence of every lane's polynomial (uniform);
//   B  interval walk: cheap transitions (pop / split bookkeeping / emit) advance until the lane needs ONE
//      sturm_signchanges evaluation, which all lanes then execute together; isolated intervals are only RECORDED,
//      in the order the serial routine would refine them;
//   C  the recorded intervals of the whole warp are dealt out to the lanes evenly (prefix sum + binary search) and
//      refined by sturm_ridders_newton with the owner's polynomial read from shared memory;
//   D  every lane compacts its results in recording order, applying the n_roots < 10 guards of the serial routine.
// Functions, operands and per-polynomial operation order are those of sturm_bisect10: results are bit-identical.
constexpr int RT_MAXB = 16; // recorded intervals per polynomial; more (never seen) falls back to the serial routine
struct RootsShared {        // per warp
    double fvec[21][32];
    double a[RT_MAXB][32]; // interval start; overwritten by the refined root
    double b[RT_MAXB][32]; // interval end;   overwritten by 1.0 / 0.0 = root valid / not
    int prefix[33];
};
// c: 11 ascending coefficients (registers); returns the number of roots written to roots[0..n)
PLB_DEV int sturm_bisect10_warp(const double *c, bool has_poly, double *roots, RootsShared *S, int lane) {
    constexpr int N = 10;
    const double tol = 1e-10;
    double fvec[21], svec[30];
    bool done = !has_poly || c[N] == 0.0;
    {
        const double c_inv = done ? 1.0 : 1.0 / c[N];
#pragma unroll
        for (int i = 0; i < N; ++i) fvec[i] = (has_poly ? c[i] : 0.0) * c_inv;
        fvec[N] = 1.0;
#pragma unroll
        for (int i = 0; i < N - 1; ++i) fvec[N + 1 + i] = fvec[i + 1] * ((i + 1) / double(N));
        fvec[2 * N] = 1.0;
#pragma unroll
        for (int i = 0; i < 21; ++i) S->fvec[i][lane] = fvec[i];
    }
    sturm_build_seq(fvec, svec);
    double mx = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) mx = fmax(mx, fabs(fvec[i]));
    const double r0 = 1.0 + mx;
    const int s_lo = sturm_signchanges(svec, -r0), s_hi = sturm_signchanges(svec, r0);
    if (s_lo - s_hi == 0) done = true;
    // ---- phase B
    double st_a[12], st_b[12];
    int st_sa[12], st_sb[12], st_depth[12];
    int sp = 0, nb = 0;
    unsigned degenerate = 0; // bit j: recorded interval j is a terminal-width one whose upper end is the root
    bool overflow = false;
    if (!done) {
        st_a[0] = -r0; st_b[0] = r0; st_sa[0] = s_lo; st_sb[0] = s_hi; st_depth[0] = 0;
        sp = 1;
    }
    double a = 0, b = 0;
    int sa = 0, sb = 0, depth = 0;
    bool walking = false;
    for (;;) {
        bool need = false;
        double cm = 0.0;
        while (!done && !need) {
            if (!walking) {
                if (sp == 0) {
                    done = true;
                    break;
                }
                --sp;
                a = st_a[sp]; b = st_b[sp]; sa = st_sa[sp]; sb = st_sb[sp]; depth = st_depth[sp];
                walking = true;
            }
            if (depth > 300) {
                walking = false;
            } else if (b - a < tol) {
                if (nb < RT_MAXB) {
                    S->a[nb][lane] = a;
                    S->b[nb][lane] = b;
                    degenerate |= 1u << nb;
                    ++nb;
                } else {
                    overflow = true;
                }
                walking = false;
            } else {
                const int n_rts = sa - sb;
                if (n_rts > 1) {
                    cm = (a + b) * 0.5;
                    need = true;
                } else {
                    if (n_rts == 1) {
                        if (nb < RT_MAXB) {
                            S->a[nb][lane] = a;
                            S->b[nb][lane] = b;
                            ++nb;
                        } else {
                            overflow = true;
                        }
                    }
                    walking = false;
                }
            }
        }
        if (!__any_sync(0xffffffffu, need)) break;
        int sc = 0;
        if (need) sc = sturm_signchanges(svec, cm);
        if (need) {
            if (sp < 12 && ((sc - sb) >= 1 || (b - cm) < tol)) {
                st_a[sp] = cm; st_b[sp] = b; st_sa[sp] = sc; st_sb[sp] = sb; st_depth[sp] = depth + 1;
                ++sp;
            }
            b = cm;
            sb = sc;
            ++depth;
        }
    }
    // ---- phase C: deal the recorded intervals of the warp out to the lanes
    int incl = nb;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    S->prefix[lane + 1] = incl;
    if (lane == 0) S->prefix[0] = 0;
    __syncwarp();
    const int total = S->prefix[32];
    for (int t = lane; t < ((total + 31) & ~31); t += 32) {
        const bool live = t < total;
        int owner = 0, j = 0;
        if (live) {
            int lo = 0, hi = 31; // largest owner with prefix[owner] <= t
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (S->prefix[mid] <= t) lo = mid;
                else hi = mid - 1;
            }
            owner = lo;
            j = t - S->prefix[owner];
        }
        const unsigned deg_owner = __shfl_sync(0xffffffffu, degenerate, owner);
        if (live) {
            const double ia = S->a[j][owner], ib = S->b[j][owner];
            double root = ib;
            int got = 1;
            if (!((deg_owner >> j) & 1u)) {
                double f[21];
#pragma unroll
                for (int i = 0; i < 21; ++i) f[i] = S->fvec[i][owner];
                got = 0;
                sturm_ridders_newton(f, ia, ib, &root, got, tol);
            }
            S->a[j][owner] = root;
            S->b[j][owner] = got ? 1.0 : 0.0;
        }
    }
    __syncwarp();
    // ---- phase D
    int n_roots = 0;
    for (int j = 0; j < nb; ++j)
        if (n_roots < 10 && S->b[j][lane] != 0.0) roots[n_roots++] = S->a[j][lane];
    __syncwarp();
    if (overflow) { // never observed; keeps the routine total
        SturmWork w;
        n_roots = sturm_bisect10(c, roots, &w);
    }
    return n_roots;
}

// ================================ relpose_5pt (Nister) =====================================================
// Back-substitution for one root z of the determinant polynomial: E (row-major 9) from the polynomial matrix A (3x13)
// and the nullspace basis Nb (relpose_5pt.cc:359-392).
// A / Nb: anything indexable (plain pointers, or StridedD views of the entry-major per-sample blocks).
struct StridedD {
    const double *p;
    size_t stride;
    PLB_DEV double operator[](int i) const { return p[(size_t)i * stride]; }
    PLB_DEV StridedD operator+(int o) const { return StridedD{p + (size_t)o * stride, stride}; }
};
template <class VA, class VN> PLB_DEV void backsub_5pt(VA A, VN Nb, double z, double *E) {
    {
        const double z2 = z * z, z3 = z2 * z, z4 = z2 * z2;
        double B[3][2], bb[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            B[r][0] = A[13 * r + 0] * z3 + A[13 * r + 1] * z2 + A[13 * r + 2] * z + A[13 * r + 3];
            B[r][1] = A[13 * r + 4] * z3 + A[13 * r + 5] * z2 + A[13 * r + 6] * z + A[13 * r + 7];
            bb[r] = A[13 * r + 8] * z4 + A[13 * r + 9] * z3 + A[13 * r + 10] * z2 + A[13 * r + 11] * z + A[13 * r + 12];
        }
        const double det = B[0][0] * B[1][1] - B[0][1] * B[1][0];
        const double id = 1.0 / det;
        const double i00 = B[1][1] * id, i01 = -B[0][1] * id, i10 = -B[1][0] * id, i11 = B[0][0] * id;
        double s0 = i00 * bb[0] + i01 * bb[1], s1 = i10 * bb[0] + i11 * bb[1];
        if (fabs(B[2][0] * s0 + B[2][1] * s1 - bb[2]) > 1e-6) {
            // rare fallback (:380-382): column-pivoted Householder least squares on the 3x2 system
            double Aq[3][2] = {{B[0][0], B[0][1]}, {B[1][0], B[1][1]}, {B[2][0], B[2][1]}};
            double rhs[3] = {bb[0], bb[1], bb[2]};
            int p0 = 0, p1 = 1;
            const double n0 = Aq[0][0] * Aq[0][0] + Aq[1][0] * Aq[1][0] + Aq[2][0] * Aq[2][0];
            const double n1 = Aq[0][1] * Aq[0][1] + Aq[1][1] * Aq[1][1] + Aq[2][1] * Aq[2][1];
            if (n1 > n0) {
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const double t = Aq[r][0];
                    Aq[r][0] = Aq[r][1];
                    Aq[r][1] = t;
                }
                p0 = 1;
                p1 = 0;
            }
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                double tail_sq = 0.0;
#pragma unroll
                for (int r = k + 1; r < 3; ++r) tail_sq += Aq[r][k] * Aq[r][k];
                const double c0 = Aq[k][k];
                double tau = 0.0, beta = c0, ess[3] = {0, 0, 0};
                if (tail_sq > 2.2250738585072014e-308) {
                    beta = sqrt(c0 * c0 + tail_sq);
                    if (c0 >= 0) beta = -beta;
#pragma unroll
                    for (int r = k + 1; r < 3; ++r) ess[r] = Aq[r][k] / (c0 - beta);
                    tau = (beta - c0) / beta;
                }
                Aq[k][k] = beta;
                if (tau != 0.0) {
                    if (k == 0) {
                        double tmp = Aq[0][1];
#pragma unroll
                        for (int r = 1; r < 3; ++r) tmp += ess[r] * Aq[r][1];
                        Aq[0][1] -= tau * tmp;
#pragma unroll
                        for (int r = 1; r < 3; ++r) Aq[r][1] -= tau * ess[r] * tmp;
                    }
                    double tmp = rhs[k];
#pragma unroll
                    for (int r = k + 1; r < 3; ++r) tmp += ess[r] * rhs[r];
                    rhs[k] -= tau * tmp;
#pragma unroll
                    for (int r = k + 1; r < 3; ++r) rhs[r] -= tau * ess[r] * tmp;
                }
            }
            const double y1 = rhs[1] / Aq[1][1];
            const double y0 = (rhs[0] - Aq[0][1] * y1) / Aq[0][0];
            if (p0 == 0) { s0 = y0; s1 = y1; } else { s1 = y0; s0 = y1; }
            (void)p1;
        }
        const double x = -s0, y = -s1;
        const double inv_norm = 1.0 / sqrt(x * x + y * y + z * z + 1.0);
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            const double e = Nb[4 * k + 0] * x + Nb[4 * k + 1] * y + Nb[4 * k + 2] * z + Nb[4 * k + 3];
            E[3 * (k % 3) + (k / 3)] = e * inv_norm; // k is the column-major index
        }
    }
}

// Four motion hypotheses of an essential matrix, filtered by cheirality on the sample (misc/essential.cc:103-169).
// E: row-major; x1s/x2s: ns unit bearings each.  Returns a 4-bit mask of accepted candidates and writes all four
// candidate poses to cand[4][7] (registers of the calling lane).
template <class VX> PLB_DEV unsigned motions_from_E(const double *E9, VX x1s, VX x2s, int ns, double cand[4][7]) {
    m3 E;
#pragma unroll
    for (int k = 0; k < 9; ++k) E.a[k] = E9[k];
    const d3 e0 = mcol(E, 0), e1 = mcol(E, 1), e2 = mcol(E, 2);
    const d3 u12 = cross(e0, e1), u13 = cross(e0, e2), u23 = cross(e1, e2);
    const double n12 = dot(u12, u12), n13 = dot(u13, u13), n23 = dot(u23, u23);
    d3 c1, c2;
    if (n12 > n13) {
        if (n12 > n23) { c1 = unit(e0); c2 = u12 / sqrt(n12); }
        else { c1 = unit(e1); c2 = u23 / sqrt(n23); }
    } else {
        if (n13 > n23) { c1 = unit(e0); c2 = u13 / sqrt(n13); }
        else { c1 = unit(e1); c2 = u23 / sqrt(n23); }
    }
    const d3 c0 = -cross(c2, c1);
    d3 v0 = mtvec(E, c1);
    d3 v1 = mtvec(E, -c0);
    v0 = unit(v0);
    v1 = v1 - dot(v0, v1) * v0;
    v1 = unit(v1);
    m3 Vt;
    set_row(Vt, 0, v0);
    set_row(Vt, 1, v1);
    set_row(Vt, 2, cross(v0, v1));
    m3 UW;
    set_col(UW, 0, c0);
    set_col(UW, 1, c1);
    set_col(UW, 2, c2);
    double qa[4], qb[4];
    rot_to_quat(mmul(UW, Vt), qa);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        UW(r, 0) = -UW(r, 0);
        UW(r, 1) = -UW(r, 1);
    }
    rot_to_quat(mmul(UW, Vt), qb);
    // The four candidates are (qa, t), (qa, -t), (qb, -t), (qb, t) (reference order).  check_cheirality
    // (misc/essential.cc:40-57) of (q, -t) yields exactly the negated depths of (q, t): dot products, products and the
    // two-term sums are symmetric under negation in round-to-nearest, and min_depth = 0 makes the bound a signed zero.
    // So one evaluation per (rotation, point) decides both translation signs — half the work, and without the
    // per-candidate early exits that kept half the lanes of k5_back idle.
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const double *q = (c < 2) ? qa : qb;
        const double sgn = (c == 0 || c == 3) ? 1.0 : -1.0;
        cand[c][0] = q[0]; cand[c][1] = q[1]; cand[c][2] = q[2]; cand[c][3] = q[3];
        cand[c][4] = sgn * c2.x; cand[c][5] = sgn * c2.y; cand[c][6] = sgn * c2.z;
    }
    unsigned mask = 0;
#pragma unroll
    for (int rot = 0; rot < 2; ++rot) {
        const double *q = rot ? qb : qa;
        bool okp = true, okm = true; // translation +c2 / -c2
        for (int i = 0; i < ns; ++i) {
            const d3 a = mk(x1s[3 * i], x1s[3 * i + 1], x1s[3 * i + 2]);
            const d3 b = mk(x2s[3 * i], x2s[3 * i + 1], x2s[3 * i + 2]);
            const d3 Rx1 = quat_rotate(q, a);
            const double ca = -dot(Rx1, b);
            const double b1 = -dot(Rx1, c2);
            const double b2 = dot(b, c2);
            const double lambda1 = b1 - ca * b2;
            const double lambda2 = -ca * b1 + b2;
            const double md = 0.0 * (1 - ca * ca);
            okp = okp && (lambda1 > md && lambda2 > md);
            okm = okm && (-lambda1 > md && -lambda2 > md);
            if (!okp && !okm) break;
        }
        if (rot == 0) {
            if (okp) mask |= 1u;
            if (okm) mask |= 2u;
        } else {
            if (okm) mask |= 4u;
            if (okp) mask |= 8u;
        }
    }
    return mask;
}

// robust/utils.cc:646-672 — note the reference stores the products in `float`
PLB_DEV bool rfc_ok(const double *Fc /*column-major*/) {
#define F_(r, c) Fc[3 * (c) + (r)]
    float den, num;
    den = F_(0, 0) * F_(0, 1) * F_(2, 0) * F_(2, 2) - F_(0, 0) * F_(0, 2) * F_(2, 0) * F_(2, 1) +
          F_(0, 1) * F_(0, 1) * F_(2, 1) * F_(2, 2) - F_(0, 1) * F_(0, 2) * F_(2, 1) * F_(2, 1) +
          F_(1, 0) * F_(1, 1) * F_(2, 0) * F_(2, 2) - F_(1, 0) * F_(1, 2) * F_(2, 0) * F_(2, 1) +
          F_(1, 1) * F_(1, 1) * F_(2, 1) * F_(2, 2) - F_(1, 1) * F_(1, 2) * F_(2, 1) * F_(2, 1);
    num = -F_(2, 2) * (F_(0, 1) * F_(0, 2) * F_(2, 2) - F_(0, 2) * F_(0, 2) * F_(2, 1) + F_(1, 1) * F_(1, 2) * F_(2, 2) -
                       F_(1, 2) * F_(1, 2) * F_(2, 1));
    if (num * den < 0) return false;
    den = F_(0, 0) * F_(1, 0) * F_(0, 2) * F_(2, 2) - F_(0, 0) * F_(2, 0) * F_(0, 2) * F_(1, 2) +
          F_(1, 0) * F_(1, 0) * F_(1, 2) * F_(2, 2) - F_(1, 0) * F_(2, 0) * F_(1, 2) * F_(1, 2) +
          F_(0, 1) * F_(1, 1) * F_(0, 2) * F_(2, 2) - F_(0, 1) * F_(2, 1) * F_(0, 2) * F_(1, 2) +
          F_(1, 1) * F_(1, 1) * F_(1, 2) * F_(2, 2) - F_(1, 1) * F_(2, 1) * F_(1, 2) * F_(1, 2);
    num = -F_(2, 2) * (F_(1, 0) * F_(2, 0) * F_(2, 2) - F_(2, 0) * F_(2, 0) * F_(1, 2) + F_(1, 1) * F_(2, 1) * F_(2, 2) -
                       F_(2, 1) * F_(2, 1) * F_(1, 2));
    if (num * den < 0) return false;
    return true;
#undef F_
}

// ================================ relpose_7pt ==============================================================
// F matrices (column-major) of 7 bearing pairs into F[0..n), n returned; only those for which keep(f) holds are listed,
// order preserved (the real-focal check of estimators/relative_pose.cc:393-398).  relpose_7pt.cc:10-60
// W: the thread's 63-double scratch (the 9 x 7 system for lane5::nullspace_9xC).
template <class Keep> PLB_DEV int fundamental_7pt(const double *x1s, const double *x2s, double *W, Keep &&keep, double F[3][9]) {
#pragma unroll
    for (int e = 0; e < 63; ++e) {
        const int i = e / 9, k = e % 9;
        W[e] = x1s[3 * i + k / 3] * x2s[3 * i + k % 3];
    }
    double nn[18];
    lane5::nullspace_9xC<7>(W, nn);
    const double *n0 = nn, *n1 = nn + 9;
    // mixed determinants: column j of the 3x3 (col-major 9-vector) taken from a, b, c respectively
    auto detc = [](const double *a, const double *b, const double *c) -> double {
        const double *c0 = a, *c1 = b + 3, *c2 = c + 6;
        return c0[0] * (c1[1] * c2[2] - c1[2] * c2[1]) - c1[0] * (c0[1] * c2[2] - c0[2] * c2[1]) +
               c2[0] * (c0[1] * c1[2] - c0[2] * c1[1]);
    };
    const double c3 = detc(n0, n0, n0);
    const double c2 = detc(n1, n0, n0) + detc(n0, n1, n0) + detc(n0, n0, n1);
    const double c1 = detc(n0, n1, n1) + detc(n1, n0, n1) + detc(n1, n1, n0);
    const double c0 = detc(n1, n1, n1);
    double roots[3];
    int n_roots;
    if (fabs(c3) < 1e-14) {
        n_roots = quadratic_real(c2, c1, c0, roots);
    } else {
        const double inv_c3 = 1.0 / c3;
        n_roots = cubic_real(c2 * inv_c3, c1 * inv_c3, c0 * inv_c3, roots);
    }
    int nm = 0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        if (j < n_roots) {
            const double r = roots[j];
            double f[9];
            double n2 = 0.0;
#pragma unroll
            for (int k = 0; k < 9; ++k) {
                f[k] = n0[k] * r + n1[k];
                n2 += f[k] * f[k];
            }
            if (n2 > 0) {
                const double nrm = sqrt(n2);
#pragma unroll
                for (int k = 0; k < 9; ++k) f[k] /= nrm;
            }
            if (keep(f)) {
                // nm is 0, 1 or 2 here: predicated copies keep F in registers
#pragma unroll
                for (int m = 0; m < 3; ++m)
                    if (m == nm) {
#pragma unroll
                        for (int k = 0; k < 9; ++k) F[m][k] = f[k];
                    }
                ++nm;
            }
        }
    }
    return nm;
}

} // namespace plb
