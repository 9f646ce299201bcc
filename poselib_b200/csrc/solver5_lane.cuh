// relpose_5pt, first half (nullspace, trace / determinant constraints, elimination, determinant polynomial) with ONE
// THREAD PER MINIMAL SAMPLE.
//
// Most steps of this half are only 5..20 wide, so a thread owns a sample.  The monomial tables are compile-time
// constants: the nullspace basis and the quadratic blocks live in registers with static indices, and only the left
// 10 x 10 block of the elimination matrix (dynamic pivot rows) sits in the thread's slice of shared memory while the
// right-hand sides are parked elsewhere.  Every value is produced by the same sequence of IEEE operations as in the CPU
// restatement (the file is compiled with -fmad=false), so the outputs are bit-identical;
// tests/test_solver5_lane_host.py checks that on the host build of this very source.
//
// Reference: PoseLib/solvers/relpose_5pt.cc:101-157 (constraints), :159-189 (nullspace, elimination), :191-352
// (determinant polynomial).  Eigen's FullPivHouseholderQR / PartialPivLU are restated below.
#pragma once
#include <cmath>
#include <type_traits>
#include <utility>

#ifndef PLB_L5
#define PLB_L5 __host__ __device__ __forceinline__
#endif

namespace plb {
namespace lane5 {

template <class F, int... I> PLB_L5 void static_for_impl(F &&f, std::integer_sequence<int, I...>) {
    (f(std::integral_constant<int, I>{}), ...);
}
template <int N, class F> PLB_L5 void static_for(F &&f) { static_for_impl(f, std::make_integer_sequence<int, N>{}); }

// quadratic monomials [x^2, xy, xz, x, y^2, yz, y, z^2, z, 1] as (i <= j) pairs of the linear ones [x, y, z, 1]
// (relpose_5pt.cc:11-12); cubic monomials [x^3,y^3,x^2y,xy^2,x^2z,x^2,y^2z,y^2,xyz,xy,xz^2,xz,x,yz^2,yz,y,z^3,z^2,z,1]
// (:54-55) as their (quadratic, linear) factorisations in (q, l) lexicographic order
struct Tables {
    int quad_i[10], quad_j[10];
    int cub_n[20], cub_q[20][3], cub_l[20][3];
};
constexpr Tables make_tables() {
    Tables T{};
    const int qexp[10][3] = {{2, 0, 0}, {1, 1, 0}, {1, 0, 1}, {1, 0, 0}, {0, 2, 0},
                             {0, 1, 1}, {0, 1, 0}, {0, 0, 2}, {0, 0, 1}, {0, 0, 0}};
    const int cexp[20][3] = {{3, 0, 0}, {0, 3, 0}, {2, 1, 0}, {1, 2, 0}, {2, 0, 1}, {2, 0, 0}, {0, 2, 1},
                             {0, 2, 0}, {1, 1, 1}, {1, 1, 0}, {1, 0, 2}, {1, 0, 1}, {1, 0, 0}, {0, 1, 2},
                             {0, 1, 1}, {0, 1, 0}, {0, 0, 3}, {0, 0, 2}, {0, 0, 1}, {0, 0, 0}};
    const int lexp[4][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {0, 0, 0}};
    int qn = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = i; j < 4; ++j) {
            T.quad_i[qn] = i;
            T.quad_j[qn] = j;
            ++qn;
        }
    for (int ci = 0; ci < 20; ++ci) {
        int n = 0;
        for (int q = 0; q < 10; ++q)
            for (int l = 0; l < 4; ++l)
                if (qexp[q][0] + lexp[l][0] == cexp[ci][0] && qexp[q][1] + lexp[l][1] == cexp[ci][1] &&
                    qexp[q][2] + lexp[l][2] == cexp[ci][2]) {
                    T.cub_q[ci][n] = q;
                    T.cub_l[ci][n] = l;
                    ++n;
                }
        T.cub_n[ci] = n;
    }
    return T;
}
constexpr Tables TB = make_tables();

// ---- nullspace of the 9 x C epipolar matrix (C = 5: relpose_5pt, C = 7: relpose_7pt) --------------------------------------------------------------------------
// a: 9 C doubles, column-major (a[c * 9 + r]), overwritten; put(s, r, v) receives entry r of the s-th basis vector =
// column C + s of the Householder Q of the full-pivoting QR (relpose_5pt.cc:167-168, relpose_7pt.cc:18-19): Eigen's
// pivot rule (largest |entry|, first in column-major order on ties), reflectors and order of the row transpositions.
// s and r are compile-time after unrolling, so the basis can go straight to registers or to its final place.
template <int COLS, class Sink> PLB_L5 void nullspace_basis(double *a, Sink &&put) {
    constexpr int ROWS = 9;
    double tau_k[COLS];
    int rt_k[COLS];
    const double precision = 2.220446049250313e-16 * double(COLS);
    double biggest = 0.0;
    bool stopped = false;
#pragma unroll
    for (int k = 0; k < COLS; ++k) {
        double best = -1.0;
        int cb = k, rb = k;
        for (int c = k; c < COLS; ++c)
            for (int r = k; r < ROWS; ++r) {
                const double v = fabs(a[c * ROWS + r]);
                if (v > best) {
                    best = v;
                    cb = c;
                    rb = r;
                }
            }
        if (k == 0) biggest = best;
        if (!stopped && fabs(best) <= fabs(biggest) * precision) stopped = true;
        if (stopped) {
            cb = k;
            rb = k;
        }
        rt_k[k] = rb;
        // row transposition on the columns still active, then the column transposition (all rows); with rb == k or
        // cb == k they leave the matrix as it is
        for (int c = k; c < COLS; ++c) {
            const double t = a[c * ROWS + k];
            a[c * ROWS + k] = a[c * ROWS + rb];
            a[c * ROWS + rb] = t;
        }
        for (int r = 0; r < ROWS; ++r) {
            const double t = a[k * ROWS + r];
            a[k * ROWS + r] = a[cb * ROWS + r];
            a[cb * ROWS + r] = t;
        }
        double v[ROWS]; // the reflector's essential part, kept in registers for the updates below
        double tail_sq = 0.0;
#pragma unroll
        for (int r = 0; r < ROWS; ++r)
            if (r > k) {
                v[r] = a[k * ROWS + r];
                tail_sq += v[r] * v[r];
            }
        const double c0 = a[k * ROWS + k];
        double tau = 0.0;
        if (!stopped) {
            double beta;
            if (tail_sq <= 2.2250738585072014e-308) {
                beta = c0;
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
                    if (r > k) v[r] = 0.0;
            } else {
                beta = sqrt(c0 * c0 + tail_sq);
                if (c0 >= 0) beta = -beta;
                const double den = c0 - beta;
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
                    if (r > k) v[r] = v[r] / den;
                tau = (beta - c0) / beta;
            }
#pragma unroll
            for (int r = 0; r < ROWS; ++r)
                if (r > k) a[k * ROWS + r] = v[r];
            a[k * ROWS + k] = beta;
        }
        tau_k[k] = tau;
        if (tau != 0.0) {
            for (int c = k + 1; c < COLS; ++c) {
                double *col = a + c * ROWS;
                double cr[ROWS];
                double tmp = 0.0;
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
                    if (r > k) {
                        cr[r] = col[r];
                        tmp += v[r] * cr[r];
                    }
                const double ck = col[k];
                tmp += ck;
                col[k] = ck - tau * tmp;
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
                    if (r > k) col[r] = cr[r] - tau * v[r] * tmp;
            }
        }
    }
    // the four basis vectors together: the reflector of a step is read once and the four chains are independent
    double q[ROWS - COLS][ROWS];
#pragma unroll
    for (int s = 0; s < ROWS - COLS; ++s)
#pragma unroll
        for (int r = 0; r < ROWS; ++r) q[s][r] = (r == COLS + s) ? 1.0 : 0.0;
#pragma unroll
    for (int k = COLS - 1; k >= 0; --k) {
        const double tau = tau_k[k];
        if (tau != 0.0) {
            double vr[ROWS];
#pragma unroll
            for (int r = 0; r < ROWS; ++r)
                if (r > k) vr[r] = a[k * ROWS + r];
#pragma unroll
            for (int s = 0; s < ROWS - COLS; ++s) {
                double tmp = 0.0;
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
                    if (r > k) tmp += vr[r] * q[s][r];
                tmp += q[s][k];
                q[s][k] -= tau * tmp;
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
                    if (r > k) q[s][r] -= tau * vr[r] * tmp;
            }
        }
        const int rt = rt_k[k];
        if (rt != k) {
#pragma unroll
            for (int s = 0; s < ROWS - COLS; ++s) {
                const double qk = q[s][k];
                double qr = 0.0;
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
                    if (r == rt) qr = q[s][r];
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
                    if (r == rt) q[s][r] = qk;
                q[s][k] = qr;
            }
        }
    }
#pragma unroll
    for (int s = 0; s < ROWS - COLS; ++s)
#pragma unroll
        for (int r = 0; r < ROWS; ++r) put(s, r, q[s][r]);
}
// qn: 9 (9 - C) doubles, qn[9 * s + r] = entry r of the s-th basis vector
template <int COLS> PLB_L5 void nullspace_9xC(double *a, double *qn) {
    nullspace_basis<COLS>(a, [&](int s, int r, double v) { qn[9 * s + r] = v; });
}
PLB_L5 void nullspace_9x5(double *a, double *qn) { nullspace_9xC<5>(a, qn); }

// ---- constraints -> 10 x 20 coefficient matrix ---------------------------------------------------------------------
// Nb[4 * k + r]: coefficient of basis r (x, y, z, 1) in entry k (column-major) of E.  E(i, j) as a linear polynomial:
#define PLB_L5_E(i, j, q) Nb[4 * (3 * (j) + (i)) + (q)]

// One quadratic block (10 coefficients): BLK 0..5 = entries (0,0),(0,1),(0,2),(1,1),(1,2),(2,2) of E E^T, BLK 6..8 = the
// minors d_t of the cofactor expansion of det(E) along its last row (relpose_5pt.cc:113-123,129-138).
template <int BLK> PLB_L5 void quad_block(const double *Nb, double *qv) {
    static_for<10>([&](auto mc) {
        constexpr int m = decltype(mc)::value;
        constexpr int qi = TB.quad_i[m], qj = TB.quad_j[m];
        constexpr bool same = qi == qj;
        double v = 0.0;
        if constexpr (BLK < 6) {
            constexpr int i = (BLK < 3) ? 0 : (BLK < 5 ? 1 : 2);
            constexpr int j = (BLK < 3) ? BLK : (BLK < 5 ? BLK - 2 : 2);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                v = v + PLB_L5_E(i, k, qi) * PLB_L5_E(j, k, qj);
                if (!same) v = v + PLB_L5_E(i, k, qj) * PLB_L5_E(j, k, qi);
            }
        } else {
            constexpr int t = BLK - 6;
            constexpr int c1 = (t == 0) ? 1 : (t == 1 ? 2 : 0);
            constexpr int c2 = (t == 0) ? 2 : (t == 1 ? 0 : 1);
            v = v + PLB_L5_E(0, c1, qi) * PLB_L5_E(1, c2, qj);
            if (!same) v = v + PLB_L5_E(0, c1, qj) * PLB_L5_E(1, c2, qi);
            v = v - PLB_L5_E(0, c2, qi) * PLB_L5_E(1, c1, qj);
            if (!same) v = v - PLB_L5_E(0, c2, qj) * PLB_L5_E(1, c1, qi);
        }
        qv[m] = v;
    });
}

// Rows 3 i .. 3 i + 2 of the coefficient matrix from the three blocks (E E^T - trace / 2)(i, 0..2)  (:146-154)
template <int I, class Sink> PLB_L5 void cubic_rows(const double *Nb, const double *q0, const double *q1, const double *q2, Sink &&put) {
    static_for<20>([&](auto cc) {
        constexpr int ci = decltype(cc)::value;
        constexpr int np = TB.cub_n[ci];
        constexpr int a0 = TB.cub_q[ci][0], a1 = TB.cub_q[ci][1], a2 = TB.cub_q[ci][2];
        constexpr int l0 = TB.cub_l[ci][0], l1 = TB.cub_l[ci][1], l2 = TB.cub_l[ci][2];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            double v = 0.0;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const double *Q = (k == 0) ? q0 : (k == 1 ? q1 : q2);
                v += Q[a0] * PLB_L5_E(k, j, l0);
                if (np > 1) v += Q[a1] * PLB_L5_E(k, j, l1);
                if (np > 2) v += Q[a2] * PLB_L5_E(k, j, l2);
            }
            put(3 * I + j, cc, v);
        }
    });
}
// Row 9: det(E) = sum_t d_t E(2, t)  (:113-125)
template <class Sink> PLB_L5 void cubic_det_row(const double *Nb, const double *d0, const double *d1, const double *d2, Sink &&put) {
    static_for<20>([&](auto cc) {
        constexpr int ci = decltype(cc)::value;
        constexpr int np = TB.cub_n[ci];
        constexpr int a0 = TB.cub_q[ci][0], a1 = TB.cub_q[ci][1], a2 = TB.cub_q[ci][2];
        constexpr int l0 = TB.cub_l[ci][0], l1 = TB.cub_l[ci][1], l2 = TB.cub_l[ci][2];
        double v = 0.0;
#pragma unroll
        for (int t = 0; t < 3; ++t) {
            const double *Q = (t == 0) ? d0 : (t == 1 ? d1 : d2);
            v += Q[a0] * PLB_L5_E(2, t, l0);
            if (np > 1) v += Q[a1] * PLB_L5_E(2, t, l1);
            if (np > 2) v += Q[a2] * PLB_L5_E(2, t, l2);
        }
        put(9, cc, v);
    });
}

// Nb (36, registers) -> the 10 x 20 coefficient matrix, entry by entry through put(row, integral_constant<ci>, value).
// The blocks are formed group by group so that at most three of them (plus the trace term) are live at a time.
template <class Sink> PLB_L5 void build_coeffs(const double *Nb, Sink &&put) {
    {
        double d0[10], d1[10], d2[10];
        quad_block<6>(Nb, d0);
        quad_block<7>(Nb, d1);
        quad_block<8>(Nb, d2);
        cubic_det_row(Nb, d0, d1, d2, put);
    }
    double tr[10]; // half the trace of E E^T (:139-144)
    {
        double a[10], b[10], c[10];
        quad_block<0>(Nb, a);
        quad_block<3>(Nb, b);
        quad_block<5>(Nb, c);
#pragma unroll
        for (int m = 0; m < 10; ++m) tr[m] = 0.5 * (a[m] + b[m] + c[m]);
    }
    {
        double q0[10], q1[10], q2[10];
        quad_block<0>(Nb, q0);
        quad_block<1>(Nb, q1);
        quad_block<2>(Nb, q2);
#pragma unroll
        for (int m = 0; m < 10; ++m) q0[m] -= tr[m];
        cubic_rows<0>(Nb, q0, q1, q2, put);
    }
    {
        double q0[10], q1[10], q2[10];
        quad_block<1>(Nb, q0);
        quad_block<3>(Nb, q1);
        quad_block<4>(Nb, q2);
#pragma unroll
        for (int m = 0; m < 10; ++m) q1[m] -= tr[m];
        cubic_rows<1>(Nb, q0, q1, q2, put);
    }
    {
        double q0[10], q1[10], q2[10];
        quad_block<2>(Nb, q0);
        quad_block<4>(Nb, q1);
        quad_block<5>(Nb, q2);
#pragma unroll
        for (int m = 0; m < 10; ++m) q2[m] -= tr[m];
        cubic_rows<2>(Nb, q0, q1, q2, put);
    }
}
#undef PLB_L5_E

// ---- [A | B] -> rows 4..9 of A^{-1} B (:173) ---------------------------------------------------------------------------
// Only the left 10 x 10 block is kept in the thread's scratch (CL, row-major, stride 10); the right-hand sides are
// parked elsewhere (global memory on the device) while it is factored, and then come back one column at a time.
//
// lu_left: partial-pivot LU in place, full-row transpositions, multipliers stored below the diagonal (the LAPACK
// arrangement).  idx[r] = original row that ends up at position r.  S: 10 doubles of scratch.
PLB_L5 void lu_left(double *CL, double *S, int *idx) {
    // row bookkeeping in the double scratch (small integers are exact; no second type aliasing the same bytes)
#pragma unroll
    for (int r = 0; r < 10; ++r) S[r] = (double)r;
#pragma unroll
    for (int k = 0; k < 10; ++k) {
        int p = k;
        double best = fabs(CL[k * 10 + k]);
#pragma unroll
        for (int r = k + 1; r < 10; ++r) {
            const double v = fabs(CL[r * 10 + k]);
            if (v > best) {
                best = v;
                p = r;
            }
        }
        {
            const double t = S[k]; // p == k: no change
            S[k] = S[p];
            S[p] = t;
        }
        double *rk = CL + k * 10, *rp = CL + p * 10;
#pragma unroll
        for (int c = 0; c < 10; ++c) {
            const double t = rk[c];
            rk[c] = rp[c];
            rp[c] = t;
        }
        const double pv = rk[k];
        double lmul[10];
#pragma unroll
        for (int r = 0; r < 10; ++r)
            if (r > k) {
                const double v = CL[r * 10 + k];
                lmul[r] = (best != 0.0) ? v / pv : v;
                CL[r * 10 + k] = lmul[r];
            }
#pragma unroll
        for (int c = 0; c < 10; ++c)
            if (c > k) {
                const double ckc = rk[c];
#pragma unroll
                for (int r = 0; r < 10; ++r)
                    if (r > k) CL[r * 10 + c] -= lmul[r] * ckc;
            }
    }
#pragma unroll
    for (int r = 0; r < 10; ++r) idx[r] = (int)S[r];
}

// The right-hand sides: get(row, column) returns the parked entry; each column is permuted (through S), run through
// the unit-lower solve (per element the same products, subtracted in the same order, as the rank-1 updates of the fused
// form) and the back substitution of rows 9..4.  X (60 doubles, may alias CL: the factors are in registers by then)
// receives rows 4..9 of A^{-1} B, X[(r - 4) * 10 + column].
template <class Get> PLB_L5 void solve_rhs(const double *CL, double *S, const int *idx, Get &&get, double *X) {
    double L[10][10], U[10][10], diag[10]; // static indices: 45 + 15 + 6 values in registers
#pragma unroll
    for (int r = 0; r < 10; ++r)
#pragma unroll
        for (int k = 0; k < 10; ++k) {
            if (k < r) L[r][k] = CL[r * 10 + k];
            if (r >= 4 && k > r) U[r][k] = CL[r * 10 + k];
        }
#pragma unroll
    for (int r = 4; r < 10; ++r) diag[r] = CL[r * 10 + r];
#pragma unroll 1
    for (int c = 0; c < 10; ++c) {
        double b[10];
#pragma unroll
        for (int r = 0; r < 10; ++r) S[r] = get(r, c);
#pragma unroll
        for (int r = 0; r < 10; ++r) b[r] = S[idx[r]];
#pragma unroll
        for (int k = 0; k < 9; ++k)
#pragma unroll
            for (int r = k + 1; r < 10; ++r) b[r] -= L[r][k] * b[k];
#pragma unroll
        for (int r = 9; r >= 4; --r) {
            double sum = b[r];
#pragma unroll
            for (int k = 0; k < 10; ++k)
                if (k > r) sum -= U[r][k] * b[k];
            b[r] = sum / diag[r];
            X[(r - 4) * 10 + c] = b[r];
        }
    }
}

// ---- 3 x 13 polynomial matrix (:176-189) and det(A(z)), ascending coefficients (:191-352) ----------------------------
PLB_L5 void poly_matrix(const double *X, double *A) {
#pragma unroll
    for (int e = 0; e < 39; ++e) {
        const int i = e / 13, c = e % 13;
        const double *top = X + (2 * i) * 10, *bot = X + (2 * i + 1) * 10;
        const int g0 = (c < 4) ? 0 : (c < 8 ? 4 : 8), src0 = (c < 4) ? 0 : (c < 8 ? 3 : 6);
        const int w = (c < 8) ? 3 : 4, o = c - g0;
        double v = 0.0;
        if (o >= 1) v = top[src0 + o - 1];
        if (o < w) v -= bot[src0 + o];
        A[e] = v;
    }
}
// p_ij ascending: p_i0[k] = A[i][3-k], p_i1[k] = A[i][7-k], p_i2[k] = A[i][12-k]
#define PLB_L5_P(i, j, k) (((j) == 0) ? A[13 * (i) + 3 - (k)] : ((j) == 1 ? A[13 * (i) + 7 - (k)] : A[13 * (i) + 12 - (k)]))
PLB_L5 void det_poly(const double *A, double *cp) {
    double minors[3][8];
    static_for<3>([&](auto tc) {
        constexpr int t = decltype(tc)::value;
        constexpr int ja = (t == 0) ? 1 : 0, jb = (t == 2) ? 1 : 2;
        constexpr int da = 3, db = (jb == 2) ? 4 : 3;
        static_for<8>([&](auto kc) {
            constexpr int k = decltype(kc)::value;
            double v = 0.0;
            if constexpr (k <= da + db) {
                double s1 = 0.0, s2 = 0.0;
#pragma unroll
                for (int i = 0; i <= da; ++i) {
                    const int j = k - i;
                    if (j >= 0 && j <= db) s1 += PLB_L5_P(1, ja, i) * PLB_L5_P(2, jb, j);
                }
#pragma unroll
                for (int i = 0; i <= db; ++i) {
                    const int j = k - i;
                    if (j >= 0 && j <= da) s2 += PLB_L5_P(1, jb, i) * PLB_L5_P(2, ja, j);
                }
                v = s1 - s2;
            }
            minors[t][k] = v;
        });
    });
    static_for<11>([&](auto kc) {
        constexpr int k = decltype(kc)::value;
        double t0 = 0.0, t1 = 0.0, t2 = 0.0;
#pragma unroll
        for (int i = 0; i <= 3; ++i) {
            const int j = k - i;
            if (j >= 0 && j <= 7) t0 += PLB_L5_P(0, 0, i) * minors[0][j];
        }
#pragma unroll
        for (int i = 0; i <= 3; ++i) {
            const int j = k - i;
            if (j >= 0 && j <= 7) t1 += PLB_L5_P(0, 1, i) * minors[1][j];
        }
#pragma unroll
        for (int i = 0; i <= 4; ++i) {
            const int j = k - i;
            if (j >= 0 && j <= 6) t2 += PLB_L5_P(0, 2, i) * minors[2][j];
        }
        double c = 0.0;
        c += t0;
        c -= t1;
        c += t2;
        cp[k] = c;
    });
}
#undef PLB_L5_P

// Whole first half on plain arrays (the host test's entry; the device kernels k5_null and k5_elim string the same pieces
// together with their shared-memory slices and a parking buffer in global memory).  W: >= 210 doubles; xs: the 5 + 5 bearings (x1s | x2s).
PLB_L5 void solve_5pt_poly_lane(double *W, const double *xs, double *Nb, double *A, double *cp) {
    // 9 x 5 epipolar constraints (:163-166): entry 3a+b of column i = x1[i][a] * x2[i][b]
#pragma unroll
    for (int e = 0; e < 45; ++e) {
        const int i = e / 9, k = e % 9;
        W[e] = xs[3 * i + k / 3] * xs[15 + 3 * i + k % 3];
    }
    nullspace_9x5(W, W + 45);
#pragma unroll
    for (int e = 0; e < 36; ++e) {
        const int r = e / 9, k = e % 9;
        Nb[4 * k + r] = W[45 + 9 * r + k];
    }
    double *CL = W, *S = W + 100, *park = W + 110;
    build_coeffs(Nb, [&](int row, auto cc, double v) {
        constexpr int ci = decltype(cc)::value;
        if constexpr (ci < 10) CL[row * 10 + ci] = v;
        else park[row * 10 + (ci - 10)] = v;
    });
    int idx[10];
    lu_left(CL, S, idx);
    solve_rhs(CL, S, idx, [&](int r, int c) { return park[r * 10 + c]; }, CL);
    poly_matrix(CL, A);
    det_poly(A, cp);
}

} // namespace lane5
} // namespace plb
