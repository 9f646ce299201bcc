// poselib_b200 — CUDA kernels of the LO-RANSAC hot path for sm_90a (H100).
//
//   k_transpose        caller AoS doubles -> SoA fp64 (+ fp32 copy) in HBM, coalesced both ways
//   k_hyp<KIND>        persistent, one warp = one minimal sample: gather -> minimal solve -> MSAC score of every
//                      model over all correspondences (lanes stride the SoA arrays, warp-shuffle reduction)
//   k_score_models     exact rescoring of explicit models (initial model, fast-mode confirmation)
//   k_lm<KIND>         Levenberg-Marquardt refit (LO step + final polish): one CTA per job, block-wide reductions of
//                      the normal equations, scalar LM logic on thread 0
//   k_inlier_mask      final inlier masks
//   k_solver_batch     the solvers/*.h surface: one warp per instance
//
// Compiled with -fmad=false (see device_math.cuh).  Reference citations are relative to /root/reference.
#include "kernels.cuh"
#include "solvers.cuh"
#include "screen_math.cuh"
#include "solver5_lane.cuh"
#include <cooperative_groups.h>
#include <type_traits>
#include <cstdlib>
#include <cstring>
#include <algorithm>

namespace plb {

PLB_DEV int min_i(int a, int b) { return a < b ? a : b; }

// ============================================================================================================
// layout transform
// ============================================================================================================
// Per-problem maximum |coordinate| of every SoA array (of the fp64 values, rounded up to float): the error bounds of the
// fp32 screening pass are built on them (screen_math.cuh).  All 32 lanes of a warp call it (n_pad is a multiple of 32).
// NaN coordinates order above every finite value as unsigned bit patterns, so they poison the maximum (and with it the
// bounds: every model of such a problem is rescored exactly).
PLB_DEV void coord_max(float *cmax, int c, double v) {
    if (!cmax) return;
    const unsigned bits = __float_as_uint(scr::f_up(fabs(v)));
    const unsigned m = __reduce_max_sync(0xffffffffu, bits);
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned *>(cmax) + c, m);
}
__global__ void k_transpose(const TransposeDesc *__restrict__ descs) {
    const TransposeDesc &d = descs[blockIdx.y];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= d.n_pad) return;
    const int idx = (k < d.n) ? k : (d.n - 1); // pad by repeating the last point (never read by the kernels)
    double a0 = d.a[2 * (size_t)idx], a1 = d.a[2 * (size_t)idx + 1];
    if (d.mode == 2) {
        // tangent-Sampson pre-step: scaled pixels -> unit bearing + unprojection Jacobian of both images
        double v[9];
        cam_unproject_with_jac(d.cam_a, a0 * d.scale, a1 * d.scale, v, v + 3);
#pragma unroll
        for (int j = 0; j < 3; ++j) d.s64[(size_t)j * d.n_pad + k] = v[j];
#pragma unroll
        for (int j = 0; j < 6; ++j) d.s64[(size_t)(6 + j) * d.n_pad + k] = v[3 + j];
        const double b0 = d.b[2 * (size_t)idx], b1 = d.b[2 * (size_t)idx + 1];
        cam_unproject_with_jac(d.cam_b, b0 * d.scale, b1 * d.scale, v, v + 3);
#pragma unroll
        for (int j = 0; j < 3; ++j) d.s64[(size_t)(3 + j) * d.n_pad + k] = v[j];
#pragma unroll
        for (int j = 0; j < 6; ++j) d.s64[(size_t)(12 + j) * d.n_pad + k] = v[3 + j];
        return;
    }
    if (d.mode == 1) cam_unproject2(d.cam_a, a0, a1, a0, a1);
    if (d.mode == 1 && d.b_dim == 2) {
        double b0, b1;
        cam_unproject2(d.cam_b, d.b[2 * (size_t)idx], d.b[2 * (size_t)idx + 1], b0, b1);
        d.s64[0 * (size_t)d.n_pad + k] = a0;
        d.s64[1 * (size_t)d.n_pad + k] = a1;
        d.s64[2 * (size_t)d.n_pad + k] = b0;
        d.s64[3 * (size_t)d.n_pad + k] = b1;
        d.s32[0 * (size_t)d.n_pad + k] = (float)a0;
        d.s32[1 * (size_t)d.n_pad + k] = (float)a1;
        d.s32[2 * (size_t)d.n_pad + k] = (float)b0;
        d.s32[3 * (size_t)d.n_pad + k] = (float)b1;
        coord_max(d.cmax, 0, a0);
        coord_max(d.cmax, 1, a1);
        coord_max(d.cmax, 2, b0);
        coord_max(d.cmax, 3, b1);
        return;
    }
    d.s64[0 * (size_t)d.n_pad + k] = a0;
    d.s64[1 * (size_t)d.n_pad + k] = a1;
    d.s32[0 * (size_t)d.n_pad + k] = (float)a0;
    d.s32[1 * (size_t)d.n_pad + k] = (float)a1;
    coord_max(d.cmax, 0, a0);
    coord_max(d.cmax, 1, a1);
    for (int c = 0; c < d.b_dim; ++c) {
        const double v = d.b[(size_t)d.b_dim * idx + c];
        d.s64[(2 + c) * (size_t)d.n_pad + k] = v;
        d.s32[(2 + c) * (size_t)d.n_pad + k] = (float)v;
        coord_max(d.cmax, 2 + c, v);
    }
}
// normalize_points (robust/utils.cc:584-644, shared scale) of one problem per CTA, in place on the AoS doubles the caller
// uploaded: optional centroid shift, then division by the mean norm / sqrt(2).  The two reductions run in the order of
// the reference's loops — one thread adds the terms one after the other (centroid: x1[k], x2[k] for k = 0..n-1 in four
// independent chains; scale: |x1[0]|, |x2[0]|, |x1[1]|, ... in one chain) — so the normalised coordinates, and with
// them every inlier decision downstream, are the bits the CPU path produces.  Everything around the two chains (loads,
// the subtraction, the norms, the division) is done by the whole CTA, tile by tile through shared memory.
constexpr int NORM_THREADS = 256, NORM_TILE = 1024;
__global__ void __launch_bounds__(NORM_THREADS) k_normalize(const NormDesc *__restrict__ descs) {
    __shared__ double tile[4][NORM_TILE];
    __shared__ double sh[5];
    const NormDesc d = descs[blockIdx.x];
    const int n = d.n, tid = threadIdx.x;
    double c[4] = {0.0, 0.0, 0.0, 0.0};
    if (d.centroid) {
        for (int t0 = 0; t0 < n; t0 += NORM_TILE) {
            const int m = min_i(NORM_TILE, n - t0);
            for (int i = tid; i < m; i += NORM_THREADS) {
                tile[0][i] = d.a[2 * (size_t)(t0 + i)];
                tile[1][i] = d.a[2 * (size_t)(t0 + i) + 1];
                tile[2][i] = d.b[2 * (size_t)(t0 + i)];
                tile[3][i] = d.b[2 * (size_t)(t0 + i) + 1];
            }
            __syncthreads();
            if (tid == 0)
                for (int i = 0; i < m; ++i) {
                    c[0] += tile[0][i];
                    c[1] += tile[1][i];
                    c[2] += tile[2][i];
                    c[3] += tile[3][i];
                }
            __syncthreads();
        }
        if (tid == 0)
            for (int j = 0; j < 4; ++j) sh[j] = c[j] / (double)n; // centroid /= x.size()
        __syncthreads();
        for (int j = 0; j < 4; ++j) c[j] = sh[j];
    }
    double scale = 0.0;
    for (int t0 = 0; t0 < n; t0 += NORM_TILE) {
        const int m = min_i(NORM_TILE, n - t0);
        for (int i = tid; i < m; i += NORM_THREADS) {
            double x0 = d.a[2 * (size_t)(t0 + i)], x1 = d.a[2 * (size_t)(t0 + i) + 1];
            double y0 = d.b[2 * (size_t)(t0 + i)], y1 = d.b[2 * (size_t)(t0 + i) + 1];
            if (d.centroid) {
                x0 -= c[0]; x1 -= c[1]; y0 -= c[2]; y1 -= c[3];
                d.a[2 * (size_t)(t0 + i)] = x0;
                d.a[2 * (size_t)(t0 + i) + 1] = x1;
                d.b[2 * (size_t)(t0 + i)] = y0;
                d.b[2 * (size_t)(t0 + i) + 1] = y1;
            }
            tile[0][i] = sqrt(x0 * x0 + x1 * x1);
            tile[1][i] = sqrt(y0 * y0 + y1 * y1);
        }
        __syncthreads();
        if (tid == 0)
            for (int i = 0; i < m; ++i) {
                scale += tile[0][i];
                scale += tile[1][i];
            }
        __syncthreads();
    }
    if (tid == 0) {
        scale /= sqrt(2.0) * (double)n; // utils.cc: scale /= std::sqrt(2) * x1.size()
        sh[4] = scale;
        for (int j = 0; j < 4; ++j) d.out[j] = d.centroid ? c[j] : 0.0;
        d.out[4] = scale;
    }
    __syncthreads();
    scale = sh[4];
    for (size_t i = tid; i < 2 * (size_t)n; i += NORM_THREADS) {
        d.a[i] = d.a[i] / scale;
        d.b[i] = d.b[i] / scale;
    }
}
void launch_normalize(const NormDesc *descs_dev, int n_desc, cudaStream_t stream) {
    if (n_desc <= 0) return;
    k_normalize<<<n_desc, NORM_THREADS, 0, stream>>>(descs_dev);
}
void launch_transpose(const TransposeDesc *descs_dev, int n_desc, int max_n_pad, cudaStream_t stream) {
    if (n_desc <= 0) return;
    const int threads = 256;
    dim3 grid((max_n_pad + threads - 1) / threads, n_desc, 1);
    k_transpose<<<grid, threads, 0, stream>>>(descs_dev);
}

// ============================================================================================================
// exact fp64 MSAC scoring of one model by one warp
// ============================================================================================================
template <int KIND> struct ModelCtx;

// reprojection error with z2 <= 0 skip (robust/utils.cc:36-63)
template <> struct ModelCtx<KIND_PNP> {
    double P[12];
    PLB_DEV void init(const double *m) {
        const m3 R = quat_to_rot(m);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            P[4 * r + 0] = R(r, 0); P[4 * r + 1] = R(r, 1); P[4 * r + 2] = R(r, 2); P[4 * r + 3] = m[4 + r];
        }
    }
};
// Sampson error + cheirality on candidates under threshold (robust/utils.cc:158-201)
template <> struct ModelCtx<KIND_RELPOSE> {
    double E[9];
    double q[4], t[3];
    PLB_DEV void init(const double *m) {
#pragma unroll
        for (int i = 0; i < 4; ++i) q[i] = m[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) t[i] = m[4 + i];
        const m3 Em = essential_from_pose(q, t);
#pragma unroll
        for (int i = 0; i < 9; ++i) E[i] = Em.a[i];
    }
};
// tangent Sampson error + cheirality (robust/utils.cc:269-298): same model constants as KIND_RELPOSE
template <> struct ModelCtx<KIND_RELPOSE_TS> : ModelCtx<KIND_RELPOSE> {};
// Sampson error (robust/utils.cc:204-239); model is column-major
template <> struct ModelCtx<KIND_FUND> {
    double E[9];
    PLB_DEV void init(const double *m) {
#pragma unroll
        for (int k = 0; k < 9; ++k) E[3 * (k % 3) + k / 3] = m[k];
    }
};
// one-way transfer error (robust/utils.cc:300-329); model is column-major
template <> struct ModelCtx<KIND_HOMOG> {
    double H[9];
    PLB_DEV void init(const double *m) {
#pragma unroll
        for (int k = 0; k < 9; ++k) H[3 * (k % 3) + k / 3] = m[k];
    }
};

PLB_DEV double sampson_r2(const double *E, double x1_0, double x1_1, double x2_0, double x2_1) {
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
// Epipolar constraint C = d2^T E d1 and its image-space gradient J_C = [M1^T E^T d2 ; M2^T E d1] for unit bearings
// d1,d2 with unprojection Jacobians M1,M2 (3x2 row-major).  Eigen evaluates `M^T * E * d` left to right, i.e. the 2x3
// product first (robust/utils.cc:282-284, optim/relative.h:184-187,210-213); the association is kept.
PLB_DEV void tangent_terms(const double *E, const double *d1, const double *d2, const double *M1, const double *M2,
                           double &C, double *JC) {
    const double Ed0 = E[0] * d1[0] + E[1] * d1[1] + E[2] * d1[2];
    const double Ed1 = E[3] * d1[0] + E[4] * d1[1] + E[5] * d1[2];
    const double Ed2 = E[6] * d1[0] + E[7] * d1[1] + E[8] * d1[2];
    C = d2[0] * Ed0 + d2[1] * Ed1 + d2[2] * Ed2;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        double T1[3], T2[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            T1[j] = M1[i] * E[3 * j] + M1[2 + i] * E[3 * j + 1] + M1[4 + i] * E[3 * j + 2];
            T2[j] = M2[i] * E[j] + M2[2 + i] * E[3 + j] + M2[4 + i] * E[6 + j];
        }
        JC[i] = T1[0] * d2[0] + T1[1] * d2[1] + T1[2] * d2[2];
        JC[2 + i] = T2[0] * d1[0] + T2[1] * d1[1] + T2[2] * d1[2];
    }
}
PLB_DEV double tangent_r2(const double *E, const double *v) { // v: the 18 values of one correspondence
    double C, JC[4];
    tangent_terms(E, v, v + 3, v + 6, v + 12, C, JC);
    const double denom2 = (JC[2] * JC[2] + JC[3] * JC[3]) + (JC[0] * JC[0] + JC[1] * JC[1]);
    return C * C / denom2;
}
PLB_DEV void load_ts(const ProblemDev &P, int k, double *v) {
#pragma unroll
    for (int j = 0; j < TS_ARRAYS; ++j) v[j] = P.ts[(size_t)j * P.n_pad + k];
}
PLB_DEV double homography_r2(const double *H, double x1_0, double x1_1, double x2_0, double x2_1) {
    const double Hx1_0 = H[0] * x1_0 + H[1] * x1_1 + H[2];
    const double Hx1_1 = H[3] * x1_0 + H[4] * x1_1 + H[5];
    const double inv_Hx1_2 = 1.0 / (H[6] * x1_0 + H[7] * x1_1 + H[8]);
    const double r0 = Hx1_0 * inv_Hx1_2 - x2_0;
    const double r1 = Hx1_1 * inv_Hx1_2 - x2_1;
    return r0 * r0 + r1 * r1;
}

// Scores `model` over all correspondences with the first SCORE_THREADS (=256) threads of the CTA; every thread of
// the CTA must call it (it contains CTA barriers) and receives the same (count, score).
// The summation order is fixed — thread-strided partial sums, xor-butterfly inside each warp, the 8 warp partials
// added left to right — so the same model gets the same score bits wherever it is scored (hypothesis scoring,
// LO rescoring, explicit rescoring): the equalities the serial loop relies on (ransac_impl.h:127,143) are preserved.
constexpr int SCORE_THREADS = 256;
constexpr int SCORE_WARPS = SCORE_THREADS / 32;
struct ScoreRed {
    double s[SCORE_WARPS];
    uint32_t c[SCORE_WARPS];
};
template <int KIND, int NT = SCORE_THREADS>
PLB_DEV void cta_score(const ProblemDev &P, const double *model, double sq_thr, ScoreRed *red, uint32_t &count_out,
                       double &score_out) {
    // NT physical threads (256, or 128 in the two-jobs-per-SM LM build) stand for the SCORE_THREADS = 256 threads of the
    // fixed summation order: thread tid accumulates the partial sums of the "virtual" threads tid, tid + NT, ... in
    // separate registers and reduces them as the virtual warps they belong to — same bits for any NT.
    static_assert(SCORE_THREADS % NT == 0 && NT % 32 == 0, "NT must divide the virtual thread count");
    constexpr int VPT = SCORE_THREADS / NT;
    const int tid = threadIdx.x, lane = tid & 31;
    const int n = P.n;
    if (tid < NT) {
        ModelCtx<KIND> C;
        C.init(model);
#pragma unroll
        for (int v = 0; v < VPT; ++v) {
            const int vt = tid + v * NT;
            uint32_t cnt = 0;
            double score = 0.0;
            if (KIND == KIND_PNP) {
                const double *__restrict__ xx = P.p[0], *__restrict__ xy = P.p[1];
                const double *__restrict__ Xx = P.p[2], *__restrict__ Xy = P.p[3], *__restrict__ Xz = P.p[4];
                const double *Pm = reinterpret_cast<const double *>(&C);
                for (int k = vt; k < n; k += SCORE_THREADS) {
                    const double X0 = Xx[k], X1 = Xy[k], X2 = Xz[k];
                    const double x0 = xx[k], x1 = xy[k];
                    const double z0 = Pm[0] * X0 + Pm[1] * X1 + Pm[2] * X2 + Pm[3];
                    const double z1 = Pm[4] * X0 + Pm[5] * X1 + Pm[6] * X2 + Pm[7];
                    const double z2 = Pm[8] * X0 + Pm[9] * X1 + Pm[10] * X2 + Pm[11];
                    if (z2 <= 0.0) continue;
                    const double inv_z2 = 1.0 / z2;
                    const double r_0 = z0 * inv_z2 - x0;
                    const double r_1 = z1 * inv_z2 - x1;
                    const double r_sq = r_0 * r_0 + r_1 * r_1;
                    if (r_sq < sq_thr) {
                        ++cnt;
                        score += r_sq;
                    }
                }
            } else if (KIND == KIND_RELPOSE_TS) {
                const double *M = reinterpret_cast<const double *>(&C);
                for (int k = vt; k < n; k += SCORE_THREADS) {
                    double vv[TS_ARRAYS];
                    load_ts(P, k, vv);
                    const double r2 = tangent_r2(M, vv);
                    bool inl = r2 < sq_thr;
                    if (inl) inl = cheirality_ok(M + 9, M + 13, mk(vv[0], vv[1], vv[2]), mk(vv[3], vv[4], vv[5]), 0.01);
                    if (inl) {
                        ++cnt;
                        score += r2;
                    }
                }
            } else {
                const double *__restrict__ ax = P.p[0], *__restrict__ ay = P.p[1];
                const double *__restrict__ bx = P.p[2], *__restrict__ by = P.p[3];
                const double *M = reinterpret_cast<const double *>(&C); // first 9 doubles: E / F / H row-major
                for (int k = vt; k < n; k += SCORE_THREADS) {
                    const double x1_0 = ax[k], x1_1 = ay[k], x2_0 = bx[k], x2_1 = by[k];
                    double r2;
                    if (KIND == KIND_HOMOG) r2 = homography_r2(M, x1_0, x1_1, x2_0, x2_1);
                    else r2 = sampson_r2(M, x1_0, x1_1, x2_0, x2_1);
                    bool inl = r2 < sq_thr;
                    if (KIND == KIND_RELPOSE) {
                        if (inl) inl = cheirality_ok(M + 9, M + 13, bearing(x1_0, x1_1), bearing(x2_0, x2_1), 0.01);
                    }
                    if (inl) {
                        ++cnt;
                        score += r2;
                    }
                }
            }
            cnt = warp_sum_u(cnt);
            score = warp_sum(score);
            if (lane == 0) {
                red->c[vt >> 5] = cnt;
                red->s[vt >> 5] = score;
            }
        }
    }
    __syncthreads();
    uint32_t ct = 0;
    double st = 0.0;
#pragma unroll
    for (int w = 0; w < SCORE_WARPS; ++w) {
        ct += red->c[w];
        st += red->s[w];
    }
    // Outliers contribute (n - count) * thr in ONE product for every kind (the reference does so for reprojection
    // scores, robust/utils.cc:62, and adds thr per outlier for the others).  Position-independent on purpose: models
    // supported only by their own minimal sample all score (n - K) thr to the last bit, as in the CPU's sequential
    // sum where the K negligible residuals are absorbed — so such ties are not "better scores" (ransac_impl.h:116).
    st += (double)(n - (int)ct) * sq_thr;
    __syncthreads();
    count_out = ct;
    score_out = st;
}

// ============================================================================================================
// fused hypothesis kernel
// ============================================================================================================
constexpr int HYP_WARPS = 8;

template <int KIND> struct HypScratch;
template <> struct HypScratch<KIND_PNP> {
    double models[4 * 7];
};
template <> struct HypScratch<KIND_RELPOSE> {
    Scratch5 s5;
    double xs[30]; // x1s[15], x2s[15]
    double models[40 * 7];
};
template <> struct HypScratch<KIND_FUND> {
    Scratch7 s7;
    double xs[42];
    double models[3 * 9];
};
template <> struct HypScratch<KIND_HOMOG> {
    double models[9];
};

// Gathers the sample and runs the minimal solver; models land in W->models.  Returns the number of models.
template <int KIND>
PLB_DEV int warp_generate_models(const ProblemDev &P, const uint32_t *sample, HypScratch<KIND> *W,
                                 const MonoTables *T, int lane) {
    if (KIND == KIND_PNP) {
        d3 xs[3], Xs[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const uint32_t id = sample[i];
            xs[i] = bearing(P.p[0][id], P.p[1][id]);
            Xs[i] = mk(P.p[2][id], P.p[3][id], P.p[4][id]);
        }
        return solve_p3p(xs, Xs, reinterpret_cast<double *>(W), lane);
    } else if (KIND == KIND_HOMOG) {
        d3 a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t id = sample[i];
            a[i] = bearing(P.p[0][id], P.p[1][id]);
            b[i] = bearing(P.p[2][id], P.p[3][id]);
        }
        return solve_h4(a, b, reinterpret_cast<double *>(W), lane, true);
    } else if (KIND == KIND_RELPOSE) {
        HypScratch<KIND_RELPOSE> *S = reinterpret_cast<HypScratch<KIND_RELPOSE> *>(W);
        if (lane < 10) {
            const int i = lane % 5, side = lane / 5;
            const uint32_t id = sample[i];
            const d3 v = bearing(P.p[2 * side][id], P.p[2 * side + 1][id]);
            double *o = S->xs + 15 * side + 3 * i;
            o[0] = v.x; o[1] = v.y; o[2] = v.z;
        }
        __syncwarp();
        return solve_5pt_poses(S->xs, S->xs + 15, &S->s5, T, S->models, lane);
    } else {
        HypScratch<KIND_FUND> *S = reinterpret_cast<HypScratch<KIND_FUND> *>(W);
        if (lane < 14) {
            const int i = lane % 7, side = lane / 7;
            const uint32_t id = sample[i];
            const d3 v = bearing(P.p[2 * side][id], P.p[2 * side + 1][id]);
            double *o = S->xs + 21 * side + 3 * i;
            o[0] = v.x; o[1] = v.y; o[2] = v.z;
        }
        __syncwarp();
        int nm = solve_7pt(S->xs, S->xs + 21, &S->s7, S->models, lane);
        if (P.rfc) {
            // estimators/relative_pose.cc:393-398: drop models failing the real-focal check, order preserved
            bool keep = false;
            double f[9];
            if (lane < nm) {
#pragma unroll
                for (int k = 0; k < 9; ++k) f[k] = S->models[9 * lane + k];
                keep = rfc_ok(f);
            }
            const unsigned km = __ballot_sync(0xffffffffu, keep);
            __syncwarp();
            if (keep) {
                const int pos = __popc(km & ((1u << lane) - 1u));
#pragma unroll
                for (int k = 0; k < 9; ++k) S->models[9 * pos + k] = f[k];
            }
            __syncwarp();
            nm = __popc(km);
        }
        return nm;
    }
}

PLB_DEV int sample_problem_slot(const RoundDesc &R, int g) {
    int lo = 0, hi = R.n_active - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(R.g_off + mid + 1) <= g) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// Solve kernel: persistent, one warp = one minimal sample of one problem of the group.  Models are appended to a
// compact list (slot range reserved with one atomicAdd per sample); n_models[g] / first_slot[g] let the host walk them
// in (sample, model) order per problem.
template <int KIND>
__global__ void __launch_bounds__(HYP_WARPS * 32, 3) k_solve(const RoundDesc R, int *work_counter, HypOut out) {
    constexpr int K = (KIND == KIND_PNP) ? 3 : (KIND == KIND_RELPOSE) ? 5 : (KIND == KIND_FUND) ? 7 : 4;
    constexpr int MSZ = kind_model_size(KIND);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MonoTables *T = reinterpret_cast<MonoTables *>(smem_raw);
    HypScratch<KIND> *Wall = reinterpret_cast<HypScratch<KIND> *>(smem_raw + 256);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    HypScratch<KIND> *W = Wall + warp;
    if (KIND == KIND_RELPOSE) {
        fill_tables(T);
        __syncthreads();
    }
    for (;;) {
        int g = 0;
        if (lane == 0) g = atomicAdd(work_counter, 1);
        g = __shfl_sync(0xffffffffu, g, 0);
        if (g >= R.n_total) break;
        const int aslot = sample_problem_slot(R, g);
        const int pidx = __ldg(R.active + aslot);
        const ProblemDev &P = R.probs[pidx];
        uint32_t sample[K];
#pragma unroll
        for (int i = 0; i < K; ++i) sample[i] = R.samples[(size_t)g * K + i];
        int nm = warp_generate_models<KIND>(P, sample, W, T, lane);
        int base = 0;
        if (lane == 0) {
            if (nm) {
                const int loc = atomicAdd(out.prob_count + aslot, nm);
                if (loc + nm > __ldg(out.seg_cap + aslot)) { // cannot happen with the worst-case capacity; the engine
                    atomicExch(out.overflow, 1);             // redoes the round with it when the optimistic one fails
                    nm = 0;
                }
                base = __ldg(out.seg_base + aslot) + loc;
            }
            out.n_models[g] = nm;
            out.first_slot[g] = base;
        }
        base = __shfl_sync(0xffffffffu, base, 0);
        nm = __shfl_sync(0xffffffffu, nm, 0);
        const double *models = W->models;
        for (int e = lane; e < nm * MSZ; e += 32) out.models[(size_t)base * MSZ + e] = models[e];
        if (lane < nm) out.model_prob[base + lane] = pidx;
        for (int m = 32 + lane; m < nm; m += 32) out.model_prob[base + m] = pidx;
        __syncwarp();
    }
}

// p3p and homography_4pt are closed forms without any use for a warp (solvers.cuh: in k_solve all 32 lanes evaluate the
// same scalar program): here every THREAD solves its own minimal sample — 32 samples per warp instead of one.  Same
// scalar code, hence the same model bits; the lanes of a warp diverge where their samples take different branches
// (number of real roots, Newton iterations).
template <int KIND>
__global__ void __launch_bounds__(128) k_solve_lane(const RoundDesc R, HypOut out) {
    static_assert(KIND == KIND_PNP || KIND == KIND_HOMOG, "closed-form solvers only");
    constexpr int MSZ = kind_model_size(KIND), MAXM = kind_max_models(KIND);
    const int g_raw = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    const bool live = g_raw < R.n_total;
    const int g = live ? g_raw : R.n_total - 1; // idle lanes redo the last sample, nothing is stored
    const int aslot = sample_problem_slot(R, g);
    const int pidx = __ldg(R.active + aslot);
    const ProblemDev &P = R.probs[pidx];
    double models[MAXM * MSZ];
    int nm;
    if (KIND == KIND_PNP) {
        d3 xs[3], Xs[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const uint32_t id = R.samples[(size_t)g * 3 + i];
            xs[i] = bearing(P.p[0][id], P.p[1][id]);
            Xs[i] = mk(P.p[2][id], P.p[3][id], P.p[4][id]);
        }
        nm = solve_p3p(xs, Xs, models, 0, false);
    } else {
        d3 a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t id = R.samples[(size_t)g * 4 + i];
            a[i] = bearing(P.p[0][id], P.p[1][id]);
            b[i] = bearing(P.p[2][id], P.p[3][id]);
        }
        nm = solve_h4(a, b, models, 0, true, false);
    }
    if (!live) return;
    int base = 0;
    if (nm) {
        const int loc = atomicAdd(out.prob_count + aslot, nm);
        if (loc + nm > __ldg(out.seg_cap + aslot)) { // cannot happen with the worst-case capacity these kinds use
            atomicExch(out.overflow, 1);
            nm = 0;
        }
        base = __ldg(out.seg_base + aslot) + loc;
    }
    out.n_models[g] = nm;
    out.first_slot[g] = base;
    for (int m = 0; m < nm; ++m) {
#pragma unroll
        for (int k = 0; k < MSZ; ++k) out.models[(size_t)(base + m) * MSZ + k] = models[m * MSZ + k];
        out.model_prob[base + m] = pidx;
    }
}

// relpose_7pt with FOUR minimal samples per warp (8 lanes each), like k5_prep: the pivoted-QR nullspace of the 9 x 7
// system is the group-of-8 routine of the 5-point solver (one lane per column), the cubic in the pencil of the two
// nullspace vectors and its roots are scalar (every lane of the group evaluates them, lanes 0..2 build one F each), the
// real-focal check keeps the surviving models in order (estimators/relative_pose.cc:393-398).  Same arithmetic as the
// warp-per-sample solve_7pt (solvers.cuh), a quarter of the warps.
constexpr int P7_M = 0, P7_N = 63, P7_XS = 81, P7_OUT = 123, P7_STRIDE = 152; // 152 = 8 (mod 16): see P5_STRIDE
constexpr size_t K7_SMEM = sizeof(double) * P7_STRIDE * 4 * HYP_WARPS;
__global__ void __launch_bounds__(HYP_WARPS * 32) k7_solve(const RoundDesc R, int *work_counter, HypOut out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, sl = lane & 7, grp = lane >> 3;
    double *W = reinterpret_cast<double *>(smem_raw) + (size_t)((threadIdx.x >> 5) * 4 + grp) * P7_STRIDE;
    const unsigned gmask = 0xffu << (8 * grp);
    for (;;) {
        int g0 = 0;
        if (lane == 0) g0 = atomicAdd(work_counter, 4);
        g0 = __shfl_sync(0xffffffffu, g0, 0);
        if (g0 >= R.n_total) break;
        int g = g0 + grp;
        const bool live = g < R.n_total;
        if (!live) g = R.n_total - 1; // idle groups redo the last sample (uniform control flow), nothing is stored
        const int aslot = sample_problem_slot(R, g);
        const int pidx = __ldg(R.active + aslot);
        const ProblemDev &P = R.probs[pidx];
        double *x1s = W + P7_XS, *x2s = W + P7_XS + 21;
        for (int idx = sl; idx < 14; idx += 8) {
            const int i = idx % 7, side = idx / 7;
            const uint32_t id = R.samples[(size_t)g * 7 + i];
            const d3 v = bearing(P.p[2 * side][id], P.p[2 * side + 1][id]);
            double *o = W + P7_XS + 21 * side + 3 * i;
            o[0] = v.x; o[1] = v.y; o[2] = v.z;
        }
        __syncwarp();
        for (int e = sl; e < 63; e += 8) {
            const int i = e / 9, k = e % 9;
            W[P7_M + e] = x1s[3 * i + k / 3] * x2s[3 * i + k % 3];
        }
        __syncwarp();
        grp8_nullspace_9xC<7>(W + P7_M, W + P7_N, sl);
        const double *n0 = W + P7_N, *n1 = W + P7_N + 9;
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
        bool keep = false;
        double f[9];
        if (sl < n_roots) {
            double r = roots[0];
            if (sl == 1) r = roots[1];
            if (sl == 2) r = roots[2];
            double n2 = 0.0;
#pragma unroll
            for (int k = 0; k < 9; ++k) {
                f[k] = n0[k] * r + n1[k];
                n2 += f[k] * f[k];
            }
            if (n2 > 0) {
                const double nn = sqrt(n2);
#pragma unroll
                for (int k = 0; k < 9; ++k) f[k] /= nn;
            }
            keep = P.rfc ? rfc_ok(f) : true;
        }
        const unsigned km = __ballot_sync(0xffffffffu, keep) & gmask;
        const int nm_all = __popc(km);
        int nm = nm_all, base = 0;
        if (sl == 0 && live) {
            if (nm) {
                const int loc = atomicAdd(out.prob_count + aslot, nm);
                if (loc + nm > __ldg(out.seg_cap + aslot)) { // cannot happen: this kind uses the worst-case capacity
                    atomicExch(out.overflow, 1);
                    nm = 0;
                }
                base = __ldg(out.seg_base + aslot) + loc;
            }
            out.n_models[g] = nm;
            out.first_slot[g] = base;
        }
        base = __shfl_sync(0xffffffffu, base, 8 * grp);
        nm = __shfl_sync(0xffffffffu, nm, 8 * grp);
        if (keep && live && nm) {
            const int pos = base + __popc(km & ((1u << lane) - 1u));
#pragma unroll
            for (int k = 0; k < 9; ++k) out.models[(size_t)pos * 9 + k] = f[k];
            out.model_prob[pos] = pidx;
        }
        __syncwarp();
    }
}

// relpose_7pt with ONE THREAD PER SAMPLE: the scalar nullspace routine of solver5_lane.cuh on a 63-double slice of shared
// memory (odd stride: conflict-free), the rest is the scalar code of k7_solve.  Same arithmetic, same model bits.
constexpr int K7L_THREADS = 256;
constexpr int K7L_STRIDE = 63;
constexpr size_t K7L_SMEM = sizeof(double) * K7L_STRIDE * K7L_THREADS;
__global__ void __launch_bounds__(K7L_THREADS) k7_solve_lane(const RoundDesc R, HypOut out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *W = reinterpret_cast<double *>(smem_raw) + (size_t)threadIdx.x * K7L_STRIDE;
    const int g_raw = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    const bool live = g_raw < R.n_total;
    const int g = live ? g_raw : R.n_total - 1; // idle lanes redo the last sample, nothing is stored
    const int aslot = sample_problem_slot(R, g);
    const int pidx = __ldg(R.active + aslot);
    const ProblemDev &P = R.probs[pidx];
    {
        double x1s[21], x2s[21];
#pragma unroll
        for (int i = 0; i < 7; ++i) {
            const uint32_t id = R.samples[(size_t)g * 7 + i];
            const d3 a = bearing(P.p[0][id], P.p[1][id]), b = bearing(P.p[2][id], P.p[3][id]);
            x1s[3 * i] = a.x; x1s[3 * i + 1] = a.y; x1s[3 * i + 2] = a.z;
            x2s[3 * i] = b.x; x2s[3 * i + 1] = b.y; x2s[3 * i + 2] = b.z;
        }
#pragma unroll
        for (int e = 0; e < 63; ++e) {
            const int i = e / 9, k = e % 9;
            W[e] = x1s[3 * i + k / 3] * x2s[3 * i + k % 3];
        }
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
    if (!live) return;
    double F[3][9];
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
            if (P.rfc ? rfc_ok(f) : true) {
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
    int base = 0;
    if (nm) {
        const int loc = atomicAdd(out.prob_count + aslot, nm);
        if (loc + nm > __ldg(out.seg_cap + aslot)) { // cannot happen: this kind uses the worst-case capacity
            atomicExch(out.overflow, 1);
            nm = 0;
        }
        base = __ldg(out.seg_base + aslot) + loc;
    }
    out.n_models[g] = nm;
    out.first_slot[g] = base;
#pragma unroll
    for (int m = 0; m < 3; ++m)
        if (m < nm) {
#pragma unroll
            for (int k = 0; k < 9; ++k) out.models[(size_t)(base + m) * 9 + k] = F[m][k];
            out.model_prob[base + m] = pidx;
        }
}

// ---- relpose_5pt as three phase kernels -------------------------------------------------------------------------
// The fused warp-per-sample 5-point solver is a large body of code and runs its Sturm root isolation on one lane; 16
// warps per SM at different places of that code starve on instruction fetch.  The
// arithmetic is unchanged, only regrouped so that each kernel's code is small and every phase uses the lanes it can:
//   k5_prep  : warp  = sample   gather, pivoted-QR nullspace, trace constraints, LU, determinant polynomial
//   k5_roots : lane  = sample   Sturm bracketing + Ridders/Newton (scalar, data dependent)
//   k5_back  : lane  = (sample, root)  back-substitution, motion decomposition, cheirality; 3 samples per warp
constexpr int S5_BLK = 105;

constexpr int PREP_SAMPLES_PER_WARP = 4;
constexpr size_t PREP_SMEM = 256 + sizeof(double) * P5_STRIDE * PREP_SAMPLES_PER_WARP * HYP_WARPS;
__global__ void __launch_bounds__(HYP_WARPS * 32) k5_prep(const RoundDesc R, int *work_counter, HypOut out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MonoTables *T = reinterpret_cast<MonoTables *>(smem_raw);
    const int lane = threadIdx.x & 31, sl = lane & 7, grp = lane >> 3;
    double *W = reinterpret_cast<double *>(smem_raw + 256) +
                (size_t)((threadIdx.x >> 5) * PREP_SAMPLES_PER_WARP + grp) * P5_STRIDE;
    fill_tables(T);
    __syncthreads();
    for (;;) {
        int g0 = 0;
        if (lane == 0) g0 = atomicAdd(work_counter, PREP_SAMPLES_PER_WARP);
        g0 = __shfl_sync(0xffffffffu, g0, 0);
        if (g0 >= R.n_total) break;
        int g = g0 + grp;
        const bool live = g < R.n_total;
        if (!live) g = R.n_total - 1; // idle groups redo the last sample (uniform control flow), nothing is stored
        const ProblemDev &P = R.probs[__ldg(R.active + sample_problem_slot(R, g))];
        // bearings of the 5 sampled correspondences (estimators/relative_pose.cc:51-54,90-94)
        for (int idx = sl; idx < 10; idx += 8) {
            const int i = idx % 5, side = idx / 5;
            const uint32_t id = R.samples[(size_t)g * 5 + i];
            d3 v;
            if (P.kind == KIND_RELPOSE_TS) {
                const double *t = P.ts + (size_t)(3 * side) * P.n_pad + id;
                v = mk(t[0], t[P.n_pad], t[2 * (size_t)P.n_pad]);
            } else {
                v = bearing(P.p[2 * side][id], P.p[2 * side + 1][id]);
            }
            double *o = W + P5_XS + 15 * side + 3 * i;
            o[0] = v.x; o[1] = v.y; o[2] = v.z;
        }
        __syncwarp();
        solve_5pt_poly_grp8(W, T, sl);
        if (live) {
            double *blk = out.s5_blk + g; // entry-major: blk[e * n_total]
            const size_t nt = (size_t)R.n_total;
            for (int e = sl; e < 39; e += 8) blk[e * nt] = W[P5_A + e];
            for (int e = sl; e < 36; e += 8) blk[(39 + e) * nt] = W[P5_NB + e];
            for (int e = sl; e < 30; e += 8) blk[(75 + e) * nt] = W[P5_XS + e];
            for (int k = sl; k < 11; k += 8) out.s5_cpoly[(size_t)k * R.n_total + g] = W[P5_CPOLY + k];
        }
        __syncwarp();
    }
}

// Bearings of the 5 sampled correspondences of every sample (estimators/relative_pose.cc:51-54,90-94) into the
// entry-major per-sample block (entries 75..104).  Its chain of dependent global loads (problem slot -> problem ->
// sample ids -> points) is a kernel of its own, at full occupancy: inside k5_prep_lane (4 warps per SM) it was 19 % of
// that kernel's time.
__global__ void __launch_bounds__(256) k5_gather(const RoundDesc R, HypOut out) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= R.n_total) return;
    const ProblemDev &P = R.probs[__ldg(R.active + sample_problem_slot(R, g))];
    const size_t nt = (size_t)R.n_total;
    double *blk = out.s5_blk + g;
    uint32_t id[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) id[i] = R.samples[(size_t)g * 5 + i];
#pragma unroll
    for (int i = 0; i < 5; ++i) {
#pragma unroll
        for (int side = 0; side < 2; ++side) {
            d3 v;
            if (P.kind == KIND_RELPOSE_TS) {
                const double *t = P.ts + (size_t)(3 * side) * P.n_pad + id[i];
                v = mk(t[0], t[P.n_pad], t[2 * (size_t)P.n_pad]);
            } else {
                v = bearing(P.p[2 * side][id[i]], P.p[2 * side + 1][id[i]]);
            }
            blk[(75 + 15 * side + 3 * i) * nt] = v.x;
            blk[(75 + 15 * side + 3 * i + 1) * nt] = v.y;
            blk[(75 + 15 * side + 3 * i + 2) * nt] = v.z;
        }
    }
}

// The same phase with ONE THREAD PER SAMPLE (solver5_lane.cuh): the nullspace basis and the quadratic blocks live in
// registers (compile-time monomial tables); shared memory holds only the LEFT 10 x 10 block of the elimination matrix
// (dynamic pivot rows) plus 10 doubles of scratch per thread, the right-hand sides are parked in global memory (L2)
// while the block is factored and come back column by column.  111 doubles per thread (odd: the 32 lanes of a warp
// spread over all bank pairs) x 256 threads = 222 KB: one CTA, 8 warps per SM.
constexpr int PREPL_THREADS = 256;
constexpr int PREPL_STRIDE = 111;
constexpr size_t PREPL_SMEM = sizeof(double) * PREPL_STRIDE * PREPL_THREADS;
template <int UNR>
__global__ void __launch_bounds__(PREPL_THREADS, 1) k5_prep_lane(const RoundDesc R, HypOut out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *W = reinterpret_cast<double *>(smem_raw) + (size_t)threadIdx.x * PREPL_STRIDE;
    double *CL = W, *S = W + 100;
    int g = blockIdx.x * PREPL_THREADS + threadIdx.x;
    const bool live = g < R.n_total;
    if (!live) g = R.n_total - 1; // idle threads of the last CTA redo the last sample (same values, harmless stores)
    const size_t nt = (size_t)R.n_total;
    double *blk = out.s5_blk + g;   // entry-major: blk[e * n_total]
    double *park = out.s5_park + g; // right-hand sides, entry-major: park[(row * 10 + column) * n_total]
    {
        double xs[30]; // the sample's bearings, written by k5_gather: 30 independent coalesced loads
#pragma unroll
        for (int e = 0; e < 30; ++e) xs[e] = blk[(75 + e) * nt];
        // 9 x 5 epipolar constraints (relpose_5pt.cc:163-166): entry 3a+b of column i = x1[i][a] * x2[i][b]
#pragma unroll
        for (int e = 0; e < 45; ++e) {
            const int i = e / 9, k = e % 9;
            W[e] = xs[3 * i + k / 3] * xs[15 + 3 * i + k % 3];
        }
    }
    lane5::nullspace_9x5(W, W + 45);
    {
        double Nb[36];
#pragma unroll
        for (int e = 0; e < 36; ++e) {
            const int r = e / 9, k = e % 9;
            Nb[4 * k + r] = W[45 + 9 * r + k];
        }
#pragma unroll
        for (int e = 0; e < 36; ++e) blk[(39 + e) * nt] = Nb[e];
        lane5::build_coeffs(Nb, [&](int row, auto cc, double v) {
            constexpr int ci = decltype(cc)::value;
            if constexpr (ci < 10) CL[row * 10 + ci] = v;
            else park[(size_t)(row * 10 + (ci - 10)) * nt] = v;
        });
    }
    int idx[10];
    lane5::lu_left(CL, S, idx);
    lane5::solve_rhs<UNR>(CL, S, idx, [&](int r, int c) { return park[(size_t)(r * 10 + c) * nt]; }, CL);
    double A[39], cp[11];
    lane5::poly_matrix(CL, A);
#pragma unroll
    for (int e = 0; e < 39; ++e) blk[e * nt] = A[e];
    lane5::det_poly(A, cp);
#pragma unroll
    for (int k = 0; k < 11; ++k) out.s5_cpoly[(size_t)k * nt + g] = cp[k];
}

constexpr int ROOTS_THREADS = 64;
__global__ void __launch_bounds__(ROOTS_THREADS) k5_roots(int n_total, HypOut out) {
    __shared__ RootsShared S[ROOTS_THREADS / 32];
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    const bool has = g < n_total;
    double c[11], roots[10];
#pragma unroll
    for (int k = 0; k < 11; ++k) c[k] = has ? out.s5_cpoly[(size_t)k * n_total + g] : 0.0;
    const int n = sturm_bisect10_warp(c, has, roots, &S[threadIdx.x >> 5], threadIdx.x & 31);
    if (has) {
        out.s5_nroots[g] = n;
        double *o = out.s5_roots + (size_t)g * 10;
        for (int k = 0; k < n; ++k) o[k] = roots[k];
    }
}

// A warp owns 32 consecutive samples.  Their real roots (0..10 each, ~2.6 on average) are dealt out to the lanes in
// passes of up to 32 roots made of WHOLE samples, so that the per-sample model count / segment reservation stays a
// warp-local segmented sum; a fixed lane = (sample, root slot) mapping keeps only ~8 of 32 lanes busy.
__global__ void __launch_bounds__(128) k5_back(const RoundDesc R, HypOut out) {
    __shared__ int s_incl[4][33];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int g0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32;
    if (g0 >= R.n_total) return; // whole warp
    int *P = s_incl[w];
    {
        const int gs = g0 + lane;
        const bool has = gs < R.n_total;
        const int nr = has ? out.s5_nroots[gs] : 0;
        if (has && nr == 0) { // no essential matrix, no model
            out.n_models[gs] = 0;
            out.first_slot[gs] = 0;
        }
        int incl = nr;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        P[lane + 1] = incl;
        if (lane == 0) P[0] = 0;
    }
    __syncwarp();
    const int T = P[32];
    const int my_incl = P[lane + 1];
    int b0 = 0;
    while (b0 < 32) {
        const int base_roots = P[b0];
        if (base_roots == T) break;
        // samples [b0, e) = the longest run whose roots fit into the 32 lanes (a sample has <= 10 roots, so e > b0)
        const unsigned fm = __ballot_sync(0xffffffffu, lane >= b0 && (my_incl - base_roots) <= 32);
        const int e = b0 + __popc(fm);
        const int cnt = P[e] - base_roots;
        const bool valid = lane < cnt;
        int s = b0, r = 0, nrs = 0;
        if (valid) {
            const int t = base_roots + lane;
            int lo = b0, hi = e - 1; // largest s with P[s] <= t
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (P[mid] <= t) lo = mid;
                else hi = mid - 1;
            }
            s = lo;
            r = t - P[s];
            nrs = P[s + 1] - P[s];
        }
        const int g = g0 + s;
        double cand[4][7];
        unsigned mask = 0;
        if (valid) {
            const StridedD blk{out.s5_blk + g, (size_t)R.n_total}; // entry-major (k5_prep_lane)
            double E[9];
            backsub_5pt(blk, blk + 39, out.s5_roots[(size_t)g * 10 + r], E);
            mask = motions_from_E(E, blk + 75, blk + 90, 5, cand);
        }
        const int mine = __popc(mask);
        // exclusive prefix / total inside the sample's lane segment (root-major, candidate-minor order of the reference)
        const int start = lane - r;
        int pre = 0, total = 0;
#pragma unroll
        for (int j = 0; j < 10; ++j) {
            const int v = __shfl_sync(0xffffffffu, mine, (start + j) & 31);
            if (j < nrs) {
                if (j < r) pre += v;
                total += v;
            }
        }
        int base = 0, pidx = 0;
        if (valid && r == 0) {
            const int aslot = sample_problem_slot(R, g);
            pidx = __ldg(R.active + aslot);
            if (total) {
                const int loc = atomicAdd(out.prob_count + aslot, total);
                if (loc + total > __ldg(out.seg_cap + aslot)) {
                    atomicExch(out.overflow, 1);
                    total = 0;
                }
                base = __ldg(out.seg_base + aslot) + loc;
            }
            out.n_models[g] = total;
            out.first_slot[g] = base;
        }
        base = __shfl_sync(0xffffffffu, base, start & 31);
        total = __shfl_sync(0xffffffffu, total, start & 31);
        pidx = __shfl_sync(0xffffffffu, pidx, start & 31);
        if (valid && total) {
            int pos = base + pre;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                if (mask & (1u << c)) {
                    double *o = out.models + (size_t)pos * 7;
#pragma unroll
                    for (int k = 0; k < 7; ++k) o[k] = cand[c][k];
                    out.model_prob[pos] = pidx;
                    ++pos;
                }
            }
        }
        b0 = e;
    }
}

// Score kernel: persistent grid of 256-thread CTAs, one CTA scores one model at a time over all correspondences of
// the model's problem.
template <int KIND>
__global__ void __launch_bounds__(SCORE_THREADS, 4)
    k_score(const ProblemDev *__restrict__ probs, const double *__restrict__ models, const int *__restrict__ model_prob,
            const int *__restrict__ model_count, int cap, uint32_t *counts, double *scores) {
    constexpr int MSZ = kind_model_size(KIND);
    __shared__ ScoreRed red;
    int nmod = *model_count;
    if (nmod > cap) nmod = cap;
    for (int m = blockIdx.x; m < nmod; m += gridDim.x) {
        const ProblemDev P = probs[model_prob[m]];
        double mdl[MSZ];
#pragma unroll
        for (int k = 0; k < MSZ; ++k) mdl[k] = models[(size_t)m * MSZ + k];
        uint32_t cnt;
        double score;
        cta_score<KIND>(P, mdl, P.sq_thr, &red, cnt, score);
        if (threadIdx.x == 0) {
            counts[m] = cnt;
            scores[m] = score;
        }
    }
}

// Tiled score kernel of the round path: CTA (x, a) scores tiles of SCORE_TM models of active problem a.  Every thread
// loads a correspondence ONCE and evaluates all models of the tile against it (model constants are broadcast reads from
// shared memory), which divides the L2 -> SM traffic of the one-CTA-per-model kernel by the tile size; the per-model
// summation order is exactly that of cta_score, so both kernels produce the same bits for the same model.
constexpr int SCORE_TM = 4;
// the tangent-Sampson kind carries 18 values per correspondence: two models per tile keep it inside 128 registers
template <int KIND> constexpr __host__ __device__ int score_tm() { return KIND == KIND_RELPOSE_TS ? 2 : SCORE_TM; }
template <int KIND>
__global__ void __launch_bounds__(SCORE_THREADS, 2)
    k_score_tiled(const RoundDesc R, HypOut out) {
    constexpr int MSZ = kind_model_size(KIND);
    constexpr int CTX = (KIND == KIND_PNP) ? 12 : kind_is_relpose(KIND) ? 16 : 9;
    constexpr int TM = score_tm<KIND>();
    __shared__ double ctx[TM][16];
    __shared__ double red_s[SCORE_WARPS][TM];
    __shared__ uint32_t red_c[SCORE_WARPS][TM];
    const int a = blockIdx.y;
    const int count = out.prob_count[a];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (blockIdx.x * TM >= count) return;
    const ProblemDev P = R.probs[R.active[a]];
    const int n = P.n;
    const double sq_thr = P.sq_thr;
    const int seg = out.seg_base[a];
    for (int m0 = blockIdx.x * TM; m0 < count; m0 += gridDim.x * TM) {
        const int tm = (count - m0 < TM) ? (count - m0) : TM;
        __syncthreads();
        if (tid < tm) {
            double mdl[MSZ];
#pragma unroll
            for (int k = 0; k < MSZ; ++k) mdl[k] = out.models[(size_t)(seg + m0 + tid) * MSZ + k];
            ModelCtx<KIND> C;
            C.init(mdl);
            const double *cp = reinterpret_cast<const double *>(&C);
#pragma unroll
            for (int k = 0; k < CTX; ++k) ctx[tid][k] = cp[k];
        }
        __syncthreads();
        uint32_t cnt[TM];
        double sc[TM];
#pragma unroll
        for (int i = 0; i < TM; ++i) {
            cnt[i] = 0;
            sc[i] = 0.0;
        }
        if (KIND == KIND_PNP) {
            const double *__restrict__ xx = P.p[0], *__restrict__ xy = P.p[1];
            const double *__restrict__ Xx = P.p[2], *__restrict__ Xy = P.p[3], *__restrict__ Xz = P.p[4];
            for (int k = tid; k < n; k += SCORE_THREADS) {
                const double X0 = Xx[k], X1 = Xy[k], X2 = Xz[k];
                const double x0 = xx[k], x1 = xy[k];
#pragma unroll
                for (int i = 0; i < TM; ++i) {
                    if (i < tm) {
                        const double *Pm = ctx[i];
                        const double z0 = Pm[0] * X0 + Pm[1] * X1 + Pm[2] * X2 + Pm[3];
                        const double z1 = Pm[4] * X0 + Pm[5] * X1 + Pm[6] * X2 + Pm[7];
                        const double z2 = Pm[8] * X0 + Pm[9] * X1 + Pm[10] * X2 + Pm[11];
                        if (z2 > 0.0) {
                            const double inv_z2 = 1.0 / z2;
                            const double r_0 = z0 * inv_z2 - x0;
                            const double r_1 = z1 * inv_z2 - x1;
                            const double r_sq = r_0 * r_0 + r_1 * r_1;
                            if (r_sq < sq_thr) {
                                ++cnt[i];
                                sc[i] += r_sq;
                            }
                        }
                    }
                }
            }
        } else if (KIND == KIND_RELPOSE_TS) {
            for (int k = tid; k < n; k += SCORE_THREADS) {
                double v[TS_ARRAYS];
                load_ts(P, k, v);
#pragma unroll
                for (int i = 0; i < TM; ++i) {
                    if (i < tm) {
                        const double r2 = tangent_r2(ctx[i], v);
                        bool inl = r2 < sq_thr;
                        if (inl)
                            inl = cheirality_ok(ctx[i] + 9, ctx[i] + 13, mk(v[0], v[1], v[2]), mk(v[3], v[4], v[5]), 0.01);
                        if (inl) {
                            ++cnt[i];
                            sc[i] += r2;
                        }
                    }
                }
            }
        } else {
            const double *__restrict__ ax = P.p[0], *__restrict__ ay = P.p[1];
            const double *__restrict__ bx = P.p[2], *__restrict__ by = P.p[3];
            for (int k = tid; k < n; k += SCORE_THREADS) {
                const double x1_0 = ax[k], x1_1 = ay[k], x2_0 = bx[k], x2_1 = by[k];
                double r2v[TM];
                unsigned under = 0; // models whose residual is under the threshold at this correspondence
#pragma unroll
                for (int i = 0; i < TM; ++i) {
                    if (i < tm) {
                        const double *M = ctx[i];
                        if (KIND == KIND_HOMOG) r2v[i] = homography_r2(M, x1_0, x1_1, x2_0, x2_1);
                        else r2v[i] = sampson_r2(M, x1_0, x1_1, x2_0, x2_1);
                        if (r2v[i] < sq_thr) under |= 1u << i;
                    }
                }
                if (KIND == KIND_RELPOSE && under) {
                    // cheirality only for candidates under the threshold (robust/utils.cc:187-197); the normalised
                    // bearings depend on the correspondence alone and are computed once
                    const d3 b1 = bearing(x1_0, x1_1), b2 = bearing(x2_0, x2_1);
#pragma unroll 1
                    for (int i = 0; i < TM; ++i)
                        if ((under >> i) & 1u)
                            if (!cheirality_ok(ctx[i] + 9, ctx[i] + 13, b1, b2, 0.01)) under &= ~(1u << i);
                }
#pragma unroll
                for (int i = 0; i < TM; ++i) {
                    if (i < tm) {
                        if ((under >> i) & 1u) {
                            ++cnt[i];
                            sc[i] += r2v[i];
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int i = 0; i < TM; ++i) {
            const uint32_t c = warp_sum_u(cnt[i]);
            const double v = warp_sum(sc[i]);
            if (lane == 0) {
                red_c[warp][i] = c;
                red_s[warp][i] = v;
            }
        }
        __syncthreads();
        if (tid < tm) {
            uint32_t ct = 0;
            double st = 0.0;
#pragma unroll
            for (int w = 0; w < SCORE_WARPS; ++w) {
                ct += red_c[w][tid];
                st += red_s[w][tid];
            }
            st += (double)(n - (int)ct) * sq_thr; // see cta_score
            out.counts[seg + m0 + tid] = ct;
            out.scores[seg + m0 + tid] = st;
        }
    }
}

// ============================================================================================================
// fp32 screening pass (fast mode)
// ============================================================================================================
// Scores EVERY model of the round in fp32 from the fp32 SoA copy of the correspondences (16 B / 2D-2D corr, 20 B /
// 2D-3D corr).  The CTA stages its problem's arrays into shared memory with TMA bulk copies (cp.async.bulk, one
// mbarrier) and then walks that problem's model tiles; every thread evaluates SCR_TM models per correspondence read
// from shared memory.  The records (count32, score32) only decide which models COULD change the RANSAC state; those
// candidates are rescored in fp64 (k_score_list) before the serial replay, so results are those of the exact mode.
constexpr int SCR_THREADS = 512;
constexpr int SCR_WARPS = SCR_THREADS / 32;
constexpr int SCR_TM = 8;
constexpr int SCR_RQ_TAKE = 8; // cases a lane may queue per pass of the warp-compacted handling

PLB_DEV uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
PLB_DEV void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
PLB_DEV void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
PLB_DEV void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
PLB_DEV void mbar_wait(uint64_t *bar, uint32_t phase) {
    asm volatile("{\n"
                 ".reg .pred P1;\n"
                 "LAB_WAIT:\n"
                 "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
                 "@P1 bra DONE;\n"
                 "bra LAB_WAIT;\n"
                 "DONE:\n"
                 "}" ::"r"(smem_u32(bar)),
                 "r"(phase)
                 : "memory");
}

// Model constants are re-read from shared memory for every (model, step) on purpose: left to itself the compiler hoists
// the loop-invariant loads of all SCR_TM models out of the streaming loop and spills them.
PLB_DEV void lds_v4(const float *p, float *o) {
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(o[0]), "=f"(o[1]), "=f"(o[2]), "=f"(o[3]) : "r"(smem_u32(p)));
}
PLB_DEV float2 lds_f2(const float2 *p) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(smem_u32(p)));
    return v;
}
PLB_DEV float warp_sum_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// NTHR: threads per CTA.  512 (one CTA per SM next to a 160 KB staging buffer) for the large problems the kernel was
// shaped for; 128 (four CTAs per SM) for small ones (BASELINE config 1: 200 correspondences), where a 512-thread CTA
// leaves most threads without a correspondence and the per-tile setup / reduction is what costs.
template <int KIND, int NTHR>
__global__ void __launch_bounds__(NTHR, NTHR >= 512 ? 1 : 4) k_screen(const RoundDesc R, HypOut out, int use_smem) {
    constexpr int SCR_THREADS = NTHR, SCR_WARPS = NTHR / 32; // shadow the file-scope defaults
    constexpr int MSZ = kind_model_size(KIND);
    constexpr int CTX = (KIND == KIND_PNP) ? 12 : kind_is_relpose(KIND) ? 16 : 9;
    constexpr int NARR = (KIND == KIND_PNP) ? 5 : 4;
    extern __shared__ __align__(128) unsigned char scr_smem[];
    __shared__ __align__(8) uint64_t bar;
    __shared__ __align__(16) float ctx[SCR_TM][scr::CTX_FLOATS];
    __shared__ float red_s[SCR_WARPS][SCR_TM];
    __shared__ float red_e[SCR_WARPS][SCR_TM];
    __shared__ uint32_t red_c[SCR_WARPS][SCR_TM];
    __shared__ uint32_t s_border[SCR_TM];
    __shared__ uint16_t rq[SCR_WARPS][32 * SCR_RQ_TAKE]; // per-warp queue of recorded cases: lane << 8 | bit << 3 | model
    // ---- static, cost-balanced partition of the round's (problem, tile) list over the CTAs of the grid ------------
    // cost of a tile = correspondences of its problem; CTA c owns the tiles whose start cost lies in
    // [W c / G, W (c+1) / G).  The grid is ONE wave (resident CTAs x SMs), so there is no tail wave; a CTA touches a
    // contiguous range of problems (usually one or two) and re-stages the shared-memory arrays when it moves on.
    __shared__ long long s_warp[SCR_WARPS];
    __shared__ long long s_pre[SCR_THREADS];
    __shared__ int s_first, s_last;
    __shared__ long long s_first_pre, s_total, s_clo, s_chi, s_Sa;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int na = R.n_active;
    auto tiles_of = [&](int a) -> int { return (out.prob_count[a] + SCR_TM - 1) / SCR_TM; };
    auto n_of = [&](int a) -> int { return R.probs[R.active[a]].n; };
    const int per = (na + SCR_THREADS - 1) / SCR_THREADS;
    const int own_lo = min_i(tid * per, na), own_hi = min_i(own_lo + per, na);
    {
        long long loc = 0;
        for (int a = own_lo; a < own_hi; ++a) loc += (long long)tiles_of(a) * n_of(a);
        long long inc = loc;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (lane == 31) s_warp[warp] = inc;
        if (tid == 0) {
            s_first = 0x7fffffff;
            s_last = -1;
        }
        __syncthreads();
        long long base = 0;
        for (int w = 0; w < warp; ++w) base += s_warp[w];
        s_pre[tid] = base + inc - loc;
        if (tid == SCR_THREADS - 1) s_total = base + inc;
        __syncthreads();
    }
    const long long total_cost = s_total;
    if (total_cost == 0) return;
    if (tid == 0) { // kept in shared memory: long-lived 64-bit values would otherwise spill around the hot loop
        s_clo = total_cost * (long long)blockIdx.x / (long long)gridDim.x;
        s_chi = total_cost * (long long)(blockIdx.x + 1) / (long long)gridDim.x;
    }
    __syncthreads();
    auto tile_range = [&](long long S, int tiles, int nn, int &t0, int &t1) {
        // tiles t with c_lo <= S + t*nn < c_hi
        const long long c_lo = s_clo, c_hi = s_chi;
        long long a0 = (c_lo > S) ? (c_lo - S + nn - 1) / nn : 0;
        long long a1 = (c_hi > S) ? (c_hi - S + nn - 1) / nn : 0;
        if (a1 > tiles) a1 = tiles;
        t0 = (int)a0;
        t1 = (int)a1;
    };
    {
        long long S = s_pre[tid];
        for (int a = own_lo; a < own_hi; ++a) {
            const int tl = tiles_of(a), nn = n_of(a);
            if (tl > 0 && nn > 0) {
                int t0, t1;
                tile_range(S, tl, nn, t0, t1);
                if (t0 < t1) {
                    atomicMin(&s_first, a);
                    atomicMax(&s_last, a);
                }
            }
            S += (long long)tl * nn;
        }
        __syncthreads();
        if (tid == 0 && s_last >= 0) {
            const int owner = s_first / per;
            long long Sf = s_pre[owner];
            for (int a = owner * per; a < s_first; ++a) Sf += (long long)tiles_of(a) * n_of(a);
            s_first_pre = Sf;
        }
        __syncthreads();
    }
    if (s_last < 0) return;
    if (tid == 0) {
        s_Sa = s_first_pre;
        if (use_smem) mbar_init(&bar, 1);
    }
    __syncthreads();
    uint32_t phase = 0;
    for (int a = s_first; a <= s_last; ++a) {
    const int count = out.prob_count[a];
    const ProblemDev P = R.probs[R.active[a]];
    const int n = P.n, n_pad = (n + 31) & ~31;
    int t_begin = 0, t_end = 0;
    {
        const int tl = (count + SCR_TM - 1) / SCR_TM;
        const long long S_a = s_Sa;
        if (tl > 0 && n > 0) tile_range(S_a, tl, n, t_begin, t_end);
        __syncthreads();
        if (tid == 0) s_Sa = S_a + (long long)tl * n;
        __syncthreads();
    }
    if (t_begin >= t_end) continue;
    const float thr = (float)P.sq_thr;
    const int seg = out.seg_base[a];
    const float *arr[NARR];
    if (use_smem) {
        float *pts = reinterpret_cast<float *>(scr_smem);
        __syncthreads(); // every thread is done with the previous problem's arrays
        if (tid == 0) {
            const uint32_t bytes = (uint32_t)n_pad * 4u;
            mbar_expect_tx(&bar, bytes * NARR);
#pragma unroll
            for (int c = 0; c < NARR; ++c) tma_bulk_g2s(pts + (size_t)c * n_pad, P.f[c], bytes, &bar);
        }
        mbar_wait(&bar, phase);
        phase ^= 1u;
#pragma unroll
        for (int c = 0; c < NARR; ++c) arr[c] = pts + (size_t)c * n_pad;
    } else {
#pragma unroll
        for (int c = 0; c < NARR; ++c) arr[c] = P.f[c];
    }
    for (int m0 = t_begin * SCR_TM; m0 < t_end * SCR_TM; m0 += SCR_TM) {
        const int tm = (count - m0 < SCR_TM) ? (count - m0) : SCR_TM;
        __syncthreads();
        if (tid < SCR_TM) s_border[tid] = 0u;
        if (tid < tm) {
            double mdl[MSZ];
#pragma unroll
            for (int k = 0; k < MSZ; ++k) mdl[k] = out.models[(size_t)(seg + m0 + tid) * MSZ + k];
            ModelCtx<KIND> C;
            C.init(mdl);
            const double *cp = reinterpret_cast<const double *>(&C);
#pragma unroll
            for (int k = 0; k < CTX; ++k) ctx[tid][k] = (float)cp[k];
            // per-model constants of the error bounds (screen_math.cuh), from the fp64 model and the problem's maxima
            float cm[5];
#pragma unroll
            for (int c = 0; c < NARR; ++c) cm[c] = P.cmax[c];
            if (KIND == KIND_PNP) scr::transfer_setup<3>(cp, cm + 2, cm, P.sq_thr, ctx[tid]);
            else if (KIND == KIND_HOMOG) scr::transfer_setup<2>(cp, cm, cm + 2, P.sq_thr, ctx[tid]);
            else scr::sampson_setup(cp, cm, P.sq_thr, ctx[tid]);
            if (KIND == KIND_RELPOSE) scr::cheirality_setup(cp + 9, cp + 13, ctx[tid]);
        }
        __syncthreads();
        uint32_t cnt[SCR_TM];
        float sc[SCR_TM], er[SCR_TM];
#pragma unroll
        for (int i = 0; i < SCR_TM; ++i) {
            cnt[i] = 0;
            sc[i] = 0.f;
            er[i] = 0.f;
        }
        {
            // sc[i] accumulates sum over inliers of (r2 - thr); n*thr is added at the end.
            // The streaming pass is branch-free: the residual terms, one test "could this correspondence be an inlier
            // of model i in fp64" (the plain fp32 test widened by the rigorous error bound, screen_math.cuh) and a
            // predicated OR that records the correspondence in a per-lane bit mask.  SCR_PB correspondences per thread
            // per step reuse the model constants fetched (broadcast) from shared memory.  The recorded cases (plain
            // decision, is it provably the fp64 decision, cheirality, division, accumulation of score and error bound)
            // are handled afterwards in a compacted loop in which every lane pops one of ITS recorded cases per
            // iteration — handled inline they cost a divergent detour for the whole warp whenever one lane of 32 hits.
            constexpr int SCR_PB = 4;
            auto maybe = [&](const float *M, const float *p) -> bool {
                if (KIND == KIND_PNP) return scr::transfer_maybe<true>(M, scr::pnp_terms(M, p[0], p[1], p[2], p[3], p[4]));
                if (KIND == KIND_HOMOG) return scr::transfer_maybe<false>(M, scr::homography_terms(M, p[0], p[1], p[2], p[3]));
                return scr::sampson_maybe(M, p[0], p[1], p[2], p[3]);
            };
            for (int base = 0; base < n; base += 32 * SCR_THREADS) {
                const int lim = min_i(n, base + 32 * SCR_THREADS);
                uint32_t hit[SCR_TM];
#pragma unroll
                for (int i = 0; i < SCR_TM; ++i) hit[i] = 0u;
                int k0 = base + tid;
                uint32_t qbit = 1u;
                for (; k0 + (SCR_PB - 1) * SCR_THREADS < lim; k0 += SCR_THREADS * SCR_PB, qbit <<= SCR_PB) {
                    float p[SCR_PB][NARR];
#pragma unroll
                    for (int j = 0; j < SCR_PB; ++j) {
                        const int k = k0 + j * SCR_THREADS;
#pragma unroll
                        for (int c = 0; c < NARR; ++c) p[j][c] = arr[c][k];
                    }
#pragma unroll
                    for (int i = 0; i < SCR_TM; ++i) {
                        if (i < tm) {
                            float Mr[20]; // [0..11] model, [16..19] constants of the streaming test
                            lds_v4(ctx[i], Mr);
                            lds_v4(ctx[i] + 4, Mr + 4);
                            lds_v4(ctx[i] + 8, Mr + 8);
                            lds_v4(ctx[i] + 16, Mr + 16);
#pragma unroll
                            for (int j = 0; j < SCR_PB; ++j)
                                if (maybe(Mr, p[j])) hit[i] |= qbit << j;
                        }
                    }
                }
                for (; k0 < lim; k0 += SCR_THREADS, qbit <<= 1) { // remainder
                    float p[NARR];
#pragma unroll
                    for (int c = 0; c < NARR; ++c) p[c] = arr[c][k0];
#pragma unroll
                    for (int i = 0; i < SCR_TM; ++i) {
                        if (i < tm) {
                            if (maybe(ctx[i], p)) hit[i] |= qbit;
                        }
                    }
                }
                // Handling of the recorded cases, compacted across the WARP: the lanes list their cases (model, bit, lane)
                // in a per-warp queue in shared memory — at most SCR_RQ_TAKE per lane and pass, so the queue cannot
                // overflow — and the warp then works through the queue 32 entries at a time.  A case is evaluated by
                // whichever lane picks it up and lands in THAT lane's accumulators of the model (the per-model sums over
                // lanes come later anyway).  Handling them lane-locally left most lanes idle: a model has a few dozen
                // inliers among 10 000 correspondences, 1-5 lanes of a warp had work per iteration.
                for (;;) {
                    int mine = 0;
#pragma unroll
                    for (int i = 0; i < SCR_TM; ++i) mine += __popc(hit[i]);
                    if (!__any_sync(0xffffffffu, mine > 0)) break;
                    const int take = mine < SCR_RQ_TAKE ? mine : SCR_RQ_TAKE;
                    int incl = take;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const int t = __shfl_up_sync(0xffffffffu, incl, o);
                        if (lane >= o) incl += t;
                    }
                    const int total = __shfl_sync(0xffffffffu, incl, 31);
                    int wpos = incl - take;
                    for (int t = 0; t < take; ++t) {
                        int mi = 0;
                        uint32_t hm = 0u;
#pragma unroll
                        for (int i = SCR_TM - 1; i >= 0; --i)
                            if (hit[i] != 0u) {
                                mi = i;
                                hm = hit[i];
                            }
                        const int q = __ffs((int)hm) - 1;
                        const uint32_t cleared = hm & (hm - 1u);
#pragma unroll
                        for (int i = 0; i < SCR_TM; ++i)
                            if (i == mi) hit[i] = cleared;
                        rq[warp][wpos++] = (uint16_t)((lane << 8) | (q << 3) | mi);
                    }
                    __syncwarp();
                    for (int eidx = lane; eidx < total; eidx += 32) {
                        const uint32_t ent = rq[warp][eidx];
                        const int mi = (int)(ent & 7u), q = (int)((ent >> 3) & 31u), otid = warp * 32 + (int)(ent >> 8);
                        const int k = base + otid + q * SCR_THREADS;
                        float p[NARR];
#pragma unroll
                        for (int c = 0; c < NARR; ++c) p[c] = arr[c][k];
                        const float *M = ctx[mi];
                        bool plain = false, border = false;
                        float v = 0.f, e = 0.f;
                        if (KIND == KIND_PNP) {
                            scr::transfer_point<true>(M, scr::pnp_terms(M, p[0], p[1], p[2], p[3], p[4]), plain, border, v, e);
                        } else if (KIND == KIND_HOMOG) {
                            scr::transfer_point<false>(M, scr::homography_terms(M, p[0], p[1], p[2], p[3]), plain, border, v, e);
                        } else {
                            scr::sampson_point(M, p[0], p[1], p[2], p[3], plain, border, v, e);
                            if (KIND == KIND_RELPOSE && (plain || border)) {
                                bool ok, cb;
                                scr::cheirality_point(M + 9, M[scr::S_EH], p[0], p[1], p[2], p[3], ok, cb);
                                if (cb) { // the cheirality decision itself is uncertain: +-1 inlier, up to thr of score
                                    border = true;
                                    e += thr;
                                } else if (!ok) {
                                    border = false; // certainly behind a camera: not an inlier whatever the residual
                                }
                                plain = plain && ok;
                            }
                        }
                        if (border) atomicAdd(&s_border[mi], 1u);
                        if (plain || border) {
#pragma unroll
                            for (int i = 0; i < SCR_TM; ++i)
                                if (i == mi) {
                                    if (plain) {
                                        ++cnt[i];
                                        sc[i] += v;
                                    }
                                    er[i] += e;
                                }
                        }
                    }
                    __syncwarp();
                }
            }
        }
#pragma unroll
        for (int i = 0; i < SCR_TM; ++i) {
            const uint32_t c = warp_sum_u(cnt[i]);
            const float v = warp_sum_f(sc[i]);
            const float ev = warp_sum_f(er[i]);
            if (lane == 0) {
                red_c[warp][i] = c;
                red_s[warp][i] = v;
                red_e[warp][i] = ev;
            }
        }
        __syncthreads();
        if (tid < tm) {
            uint32_t ct = 0;
            float st = 0.f, et = 0.f;
#pragma unroll
            for (int w = 0; w < SCR_WARPS; ++w) {
                ct += red_c[w][tid];
                st += red_s[w][tid];
                et += red_e[w][tid];
            }
            st += (float)n * thr; // the per-correspondence sums hold (r2 - thr) of the inliers only
            // + the rounding of the fp32 sums themselves: at most n/SCR_THREADS + 24 additions deep over terms of
            //   magnitude <= thr each (ct of them), and the final n * thr product and addition
            const float depth = (float)(n / SCR_THREADS + 24);
            et = et * (1.f + 1e-5f) + scr::U * thr * (depth * (float)ct + 2.2f * (float)n);
            out.fcounts[seg + m0 + tid] = ct;
            out.fscores[seg + m0 + tid] = st;
            out.fborder[seg + m0 + tid] = s_border[tid];
            out.ferr[seg + m0 + tid] = et * (1.f + 1e-5f);
        }
    }
    } // problems of this CTA
}

// Exact fp64 rescoring of a list of model slots (fast mode confirmation): one CTA per listed slot.
template <int KIND>
__global__ void __launch_bounds__(SCORE_THREADS, 4)
    k_score_list(const ProblemDev *__restrict__ probs, const double *__restrict__ models,
                 const int *__restrict__ model_prob, const int *__restrict__ slots, int n_slots, uint32_t *counts,
                 double *scores) {
    constexpr int MSZ = kind_model_size(KIND);
    __shared__ ScoreRed red;
    for (int j = blockIdx.x; j < n_slots; j += gridDim.x) {
        const int m = slots[j];
        const ProblemDev P = probs[model_prob[m]];
        double mdl[MSZ];
#pragma unroll
        for (int k = 0; k < MSZ; ++k) mdl[k] = models[(size_t)m * MSZ + k];
        uint32_t cnt;
        double score;
        cta_score<KIND>(P, mdl, P.sq_thr, &red, cnt, score);
        if (threadIdx.x == 0) {
            counts[m] = cnt;
            scores[m] = score;
        }
    }
}

// fast mode confirmation driven by the device-side candidate lists of k_select: CTA (x, a) rescores the candidates
// x, x + gridDim.x, ... of active problem a in fp64 (same cta_score routine, hence the same bits, as everywhere else).
template <int KIND>
__global__ void __launch_bounds__(SCORE_THREADS, 4)
    k_confirm(const ProblemDev *__restrict__ probs, const SelectArgs A, const double *__restrict__ models) {
    constexpr int MSZ = kind_model_size(KIND);
    __shared__ ScoreRed red;
    const int a = blockIdx.y;
    const int nc = A.n_cand[a];
    if ((int)blockIdx.x >= nc) return;
    const RoundProb R = A.rp[a];
    const ProblemDev P = probs[R.pidx];
    for (int j = blockIdx.x; j < nc; j += gridDim.x) {
        const int m = A.cand_slot[R.seg_base + j];
        double mdl[MSZ];
#pragma unroll
        for (int k = 0; k < MSZ; ++k) mdl[k] = models[(size_t)m * MSZ + k];
        uint32_t cnt;
        double score;
        cta_score<KIND>(P, mdl, P.sq_thr, &red, cnt, score);
        if (threadIdx.x == 0) {
            A.counts[m] = cnt;
            A.scores[m] = score;
        }
    }
}

template <int KIND> static size_t hyp_smem_bytes() { return 256 + sizeof(HypScratch<KIND>) * HYP_WARPS; }

// Occupancy figures and opt-in attributes are per device: the caches below are indexed by the current device so that a
// process driving several GPUs (plb_set_device from different threads) configures each of them.
constexpr int MAX_DEVICES = 64;
static int cur_dev() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev >= 0 && dev < MAX_DEVICES) ? dev : 0;
}
static int sm_count() {
    static int cached[MAX_DEVICES] = {0};
    const int dev = cur_dev();
    if (cached[dev] == 0) {
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        cached[dev] = n > 0 ? n : 132;
    }
    return cached[dev];
}

template <int KIND> static int solve_blocks_per_sm() {
    static int cached_dev[MAX_DEVICES] = {0};
    int &cached = cached_dev[cur_dev()];
    if (cached <= 0) {
        const size_t smem = hyp_smem_bytes<KIND>();
        cudaFuncSetAttribute(k_solve<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        int nb = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_solve<KIND>, HYP_WARPS * 32, smem);
        cached = nb > 0 ? nb : 1;
    }
    return cached;
}
template <int KIND> static int score_blocks_per_sm() {
    static int cached_dev[MAX_DEVICES] = {0};
    int &cached = cached_dev[cur_dev()];
    if (cached <= 0) {
        int nb = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_score<KIND>, SCORE_THREADS, 0);
        cached = nb > 0 ? nb : 1;
    }
    return cached;
}
int device_sm_count() { return sm_count(); }

static int prep_blocks_per_sm() {
    static int cached_dev[MAX_DEVICES] = {0};
    int &cached = cached_dev[cur_dev()];
    if (cached <= 0) {
        const size_t smem = PREP_SMEM;
        cudaFuncSetAttribute(k5_prep, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        int nb = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k5_prep, HYP_WARPS * 32, smem);
        cached = nb > 0 ? nb : 1;
    }
    return cached;
}

template <int KIND>
static void launch_hyp_t(const RoundDesc &R, int *work, const HypOut &out, int mode, int max_n_pad, cudaStream_t stream,
                         cudaEvent_t ev_between) {
    // persistent grids: a multiple of the SM count (resident CTAs per SM from the occupancy API), never more CTAs
    // than there is work for
    if constexpr (KIND == KIND_RELPOSE_TS) mode = 0; // no fp32 screening copy of the 18-array layout: exact scoring
    if (kind_is_relpose(KIND) && (KIND == KIND_RELPOSE_TS || out.s5_blk != nullptr)) {
        // first half: one thread per sample (PLB_PREP_LANE=0: four samples per warp, k5_prep)
        static const bool lane_prep = [] {
            const char *e = std::getenv("PLB_PREP_LANE");
            return e ? std::atoi(e) != 0 : true;
        }();
        if (lane_prep) {
            static const int unr = [] {
                const char *e = std::getenv("PLB_PREP_UNR"); // columns of the right-hand side solved per loop pass
                return e ? std::atoi(e) : 1;
            }();
            static bool attr_set[MAX_DEVICES] = {false};
            if (!attr_set[cur_dev()]) {
                cudaFuncSetAttribute(k5_prep_lane<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PREPL_SMEM);
                cudaFuncSetAttribute(k5_prep_lane<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PREPL_SMEM);
                attr_set[cur_dev()] = true;
            }
            k5_gather<<<(R.n_total + 255) / 256, 256, 0, stream>>>(R, out);
            const unsigned grid = (unsigned)((R.n_total + PREPL_THREADS - 1) / PREPL_THREADS);
            if (unr == 1) k5_prep_lane<1><<<grid, PREPL_THREADS, PREPL_SMEM, stream>>>(R, out);
            else k5_prep_lane<2><<<grid, PREPL_THREADS, PREPL_SMEM, stream>>>(R, out);
        } else {
            int blocks = prep_blocks_per_sm() * sm_count();
            const int per_cta = HYP_WARPS * PREP_SAMPLES_PER_WARP;
            const int need = (R.n_total + per_cta - 1) / per_cta;
            if (blocks > need) blocks = need;
            if (blocks < 1) blocks = 1;
            k5_prep<<<blocks, HYP_WARPS * 32, PREP_SMEM, stream>>>(R, work, out);
        }
        k5_roots<<<(R.n_total + ROOTS_THREADS - 1) / ROOTS_THREADS, ROOTS_THREADS, 0, stream>>>(R.n_total, out);
        const int warps = (R.n_total + 31) / 32;
        k5_back<<<(warps * 32 + 127) / 128, 128, 0, stream>>>(R, out);
    } else if constexpr (KIND == KIND_PNP || KIND == KIND_HOMOG) {
        // closed-form solvers: one thread per minimal sample (PLB_SOLVE_LANE=0: the warp-per-sample kernel)
        static const bool lane_solve = [] {
            const char *e = std::getenv("PLB_SOLVE_LANE");
            return e ? std::atoi(e) != 0 : true;
        }();
        if (lane_solve) {
            k_solve_lane<KIND><<<(R.n_total + 127) / 128, 128, 0, stream>>>(R, out);
        } else {
            int blocks = solve_blocks_per_sm<KIND>() * sm_count();
            const int need = (R.n_total + HYP_WARPS - 1) / HYP_WARPS;
            if (blocks > need) blocks = need;
            if (blocks < 1) blocks = 1;
            k_solve<KIND><<<blocks, HYP_WARPS * 32, hyp_smem_bytes<KIND>(), stream>>>(R, work, out);
        }
    } else if constexpr (KIND == KIND_FUND) {
        // relpose_7pt: one thread per sample (PLB_SOLVE7_LANE=0: four samples per warp; PLB_SOLVE7_GRP=0: the
        // warp-per-sample kernel)
        static const bool lane7 = [] {
            const char *e = std::getenv("PLB_SOLVE7_LANE");
            return e ? std::atoi(e) != 0 : true;
        }();
        static const bool grp7 = [] {
            const char *e = std::getenv("PLB_SOLVE7_GRP");
            return e ? std::atoi(e) != 0 : true;
        }();
        if (lane7) {
            static bool attr_set[MAX_DEVICES] = {false};
            if (!attr_set[cur_dev()]) {
                cudaFuncSetAttribute(k7_solve_lane, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K7L_SMEM);
                attr_set[cur_dev()] = true;
            }
            k7_solve_lane<<<(R.n_total + K7L_THREADS - 1) / K7L_THREADS, K7L_THREADS, K7L_SMEM, stream>>>(R, out);
        } else if (grp7) {
            static int per_sm_dev[MAX_DEVICES] = {0};
            int &per_sm = per_sm_dev[cur_dev()];
            if (per_sm <= 0) {
                cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k7_solve, HYP_WARPS * 32, K7_SMEM);
                if (per_sm < 1) per_sm = 1;
            }
            int blocks = per_sm * sm_count();
            const int need = (R.n_total + 4 * HYP_WARPS - 1) / (4 * HYP_WARPS);
            if (blocks > need) blocks = need;
            if (blocks < 1) blocks = 1;
            k7_solve<<<blocks, HYP_WARPS * 32, K7_SMEM, stream>>>(R, work, out);
        } else {
            int blocks = solve_blocks_per_sm<KIND>() * sm_count();
            const int need = (R.n_total + HYP_WARPS - 1) / HYP_WARPS;
            if (blocks > need) blocks = need;
            if (blocks < 1) blocks = 1;
            k_solve<KIND><<<blocks, HYP_WARPS * 32, hyp_smem_bytes<KIND>(), stream>>>(R, work, out);
        }
    } else if constexpr (KIND != KIND_RELPOSE_TS) {
        int blocks = solve_blocks_per_sm<KIND>() * sm_count();
        const int need = (R.n_total + HYP_WARPS - 1) / HYP_WARPS;
        if (blocks > need) blocks = need;
        if (blocks < 1) blocks = 1;
        k_solve<KIND><<<blocks, HYP_WARPS * 32, hyp_smem_bytes<KIND>(), stream>>>(R, work, out);
    }
    if (ev_between) cudaEventRecord(ev_between, stream); // solve | score boundary for the per-kernel timing
    if (mode == 0) {
        // tiled exact scoring: grid.y = active problem, grid.x CTAs stride over that problem's tiles of SCORE_TM models
        int tiles = (out.max_seg_cap + score_tm<KIND>() - 1) / score_tm<KIND>();
        int gx = (4 * 8 * sm_count() + R.n_active - 1) / R.n_active; // ~4 waves of 8 CTAs per SM over the whole group
        if (gx > tiles) gx = tiles;
        if (gx < 1) gx = 1;
        k_score_tiled<KIND><<<dim3(gx, R.n_active, 1), SCORE_THREADS, 0, stream>>>(R, out);
    } else if constexpr (KIND != KIND_RELPOSE_TS) {
        // fp32 screening: one CTA holds one problem's fp32 arrays in shared memory (TMA) and strides over its tiles
        constexpr int NARR = (KIND == KIND_PNP) ? 5 : 4;
        const size_t bytes = (size_t)NARR * (size_t)max_n_pad * 4;
        const int use_smem = bytes <= 200 * 1024 ? 1 : 0;
        static bool attr_done_dev[MAX_DEVICES] = {false};
        bool &attr_done = attr_done_dev[cur_dev()];
        const bool small = max_n_pad <= 2048; // few correspondences per problem: 128-thread CTAs, four per SM
        auto kern = small ? k_screen<KIND, 128> : k_screen<KIND, 512>;
        const int nthr = small ? 128 : 512;
        if (!attr_done) {
            cudaFuncSetAttribute(k_screen<KIND, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
            attr_done = true;
        }
        // one wave: resident CTAs per SM (occupancy API for this shared-memory size) x SMs; the kernel partitions the
        // (problem, tile) list over the CTAs by cost itself
        int per_sm = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, nthr, use_smem ? bytes : 0);
        if (per_sm < 1) per_sm = 1;
        long long tiles = ((long long)out.max_seg_cap + SCR_TM - 1) / SCR_TM * (long long)R.n_active;
        int gx = per_sm * sm_count();
        if ((long long)gx > tiles) gx = (int)tiles;
        if (gx < 1) gx = 1;
        kern<<<gx, nthr, use_smem ? bytes : 0, stream>>>(R, out, use_smem);
    }
}
void launch_hypotheses(int kind, const RoundDesc &R, int *work, const HypOut &out, int mode, int max_n_pad,
                       cudaStream_t stream, cudaEvent_t ev_between) {
    cudaMemsetAsync(work, 0, 3 * sizeof(int), stream); // [0] sample queue, [2] overflow flag
    cudaMemsetAsync(out.prob_count, 0, sizeof(int) * R.n_active, stream);
    switch (kind) {
    case KIND_PNP: launch_hyp_t<KIND_PNP>(R, work, out, mode, max_n_pad, stream, ev_between); break;
    case KIND_RELPOSE: launch_hyp_t<KIND_RELPOSE>(R, work, out, mode, max_n_pad, stream, ev_between); break;
    case KIND_FUND: launch_hyp_t<KIND_FUND>(R, work, out, mode, max_n_pad, stream, ev_between); break;
    case KIND_RELPOSE_TS: launch_hyp_t<KIND_RELPOSE_TS>(R, work, out, mode, max_n_pad, stream, ev_between); break;
    default: launch_hyp_t<KIND_HOMOG>(R, work, out, mode, max_n_pad, stream, ev_between); break;
    }
}
void launch_score_list(int kind, const ProblemDev *probs, const double *models, const int *model_prob, const int *slots,
                       int n_slots, uint32_t *counts, double *scores, cudaStream_t stream) {
    if (n_slots <= 0) return;
    int blocks = n_slots;
    if (blocks > 8 * sm_count()) blocks = 8 * sm_count();
    switch (kind) {
    case KIND_PNP: k_score_list<KIND_PNP><<<blocks, SCORE_THREADS, 0, stream>>>(probs, models, model_prob, slots, n_slots, counts, scores); break;
    case KIND_RELPOSE: k_score_list<KIND_RELPOSE><<<blocks, SCORE_THREADS, 0, stream>>>(probs, models, model_prob, slots, n_slots, counts, scores); break;
    case KIND_FUND: k_score_list<KIND_FUND><<<blocks, SCORE_THREADS, 0, stream>>>(probs, models, model_prob, slots, n_slots, counts, scores); break;
    case KIND_RELPOSE_TS: k_score_list<KIND_RELPOSE_TS><<<blocks, SCORE_THREADS, 0, stream>>>(probs, models, model_prob, slots, n_slots, counts, scores); break;
    default: k_score_list<KIND_HOMOG><<<blocks, SCORE_THREADS, 0, stream>>>(probs, models, model_prob, slots, n_slots, counts, scores); break;
    }
}

void launch_confirm(int kind, const ProblemDev *probs, const SelectArgs &A, const double *models, cudaStream_t stream) {
    if (A.na <= 0) return;
    int gx = (8 * sm_count() + A.na - 1) / A.na;
    if (gx > 64) gx = 64;
    if (gx < 1) gx = 1;
    const dim3 grid((unsigned)gx, (unsigned)A.na, 1);
    switch (kind) {
    case KIND_PNP: k_confirm<KIND_PNP><<<grid, SCORE_THREADS, 0, stream>>>(probs, A, models); break;
    case KIND_RELPOSE: k_confirm<KIND_RELPOSE><<<grid, SCORE_THREADS, 0, stream>>>(probs, A, models); break;
    case KIND_FUND: k_confirm<KIND_FUND><<<grid, SCORE_THREADS, 0, stream>>>(probs, A, models); break;
    case KIND_RELPOSE_TS: k_confirm<KIND_RELPOSE_TS><<<grid, SCORE_THREADS, 0, stream>>>(probs, A, models); break;
    default: k_confirm<KIND_HOMOG><<<grid, SCORE_THREADS, 0, stream>>>(probs, A, models); break;
    }
}

// ============================================================================================================
// explicit model scoring
// ============================================================================================================
void launch_score_models(int kind, const ProblemDev *probs, const double *models, const int *model_prob, int n_models,
                         const int *n_models_dev, uint32_t *counts, double *scores, cudaStream_t stream) {
    if (n_models <= 0) return;
    int blocks = n_models;
    if (blocks > 8 * sm_count()) blocks = 8 * sm_count();
    switch (kind) {
    case KIND_PNP: k_score<KIND_PNP><<<blocks, SCORE_THREADS, 0, stream>>>(probs, models, model_prob, n_models_dev, n_models, counts, scores); break;
    case KIND_RELPOSE: k_score<KIND_RELPOSE><<<blocks, SCORE_THREADS, 0, stream>>>(probs, models, model_prob, n_models_dev, n_models, counts, scores); break;
    case KIND_FUND: k_score<KIND_FUND><<<blocks, SCORE_THREADS, 0, stream>>>(probs, models, model_prob, n_models_dev, n_models, counts, scores); break;
    case KIND_RELPOSE_TS: k_score<KIND_RELPOSE_TS><<<blocks, SCORE_THREADS, 0, stream>>>(probs, models, model_prob, n_models_dev, n_models, counts, scores); break;
    default: k_score<KIND_HOMOG><<<blocks, SCORE_THREADS, 0, stream>>>(probs, models, model_prob, n_models_dev, n_models, counts, scores); break;
    }
}

// ============================================================================================================
// inlier masks
// ============================================================================================================
template <int KIND>
__global__ void k_inlier_mask(const ProblemDev *__restrict__ probs, const MaskDesc *__restrict__ descs, char *mask_base) {
    constexpr int MSZ = kind_model_size(KIND);
    const MaskDesc &D = descs[blockIdx.y];
    const ProblemDev P = probs[D.pidx];
    const double sq_thr = P.sq_thr;
    char *mask = mask_base + D.mask_off;
    double mdl[MSZ];
#pragma unroll
    for (int k = 0; k < MSZ; ++k) mdl[k] = D.model[k];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P.n) return;
    if (KIND == KIND_PNP) {
        // robust/utils.cc:374-383: Z = R*X + t ; r2 = |Z.hnormalized() - x|^2 ; inlier iff r2 < thr && Z(2) > 0
        const m3 R = quat_to_rot(mdl);
        const d3 Z = mvec(R, mk(P.p[2][k], P.p[3][k], P.p[4][k])) + mk(mdl[4], mdl[5], mdl[6]);
        const double d0 = Z.x / Z.z - P.p[0][k], d1 = Z.y / Z.z - P.p[1][k];
        const double r2 = d0 * d0 + d1 * d1;
        mask[k] = (r2 < sq_thr && Z.z > 0.0) ? 1 : 0;
    } else if (KIND == KIND_RELPOSE_TS) { // robust/utils.cc:541-569
        ModelCtx<KIND> C;
        C.init(mdl);
        const double *M = reinterpret_cast<const double *>(&C);
        double v[TS_ARRAYS];
        load_ts(P, k, v);
        bool inl = tangent_r2(M, v) < sq_thr;
        if (inl) inl = cheirality_ok(M + 9, M + 13, mk(v[0], v[1], v[2]), mk(v[3], v[4], v[5]), 0.01);
        mask[k] = inl ? 1 : 0;
    } else {
        ModelCtx<KIND> C;
        C.init(mdl);
        const double *M = reinterpret_cast<const double *>(&C);
        const double x1_0 = P.p[0][k], x1_1 = P.p[1][k], x2_0 = P.p[2][k], x2_1 = P.p[3][k];
        double r2;
        if (KIND == KIND_HOMOG) r2 = homography_r2(M, x1_0, x1_1, x2_0, x2_1);
        else r2 = sampson_r2(M, x1_0, x1_1, x2_0, x2_1);
        bool inl = r2 < sq_thr;
        if (KIND == KIND_RELPOSE && inl)
            inl = cheirality_ok(M + 9, M + 13, bearing(x1_0, x1_1), bearing(x2_0, x2_1), 0.01);
        mask[k] = inl ? 1 : 0;
    }
}
// One bit per correspondence for the trip over PCIe (the host expands them to the caller's char[n]).
__global__ void k_pack_mask(const char *__restrict__ mask, uint32_t *__restrict__ bits, size_t n_bytes) {
    const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_bytes) return; // n_bytes is a multiple of 32: whole warps leave together
    const unsigned b = __ballot_sync(0xffffffffu, mask[k] != 0);
    if ((threadIdx.x & 31) == 0) bits[k >> 5] = b;
}
void launch_pack_mask(const char *mask, uint32_t *bits, size_t n_bytes, cudaStream_t stream) {
    if (n_bytes == 0) return;
    k_pack_mask<<<(unsigned)((n_bytes + 255) / 256), 256, 0, stream>>>(mask, bits, n_bytes);
}
void launch_inlier_masks(int kind, const ProblemDev *probs, const MaskDesc *descs_dev, int n_desc, int max_n,
                         char *mask_base, cudaStream_t stream) {
    if (n_desc <= 0 || max_n <= 0) return;
    const int threads = 256;
    dim3 grid((max_n + threads - 1) / threads, n_desc, 1);
    switch (kind) {
    case KIND_PNP: k_inlier_mask<KIND_PNP><<<grid, threads, 0, stream>>>(probs, descs_dev, mask_base); break;
    case KIND_RELPOSE: k_inlier_mask<KIND_RELPOSE><<<grid, threads, 0, stream>>>(probs, descs_dev, mask_base); break;
    case KIND_FUND: k_inlier_mask<KIND_FUND><<<grid, threads, 0, stream>>>(probs, descs_dev, mask_base); break;
    case KIND_RELPOSE_TS: k_inlier_mask<KIND_RELPOSE_TS><<<grid, threads, 0, stream>>>(probs, descs_dev, mask_base); break;
    default: k_inlier_mask<KIND_HOMOG><<<grid, threads, 0, stream>>>(probs, descs_dev, mask_base); break;
    }
}

// ============================================================================================================
// Levenberg-Marquardt refit: one CTA per job
// ============================================================================================================
constexpr int LM_THREADS = 256;
constexpr int LM_WARPS = LM_THREADS / 32;
constexpr int LM_MAX_CLUSTER = 8;
constexpr int LM_NV_MAX = 56;

struct LossFn { // robust/robust_loss.h:41-67,125-136
    int type;
    double thr, sq_thr, inv_sq_thr;
    PLB_DEV double loss(double r2) const {
        switch (type) {
        case 1: return fmin(r2, sq_thr);
        case 2: {
            const double r = sqrt(r2);
            return (r <= thr) ? r2 : thr * (2.0 * r - thr);
        }
        case 3: return sq_thr * log1p(r2 * inv_sq_thr);
        default: return r2;
        }
    }
    PLB_DEV double weight(double r2) const {
        switch (type) {
        case 1: return (r2 < sq_thr) ? 1.0 : 0.0;
        case 2: {
            const double r = sqrt(r2);
            return (r <= thr) ? 1.0 : thr / r;
        }
        case 3: return fmax(2.2250738585072014e-308, 1.0 / (1.0 + r2 * inv_sq_thr));
        default: return 1.0;
        }
    }
};

template <int KIND> struct LmDims;
template <> struct LmDims<KIND_PNP> { static constexpr int NP = 6, CTX = 12; };
template <> struct LmDims<KIND_RELPOSE> { static constexpr int NP = 5, CTX = 9 + 45; };
template <> struct LmDims<KIND_RELPOSE_TS> { static constexpr int NP = 5, CTX = 9 + 45; };
template <> struct LmDims<KIND_FUND> { static constexpr int NP = 7, CTX = 9 + 63; };
template <> struct LmDims<KIND_HOMOG> { static constexpr int NP = 8, CTX = 18; };

// one-sided Jacobi SVD of a 3x3 (stands in for Eigen::JacobiSVD, optim_utils.h:59-73).  Row-major in/out.
PLB_DEV void svd3_dev(const m3 &F, m3 &U, double *s, m3 &V) {
    m3 A = F;
#pragma unroll
    for (int k = 0; k < 9; ++k) V.a[k] = (k % 4 == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = 0; i < 3; ++i) {
                    alpha += A(i, p) * A(i, p);
                    beta += A(i, q) * A(i, q);
                    gamma += A(i, p) * A(i, q);
                }
                if (gamma == 0.0) continue;
                off = fmax(off, fabs(gamma) / sqrt(alpha * beta + 1e-300));
                const double zeta = (beta - alpha) / (2.0 * gamma);
                const double t = ((zeta >= 0) ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
                for (int i = 0; i < 3; ++i) {
                    const double ap = A(i, p), aq = A(i, q);
                    A(i, p) = c * ap - sn * aq;
                    A(i, q) = sn * ap + c * aq;
                    const double vp = V(i, p), vq = V(i, q);
                    V(i, p) = c * vp - sn * vq;
                    V(i, q) = sn * vp + c * vq;
                }
            }
        if (off < 1e-16) break;
    }
    double sv[3];
    for (int j = 0; j < 3; ++j) sv[j] = sqrt(dot(mcol(A, j), mcol(A, j)));
    int idx[3] = {0, 1, 2};
    // sort descending (3 elements)
    if (sv[idx[1]] > sv[idx[0]]) { int t = idx[0]; idx[0] = idx[1]; idx[1] = t; }
    if (sv[idx[2]] > sv[idx[1]]) { int t = idx[1]; idx[1] = idx[2]; idx[2] = t; }
    if (sv[idx[1]] > sv[idx[0]]) { int t = idx[0]; idx[0] = idx[1]; idx[1] = t; }
    m3 Vs, Us;
    for (int j = 0; j < 3; ++j) {
        s[j] = sv[idx[j]];
        set_col(Vs, j, mcol(V, idx[j]));
        if (s[j] > 0) set_col(Us, j, mcol(A, idx[j]) / s[j]);
        else set_col(Us, j, mk(0, 0, 0));
    }
    if (!(s[2] > 1e-14 * s[0])) set_col(Us, 2, cross(mcol(Us, 0), mcol(Us, 1)));
    if (!(s[1] > 0)) {
        const d3 u0 = mcol(Us, 0);
        const d3 e = (fabs(u0.x) < 0.9) ? mk(1, 0, 0) : mk(0, 1, 0);
        const d3 u1 = unit(cross(u0, e));
        set_col(Us, 1, u1);
        set_col(Us, 2, cross(u0, u1));
    }
    U = Us;
    V = Vs;
}

// F (row-major) from the factorised representation (qU,qV,sigma)  (optim_utils.h:74-78)
PLB_DEV m3 ff_to_F(const double *par) {
    const m3 U = quat_to_rot(par), V = quat_to_rot(par + 4);
    const double sigma = par[8];
    m3 F;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) F(r, c) = U(r, 0) * V(c, 0) + sigma * U(r, 1) * V(c, 1);
    return F;
}

// Builds the evaluation context of the current parameters (executed by thread 0).
//   PNP     : ctx[0..8] = R row-major, ctx[9..11] = t
//   RELPOSE : ctx[0..8] = E row-major, ctx[9 + 5*m + p] = d vec(E)_m / d param_p (vec column-major), tb = tangent basis
//   FUND    : ctx[0..8] = F row-major, ctx[9 + 7*m + p]
//   HOMOG   : ctx[0..8] = H row-major, ctx[9..17] = adj(H) row-major
template <int KIND> PLB_DEV void lm_build_ctx(const double *par, double *ctx, double *tb, bool with_jac) {
    if (KIND == KIND_PNP) {
        const m3 R = quat_to_rot(par);
#pragma unroll
        for (int k = 0; k < 9; ++k) ctx[k] = R.a[k];
        ctx[9] = par[4]; ctx[10] = par[5]; ctx[11] = par[6];
    } else if (kind_is_relpose(KIND)) {
        const m3 E = essential_from_pose(par, par + 4);
#pragma unroll
        for (int k = 0; k < 9; ++k) ctx[k] = E.a[k];
        if (with_jac) {
            const m3 R = quat_to_rot(par);
            const d3 t = mk(par[4], par[5], par[6]);
            // tangent basis (optim/relative.h:62-82)
            d3 b0;
            const double ax = fabs(t.x), ay = fabs(t.y), az = fabs(t.z);
            if (ax < ay) {
                if (ax < az) b0 = unit(cross(t, mk(1, 0, 0)));
                else b0 = unit(cross(t, mk(0, 0, 1)));
            } else {
                if (ay < az) b0 = unit(cross(t, mk(0, 1, 0)));
                else b0 = unit(cross(t, mk(0, 0, 1)));
            }
            const d3 b1 = unit(cross(b0, t));
            tb[0] = b0.x; tb[1] = b1.x; tb[2] = b0.y; tb[3] = b1.y; tb[4] = b0.z; tb[5] = b1.z;
            // d vec(E) / d(rotation, translation)  (optim/relative.h:39-60)
            const d3 e0 = mcol(E, 0), e1 = mcol(E, 1), e2 = mcol(E, 2);
            const double e0a[3] = {e0.x, e0.y, e0.z}, e1a[3] = {e1.x, e1.y, e1.z}, e2a[3] = {e2.x, e2.y, e2.z};
            double *D = ctx + 9;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                D[5 * r + 0] = 0.0;           D[5 * r + 1] = -e2a[r];          D[5 * r + 2] = e1a[r];
                D[5 * (3 + r) + 0] = e2a[r];  D[5 * (3 + r) + 1] = 0.0;        D[5 * (3 + r) + 2] = -e0a[r];
                D[5 * (6 + r) + 0] = -e1a[r]; D[5 * (6 + r) + 1] = e0a[r];     D[5 * (6 + r) + 2] = 0.0;
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const d3 v0 = cross(b0, mcol(R, c)), v1 = cross(b1, mcol(R, c));
                D[5 * (3 * c + 0) + 3] = v0.x; D[5 * (3 * c + 0) + 4] = v1.x;
                D[5 * (3 * c + 1) + 3] = v0.y; D[5 * (3 * c + 1) + 4] = v1.y;
                D[5 * (3 * c + 2) + 3] = v0.z; D[5 * (3 * c + 2) + 4] = v1.z;
            }
        }
    } else if (KIND == KIND_FUND) {
        const m3 F = ff_to_F(par);
#pragma unroll
        for (int k = 0; k < 9; ++k) ctx[k] = F.a[k];
        if (with_jac) {
            const m3 U = quat_to_rot(par), V = quat_to_rot(par + 4);
            double *D = ctx + 9;
            // optim/fundamental.h:68-77: U' = exp([w]x)U -> [e_k]x F ; V' = exp([w]x)V -> -F[e_k]x ; sigma -> u1 v1^T
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const int m = 3 * c + r;
                    const double f0 = F(0, c), f1 = F(1, c), f2 = F(2, c);
                    D[7 * m + 0] = (r == 0) ? 0.0 : (r == 1 ? -f2 : f1);
                    D[7 * m + 1] = (r == 0) ? f2 : (r == 1 ? 0.0 : -f0);
                    D[7 * m + 2] = (r == 0) ? -f1 : (r == 1 ? f0 : 0.0);
                    const double g0 = F(r, 0), g1 = F(r, 1), g2 = F(r, 2);
                    D[7 * m + 3] = (c == 0) ? 0.0 : (c == 1 ? -g2 : g1);
                    D[7 * m + 4] = (c == 0) ? g2 : (c == 1 ? 0.0 : -g0);
                    D[7 * m + 5] = (c == 0) ? -g1 : (c == 1 ? g0 : 0.0);
                    D[7 * m + 6] = U(r, 1) * V(c, 1);
                }
        }
    } else {
        // par is column-major H
        m3 H;
#pragma unroll
        for (int k = 0; k < 9; ++k) H.a[3 * (k % 3) + k / 3] = par[k];
#pragma unroll
        for (int k = 0; k < 9; ++k) ctx[k] = H.a[k];
        double *G = ctx + 9; // adjugate (optim/homography.h:160-175)
        G[0] = H(1, 1) * H(2, 2) - H(1, 2) * H(2, 1);
        G[1] = H(0, 2) * H(2, 1) - H(0, 1) * H(2, 2);
        G[2] = H(0, 1) * H(1, 2) - H(0, 2) * H(1, 1);
        G[3] = H(1, 2) * H(2, 0) - H(1, 0) * H(2, 2);
        G[4] = H(0, 0) * H(2, 2) - H(0, 2) * H(2, 0);
        G[5] = H(0, 2) * H(1, 0) - H(0, 0) * H(1, 2);
        G[6] = H(1, 0) * H(2, 1) - H(1, 1) * H(2, 0);
        G[7] = H(0, 1) * H(2, 0) - H(0, 0) * H(2, 1);
        G[8] = H(0, 0) * H(1, 1) - H(0, 1) * H(1, 0);
    }
}

// parameter update  (optim/absolute.h:146-160, relative.h:152-157, fundamental.h:106-112, homography.h:157-161)
template <int KIND> PLB_DEV void lm_step(const double *par, const double *dp, const double *tb, double *out) {
    if (KIND == KIND_PNP) {
        double e[4];
        quat_exp(mk(dp[0], dp[1], dp[2]), e);
        quat_mul(par, e, out);
        const d3 rt = quat_rotate(par, mk(dp[3], dp[4], dp[5]));
        out[4] = par[4] + rt.x; out[5] = par[5] + rt.y; out[6] = par[6] + rt.z;
    } else if (kind_is_relpose(KIND)) {
        double e[4];
        quat_exp(mk(dp[0], dp[1], dp[2]), e);
        quat_mul(par, e, out);
#pragma unroll
        for (int r = 0; r < 3; ++r) out[4 + r] = par[4 + r] + (tb[2 * r] * dp[3] + tb[2 * r + 1] * dp[4]);
    } else if (KIND == KIND_FUND) {
        double e[4];
        quat_exp(mk(dp[0], dp[1], dp[2]), e);
        quat_mul(e, par, out);
        quat_exp(mk(dp[3], dp[4], dp[5]), e);
        quat_mul(e, par + 4, out + 4);
        out[8] = par[8] + dp[6];
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) out[k] = par[k] + dp[k];
        out[8] = par[8];
    }
}

// Sampson residual and its derivative wrt vec(E) (column-major)   (optim/relative.h:118-149)
PLB_DEV void sampson_res_dF(const double *E, double a0, double a1, double b0, double b1, double &r, double *dF) {
    const double Ex0 = E[0] * a0 + E[1] * a1 + E[2] * 1.0;
    const double Ex1 = E[3] * a0 + E[4] * a1 + E[5] * 1.0;
    const double Ex2 = E[6] * a0 + E[7] * a1 + E[8] * 1.0;
    const double C = b0 * Ex0 + b1 * Ex1 + 1.0 * Ex2;
    const double J0 = E[0] * b0 + E[3] * b1 + E[6];
    const double J1 = E[1] * b0 + E[4] * b1 + E[7];
    const double J2 = E[0] * a0 + E[1] * a1 + E[2];
    const double J3 = E[3] * a0 + E[4] * a1 + E[5];
    const double nJ = sqrt(J0 * J0 + J1 * J1 + J2 * J2 + J3 * J3);
    const double inv = 1.0 / nJ;
    r = C * inv;
    const double s = C * inv * inv;
    dF[0] = a0 * b0 - s * (J2 * a0 + J0 * b0);
    dF[1] = a0 * b1 - s * (J3 * a0 + J0 * b1);
    dF[2] = a0 - s * (J0);
    dF[3] = a1 * b0 - s * (J2 * a1 + J1 * b0);
    dF[4] = a1 * b1 - s * (J3 * a1 + J1 * b1);
    dF[5] = a1 - s * (J1);
    dF[6] = b0 - s * (J2);
    dF[7] = b1 - s * (J3);
    dF[8] = 1.0;
#pragma unroll
    for (int k = 0; k < 9; ++k) dF[k] *= inv;
}
// residual only (optim/relative.h:98-105)
PLB_DEV double sampson_res(const double *E, double a0, double a1, double b0, double b1) {
    const double Ex0 = E[0] * a0 + E[1] * a1 + E[2] * 1.0;
    const double Ex1 = E[3] * a0 + E[4] * a1 + E[5] * 1.0;
    const double Ex2 = E[6] * a0 + E[7] * a1 + E[8] * 1.0;
    const double C = b0 * Ex0 + b1 * Ex1 + 1.0 * Ex2;
    const double n1 = Ex0 * Ex0 + Ex1 * Ex1;
    const double t0 = E[0] * b0 + E[3] * b1 + E[6] * 1.0;
    const double t1 = E[1] * b0 + E[4] * b1 + E[7] * 1.0;
    return C / sqrt(n1 + (t0 * t0 + t1 * t1));
}

template <int NP> struct JacAcc {
    static constexpr int NT = NP * (NP + 1) / 2;
    double jtj[NT];
    double jtr[NP];
    double cnt;
    PLB_DEV void zero() {
#pragma unroll
        for (int i = 0; i < NT; ++i) jtj[i] = 0.0;
#pragma unroll
        for (int i = 0; i < NP; ++i) jtr[i] = 0.0;
        cnt = 0.0;
    }
    // 1-dim residual (jacobian_accumulator.h:125-141)
    PLB_DEV void add1(const LossFn &L, double res, const double *J) {
        const double w = L.weight(res * res);
        if (w == 0) return;
        int t = 0;
#pragma unroll
        for (int i = 0; i < NP; ++i)
#pragma unroll
            for (int j = 0; j <= i; ++j) jtj[t++] += w * (J[i] * J[j]);
        const double wr = w * res;
#pragma unroll
        for (int i = 0; i < NP; ++i) jtr[i] += wr * J[i];
        cnt += 1.0;
    }
    // 2-dim residual (jacobian_accumulator.h:87-104)
    PLB_DEV void add2(const LossFn &L, double r0, double r1, const double *J0, const double *J1) {
        const double w = L.weight(r0 * r0 + r1 * r1);
        if (w == 0) return;
        int t = 0;
#pragma unroll
        for (int i = 0; i < NP; ++i)
#pragma unroll
            for (int j = 0; j <= i; ++j) jtj[t++] += w * (J0[i] * J0[j] + J1[i] * J1[j]);
        const double wr0 = w * r0, wr1 = w * r1;
#pragma unroll
        for (int i = 0; i < NP; ++i) jtr[i] += J0[i] * wr0 + J1[i] * wr1;
        cnt += 1.0;
    }
};

struct LmShared {
    double par[9], par_new[9];
    double ctx[80];
    double tb[6], tb_new[6];
    double red[LM_WARPS][LM_NV_MAX];
    double sums[2][LM_NV_MAX]; // CTA partial sums, double-buffered: read by the other CTAs of the cluster (DSMEM)
    double tot[LM_NV_MAX];     // cluster totals (identical in every CTA)
    ScoreRed sred;
    int wcount[LM_WARPS];
    int flag;
};

// Cluster-wide deterministic sum of NV per-thread values -> S->tot[0..NV) in every CTA of the cluster.
// Order: xor-butterfly inside a warp, warps left to right, CTAs in rank order.
template <int NV> PLB_DEV void cluster_sum(LmShared *S, const double *v, int &buf, int csize) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const double s = warp_sum(v[i]);
        if (lane == 0) S->red[warp][i] = s;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        double s = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += S->red[w][threadIdx.x];
        S->sums[buf][threadIdx.x] = s;
    }
    cluster.sync();
    if (threadIdx.x < NV) {
        double t = 0.0;
        for (int r = 0; r < csize; ++r) {
            const double *remote = cluster.map_shared_rank(&S->sums[buf][0], r);
            t += remote[threadIdx.x];
        }
        S->tot[threadIdx.x] = t;
    }
    __syncthreads();
    buf ^= 1;
}

// thread 0 -> whole CTA broadcast of a small integer (two barriers: the slot can be reused right away)
PLB_DEV int block_bcast(LmShared *S, int v) {
    if (threadIdx.x == 0) S->flag = v;
    __syncthreads();
    const int r = S->flag;
    __syncthreads();
    return r;
}

// One evaluation pass at the parameters whose context is in S->ctx: robust cost + row count (compute_residual of the
// refiners) AND the normal equations JtJ (lower triangle, packed row-major), Jtr + count of non-zero-weight rows
// (compute_jacobian), accumulated separately exactly as two passes of the reference would.
// Output layout in S->tot: [0] loss sum, [1] residual rows, [2..2+NT) JtJ, [2+NT..2+NT+NP) Jtr, [2+NT+NP] jac rows.
template <int KIND>
PLB_DEV void lm_eval_pass(const ProblemDev &P, const LmParams &prm, const LossFn &L, const int *list, int lo, int na,
                          LmShared *S, int &buf, int csize) {
    constexpr int NP = LmDims<KIND>::NP;
    constexpr int NT = NP * (NP + 1) / 2;
    const double *ctx = S->ctx;
    JacAcc<NP> A;
    A.zero();
    double lsum = 0.0, rows = 0.0;
    for (int i = threadIdx.x; i < na; i += (int)blockDim.x) {
        const int k = list ? list[i] : lo + i;
        if (KIND == KIND_PNP) {
            const double X0 = P.p[2][k], X1 = P.p[3][k], X2 = P.p[4][k];
            const double Z0 = ctx[0] * X0 + ctx[1] * X1 + ctx[2] * X2 + ctx[9];
            const double Z1 = ctx[3] * X0 + ctx[4] * X1 + ctx[5] * X2 + ctx[10];
            const double Z2 = ctx[6] * X0 + ctx[7] * X1 + ctx[8] * X2 + ctx[11];
            if (Z2 < 0) continue; // optim/absolute.h:57-58,93-94
            double zp0, zp1, xr0, xr1, Jp[2][3];
            if (prm.use_camera) { // <Model>::project for the residual, ::project_with_jac for the Jacobian pass
                cam_project(prm.cam, Z0, Z1, Z2, xr0, xr1); // (optim/absolute.h:59-61,97-104)
                cam_project_with_jac(prm.cam, Z0, Z1, Z2, zp0, zp1, &Jp[0][0]);
            } else { // NullCameraModel (camera_models.cc:2708-2722)
                zp0 = Z0 / Z2;
                zp1 = Z1 / Z2;
                xr0 = zp0;
                xr1 = zp1;
                const double z_inv = 1.0 / Z2;
                Jp[0][0] = z_inv; Jp[0][1] = 0.0; Jp[0][2] = -zp0 * z_inv;
                Jp[1][0] = 0.0; Jp[1][1] = z_inv; Jp[1][2] = -zp1 * z_inv;
            }
            const double x0 = P.p[0][k], x1 = P.p[1][k];
            {
                const double q0 = xr0 - x0, q1 = xr1 - x1;
                lsum += L.loss(q0 * q0 + q1 * q1);
                rows += 1.0;
            }
            const double r0 = zp0 - x0, r1 = zp1 - x1;
            double J[2][6];
#pragma unroll
            for (int a = 0; a < 2; ++a) {
                double dZ[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) dZ[c] = Jp[a][0] * ctx[c] + Jp[a][1] * ctx[3 + c] + Jp[a][2] * ctx[6 + c];
                J[a][0] = -X2 * dZ[1] + X1 * dZ[2];
                J[a][1] = X2 * dZ[0] - X0 * dZ[2];
                J[a][2] = -X1 * dZ[0] + X0 * dZ[1];
                J[a][3] = dZ[0]; J[a][4] = dZ[1]; J[a][5] = dZ[2];
            }
            A.add2(L, r0, r1, J[0], J[1]);
        } else if (KIND == KIND_HOMOG) {
            const double a0 = P.p[0][k], a1 = P.p[1][k], b0 = P.p[2][k], b1 = P.p[3][k];
            const double *H = ctx, *G = ctx + 9;
            // forward transfer (optim/homography.h:63-71,107-123); parameters = H00,H10,H20,H01,H11,H21,H02,H12
            const double Hx0 = H[0] * a0 + H[1] * a1 + H[2];
            const double Hx1 = H[3] * a0 + H[4] * a1 + H[5];
            const double iw = 1.0 / (H[6] * a0 + H[7] * a1 + H[8]);
            const double z0 = Hx0 * iw, z1 = Hx1 * iw;
            const double r0 = z0 - b0, r1 = z1 - b1;
            lsum += L.loss(r0 * r0 + r1 * r1);
            double J0[8] = {a0, 0.0, -a0 * z0, a1, 0.0, -a1 * z0, 1.0, 0.0};
            double J1[8] = {0.0, a0, -a0 * z1, 0.0, a1, -a1 * z1, 0.0, 1.0};
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                J0[m] = J0[m] * iw;
                J1[m] = J1[m] * iw;
            }
            A.add2(L, r0, r1, J0, J1);
            // backward transfer through adj(H) (optim/homography.h:73-81,125-152):  y = pi(G x2),
            // dy_i/dH_k = ( (dG/dH_k x2)_i - y_i (dG/dH_k x2)_2 ) / (G x2)_2
            const double Gx0 = G[0] * b0 + G[1] * b1 + G[2];
            const double Gx1 = G[3] * b0 + G[4] * b1 + G[5];
            const double iv = 1.0 / (G[6] * b0 + G[7] * b1 + G[8]);
            const double y0 = Gx0 * iv, y1 = Gx1 * iv;
            const double s0 = y0 - a0, s1 = y1 - a1;
            lsum += L.loss(s0 * s0 + s1 * s1);
            rows += 2.0;
            const double y0b1 = y0 * b1, y0b0 = y0 * b0, y1b1 = y1 * b1, y1b0 = y1 * b0;
            const double H00 = H[0], H01 = H[1], H02 = H[2], H10 = H[3], H11 = H[4], H12 = H[5], H20 = H[6],
                         H21 = H[7], H22 = H[8];
            double K0[8], K1[8];
            K0[0] = H21 * y0b1 - H11 * y0;
            K0[1] = H01 * y0 - H21 * y0b0;
            K0[2] = H11 * y0b0 - H01 * y0b1;
            K0[3] = H12 - H22 * b1 + H10 * y0 - H20 * y0b1;
            K0[4] = H22 * b0 - H02 - H00 * y0 + H20 * y0b0;
            K0[5] = H02 * b1 - H12 * b0 + H00 * y0b1 - H10 * y0b0;
            K0[6] = H21 * b1 - H11;
            K0[7] = H01 - H21 * b0;
            K1[0] = H22 * b1 - H12 - H11 * y1 + H21 * y1b1;
            K1[1] = H02 - H22 * b0 + H01 * y1 - H21 * y1b0;
            K1[2] = H12 * b0 - H02 * b1 - H01 * y1b1 + H11 * y1b0;
            K1[3] = H10 * y1 - H20 * y1b1;
            K1[4] = H20 * y1b0 - H00 * y1;
            K1[5] = H00 * y1b1 - H10 * y1b0;
            K1[6] = H10 - H20 * b1;
            K1[7] = H20 * b0 - H00;
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                K0[m] = K0[m] * iv;
                K1[m] = K1[m] * iv;
            }
            A.add2(L, s0, s1, K0, K1);
        } else if (KIND == KIND_RELPOSE_TS) {
            // FixCameraRelativePoseRefiner (optim/relative.h:181-249)
            double v[TS_ARRAYS];
            load_ts(P, k, v);
            double C, JC[4];
            tangent_terms(ctx, v, v + 3, v + 6, v + 12, C, JC);
            {
                const double nJc_sq = (JC[2] * JC[2] + JC[3] * JC[3]) + (JC[0] * JC[0] + JC[1] * JC[1]);
                const double rr = C / sqrt(nJc_sq);
                lsum += L.loss(rr * rr);
                rows += 1.0;
            }
            const double nJ_C = sqrt((JC[0] * JC[0] + JC[2] * JC[2]) + (JC[1] * JC[1] + JC[3] * JC[3]));
            const double inv = 1.0 / nJ_C;
            const double r = C * inv;
            const double s = C * inv * inv;
            const double *d1 = v, *d2 = v + 3, *M1 = v + 6, *M2 = v + 12;
            double dF[9], J[NP];
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int rr = 0; rr < 3; ++rr) {
                    double e = d1[c] * d2[rr];
                    e -= s * (JC[0] * M1[2 * c] * d2[rr] + JC[1] * M1[2 * c + 1] * d2[rr] + JC[2] * M2[2 * rr] * d1[c] +
                              JC[3] * M2[2 * rr + 1] * d1[c]);
                    dF[3 * c + rr] = e * inv;
                }
            const double *D = ctx + 9;
#pragma unroll
            for (int p = 0; p < NP; ++p) {
                double t = 0.0;
#pragma unroll
                for (int m = 0; m < 9; ++m) t += dF[m] * D[NP * m + p];
                J[p] = t;
            }
            A.add1(L, r, J);
        } else {
            const double a0 = P.p[0][k], a1 = P.p[1][k], b0 = P.p[2][k], b1 = P.p[3][k];
            {
                const double rr = sampson_res(ctx, a0, a1, b0, b1);
                lsum += L.loss(rr * rr);
                rows += 1.0;
            }
            double r, dF[9], J[NP];
            sampson_res_dF(ctx, a0, a1, b0, b1, r, dF);
            const double *D = ctx + 9;
#pragma unroll
            for (int p = 0; p < NP; ++p) {
                double s = 0.0;
#pragma unroll
                for (int m = 0; m < 9; ++m) s += dF[m] * D[NP * m + p];
                J[p] = s;
            }
            A.add1(L, r, J);
        }
    }
    constexpr int NV = 2 + NT + NP + 1;
    double v[NV];
    v[0] = lsum;
    v[1] = rows;
#pragma unroll
    for (int i = 0; i < NT; ++i) v[2 + i] = A.jtj[i];
#pragma unroll
    for (int i = 0; i < NP; ++i) v[2 + NT + i] = A.jtr[i];
    v[NV - 1] = A.cnt;
    cluster_sum<NV>(S, v, buf, csize);
}

// lower Cholesky solve of (A) x = rhs, only the lower triangle of A read (jacobian_accumulator.h:145-154)
template <int NP> PLB_DEV void llt_solve(const double *A, const double *rhs, double *x) {
    double Lm[NP * NP];
    for (int j = 0; j < NP; ++j) {
        double d = A[j * NP + j];
        for (int k = 0; k < j; ++k) d -= Lm[j * NP + k] * Lm[j * NP + k];
        const double ljj = sqrt(d);
        Lm[j * NP + j] = ljj;
        for (int i = j + 1; i < NP; ++i) {
            double s = A[i * NP + j];
            for (int k = 0; k < j; ++k) s -= Lm[i * NP + k] * Lm[j * NP + k];
            Lm[i * NP + j] = s / ljj;
        }
    }
    double y[NP];
    for (int i = 0; i < NP; ++i) {
        double s = rhs[i];
        for (int k = 0; k < i; ++k) s -= Lm[i * NP + k] * y[k];
        y[i] = s / Lm[i * NP + i];
    }
    for (int i = NP - 1; i >= 0; --i) {
        double s = y[i];
        for (int k = i + 1; k < NP; ++k) s -= Lm[k * NP + i] * x[k];
        x[i] = s / Lm[i * NP + i];
    }
}

// One thread-block CLUSTER per job (1..8 CTAs of 256 threads, DSMEM reductions); CTA r owns the correspondences
// [r*chunk, (r+1)*chunk).  Every CTA runs the scalar LM logic (optim/lm_impl.h:56-140) redundantly on identical
// cluster totals, so no broadcast between CTAs is needed.  The reference evaluates the residual of a trial step and,
// if accepted, the Jacobian at the same parameters in a second pass; here both come from one pass.
template <int KIND, int MINB>
__global__ void __launch_bounds__(LM_THREADS / MINB, MINB)
    k_lm(const ProblemDev *__restrict__ probs, const LmJob *__restrict__ jobs, const LoJobSrc *__restrict__ job_src,
         const double *__restrict__ models_in, const int *__restrict__ n_jobs_dev, int n_jobs, const char *mask_base,
         int *idx_scratch, int scratch_stride, LmJobOut *outs) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    constexpr int NP = LmDims<KIND>::NP;
    constexpr int NT = NP * (NP + 1) / 2;
    constexpr int MSZ = kind_model_size(KIND);
    __shared__ LmShared S;
    const int csize = (int)cluster.num_blocks(), crank = (int)cluster.block_rank();
    // The grid is a set of clusters that walk the job list: explicit jobs (jobs[j], model j of models_in, stride 9) or
    // the LO jobs k_pass1 listed on the device (template jobs[job_src[j].pidx], model slot job_src[j].slot of the
    // round's model list, stride MSZ; the count is read from device memory and clamped to n_jobs).
    const int n_clusters = (int)gridDim.x / csize, cluster_id = (int)blockIdx.x / csize;
    int nj = n_jobs;
    if (n_jobs_dev) {
        const int v = *n_jobs_dev;
        if (v < nj) nj = v;
    }
    int buf = 0;
    for (int job = cluster_id; job < nj; job += n_clusters) {
    const LmJob &J = job_src ? jobs[job_src[job].pidx] : jobs[job];
    const ProblemDev P = probs[J.pidx];
    const LmParams prm = J.prm;
    const char *mask_in = (J.mask_off >= 0) ? mask_base + J.mask_off : nullptr;
    const double *min = job_src ? models_in + (size_t)job_src[job].slot * MSZ : models_in + (size_t)job * 9;
    LmJobOut *out = outs + job;
    LossFn L;
    L.type = prm.loss_type;
    L.thr = prm.loss_scale;
    L.sq_thr = prm.loss_scale * prm.loss_scale;
    L.inv_sq_thr = 1.0 / L.sq_thr;

    // ---- this CTA's slice and its active-point list ------------------------------------------------------------
    const int chunk = (((P.n + csize - 1) / csize) + 31) & ~31;
    const int lo = min_i(crank * chunk, P.n), hi = min_i(lo + chunk, P.n);
    int na = hi - lo;
    const int *list = nullptr;
    bool untouched = false;
    if (prm.subset_mode != 0) {
        int *mylist = idx_scratch + (size_t)cluster_id * (size_t)scratch_stride + lo;
        ModelCtx<KIND_RELPOSE> C;
        if (KIND == KIND_RELPOSE && prm.subset_mode == 1) C.init(min);
        const double *M = reinterpret_cast<const double *>(&C);
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        int base = 0;
        for (int t0 = lo; t0 < hi; t0 += (int)blockDim.x) {
            const int k = t0 + threadIdx.x;
            bool keep = false;
            if (k < hi) {
                if (prm.subset_mode == 2) {
                    keep = mask_in[k] != 0;
                } else if (KIND == KIND_RELPOSE) {
                    // relpose LO subset: inliers of the start pose at 5*thr^2 (estimators/relative_pose.cc:62-86)
                    const double a0 = P.p[0][k], a1 = P.p[1][k], b0 = P.p[2][k], b1 = P.p[3][k];
                    keep = sampson_r2(M, a0, a1, b0, b1) < prm.subset_sq_thr;
                    if (keep) keep = cheirality_ok(M + 9, M + 13, bearing(a0, a1), bearing(b0, b1), 0.01);
                }
            }
            const unsigned bal = __ballot_sync(0xffffffffu, keep);
            if (lane == 0) S.wcount[warp] = __popc(bal);
            __syncthreads();
            int off = base;
            for (int w = 0; w < warp; ++w) off += S.wcount[w];
            int tile = 0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tile += S.wcount[w];
            if (keep) mylist[off + __popc(bal & ((1u << lane) - 1u))] = k;
            base += tile;
            __syncthreads();
        }
        na = base;
        list = mylist;
        __syncthreads();
        if (KIND == KIND_RELPOSE && prm.subset_mode == 1) {
            double c[1] = {threadIdx.x == 0 ? (double)na : 0.0};
            cluster_sum<1>(&S, c, buf, csize);
            untouched = !(S.tot[0] > 5.0);
        }
    }

    // ---- initial parameters
    if (threadIdx.x == 0) {
        if (KIND == KIND_FUND) {
            m3 F, U, V;
#pragma unroll
            for (int k = 0; k < 9; ++k) F.a[3 * (k % 3) + k / 3] = min[k];
            double sv[3];
            svd3_dev(F, U, sv, V);
            if (det3(U) < 0)
                for (int k = 0; k < 9; ++k) U.a[k] = -U.a[k];
            if (det3(V) < 0)
                for (int k = 0; k < 9; ++k) V.a[k] = -V.a[k];
            rot_to_quat(U, S.par);
            rot_to_quat(V, S.par + 4);
            S.par[8] = sv[1] / sv[0];
        } else {
            for (int k = 0; k < MSZ; ++k) S.par[k] = min[k];
            for (int k = MSZ; k < 9; ++k) S.par[k] = 0.0;
        }
    }
    __syncthreads();

    int iterations = 0;
    double cost = 0.0, initial_cost = 0.0;
    if (!untouched) {
        // scalar LM state (thread 0 of every CTA); rc mirrors NormalAccumulator::residual_count
        double lambda = prm.initial_lambda, nu = 2.0, rc = 0.0;
        double JtJ[NP * NP], Jtr[NP], sol[NP];
        bool recompute_jac = true;
        if (threadIdx.x == 0) lm_build_ctx<KIND>(S.par, S.ctx, S.tb, true);
        __syncthreads();
        lm_eval_pass<KIND>(P, prm, L, list, lo, na, &S, buf, csize);
        if (threadIdx.x == 0) {
            cost = S.tot[0] * (1.0 / fmax(1.0, S.tot[1])); // acc.get_residual() after the residual pass
            initial_cost = cost;
            int t = 0;
            for (int i = 0; i < NP; ++i)
                for (int j = 0; j <= i; ++j) JtJ[i * NP + j] = S.tot[2 + t++];
            for (int i = 0; i < NP; ++i) Jtr[i] = S.tot[2 + NT + i];
            rc = S.tot[2 + NT + NP]; // residual_count after the Jacobian pass
        }
        for (int it = 0; it < prm.max_iterations; ++it) {
            iterations = it;
            int stop = 0;
            if (threadIdx.x == 0) {
                if (recompute_jac) {
                    double g = 0.0;
                    for (int i = 0; i < NP; ++i) g += Jtr[i] * Jtr[i];
                    const double grad_norm = (1.0 / fmax(1.0, rc)) * sqrt(g);
                    if (grad_norm < prm.gradient_tol) stop = 1;
                }
                if (!stop) {
                    const double scale = 1.0 / fmax(1.0, rc);
                    double Am[NP * NP], rhs[NP];
                    for (int i = 0; i < NP; ++i)
                        for (int j = 0; j <= i; ++j) Am[i * NP + j] = scale * JtJ[i * NP + j];
                    for (int i = 0; i < NP; ++i) Am[i * NP + i] += lambda;
                    for (int i = 0; i < NP; ++i) rhs[i] = -(scale * Jtr[i]);
                    llt_solve<NP>(Am, rhs, sol);
                    double sn = 0.0;
                    for (int i = 0; i < NP; ++i) sn += sol[i] * sol[i];
                    if (sqrt(sn) < prm.step_tol) stop = 1;
                }
                if (!stop) {
                    lm_step<KIND>(S.par, sol, S.tb, S.par_new);
                    lm_build_ctx<KIND>(S.par_new, S.ctx, S.tb_new, true);
                }
            }
            if (block_bcast(&S, stop)) break;
            lm_eval_pass<KIND>(P, prm, L, list, lo, na, &S, buf, csize);
            int brk = 0;
            if (threadIdx.x == 0) {
                rc = S.tot[1]; // residual_count after the residual pass of the trial point
                const double cost_new = S.tot[0] * (1.0 / fmax(1.0, rc));
                if (cost_new < cost) {
                    const double cost_decrease = cost - cost_new;
                    for (int k = 0; k < 9; ++k) S.par[k] = S.par_new[k];
                    for (int k = 0; k < 6; ++k) S.tb[k] = S.tb_new[k];
                    cost = cost_new;
                    recompute_jac = true;
                    const double scale = 1.0 / fmax(1.0, rc);
                    double pred = 0.0;
                    for (int i = 0; i < NP; ++i) pred += sol[i] * (lambda * sol[i] + scale * Jtr[i]);
                    pred = -pred;
                    if (pred > 0) {
                        const double rho = cost_decrease / pred;
                        const double factor = 1.0 - pow(2.0 * rho - 1.0, 3.0);
                        lambda *= fmax(1.0 / 3.0, factor);
                    } else {
                        lambda *= 1.0 / 3.0;
                    }
                    nu = 2.0;
                    lambda = fmax(prm.min_lambda, lambda);
                    if (cost > 0 && cost_decrease / cost < prm.relative_cost_tol) brk = 1;
                    // the Jacobian pass the reference would run next at the accepted parameters
                    int t = 0;
                    for (int i = 0; i < NP; ++i)
                        for (int j = 0; j <= i; ++j) JtJ[i * NP + j] = S.tot[2 + t++];
                    for (int i = 0; i < NP; ++i) Jtr[i] = S.tot[2 + NT + i];
                    if (!brk && it + 1 < prm.max_iterations) rc = S.tot[2 + NT + NP];
                } else {
                    recompute_jac = false;
                    lambda *= nu;
                    nu *= 2.0;
                    lambda = fmin(prm.max_lambda, lambda);
                }
                if (it + 1 >= prm.max_iterations && !brk) iterations = it + 1;
            }
            if (block_bcast(&S, brk)) break;
        }
    }
    // ---- output (CTA 0 of the cluster)
    __syncthreads();
    if (threadIdx.x == 0) {
        if (KIND == KIND_FUND) {
            if (untouched) {
                for (int k = 0; k < 9; ++k) S.par_new[k] = min[k];
            } else {
                const m3 F = ff_to_F(S.par);
                for (int k = 0; k < 9; ++k) S.par_new[k] = F.a[3 * (k % 3) + k / 3];
            }
        } else {
            for (int k = 0; k < MSZ; ++k) S.par_new[k] = untouched ? min[k] : S.par[k];
            for (int k = MSZ; k < 9; ++k) S.par_new[k] = 0.0;
        }
        if (crank == 0) {
            for (int k = 0; k < 9; ++k) out->model[k] = S.par_new[k];
            out->iterations = iterations;
            out->cost = cost;
            out->initial_cost = initial_cost;
        }
    }
    __syncthreads();
    if (prm.score_after && crank == 0) {
        uint32_t cnt;
        double score;
        double mdl[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) mdl[k] = S.par_new[k];
        cta_score<KIND, LM_THREADS / MINB>(P, mdl, P.sq_thr, &S.sred, cnt, score);
        if (threadIdx.x == 0) {
            out->count = cnt;
            out->score = score;
        }
    }
    cluster.sync(); // no CTA may exit (or start the next job) while a sibling can still read its shared memory
    } // jobs of this cluster
}

// CTAs of k_lm per SM.  k_lm needs ~255 registers per thread.  1: 256 threads, one CTA (one job, or one slice of a job's
// cluster) per SM.  2 (PLB_LM_MINB=2): 128 threads per CTA, still 255 registers, two CTAs per SM — every job gets half the
// threads but twice as many jobs are in flight; the LM passes are latency bound (few correspondences per thread, a
// cluster-wide reduction and a scalar solve per iteration).
static int lm_minb() {
    static const int minb = [] {
        const char *e = std::getenv("PLB_LM_MINB");
        return (e && std::atoi(e) == 2) ? 2 : 1;
    }();
    return minb;
}
static thread_local int t_lm_sm_share = 50;
void lm_set_sm_share(int pct) { t_lm_sm_share = (pct > 0 && pct <= 100) ? pct : 50; }
static int lm_cluster_size(int n_jobs, int max_n) {
    static const int per_cta = [] { // correspondences per CTA before another CTA of the cluster pays off
        const char *e = std::getenv("PLB_LM_PER_CTA");
        const int v = e ? std::atoi(e) : 0;
        return v > 0 ? v : 2048;
    }();
    int csize = (max_n + per_cta - 1) / per_cta;
    if (csize < 1) csize = 1;
    if (csize > LM_MAX_CLUSTER) csize = LM_MAX_CLUSTER;
    if (csize > 4 && csize < 8) csize = 4;
    if (csize == 3) csize = 2;
    // k_lm needs the whole register file of an SM per CTA: with many jobs in one launch (batch groups) wide clusters
    // only take SMs away from the co-running hypothesis kernels, so the cluster shrinks as the job count grows
    // SMs (percent of the device) the LO clusters of one launch may cover: half when other lock-step groups share the GPU
    // (their hypothesis kernels want the other half: +5 % on the batch workload), all of it for a call that runs alone
    // (C4 single call 2.7 -> 2.2 ms).  PLB_LM_SM_PCT overrides.
    static const int forced = [] {
        const char *e = std::getenv("PLB_LM_SM_PCT");
        const int v = e ? std::atoi(e) : 0;
        return (v > 0 && v <= 100) ? v : 0;
    }();
    const int sm_share = forced ? forced : t_lm_sm_share;
    while (csize > 1 && n_jobs * csize > sm_count() * sm_share / 100) csize /= 2;
    return csize;
}
template <int KIND>
static void launch_lm_t(const ProblemDev *probs, const LmJob *jobs, const LoJobSrc *job_src, const double *models_in,
                        const int *n_jobs_dev, int n_jobs, int n_clusters, int csize, const char *mask_base,
                        int *idx_scratch, int scratch_stride, LmJobOut *out, cudaStream_t stream) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)(n_clusters * csize), 1, 1);
    cfg.blockDim = dim3((unsigned)(LM_THREADS / lm_minb()), 1, 1);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)csize;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (lm_minb() == 2)
        cudaLaunchKernelEx(&cfg, k_lm<KIND, 2>, probs, jobs, job_src, models_in, n_jobs_dev, n_jobs, mask_base, idx_scratch,
                           scratch_stride, out);
    else
        cudaLaunchKernelEx(&cfg, k_lm<KIND, 1>, probs, jobs, job_src, models_in, n_jobs_dev, n_jobs, mask_base, idx_scratch,
                           scratch_stride, out);
}
static void launch_lm_any(int kind, const ProblemDev *probs, const LmJob *jobs, const LoJobSrc *job_src,
                          const double *models_in, const int *n_jobs_dev, int n_jobs, int n_clusters, int csize,
                          const char *mask_base, int *idx_scratch, int scratch_stride, LmJobOut *out, cudaStream_t stream) {
    switch (kind) {
    case KIND_PNP: launch_lm_t<KIND_PNP>(probs, jobs, job_src, models_in, n_jobs_dev, n_jobs, n_clusters, csize, mask_base, idx_scratch, scratch_stride, out, stream); break;
    case KIND_RELPOSE: launch_lm_t<KIND_RELPOSE>(probs, jobs, job_src, models_in, n_jobs_dev, n_jobs, n_clusters, csize, mask_base, idx_scratch, scratch_stride, out, stream); break;
    case KIND_FUND: launch_lm_t<KIND_FUND>(probs, jobs, job_src, models_in, n_jobs_dev, n_jobs, n_clusters, csize, mask_base, idx_scratch, scratch_stride, out, stream); break;
    case KIND_RELPOSE_TS: launch_lm_t<KIND_RELPOSE_TS>(probs, jobs, job_src, models_in, n_jobs_dev, n_jobs, n_clusters, csize, mask_base, idx_scratch, scratch_stride, out, stream); break;
    default: launch_lm_t<KIND_HOMOG>(probs, jobs, job_src, models_in, n_jobs_dev, n_jobs, n_clusters, csize, mask_base, idx_scratch, scratch_stride, out, stream); break;
    }
}
void launch_lm(int kind, const ProblemDev *probs, const LmJob *jobs_dev, const double *models_in, int n_jobs,
               int max_n, const char *mask_base, int *idx_scratch, int scratch_stride, LmJobOut *out, cudaStream_t stream) {
    if (n_jobs <= 0) return;
    const int csize = lm_cluster_size(n_jobs, max_n);
    launch_lm_any(kind, probs, jobs_dev, nullptr, models_in, nullptr, n_jobs, n_jobs, csize, mask_base, idx_scratch,
                  scratch_stride, out, stream);
}
// Clusters of a round's LO launch: at most one wave (a k_lm CTA owns an SM), at most the estimated number of jobs.
int lm_round_max_clusters(int kind, int est_jobs, int max_n) {
    (void)kind;
    if (est_jobs < 1) est_jobs = 1;
    const int csize = lm_cluster_size(est_jobs, max_n);
    int nc = lm_minb() * sm_count() / csize;
    if (nc > est_jobs) nc = est_jobs;
    return nc < 1 ? 1 : nc;
}
void launch_lm_round(int kind, const ProblemDev *probs, const LmJob *tmpl, const LoJobSrc *job_src,
                     const double *models, const int *n_jobs_dev, int job_cap, int est_jobs, int max_n,
                     int *idx_scratch, int scratch_stride, LmJobOut *out, cudaStream_t stream) {
    if (est_jobs < 1) est_jobs = 1;
    const int csize = lm_cluster_size(est_jobs, max_n);
    const int nc = lm_round_max_clusters(kind, est_jobs, max_n);
    launch_lm_any(kind, probs, tmpl, job_src, models, n_jobs_dev, job_cap, nc, csize, nullptr, idx_scratch, scratch_stride,
                  out, stream);
}

// ============================================================================================================
// relpose_8pt / essential_matrix_8pt (solvers/relpose_8pt.cc:52-95): non-minimal essential matrix from n >= 8 bearings
// ============================================================================================================
// One warp per instance.  Row i of the n x 9 system is [x2.x x1^T, x2.y x1^T, x2.z x1^T] (:41-49).
//   n == 8: last column of the Householder Q of the transposed system (:63-67), no pivoting (lane 0, 9x8).
//   n  > 8: eigenvector of the smallest eigenvalue of A^T A (:68-72).  Lane <-> entry (p, q) of the Gram matrix, every
//           lane sums ITS entry over the correspondences in order (the summation order of a sequential loop); then a
//           cyclic Jacobi eigen-iteration on lane 0 (Eigen's SelfAdjointEigenSolver is iterative too: parity to tolerance).
// Then the closest essential matrix in Frobenius norm, singular values (a, b, c) -> ((a+b)/2, (a+b)/2, 0) (:74-81), and
// for the pose variant motion_from_essential with the cheirality test on ALL n correspondences (misc/essential.cc:103-169).
struct EightScratch {
    double G[81];
    double V[81];
    double e[9];
    double E[9];
};
PLB_DEV void sym_eigen_jacobi9(double *A /*9x9 row-major, symmetric, destroyed*/, double *V /*column c at V[9c..]*/, double *e_min) {
    constexpr int N = 9;
    for (int c = 0; c < N; ++c)
        for (int r = 0; r < N; ++r) V[c * N + r] = (r == c) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 100; ++sweep) {
        double off = 0.0, diag = 0.0;
        for (int i = 0; i < N; ++i) {
            diag += A[i * N + i] * A[i * N + i];
            for (int j = i + 1; j < N; ++j) off += A[i * N + j] * A[i * N + j];
        }
        if (off <= 1e-32 * diag || off == 0.0) break;
        for (int p = 0; p < N - 1; ++p)
            for (int q = p + 1; q < N; ++q) {
                if (A[p * N + q] == 0.0) continue;
                const double theta = (A[q * N + q] - A[p * N + p]) / (2.0 * A[p * N + q]);
                const double t = ((theta >= 0) ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
                for (int k = 0; k < N; ++k) { // A <- A J
                    const double akp = A[k * N + p], akq = A[k * N + q];
                    A[k * N + p] = c * akp - sn * akq;
                    A[k * N + q] = sn * akp + c * akq;
                }
                for (int k = 0; k < N; ++k) { // A <- J^T A
                    const double apk = A[p * N + k], aqk = A[q * N + k];
                    A[p * N + k] = c * apk - sn * aqk;
                    A[q * N + k] = sn * apk + c * aqk;
                }
                for (int k = 0; k < N; ++k) {
                    const double vkp = V[p * N + k], vkq = V[q * N + k];
                    V[p * N + k] = c * vkp - sn * vkq;
                    V[q * N + k] = sn * vkp + c * vkq;
                }
            }
    }
    int best = 0; // first index of the smallest eigenvalue (ascending sort keeps the first of equal values in front)
    for (int i = 1; i < N; ++i)
        if (A[i * N + i] < A[best * N + best]) best = i;
    for (int r = 0; r < N; ++r) e_min[r] = V[best * N + r];
}
// householderQr().householderQ().col(8) of the 9 x 8 matrix whose column i is row i of the system (column-major a[c*9+r])
PLB_DEV void householder_lastcol_9x8(double *a, double *q8) {
    constexpr int ROWS = 9, COLS = 8;
    double hc[COLS];
    for (int k = 0; k < COLS; ++k) {
        double tail_sq = 0.0;
        for (int r = k + 1; r < ROWS; ++r) tail_sq += a[k * ROWS + r] * a[k * ROWS + r];
        const double c0 = a[k * ROWS + k];
        double tau, beta;
        if (tail_sq <= 2.2250738585072014e-308) {
            tau = 0.0;
            beta = c0;
            for (int r = k + 1; r < ROWS; ++r) a[k * ROWS + r] = 0.0;
        } else {
            beta = sqrt(c0 * c0 + tail_sq);
            if (c0 >= 0) beta = -beta;
            for (int r = k + 1; r < ROWS; ++r) a[k * ROWS + r] = a[k * ROWS + r] / (c0 - beta);
            tau = (beta - c0) / beta;
        }
        hc[k] = tau;
        a[k * ROWS + k] = beta;
        if (tau != 0.0) {
            for (int c = k + 1; c < COLS; ++c) {
                double tmp = 0.0;
                for (int r = k + 1; r < ROWS; ++r) tmp += a[k * ROWS + r] * a[c * ROWS + r];
                tmp += a[c * ROWS + k];
                a[c * ROWS + k] -= tau * tmp;
                for (int r = k + 1; r < ROWS; ++r) a[c * ROWS + r] -= tau * a[k * ROWS + r] * tmp;
            }
        }
    }
    for (int r = 0; r < ROWS; ++r) q8[r] = (r == 8) ? 1.0 : 0.0;
    for (int k = COLS - 1; k >= 0; --k) {
        const double tau = hc[k];
        if (tau == 0.0) continue;
        double tmp = 0.0;
        for (int r = k + 1; r < ROWS; ++r) tmp += a[k * ROWS + r] * q8[r];
        tmp += q8[k];
        q8[k] -= tau * tmp;
        for (int r = k + 1; r < ROWS; ++r) q8[r] -= tau * a[k * ROWS + r] * tmp;
    }
}
// want_poses == 0: E_out (count x 9, COLUMN-major like Eigen::Matrix3d); else poses_out (count x 4 x 7) + n_out.
__global__ void __launch_bounds__(128) k_eightpt(size_t count, int n, const double *__restrict__ x1, const double *__restrict__ x2,
                                                 int want_poses, double *E_out, double *poses_out, int *n_out) {
    __shared__ EightScratch scratch[4];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const size_t inst = (size_t)blockIdx.x * 4 + w;
    if (inst >= count) return;
    EightScratch &S = scratch[w];
    const double *a = x1 + inst * (size_t)n * 3, *b = x2 + inst * (size_t)n * 3;
    if (n == 8) {
        if (lane == 0) {
            double At[72];
            for (int i = 0; i < 8; ++i)
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 3; ++c) At[9 * i + 3 * r + c] = b[3 * i + r] * a[3 * i + c];
            householder_lastcol_9x8(At, S.e);
        }
    } else {
        for (int ent = lane; ent < 81; ent += 32) {
            const int p = ent / 9, q = ent % 9;
            double s = 0.0;
            for (int i = 0; i < n; ++i) {
                const double rp = b[3 * i + p / 3] * a[3 * i + p % 3], rq = b[3 * i + q / 3] * a[3 * i + q % 3];
                s = (i == 0) ? rp * rq : s + rp * rq;
            }
            S.G[ent] = s;
        }
        __syncwarp();
        if (lane == 0) {
            for (int i = 0; i < 9; ++i) // the solver reads the lower triangle
                for (int j = i + 1; j < 9; ++j) S.G[i * 9 + j] = S.G[j * 9 + i];
            sym_eigen_jacobi9(S.G, S.V, S.e);
        }
    }
    __syncwarp();
    if (lane == 0) {
        m3 E, U, V;
        for (int k = 0; k < 9; ++k) E.a[k] = S.e[k]; // Map<const RowMajor 3x3>
        double d[3];
        svd3_dev(E, U, d, V);
        const double m = (d[0] + d[1]) / 2.;
        m3 UD;
        for (int r = 0; r < 3; ++r) {
            UD(r, 0) = U(r, 0) * m;
            UD(r, 1) = U(r, 1) * m;
            UD(r, 2) = U(r, 2) * 0.0;
        }
        m3 Vt;
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) Vt(r, c) = V(c, r);
        const m3 Ef = mmul(UD, Vt);
        for (int k = 0; k < 9; ++k) S.E[k] = Ef.a[k];
        if (!want_poses) {
            for (int k = 0; k < 9; ++k) E_out[inst * 9 + k] = Ef.a[3 * (k % 3) + k / 3];
        } else {
            double cand[4][7];
            const unsigned mask = motions_from_E(S.E, a, b, n, cand);
            int cnt = 0;
            for (int c = 0; c < 4; ++c)
                if (mask & (1u << c)) {
                    for (int k = 0; k < 7; ++k) poses_out[(inst * 4 + cnt) * 7 + k] = cand[c][k];
                    ++cnt;
                }
            n_out[inst] = cnt;
        }
    }
}
void launch_eightpt(size_t count, int n, const double *x1, const double *x2, int want_poses, double *E_out, double *poses_out,
                    int *n_out, cudaStream_t stream) {
    if (count == 0) return;
    k_eightpt<<<(unsigned)((count + 3) / 4), 128, 0, stream>>>(count, n, x1, x2, want_poses, E_out, poses_out, n_out);
}

// ============================================================================================================
// direct solver surface: one warp per instance
// ============================================================================================================
// variant: 0 = native output (p3p poses / 5pt E / 7pt F / H), 1 = 5pt poses / p3p_lambdatwist
template <int KIND, int VARIANT>
__global__ void __launch_bounds__(HYP_WARPS * 32)
    k_solver_batch(size_t count, const double *__restrict__ a, const double *__restrict__ b, double *out, int *n_out,
                   int flags) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MonoTables *T = reinterpret_cast<MonoTables *>(smem_raw);
    HypScratch<KIND> *W = reinterpret_cast<HypScratch<KIND> *>(smem_raw + 256) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (KIND == KIND_RELPOSE) {
        fill_tables(T);
        __syncthreads();
    }
    const size_t gw = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t i = gw; i < count; i += nw) {
        if (KIND == KIND_PNP) {
            d3 xs[3], Xs[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                xs[k] = mk(a[9 * i + 3 * k], a[9 * i + 3 * k + 1], a[9 * i + 3 * k + 2]);
                Xs[k] = mk(b[9 * i + 3 * k], b[9 * i + 3 * k + 1], b[9 * i + 3 * k + 2]);
            }
            double *models = reinterpret_cast<double *>(W);
            const int n = (VARIANT == 1) ? solve_p3p_lambdatwist(xs, Xs, models, lane) : solve_p3p(xs, Xs, models, lane);
            if (lane < 28) out[28 * i + lane] = (lane < 7 * n) ? models[lane] : 0.0;
            if (lane == 0) n_out[i] = n;
        } else if (KIND == KIND_HOMOG) {
            d3 xa[4], xb[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                xa[k] = mk(a[12 * i + 3 * k], a[12 * i + 3 * k + 1], a[12 * i + 3 * k + 2]);
                xb[k] = mk(b[12 * i + 3 * k], b[12 * i + 3 * k + 1], b[12 * i + 3 * k + 2]);
            }
            double *models = reinterpret_cast<double *>(W);
            const int n = solve_h4(xa, xb, models, lane, flags != 0);
            if (lane < 9) out[9 * i + lane] = n ? models[lane] : 0.0;
            if (lane == 0) n_out[i] = n;
        } else if (KIND == KIND_RELPOSE) {
            HypScratch<KIND_RELPOSE> *S = reinterpret_cast<HypScratch<KIND_RELPOSE> *>(W);
            if (lane < 30) S->xs[lane] = (lane < 15) ? a[15 * i + lane] : b[15 * i + lane - 15];
            __syncwarp();
            if (VARIANT == 0) {
                const int n = solve_5pt_E(S->xs, S->xs + 15, &S->s5, T, lane);
                for (int e = lane; e < 90; e += 32) {
                    const int m = e / 9, k = e % 9; // output column-major
                    out[90 * i + e] = (m < n) ? S->s5.Es[9 * m + 3 * (k % 3) + k / 3] : 0.0;
                }
                if (lane == 0) n_out[i] = n;
            } else {
                const int n = solve_5pt_poses(S->xs, S->xs + 15, &S->s5, T, S->models, lane);
                for (int e = lane; e < 280; e += 32) out[280 * i + e] = (e < 7 * n) ? S->models[e] : 0.0;
                if (lane == 0) n_out[i] = n;
            }
        } else {
            HypScratch<KIND_FUND> *S = reinterpret_cast<HypScratch<KIND_FUND> *>(W);
            for (int e = lane; e < 42; e += 32) S->xs[e] = (e < 21) ? a[21 * i + e] : b[21 * i + e - 21];
            __syncwarp();
            const int n = solve_7pt(S->xs, S->xs + 21, &S->s7, S->models, lane);
            if (lane < 27) out[27 * i + lane] = (lane < 9 * n) ? S->models[lane] : 0.0;
            if (lane == 0) n_out[i] = n;
        }
        __syncwarp();
    }
}

template <int KIND, int VARIANT>
static void launch_solver_t(size_t count, const double *a, const double *b, double *out, int *n_out, int flags,
                            cudaStream_t stream) {
    const size_t smem = hyp_smem_bytes<KIND>();
    cudaFuncSetAttribute(k_solver_batch<KIND, VARIANT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    size_t blocks = (count + HYP_WARPS - 1) / HYP_WARPS;
    const size_t cap = (size_t)sm_count() * 4;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    k_solver_batch<KIND, VARIANT><<<(unsigned)blocks, HYP_WARPS * 32, smem, stream>>>(count, a, b, out, n_out, flags);
}
void launch_solver_batch(int kind, int variant, size_t count, const double *a, const double *b, double *out,
                         int *n_out, int flags, cudaStream_t stream) {
    if (count == 0) return;
    switch (kind) {
    case KIND_PNP:
        if (variant == 0) launch_solver_t<KIND_PNP, 0>(count, a, b, out, n_out, flags, stream);
        else launch_solver_t<KIND_PNP, 1>(count, a, b, out, n_out, flags, stream);
        break;
    case KIND_RELPOSE:
        if (variant == 0) launch_solver_t<KIND_RELPOSE, 0>(count, a, b, out, n_out, flags, stream);
        else launch_solver_t<KIND_RELPOSE, 1>(count, a, b, out, n_out, flags, stream);
        break;
    case KIND_FUND: launch_solver_t<KIND_FUND, 0>(count, a, b, out, n_out, flags, stream); break;
    default: launch_solver_t<KIND_HOMOG, 0>(count, a, b, out, n_out, flags, stream); break;
    }
}

} // namespace plb
