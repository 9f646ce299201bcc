// poselib_b200 — CUDA kernels of the LO-RANSAC hot path for sm_90a (H100).
//
//   k_ingest           device-resident caller arrays (fp32 / fp64) -> the engine's fp64 AoS input buffer
//   k_transpose        caller AoS doubles -> SoA fp64 (+ fp32 copy) in HBM, coalesced both ways
//   k_solve_lane<KIND> / k7_solve_lane / k5_gather -> k5_null -> k5_elim -> k5_roots -> k5_back
//                      minimal solvers of a round, one thread per minimal sample (the 5-point solver in phases)
//   k_score_tiled / k_screen
//                      MSAC scoring of every model of a round over all correspondences (exact fp64 / fp32 screening)
//   k_score            exact scoring (and masks) of explicit models: initial models, plb_score_batch
//   k_confirm          exact rescoring of the fast-mode candidates of a round
//   k_lm<KIND, CAM>    Levenberg-Marquardt refit (LO step + final polish): one cluster per job, cluster-wide reductions
//                      of the normal equations, scalar LM logic on thread 0; CAM refines PnP camera parameters too
//   k_inlier_mask      final inlier masks (k_scatter_masks: into the callers' device buffers)
//   Every exact score (k_score_tiled, k_score, k_confirm, the rescoring in k_lm) comes from one routine, msac_score,
//   and every fp64 inlier decision (those, k_inlier_mask, the LO subset in k_lm) from one test per kind, under_thr
//   (+ cheirality for the relpose kinds); the PnP mask alone keeps the reference's own formula.
//   k_solver_batch     the solvers/*.h surface: one thread per instance (relpose_5pt: k5_load -> k5_null -> k5_elim
//                      -> k5_roots -> k5_solver_out)
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
// bounds: the setups then set scr::REC_ERR0 = +inf and every model of such a problem is rescored exactly).
PLB_DEV void coord_max(float *cmax, int c, double v) {
    if (!cmax) return;
    const unsigned bits = __float_as_uint(scr::f_up(fabs(v)));
    const unsigned m = __reduce_max_sync(0xffffffffu, bits);
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned *>(cmax) + c, m);
}
// X: some camera of the launch is a fisheye or division model (camera.cuh)
template <bool X> __global__ void k_transpose(const TransposeDesc *__restrict__ descs) {
    const TransposeDesc &d = descs[blockIdx.y];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= d.n_pad) return;
    const int idx = (k < d.n) ? k : (d.n - 1); // pad by repeating the last point (never read by the kernels)
    double a0 = d.a[2 * (size_t)idx], a1 = d.a[2 * (size_t)idx + 1];
    if (d.px) { // before mode 1 unprojects a0, a1 in place
        d.px[k] = a0 * d.px_scale;
        d.px[(size_t)d.n_pad + k] = a1 * d.px_scale;
        if (d.b_dim == 2) {
            d.px[2 * (size_t)d.n_pad + k] = d.b[2 * (size_t)idx] * d.px_scale;
            d.px[3 * (size_t)d.n_pad + k] = d.b[2 * (size_t)idx + 1] * d.px_scale;
        }
    }
    if (d.mode == 2) {
        // tangent-Sampson pre-step: scaled pixels -> unit bearing + unprojection Jacobian of both images
        double v[9];
        cam_unproject_with_jac<X>(d.cam_a, a0 * d.scale, a1 * d.scale, v, v + 3);
#pragma unroll
        for (int j = 0; j < 3; ++j) d.s64[(size_t)j * d.n_pad + k] = v[j];
#pragma unroll
        for (int j = 0; j < 6; ++j) d.s64[(size_t)(6 + j) * d.n_pad + k] = v[3 + j];
        const double b0 = d.b[2 * (size_t)idx], b1 = d.b[2 * (size_t)idx + 1];
        cam_unproject_with_jac<X>(d.cam_b, b0 * d.scale, b1 * d.scale, v, v + 3);
#pragma unroll
        for (int j = 0; j < 3; ++j) d.s64[(size_t)(3 + j) * d.n_pad + k] = v[j];
#pragma unroll
        for (int j = 0; j < 6; ++j) d.s64[(size_t)(12 + j) * d.n_pad + k] = v[3 + j];
        return;
    }
    if (d.mode == 1) cam_unproject2<X>(d.cam_a, a0, a1, a0, a1);
    if (d.mode == 1 && d.b_dim == 2) {
        double b0, b1;
        cam_unproject2<X>(d.cam_b, d.b[2 * (size_t)idx], d.b[2 * (size_t)idx + 1], b0, b1);
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
// The integer rows of the Sampson kinds' streaming test (screen_math.cuh), once per problem; zero rows in [n, n_pad).
__global__ void k_qrows(const TransposeDesc *__restrict__ descs) {
    const TransposeDesc &d = descs[blockIdx.y];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (!d.q || k >= d.n_pad) return;
    uint32_t w[4] = {0u, 0u, 0u, 0u};
    if (k < d.n) {
        int e[8];
        scr::sampson_qscale(d.cmax, e);
        float f[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = ldexpf(1.f, 15 - e[j]);
        const float *s = d.s32;
        scr::sampson_qrow(s[k], s[(size_t)d.n_pad + k], s[2 * (size_t)d.n_pad + k], s[3 * (size_t)d.n_pad + k], f, w);
    }
    d.q[k] = make_uint4(w[0], w[1], w[2], w[3]);
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
// Device-resident inputs (plb_estimate_batch_device, plb_refine_batch_device) -> the fp64 AoS the host path would have
// uploaded (a, b, then the weights), one problem per blockIdx.y.  fp32 -> fp64 is exact, so everything downstream sees
// the values the host path sees for the widened input.  The copy also keeps the caller's arrays read-only: k_normalize
// works in place on the engine's buffer.
constexpr int INGEST_THREADS = 256, INGEST_MAX_BLOCKS = 512;
__global__ void __launch_bounds__(INGEST_THREADS) k_ingest(const IngestDesc *__restrict__ descs) {
    const IngestDesc d = descs[blockIdx.y];
    const size_t na = 2 * (size_t)d.n, nb = na + (size_t)d.b_dim * d.n, total = nb + (d.w ? (size_t)d.n : 0);
    for (size_t i = (size_t)blockIdx.x * INGEST_THREADS + threadIdx.x; i < total; i += (size_t)gridDim.x * INGEST_THREADS) {
        const size_t j = i < na ? i : i < nb ? i - na : i - nb;
        const void *src = i < na ? d.a : i < nb ? d.b : d.w;
        d.dst[i] = d.f32 ? (double)static_cast<const float *>(src)[j] : static_cast<const double *>(src)[j];
    }
}
void launch_ingest(const IngestDesc *descs_dev, int n_desc, size_t max_vals, cudaStream_t stream) {
    if (n_desc <= 0 || max_vals == 0) return;
    const unsigned bx = (unsigned)std::min<size_t>((max_vals + INGEST_THREADS - 1) / INGEST_THREADS, INGEST_MAX_BLOCKS);
    k_ingest<<<dim3(bx, n_desc, 1), INGEST_THREADS, 0, stream>>>(descs_dev);
}
// Final masks into the callers' device buffers (plb_estimate_batch_device), one problem per blockIdx.y: the 0 / 1 bytes
// the host path expands from the packed bits.
__global__ void __launch_bounds__(INGEST_THREADS) k_scatter_masks(const char *__restrict__ mask,
                                                                  const ScatterDesc *__restrict__ descs) {
    const ScatterDesc d = descs[blockIdx.y];
    const char *src = mask + d.mask_off;
    for (int k = blockIdx.x * INGEST_THREADS + threadIdx.x; k < d.n; k += gridDim.x * INGEST_THREADS)
        d.dst[k] = src[k] != 0 ? 1 : 0;
}
void launch_scatter_masks(const char *mask, const ScatterDesc *descs_dev, int n_desc, int max_n, cudaStream_t stream) {
    if (n_desc <= 0 || max_n <= 0) return;
    const unsigned bx = (unsigned)std::min((max_n + INGEST_THREADS - 1) / INGEST_THREADS, INGEST_MAX_BLOCKS);
    k_scatter_masks<<<dim3(bx, n_desc, 1), INGEST_THREADS, 0, stream>>>(mask, descs_dev);
}
void launch_normalize(const NormDesc *descs_dev, int n_desc, cudaStream_t stream) {
    if (n_desc <= 0) return;
    k_normalize<<<n_desc, NORM_THREADS, 0, stream>>>(descs_dev);
}
void launch_qrows(const TransposeDesc *descs_dev, int n_desc, int max_n_pad, cudaStream_t stream) {
    if (n_desc <= 0) return;
    k_qrows<<<dim3((max_n_pad + 255) / 256, n_desc, 1), 256, 0, stream>>>(descs_dev);
}
void launch_transpose(const TransposeDesc *descs_dev, int n_desc, int max_n_pad, bool xcam, cudaStream_t stream) {
    if (n_desc <= 0) return;
    const int threads = 256;
    dim3 grid((max_n_pad + threads - 1) / threads, n_desc, 1);
    if (xcam)
        k_transpose<true><<<grid, threads, 0, stream>>>(descs_dev);
    else
        k_transpose<false><<<grid, threads, 0, stream>>>(descs_dev);
}

// ============================================================================================================
// exact fp64 inlier test and MSAC scoring
// ============================================================================================================
// The model context: the per-model constants of the inlier test, row-major doubles.
//   PnP              [R | t] as a 3x4 matrix
//   relpose kinds    E = [t]x R, then q at 9..12 and t at 13..15 (cheirality)
//   F / H            the column-major model transposed
constexpr __host__ __device__ int kind_ctx_size(int kind) { return kind == KIND_PNP ? 12 : kind_is_relpose(kind) ? 16 : 9; }
constexpr int CTX_MAX = 16;
template <int KIND> PLB_DEV void model_ctx(const double *m, double *ctx) {
    if constexpr (KIND == KIND_PNP) {
        const m3 R = quat_to_rot(m);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            ctx[4 * r + 0] = R(r, 0); ctx[4 * r + 1] = R(r, 1); ctx[4 * r + 2] = R(r, 2); ctx[4 * r + 3] = m[4 + r];
        }
    } else if constexpr (kind_is_relpose(KIND)) {
        const m3 E = essential_from_pose(m, m + 4);
#pragma unroll
        for (int i = 0; i < 9; ++i) ctx[i] = E.a[i];
#pragma unroll
        for (int i = 0; i < 7; ++i) ctx[9 + i] = m[i];
    } else {
#pragma unroll
        for (int k = 0; k < 9; ++k) ctx[3 * (k % 3) + k / 3] = m[k];
    }
}

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

// One correspondence as the inlier test reads it: x.x x.y X.x X.y X.z (PnP), x1.x x1.y x2.x x2.y (relpose, F, H) or
// the 18 tangent-Sampson values.
constexpr __host__ __device__ int kind_corr_size(int kind) { return kind == KIND_PNP ? 5 : kind == KIND_RELPOSE_TS ? TS_ARRAYS : 4; }
template <int KIND> PLB_DEV void load_corr(const ProblemDev &P, int k, double *v) {
    if constexpr (KIND == KIND_RELPOSE_TS) {
        load_ts(P, k, v);
    } else {
#pragma unroll
        for (int j = 0; j < kind_corr_size(KIND); ++j) v[j] = P.p[j][k];
    }
}
// The fp64 inlier test, split so that a tile of models can share one load of the correspondence and one computation
// of its bearings.  under_thr: r2 of correspondence v under model context C, and r2 < sq_thr.
//   PnP              reprojection error, points with z2 <= 0 skipped (robust/utils.cc:36-63)
//   relpose, F       Sampson error (robust/utils.cc:158-201, 204-239)
//   tangent Sampson  robust/utils.cc:269-298
//   H                one-way transfer error (robust/utils.cc:300-329)
template <int KIND> PLB_DEV bool under_thr(const double *C, const double *v, double sq_thr, double &r2) {
    if constexpr (KIND == KIND_PNP) {
        const double z0 = C[0] * v[2] + C[1] * v[3] + C[2] * v[4] + C[3];
        const double z1 = C[4] * v[2] + C[5] * v[3] + C[6] * v[4] + C[7];
        const double z2 = C[8] * v[2] + C[9] * v[3] + C[10] * v[4] + C[11];
        if (z2 <= 0.0) return false;
        const double inv_z2 = 1.0 / z2;
        const double r_0 = z0 * inv_z2 - v[0];
        const double r_1 = z1 * inv_z2 - v[1];
        r2 = r_0 * r_0 + r_1 * r_1;
    } else if constexpr (KIND == KIND_RELPOSE_TS) {
        r2 = tangent_r2(C, v);
    } else if constexpr (KIND == KIND_HOMOG) {
        r2 = homography_r2(C, v[0], v[1], v[2], v[3]);
    } else {
        r2 = sampson_r2(C, v[0], v[1], v[2], v[3]);
    }
    return r2 < sq_thr;
}
// Relpose kinds: cheirality, tested only for correspondences under the threshold (robust/utils.cc:187-197), on the unit
// bearings of the correspondence.
template <int KIND> PLB_DEV void corr_bearings(const double *v, d3 &b1, d3 &b2) {
    if constexpr (KIND == KIND_RELPOSE_TS) {
        b1 = mk(v[0], v[1], v[2]);
        b2 = mk(v[3], v[4], v[5]);
    } else {
        b1 = bearing(v[0], v[1]);
        b2 = bearing(v[2], v[3]);
    }
}
PLB_DEV bool cheirality_ctx(const double *C, d3 b1, d3 b2) { return cheirality_ok(C + 9, C + 13, b1, b2, 0.01); }
// The PnP mask keeps its own formula on purpose (DESIGN.md §3): the reference's get_inliers (robust/utils.cc:374-383)
// divides, r2 = |Z.hnormalized() - x|^2 with Z = R*X + t, and tests Z(2) > 0 after the threshold, while its scorer
// (under_thr) multiplies by 1/z2 and skips z2 <= 0 first.  The two give different bits.  C: the PnP model context;
// v(j): value j of the correspondence as load_corr lays it out (x.x x.y X.x X.y X.z).
template <class V> PLB_DEV bool pnp_get_inlier(const double *C, V v, double sq_thr) {
    const double X0 = v(2), X1 = v(3), X2 = v(4);
    const double z0 = C[0] * X0 + C[1] * X1 + C[2] * X2 + C[3];
    const double z1 = C[4] * X0 + C[5] * X1 + C[6] * X2 + C[7];
    const double z2 = C[8] * X0 + C[9] * X1 + C[10] * X2 + C[11];
    const double d0 = z0 / z2 - v(0), d1 = z1 / z2 - v(1);
    const double r2 = d0 * d0 + d1 * d1;
    return r2 < sq_thr && z2 > 0.0;
}
template <int KIND> PLB_DEV bool is_inlier(const double *C, const double *v, double sq_thr) {
    double r2;
    if (!under_thr<KIND>(C, v, sq_thr, r2)) return false;
    if constexpr (kind_is_relpose(KIND)) {
        d3 b1, b2;
        corr_bearings<KIND>(v, b1, b2);
        return cheirality_ctx(C, b1, b2);
    }
    return true;
}

// Exact MSAC scoring of a tile of models (contexts ctx[0..tm), tm <= TM) over all correspondences of P, by the CTA's
// SCORE_THREADS (=256) threads, all of which must call it (it contains CTA barriers and warp reductions).
// Model i's record goes to counts[i], scores[i].  Every correspondence is loaded once for the whole tile.
// A model's summation order depends neither on TM nor on its place in the tile — thread-strided partial sums,
// xor-butterfly inside each warp, the 8 warp partials added left to right — so the same model gets the same score bits
// wherever it is scored (round tiles, initial models, LO rescoring, fast-mode confirmation): the equalities the serial
// loop relies on (ransac_impl.h:127,143) are preserved.
constexpr int SCORE_THREADS = 256;
constexpr int SCORE_WARPS = SCORE_THREADS / 32;
template <int TM> struct ScoreRed {
    double s[SCORE_WARPS][TM];
    uint32_t c[SCORE_WARPS][TM];
};
// MASK: also write model i's decision on correspondence k to mask[i * mask_stride + k] (get_inliers: is_inlier, and
// pnp_get_inlier for PnP), from the correspondence loaded for the score.
template <int KIND, int TM, bool MASK = false>
PLB_DEV void msac_score(const ProblemDev &P, const double (&ctx)[TM][CTX_MAX], int tm, ScoreRed<TM> &red,
                        uint32_t *counts, double *scores, char *mask = nullptr, long long mask_stride = 0) {
    const int tid = threadIdx.x, lane = tid & 31;
    const int n = P.n;
    const double sq_thr = P.sq_thr;
    uint32_t cnt[TM];
    double sc[TM];
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        cnt[i] = 0;
        sc[i] = 0.0;
    }
    // One correspondence per iteration: unrolled, the loop keeps the problem's array pointers of several iterations
    // live, and the 64-register one-model kernels (k_score, k_confirm) spill them.
#pragma unroll 1
    for (int k = tid; k < n; k += SCORE_THREADS) {
        double v[kind_corr_size(KIND)];
        load_corr<KIND>(P, k, v);
        // Without cheirality a model under the threshold is an inlier and is accumulated at once; the relpose kinds
        // collect the models under the threshold first, so that the bearings are computed once for the tile.
        double r2u[TM];
        unsigned under = 0, dec = 0;
#pragma unroll
        for (int i = 0; i < TM; ++i) {
            double r2;
            if (i < tm && under_thr<KIND>(ctx[i], v, sq_thr, r2)) {
                if constexpr (kind_is_relpose(KIND)) {
                    r2u[i] = r2;
                    under |= 1u << i;
                } else {
                    ++cnt[i];
                    sc[i] += r2;
                    dec |= 1u << i;
                }
            }
        }
        if (kind_is_relpose(KIND) && under) {
            d3 b1, b2;
            corr_bearings<KIND>(v, b1, b2);
#pragma unroll 1
            for (int i = 0; i < TM; ++i)
                if (((under >> i) & 1u) && !cheirality_ctx(ctx[i], b1, b2)) under &= ~(1u << i);
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                if ((under >> i) & 1u) {
                    ++cnt[i];
                    sc[i] += r2u[i];
                }
            }
        }
        if constexpr (MASK) {
            if constexpr (kind_is_relpose(KIND)) dec = under;
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                if (i >= tm) break;
                bool in = (dec >> i) & 1u;
                if constexpr (KIND == KIND_PNP) in = pnp_get_inlier(ctx[i], [&](int j) { return v[j]; }, sq_thr);
                mask[i * mask_stride + k] = in ? 1 : 0;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const uint32_t c = warp_sum_u(cnt[i]);
        const double s = warp_sum(sc[i]);
        if (lane == 0) {
            red.c[tid >> 5][i] = c;
            red.s[tid >> 5][i] = s;
        }
    }
    __syncthreads();
    if (tid < tm) {
        uint32_t ct = 0;
        double st = 0.0;
#pragma unroll
        for (int w = 0; w < SCORE_WARPS; ++w) {
            ct += red.c[w][tid];
            st += red.s[w][tid];
        }
        // Outliers contribute (n - count) * thr in ONE product for every kind (the reference does so for reprojection
        // scores, robust/utils.cc:62, and adds thr per outlier for the others).  Position-independent on purpose:
        // models supported only by their own minimal sample all score (n - K) thr to the last bit, as in the CPU's
        // sequential sum where the K negligible residuals are absorbed — so such ties are not "better scores"
        // (ransac_impl.h:116).
        st += (double)(n - (int)ct) * sq_thr;
        counts[tid] = ct;
        scores[tid] = st;
    }
    __syncthreads(); // red and ctx may be rewritten after this
}
// One model, its context built by every thread in registers.
template <int KIND>
PLB_DEV void cta_score(const ProblemDev &P, const double *model, ScoreRed<1> &red, uint32_t *count, double *score) {
    double ctx[1][CTX_MAX];
    model_ctx<KIND>(model, ctx[0]);
    msac_score<KIND, 1>(P, ctx, 1, red, count, score);
}

// ============================================================================================================
// hypothesis kernels: one minimal solve per thread
// ============================================================================================================
PLB_DEV int sample_problem_slot(const RoundDesc &R, int g) {
    int lo = 0, hi = R.n_active - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(R.g_off + mid + 1) <= g) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// p3p and homography_4pt: every thread solves its own minimal sample with the scalar closed form; the lanes of a warp
// diverge where their samples take different branches (number of real roots, Newton iterations).  Models are appended
// to the problem's segment (slot range reserved with one atomicAdd per sample); n_models[g] / first_slot[g] let the
// ordered scans walk them in (sample, model) order per problem.
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
        nm = solve_p3p(xs, Xs, models);
    } else {
        d3 a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t id = R.samples[(size_t)g * 4 + i];
            a[i] = bearing(P.p[0][id], P.p[1][id]);
            b[i] = bearing(P.p[2][id], P.p[3][id]);
        }
        nm = solve_h4(a, b, models, true);
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

// relpose_7pt with ONE THREAD PER SAMPLE: fundamental_7pt on a 63-double slice of shared memory per thread (odd stride:
// conflict-free).
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
    double x1s[21], x2s[21];
#pragma unroll
    for (int i = 0; i < 7; ++i) {
        const uint32_t id = R.samples[(size_t)g * 7 + i];
        const d3 a = bearing(P.p[0][id], P.p[1][id]), b = bearing(P.p[2][id], P.p[3][id]);
        x1s[3 * i] = a.x; x1s[3 * i + 1] = a.y; x1s[3 * i + 2] = a.z;
        x2s[3 * i] = b.x; x2s[3 * i + 1] = b.y; x2s[3 * i + 2] = b.z;
    }
    double F[3][9];
    // P.rfc is read after the solve (loaded up front, it would stay live across the nullspace routine)
    int nm = fundamental_7pt(x1s, x2s, W, [&](const double *f) { return P.rfc ? rfc_ok(f) : true; }, F);
    if (!live) return;
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

// ---- relpose_5pt as phase kernels ----------------------------------------------------------------------------------
// The 5-point solver is a large body of code; as one kernel, warps at different places of it starve on instruction
// fetch.  Split into phases, each kernel's code is small and every phase maps its threads to the work it has:
//   k5_gather    : thread = sample          the sample's bearings
//   k5_null      : thread = sample          pivoted-QR nullspace
//   k5_elim      : thread = sample          trace constraints, LU, determinant polynomial
//   k5_roots     : lane   = sample          Sturm bracketing + Ridders/Newton, warp-cooperative
//   k5_back      : lane   = (sample, root)  back-substitution, motion decomposition, cheirality
// The solver surface (k5_load, k5_solver_out) runs k5_null, k5_elim and k5_roots on the caller's instances.
constexpr int S5_BLK = 105;

// Bearings of the 5 sampled correspondences of every sample (estimators/relative_pose.cc:51-54,90-94) into the
// entry-major per-sample block (entries 75..104).  Its chain of dependent global loads (problem slot -> problem ->
// sample ids -> points) is a kernel of its own, at full occupancy: inside the first-half kernel (4 warps per SM) it was
// 19 % of that kernel's time.
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

// First half with ONE THREAD PER SAMPLE (solver5_lane.cuh), in two kernels split at the nullspace.  As one kernel its
// 200 KB of straight-line code starved on instruction fetch, and the nullspace, which needs far fewer registers, ran at
// the occupancy the elimination imposes.
//
// k5_null: the 9 x 5 epipolar matrix in a 45-double slice of shared memory (odd stride: the 32 lanes of a warp spread
// over all bank pairs; the pivoted QR indexes it dynamically), its nullspace basis Nb straight from registers to
// entries 39..74 of the sample's block, where k5_elim and k5_back read it.  Four CTAs of 128 threads, 16 warps per SM
// (128 registers, no spills; 7 % faster on the H100 than 12 warps at 162 registers).
constexpr int NULL_THREADS = 128;
constexpr int NULL_STRIDE = 45;
__global__ void __launch_bounds__(NULL_THREADS, 4) k5_null(const int n_total, HypOut out) {
    __shared__ double sW[NULL_THREADS * NULL_STRIDE];
    double *W = sW + threadIdx.x * NULL_STRIDE;
    const int g = blockIdx.x * NULL_THREADS + threadIdx.x;
    if (g >= n_total) return;
    const size_t nt = (size_t)n_total;
    double *blk = out.s5_blk + g; // entry-major: blk[e * n_total]
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
    // Nb[4 * k + r] = entry k of basis vector r
    lane5::nullspace_basis<5>(W, [&](int r, int k, double v) { blk[(39 + 4 * k + r) * nt] = v; });
}

// k5_elim: Nb (registers) -> trace / determinant constraints -> elimination -> determinant polynomial.  The quadratic
// blocks live in registers (compile-time monomial tables); shared memory holds only the LEFT 10 x 10 block of the
// elimination matrix (dynamic pivot rows) plus 10 doubles of scratch per thread, the right-hand sides are parked in
// global memory (L2) while the block is factored and come back column by column.  111 doubles per thread (odd) x 256
// threads = 222 KB: one CTA, 8 warps per SM.
constexpr int ELIM_THREADS = 256;
constexpr int ELIM_STRIDE = 111;
constexpr size_t ELIM_SMEM = sizeof(double) * ELIM_STRIDE * ELIM_THREADS;
// Of R, only n_total is read.  (With an int parameter in its place the compiler schedules this kernel differently.)
__global__ void __launch_bounds__(ELIM_THREADS, 1) k5_elim(const RoundDesc R, HypOut out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *W = reinterpret_cast<double *>(smem_raw) + (size_t)threadIdx.x * ELIM_STRIDE;
    double *CL = W, *S = W + 100;
    int g = blockIdx.x * ELIM_THREADS + threadIdx.x;
    const bool live = g < R.n_total;
    if (!live) g = R.n_total - 1; // idle threads of the last CTA redo the last sample (same values, harmless stores)
    const size_t nt = (size_t)R.n_total;
    double *blk = out.s5_blk + g;   // entry-major: blk[e * n_total]
    double *park = out.s5_park + g; // right-hand sides, entry-major: park[(row * 10 + column) * n_total]
    {
        double Nb[36];
#pragma unroll
        for (int e = 0; e < 36; ++e) Nb[e] = blk[(39 + e) * nt];
        lane5::build_coeffs(Nb, [&](int row, auto cc, double v) {
            constexpr int ci = decltype(cc)::value;
            if constexpr (ci < 10) CL[row * 10 + ci] = v;
            else park[(size_t)(row * 10 + (ci - 10)) * nt] = v;
        });
    }
    int idx[10];
    lane5::lu_left(CL, S, idx);
    lane5::solve_rhs(CL, S, idx, [&](int r, int c) { return park[(size_t)(r * 10 + c) * nt]; }, CL);
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
            const StridedD blk{out.s5_blk + g, (size_t)R.n_total}; // entry-major (k5_null, k5_elim)
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

// Models the scoring kernels evaluate in active problem a's segment.  prob_count[a] keeps the whole atomicAdd total
// even when the segment overflowed (the solve kernels then set out.overflow and drop the samples that did not fit), so
// it is clamped to the segment: an overflowed round is redone, but its scoring must stay inside the problem's slots.
__device__ __forceinline__ int seg_models(const HypOut &out, int a) {
    const int c = out.prob_count[a], cap = __ldg(out.seg_cap + a);
    return c < cap ? c : cap;
}

// Tiled score kernel of the round path: CTA (x, a) scores tiles of SCORE_TM models of active problem a (model constants
// are broadcast reads from shared memory), which divides the L2 -> SM traffic of one CTA per model by the tile size.
constexpr int SCORE_TM = 4;
// the tangent-Sampson kind carries 18 values per correspondence: two models per tile keep it inside 128 registers
template <int KIND> constexpr __host__ __device__ int score_tm() { return KIND == KIND_RELPOSE_TS ? 2 : SCORE_TM; }

// Explicit-model scorer: a persistent 1D grid of 256-thread CTAs walks the (problem, first model, tile size) items of
// the descriptors — descriptor d owns tiles [tile0, tile0 + ceil(m / tm_max)), tile j of it models j*tm_max .. — and
// scores each tile with msac_score, every correspondence loaded once per tile.  tm_max is score_tm<KIND>() or 1 (the
// initial models); a record's bits depend on neither.  MASK: the descriptors' masks are written in the same pass.
template <int KIND, bool MASK>
__global__ void __launch_bounds__(SCORE_THREADS, 2)
    k_score(const ProblemDev *__restrict__ probs, const ScoreDesc *__restrict__ descs, int n_desc, long long n_tiles,
            int tm_max) {
    constexpr int MSZ = kind_model_size(KIND);
    constexpr int TM = score_tm<KIND>();
    __shared__ double ctx[TM][CTX_MAX];
    __shared__ ScoreRed<TM> red;
    __shared__ uint32_t cnt[TM];
    __shared__ double sc[TM];
    // the tile's item, read back from shared memory after the scoring pass rather than kept live through it (the
    // 128-register budget of the pass has no room for it)
    __shared__ const ScoreDesc *item;
    __shared__ long long item_m0;
    __shared__ int item_tm;
    const int tid = threadIdx.x;
    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        if (tid == 0) {
            int lo = 0, hi = n_desc - 1; // the last descriptor with tile0 <= t
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (descs[mid].tile0 <= t) lo = mid;
                else hi = mid - 1;
            }
            const long long m0 = (t - descs[lo].tile0) * tm_max;
            item = descs + lo;
            item_m0 = m0;
            item_tm = (int)(descs[lo].m - m0 < tm_max ? descs[lo].m - m0 : tm_max);
        }
        __syncthreads();
        {
            const ScoreDesc &D = *item;
            const long long m0 = item_m0;
            const int tm = item_tm;
            if (tid < tm) {
                double mdl[MSZ];
#pragma unroll
                for (int k = 0; k < MSZ; ++k) mdl[k] = D.models[(size_t)(m0 + tid) * MSZ + k];
                model_ctx<KIND>(mdl, ctx[tid]);
            }
            __syncthreads();
            msac_score<KIND, TM, MASK>(probs[D.pidx], ctx, tm, red, cnt, sc,
                                       MASK ? D.mask + m0 * D.mask_stride : nullptr, D.mask_stride);
        }
        if (tid < item_tm) { // msac_score ends with a barrier; thread tid wrote cnt[tid], sc[tid]
            if (item->counts) item->counts[item_m0 + tid] = cnt[tid];
            else item->counts32[item_m0 + tid] = cnt[tid];
            item->scores[item_m0 + tid] = sc[tid];
        }
        __syncthreads(); // item is rewritten for the next tile
    }
}
template <int KIND>
__global__ void __launch_bounds__(SCORE_THREADS, 2)
    k_score_tiled(const RoundDesc R, HypOut out) {
    constexpr int MSZ = kind_model_size(KIND);
    constexpr int TM = score_tm<KIND>();
    __shared__ double ctx[TM][CTX_MAX];
    __shared__ ScoreRed<TM> red;
    const int a = blockIdx.y;
    const int count = seg_models(out, a);
    const int tid = threadIdx.x;
    if (blockIdx.x * TM >= count) return;
    const ProblemDev P = R.probs[R.active[a]];
    const int seg = out.seg_base[a];
    for (int m0 = blockIdx.x * TM; m0 < count; m0 += gridDim.x * TM) {
        const int tm = (count - m0 < TM) ? (count - m0) : TM;
        if (tid < tm) {
            double mdl[MSZ];
#pragma unroll
            for (int k = 0; k < MSZ; ++k) mdl[k] = out.models[(size_t)(seg + m0 + tid) * MSZ + k];
            model_ctx<KIND>(mdl, ctx[tid]);
        }
        __syncthreads();
        msac_score<KIND, TM>(P, ctx, tm, red, out.counts + seg + m0, out.scores + seg + m0);
    }
}

// ============================================================================================================
// fp32 screening pass (fast mode)
// ============================================================================================================
// Scores EVERY model of the round in fp32 from the fp32 SoA copy of the correspondences (16 B / 2D-2D corr, 20 B /
// 2D-3D corr).  The CTA stages its problem's arrays into shared memory with TMA bulk copies (cp.async.bulk, one
// mbarrier) and then walks that problem's model tiles; every thread evaluates SCR_TM models per correspondence read
// from shared memory.  The records (count32, score32) only decide which models COULD change the RANSAC state; those
// candidates are rescored in fp64 (k_confirm) before the serial replay, so results are those of the exact mode.
constexpr int SCR_THREADS = 512;
constexpr int SCR_WARPS = SCR_THREADS / 32;
constexpr int SCR_TM = 8;
constexpr int SCR_RQ_TAKE = 8; // cases a lane may queue per pass of the warp-compacted handling
constexpr int SCR_PB = 4;      // correspondences per thread and step of the streaming pass
constexpr int SCR_CTX_THREADS = 128;
constexpr int QW = 8;          // Sampson kinds: word groups of 8 streaming steps per chunk (hit[] words of a lane)
static_assert(SCR_RQ_TAKE == scr::RQ_TAKE && SCR_TM == scr::REC_TM, "the depth bound of scr::record_depth");

// The fp32 screening constants of every model of the round (scr::CTX_FLOATS floats per model slot, fctx), one
// thread per model: the fp32 model from model_ctx and the per-model constants of the error bounds (screen_math.cuh),
// from the fp64 model and the problem's coordinate maxima.  Entries a kind does not use are 0.
template <int KIND>
__global__ void __launch_bounds__(SCR_CTX_THREADS) k_screen_ctx(const RoundDesc R, const HypOut out, float *__restrict__ fctx) {
    constexpr int MSZ = kind_model_size(KIND);
    constexpr int CTX = kind_ctx_size(KIND);
    constexpr int NARR = (KIND == KIND_PNP) ? 5 : 4;
    const int a = blockIdx.y;
    const int m = blockIdx.x * SCR_CTX_THREADS + threadIdx.x;
    if (m >= seg_models(out, a)) return;
    const ProblemDev &P = R.probs[R.active[a]];
    const size_t slot = (size_t)out.seg_base[a] + m;
    double mdl[MSZ];
#pragma unroll
    for (int k = 0; k < MSZ; ++k) mdl[k] = out.models[slot * MSZ + k];
    double cp[CTX];
    model_ctx<KIND>(mdl, cp);
    float c[scr::CTX_FLOATS];
#pragma unroll
    for (int k = 0; k < scr::CTX_FLOATS; ++k) c[k] = k < CTX ? (float)cp[k] : 0.f;
    float cm[5];
#pragma unroll
    for (int j = 0; j < NARR; ++j) cm[j] = P.cmax[j];
    if (KIND == KIND_PNP) scr::transfer_setup<3>(cp, cm + 2, cm, P.sq_thr, c);
    else if (KIND == KIND_HOMOG) scr::transfer_setup<2>(cp, cm, cm + 2, P.sq_thr, c);
    else scr::sampson_setup(cp, cm, P.sq_thr, c);
    if constexpr (KIND == KIND_RELPOSE) scr::cheirality_setup(cp + 9, cp + 13, c);
    if constexpr (KIND == KIND_RELPOSE || KIND == KIND_FUND) { // the integer streaming test (screen_math.cuh)
        uint32_t w[4];
        int qc, qoff;
        scr::sampson_qmodel(cp, cm, c[scr::S_CK], w, qc, qoff);
        c[scr::S_QH0] = __uint_as_float(w[0]);
        c[scr::S_QH1] = __uint_as_float(w[1]);
        c[scr::S_QL0] = __uint_as_float(w[2]);
        c[scr::S_QL1] = __uint_as_float(w[3]);
        c[scr::S_QC] = __int_as_float(qc);
        c[scr::S_QOFF] = __int_as_float(qoff);
    }
    float4 *dst = reinterpret_cast<float4 *>(fctx + slot * scr::CTX_FLOATS);
#pragma unroll
    for (int k = 0; k < scr::CTX_FLOATS / 4; ++k) dst[k] = make_float4(c[4 * k], c[4 * k + 1], c[4 * k + 2], c[4 * k + 3]);
}

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
PLB_DEV void cp_async16(void *dst_smem, const void *src_gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
PLB_DEV void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
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
PLB_DEV float lds_f(uint32_t saddr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr));
    return v;
}
// h |= bit if c, as one predicated LOP3 on c's predicate (left to itself the compiler selects bit-or-0 first and ORs that)
PLB_DEV void or_if(uint32_t &h, bool c, uint32_t bit) {
    asm("{\n.reg .pred p;\nsetp.ne.u32 p, %1, 0;\n@p or.b32 %0, %0, %2;\n}" : "+r"(h) : "r"((uint32_t)c), "r"(bit));
}
PLB_DEV float2 lds_f2(const float2 *p) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(smem_u32(p)));
    return v;
}
// The integer streaming test of the Sampson kinds (screen_math.cuh): the A fragment of 16 staged rows, the s8 MMA with
// int32 accumulation, and h |= bit if (uint32)v <= lim as one predicated LOP3.
PLB_DEV void ldsm_x2(uint32_t saddr, uint32_t &r0, uint32_t &r1) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(saddr));
}
PLB_DEV void mma_s8(int *d, uint32_t a0, uint32_t a1, uint32_t b, int c0, int c1) {
    asm("mma.sync.aligned.m16n8k16.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%7,%8,%7,%8};"
        : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
        : "r"(a0), "r"(a1), "r"(b), "r"(c0), "r"(c1));
}
PLB_DEV void or_if_le(uint32_t &h, uint32_t v, uint32_t lim, uint32_t bit) {
    asm("{\n.reg .pred p;\nsetp.le.u32 p, %1, %2;\n@p or.b32 %0, %0, %3;\n}" : "+r"(h) : "r"(v), "r"(lim), "r"(bit));
}
PLB_DEV float warp_sum_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Padded length of one staged array: the streaming pass then runs whole steps of SCR_PB correspondences per thread.
template <int NTHR> constexpr __host__ __device__ int scr_stage_len(int n) {
    return (n + SCR_PB * NTHR - 1) / (SCR_PB * NTHR) * (SCR_PB * NTHR);
}

// NTHR: threads per CTA.  512 (one CTA per SM next to a 160 KB staging buffer) for the large problems the kernel was
// shaped for; 128 (four CTAs per SM) for small ones (BASELINE config 1: 200 correspondences), where a 512-thread CTA
// leaves most threads without a correspondence.
//
// The pipeline of one CTA over its tiles of SCR_TM models, with one barrier per tile:
//   * the model constants come ready-made from fctx (k_screen_ctx); tile t+1's are copied (cp.async) into the other
//     half of the double-buffered ctx[] while tile t streams, and waited for just before the tile's barrier;
//   * the warps' partial records of tile t go to one half of the double-buffered red_* / s_border; the cross-warp sums
//     and the record writes of tile t are done by threads 0..SCR_TM-1 at the start of tile t+1 (the last tile of a
//     problem right after its barrier), always in warp order, so the records do not depend on timing;
//   * on the shared-memory path the staged arrays are padded with NaN to whole streaming steps (scr_stage_len), so there
//     is no remainder pass; the global-memory path runs one guarded step for the last < SCR_PB correspondences;
//   * the Sampson kinds (relpose, fundamental) stream the integer form of |C^| <= K on the int8 tensor cores instead
//     (screen_math.cuh): the CTA stages the problem's 16 B integer rows (ProblemDev::q, built once per problem by
//     k_qrows; zero rows up to scr_stage_len), a warp step is one ldmatrix and two mma.m16n8k16.s8 over 16 rows x the
//     tile's 8 models, and the queue pass reads the fp32 coordinates of a recorded case from global memory.  Unstaged,
//     the lanes read their fragment words from ProblemDev::q.  A caller that supplies no rows (q null) gets them built
//     from the fp32 arrays, by the CTA when staged and by every lane for its own words otherwise (the same bits).
template <int KIND, int NTHR>
__global__ void __launch_bounds__(NTHR, NTHR >= 512 ? 1 : 4) k_screen(const RoundDesc R, HypOut out, const float *__restrict__ fctx, int use_smem) {
    constexpr int SCR_THREADS = NTHR, SCR_WARPS = NTHR / 32; // shadow the file-scope defaults
    constexpr int NARR = (KIND == KIND_PNP) ? 5 : 4;
    constexpr bool SAMP = KIND == KIND_RELPOSE || KIND == KIND_FUND;
    constexpr int CTX_V4 = scr::CTX_FLOATS / 4;
    extern __shared__ __align__(128) unsigned char scr_smem[];
    __shared__ __align__(8) uint64_t bar;
    __shared__ __align__(16) float ctx[2][SCR_TM][scr::CTX_FLOATS];
    __shared__ float red_s[2][SCR_WARPS][SCR_TM];
    __shared__ float red_e[2][SCR_WARPS][SCR_TM];
    __shared__ uint32_t red_c[2][SCR_WARPS][SCR_TM];
    __shared__ uint32_t s_border[2][SCR_TM];
    __shared__ uint16_t rq[SCR_WARPS][32 * SCR_RQ_TAKE]; // per-warp queue of recorded cases: lane << 8 | bit << 3 | hit[] word
                                                         // (the model; Sampson kinds: the word group)
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
    auto tiles_of = [&](int a) -> int { return (seg_models(out, a) + SCR_TM - 1) / SCR_TM; };
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
    if (tid < 2 * SCR_TM) s_border[tid / SCR_TM][tid % SCR_TM] = 0u; // then reset by each tile's record writer
    __syncthreads();
    uint32_t phase = 0;
    for (int a = s_first; a <= s_last; ++a) {
    const int count = seg_models(out, a);
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
    // copy the constants of the tile of models starting at m0f (cp.async, 16 B per thread; waited for before the
    // barrier that precedes their first use)
    auto fetch_ctx = [&](int b, int m0f) {
        const int tmf = (count - m0f < SCR_TM) ? (count - m0f) : SCR_TM;
        if (tid < tmf * CTX_V4) cp_async16(&ctx[b][0][0] + 4 * tid, fctx + (size_t)(seg + m0f) * scr::CTX_FLOATS + 4 * tid);
    };
    // cross-warp sums of the tile of models starting at m0f (partials in half b), by thread tid < that tile's size
    auto write_record = [&](int b, int m0f) {
        uint32_t ct = 0;
        float st = 0.f, et = 0.f;
#pragma unroll
        for (int w = 0; w < SCR_WARPS; ++w) {
            ct += red_c[b][w][tid];
            st += red_s[b][w][tid];
            et += red_e[b][w][tid];
        }
        st += (float)n * thr; // the per-correspondence sums hold (r2 - thr) of the inliers only
        // + the rounding of the fp32 sums themselves (scr::record_err): their depth follows from the queue pass, which
        //   lets any lane of a warp add a recorded case to its sums.  The padding below adds no term (a padded
        //   correspondence is never recorded) and no chunk, and the correspondence -> (lane, bit) mapping and the queue
        //   order are those of a pass over the n correspondences alone, so the depth is unchanged.
        const uint32_t bd = s_border[b][tid];
        out.fcounts[seg + m0f + tid] = ct;
        out.fscores[seg + m0f + tid] = st;
        out.fborder[seg + m0f + tid] = bd;
        // + REC_ERR0: +inf for a model whose fp32 evaluation the bounds do not cover (overflow, non-finite data bounds)
        out.ferr[seg + m0f + tid] = scr::record_err(et, ct, bd, thr, n, SCR_THREADS) +
                                    fctx[(size_t)(seg + m0f + tid) * scr::CTX_FLOATS + scr::REC_ERR0];
        s_border[b][tid] = 0u;
    };
    fetch_ctx(0, t_begin * SCR_TM);
    const float *arr[NARR];
    uint32_t sarr[NARR] = {}; // shared-memory addresses of the staged arrays (the streaming pass reads them with LDS)
    int n_str = n; // correspondences the streaming pass runs over (padded on the shared-memory path)
    float qf[8];   // Sampson kinds: 2^(15 - e_j), the column scales of the integer rows (screen_math.cuh)
    uint32_t srow = 0; // Sampson kinds: shared-memory address of the staged rows
    if constexpr (SAMP) {
        int e[8];
        scr::sampson_qscale(P.cmax, e);
#pragma unroll
        for (int j = 0; j < 8; ++j) qf[j] = ldexpf(1.f, 15 - e[j]);
#pragma unroll
        for (int c = 0; c < NARR; ++c) arr[c] = P.f[c]; // the queue pass reads the recorded cases from L2
    }
    if (use_smem && SAMP) {
        // the integer rows (16 B each) of the problem's correspondences, zero rows up to whole streaming word groups;
        // a zero row may be recorded, the queue pass skips it (k >= n).  The rows of P.q (launch_qrows) come in by one
        // TMA bulk copy; without them the CTA builds the rows from the fp32 arrays.
        uint4 *rows = reinterpret_cast<uint4 *>(scr_smem);
        const int n_st = scr_stage_len<NTHR>(n);
        __syncthreads(); // every thread is done with the previous problem's rows
        int k_have = 0;
        if (P.q) {
            if (tid == 0) {
                mbar_expect_tx(&bar, (uint32_t)n_pad * 16u);
                tma_bulk_g2s(rows, P.q, (uint32_t)n_pad * 16u, &bar);
            }
            mbar_wait(&bar, phase);
            phase ^= 1u;
            k_have = n_pad;
        }
        for (int k = k_have + tid; k < n_st; k += SCR_THREADS) {
            uint32_t w[4] = {0u, 0u, 0u, 0u};
            if (k < n) scr::sampson_qrow(P.f[0][k], P.f[1][k], P.f[2][k], P.f[3][k], qf, w);
            rows[k] = make_uint4(w[0], w[1], w[2], w[3]);
        }
        srow = smem_u32(rows);
        n_str = n_st;
    } else if (use_smem) {
        float *pts = reinterpret_cast<float *>(scr_smem);
        const int n_st = scr_stage_len<NTHR>(n);
        __syncthreads(); // every thread is done with the previous problem's arrays
        if (tid == 0) {
            const uint32_t bytes = (uint32_t)n_pad * 4u;
            mbar_expect_tx(&bar, bytes * NARR);
#pragma unroll
            for (int c = 0; c < NARR; ++c) tma_bulk_g2s(pts + (size_t)c * n_st, P.f[c], bytes, &bar);
        }
        mbar_wait(&bar, phase);
        phase ^= 1u;
        // NaN padding of [n, n_st) of every array, written after this thread saw the bulk copies complete and made
        // visible to all by the barrier below.  A padded correspondence is never recorded: every test of the streaming
        // pass is an ordered comparison, false when an operand is NaN, and NaN coordinates make every operand NaN
        //   relpose, fundamental: C is NaN  ->  sampson_maybe_c's  |C| <= K  is false;
        //   homography: w is NaN  ->  z = fma(thr_s', |w|, c') is NaN  ->  transfer_maybe's  z > 0  is false;
        //   pnp: the depth z2 is NaN  ->  z is NaN  ->  z > 0  is false.
        // This holds whatever the model constants are, infinite ones included.
        for (int i = n + tid; i < n_st; i += SCR_THREADS)
#pragma unroll
            for (int c = 0; c < NARR; ++c) pts[(size_t)c * n_st + i] = __int_as_float(0x7fc00000);
#pragma unroll
        for (int c = 0; c < NARR; ++c) {
            arr[c] = pts + (size_t)c * n_st;
            sarr[c] = smem_u32(arr[c]);
        }
        n_str = n_st;
    } else if (!SAMP) {
#pragma unroll
        for (int c = 0; c < NARR; ++c) arr[c] = P.f[c];
    }
    cp_async_wait_all();
    __syncthreads();
    int b = 0;
    for (int m0 = t_begin * SCR_TM; m0 < t_end * SCR_TM; m0 += SCR_TM, b ^= 1) {
        const int tm = (count - m0 < SCR_TM) ? (count - m0) : SCR_TM;
        if (m0 + SCR_TM < t_end * SCR_TM) fetch_ctx(b ^ 1, m0 + SCR_TM);
        if (m0 > t_begin * SCR_TM && tid < SCR_TM) write_record(b ^ 1, m0 - SCR_TM); // only a problem's last tile is partial
        const float(*cx)[scr::CTX_FLOATS] = ctx[b];
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
            // of model i in fp64" (screen_math.cuh: for the Sampson kinds |C| <= K, a bound over the coordinate box that
            // needs neither D nor E^T x2; for the transfer kinds the plain fp32 test widened by the rigorous error bound)
            // and a predicated OR that records the correspondence in a per-lane bit mask.  SCR_PB correspondences per thread
            // per step reuse the model constants fetched (broadcast) from shared memory.  The recorded cases (plain
            // decision, is it provably the fp64 decision, cheirality, division, accumulation of score and error bound)
            // are handled afterwards in a compacted loop in which every lane pops one of ITS recorded cases per
            // iteration — handled inline they cost a divergent detour for the whole warp whenever one lane of 32 hits.
            auto transfer_maybe = [&](const float *M, const float *p) -> bool {
                if (KIND == KIND_PNP) return scr::transfer_maybe<true>(M, scr::pnp_terms(M, p[0], p[1], p[2], p[3], p[4]));
                return scr::transfer_maybe<false>(M, scr::homography_terms(M, p[0], p[1], p[2], p[3]));
            };
            // Sampson kinds: the lane's B fragments (of model lane >> 2: [e_hi; 0] and [e_lo; e_hi]) and, for the models
            // 2 (lane & 3) + {0, 1} of its accumulators, init + off and 2 off; a model missing from a partial tile
            // records nothing (off = QOFF_NONE), so the streaming pass needs no per-model guard
            uint32_t qbh = 0u, qbl = 0u, qlim[2] = {0u, 0u};
            int qc[2] = {0, 0};
            if constexpr (SAMP) {
                const int t = lane & 3, g = lane >> 2;
                if (g < tm) {
                    if (t < 2) qbh = __float_as_uint(cx[g][scr::S_QH0 + t]);
                    qbl = __float_as_uint(cx[g][t < 2 ? scr::S_QL0 + t : scr::S_QH0 + t - 2]);
                }
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int mi = 2 * t + i;
                    qc[i] = mi < tm ? __float_as_int(cx[mi][scr::S_QC]) : scr::QOFF_NONE;
                    qlim[i] = (uint32_t)(mi < tm ? __float_as_int(cx[mi][scr::S_QOFF]) : scr::QOFF_NONE) << 1;
                }
            }
            // one step: 16 rows x 8 models; bit 4 s + j of h: accumulator j of the lane, i.e. row (lane >> 2) + 8 (j >> 1)
            // of the step and model 2 (lane & 3) + (j & 1)
            auto qstep = [&](uint32_t &h, uint32_t a0, uint32_t a1, int s) {
                int d1[4], d2[4];
                mma_s8(d1, a0, a1, qbh, 0, 0);
                mma_s8(d2, a0, a1, qbl, qc[0], qc[1]);
#pragma unroll
                for (int j = 0; j < 4; ++j) or_if_le(h, (uint32_t)d1[j] * 256u + (uint32_t)d2[j], qlim[j & 1], 1u << (4 * s + j));
            };
            // the lane's word of row k for the unstaged path (zero past n, as the staged padding): from P.q, or built
            const uint32_t *qg = reinterpret_cast<const uint32_t *>(P.q);
            auto qword_ld = [&](int k) -> uint32_t { return k < n ? qg[4 * (size_t)k + (lane & 3)] : 0u; };
            auto qword_at = [&](int k) -> uint32_t {
                return k < n ? scr::sampson_qword(arr[0][k], arr[1][k], arr[2][k], arr[3][k], qf, lane & 3) : 0u;
            };
            for (int base = 0; base < n_str; base += 32 * SCR_THREADS) {
                const int lim = min_i(n_str, base + 32 * SCR_THREADS);
                uint32_t hit[SCR_TM];
#pragma unroll
                for (int i = 0; i < SCR_TM; ++i) hit[i] = 0u;
                if constexpr (SAMP) {
                    // A chunk is QW word groups of 4 NTHR rows; in group w, step s of a warp covers the 16 rows
                    // base + 4 NTHR w + 16 (s SCR_WARPS + warp) + 0..15, and its hits go to bits 4 s .. 4 s + 3 of hit[w].
                    // n_str (or, unstaged, the zero rows past n) fills whole groups.  The words are shifted in, so that
                    // hit[] is indexed by constants only.
                    static_assert(QW == SCR_TM && 4 * 8 * QW == 32 * scr::REC_TM, "bits per lane and chunk of scr::record_depth");
#pragma unroll 1
                    for (int w = 0; w < QW; ++w) {
                        const int g0 = base + w * 4 * SCR_THREADS;
                        uint32_t h = 0u;
                        if (g0 < n_str) {
                            if (use_smem) {
                                const uint32_t a = srow + 16u * (uint32_t)(g0 + 16 * warp + (lane & 15));
#pragma unroll
                                for (int s = 0; s < 8; ++s) {
                                    uint32_t a0, a1;
                                    ldsm_x2(a + (uint32_t)(s * 256 * SCR_WARPS), a0, a1);
                                    qstep(h, a0, a1, s);
                                }
                            } else if (qg) {
                                // the group's 16 words first: all loads in flight before the first MMA
                                uint32_t fa[8][2];
#pragma unroll
                                for (int s = 0; s < 8; ++s) {
                                    const int r = g0 + 16 * (s * SCR_WARPS + warp) + (lane >> 2);
                                    fa[s][0] = qword_ld(r);
                                    fa[s][1] = qword_ld(r + 8);
                                }
#pragma unroll
                                for (int s = 0; s < 8; ++s) qstep(h, fa[s][0], fa[s][1], s);
                            } else {
#pragma unroll
                                for (int s = 0; s < 8; ++s) {
                                    const int r = g0 + 16 * (s * SCR_WARPS + warp) + (lane >> 2);
                                    qstep(h, qword_at(r), qword_at(r + 8), s);
                                }
                            }
                        }
#pragma unroll
                        for (int i = 0; i + 1 < SCR_TM; ++i) hit[i] = hit[i + 1];
                        hit[SCR_TM - 1] = h;
                    }
                } else {
                int k0 = base + tid;
                uint32_t qbit = 1u;
                // GUARDED: correspondences at or past lim read as NaN (never recorded, see the padding above);
                // STAGED: the arrays are in shared memory (sarr), read with LDS rather than generic loads
                auto step = [&](auto guarded, auto staged) {
                    float p[SCR_PB][NARR];
                    uint32_t bit[SCR_PB];
#pragma unroll
                    for (int j = 0; j < SCR_PB; ++j) {
                        const int k = k0 + j * SCR_THREADS;
                        bit[j] = qbit << j;
#pragma unroll
                        for (int c = 0; c < NARR; ++c) {
                            if (decltype(staged)::value) p[j][c] = lds_f(sarr[c] + 4u * (uint32_t)k);
                            else p[j][c] = (!decltype(guarded)::value || k < lim) ? arr[c][k] : __int_as_float(0x7fc00000);
                        }
                    }
#pragma unroll
                    for (int i = 0; i < SCR_TM; ++i) {
                        if (i >= tm) continue;
                        float Mr[20]; // [0..11] model, [16..19] constants of the streaming test
                        lds_v4(cx[i], Mr);
                        lds_v4(cx[i] + 4, Mr + 4);
                        lds_v4(cx[i] + 8, Mr + 8);
                        lds_v4(cx[i] + 16, Mr + 16);
#pragma unroll
                        for (int j = 0; j < SCR_PB; ++j) or_if(hit[i], transfer_maybe(Mr, p[j]), bit[j]);
                    }
                };
                auto stream = [&](auto staged) {
                    for (; k0 + (SCR_PB - 1) * SCR_THREADS < lim; k0 += SCR_THREADS * SCR_PB, qbit <<= SCR_PB)
                        step(std::false_type{}, staged);
                    // the last < SCR_PB correspondences of this lane (the staged arrays are padded to whole steps)
                    if (!decltype(staged)::value && k0 < lim) step(std::true_type{}, staged);
                };
                if (use_smem) stream(std::true_type{});
                else stream(std::false_type{});
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
                        const int q = (int)((ent >> 3) & 31u), ol = (int)(ent >> 8);
                        int mi, k;
                        if constexpr (SAMP) { // (word group, bit) -> (row, model), see the streaming pass
                            const int s = 8 * (int)(ent & 7u) + (q >> 2), j = q & 3;
                            k = base + 16 * (s * SCR_WARPS + warp) + (ol >> 2) + 8 * (j >> 1);
                            mi = 2 * (ol & 3) + (j & 1);
                            if (k >= n) continue; // a zero row of the padding
                        } else {
                            mi = (int)(ent & 7u);
                            k = base + warp * 32 + ol + q * SCR_THREADS;
                        }
                        float p[NARR];
#pragma unroll
                        for (int c = 0; c < NARR; ++c) p[c] = arr[c][k];
                        const float *M = cx[mi];
                        bool plain = false, border = false;
                        float v = 0.f, e = 0.f;
                        if (KIND == KIND_PNP) {
                            scr::transfer_point<true>(M, scr::pnp_terms(M, p[0], p[1], p[2], p[3], p[4]), plain, border, v, e);
                        } else if (KIND == KIND_HOMOG) {
                            scr::transfer_point<false>(M, scr::homography_terms(M, p[0], p[1], p[2], p[3]), plain, border, v, e);
                        } else {
                            scr::sampson_point(M, thr, p[0], p[1], p[2], p[3], plain, border, v, e);
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
                        if (border) atomicAdd(&s_border[b][mi], 1u);
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
                red_c[b][warp][i] = c;
                red_s[b][warp][i] = v;
                red_e[b][warp][i] = ev;
            }
        }
        cp_async_wait_all(); // the next tile's constants
        __syncthreads();
    }
    // the problem's last tile (the next problem starts with a barrier before any of its tiles writes red_* / s_border)
    const int m_last = (t_end - 1) * SCR_TM;
    if (tid < ((count - m_last < SCR_TM) ? (count - m_last) : SCR_TM)) write_record(b ^ 1, m_last);
    } // problems of this CTA
}

// fast mode confirmation driven by the device-side candidate lists of k_select: CTA (x, a) rescores the candidates
// x, x + gridDim.x, ... of active problem a in fp64 (msac_score, hence the same bits as everywhere else).
template <int KIND>
__global__ void __launch_bounds__(SCORE_THREADS, 4)
    k_confirm(const ProblemDev *__restrict__ probs, const SelectArgs A, const double *__restrict__ models) {
    constexpr int MSZ = kind_model_size(KIND);
    __shared__ ScoreRed<1> red;
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
        cta_score<KIND>(P, mdl, red, A.counts + m, A.scores + m);
    }
}

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
// Calls f(std::integral_constant<int, K>{}) for the runtime kind K; unknown kinds run as KIND_HOMOG.
template <class F> static void with_kind(int kind, F &&f) {
    if (kind == KIND_PNP) f(std::integral_constant<int, KIND_PNP>{});
    else if (kind == KIND_RELPOSE) f(std::integral_constant<int, KIND_RELPOSE>{});
    else if (kind == KIND_FUND) f(std::integral_constant<int, KIND_FUND>{});
    else if (kind == KIND_RELPOSE_TS) f(std::integral_constant<int, KIND_RELPOSE_TS>{});
    else f(std::integral_constant<int, KIND_HOMOG>{});
}

// relpose_5pt first half and root isolation of the R.n_total samples whose bearings are in out.s5_blk (entries
// 75..104): the round chain and the solver surface both run them through here.
static void launch_5pt_prep_roots(const RoundDesc &R, const HypOut &out, cudaStream_t stream) {
    static bool attr_set[MAX_DEVICES] = {false};
    if (!attr_set[cur_dev()]) {
        cudaFuncSetAttribute(k5_elim, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ELIM_SMEM);
        attr_set[cur_dev()] = true;
    }
    const int n = R.n_total;
    k5_null<<<(unsigned)((n + NULL_THREADS - 1) / NULL_THREADS), NULL_THREADS, 0, stream>>>(n, out);
    k5_elim<<<(unsigned)((n + ELIM_THREADS - 1) / ELIM_THREADS), ELIM_THREADS, ELIM_SMEM, stream>>>(R, out);
    k5_roots<<<(n + ROOTS_THREADS - 1) / ROOTS_THREADS, ROOTS_THREADS, 0, stream>>>(n, out);
}

template <int KIND>
static void launch_hyp_t(const RoundDesc &R, const HypOut &out, int mode, int max_n_pad, float *fctx, cudaStream_t stream,
                         cudaEvent_t ev_between) {
    if constexpr (KIND == KIND_RELPOSE_TS) mode = 0; // no fp32 screening copy of the 18-array layout: exact scoring
    if constexpr (kind_is_relpose(KIND)) {
        k5_gather<<<(R.n_total + 255) / 256, 256, 0, stream>>>(R, out);
        launch_5pt_prep_roots(R, out, stream);
        const int warps = (R.n_total + 31) / 32;
        k5_back<<<(warps * 32 + 127) / 128, 128, 0, stream>>>(R, out);
    } else if constexpr (KIND == KIND_FUND) {
        static bool attr_set[MAX_DEVICES] = {false};
        if (!attr_set[cur_dev()]) {
            cudaFuncSetAttribute(k7_solve_lane, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K7L_SMEM);
            attr_set[cur_dev()] = true;
        }
        k7_solve_lane<<<(R.n_total + K7L_THREADS - 1) / K7L_THREADS, K7L_THREADS, K7L_SMEM, stream>>>(R, out);
    } else {
        k_solve_lane<KIND><<<(R.n_total + 127) / 128, 128, 0, stream>>>(R, out);
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
        // fp32 screening: the constants of every model once, then one CTA holds one problem's fp32 arrays in shared
        // memory (TMA) and strides over its tiles
        k_screen_ctx<KIND><<<dim3((out.max_seg_cap + SCR_CTX_THREADS - 1) / SCR_CTX_THREADS, R.n_active, 1),
                             SCR_CTX_THREADS, 0, stream>>>(R, out, fctx);
        constexpr int NARR = (KIND == KIND_PNP) ? 5 : 4;
        const bool small = max_n_pad <= 2048; // few correspondences per problem: 128-thread CTAs, four per SM
        const size_t bytes =
            (size_t)NARR * (size_t)(small ? scr_stage_len<128>(max_n_pad) : scr_stage_len<512>(max_n_pad)) * 4;
        const int use_smem = bytes <= 200 * 1024 ? 1 : 0;
        static bool attr_done_dev[MAX_DEVICES] = {false};
        bool &attr_done = attr_done_dev[cur_dev()];
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
        kern<<<gx, nthr, use_smem ? bytes : 0, stream>>>(R, out, fctx, use_smem);
    }
}
void launch_hypotheses(int kind, const RoundDesc &R, const HypOut &out, int mode, int max_n_pad, float *fctx,
                       cudaStream_t stream, cudaEvent_t ev_between) {
    cudaMemsetAsync(out.prob_count, 0, sizeof(int) * R.n_active, stream);
    with_kind(kind, [&](auto K) { launch_hyp_t<K>(R, out, mode, max_n_pad, fctx, stream, ev_between); });
}

// ---- caller-drawn samples (plb_generate_batch): the round's sample table in, its records out ------------------------
// One problem per blockIdx.y (strided: a check covers every problem of a call), blockIdx.x strides over its indices.
// CHECK writes nothing but the flag, so an index outside [0, n) is found before any kernel gathers with it.
template <bool CHECK>
__global__ void __launch_bounds__(256) k_take_samples(const TakeDesc *__restrict__ descs, int n_desc, int *bad) {
    for (int d = blockIdx.y; d < n_desc; d += gridDim.y) {
        const TakeDesc D = descs[d];
        for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < D.count; i += (long long)gridDim.x * 256) {
            const int32_t v = D.src[i];
            if (CHECK) {
                if (v < 0 || v >= D.n) *bad = 1;
            } else {
                D.dst[i] = (uint32_t)v;
            }
        }
    }
}
void launch_take_samples(const TakeDesc *descs_dev, int n_desc, long long max_count, int *bad, cudaStream_t stream) {
    if (n_desc <= 0 || max_count <= 0) return;
    const dim3 grid((unsigned)std::min<long long>((max_count + 255) / 256, 512), (unsigned)std::min(n_desc, 65535), 1);
    if (bad)
        k_take_samples<true><<<grid, 256, 0, stream>>>(descs_dev, n_desc, bad);
    else
        k_take_samples<false><<<grid, 256, 0, stream>>>(descs_dev, n_desc, nullptr);
}
// One thread per sample g of the round: its n_models[g] models of slots [first_slot[g], first_slot[g] + n_models[g]) with
// their exact records, into row j = g - g_off[a] of active problem a's descriptor (direct), or packed: problem a's used
// segment prefix moves to cbase[a] (the models of the problems before it), slot order kept.
__global__ void __launch_bounds__(256) k_put_hyps(const RoundDesc R, const HypOut out, const PutDesc *__restrict__ descs,
                                                  int msz, int maxm, int packed) {
    extern __shared__ int cbase[]; // packed: n_active entries
    if (packed && threadIdx.x == 0)
        for (int a = 0, c = 0; a < R.n_active; ++a) {
            cbase[a] = c;
            c += seg_models(out, a);
        }
    __syncthreads();
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= R.n_total) return;
    const int a = sample_problem_slot(R, g);
    const int j = g - __ldg(R.g_off + a);
    const PutDesc &D = descs[a];
    const int nm = out.n_models[g], fs = out.first_slot[g];
    const long long o = packed ? (long long)cbase[a] + fs - __ldg(out.seg_base + a) : (long long)j * maxm;
    D.n_models[j] = nm;
    if (packed) D.offsets[j] = (int)o;
    double *models = D.models + o * msz, *scores = D.scores + o;
    long long *counts = D.counts + o;
    for (int m = 0; m < nm; ++m) {
        for (int k = 0; k < msz; ++k) models[m * msz + k] = out.models[(size_t)(fs + m) * msz + k];
        scores[m] = out.scores[fs + m];
        counts[m] = out.counts[fs + m];
    }
}
void launch_put_hyps(const RoundDesc &R, const HypOut &out, const PutDesc *descs_dev, int msz, int maxm, bool packed,
                     cudaStream_t stream) {
    if (R.n_total <= 0) return;
    const size_t smem = packed ? sizeof(int) * (size_t)R.n_active : 0;
    k_put_hyps<<<(R.n_total + 255) / 256, 256, smem, stream>>>(R, out, descs_dev, msz, maxm, packed ? 1 : 0);
}
void launch_confirm(int kind, const ProblemDev *probs, const SelectArgs &A, const double *models, cudaStream_t stream) {
    if (A.na <= 0) return;
    int gx = (8 * sm_count() + A.na - 1) / A.na;
    if (gx > 64) gx = 64;
    if (gx < 1) gx = 1;
    const dim3 grid((unsigned)gx, (unsigned)A.na, 1);
    with_kind(kind, [&](auto K) { k_confirm<K><<<grid, SCORE_THREADS, 0, stream>>>(probs, A, models); });
}

// ============================================================================================================
// explicit model scoring
// ============================================================================================================
int score_tile_models(int kind) {
    int tm = 0;
    with_kind(kind, [&](auto K) { tm = score_tm<K>(); });
    return tm;
}
void launch_score_models(int kind, bool mask, const ProblemDev *probs, const ScoreDesc *descs_dev, int n_desc,
                         long long n_tiles, int tm_max, cudaStream_t stream) {
    if (n_desc <= 0 || n_tiles <= 0) return;
    const long long blocks = n_tiles < 8LL * sm_count() ? n_tiles : 8LL * sm_count();
    with_kind(kind, [&](auto K) {
        if (mask)
            k_score<K, true><<<(unsigned)blocks, SCORE_THREADS, 0, stream>>>(probs, descs_dev, n_desc, n_tiles, tm_max);
        else
            k_score<K, false><<<(unsigned)blocks, SCORE_THREADS, 0, stream>>>(probs, descs_dev, n_desc, n_tiles, tm_max);
    });
}
// One-model descriptors of a device list of (model, problem index) pairs.
__global__ void k_score_list(const double *models, const int *model_prob, int n_models, int msz, uint32_t *counts,
                             double *scores, ScoreDesc *descs) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_models) return;
    descs[m] = {models + (size_t)m * msz, nullptr, scores + m, nullptr, 0, m, 1, model_prob[m], 0, counts + m};
}
void launch_score_models(int kind, const ProblemDev *probs, const double *models, const int *model_prob, int n_models,
                         uint32_t *counts, double *scores, cudaStream_t stream) {
    if (n_models <= 0) return;
    ScoreDesc *descs = nullptr;
    if (cudaMallocAsync(&descs, sizeof(ScoreDesc) * n_models, stream) != cudaSuccess) return;
    k_score_list<<<(n_models + 255) / 256, 256, 0, stream>>>(models, model_prob, n_models, kind_model_size(kind), counts,
                                                              scores, descs);
    launch_score_models(kind, false, probs, descs, n_models, n_models, 1, stream);
    cudaFreeAsync(descs, stream);
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
    double C[kind_ctx_size(KIND)];
    model_ctx<KIND>(mdl, C);
    if constexpr (KIND == KIND_PNP) {
        mask[k] = pnp_get_inlier(C, [&](int j) { return P.p[j][k]; }, sq_thr) ? 1 : 0;
    } else { // the scorer's test (tangent Sampson: robust/utils.cc:541-569)
        double v[kind_corr_size(KIND)];
        load_corr<KIND>(P, k, v);
        mask[k] = is_inlier<KIND>(C, v, sq_thr) ? 1 : 0;
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
    with_kind(kind, [&](auto K) { k_inlier_mask<K><<<grid, threads, 0, stream>>>(probs, descs_dev, mask_base); });
}

// ============================================================================================================
// Levenberg-Marquardt refit: one CTA per job
// ============================================================================================================
constexpr int LM_THREADS = 256;
static_assert(LM_THREADS == SCORE_THREADS, "k_lm rescores its result with msac_score");
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
    // 1-dim residual (jacobian_accumulator.h:125-141); W: the residual's weight wk, w = wk * loss weight (:122)
    template <bool W = false> PLB_DEV void add1(const LossFn &L, double res, const double *J, double wk = 1.0) {
        const double w = W ? wk * L.weight(res * res) : L.weight(res * res);
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
    // 2-dim residual (jacobian_accumulator.h:87-104); W as in add1 (:86)
    template <bool W = false>
    PLB_DEV void add2(const LossFn &L, double r0, double r1, const double *J0, const double *J1, double wk = 1.0) {
        const double w = W ? wk * L.weight(r0 * r0 + r1 * r1) : L.weight(r0 * r0 + r1 * r1);
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

// The refiners with camera parameters: the pose and, per camera, m <= CAM_MAX_PARAMS parameters, padded to NP.
//   KIND_PNP        AbsolutePoseRefiner with a non-empty camera_refine_idx (optim/absolute.h:40-171): pose 6, one
//                   camera, a 2-dim residual per point
//   KIND_RELPOSE_TS CameraRelativePoseRefiner, shared_intrinsics false (optim/relative.h:268-483, bundle.cc:249-254):
//                   rotation 3, tangent translation 2, camera 1 then camera 2, a 1-dim residual per point
// The padded rows and columns of JtJ and Jtr are zero, their damped diagonal is lambda and their step component zero, so
// the Cholesky solve, the step, its norm and the predicted decrease are those of the unpadded system.
// Tile row of one point: R Jacobian rows (NP each) | w*r (R) | w | loss | residual row | jac row | staging (STAGE):
//   PnP : jac_params of the point (2 x CAM_MAX_PARAMS)
//   TS  : jac_params of unproject_with_jac at x1, at x2 and at the finite-difference point (3 x 3 x CAM_MAX_PARAMS)
template <int KIND> struct LmCamDims;
template <> struct LmCamDims<KIND_PNP> {
    static constexpr int NPOSE = 6, NCAM = 1, R = 2, STAGE = 2 * CAM_MAX_PARAMS, CTX = 12;
};
template <> struct LmCamDims<KIND_RELPOSE_TS> {
    static constexpr int NPOSE = 5, NCAM = 2, R = 1, STAGE = 9 * CAM_MAX_PARAMS, CTX = 9 + 45;
};
template <int KIND> struct LmCamLayout : LmCamDims<KIND> {
    using D = LmCamDims<KIND>;
    static constexpr int NP = D::NPOSE + D::NCAM * CAM_MAX_PARAMS;
    static constexpr int NT = NP * (NP + 1) / 2;
    static constexpr int NV = 2 + NT + NP + 1; // [loss, residual rows, JtJ (packed lower, row-major), Jtr, jac rows]
    static constexpr int WR = D::R * NP, WT = WR + D::R, LOSS = WT + 1, ROW = LOSS + 1, JROW = ROW + 1, JP = JROW + 1,
                         W = JP + D::STAGE;
    static constexpr size_t TILE_BYTES = sizeof(double) * W * LM_THREADS;
    static_assert(NV <= LM_THREADS, "one owner thread per reduced value");
};

// Shared memory of one k_lm CTA that both refiners use: the parameters, the scalar LM state of thread 0 (JtJ and its
// damped copy Am NP x NP row-major, lower triangle used) and the cluster reduction of NV values.
template <int NP, int NV> struct LmCore {
    double par[9], par_new[9];
    double tb[6], tb_new[6]; // relpose: tangent basis of par / par_new
    double JtJ[NP * NP], Am[NP * NP], Jtr[NP], rhs[NP], sol[NP];
    double sums[2][NV]; // CTA partial sums, double-buffered: read by the other CTAs of the cluster (DSMEM)
    double tot[NV];     // cluster totals (identical in every CTA)
    int wcount[LM_WARPS];
    int flag;
};
// fixed camera: per-warp partial sums of the packed normal equations (cluster_sum), the rescoring of the result
template <int NP> struct LmShared : LmCore<NP, LM_NV_MAX> {
    double ctx[80];
    double red[LM_WARPS][LM_NV_MAX];
    ScoreRed<1> sred;
};
// camera refinement: the camera parameters of par / par_new and the refined indices idx[i][0..m[i]) of every camera;
// the tile rows of lmi_eval_pass are dynamic shared memory
template <int KIND> struct LmCamShared : LmCore<LmCamLayout<KIND>::NP, LmCamLayout<KIND>::NV> {
    static constexpr int NC = LmCamDims<KIND>::NCAM;
    double ctx[LmCamDims<KIND>::CTX];
    double cam[NC][CAM_MAX_PARAMS], cam_new[NC][CAM_MAX_PARAMS];
    int idx[NC][CAM_MAX_PARAMS];
    int m[NC];
};

// Cluster totals of the CTA partial sums S->sums[buf][0..nv) -> S->tot[0..nv) in every CTA, CTAs in rank order.
template <class Shared> PLB_DEV void cluster_total(Shared *S, int nv, int &buf, int csize) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    cluster.sync();
    if ((int)threadIdx.x < nv) {
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

// Cluster-wide deterministic sum of NV per-thread values -> S->tot[0..NV) in every CTA of the cluster.
// Order: xor-butterfly inside a warp, warps left to right, CTAs in rank order.
template <int NV, class Shared> PLB_DEV void cluster_sum(Shared *S, const double *v, int &buf, int csize) {
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
    cluster_total(S, NV, buf, csize);
}

// thread 0 -> whole CTA broadcast of a small integer (two barriers: the slot can be reused right away)
template <class Shared> PLB_DEV int block_bcast(Shared *S, int v) {
    if (threadIdx.x == 0) S->flag = v;
    __syncthreads();
    const int r = S->flag;
    __syncthreads();
    return r;
}

// The weight of point k's residuals: wt[k] (W, uniform where wt is null), 1 otherwise; wmul<W>(wk, v) is wk * v (W) or v
template <bool W> PLB_DEV double lm_weight(const double *wt, int k) {
    if constexpr (W) return wt ? wt[k] : 1.0;
    else return 1.0;
}
template <bool W> PLB_DEV double wmul(double wk, double v) {
    if constexpr (W) return wk * v;
    else return v;
}

// One evaluation pass at the parameters whose context is in S->ctx: robust cost + row count (compute_residual of the
// refiners) AND the normal equations JtJ (lower triangle, packed row-major), Jtr + count of non-zero-weight rows
// (compute_jacobian), accumulated separately exactly as two passes of the reference would.
// Output layout in S->tot: [0] loss sum, [1] residual rows, [2..2+NT) JtJ, [2+NT..2+NT+NP) Jtr, [2+NT+NP] jac rows.
// W: point k's residuals carry the weight wt[k] (uniform where wt is null): its loss terms are wt[k] * loss and its
// Jacobian weight wt[k] * loss weight (jacobian_accumulator.h:65-74,83-133); every residual still counts as a row.
template <int KIND, bool X = false, bool W = false>
PLB_DEV void lm_eval_pass(const ProblemDev &P, const LossFn &L, const double *wt, const int *list, int lo, int na,
                          LmShared<LmDims<KIND>::NP> *S, int &buf, int csize) {
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
            const double wk = lm_weight<W>(wt, k);
            double zp0, zp1, xr0, xr1, Jp[2][3];
            if (P.cam[0].model != CAMM_NULL) { // <Model>::project for the residual, ::project_with_jac for the Jacobian pass
                cam_project<X>(P.cam[0], Z0, Z1, Z2, xr0, xr1); // (optim/absolute.h:59-61,97-104)
                cam_project_with_jac<X>(P.cam[0], Z0, Z1, Z2, zp0, zp1, &Jp[0][0]);
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
                lsum += wmul<W>(wk, L.loss(q0 * q0 + q1 * q1));
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
            A.template add2<W>(L, r0, r1, J[0], J[1], wk);
        } else if (KIND == KIND_HOMOG) {
            const double a0 = P.p[0][k], a1 = P.p[1][k], b0 = P.p[2][k], b1 = P.p[3][k];
            const double wk = lm_weight<W>(wt, k); // one weight for both transfers (optim/homography.h:75,84,121,147)
            const double *H = ctx, *G = ctx + 9;
            // forward transfer (optim/homography.h:63-71,107-123); parameters = H00,H10,H20,H01,H11,H21,H02,H12
            const double Hx0 = H[0] * a0 + H[1] * a1 + H[2];
            const double Hx1 = H[3] * a0 + H[4] * a1 + H[5];
            const double iw = 1.0 / (H[6] * a0 + H[7] * a1 + H[8]);
            const double z0 = Hx0 * iw, z1 = Hx1 * iw;
            const double r0 = z0 - b0, r1 = z1 - b1;
            lsum += wmul<W>(wk, L.loss(r0 * r0 + r1 * r1));
            double J0[8] = {a0, 0.0, -a0 * z0, a1, 0.0, -a1 * z0, 1.0, 0.0};
            double J1[8] = {0.0, a0, -a0 * z1, 0.0, a1, -a1 * z1, 0.0, 1.0};
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                J0[m] = J0[m] * iw;
                J1[m] = J1[m] * iw;
            }
            A.template add2<W>(L, r0, r1, J0, J1, wk);
            // backward transfer through adj(H) (optim/homography.h:73-81,125-152):  y = pi(G x2),
            // dy_i/dH_k = ( (dG/dH_k x2)_i - y_i (dG/dH_k x2)_2 ) / (G x2)_2
            const double Gx0 = G[0] * b0 + G[1] * b1 + G[2];
            const double Gx1 = G[3] * b0 + G[4] * b1 + G[5];
            const double iv = 1.0 / (G[6] * b0 + G[7] * b1 + G[8]);
            const double y0 = Gx0 * iv, y1 = Gx1 * iv;
            const double s0 = y0 - a0, s1 = y1 - a1;
            lsum += wmul<W>(wk, L.loss(s0 * s0 + s1 * s1));
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
            A.template add2<W>(L, s0, s1, K0, K1, wk);
        } else if (KIND == KIND_RELPOSE_TS) {
            // FixCameraRelativePoseRefiner (optim/relative.h:181-249)
            double v[TS_ARRAYS];
            load_ts(P, k, v);
            const double wk = lm_weight<W>(wt, k);
            double C, JC[4];
            tangent_terms(ctx, v, v + 3, v + 6, v + 12, C, JC);
            {
                const double nJc_sq = (JC[2] * JC[2] + JC[3] * JC[3]) + (JC[0] * JC[0] + JC[1] * JC[1]);
                const double rr = C / sqrt(nJc_sq);
                lsum += wmul<W>(wk, L.loss(rr * rr));
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
            A.template add1<W>(L, r, J, wk);
        } else {
            const double a0 = P.p[0][k], a1 = P.p[1][k], b0 = P.p[2][k], b1 = P.p[3][k];
            const double wk = lm_weight<W>(wt, k);
            {
                const double rr = sampson_res(ctx, a0, a1, b0, b1);
                lsum += wmul<W>(wk, L.loss(rr * rr));
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
            A.template add1<W>(L, r, J, wk);
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

// Tangent-Sampson row of one correspondence for CameraRelativePoseRefiner::compute_jacobian (optim/relative.h:333-437):
// the pose columns tr[0..5) and the camera columns tr[5 ..) of the tile row, from the pixels (a0, a1), (b0, b1), the
// bearings d1, d2 and the unprojection Jacobians M1, M2 at cameras c1, c2, C and J_C of tangent_terms.  The jac_params
// of both points are staged at st (d1_p) and st + 3 * CAM_MAX_PARAMS (d2_p); st + 6 * CAM_MAX_PARAMS is the scratch of
// the finite-difference points.  Operation order of the reference on mini-Eigen (products and dots left to right).
template <int NP, bool X = false>
PLB_DEV void ts_cam_row(const double *E, const double *D, const CamDev &c1, const CamDev &c2, double a0, double a1,
                        double b0, double b1, const double *d1, const double *d2, const double *M1, const double *M2,
                        double C, const double *JC, const int (*idx)[CAM_MAX_PARAMS], const int *m, double *st,
                        double *tr) {
    const double nJ_C = sqrt((JC[0] * JC[0] + JC[2] * JC[2]) + (JC[1] * JC[1] + JC[3] * JC[3]));
    const double inv = 1.0 / nJ_C;
    const double s = C * inv * inv;
    {
        double dF[9];
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int rr = 0; rr < 3; ++rr) {
                double e = d1[c] * d2[rr];
                e -= s * (JC[0] * M1[2 * c] * d2[rr] + JC[1] * M1[2 * c + 1] * d2[rr] + JC[2] * M2[2 * rr] * d1[c] +
                          JC[3] * M2[2 * rr + 1] * d1[c]);
                dF[3 * c + rr] = e * inv;
            }
#pragma unroll
        for (int p = 0; p < 5; ++p) {
            double t = 0.0;
#pragma unroll
            for (int q = 0; q < 9; ++q) t += dF[q] * D[5 * q + p];
            tr[p] = t;
        }
    }
    constexpr double eps = 1e-6;
    const double sig = (-s) * inv; // -s * inv_nJ_C of J_M11 .. J_M22
    double *tmp = st + 6 * CAM_MAX_PARAMS;
    int col = 5;
#pragma unroll 1
    for (int cam = 0; cam < 2; ++cam) {
        // this camera's point d, its partner's point e, its M and the partner's M: J_d = (e^T G - s (d^T G^T Mo Mo^T G)) inv
        // with G = E (camera 1) or E^T (camera 2); J_Mq = sig * Mc.col(q)^T G^T e e^T G
        const double *d = cam ? d2 : d1, *e = cam ? d1 : d2, *Mc = cam ? M2 : M1, *Mo = cam ? M1 : M2;
        auto G = [&](int r, int c) { return cam ? E[3 * c + r] : E[3 * r + c]; };
        double Jd[3], JM[2][3];
        {
            double a[3], b[2], c[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) a[j] = d[0] * G(j, 0) + d[1] * G(j, 1) + d[2] * G(j, 2); // d^T G^T
#pragma unroll
            for (int q = 0; q < 2; ++q) b[q] = a[0] * Mo[q] + a[1] * Mo[2 + q] + a[2] * Mo[4 + q];
#pragma unroll
            for (int j = 0; j < 3; ++j) c[j] = b[0] * Mo[2 * j] + b[1] * Mo[2 * j + 1];
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const double eg = e[0] * G(0, j) + e[1] * G(1, j) + e[2] * G(2, j);
                const double cg = c[0] * G(0, j) + c[1] * G(1, j) + c[2] * G(2, j);
                Jd[j] = (eg - s * cg) * inv;
            }
        }
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            double g[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) g[k] = sig * Mc[2 * k + q];
            double h[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) h[j] = g[0] * G(j, 0) + g[1] * G(j, 1) + g[2] * G(j, 2); // (..) G^T
            const double hs = h[0] * e[0] + h[1] * e[1] + h[2] * e[2];
            double u[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) u[k] = hs * e[k];
#pragma unroll
            for (int j = 0; j < 3; ++j) JM[q][j] = u[0] * G(0, j) + u[1] * G(1, j) + u[2] * G(2, j);
        }
        const CamDev &cc = cam ? c2 : c1;
        const double *dp = st + 3 * CAM_MAX_PARAMS * cam;
        const double x0 = cam ? b0 : a0, x1 = cam ? b1 : a1;
        for (int i = 0; i < m[cam]; ++i) {
            const int j = idx[cam][i];
            tr[col + i] = Jd[0] * dp[j] + Jd[1] * dp[CAM_MAX_PARAMS + j] + Jd[2] * dp[2 * CAM_MAX_PARAMS + j];
        }
#pragma unroll 1
        for (int q = 0; q < 2; ++q) { // x + eps e_q: dp_e = (jac_params(x + eps e_q) - d_p) / eps
            double dd[3], dM[6];
            cam_unproject_with_jac_params<X>(cc, q == 0 ? x0 + eps : x0, q == 1 ? x1 + eps : x1, dd, dM, tmp);
            for (int i = 0; i < m[cam]; ++i) {
                const int j = idx[cam][i];
                double f[3];
#pragma unroll
                for (int r = 0; r < 3; ++r) f[r] = (tmp[CAM_MAX_PARAMS * r + j] - dp[CAM_MAX_PARAMS * r + j]) / eps;
                tr[col + i] += JM[q][0] * f[0] + JM[q][1] * f[1] + JM[q][2] * f[2];
            }
        }
        col += m[cam];
    }
    for (; col < NP; ++col) tr[col] = 0.0;
}

// One evaluation pass at the pose whose context is in S->ctx and the camera parameters cp[i] of camera i: robust cost
// and residual rows (compute_residual) and JtJ, Jtr, jacobian rows (compute_jacobian) -> S->tot, in lm_eval_pass's
// layout.
//   PnP : <Model>::project / project_with_jac with jac_params (optim/absolute.h:55-143)
//   TS  : unproject_with_jac of both pixels at the (trial) cameras, the tangent Sampson residual, the pose columns of
//         the fixed-camera refiner and the camera columns of ts_cam_row (optim/relative.h:289-441)
// Every 256 points each thread writes its point's row of the tile; thread e < NV then adds value e of every row in point
// order.  Order of the sums: points in order inside a CTA, CTAs in rank order (deterministic for a given cluster size).
// W: the residual weights of lm_eval_pass, folded into the row's loss and w columns.
template <int KIND, bool X = false, bool W = false>
PLB_DEV void lmi_eval_pass(const ProblemDev &P, const LossFn &L, const double *wt, const CamDev *cams,
                           const double (*cp)[CAM_MAX_PARAMS], const int *m, const int (*idx)[CAM_MAX_PARAMS],
                           const int *list, int lo, int na, LmCamShared<KIND> *S, double *tile, int &buf, int csize) {
    using Y = LmCamLayout<KIND>;
    constexpr int NP = Y::NP, NC = Y::NCAM;
    const double *ctx = S->ctx;
    CamDev cam[NC];
#pragma unroll
    for (int i = 0; i < NC; ++i) {
        cam[i].model = cams[i].model;
        cam[i].reserved = 0;
#pragma unroll
        for (int c = 0; c < CAM_MAX_PARAMS; ++c) cam[i].p[c] = cp[i][c];
    }
    // the value this thread owns: kind 0 column sum of column a, 1 JtJ(a, b), 2 Jtr(a), -1 none (or a padded entry)
    int np = Y::NPOSE;
#pragma unroll
    for (int i = 0; i < NC; ++i) np += m[i];
    const int e = threadIdx.x;
    int kind = -1, a = 0, b = 0;
    if (e == 0) {
        kind = 0; a = Y::LOSS;
    } else if (e == 1) {
        kind = 0; a = Y::ROW;
    } else if (e < 2 + Y::NT) {
        const int t = e - 2;
        while ((a + 1) * (a + 2) / 2 <= t) ++a;
        b = t - a * (a + 1) / 2;
        if (a < np) kind = 1;
    } else if (e < 2 + Y::NT + NP) {
        a = e - 2 - Y::NT;
        if (a < np) kind = 2;
    } else if (e == Y::NV - 1) {
        kind = 0; a = Y::JROW;
    }
    double acc = 0.0;
    for (int t0 = 0; t0 < na; t0 += (int)blockDim.x) {
        const int i = t0 + threadIdx.x;
        double *tr = tile + (size_t)threadIdx.x * Y::W;
        bool filled = false;
        tr[Y::LOSS] = 0.0;
        tr[Y::ROW] = 0.0;
        tr[Y::JROW] = 0.0;
        if (i < na) {
            const int k = list ? list[i] : lo + i;
            if constexpr (KIND == KIND_PNP) {
                const double X0 = P.p[2][k], X1 = P.p[3][k], X2 = P.p[4][k];
                const double Z0 = ctx[0] * X0 + ctx[1] * X1 + ctx[2] * X2 + ctx[9];
                const double Z1 = ctx[3] * X0 + ctx[4] * X1 + ctx[5] * X2 + ctx[10];
                const double Z2 = ctx[6] * X0 + ctx[7] * X1 + ctx[8] * X2 + ctx[11];
                if (!(Z2 < 0)) { // optim/absolute.h:57-58,93-94
                    const double wk = lm_weight<W>(wt, k);
                    double xr0, xr1, zp0, zp1, Jp[2][3];
                    cam_project<X>(cam[0], Z0, Z1, Z2, xr0, xr1);
                    cam_project_with_jac<X>(cam[0], Z0, Z1, Z2, zp0, zp1, &Jp[0][0]);
                    const double x0 = P.p[0][k], x1 = P.p[1][k];
                    const double q0 = xr0 - x0, q1 = xr1 - x1;
                    tr[Y::LOSS] = wmul<W>(wk, L.loss(q0 * q0 + q1 * q1));
                    tr[Y::ROW] = 1.0;
                    const double r0 = zp0 - x0, r1 = zp1 - x1;
                    const double w = wmul<W>(wk, L.weight(r0 * r0 + r1 * r1));
                    if (w != 0) { // jacobian_accumulator.h:87-104
                        filled = true;
                        tr[Y::JROW] = 1.0;
                        tr[Y::WT] = w;
                        tr[Y::WR] = w * r0;
                        tr[Y::WR + 1] = w * r1;
#pragma unroll
                        for (int q = 0; q < 2; ++q) {
                            double dZ[3];
#pragma unroll
                            for (int c = 0; c < 3; ++c)
                                dZ[c] = Jp[q][0] * ctx[c] + Jp[q][1] * ctx[3 + c] + Jp[q][2] * ctx[6 + c];
                            double *Jr = tr + q * NP;
                            Jr[0] = -X2 * dZ[1] + X1 * dZ[2];
                            Jr[1] = X2 * dZ[0] - X0 * dZ[2];
                            Jr[2] = -X1 * dZ[0] + X0 * dZ[1];
                            Jr[3] = dZ[0]; Jr[4] = dZ[1]; Jr[5] = dZ[2];
                        }
                        // J.col(6 + c) = J_params.col(camera_refine_idx[c]); jac_params is staged in the row's tail
                        cam_jac_params<X>(cam[0], Z0, Z1, Z2, tr + Y::JP);
#pragma unroll
                        for (int c = 0; c < NP - 6; ++c) {
                            tr[6 + c] = c < m[0] ? tr[Y::JP + idx[0][c]] : 0.0;
                            tr[NP + 6 + c] = c < m[0] ? tr[Y::JP + CAM_MAX_PARAMS + idx[0][c]] : 0.0;
                        }
                    }
                }
            } else { // KIND_RELPOSE_TS
                const double a0 = P.p[0][k], a1 = P.p[1][k], b0 = P.p[2][k], b1 = P.p[3][k];
                const double wk = lm_weight<W>(wt, k);
                double d1[3], d2[3], M1[6], M2[6];
                cam_unproject_with_jac_params<X>(cam[0], a0, a1, d1, M1, tr + Y::JP);
                cam_unproject_with_jac_params<X>(cam[1], b0, b1, d2, M2, tr + Y::JP + 3 * CAM_MAX_PARAMS);
                double C, JC[4];
                tangent_terms(ctx, d1, d2, M1, M2, C, JC);
                {
                    const double nJc_sq = (JC[2] * JC[2] + JC[3] * JC[3]) + (JC[0] * JC[0] + JC[1] * JC[1]);
                    const double rr = C / sqrt(nJc_sq);
                    tr[Y::LOSS] = wmul<W>(wk, L.loss(rr * rr));
                    tr[Y::ROW] = 1.0;
                }
                const double nJ_C = sqrt((JC[0] * JC[0] + JC[2] * JC[2]) + (JC[1] * JC[1] + JC[3] * JC[3]));
                const double r = C * (1.0 / nJ_C);
                const double w = wmul<W>(wk, L.weight(r * r));
                if (w != 0) { // jacobian_accumulator.h:125-141
                    filled = true;
                    tr[Y::JROW] = 1.0;
                    tr[Y::WT] = w;
                    tr[Y::WR] = w * r;
                    ts_cam_row<NP, X>(ctx, ctx + 9, cam[0], cam[1], a0, a1, b0, b1, d1, d2, M1, M2, C, JC, idx, m,
                                   tr + Y::JP, tr);
                }
            }
        }
        if (!filled) { // no Jacobian contribution: a zero row (reference: add_jacobian returns early)
            for (int c = 0; c < Y::R * NP; ++c) tr[c] = 0.0;
            tr[Y::WT] = 0.0;
#pragma unroll
            for (int q = 0; q < Y::R; ++q) tr[Y::WR + q] = 0.0;
        }
        __syncthreads();
        const int rows = min_i((int)blockDim.x, na - t0);
        if (kind == 0) {
            for (int r = 0; r < rows; ++r) acc += tile[r * Y::W + a];
        } else if (kind == 1) {
            for (int r = 0; r < rows; ++r) {
                const double *q = tile + r * Y::W;
                if constexpr (Y::R == 2) acc += q[Y::WT] * (q[a] * q[b] + q[NP + a] * q[NP + b]);
                else acc += q[Y::WT] * (q[a] * q[b]);
            }
        } else if (kind == 2) {
            for (int r = 0; r < rows; ++r) {
                const double *q = tile + r * Y::W;
                if constexpr (Y::R == 2) acc += q[a] * q[Y::WR] + q[NP + a] * q[Y::WR + 1];
                else acc += q[a] * q[Y::WR];
            }
        }
        __syncthreads();
    }
    if (e < Y::NV) S->sums[buf][e] = acc;
    cluster_total(S, Y::NV, buf, csize);
}

// Lower Cholesky solve of (A) x = rhs, n x n row-major, only the lower triangle of A read and the factor written over it
// (jacobian_accumulator.h:145-154).  Unrolled for the fixed-camera sizes (n <= 8): the step is on the critical path of
// every LM iteration, and as loops over shared memory it makes the LO of small problems half as slow again.  The 14 x 14
// camera system stays a loop: unrolled, it would take the registers of the evaluation pass (spills).
PLB_DEV void llt_solve_n(double *A, const double *rhs, double *x, int n) {
#pragma unroll 8
    for (int j = 0; j < n; ++j) {
        double d = A[j * n + j];
#pragma unroll 8
        for (int k = 0; k < j; ++k) d -= A[j * n + k] * A[j * n + k];
        const double ljj = sqrt(d);
        A[j * n + j] = ljj;
#pragma unroll 8
        for (int i = j + 1; i < n; ++i) {
            double s = A[i * n + j];
#pragma unroll 8
            for (int k = 0; k < j; ++k) s -= A[i * n + k] * A[j * n + k];
            A[i * n + j] = s / ljj;
        }
    }
#pragma unroll 8
    for (int i = 0; i < n; ++i) {
        double s = rhs[i];
#pragma unroll 8
        for (int k = 0; k < i; ++k) s -= A[i * n + k] * x[k];
        x[i] = s / A[i * n + i];
    }
#pragma unroll 8
    for (int i = n - 1; i >= 0; --i) {
        double s = x[i];
#pragma unroll 8
        for (int k = i + 1; k < n; ++k) s -= A[k * n + i] * x[k];
        x[i] = s / A[i * n + i];
    }
}

// The points k of this CTA's slice [lo, hi) with keep(k), in point order -> list; returns their number.
template <class Shared, class Keep> PLB_DEV int lm_compact(Shared *S, int lo, int hi, int *list, Keep keep) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int base = 0;
    for (int t0 = lo; t0 < hi; t0 += (int)blockDim.x) {
        const int k = t0 + threadIdx.x;
        const bool kept = k < hi && keep(k);
        const unsigned bal = __ballot_sync(0xffffffffu, kept);
        if (lane == 0) S->wcount[warp] = __popc(bal);
        __syncthreads();
        int off = base;
        for (int w = 0; w < warp; ++w) off += S->wcount[w];
        int tile = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tile += S->wcount[w];
        if (kept) list[off + __popc(bal & ((1u << lane) - 1u))] = k;
        base += tile;
        __syncthreads();
    }
    return base;
}

// One thread-block CLUSTER per job (1..8 CTAs of 256 threads, DSMEM reductions); CTA r owns the correspondences
// [r*chunk, (r+1)*chunk).  Every CTA runs the scalar LM logic (optim/lm_impl.h:56-140) redundantly on identical
// cluster totals, so no broadcast between CTAs is needed.  The reference evaluates the residual of a trial step and,
// if accepted, the Jacobian at the same parameters in a second pass; here both come from one pass.
// Two refiners: the fixed-camera one of every kind (lm_eval_pass: per-thread packed normal equations, cluster_sum), and
// CAM, the refiner with camera parameters (lmi_eval_pass: the shared-memory tile summed in point order, which ~255
// registers of per-thread accumulators for 14 or 21 parameters would not leave room for):
//   KIND_PNP        AbsolutePoseRefiner, KIND_RELPOSE_TS CameraRelativePoseRefiner: the parameters
//                   cam_refine_idx(P.cam[i].model, job.cam_refine) of every camera P.cam[i] of the job's problem
// CAM writes camera i of job j to cam_outs[(j * kind_cam_count(KIND) + i) * CAM_MAX_PARAMS ..].
template <int KIND, bool CAM> struct LmNP { static constexpr int v = LmDims<KIND>::NP; };
template <int KIND> struct LmNP<KIND, true> { static constexpr int v = LmCamLayout<KIND>::NP; };
template <int KIND, bool CAM, bool X = false, bool W = false>
__global__ void __launch_bounds__(LM_THREADS, 1)
    k_lm(const ProblemDev *__restrict__ probs, const LmJob *__restrict__ jobs, const LoJobSrc *__restrict__ job_src,
         const double *__restrict__ models_in, const int *__restrict__ n_jobs_dev, int n_jobs, const char *mask_base,
         int *idx_scratch, int scratch_stride, LmJobOut *outs, double *cam_outs) {
    static_assert(!CAM || KIND == KIND_PNP || KIND == KIND_RELPOSE_TS, "camera refinement: absolute and tangent-Sampson relative pose");
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    constexpr int NP = LmNP<KIND, CAM>::v;
    constexpr int NT = NP * (NP + 1) / 2;
    constexpr int MSZ = kind_model_size(KIND);
    __shared__ std::conditional_t<CAM, LmCamShared<KIND>, LmShared<NP>> S;
    extern __shared__ double lmi_tile[]; // CAM: LmCamLayout<KIND>::TILE_BYTES
    const int csize = (int)cluster.num_blocks(), crank = (int)cluster.block_rank();
    // The grid is a set of clusters that walk the job list: explicit jobs (jobs[j], model j of models_in, stride 9) or
    // the LO jobs k_pass1 listed on the device (template jobs[job_src[j].pidx], model slot job_src[j].slot of the
    // round's model list, stride MSZ; the count is read from device memory and clamped to n_jobs).  For the LO launch of
    // a round n_jobs_dev is &ctl[CTL_JOB_TOTAL] of the round's control words: a round whose records overflowed
    // (CTL_FLAGS: k_pass1 left job entries unwritten) is redone by the host, so no job of it runs.
    const int n_clusters = (int)gridDim.x / csize, cluster_id = (int)blockIdx.x / csize;
    int nj = n_jobs;
    if (n_jobs_dev) {
        const int v = n_jobs_dev[CTL_FLAGS - CTL_JOB_TOTAL] != 0 ? 0 : n_jobs_dev[0];
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
        double C[kind_ctx_size(KIND_RELPOSE)];
        if (KIND == KIND_RELPOSE && prm.subset_mode == 1) model_ctx<KIND_RELPOSE>(min, C);
        na = lm_compact(&S, lo, hi, mylist, [&](int k) {
            if (prm.subset_mode == 2) return mask_in[k] != 0;
            if (KIND != KIND_RELPOSE) return false;
            // relpose LO subset: inliers of the start pose at 5*thr^2 (estimators/relative_pose.cc:62-86)
            double v[kind_corr_size(KIND_RELPOSE)];
            load_corr<KIND_RELPOSE>(P, k, v);
            return is_inlier<KIND_RELPOSE>(C, v, prm.subset_sq_thr);
        });
        list = mylist;
        __syncthreads();
        if constexpr (KIND == KIND_RELPOSE) {
            if (prm.subset_mode == 1) {
                double c[1] = {threadIdx.x == 0 ? (double)na : 0.0};
                cluster_sum<1>(&S, c, buf, csize);
                untouched = !(S.tot[0] > 5.0);
            }
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
        if constexpr (CAM) {
            for (int i = 0; i < kind_cam_count(KIND); ++i) {
                for (int c = 0; c < CAM_MAX_PARAMS; ++c) S.cam[i][c] = P.cam[i].p[c];
                for (int c = 0; c < CAM_MAX_PARAMS; ++c) S.idx[i][c] = 0;
                S.m[i] = cam_refine_idx(P.cam[i].model, J.cam_refine, S.idx[i]);
            }
        }
    }
    __syncthreads();
    constexpr int NC = kind_cam_count(KIND);
    // CAM: the cameras' models and refined parameters, in registers for the evaluation pass
    int m[NC] = {}, idx[NC][CAM_MAX_PARAMS];
    CamDev cams[NC];
    if constexpr (CAM) {
#pragma unroll
        for (int i = 0; i < NC; ++i) {
            cams[i].model = P.cam[i].model;
            m[i] = S.m[i];
#pragma unroll
            for (int c = 0; c < CAM_MAX_PARAMS; ++c) idx[i][c] = S.idx[i][c];
        }
    }
    // one evaluation pass at par (trial: par_new), totals in S.tot
    const double *wt = W ? J.w : nullptr;
    auto eval = [&](bool trial) {
        if constexpr (CAM)
            lmi_eval_pass<KIND, X, W>(P, L, wt, cams, trial ? S.cam_new : S.cam, m, idx, list, lo, na, &S, lmi_tile, buf,
                                      csize);
        else
            lm_eval_pass<KIND, X, W>(P, L, wt, list, lo, na, &S, buf, csize);
    };

    int iterations = 0;
    double cost = 0.0, initial_cost = 0.0;
    if (!untouched) {
        // scalar LM state (thread 0 of every CTA); rc mirrors NormalAccumulator::residual_count
        double lambda = prm.initial_lambda, nu = 2.0, rc = 0.0;
        bool recompute_jac = true;
        if (threadIdx.x == 0) lm_build_ctx<KIND>(S.par, S.ctx, S.tb, true);
        __syncthreads();
        eval(false);
        if (threadIdx.x == 0) {
            cost = S.tot[0] * (1.0 / fmax(1.0, S.tot[1])); // acc.get_residual() after the residual pass
            initial_cost = cost;
            int t = 0;
            for (int i = 0; i < NP; ++i)
                for (int j = 0; j <= i; ++j) S.JtJ[i * NP + j] = S.tot[2 + t++];
            for (int i = 0; i < NP; ++i) S.Jtr[i] = S.tot[2 + NT + i];
            rc = S.tot[2 + NT + NP]; // residual_count after the Jacobian pass
        }
        for (int it = 0; it < prm.max_iterations; ++it) {
            iterations = it;
            int stop = 0;
            if (threadIdx.x == 0) {
                if (recompute_jac) {
                    double g = 0.0;
                    for (int i = 0; i < NP; ++i) g += S.Jtr[i] * S.Jtr[i];
                    const double grad_norm = (1.0 / fmax(1.0, rc)) * sqrt(g);
                    if (grad_norm < prm.gradient_tol) stop = 1;
                }
                if (!stop) {
                    const double scale = 1.0 / fmax(1.0, rc);
                    for (int i = 0; i < NP; ++i)
                        for (int j = 0; j <= i; ++j) S.Am[i * NP + j] = scale * S.JtJ[i * NP + j];
                    for (int i = 0; i < NP; ++i) S.Am[i * NP + i] += lambda;
                    for (int i = 0; i < NP; ++i) S.rhs[i] = -(scale * S.Jtr[i]);
                    llt_solve_n(S.Am, S.rhs, S.sol, NP);
                    double sn = 0.0;
                    for (int i = 0; i < NP; ++i) sn += S.sol[i] * S.sol[i];
                    if (sqrt(sn) < prm.step_tol) stop = 1;
                }
                if (!stop) {
                    lm_step<KIND>(S.par, S.sol, S.tb, S.par_new);
                    if constexpr (CAM) { // AbsolutePoseRefiner::step (optim/absolute.h:146-160), relative.h:443-468
                        int off = LmCamDims<KIND>::NPOSE;
                        for (int i = 0; i < NC; ++i) {
                            for (int c = 0; c < CAM_MAX_PARAMS; ++c) S.cam_new[i][c] = S.cam[i][c];
                            for (int c = 0; c < S.m[i]; ++c) S.cam_new[i][S.idx[i][c]] += S.sol[off + c];
                            off += S.m[i];
                        }
                    }
                    lm_build_ctx<KIND>(S.par_new, S.ctx, S.tb_new, true);
                }
            }
            if (block_bcast(&S, stop)) break;
            eval(true);
            int brk = 0;
            if (threadIdx.x == 0) {
                rc = S.tot[1]; // residual_count after the residual pass of the trial point
                const double cost_new = S.tot[0] * (1.0 / fmax(1.0, rc));
                if (cost_new < cost) {
                    const double cost_decrease = cost - cost_new;
                    for (int k = 0; k < 9; ++k) S.par[k] = S.par_new[k];
                    for (int k = 0; k < 6; ++k) S.tb[k] = S.tb_new[k];
                    if constexpr (CAM)
                        for (int i = 0; i < NC; ++i)
                            for (int c = 0; c < CAM_MAX_PARAMS; ++c) S.cam[i][c] = S.cam_new[i][c];
                    cost = cost_new;
                    recompute_jac = true;
                    const double scale = 1.0 / fmax(1.0, rc);
                    double pred = 0.0;
                    for (int i = 0; i < NP; ++i) pred += S.sol[i] * (lambda * S.sol[i] + scale * S.Jtr[i]);
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
                        for (int j = 0; j <= i; ++j) S.JtJ[i * NP + j] = S.tot[2 + t++];
                    for (int i = 0; i < NP; ++i) S.Jtr[i] = S.tot[2 + NT + i];
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
            if constexpr (CAM)
                for (int i = 0; i < NC; ++i)
                    for (int c = 0; c < CAM_MAX_PARAMS; ++c) cam_outs[((size_t)job * NC + i) * CAM_MAX_PARAMS + c] = S.cam[i][c];
        }
    }
    __syncthreads();
    if constexpr (!CAM) {
        if (prm.score_after && crank == 0) {
            double mdl[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) mdl[k] = S.par_new[k];
            cta_score<KIND>(P, mdl, S.sred, &out->count, &out->score);
        }
    }
    cluster.sync(); // no CTA may exit (or start the next job) while a sibling can still read its shared memory
    } // jobs of this cluster
}

// k_lm needs ~255 registers per thread: one 256-thread CTA (one job, or one slice of a job's cluster) per SM.
static thread_local int t_lm_sm_share = 50;
void lm_set_sm_share(int pct) { t_lm_sm_share = (pct > 0 && pct <= 100) ? pct : 50; }
static int lm_cluster_size(int n_jobs, int max_n, int share = t_lm_sm_share) {
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
    const int sm_share = forced ? forced : share;
    while (csize > 1 && n_jobs * csize > sm_count() * sm_share / 100) csize /= 2;
    return csize;
}
// A grid of n_clusters clusters of csize CTAs over a job list: k_lm<kind> of the fixed-camera refiner, or with
// refine_camera the refiner with camera parameters of the kind (KIND_PNP or KIND_RELPOSE_TS).
// weighted: the W instantiation (LmJob::w); the LO launches of the rounds have no weights.
static void launch_lm_any(int kind, bool refine_camera, bool xcam, const ProblemDev *probs, const LmJob *jobs,
                          const LoJobSrc *job_src, const double *models_in, const int *n_jobs_dev, int n_jobs,
                          int n_clusters, int csize, const char *mask_base, int *idx_scratch, int scratch_stride,
                          LmJobOut *out, double *cam_out, cudaStream_t stream, bool weighted = false) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)(n_clusters * csize), 1, 1);
    cfg.blockDim = dim3((unsigned)LM_THREADS, 1, 1);
    const size_t tile = !refine_camera                 ? 0
                        : kind == KIND_RELPOSE_TS ? LmCamLayout<KIND_RELPOSE_TS>::TILE_BYTES
                                                  : LmCamLayout<KIND_PNP>::TILE_BYTES;
    cfg.dynamicSmemBytes = tile;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)csize;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    auto launch = [&](auto kernel) {
        cudaLaunchKernelEx(&cfg, kernel, probs, jobs, job_src, models_in, n_jobs_dev, n_jobs, mask_base, idx_scratch,
                           scratch_stride, out, cam_out);
    };
    // xcam: a camera of the jobs is a fisheye or division model.  Only the refiners that evaluate cameras have an X
    // instantiation: the PnP refiners and the tangent-Sampson camera refiner.
    if (refine_camera) {
        auto cam_kernel = kind == KIND_RELPOSE_TS ? (xcam ? k_lm<KIND_RELPOSE_TS, true, true> : k_lm<KIND_RELPOSE_TS, true>)
                                                  : (xcam ? k_lm<KIND_PNP, true, true> : k_lm<KIND_PNP, true>);
        if (weighted)
            cam_kernel = kind == KIND_RELPOSE_TS
                             ? (xcam ? k_lm<KIND_RELPOSE_TS, true, true, true> : k_lm<KIND_RELPOSE_TS, true, false, true>)
                             : (xcam ? k_lm<KIND_PNP, true, true, true> : k_lm<KIND_PNP, true, false, true>);
        cudaFuncSetAttribute(cam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tile);
        launch(cam_kernel);
    } else if (xcam && kind == KIND_PNP) {
        launch(weighted ? k_lm<KIND_PNP, false, true, true> : k_lm<KIND_PNP, false, true>);
    } else {
        with_kind(kind, [&](auto K) { launch(weighted ? k_lm<K, false, false, true> : k_lm<K, false>); });
    }
}
void launch_lm(int kind, bool refine_camera, bool xcam, bool weighted, const ProblemDev *probs, const LmJob *jobs_dev,
               const double *models_in, int n_jobs, int max_n, const char *mask_base, int *idx_scratch,
               int scratch_stride, LmJobOut *out, double *cam_out, cudaStream_t stream) {
    if (n_jobs <= 0) return;
    const int csize = lm_cluster_size(n_jobs, max_n);
    launch_lm_any(kind, refine_camera, xcam, probs, jobs_dev, nullptr, models_in, nullptr, n_jobs, n_jobs, csize, mask_base,
                  idx_scratch, scratch_stride, out, cam_out, stream, weighted);
}
int lm_lone_width(int n) { return lm_cluster_size(1, n, 100); }
void launch_lm_width(int kind, bool refine_camera, bool xcam, bool weighted, const ProblemDev *probs,
                     const LmJob *jobs_dev, const double *models_in, int n_jobs, int csize, LmJobOut *out,
                     double *cam_out, cudaStream_t stream) {
    if (n_jobs <= 0) return;
    const int nc = std::max(1, std::min(n_jobs, sm_count() / csize));
    launch_lm_any(kind, refine_camera, xcam, probs, jobs_dev, nullptr, models_in, nullptr, n_jobs, nc, csize, nullptr,
                  nullptr, 0, out, cam_out, stream, weighted);
}
// Clusters of a round's LO launch: at most one wave (a k_lm CTA owns an SM), at most the estimated number of jobs.
int lm_round_max_clusters(int kind, int est_jobs, int max_n) {
    (void)kind;
    if (est_jobs < 1) est_jobs = 1;
    const int csize = lm_cluster_size(est_jobs, max_n);
    int nc = sm_count() / csize;
    if (nc > est_jobs) nc = est_jobs;
    return nc < 1 ? 1 : nc;
}
void launch_lm_round(int kind, const ProblemDev *probs, const LmJob *tmpl, const LoJobSrc *job_src,
                     const double *models, const int *n_jobs_dev, int job_cap, int est_jobs, int max_n,
                     int *idx_scratch, int scratch_stride, LmJobOut *out, cudaStream_t stream) {
    if (est_jobs < 1) est_jobs = 1;
    const int csize = lm_cluster_size(est_jobs, max_n);
    const int nc = lm_round_max_clusters(kind, est_jobs, max_n);
    launch_lm_any(kind, false, false, probs, tmpl, job_src, models, n_jobs_dev, job_cap, nc, csize, nullptr, idx_scratch,
                  scratch_stride, out, nullptr, stream);
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
// direct solver surface (solvers/*.h): one thread per instance, the solver code of the round kernels
// ============================================================================================================
// p3p (variant 0) / p3p_lambdatwist (variant 1), homography_4pt and relpose_7pt; every output slot is written, unused
// ones with zeros.  relpose_7pt runs without the real-focal check.
template <int KIND, int VARIANT>
__global__ void __launch_bounds__(K7L_THREADS)
    k_solver_batch(size_t count, const double *__restrict__ a, const double *__restrict__ b, double *out, int *n_out,
                   int flags) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    if constexpr (KIND == KIND_PNP) {
        d3 xs[3], Xs[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            xs[k] = mk(a[9 * i + 3 * k], a[9 * i + 3 * k + 1], a[9 * i + 3 * k + 2]);
            Xs[k] = mk(b[9 * i + 3 * k], b[9 * i + 3 * k + 1], b[9 * i + 3 * k + 2]);
        }
        double models[28];
        const int n = (VARIANT == 1) ? solve_p3p_lambdatwist(xs, Xs, models) : solve_p3p(xs, Xs, models);
#pragma unroll
        for (int e = 0; e < 28; ++e) out[28 * i + e] = (e < 7 * n) ? models[e] : 0.0;
        n_out[i] = n;
    } else if constexpr (KIND == KIND_HOMOG) {
        d3 xa[4], xb[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            xa[k] = mk(a[12 * i + 3 * k], a[12 * i + 3 * k + 1], a[12 * i + 3 * k + 2]);
            xb[k] = mk(b[12 * i + 3 * k], b[12 * i + 3 * k + 1], b[12 * i + 3 * k + 2]);
        }
        double H[9];
        const int n = solve_h4(xa, xb, H, flags != 0);
#pragma unroll
        for (int k = 0; k < 9; ++k) out[9 * i + k] = n ? H[k] : 0.0;
        n_out[i] = n;
    } else {
        static_assert(KIND == KIND_FUND, "relpose_5pt runs on the phase kernels");
        extern __shared__ __align__(16) unsigned char smem_raw[];
        double *W = reinterpret_cast<double *>(smem_raw) + (size_t)threadIdx.x * K7L_STRIDE;
        double x1s[21], x2s[21];
#pragma unroll
        for (int e = 0; e < 21; ++e) {
            x1s[e] = a[21 * i + e];
            x2s[e] = b[21 * i + e];
        }
        double F[3][9];
        const int n = fundamental_7pt(x1s, x2s, W, [](const double *) { return true; }, F);
#pragma unroll
        for (int m = 0; m < 3; ++m)
#pragma unroll
            for (int k = 0; k < 9; ++k) out[27 * i + 9 * m + k] = (m < n) ? F[m][k] : 0.0;
        n_out[i] = n;
    }
}

// relpose_5pt: the caller's bearings (5 x 3 doubles per side and instance) into entries 75..104 of the entry-major
// per-instance block, where k5_null and k5_back expect the sample's bearings.
__global__ void __launch_bounds__(256) k5_load(int n, const double *__restrict__ a, const double *__restrict__ b,
                                               HypOut s5) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n) return;
    double *blk = s5.s5_blk + g;
#pragma unroll
    for (int e = 0; e < 15; ++e) {
        blk[(size_t)(75 + e) * n] = a[(size_t)g * 15 + e];
        blk[(size_t)(90 + e) * n] = b[(size_t)g * 15 + e];
    }
}

// relpose_5pt output, one thread per instance: per root, the back-substitution of k5_back.  Variant 0: up to 10 E
// (column-major, 90 doubles); variant 1: the poses of motions_from_E in the reference's order (E-major, then the four
// candidates; 280 doubles).  Unused slots are zeroed.
template <int VARIANT>
__global__ void __launch_bounds__(128) k5_solver_out(int n, HypOut s5, double *out, int *n_out) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n) return;
    const StridedD blk{s5.s5_blk + g, (size_t)n};
    const int nr = s5.s5_nroots[g];
    const double *roots = s5.s5_roots + (size_t)g * 10;
    if constexpr (VARIANT == 0) {
        double *o = out + (size_t)g * 90;
        for (int m = 0; m < 10; ++m) {
            double E[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
            if (m < nr) backsub_5pt(blk, blk + 39, roots[m], E);
#pragma unroll
            for (int k = 0; k < 9; ++k) o[9 * m + k] = E[3 * (k % 3) + k / 3];
        }
        n_out[g] = nr;
    } else {
        double *o = out + (size_t)g * 280;
        int pos = 0;
        for (int r = 0; r < nr; ++r) {
            double E[9], cand[4][7];
            backsub_5pt(blk, blk + 39, roots[r], E);
            const unsigned mask = motions_from_E(E, blk + 75, blk + 90, 5, cand);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                if (mask & (1u << c)) {
#pragma unroll
                    for (int k = 0; k < 7; ++k) o[7 * pos + k] = cand[c][k];
                    ++pos;
                }
            }
        }
        for (int e = 7 * pos; e < 280; ++e) o[e] = 0.0;
        n_out[g] = pos;
    }
}

template <int KIND, int VARIANT>
static void launch_solver_t(size_t count, const double *a, const double *b, double *out, int *n_out, int flags,
                            cudaStream_t stream) {
    size_t smem = 0;
    if constexpr (KIND == KIND_FUND) {
        smem = K7L_SMEM;
        static bool attr_set[MAX_DEVICES] = {false};
        if (!attr_set[cur_dev()]) {
            cudaFuncSetAttribute(k_solver_batch<KIND, VARIANT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            attr_set[cur_dev()] = true;
        }
    }
    k_solver_batch<KIND, VARIANT><<<(unsigned)((count + K7L_THREADS - 1) / K7L_THREADS), K7L_THREADS, smem, stream>>>(
        count, a, b, out, n_out, flags);
}
int launch_solver_batch(int kind, int variant, size_t count, const double *a, const double *b, double *out, int *n_out,
                        int flags, const HypOut &s5, cudaStream_t stream) {
    if (count == 0) return 0;
    switch (kind) {
    case KIND_PNP:
        if (variant == 0) launch_solver_t<KIND_PNP, 0>(count, a, b, out, n_out, flags, stream);
        else launch_solver_t<KIND_PNP, 1>(count, a, b, out, n_out, flags, stream);
        return 1;
    case KIND_RELPOSE: {
        const int n = (int)count; // the s5 buffers of `count` instances bound it far below INT_MAX
        RoundDesc R{};
        R.n_total = n;
        k5_load<<<(n + 255) / 256, 256, 0, stream>>>(n, a, b, s5);
        launch_5pt_prep_roots(R, s5, stream);
        if (variant == 0) k5_solver_out<0><<<(n + 127) / 128, 128, 0, stream>>>(n, s5, out, n_out);
        else k5_solver_out<1><<<(n + 127) / 128, 128, 0, stream>>>(n, s5, out, n_out);
        return 5;
    }
    case KIND_FUND: launch_solver_t<KIND_FUND, 0>(count, a, b, out, n_out, flags, stream); return 1;
    default: launch_solver_t<KIND_HOMOG, 0>(count, a, b, out, n_out, flags, stream); return 1;
    }
}

} // namespace plb
