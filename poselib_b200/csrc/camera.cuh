// poselib_b200 — camera models of the estimate_* pre-step, evaluated on the device (row N3 of SURVEY.md §8f):
// NULL, SIMPLE_PINHOLE, PINHOLE, SIMPLE_RADIAL, RADIAL, OPENCV  (misc/camera_models.{h,cc} of the reference,
// citations relative to /root/reference/PoseLib).  Compiled with -fmad=false like the rest of the fp64 path, so the
// calibrated points / bearings / unprojection Jacobians are the doubles a baseline x86-64 build computes.
#pragma once
#include "device_math.cuh"

namespace plb {

enum { CAMM_NULL = -1, CAMM_SIMPLE_PINHOLE = 0, CAMM_PINHOLE = 1, CAMM_SIMPLE_RADIAL = 2, CAMM_RADIAL = 3, CAMM_OPENCV = 4 };

struct CamDev { // Camera: model id + parameter vector (camera_models.h:59-66)
    int model;
    int reserved;
    double p[8];
};

#define PLB_HD __host__ __device__ __forceinline__

constexpr double CAM_UNDIST_TOL = 1e-10; // camera_models.cc:41
constexpr int CAM_UNDIST_MAX_ITER = 100; // camera_models.cc:42

// undistort_poly1 / undistort_poly2 (camera_models.cc:579-613): Newton on k2 r^5 + k1 r^3 + r - rd
PLB_HD double cam_undistort_poly(double k1, double k2, bool two, double rd) {
    double r = rd;
    for (int iter = 0; iter < CAM_UNDIST_MAX_ITER; ++iter) {
        const double r2 = r * r;
        double f, fp;
        if (two) {
            f = k2 * r2 * r2 * r + k1 * r2 * r + r - rd;
            if (fabs(f) < CAM_UNDIST_TOL) break;
            fp = 5.0 * k2 * r2 * r2 + 3.0 * k1 * r2 + 1.0;
        } else {
            f = k1 * r2 * r + r - rd;
            if (fabs(f) < CAM_UNDIST_TOL) break;
            fp = 3.0 * k1 * r2 + 1.0;
        }
        r = r - f / fp;
    }
    return r;
}

// compute_opencv_distortion(_jac) (camera_models.cc:919-950)
PLB_HD void cam_opencv_distortion(const double *p, double u, double v, double &xd, double &yd) {
    const double k1 = p[4], k2 = p[5], p1 = p[6], p2 = p[7];
    const double u2 = u * u, uv = u * v, v2 = v * v;
    const double r2 = u * u + v * v;
    const double alpha = 1.0 + k1 * r2 + k2 * r2 * r2;
    xd = alpha * u + 2.0 * p1 * uv + p2 * (r2 + 2.0 * u2);
    yd = alpha * v + 2.0 * p2 * uv + p1 * (r2 + 2.0 * v2);
}
PLB_HD void cam_opencv_distortion_jac(const double *p, double u, double v, double &xd, double &yd, double *j) {
    const double k1 = p[4], k2 = p[5], p1 = p[6], p2 = p[7];
    const double r2 = u * u + v * v;
    j[0] = k2 * r2 * r2 + 6 * p2 * u + 2 * p1 * v + u * (2 * k1 * u + 4 * k2 * u * r2) + k1 * r2 + 1.0;
    j[1] = 2 * p1 * u + 2 * p2 * v + v * (2 * k1 * u + 4 * k2 * u * r2);
    j[2] = 2 * p1 * u + 2 * p2 * v + u * (2 * k1 * v + 4 * k2 * v * r2);
    j[3] = k2 * r2 * r2 + 2 * p2 * u + 6 * p1 * v + v * (2 * k1 * v + 4 * k2 * v * r2) + k1 * r2 + 1.0;
    cam_opencv_distortion(p, u, v, xd, yd);
}
// undistort_opencv (camera_models.cc:972-991): damped Newton with the closed-form 2x2 inverse
PLB_HD void cam_undistort_opencv(const double *p, double xp0, double xp1, double &x0, double &x1) {
    x0 = xp0;
    x1 = xp1;
    const double lambda = 1e-8;
    for (int iter = 0; iter < CAM_UNDIST_MAX_ITER; ++iter) {
        double xd, yd, j[4];
        cam_opencv_distortion_jac(p, x0, x1, xd, yd, j);
        j[0] += lambda;
        j[3] += lambda;
        const double res0 = xd - xp0, res1 = yd - xp1;
        if (sqrt(res0 * res0 + res1 * res1) < CAM_UNDIST_TOL) break;
        const double det = j[0] * j[3] - j[2] * j[1];
        const double invdet = 1.0 / det;
        const double i00 = j[3] * invdet, i01 = -j[1] * invdet, i10 = -j[2] * invdet, i11 = j[0] * invdet;
        x0 = x0 - (i00 * res0 + i01 * res1);
        x1 = x1 - (i10 * res0 + i11 * res1);
    }
}

PLB_HD void cam_normalize3(double *x) { // Eigen normalize()
    const double n2 = x[0] * x[0] + x[1] * x[1] + x[2] * x[2];
    if (n2 > 0) {
        const double n = sqrt(n2);
        x[0] /= n;
        x[1] /= n;
        x[2] /= n;
    }
}

// <Model>::unproject: pixel -> unit bearing (camera_models.cc:700-705,745-751,819-831,895-907,1025-1033,2724-2726)
PLB_HD void cam_unproject(const CamDev &c, double u, double v, double *x) {
    const double *p = c.p;
    switch (c.model) {
    case CAMM_NULL:
        x[0] = u; x[1] = v; x[2] = 1.0;
        return;
    case CAMM_SIMPLE_PINHOLE:
        x[0] = (u - p[1]) / p[0]; x[1] = (v - p[2]) / p[0]; x[2] = 1.0;
        cam_normalize3(x);
        return;
    case CAMM_PINHOLE:
        x[0] = (u - p[2]) / p[0]; x[1] = (v - p[3]) / p[1]; x[2] = 1.0;
        cam_normalize3(x);
        return;
    case CAMM_SIMPLE_RADIAL:
    case CAMM_RADIAL: {
        x[0] = (u - p[1]) / p[0]; x[1] = (v - p[2]) / p[0]; x[2] = 0.0;
        const double r0 = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
        if (fabs(r0) > 1e-8) {
            const double r = cam_undistort_poly(p[3], c.model == CAMM_RADIAL ? p[4] : 0.0, c.model == CAMM_RADIAL, r0);
            const double s = r / r0;
            x[0] *= s; x[1] *= s; x[2] *= s;
        }
        x[2] = 1.0;
        cam_normalize3(x);
        return;
    }
    default: { // CAMM_OPENCV
        double x0, x1;
        cam_undistort_opencv(p, (u - p[2]) / p[0], (v - p[3]) / p[1], x0, x1);
        x[0] = x0; x[1] = x1; x[2] = 1.0;
        cam_normalize3(x);
        return;
    }
    }
}

// Camera::unproject to a 2D point: the bearing, hnormalized (camera_models.h:98-102)
PLB_HD void cam_unproject2(const CamDev &c, double u, double v, double &ox, double &oy) {
    double x[3];
    cam_unproject(c, u, v, x);
    ox = x[0] / x[2];
    oy = x[1] / x[2];
}

// <Model>::project (camera_models.cc:668-671,716-720,766-772,849-857,965-970,2708-2710)
PLB_HD void cam_project(const CamDev &c, double X, double Y, double Z, double &u, double &v) {
    const double *p = c.p;
    switch (c.model) {
    case CAMM_NULL: u = X / Z; v = Y / Z; return;
    case CAMM_SIMPLE_PINHOLE: u = p[0] * X / Z + p[1]; v = p[0] * Y / Z + p[2]; return;
    case CAMM_PINHOLE: u = p[0] * X / Z + p[2]; v = p[1] * Y / Z + p[3]; return;
    case CAMM_SIMPLE_RADIAL: {
        const double inv_z = 1.0 / Z;
        const double px = X * inv_z, py = Y * inv_z;
        const double r2 = px * px + py * py;
        const double alpha = (1.0 + p[3] * r2);
        u = p[0] * alpha * px + p[1];
        v = p[0] * alpha * py + p[2];
        return;
    }
    case CAMM_RADIAL: {
        const double hx = X / Z, hy = Y / Z;
        const double r2 = hx * hx + hy * hy;
        const double alpha = (1.0 + p[3] * r2 + p[4] * r2 * r2);
        u = p[0] * alpha * hx + p[1];
        v = p[0] * alpha * hy + p[2];
        return;
    }
    default: {
        double xd, yd;
        cam_opencv_distortion(p, X / Z, Y / Z, xd, yd);
        u = p[0] * xd + p[2];
        v = p[1] * yd + p[3];
        return;
    }
    }
}

PLB_HD void cam_left_mul_2x2(const double *jd, double *J) { // J (2x3 row-major) <- jd (2x2 row-major) * J
    double o[6];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int k = 0; k < 3; ++k) o[3 * r + k] = jd[2 * r] * J[k] + jd[2 * r + 1] * J[3 + k];
#pragma unroll
    for (int k = 0; k < 6; ++k) J[k] = o[k];
}

// <Model>::project_with_jac, point Jacobian J (2x3 row-major)
// (camera_models.cc:672-699,721-744,773-818,858-893,992-1024,2711-2723)
PLB_HD void cam_project_with_jac(const CamDev &c, double X, double Y, double Z, double &u, double &v, double *J) {
    const double *p = c.p;
    switch (c.model) {
    case CAMM_NULL: {
        u = X / Z;
        v = Y / Z;
        const double z_inv = 1.0 / Z;
        J[0] = z_inv; J[1] = 0.0; J[2] = -u * z_inv;
        J[3] = 0.0; J[4] = z_inv; J[5] = -v * z_inv;
        return;
    }
    case CAMM_SIMPLE_PINHOLE:
    case CAMM_PINHOLE: {
        const bool two = c.model == CAMM_PINHOLE;
        const double fx = p[0], fy = two ? p[1] : p[0], cx = two ? p[2] : p[1], cy = two ? p[3] : p[2];
        const double inv_z = 1.0 / Z;
        const double px = fx * X * inv_z, py = fy * Y * inv_z;
        u = px + cx;
        v = py + cy;
        J[0] = fx * inv_z; J[1] = 0.0; J[2] = -px * inv_z;
        J[3] = 0.0; J[4] = fy * inv_z; J[5] = -py * inv_z;
        return;
    }
    case CAMM_SIMPLE_RADIAL:
    case CAMM_RADIAL: {
        const double inv_z = 1.0 / Z;
        const double px = X * inv_z, py = Y * inv_z;
        const double r2 = px * px + py * py;
        double jd[4], alpha;
        if (c.model == CAMM_SIMPLE_RADIAL) {
            alpha = (1.0 + p[3] * r2);
            jd[0] = (2.0 * p[3] * px * px + alpha) * p[0];
            jd[1] = (2.0 * p[3] * px * py) * p[0];
            jd[2] = jd[1];
            jd[3] = (2.0 * p[3] * py * py + alpha) * p[0];
        } else {
            alpha = (1.0 + p[3] * r2 + p[4] * r2 * r2);
            const double alphap = (2.0 * p[3] + 4.0 * p[4] * r2);
            jd[0] = (alphap * px * px + alpha) * p[0];
            jd[1] = (alphap * px * py) * p[0];
            jd[2] = jd[1];
            jd[3] = (alphap * py * py + alpha) * p[0];
        }
        J[0] = inv_z; J[1] = 0; J[2] = -px * inv_z;
        J[3] = 0; J[4] = inv_z; J[5] = -py * inv_z;
        cam_left_mul_2x2(jd, J);
        u = p[0] * alpha * px + p[1];
        v = p[0] * alpha * py + p[2];
        return;
    }
    default: {
        const double x0 = X / Z, x1 = Y / Z;
        double xd, yd, j0[4];
        cam_opencv_distortion_jac(p, x0, x1, xd, yd, j0);
        J[0] = 1.0 / Z; J[1] = 0.0; J[2] = -x0 / Z;
        J[3] = 0.0; J[4] = 1.0 / Z; J[5] = -x1 / Z;
        cam_left_mul_2x2(j0, J);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            J[k] *= p[0];
            J[3 + k] *= p[1];
        }
        u = p[0] * xd + p[2];
        v = p[1] * yd + p[3];
        return;
    }
    }
}

constexpr int CAM_MAX_PARAMS = 8;

// jac_params of <Model>::project_with_jac: d(u, v) / d(params), 2 x CAM_MAX_PARAMS row-major (jp[c] row u,
// jp[CAM_MAX_PARAMS + c] row v); columns past the model's parameter count are left untouched.
// (camera_models.cc:688-697,737-743,800-816,878-891,939-949,1011-1021,2719-2722)
PLB_HD void cam_jac_params(const CamDev &c, double X, double Y, double Z, double *jp) {
    const double *p = c.p;
    double *j0 = jp, *j1 = jp + CAM_MAX_PARAMS;
    switch (c.model) {
    case CAMM_NULL: return;
    case CAMM_SIMPLE_PINHOLE: {
        const double inv_z = 1.0 / Z;
        j0[0] = X * inv_z; j1[0] = Y * inv_z;
        j0[1] = 1.0; j1[1] = 0.0;
        j0[2] = 0.0; j1[2] = 1.0;
        return;
    }
    case CAMM_PINHOLE: {
        const double inv_z = 1.0 / Z;
        j0[0] = X * inv_z; j1[0] = 0.0;
        j0[1] = 0.0; j1[1] = Y * inv_z;
        j0[2] = 1.0; j1[2] = 0.0;
        j0[3] = 0.0; j1[3] = 1.0;
        return;
    }
    case CAMM_SIMPLE_RADIAL:
    case CAMM_RADIAL: {
        const double inv_z = 1.0 / Z;
        const double px = X * inv_z, py = Y * inv_z;
        const double r2 = px * px + py * py;
        const double alpha = c.model == CAMM_RADIAL ? (1.0 + p[3] * r2 + p[4] * r2 * r2) : (1.0 + p[3] * r2);
        j0[0] = alpha * px; j1[0] = alpha * py;
        j0[1] = 1.0; j1[1] = 0.0;
        j0[2] = 0.0; j1[2] = 1.0;
        j0[3] = p[0] * r2 * px; j1[3] = p[0] * r2 * py;
        if (c.model == CAMM_RADIAL) {
            j0[4] = p[0] * r2 * r2 * px;
            j1[4] = p[0] * r2 * r2 * py;
        }
        return;
    }
    default: {
        const double u = X / Z, v = Y / Z;
        double xd, yd;
        cam_opencv_distortion(p, u, v, xd, yd);
        const double uv = u * v, r2 = u * u + v * v;
        j0[0] = xd; j1[0] = 0.0;
        j0[1] = 0.0; j1[1] = yd;
        j0[2] = 1.0; j1[2] = 0.0;
        j0[3] = 0.0; j1[3] = 1.0;
        j0[4] = p[0] * (r2 * u); j1[4] = p[1] * (r2 * v);
        j0[5] = p[0] * (r2 * r2 * u); j1[5] = p[1] * (r2 * r2 * v);
        j0[6] = p[0] * (2.0 * uv); j1[6] = p[1] * (r2 + 2.0 * (v * v));
        j0[7] = p[0] * (r2 + 2.0 * (u * u)); j1[7] = p[1] * (2.0 * uv);
        return;
    }
    }
}

// Refinement flags of BundleOptions as one bit set (refine_focal_length, refine_principal_point, refine_extra_params)
enum { CAM_REFINE_FOCAL = 1, CAM_REFINE_PP = 2, CAM_REFINE_EXTRA = 4 };

// Camera::get_param_refinement_idx (camera_models.cc:545-561): focal indices, then principal point, then the extra
// parameters of the model (index tables :708-710,759-761,834-836,911-913,1036-1038,2730-2732).  Returns the count.
PLB_HD int cam_refine_idx(int model, int flags, int *idx) {
    int nf = 0, npp = 0, ne = 0; // focal count, principal point at [nf, nf + npp), extras at [nf + npp, + ne)
    switch (model) {
    case CAMM_SIMPLE_PINHOLE: nf = 1; npp = 2; ne = 0; break;
    case CAMM_PINHOLE: nf = 2; npp = 2; ne = 0; break;
    case CAMM_SIMPLE_RADIAL: nf = 1; npp = 2; ne = 1; break;
    case CAMM_RADIAL: nf = 1; npp = 2; ne = 2; break;
    case CAMM_OPENCV: nf = 2; npp = 2; ne = 4; break;
    default: return 0;
    }
    int m = 0;
    if (flags & CAM_REFINE_FOCAL)
        for (int i = 0; i < nf; ++i) idx[m++] = i;
    if (flags & CAM_REFINE_PP)
        for (int i = 0; i < npp; ++i) idx[m++] = nf + i;
    if (flags & CAM_REFINE_EXTRA)
        for (int i = 0; i < ne; ++i) idx[m++] = nf + npp + i;
    return m;
}

// default <Model>::unproject_with_jac (camera_models.cc:456-489): bearing d and M = J^T (J J^T)^-1 (3x2 row-major)
PLB_HD void cam_unproject_with_jac(const CamDev &c, double u, double v, double *d, double *M) {
    cam_unproject(c, u, v, d);
    double J[6], pu, pv;
    cam_project_with_jac(c, d[0], d[1], d[2], pu, pv, J);
    double B[4];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int q = 0; q < 2; ++q) B[2 * r + q] = J[3 * r] * J[3 * q] + J[3 * r + 1] * J[3 * q + 1] + J[3 * r + 2] * J[3 * q + 2];
    const double det = B[0] * B[3] - B[1] * B[2];
    double Bi[4] = {B[3], -B[1], -B[2], B[0]};
#pragma unroll
    for (int k = 0; k < 4; ++k) Bi[k] /= det;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int q = 0; q < 2; ++q) M[2 * i + q] = J[i] * Bi[q] + J[3 + i] * Bi[2 + q];
}

// default <Model>::unproject_with_jac with jac_params (camera_models.cc:456-489): d, M as above and
// dp = d(bearing) / d(params), 3 x CAM_MAX_PARAMS row-major, = -M * jac_params of project_with_jac at d; columns past
// the model's parameter count are left untouched.  The reference has two orders: -(J^T B^-1) Jp with a jac_point
// (:480-483) and -J^T B^-1 Jp without (:486-488).  Negation is exact and commutes with every rounding, so both give
// these bits.
PLB_HD void cam_unproject_with_jac_params(const CamDev &c, double u, double v, double *d, double *M, double *dp) {
    cam_unproject_with_jac(c, u, v, d, M);
    double jp[2 * CAM_MAX_PARAMS];
    cam_jac_params(c, d[0], d[1], d[2], jp);
    const int np = c.model == CAMM_NULL ? 0 : c.model == CAMM_SIMPLE_PINHOLE ? 3 : c.model == CAMM_RADIAL ? 5
                   : c.model == CAMM_OPENCV ? 8 : 4;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < np; ++j)
            dp[CAM_MAX_PARAMS * i + j] = (-M[2 * i]) * jp[j] + (-M[2 * i + 1]) * jp[CAM_MAX_PARAMS + j];
}

} // namespace plb
