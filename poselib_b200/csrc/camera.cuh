// poselib_b200 — camera models of the estimate_* pre-step, evaluated on the device (row N3 of SURVEY.md §8f):
// NULL, SIMPLE_PINHOLE, PINHOLE, SIMPLE_RADIAL, RADIAL, OPENCV, SIMPLE_RADIAL_FISHEYE, RADIAL_FISHEYE, DIVISION,
// SIMPLE_DIVISION  (misc/camera_models.{h,cc} of the reference, citations relative to /root/reference/PoseLib).
// Compiled with -fmad=false like the rest of the fp64 path, so the calibrated points / bearings / unprojection Jacobians
// are the doubles a baseline x86-64 build computes (the fisheye models' atan2 / tan, and pow in the division models'
// parameter Jacobian, are CUDA's on the device: not correctly rounded, they can differ from glibc in the last bits).
#pragma once
#include "device_math.cuh"

namespace plb {

enum {
    CAMM_NULL = -1, CAMM_SIMPLE_PINHOLE = 0, CAMM_PINHOLE = 1, CAMM_SIMPLE_RADIAL = 2, CAMM_RADIAL = 3, CAMM_OPENCV = 4,
    CAMM_SIMPLE_RADIAL_FISHEYE = 8, CAMM_RADIAL_FISHEYE = 9, CAMM_DIVISION = 101, CAMM_SIMPLE_DIVISION = 102
};

struct CamDev { // Camera: model id + parameter vector (camera_models.h:59-66)
    int model;
    int reserved;
    double p[8];
};

#define PLB_HD __host__ __device__ __forceinline__
constexpr int CAM_MAX_PARAMS = 8;
// The fisheye and division models (ids past OPENCV) sit behind the template flag X of the camera functions below: with
// X = false (the default) a function is the switch over the six older models and nothing else, so the kernels built
// without X compile to what they were before these models existed; the host launches the X instantiation of a kernel
// only for work that has such a camera.  With X the four models are called, not inlined (atan2 / tan, Newton loops),
// arguments and results by value so the caller's camera and outputs need no stack copy.
#define PLB_HD_CALL static __host__ __device__ __noinline__

// The parameter layout of every model on the path: focal lengths at [0, nf), principal point at [nf, nf + npp), the
// model's extra parameters at [nf + npp, np) (focal_idx / principal_point_idx / extra_idx and num_params of each model,
// camera_models.cc).  Camera::focal, Camera::rescale, get_param_refinement_idx and the parameter count all read it.
struct CamLayout {
    int nf, npp, ne;
    PLB_HD int np() const { return nf + npp + ne; }
};
// false (and an empty layout) for a model id the path does not run
PLB_HD bool cam_layout(int model, CamLayout &L) {
    switch (model) {
    case CAMM_NULL: L = {0, 0, 0}; return true;
    case CAMM_SIMPLE_PINHOLE: L = {1, 2, 0}; return true;        // :708-710
    case CAMM_PINHOLE: L = {2, 2, 0}; return true;               // :759-761
    case CAMM_SIMPLE_RADIAL: L = {1, 2, 1}; return true;         // :834-836
    case CAMM_RADIAL: L = {1, 2, 2}; return true;                // :911-913
    case CAMM_OPENCV: L = {2, 2, 4}; return true;                // :1036-1038
    case CAMM_SIMPLE_RADIAL_FISHEYE: L = {1, 2, 1}; return true; // :1654-1658
    case CAMM_RADIAL_FISHEYE: L = {1, 2, 2}; return true;        // :1792-1796
    case CAMM_DIVISION: L = {2, 2, 1}; return true;              // :2542-2546
    case CAMM_SIMPLE_DIVISION: L = {1, 2, 1}; return true;       // :2697-2701
    default: L = {0, 0, 0}; return false;
    }
}
PLB_HD int cam_num_params(int model) {
    CamLayout L;
    cam_layout(model, L);
    return L.np();
}

// Camera::focal (camera_models.cc:304-324): the mean of the focal lengths, 1 for the NULL camera
PLB_HD double cam_focal(const CamDev &c) {
    CamLayout L;
    cam_layout(c.model, L);
    if (L.nf == 0) return 1.0;
    double f = 0.0;
    for (int i = 0; i < L.nf; ++i) f += c.p[i] / L.nf;
    return f;
}
// Camera::rescale (camera_models.cc:432-454): focal lengths and principal point times scale
PLB_HD void cam_rescale(CamDev &c, double scale) {
    CamLayout L;
    cam_layout(c.model, L);
    for (int i = 0; i < L.nf + L.npp; ++i) c.p[i] *= scale;
}

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

// ---- fisheye and division models (called, not inlined) -----------------------------------------------------------------
struct CamX { // model id and the first five parameters (all these models have at most five)
    int model;
    double p[5];
};
PLB_HD CamX cam_x(const CamDev &c) {
    CamX e;
    e.model = c.model;
#pragma unroll
    for (int i = 0; i < 5; ++i) e.p[i] = c.p[i];
    return e;
}
// Results of the called functions, each no larger than its caller needs
struct CamV2 {
    double u, v;
};
struct CamV3 {
    double x[3];
};
struct CamPJ { // projection and point Jacobian (2x3 row-major)
    double u, v, J[6];
};
struct CamJP { // jac_params (2 x 5 row-major)
    double jp[10];
};
struct CamPJX { // projection, point Jacobian and jac_params
    double u, v, J[6], jp[10];
};
struct CamUJ { // bearing and unproject Jacobian M (3x2 row-major)
    double d[3], M[6];
};
struct CamUJP { // bearing, M and jac_params (3 x 5 row-major)
    double d[3], M[6], dp[15];
};

// M = J^T (J J^T)^-1 of the default <Model>::unproject_with_jac (camera_models.cc:474-480), J 2x3 row-major
PLB_HD void cam_default_M(const double *J, double *M) {
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

// undistort_theta_poly_newton (camera_models.cc:613-637): the inner loop runs over the model's parameters from k0 = 3
PLB_HD double cam_theta_newton(const double *p, int np, double rd, double &theta) {
    double f = 0.0, fp;
    for (int iter = 0; iter < CAM_UNDIST_MAX_ITER; iter++) {
        f = 1.0;
        fp = 1.0;
        const double theta2 = theta * theta;
        double theta2k = theta2;
        double factor = 3.0;
        for (int k = 3; k < np; ++k) {
            const double t = theta2k * p[k];
            f += t;
            fp += factor * t;
            theta2k *= theta2;
            factor += 2.0;
        }
        f *= theta;
        f -= rd;
        if (fabs(f) < CAM_UNDIST_TOL) return fabs(f);
        theta = theta - f / fp;
    }
    return fabs(f);
}
// undistort_theta_poly (camera_models.cc:639-662): Newton from 0, rd, 0.5 rd, 1.5 rd
PLB_HD double cam_undistort_theta(const double *p, int np, double rd) {
    double theta = 0;
    double res = cam_theta_newton(p, np, rd, theta);
    if (res > CAM_UNDIST_TOL || theta < 0) {
        theta = rd;
        res = cam_theta_newton(p, np, rd, theta);
        if (res > CAM_UNDIST_TOL || theta < 0) {
            theta = 0.5 * rd;
            res = cam_theta_newton(p, np, rd, theta);
            if (res > CAM_UNDIST_TOL || theta < 0) {
                theta = 1.5 * rd;
                res = cam_theta_newton(p, np, rd, theta);
            }
        }
    }
    return theta;
}

// SimpleRadialFisheye / RadialFisheye / Division / SimpleDivision ::unproject (camera_models.cc:1628-1652,1766-1790,
// 2475-2484,2630-2640)
PLB_HD CamV3 camx_unproject_w(const CamX &c, double u, double v) {
    const double *p = c.p;
    CamV3 r;
    double *x = r.x;
    if (c.model == CAMM_SIMPLE_RADIAL_FISHEYE || c.model == CAMM_RADIAL_FISHEYE) {
        const double px = (u - p[1]) / p[0];
        const double py = (v - p[2]) / p[0];
        const double rd = sqrt(px * px + py * py);
        if (rd > 1e-8) {
            const double theta = cam_undistort_theta(p, c.model == CAMM_RADIAL_FISHEYE ? 5 : 4, rd);
            x[0] = px / rd;
            x[1] = py / rd;
            if (fabs(theta - 1.57079632679489661923) > 1e-8) // M_PI_2
                x[2] = 1.0 / tan(theta);
            else
                x[2] = 0.0;
        } else {
            x[0] = px;
            x[1] = py;
            x[2] = sqrt(1 - rd * rd);
        }
    } else {
        const bool two = c.model == CAMM_DIVISION;
        const double x0 = (u - p[two ? 2 : 1]) / p[0];
        const double y0 = (v - p[two ? 3 : 2]) / p[two ? 1 : 0];
        const double r2 = x0 * x0 + y0 * y0;
        x[0] = x0;
        x[1] = y0;
        x[2] = 1.0 + p[two ? 4 : 3] * r2;
    }
    cam_normalize3(x);
    return r;
}

// SimpleRadialFisheye / RadialFisheye / Division / SimpleDivision ::project (camera_models.cc:1517-1535,1664-1683,
// 2395-2413,2552-2571)
PLB_HD_CALL CamV2 camx_project(CamX c, double X, double Y, double Z) {
    const double *p = c.p;
    CamV2 r;
    const double rho = sqrt(X * X + Y * Y);
    if (c.model == CAMM_SIMPLE_RADIAL_FISHEYE || c.model == CAMM_RADIAL_FISHEYE) {
        if (rho > 1e-8) {
            const double theta = atan2(rho, Z);
            const double theta2 = theta * theta;
            double rd;
            if (c.model == CAMM_RADIAL_FISHEYE) {
                const double theta4 = theta2 * theta2;
                rd = theta * (1.0 + theta2 * p[3] + theta4 * p[4]);
            } else {
                rd = theta * (1.0 + theta2 * p[3]);
            }
            const double inv_r = 1.0 / rho;
            r.u = p[0] * X * inv_r * rd + p[1];
            r.v = p[0] * Y * inv_r * rd + p[2];
        } else { // very close to the principal axis: distortion ignored
            r.u = p[0] * X + p[1];
            r.v = p[0] * Y + p[2];
        }
        return r;
    }
    const bool two = c.model == CAMM_DIVISION;
    const double disc2 = Z * Z - 4.0 * rho * rho * p[two ? 4 : 3];
    if (disc2 < 0) {
        r.u = r.v = 0.0;
        return r;
    }
    const double sq = sqrt(disc2);
    const double rr = 2.0 / (Z + sq);
    r.u = p[0] * rr * X + p[two ? 2 : 1];
    r.v = p[two ? 1 : 0] * rr * Y + p[two ? 3 : 2];
    return r;
}

// SimpleRadialFisheye / RadialFisheye / Division / SimpleDivision ::project_with_jac with jac_params
// (camera_models.cc:1537-1612,1685-1764,2415-2473,2573-2628); jac_params columns past the model's count are untouched
PLB_HD CamPJX camx_pwj(const CamX &c, double X, double Y, double Z) {
    const double *p = c.p;
    CamPJX r;
    double *J = r.J, *j0 = r.jp, *j1 = r.jp + 5;
    const double rho = sqrt(X * X + Y * Y);
    if (c.model == CAMM_SIMPLE_RADIAL_FISHEYE || c.model == CAMM_RADIAL_FISHEYE) {
        const bool two = c.model == CAMM_RADIAL_FISHEYE;
        if (rho > 1e-8) {
            const double theta = atan2(rho, Z);
            const double theta2 = theta * theta;
            const double theta4 = theta2 * theta2;
            const double rd = two ? theta * (1.0 + theta2 * p[3] + theta4 * p[4]) : theta * (1.0 + theta2 * p[3]);
            const double inv_r = 1.0 / rho;
            const double drho_dx = X / rho;
            const double drho_dy = Y / rho;
            const double rho_z2 = rho * rho + Z * Z;
            const double dtheta_drho = Z / rho_z2;
            const double dtheta_dz = -rho / rho_z2;
            const double drd_dtheta = two ? (1.0 + 3.0 * theta2 * p[3] + 5.0 * theta4 * p[4]) : (1.0 + 3.0 * theta2 * p[3]);
            const double drd_dx = drd_dtheta * dtheta_drho * drho_dx;
            const double drd_dy = drd_dtheta * dtheta_drho * drho_dy;
            const double drd_dz = drd_dtheta * dtheta_dz;
            const double dinv_r_drho = -1.0 / (rho * rho);
            const double dinv_r_dx = dinv_r_drho * drho_dx;
            const double dinv_r_dy = dinv_r_drho * drho_dy;
            r.u = p[0] * X * inv_r * rd + p[1];
            r.v = p[0] * Y * inv_r * rd + p[2];
            J[0] = p[0] * (inv_r * rd + X * dinv_r_dx * rd + X * inv_r * drd_dx);
            J[1] = p[0] * X * (dinv_r_dy * rd + inv_r * drd_dy);
            J[2] = p[0] * X * inv_r * drd_dz;
            J[3] = p[0] * Y * (dinv_r_dx * rd + inv_r * drd_dx);
            J[4] = p[0] * (inv_r * rd + Y * dinv_r_dy * rd + Y * inv_r * drd_dy);
            J[5] = p[0] * Y * inv_r * drd_dz;
            j0[0] = X * inv_r * rd; j1[0] = Y * inv_r * rd;
            j0[1] = 1.0; j1[1] = 0.0;
            j0[2] = 0.0; j1[2] = 1.0;
            j0[3] = p[0] * X * inv_r * theta * theta2; j1[3] = p[0] * Y * inv_r * theta * theta2;
            if (two) {
                j0[4] = p[0] * X * inv_r * theta * theta4;
                j1[4] = p[0] * Y * inv_r * theta * theta4;
            }
        } else { // very close to the principal axis: distortion ignored; jac_params zeroed, then four entries set
            r.u = p[0] * X + p[1];
            r.v = p[0] * Y + p[2];
            J[0] = p[0]; J[1] = 0.0; J[2] = 0.0;
            J[3] = 0.0; J[4] = p[0]; J[5] = 0.0;
#pragma unroll
            for (int k = 0; k < 10; ++k) r.jp[k] = 0.0;
            j0[0] = X;
            j0[1] = 1.0;
            j1[0] = Y;
            j1[2] = 1.0;
        }
        return r;
    }
    const bool two = c.model == CAMM_DIVISION;
    const double k = p[two ? 4 : 3];
    const double disc2 = Z * Z - 4.0 * rho * rho * k;
    if (disc2 < 0) {
        r.u = r.v = 0.0;
#pragma unroll
        for (int q = 0; q < 6; ++q) J[q] = 0.0;
#pragma unroll
        for (int q = 0; q < 10; ++q) r.jp[q] = 0.0;
        return r;
    }
    const double fx = p[0], fy = p[two ? 1 : 0];
    const double sq = sqrt(disc2);
    const double den = Z + sq;
    const double rr = 2.0 / den;
    const double xp0 = rr * X;
    const double xp1 = rr * Y;
    r.u = fx * xp0 + p[two ? 2 : 1];
    r.v = fy * xp1 + p[two ? 3 : 2];
    const double dd[3] = {-8.0 * k * X, -8.0 * k * Y, 2.0 * Z};
    const double dsq_ddisc2 = 0.5 / sq;
    const double dr_dden = -2.0 / (den * den);
    const double e[3] = {0.0, 0.0, 1.0};
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const double dr = dr_dden * (dsq_ddisc2 * dd[q] + e[q]);
        J[q] = X * dr;
        J[3 + q] = Y * dr;
    }
    J[0] += rr;
    J[4] += rr;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        J[q] *= fx;
        J[3 + q] *= fy;
    }
    const double dr_dk = 4.0 * rho * rho / (den * den * sq);
    if (two) {
        j0[0] = xp0; j1[0] = 0.0;
        j0[1] = 0.0; j1[1] = xp1;
        j0[2] = 1.0; j1[2] = 0.0;
        j0[3] = 0.0; j1[3] = 1.0;
        j0[4] = fx * X * dr_dk; j1[4] = fy * Y * dr_dk;
    } else {
        j0[0] = xp0; j1[0] = xp1;
        j0[1] = 1.0; j1[1] = 0.0;
        j0[2] = 0.0; j1[2] = 1.0;
        j0[3] = fx * X * dr_dk; j1[3] = fx * Y * dr_dk;
    }
    return r;
}

// Division / SimpleDivision ::unproject_with_jac, the models' own closed form (camera_models.cc:2486-2540,2642-2695),
// not the default J^T (J J^T)^-1 of :456-489: bearing, M (3x2 row-major) and jac_params (3 x np row-major)
PLB_HD CamUJP camx_division_uwj(const CamX &c, double u, double v) {
    const double *p = c.p;
    CamUJP r;
    double *x = r.d, *M = r.M, *P = r.dp;
    if (c.model == CAMM_DIVISION) {
        const double x0 = (u - p[2]) / p[0];
        const double y0 = (v - p[3]) / p[1];
        const double r2 = x0 * x0 + y0 * y0;
        x[0] = x0;
        x[1] = y0;
        x[2] = 1.0 + p[4] * r2;
        const double inv_norm = 1.0 / sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
        x[0] *= inv_norm;
        x[1] *= inv_norm;
        x[2] *= inv_norm;
        M[0] = p[0] * (1 - x[0] * x[0]) + 2 * x[0] * x[2] * p[4] * (p[2] - u);
        M[1] = x[0] * (-p[1] * x[1] + 2 * x[2] * p[4] * (p[3] - v));
        M[2] = x[1] * (-p[0] * x[0] + 2 * x[2] * p[4] * (p[2] - u));
        M[3] = p[1] * (1 - x[1] * x[1]) + 2 * x[1] * x[2] * p[4] * (p[3] - v);
        M[4] = -p[0] * x[0] * x[2] + 2 * p[4] * (p[2] - u) * (x[2] * x[2] - 1);
        M[5] = -p[1] * x[1] * x[2] + 2 * p[4] * (p[3] - v) * (x[2] * x[2] - 1);
        const double s0 = inv_norm / (p[0] * p[0]), s1 = inv_norm / (p[1] * p[1]);
        for (int i = 0; i < 3; ++i) {
            M[2 * i] *= s0;
            M[2 * i + 1] *= s1;
        }
        P[0] = (p[2] - u) * (-p[0] * (x[0] * x[0] - 1) + 2 * x[0] * x[2] * p[4] * (p[2] - u));
        P[1] = x[0] * (p[3] - v) * (-p[1] * x[1] + 2 * x[2] * p[4] * (p[3] - v));
        P[2] = p[0] * (x[0] * x[0] - 1) - 2 * x[0] * x[2] * p[4] * (p[2] - u);
        P[3] = x[0] * (p[1] * x[1] - 2 * x[2] * p[4] * (p[3] - v));
        P[4] = -x[0] * x[2] * r2;
        P[5] = x[1] * (p[2] - u) * (-p[0] * x[0] + 2 * x[2] * p[4] * (p[2] - u));
        P[6] = (p[3] - v) * (-p[1] * (x[1] * x[1] - 1) + 2 * x[1] * x[2] * p[4] * (p[3] - v));
        P[7] = x[1] * (p[0] * x[0] - 2 * x[2] * p[4] * (p[2] - u));
        P[8] = p[1] * (x[1] * x[1] - 1) - 2 * x[1] * x[2] * p[4] * (p[3] - v);
        P[9] = -x[1] * x[2] * r2;
        P[10] = (p[2] - u) * (-p[0] * x[0] * x[2] + 2 * p[4] * (p[2] - u) * (x[2] * x[2] - 1));
        P[11] = (p[3] - v) * (-p[1] * x[1] * x[2] + 2 * p[4] * (p[3] - v) * (x[2] * x[2] - 1));
        P[12] = p[0] * x[0] * x[2] - 2 * p[4] * (p[2] - u) * (x[2] * x[2] - 1);
        P[13] = p[1] * x[1] * x[2] - 2 * p[4] * (p[3] - v) * (x[2] * x[2] - 1);
        P[14] = r2 * (1 - x[2] * x[2]);
        const double c0 = pow(p[0], 3.0), c1 = pow(p[1], 3.0), c2 = pow(p[0], 2.0), c3 = pow(p[1], 2.0);
        for (int i = 0; i < 3; ++i) {
            P[5 * i] /= c0;
            P[5 * i + 1] /= c1;
            P[5 * i + 2] /= c2;
            P[5 * i + 3] /= c3;
        }
        for (int i = 0; i < 15; ++i) P[i] *= inv_norm;
        return r;
    }
    const double x0 = (u - p[1]) / p[0];
    const double y0 = (v - p[2]) / p[0];
    const double r2 = x0 * x0 + y0 * y0;
    x[0] = x0;
    x[1] = y0;
    x[2] = 1.0 + p[3] * r2;
    const double inv_norm = 1.0 / sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    x[0] *= inv_norm;
    x[1] *= inv_norm;
    x[2] *= inv_norm;
    M[0] = p[0] * (1 - x[0] * x[0]) + 2 * x[0] * x[2] * p[3] * (p[1] - u);
    M[1] = x[0] * (-p[0] * x[1] + 2 * x[2] * p[3] * (p[2] - v));
    M[2] = x[1] * (-p[0] * x[0] + 2 * x[2] * p[3] * (p[1] - u));
    M[3] = p[0] * (1 - x[1] * x[1]) + 2 * x[1] * x[2] * p[3] * (p[2] - v);
    M[4] = -p[0] * x[0] * x[2] + 2 * p[3] * (p[1] - u) * (x[2] * x[2] - 1);
    M[5] = -p[0] * x[1] * x[2] + 2 * p[3] * (p[2] - v) * (x[2] * x[2] - 1);
    const double s = inv_norm / (p[0] * p[0]);
    for (int i = 0; i < 6; ++i) M[i] *= s;
    // 3 x 4, stored with the row stride of 5
    P[0] = (p[1] - u) * (-p[0] * (x[0] * x[0] - 1) + 2 * x[0] * x[2] * p[3] * (p[1] - u));
    P[0] += x[0] * (p[2] - v) * (-p[0] * x[1] + 2 * x[2] * p[3] * (p[2] - v));
    P[1] = p[0] * (x[0] * x[0] - 1) - 2 * x[0] * x[2] * p[3] * (p[1] - u);
    P[2] = x[0] * (p[0] * x[1] - 2 * x[2] * p[3] * (p[2] - v));
    P[3] = -x[0] * x[2] * r2;
    P[5] = x[1] * (p[1] - u) * (-p[0] * x[0] + 2 * x[2] * p[3] * (p[1] - u));
    P[5] += (p[2] - v) * (-p[0] * (x[1] * x[1] - 1) + 2 * x[1] * x[2] * p[3] * (p[2] - v));
    P[6] = x[1] * (p[0] * x[0] - 2 * x[2] * p[3] * (p[1] - u));
    P[7] = p[0] * (x[1] * x[1] - 1) - 2 * x[1] * x[2] * p[3] * (p[2] - v);
    P[8] = -x[1] * x[2] * r2;
    P[10] = (p[1] - u) * (-p[0] * x[0] * x[2] + 2 * p[3] * (p[1] - u) * (x[2] * x[2] - 1));
    P[10] += (p[2] - v) * (-p[0] * x[1] * x[2] + 2 * p[3] * (p[2] - v) * (x[2] * x[2] - 1));
    P[11] = p[0] * x[0] * x[2] - 2 * p[3] * (p[1] - u) * (x[2] * x[2] - 1);
    P[12] = p[0] * x[1] * x[2] - 2 * p[3] * (p[2] - v) * (x[2] * x[2] - 1);
    P[13] = r2 * (1 - x[2] * x[2]);
    const double c0 = pow(p[0], 3.0), c1 = pow(p[0], 2.0);
    for (int i = 0; i < 3; ++i) {
        P[5 * i] /= c0;
        P[5 * i + 1] /= c1;
        P[5 * i + 2] /= c1;
        P[5 * i + 4] = 0.0;
    }
    for (int i = 0; i < 15; ++i) P[i] *= inv_norm;
    return r;
}

// The called entry points of the four models: one call per camera function at every call site.
PLB_HD_CALL CamV3 camx_unproject(CamX c, double u, double v) { return camx_unproject_w(c, u, v); }
PLB_HD_CALL CamPJ camx_project_with_jac(CamX c, double X, double Y, double Z) {
    const CamPJX a = camx_pwj(c, X, Y, Z);
    CamPJ r;
    r.u = a.u;
    r.v = a.v;
#pragma unroll
    for (int k = 0; k < 6; ++k) r.J[k] = a.J[k];
    return r;
}
PLB_HD_CALL CamJP camx_jac_params(CamX c, double X, double Y, double Z) {
    const CamPJX a = camx_pwj(c, X, Y, Z);
    CamJP r;
#pragma unroll
    for (int k = 0; k < 10; ++k) r.jp[k] = a.jp[k];
    return r;
}
// <Model>::unproject_with_jac with jac_params: the division models' own form, else the default one (camera_models.cc:
// 456-489) with dp = -M * jac_params of project_with_jac at d
PLB_HD CamUJP camx_uwj(const CamX &c, double u, double v) {
    if (c.model == CAMM_DIVISION || c.model == CAMM_SIMPLE_DIVISION) return camx_division_uwj(c, u, v);
    CamUJP r;
    const CamV3 d = camx_unproject_w(c, u, v);
#pragma unroll
    for (int k = 0; k < 3; ++k) r.d[k] = d.x[k];
    const CamPJX a = camx_pwj(c, r.d[0], r.d[1], r.d[2]);
    cam_default_M(a.J, r.M);
    const int np = cam_num_params(c.model);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < np; ++j) r.dp[5 * i + j] = (-r.M[2 * i]) * a.jp[j] + (-r.M[2 * i + 1]) * a.jp[5 + j];
    return r;
}
PLB_HD_CALL CamUJ camx_unproject_with_jac(CamX c, double u, double v) {
    const CamUJP a = camx_uwj(c, u, v);
    CamUJ r;
#pragma unroll
    for (int k = 0; k < 3; ++k) r.d[k] = a.d[k];
#pragma unroll
    for (int k = 0; k < 6; ++k) r.M[k] = a.M[k];
    return r;
}
// dp: the model's parameter columns of a 3 x CAM_MAX_PARAMS row-major block (the caller's staging memory)
PLB_HD_CALL CamUJ camx_unproject_with_jac_params(CamX c, double u, double v, double *dp) {
    const CamUJP a = camx_uwj(c, u, v);
    const int np = cam_num_params(c.model);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < np; ++j) dp[CAM_MAX_PARAMS * i + j] = a.dp[5 * i + j];
    CamUJ r;
#pragma unroll
    for (int k = 0; k < 3; ++k) r.d[k] = a.d[k];
#pragma unroll
    for (int k = 0; k < 6; ++k) r.M[k] = a.M[k];
    return r;
}

// the four models above: ids past OPENCV among those cam_layout accepts
PLB_HD bool cam_is_x(int model) { return model > CAMM_OPENCV; }

// <Model>::unproject: pixel -> unit bearing (camera_models.cc:700-705,745-751,819-831,895-907,1025-1033,2724-2726)
template <bool X = false> PLB_HD void cam_unproject(const CamDev &c, double u, double v, double *x) {
    if (X && cam_is_x(c.model)) {
        const CamV3 r = camx_unproject(cam_x(c), u, v);
        x[0] = r.x[0]; x[1] = r.x[1]; x[2] = r.x[2];
        return;
    }
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
template <bool X = false> PLB_HD void cam_unproject2(const CamDev &c, double u, double v, double &ox, double &oy) {
    double x[3];
    cam_unproject<X>(c, u, v, x);
    ox = x[0] / x[2];
    oy = x[1] / x[2];
}

// <Model>::project (camera_models.cc:668-671,716-720,766-772,849-857,965-970,2708-2710)
template <bool XM = false> PLB_HD void cam_project(const CamDev &c, double X, double Y, double Z, double &u, double &v) {
    if (XM && cam_is_x(c.model)) {
        const CamV2 r = camx_project(cam_x(c), X, Y, Z);
        u = r.u;
        v = r.v;
        return;
    }
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
template <bool XM = false>
PLB_HD void cam_project_with_jac(const CamDev &c, double X, double Y, double Z, double &u, double &v, double *J) {
    if (XM && cam_is_x(c.model)) {
        const CamPJ r = camx_project_with_jac(cam_x(c), X, Y, Z);
        u = r.u;
        v = r.v;
#pragma unroll
        for (int k = 0; k < 6; ++k) J[k] = r.J[k];
        return;
    }
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

// jac_params of <Model>::project_with_jac: d(u, v) / d(params), 2 x CAM_MAX_PARAMS row-major (jp[c] row u,
// jp[CAM_MAX_PARAMS + c] row v); columns past the model's parameter count are left untouched.
// (camera_models.cc:688-697,737-743,800-816,878-891,939-949,1011-1021,2719-2722)
template <bool XM = false> PLB_HD void cam_jac_params(const CamDev &c, double X, double Y, double Z, double *jp) {
    const double *p = c.p;
    double *j0 = jp, *j1 = jp + CAM_MAX_PARAMS;
    if (XM && cam_is_x(c.model)) {
        const CamJP r = camx_jac_params(cam_x(c), X, Y, Z);
        const int np = cam_num_params(c.model);
        for (int k = 0; k < np; ++k) {
            j0[k] = r.jp[k];
            j1[k] = r.jp[5 + k];
        }
        return;
    }
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
// parameters of the model (the layout of cam_layout).  Returns the count.
PLB_HD int cam_refine_idx(int model, int flags, int *idx) {
    CamLayout L;
    cam_layout(model, L);
    int m = 0;
    if (flags & CAM_REFINE_FOCAL)
        for (int i = 0; i < L.nf; ++i) idx[m++] = i;
    if (flags & CAM_REFINE_PP)
        for (int i = 0; i < L.npp; ++i) idx[m++] = L.nf + i;
    if (flags & CAM_REFINE_EXTRA)
        for (int i = 0; i < L.ne; ++i) idx[m++] = L.nf + L.npp + i;
    return m;
}

// <Model>::unproject_with_jac: bearing d and M (3x2 row-major).  The default (camera_models.cc:456-489) is
// M = J^T (J J^T)^-1 of the projection Jacobian at d; the division models have their own closed form.
template <bool X = false> PLB_HD void cam_unproject_with_jac(const CamDev &c, double u, double v, double *d, double *M) {
    if (X && cam_is_x(c.model)) {
        const CamUJ r = camx_unproject_with_jac(cam_x(c), u, v);
#pragma unroll
        for (int k = 0; k < 3; ++k) d[k] = r.d[k];
#pragma unroll
        for (int k = 0; k < 6; ++k) M[k] = r.M[k];
        return;
    }
    cam_unproject(c, u, v, d);
    double J[6], pu, pv;
    cam_project_with_jac(c, d[0], d[1], d[2], pu, pv, J);
    cam_default_M(J, M);
}

// <Model>::unproject_with_jac with jac_params: d, M as above and dp = d(bearing) / d(params), 3 x CAM_MAX_PARAMS
// row-major; columns past the model's parameter count are left untouched.  The default (camera_models.cc:456-489) is
// -M * jac_params of project_with_jac at d.  The reference has two orders there: -(J^T B^-1) Jp with a jac_point
// (:480-483) and -J^T B^-1 Jp without (:486-488).  Negation is exact and commutes with every rounding, so both give
// these bits.  The division models' own form computes dp in closed form, the same with or without a jac_point.
template <bool X = false>
PLB_HD void cam_unproject_with_jac_params(const CamDev &c, double u, double v, double *d, double *M, double *dp) {
    if (X && cam_is_x(c.model)) {
        const CamUJ r = camx_unproject_with_jac_params(cam_x(c), u, v, dp);
#pragma unroll
        for (int k = 0; k < 3; ++k) d[k] = r.d[k];
#pragma unroll
        for (int k = 0; k < 6; ++k) M[k] = r.M[k];
        return;
    }
    cam_unproject_with_jac(c, u, v, d, M);
    double jp[2 * CAM_MAX_PARAMS];
    cam_jac_params(c, d[0], d[1], d[2], jp);
    // the counts of cam_layout for the six older models, as the ternary the kernels built without X were compiled from
    const int np = c.model == CAMM_NULL ? 0 : c.model == CAMM_SIMPLE_PINHOLE ? 3 : c.model == CAMM_RADIAL ? 5
                   : c.model == CAMM_OPENCV ? 8 : 4;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < np; ++j)
            dp[CAM_MAX_PARAMS * i + j] = (-M[2 * i]) * jp[j] + (-M[2 * i + 1]) * jp[CAM_MAX_PARAMS + j];
}

} // namespace plb
