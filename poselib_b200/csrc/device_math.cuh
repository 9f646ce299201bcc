// poselib_b200 — small fp64 vector / quaternion helpers for the device kernels (sm_90a).
//
// The whole translation unit is compiled with -fmad=false: fp64 products and sums are rounded separately, like a
// baseline x86-64 build of the reference (CMakeLists.txt:18,23-27: no -march=native, no fast-math), so that the
// per-point inlier tests r2 < thr2 (robust/utils.cc:51-61,187-198) take the same branch as on the CPU.
// fp32 screening kernels ask for FMA explicitly through intrinsics.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace plb {

#define PLB_DEV __device__ __forceinline__

struct d3 {
    double x, y, z;
};
PLB_DEV d3 mk(double a, double b, double c) { return d3{a, b, c}; }
PLB_DEV d3 operator+(d3 a, d3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
PLB_DEV d3 operator-(d3 a, d3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
PLB_DEV d3 operator-(d3 a) { return mk(-a.x, -a.y, -a.z); }
PLB_DEV d3 operator*(double s, d3 a) { return mk(s * a.x, s * a.y, s * a.z); }
PLB_DEV d3 operator/(d3 a, double s) { return mk(a.x / s, a.y / s, a.z / s); }
PLB_DEV double dot(d3 a, d3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
PLB_DEV d3 cross(d3 a, d3 b) { return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
// Eigen normalized(): x / sqrt(x.x) when the squared norm is positive
PLB_DEV d3 unit(d3 a) {
    const double n2 = dot(a, a);
    return (n2 > 0) ? a / sqrt(n2) : a;
}
// x.homogeneous().normalized() of an image point (estimators/*.cc generate_models)
PLB_DEV d3 bearing(double u, double v) { return unit(mk(u, v, 1.0)); }

// Row-major 3x3 in registers
struct m3 {
    double a[9];
    PLB_DEV double &operator()(int r, int c) { return a[3 * r + c]; }
    PLB_DEV double operator()(int r, int c) const { return a[3 * r + c]; }
};
PLB_DEV d3 mcol(const m3 &A, int c) { return mk(A(0, c), A(1, c), A(2, c)); }
PLB_DEV d3 mrow(const m3 &A, int r) { return mk(A(r, 0), A(r, 1), A(r, 2)); }
PLB_DEV void set_col(m3 &A, int c, d3 v) { A(0, c) = v.x; A(1, c) = v.y; A(2, c) = v.z; }
PLB_DEV void set_row(m3 &A, int r, d3 v) { A(r, 0) = v.x; A(r, 1) = v.y; A(r, 2) = v.z; }
PLB_DEV m3 mmul(const m3 &A, const m3 &B) {
    m3 C;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) C(i, j) = A(i, 0) * B(0, j) + A(i, 1) * B(1, j) + A(i, 2) * B(2, j);
    return C;
}
PLB_DEV d3 mvec(const m3 &A, d3 v) {
    return mk(A(0, 0) * v.x + A(0, 1) * v.y + A(0, 2) * v.z, A(1, 0) * v.x + A(1, 1) * v.y + A(1, 2) * v.z,
              A(2, 0) * v.x + A(2, 1) * v.y + A(2, 2) * v.z);
}
// A^T v
PLB_DEV d3 mtvec(const m3 &A, d3 v) {
    return mk(A(0, 0) * v.x + A(1, 0) * v.y + A(2, 0) * v.z, A(0, 1) * v.x + A(1, 1) * v.y + A(2, 1) * v.z,
              A(0, 2) * v.x + A(1, 2) * v.y + A(2, 2) * v.z);
}
PLB_DEV double det3(const m3 &m) {
    return m(0, 0) * (m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1)) - m(0, 1) * (m(1, 0) * m(2, 2) - m(1, 2) * m(2, 0)) +
           m(0, 2) * (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0));
}
// cofactor inverse (what Eigen does for fixed 3x3; misc p3p.cc:121-122)
PLB_DEV m3 inv3(const m3 &m) {
    m3 c;
    c(0, 0) = m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1);
    c(1, 0) = m(1, 2) * m(2, 0) - m(1, 0) * m(2, 2);
    c(2, 0) = m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0);
    c(0, 1) = m(0, 2) * m(2, 1) - m(0, 1) * m(2, 2);
    c(1, 1) = m(0, 0) * m(2, 2) - m(0, 2) * m(2, 0);
    c(2, 1) = m(0, 1) * m(2, 0) - m(0, 0) * m(2, 1);
    c(0, 2) = m(0, 1) * m(1, 2) - m(0, 2) * m(1, 1);
    c(1, 2) = m(0, 2) * m(1, 0) - m(0, 0) * m(1, 2);
    c(2, 2) = m(0, 0) * m(1, 1) - m(0, 1) * m(1, 0);
    const double det = c(0, 0) * m(0, 0) + c(1, 0) * m(0, 1) + c(2, 0) * m(0, 2);
    const double id = 1.0 / det;
#pragma unroll
    for (int k = 0; k < 9; ++k) c.a[k] = c.a[k] * id;
    return c;
}

// Pose: q = (w,x,y,z), t  (camera_pose.h:40-68)
struct pose_t {
    double q[4];
    double t[3];
};
// quaternion -> rotation matrix, Eigen's toRotationMatrix op order (misc/quaternion.h:36-38)
PLB_DEV m3 quat_to_rot(const double *q) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    m3 R;
    R(0, 0) = 1 - (tyy + tzz); R(0, 1) = txy - twz;       R(0, 2) = txz + twy;
    R(1, 0) = txy + twz;       R(1, 1) = 1 - (txx + tzz); R(1, 2) = tyz - twx;
    R(2, 0) = txz - twy;       R(2, 1) = tyz + twx;       R(2, 2) = 1 - (txx + tyy);
    return R;
}
// rotation matrix -> unit quaternion (Shepperd branch selection as Eigen::Quaterniond(R), then normalise;
// misc/quaternion.h:45-51)
PLB_DEV void rot_to_quat(const m3 &R, double *qo) {
    double qx, qy, qz, qw;
    double t = R(0, 0) + R(1, 1) + R(2, 2);
    if (t > 0) {
        t = sqrt(t + 1.0);
        qw = 0.5 * t;
        t = 0.5 / t;
        qx = (R(2, 1) - R(1, 2)) * t;
        qy = (R(0, 2) - R(2, 0)) * t;
        qz = (R(1, 0) - R(0, 1)) * t;
    } else {
        int i = 0;
        if (R(1, 1) > R(0, 0)) i = 1;
        if (R(2, 2) > R(i, i)) i = 2;
        if (i == 0) {
            t = sqrt(R(0, 0) - R(1, 1) - R(2, 2) + 1.0);
            qx = 0.5 * t;
            t = 0.5 / t;
            qw = (R(2, 1) - R(1, 2)) * t;
            qy = (R(1, 0) + R(0, 1)) * t;
            qz = (R(2, 0) + R(0, 2)) * t;
        } else if (i == 1) {
            t = sqrt(R(1, 1) - R(2, 2) - R(0, 0) + 1.0);
            qy = 0.5 * t;
            t = 0.5 / t;
            qw = (R(0, 2) - R(2, 0)) * t;
            qz = (R(2, 1) + R(1, 2)) * t;
            qx = (R(0, 1) + R(1, 0)) * t;
        } else {
            t = sqrt(R(2, 2) - R(0, 0) - R(1, 1) + 1.0);
            qz = 0.5 * t;
            t = 0.5 / t;
            qw = (R(1, 0) - R(0, 1)) * t;
            qx = (R(0, 2) + R(2, 0)) * t;
            qy = (R(1, 2) + R(2, 1)) * t;
        }
    }
    const double n2 = qw * qw + qx * qx + qy * qy + qz * qz;
    if (n2 > 0) {
        const double n = sqrt(n2);
        qw /= n; qx /= n; qy /= n; qz /= n;
    }
    qo[0] = qw; qo[1] = qx; qo[2] = qy; qo[3] = qz;
}
// misc/quaternion.h:61-70
PLB_DEV d3 quat_rotate(const double *q, d3 p) {
    const double q1 = q[0], q2 = q[1], q3 = q[2], q4 = q[3];
    const double px1 = -p.x * q2 - p.y * q3 - p.z * q4;
    const double px2 = p.x * q1 - p.y * q4 + p.z * q3;
    const double px3 = p.y * q1 + p.x * q4 - p.z * q2;
    const double px4 = p.y * q2 - p.x * q3 + p.z * q1;
    return mk(px2 * q1 - px1 * q2 - px3 * q4 + px4 * q3, px3 * q1 - px1 * q3 + px2 * q4 - px4 * q2,
              px3 * q2 - px2 * q3 - px1 * q4 + px4 * q1);
}
// misc/quaternion.h:52-59
PLB_DEV void quat_mul(const double *a, const double *b, double *r) {
    const double a1 = a[0], a2 = a[1], a3 = a[2], a4 = a[3];
    const double b1 = b[0], b2 = b[1], b3 = b[2], b4 = b[3];
    r[0] = a1 * b1 - a2 * b2 - a3 * b3 - a4 * b4;
    r[1] = a1 * b2 + a2 * b1 + a3 * b4 - a4 * b3;
    r[2] = a1 * b3 + a3 * b1 - a2 * b4 + a4 * b2;
    r[3] = a1 * b4 + a2 * b3 - a3 * b2 + a4 * b1;
}
// misc/quaternion.h:73-96
PLB_DEV void quat_exp(d3 w, double *r) {
    const double theta2 = dot(w, w);
    const double theta = sqrt(theta2);
    const double th = 0.5 * theta;
    double re, im;
    if (theta > 1e-6) {
        re = cos(th);
        im = sin(th) / theta;
    } else {
        const double theta4 = theta2 * theta2;
        re = 1.0 - (1.0 / 8.0) * theta2 + (1.0 / 384.0) * theta4;
        im = 0.5 - (1.0 / 48.0) * theta2 + (1.0 / 3840.0) * theta4;
        const double s = sqrt(re * re + im * im * theta2);
        re /= s;
        im /= s;
    }
    r[0] = re; r[1] = im * w.x; r[2] = im * w.y; r[3] = im * w.z;
}
// E = [t]x R   (misc/essential.cc:35-38)
PLB_DEV m3 essential_from_pose(const double *q, const double *t) {
    m3 Tx;
    Tx(0, 0) = 0.0;   Tx(0, 1) = -t[2]; Tx(0, 2) = t[1];
    Tx(1, 0) = t[2];  Tx(1, 1) = 0.0;   Tx(1, 2) = -t[0];
    Tx(2, 0) = -t[1]; Tx(2, 1) = t[0];  Tx(2, 2) = 0.0;
    return mmul(Tx, quat_to_rot(q));
}
// misc/essential.cc:40-57 ; x1,x2 unit bearings
PLB_DEV bool cheirality_ok(const double *q, const double *t, d3 x1, d3 x2, double min_depth) {
    const d3 Rx1 = quat_rotate(q, x1);
    const d3 tt = mk(t[0], t[1], t[2]);
    const double a = -dot(Rx1, x2);
    const double b1 = -dot(Rx1, tt);
    const double b2 = dot(x2, tt);
    const double lambda1 = b1 - a * b2;
    const double lambda2 = -a * b1 + b2;
    const double md = min_depth * (1 - a * a);
    return lambda1 > md && lambda2 > md;
}

// ---- warp helpers ----------------------------------------------------------------------------------------
PLB_DEV double shfl_d(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }
PLB_DEV double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
PLB_DEV unsigned warp_sum_u(unsigned v) { return __reduce_add_sync(0xffffffffu, v); }

} // namespace plb
