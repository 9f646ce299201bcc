// The adapter's refiners with PoseLib's per-residual weights, against the same kind of stand-ins for the Eigen / PoseLib
// types as tests/adapter_intrinsics_compile_test.cc.  Built and run by tests/test_weighted_refine.py; `run` (GPU) checks
// that weights of size n give the *_weighted entry point's result, that any other size gives the unweighted result, and
// that bundle_adjust(CameraPose*) ignores its weights, as the reference does (bundle.cc:84-92).
#include "../poselib_b200/adapter/poselib_b200.hpp"

#include <cmath>
#include <cstdio>
#include <cstring>

namespace standin {
template <int N> struct Vec {
    double d[N];
    double &operator()(int i) { return d[i]; }
    double operator()(int i) const { return d[i]; }
};
using Vector2d = Vec<2>;
using Vector3d = Vec<3>;
using Vector4d = Vec<4>;
struct Matrix3d { // column-major
    double d[9];
};
struct CameraPose { // camera_pose.h:40-68
    Vector4d q{{1, 0, 0, 0}};
    Vector3d t{{0, 0, 0}};
};
struct Camera { // misc/camera_models.h:59-63
    int model_id = -1, width = 0, height = 0;
    std::vector<double> params;
};
struct Image {
    CameraPose pose;
    Camera camera;
};
struct ImagePair {
    CameraPose pose;
    Camera camera1, camera2;
};
struct BundleOptions { // types.h:60-95
    size_t max_iterations = 100;
    enum LossType { TRIVIAL, TRUNCATED, HUBER, CAUCHY, TRUNCATED_CAUCHY, TRUNCATED_LE_ZACH } loss_type = CAUCHY;
    double loss_scale = 1.0, gradient_tol = 1e-12, step_tol = 1e-8, relative_cost_tol = 1e-10, initial_lambda = 1e-3,
           min_lambda = 1e-10, max_lambda = 1e10;
    bool verbose = false;
    enum LambdaUpdateType { NIELSEN, FIXED_FACTOR } lambda_update = NIELSEN;
    double lambda_factor = 10.0;
    enum DampingType { LEVENBERG, MARQUARDT } damping = LEVENBERG;
    bool refine_focal_length = false, refine_extra_params = false, refine_principal_point = false;
};
struct BundleStats { // types.h:97-106, the fields the adapter fills
    size_t iterations = 0;
    double initial_cost = 0, cost = 0;
};
} // namespace standin

using namespace standin;

namespace {
int failures = 0;
void expect(bool ok, const char *what) {
    if (!ok) {
        std::printf("FAILED: %s\n", what);
        ++failures;
    }
}
bool same(const double *a, const double *b, int n) { return std::memcmp(a, b, sizeof(double) * n) == 0; }
bool same_stats(const BundleStats &s, const double *c) {
    return s.iterations == (size_t)c[0] && s.initial_cost == c[1] && s.cost == c[2];
}
void pose_to(const CameraPose &p, double *m) {
    for (int i = 0; i < 4; ++i) m[i] = p.q(i);
    for (int i = 0; i < 3; ++i) m[4 + i] = p.t(i);
}
bool same_pose(const CameraPose &p, const double *m) {
    double a[7];
    pose_to(p, a);
    return same(a, m, 7);
}
plb_camera cam_c(const Camera &c) {
    plb_camera o;
    std::memset(&o, 0, sizeof(o));
    o.model_id = c.model_id;
    for (size_t i = 0; i < c.params.size(); ++i) o.params[i] = c.params[i];
    return o;
}
} // namespace

int main(int argc, char **argv) {
    // a PINHOLE scene (focal 800) and its second view; every 9th observation is an outlier
    const int n = 300;
    std::vector<Vector2d> x(n), x1(n), x2(n), c1(n), c2(n);
    std::vector<Vector3d> X(n);
    std::vector<double> w(n), w_short(n - 1), w_long(n + 1, 1.0);
    for (int i = 0; i < n; ++i) {
        const double a = 0.37 * i, b = 0.11 * i;
        X[i] = Vector3d{{std::sin(a), std::cos(1.3 * a) * 0.7, 4.0 + std::sin(b)}};
        x[i] = Vector2d{{800.0 * X[i](0) / X[i](2) + 320.0, 800.0 * X[i](1) / X[i](2) + 240.0}};
        const double Y0 = X[i](0) - 0.5, Y1 = X[i](1) + 0.05, Y2 = X[i](2) + 0.1; // second camera: a translation
        x1[i] = Vector2d{{X[i](0) / X[i](2), X[i](1) / X[i](2)}};
        x2[i] = Vector2d{{Y0 / Y2, Y1 / Y2}};
        c1[i] = x[i];
        c2[i] = Vector2d{{800.0 * x2[i](0) + 320.0, 800.0 * x2[i](1) + 240.0}};
        if (i % 9 == 4) {
            x[i](0) += 25.0;
            x2[i](1) += 0.03;
            c2[i](1) += 24.0;
        }
        w[i] = i % 9 == 4 ? 0.05 : (i % 10 == 7 ? 0.0 : 0.5 + 0.01 * (i % 50));
        if (i < n - 1) w_short[i] = w[i];
    }
    BundleOptions bo;
    bo.loss_scale = 2.0;
    if (argc > 1 && std::strcmp(argv[1], "run") == 0) {
        const plb_bundle_opt c = poselib_b200::detail::bundle_to_c(bo);
        BundleOptions bn = bo;
        bn.loss_scale = 2.0 / 800.0;
        const plb_bundle_opt cn = poselib_b200::detail::bundle_to_c(bn);
        CameraPose p0;
        p0.q = Vector4d{{0.9999, 0.01, -0.005, 0.002}};
        p0.t = Vector3d{{0.01, -0.02, 0.01}};
        // bundle_adjust(x, X, Image*, opt, weights)
        {
            Image img0;
            img0.pose = p0;
            img0.camera.model_id = 1;
            img0.camera.params = {808.0, 805.0, 321.0, 239.0};
            BundleOptions b7 = bo;
            b7.refine_focal_length = b7.refine_principal_point = b7.refine_extra_params = true;
            const plb_bundle_opt c7 = poselib_b200::detail::bundle_to_c(b7);
            for (int variant = 0; variant < 3; ++variant) { // weights of size n, n - 1, n + 1
                const std::vector<double> &wv = variant == 0 ? w : variant == 1 ? w_short : w_long;
                Image img = img0;
                const BundleStats s = poselib_b200::bundle_adjust_image<BundleStats>(x, X, &img, b7, wv);
                double m[7], st[3];
                pose_to(p0, m);
                plb_camera cam = cam_c(img0.camera);
                const int rc = variant == 0
                                   ? plb_bundle_adjust_image_weighted(&x[0](0), &X[0](0), n, m, &cam, &c7, st, w.data())
                                   : plb_bundle_adjust_image(&x[0](0), &X[0](0), n, m, &cam, &c7, st);
                expect(rc == 0 && same_pose(img.pose, m) && same_stats(s, st) && same(img.camera.params.data(), cam.params, 4),
                       variant == 0 ? "bundle_adjust_image: weights of size n" : "bundle_adjust_image: other sizes");
            }
            if (failures == 0) { // the weights change the result
                Image a = img0, b = img0;
                poselib_b200::bundle_adjust_image<BundleStats>(x, X, &a, b7, w);
                poselib_b200::bundle_adjust_image<BundleStats>(x, X, &b, b7);
                expect(!same(a.camera.params.data(), b.camera.params.data(), 4), "bundle_adjust_image: weights used");
            }
        }
        // bundle_adjust(x, X, CameraPose*, opt, weights): the weights are ignored
        {
            std::vector<Vector2d> xn(n);
            for (int i = 0; i < n; ++i) xn[i] = Vector2d{{(x[i](0) - 320.0) / 800.0, (x[i](1) - 240.0) / 800.0}};
            CameraPose a = p0, b = p0;
            const BundleStats sa = poselib_b200::bundle_adjust<BundleStats>(xn, X, &a, bn, w);
            const BundleStats sb = poselib_b200::bundle_adjust<BundleStats>(xn, X, &b, bn);
            double mb[7];
            pose_to(b, mb);
            const double sbv[3] = {(double)sb.iterations, sb.initial_cost, sb.cost};
            expect(same_pose(a, mb) && same_stats(sa, sbv), "bundle_adjust(CameraPose*): weights ignored");
        }
        // refine_relpose(x1, x2, CameraPose*, opt, weights)
        CameraPose r0;
        r0.q = Vector4d{{0.99995, 0.005, -0.004, 0.003}};
        r0.t = Vector3d{{-0.97, 0.12, 0.2}};
        {
            const double nt = std::sqrt(r0.t(0) * r0.t(0) + r0.t(1) * r0.t(1) + r0.t(2) * r0.t(2));
            for (int i = 0; i < 3; ++i) r0.t(i) /= nt;
        }
        for (int variant = 0; variant < 3; ++variant) {
            const std::vector<double> &wv = variant == 0 ? w : variant == 1 ? w_short : w_long;
            CameraPose p = r0;
            const BundleStats s = poselib_b200::refine_relpose<BundleStats>(x1, x2, &p, bn, wv);
            double m[7], st[3];
            pose_to(r0, m);
            const int rc = variant == 0 ? plb_refine_relpose_weighted(&x1[0](0), &x2[0](0), n, m, &cn, st, w.data())
                                        : plb_refine_relpose(&x1[0](0), &x2[0](0), n, m, &cn, st);
            expect(rc == 0 && same_pose(p, m) && same_stats(s, st),
                   variant == 0 ? "refine_relpose: weights of size n" : "refine_relpose: other sizes");
        }
        // refine_relpose(x1, x2, ImagePair*, opt, weights), flags 0 and 7
        for (int flags = 0; flags <= 7; flags += 7) {
            ImagePair pr0;
            pr0.pose = r0;
            pr0.camera1.model_id = pr0.camera2.model_id = 1;
            pr0.camera1.params = {801.0, 802.0, 320.5, 240.5};
            pr0.camera2.params = {799.0, 800.0, 319.5, 239.0};
            BundleOptions bf = bo;
            bf.refine_focal_length = bf.refine_principal_point = bf.refine_extra_params = flags != 0;
            const plb_bundle_opt cf = poselib_b200::detail::bundle_to_c(bf);
            for (int variant = 0; variant < 3; ++variant) {
                const std::vector<double> &wv = variant == 0 ? w : variant == 1 ? w_short : w_long;
                ImagePair pr = pr0;
                const BundleStats s = poselib_b200::refine_relpose_pair<BundleStats>(c1, c2, &pr, bf, wv);
                double m[7], st[3];
                pose_to(r0, m);
                plb_camera k1 = cam_c(pr0.camera1), k2 = cam_c(pr0.camera2);
                const int rc = variant == 0 ? plb_refine_relpose_pair_weighted(&c1[0](0), &c2[0](0), n, &k1, &k2, m, &cf,
                                                                               st, w.data())
                                            : plb_refine_relpose_pair(&c1[0](0), &c2[0](0), n, &k1, &k2, m, &cf, st);
                expect(rc == 0 && same_pose(pr.pose, m) && same_stats(s, st) &&
                           same(pr.camera1.params.data(), k1.params, 4) && same(pr.camera2.params.data(), k2.params, 4),
                       variant == 0 ? "refine_relpose_pair: weights of size n" : "refine_relpose_pair: other sizes");
            }
        }
        // refine_fundamental / refine_homography: the essential matrix of the second view / a homography start
        {
            Matrix3d F0{{0.0, 0.1, -0.05, -0.1, 0.0, 0.5, 0.05, -0.5, 0.0}};
            Matrix3d H0{{1.0, 0.01, 0.0, -0.01, 1.0, 0.0, -0.12, 0.01, 1.0}};
            for (int hom = 0; hom < 2; ++hom)
                for (int variant = 0; variant < 3; ++variant) {
                    const std::vector<double> &wv = variant == 0 ? w : variant == 1 ? w_short : w_long;
                    Matrix3d M = hom ? H0 : F0, Mc = M;
                    double st[3];
                    BundleStats s;
                    int rc;
                    if (hom) {
                        s = poselib_b200::refine_homography<BundleStats>(x1, x2, &M, bn, wv);
                        rc = variant == 0 ? plb_refine_homography_weighted(&x1[0](0), &x2[0](0), n, Mc.d, &cn, st, w.data())
                                          : plb_refine_homography(&x1[0](0), &x2[0](0), n, Mc.d, &cn, st);
                    } else {
                        s = poselib_b200::refine_fundamental<BundleStats>(x1, x2, &M, bn, wv);
                        rc = variant == 0 ? plb_refine_fundamental_weighted(&x1[0](0), &x2[0](0), n, Mc.d, &cn, st, w.data())
                                          : plb_refine_fundamental(&x1[0](0), &x2[0](0), n, Mc.d, &cn, st);
                    }
                    expect(rc == 0 && same(M.d, Mc.d, 9) && same_stats(s, st),
                           hom ? "refine_homography: weights and sizes" : "refine_fundamental: weights and sizes");
                }
        }
        (void)c;
        if (failures) return 3;
        std::printf("adapter weights run ok\n");
        return 0;
    }
    // instantiate without running (link check)
    if (argc > 5) {
        Image img;
        ImagePair pr;
        CameraPose p;
        Matrix3d M{};
        poselib_b200::bundle_adjust_image<BundleStats>(x, X, &img, bo, w);
        poselib_b200::bundle_adjust<BundleStats>(x, X, &p, bo, w);
        poselib_b200::refine_relpose<BundleStats>(x1, x2, &p, bo, w);
        poselib_b200::refine_relpose_pair<BundleStats>(c1, c2, &pr, bo, w);
        poselib_b200::refine_fundamental<BundleStats>(x1, x2, &M, bo, w);
        poselib_b200::refine_homography<BundleStats>(x1, x2, &M, bo, w);
    }
    std::printf("adapter weights link ok\n");
    return 0;
}
