// A client written against PoseLib's OWN headers only — it does not know this repository exists — linked with
// poselib_b200/adapter/poselib_dropin.cc + libposelib_b200.so instead of PoseLib's CPU sources for the hot path
// (tests/test_dropin_reference_headers.py; Eigen is replaced by the test stand-in oracle/ref/mini at compile time because
// this image has no Eigen3).  Linking succeeds only if the drop-in defines every function below with exactly the
// signature PoseLib's headers declare.   oracle/_ref/dropin_client       -> link check only
//                                         oracle/_ref/dropin_client run   -> one call of every entry point on cuda:0
#include <PoseLib/robust.h>
#include <PoseLib/robust/bundle.h>
#include <PoseLib/robust/ransac.h>
#include <PoseLib/solvers/homography_4pt.h>
#include <PoseLib/solvers/p3p.h>
#include <PoseLib/solvers/p3p_lambdatwist.h>
#include <PoseLib/solvers/relpose_5pt.h>
#include <PoseLib/solvers/relpose_7pt.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>

using namespace poselib;

namespace {
struct Scene {
    std::vector<Point2D> x1, x2;     // normalised image points of two views
    std::vector<Point3D> X;          // 3D points in the frame of view 1
    CameraPose gt;                   // view 1 -> view 2
};
Scene make_scene(size_t n, double outlier_ratio, unsigned seed, bool planar) {
    std::mt19937 rng(seed);
    std::uniform_real_distribution<double> u(-1.0, 1.0);
    Scene s;
    const double a = 0.2;
    s.gt.q = Eigen::Vector4d(std::cos(a / 2), 0.0, std::sin(a / 2), 0.0); // rotation about y
    s.gt.t = Eigen::Vector3d(0.5, 0.1, 0.05);
    const double c = std::cos(a), sn = std::sin(a);
    for (size_t i = 0; i < n; ++i) {
        Point3D P(u(rng), u(rng), planar ? 4.0 : 4.0 + u(rng));
        Point3D Q(c * P(0) + sn * P(2) + s.gt.t(0), P(1) + s.gt.t(1), -sn * P(0) + c * P(2) + s.gt.t(2));
        Point2D p1(P(0) / P(2), P(1) / P(2)), p2(Q(0) / Q(2), Q(1) / Q(2));
        if (u(rng) * 0.5 + 0.5 < outlier_ratio) p2 = Point2D(0.3 * u(rng), 0.3 * u(rng));
        s.x1.push_back(p1);
        s.x2.push_back(p2);
        s.X.push_back(P);
    }
    return s;
}
int fail(const char *what) {
    std::printf("dropin client FAILED: %s\n", what);
    return 1;
}
} // namespace

int main(int argc, char **argv) {
    if (argc < 2 || std::strcmp(argv[1], "run") != 0) {
        // take the address of every entry point through the type its PoseLib declaration has: resolved at link time
        RansacStats (*e1)(const std::vector<Point2D> &, const std::vector<Point3D> &, AbsolutePoseOptions, Image *,
                          std::vector<char> *) = &estimate_absolute_pose;
        RansacStats (*e2)(const std::vector<Point2D> &, const std::vector<Point2D> &, const Camera &, const Camera &,
                          const RelativePoseOptions &, CameraPose *, std::vector<char> *) = &estimate_relative_pose;
        RansacStats (*e3)(const std::vector<Point2D> &, const std::vector<Point2D> &, const RelativePoseOptions &,
                          Eigen::Matrix3d *, std::vector<char> *) = &estimate_fundamental;
        RansacStats (*e4)(const std::vector<Point2D> &, const std::vector<Point2D> &, const HomographyOptions &,
                          Eigen::Matrix3d *, std::vector<char> *) = &estimate_homography;
        RansacStats (*r1)(const std::vector<Point2D> &, const std::vector<Point3D> &, const AbsolutePoseOptions &,
                          CameraPose *, std::vector<char> *) = &ransac_pnp;
        RansacStats (*r2)(const std::vector<Point2D> &, const std::vector<Point2D> &, const RelativePoseOptions &,
                          CameraPose *, std::vector<char> *) = &ransac_relpose;
        RansacStats (*r3)(const std::vector<Point2D> &, const std::vector<Point2D> &, const Camera &, const Camera &,
                          const RelativePoseOptions &, CameraPose *, std::vector<char> *) = &ransac_relpose;
        RansacStats (*r4)(const std::vector<Point2D> &, const std::vector<Point2D> &, const RelativePoseOptions &,
                          Eigen::Matrix3d *, std::vector<char> *) = &ransac_fundamental;
        RansacStats (*r5)(const std::vector<Point2D> &, const std::vector<Point2D> &, const HomographyOptions &,
                          Eigen::Matrix3d *, std::vector<char> *) = &ransac_homography;
        BundleStats (*b1)(const std::vector<Point2D> &, const std::vector<Point3D> &, CameraPose *, const BundleOptions &,
                          const std::vector<double> &) = &bundle_adjust;
        BundleStats (*b2)(const std::vector<Point2D> &, const std::vector<Point2D> &, CameraPose *, const BundleOptions &,
                          const std::vector<double> &) = &refine_relpose;
        BundleStats (*b3)(const std::vector<Point2D> &, const std::vector<Point2D> &, Eigen::Matrix3d *,
                          const BundleOptions &, const std::vector<double> &) = &refine_fundamental;
        BundleStats (*b4)(const std::vector<Point2D> &, const std::vector<Point2D> &, Eigen::Matrix3d *,
                          const BundleOptions &, const std::vector<double> &) = &refine_homography;
        int (*s1)(const std::vector<Eigen::Vector3d> &, const std::vector<Eigen::Vector3d> &, std::vector<CameraPose> *) = &p3p;
        int (*s2)(const std::vector<Eigen::Vector3d> &, const std::vector<Eigen::Vector3d> &,
                  std::vector<Eigen::Matrix3d> *) = &relpose_5pt;
        int (*s3)(const std::vector<Eigen::Vector3d> &, const std::vector<Eigen::Vector3d> &, std::vector<CameraPose> *) =
            &relpose_5pt;
        int (*s4)(const std::vector<Eigen::Vector3d> &, const std::vector<Eigen::Vector3d> &,
                  std::vector<Eigen::Matrix3d> *) = &relpose_7pt;
        int (*s5)(const std::vector<Eigen::Vector3d> &, const std::vector<Eigen::Vector3d> &, Eigen::Matrix3d *, bool) =
            &homography_4pt;
        int (*s6)(const std::vector<Eigen::Vector3d> &, const std::vector<Eigen::Vector3d> &, std::vector<CameraPose> *) =
            &p3p_lambdatwist;
        const void *all[] = {(void *)e1, (void *)e2, (void *)e3, (void *)e4, (void *)r1, (void *)r2, (void *)r3,
                             (void *)r4, (void *)r5, (void *)b1, (void *)b2, (void *)b3, (void *)b4, (void *)s1,
                             (void *)s2, (void *)s3, (void *)s4, (void *)s5, (void *)s6};
        for (const void *p : all)
            if (!p) return fail("null entry point");
        std::printf("dropin link ok: %zu PoseLib entry points resolved\n", sizeof(all) / sizeof(all[0]));
        return 0;
    }

    // ---- run: PoseLib call sites, CUDA implementation ------------------------------------------------------------
    const double f = 1000.0;
    Camera cam(1 /* PINHOLE */, std::vector<double>{f, f, 0.0, 0.0});
    Scene sc = make_scene(2000, 0.5, 1, false);
    std::vector<Point2D> px1 = sc.x1, px2 = sc.x2;
    for (auto &p : px1) p = p * f;
    for (auto &p : px2) p = p * f;

    RelativePoseOptions ro;
    ro.max_error = 1.0;
    ro.ransac.max_iterations = 5000;
    ro.ransac.min_iterations = 200;
    CameraPose pose;
    std::vector<char> inl;
    RansacStats st = estimate_relative_pose(px1, px2, cam, cam, ro, &pose, &inl);
    if (st.num_inliers < 900 || inl.size() != px1.size()) return fail("estimate_relative_pose inliers");
    const double dq = std::abs(std::abs(pose.q.dot(sc.gt.q)) - 1.0);
    const double dt = (pose.t.normalized() - sc.gt.t.normalized()).norm();
    std::printf("estimate_relative_pose: inliers=%zu dq=%.3g dt=%.3g\n", (size_t)st.num_inliers, dq, dt);
    if (dq > 1e-6 || dt > 2e-3) return fail("estimate_relative_pose accuracy");

    AbsolutePoseOptions ao;
    ao.max_error = 2.0;
    ao.ransac.max_iterations = 2000;
    ao.ransac.min_iterations = 100;
    Image image;
    image.camera = cam;
    std::vector<Point3D> Xw = sc.X; // world = view 1, so the absolute pose of view 2 equals the relative pose
    st = estimate_absolute_pose(px2, Xw, ao, &image, &inl);
    std::printf("estimate_absolute_pose: inliers=%zu dt=%.3g\n", (size_t)st.num_inliers, (image.pose.t - sc.gt.t).norm());
    if (st.num_inliers < 900) return fail("estimate_absolute_pose inliers");
    if ((image.pose.t - sc.gt.t).norm() > 1e-3) return fail("estimate_absolute_pose accuracy");

    Eigen::Matrix3d F;
    st = estimate_fundamental(px1, px2, ro, &F, &inl);
    std::printf("estimate_fundamental: inliers=%zu\n", (size_t)st.num_inliers);
    if (st.num_inliers < 900) return fail("estimate_fundamental inliers");

    Scene pl = make_scene(1500, 0.4, 2, true);
    std::vector<Point2D> h1 = pl.x1, h2 = pl.x2;
    for (auto &p : h1) p = p * f;
    for (auto &p : h2) p = p * f;
    HomographyOptions ho;
    ho.max_error = 1.0;
    ho.ransac.max_iterations = 2000;
    Eigen::Matrix3d H;
    st = estimate_homography(h1, h2, ho, &H, &inl);
    std::printf("estimate_homography: inliers=%zu\n", (size_t)st.num_inliers);
    if (st.num_inliers < 800) return fail("estimate_homography inliers");

    RelativePoseOptions rn = ro;
    rn.max_error = 1.0 / f;
    CameraPose p2;
    st = ransac_relpose(sc.x1, sc.x2, rn, &p2, &inl);
    std::printf("ransac_relpose: inliers=%zu\n", (size_t)st.num_inliers);
    if (st.num_inliers < 900) return fail("ransac_relpose inliers");
    BundleStats bs = refine_relpose(sc.x1, sc.x2, &p2, BundleOptions());
    std::printf("refine_relpose: cost %.6g -> %.6g\n", bs.initial_cost, bs.cost);
    if (!(bs.cost <= bs.initial_cost)) return fail("refine_relpose cost");

    std::vector<Eigen::Vector3d> b1, b2;
    for (int i = 0; i < 5; ++i) {
        b1.push_back(Eigen::Vector3d(pl.x1[i](0), pl.x1[i](1), 1.0).normalized());
        b2.push_back(Eigen::Vector3d(sc.x2[i](0), sc.x2[i](1), 1.0).normalized());
    }
    std::vector<Eigen::Matrix3d> Es;
    const int n5 = relpose_5pt(b1, b2, &Es);
    std::printf("relpose_5pt: %d solutions\n", n5);
    if (n5 != (int)Es.size()) return fail("relpose_5pt count");
    std::printf("dropin run ok\n");
    return 0;
}
