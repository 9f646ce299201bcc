// Test client of PoseLib's own estimators' generate_models and score_model: AbsolutePoseEstimator,
// RelativePoseEstimator, CameraRelativePoseEstimator, FundamentalEstimator (with and without real_focal_check) and
// HomographyEstimator, built with a seeded RansacOptions and asked for S hypothesis sets in a row, as ransac() asks them.
// The samples they draw come from the estimator's own RandomSampler; a second RandomSampler with the same options
// records them.  It is compiled against the reference's headers and linked with the reference's sources built on
// mini-Eigen (oracle/_ref/libplref2.so, or libplref2_alt.so for the other summation order);
// tests/golden/make_generate_golden.py builds it.
#include "PoseLib/misc/camera_models.h"
#include "PoseLib/robust/estimators/absolute_pose.h"
#include "PoseLib/robust/estimators/homography.h"
#include "PoseLib/robust/estimators/relative_pose.h"
#include "PoseLib/robust/sampling.h"

#include <cstdint>
#include <vector>

using namespace poselib;

namespace {
int num_params(int model) {
    switch (model) {
    case 0: return 3;
    case 1: case 2: case 8: case 102: return 4;
    case 3: case 9: case 101: return 5;
    case 4: return 8;
    default: return 0;
    }
}
Camera camera(int model, const double *params) {
    Camera c;
    c.model_id = model;
    c.width = c.height = 0;
    c.params.assign(params, params + num_params(model));
    return c;
}
std::vector<Point2D> v2(const double *a, int64_t n) {
    std::vector<Point2D> v(n);
    for (int64_t k = 0; k < n; ++k) v[k] = Point2D(a[2 * k], a[2 * k + 1]);
    return v;
}
std::vector<Point3D> v3(const double *a, int64_t n) {
    std::vector<Point3D> v(n);
    for (int64_t k = 0; k < n; ++k) v[k] = Point3D(a[3 * k], a[3 * k + 1], a[3 * k + 2]);
    return v;
}
void put(const CameraPose &p, double *out) {
    for (int i = 0; i < 4; ++i) out[i] = p.q(i);
    for (int i = 0; i < 3; ++i) out[4 + i] = p.t(i);
}
void put(const Eigen::Matrix3d &M, double *out) { // column-major
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) out[3 * c + r] = M(r, c);
}
// S calls of generate_models, each followed by score_model of every model; the sample of call j drawn again by `smp`.
// Row j of models / scores / counts holds maxm slots of msz doubles.
template <typename Est, typename Model>
void run(Est &est, RandomSampler &smp, size_t k, int64_t S, int maxm, int msz, int32_t *samples, int32_t *n_models,
         double *models, double *scores, uint64_t *counts) {
    std::vector<size_t> sample(k);
    std::vector<Model> hyp;
    for (int64_t j = 0; j < S; ++j) {
        smp.generate_sample(&sample);
        for (size_t i = 0; i < k; ++i) samples[j * k + i] = (int32_t)sample[i];
        est.generate_models(&hyp);
        n_models[j] = (int32_t)hyp.size();
        for (size_t m = 0; m < hyp.size() && (int)m < maxm; ++m) {
            put(hyp[m], models + (j * maxm + m) * msz);
            size_t cnt = 0;
            scores[j * maxm + m] = est.score_model(hyp[m], &cnt);
            counts[j * maxm + m] = cnt;
        }
    }
}
} // namespace

extern "C" {
// kind: 0 PnP, 1 relative pose, 2 relative pose with cameras (tangent Sampson), 3 fundamental, 4 homography.
// a / b: x, X (PnP) or x1, x2 (pixels of camera 1 / 2 for kind 2).  Samples S x k, models S x M x msz.
void gen_run(int kind, int real_focal_check, const double *a, const double *b, int64_t n, int model1,
             const double *params1, int model2, const double *params2, double max_error, uint64_t seed, int prosac,
             int64_t S, int32_t *samples, int32_t *n_models, double *models, double *scores, uint64_t *counts) {
    RansacOptions ro;
    ro.seed = seed;
    ro.progressive_sampling = prosac != 0;
    const std::vector<Point2D> x1 = v2(a, n);
    if (kind == 0) {
        AbsolutePoseOptions opt;
        opt.ransac = ro;
        opt.max_error = max_error;
        const std::vector<Point3D> X = v3(b, n);
        AbsolutePoseEstimator est(opt, x1, X);
        RandomSampler smp(n, 3, ro);
        run<AbsolutePoseEstimator, CameraPose>(est, smp, 3, S, 4, 7, samples, n_models, models, scores, counts);
        return;
    }
    const std::vector<Point2D> x2 = v2(b, n);
    if (kind == 4) {
        HomographyOptions opt;
        opt.ransac = ro;
        opt.max_error = max_error;
        HomographyEstimator est(opt, x1, x2);
        RandomSampler smp(n, 4, ro);
        run<HomographyEstimator, Eigen::Matrix3d>(est, smp, 4, S, 1, 9, samples, n_models, models, scores, counts);
        return;
    }
    RelativePoseOptions opt;
    opt.ransac = ro;
    opt.max_error = max_error;
    opt.real_focal_check = real_focal_check != 0;
    if (kind == 1) {
        RelativePoseEstimator est(opt, x1, x2);
        RandomSampler smp(n, 5, ro);
        run<RelativePoseEstimator, CameraPose>(est, smp, 5, S, 40, 7, samples, n_models, models, scores, counts);
    } else if (kind == 2) {
        const Camera c1 = camera(model1, params1), c2 = camera(model2, params2);
        CameraRelativePoseEstimator est(opt, x1, x2, c1, c2);
        RandomSampler smp(n, 5, ro);
        run<CameraRelativePoseEstimator, CameraPose>(est, smp, 5, S, 40, 7, samples, n_models, models, scores, counts);
    } else {
        FundamentalEstimator est(opt, x1, x2);
        RandomSampler smp(n, 7, ro);
        run<FundamentalEstimator, Eigen::Matrix3d>(est, smp, 7, S, 3, 9, samples, n_models, models, scores, counts);
    }
}
} // extern "C"
