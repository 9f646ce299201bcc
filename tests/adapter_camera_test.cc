// The adapter's project_points / unproject_points against stand-ins for the Eigen / PoseLib types.  Built and run by
// tests/test_camera_batch.py; `run` (GPU) checks each template against the C-ABI call it wraps, bit for bit, on a few
// cameras; without `run` it only links.
#include "../poselib_b200/adapter/poselib_b200.hpp"

#include <cmath>
#include <cstdio>
#include <cstring>

namespace standin {
template <int N> struct Vec {
    double d[N];
};
using Vector2d = Vec<2>;
using Vector3d = Vec<3>;
template <int R, int C> struct Mat { // column-major, as Eigen::Matrix<double, R, C>
    double d[R * C];
};
struct MatDyn { // Eigen::Matrix<double, R, Eigen::Dynamic>: resize and column-major data()
    int rows = 0, cols = 0;
    std::vector<double> v;
    void resize(int r, int c) {
        rows = r;
        cols = c;
        v.assign((size_t)r * c, 0.0);
    }
    double *data() { return v.data(); }
};
struct Camera { // misc/camera_models.h:59-63
    int model_id = -1, width = 0, height = 0;
    std::vector<double> params;
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
// the C-ABI call the templates wrap, for one camera
void direct(int op, const Camera &cam, const double *in, size_t n, std::vector<double> &out, std::vector<double> &jac,
            std::vector<double> &jp, bool jacs) {
    const int rows = op == PLB_CAMOP_PROJECT ? 2 : 3;
    plb_camera_problem q = plb_camera_problem();
    q.op = op;
    q.n = n;
    q.camera = poselib_b200::detail::camera_to_c(cam);
    const int np = poselib_b200::detail::camera_num_params(q.camera.model_id);
    out.assign(n * rows, 0.0);
    jac.assign(n * 6, 0.0);
    jp.assign(n * rows * np + 1, 0.0);
    q.in = in;
    q.out = out.data();
    q.jac = jacs ? jac.data() : nullptr;
    q.jac_params = jacs ? jp.data() : nullptr;
    if (plb_camera_batch(&q, 1, -1, 1) != PLB_OK) std::printf("FAILED: plb_camera_batch: %s\n", plb_last_error()), ++failures;
    jp.resize(n * rows * np);
}
template <typename V> bool same(const std::vector<V> &a, const std::vector<double> &b) {
    return sizeof(V) * a.size() == sizeof(double) * b.size() && std::memcmp(a.data(), b.data(), sizeof(double) * b.size()) == 0;
}
bool same_dyn(const std::vector<MatDyn> &a, const std::vector<double> &b, int rows) {
    std::vector<double> flat;
    for (const MatDyn &m : a) {
        if (m.rows != rows) return false;
        flat.insert(flat.end(), m.v.begin(), m.v.end());
    }
    return flat.size() == b.size() && std::memcmp(flat.data(), b.data(), sizeof(double) * b.size()) == 0;
}
} // namespace

int main(int argc, char **argv) {
    const bool run = argc > 1 && std::strcmp(argv[1], "run") == 0;
    std::vector<Camera> cams(3);
    cams[0].model_id = 4;
    cams[0].params = {868.993378, 866.063001, 525.942323, 420.042529, -0.399431, 0.188924, 0.000153, 0.000571};
    cams[1].model_id = 101;
    cams[1].params = {820.0, 790.0, 330.0, 245.0, -0.2};
    cams[2].model_id = 9;
    cams[2].params = {1921.45, 2156.14, 1446.19, -0.0447036, -0.00511989};
    std::vector<std::vector<Vector3d>> X(3);
    std::vector<std::vector<Vector2d>> px(3);
    for (size_t c = 0; c < 3; ++c)
        for (size_t k = 0; k < 50 + 20 * c; ++k) {
            const double u = std::sin(0.37 * k + c), v = std::cos(0.23 * k), w = 2.0 + std::sin(0.11 * k);
            X[c].push_back(Vector3d{{u, v, w}});
            px[c].push_back(Vector2d{{400.0 + 300.0 * u, 300.0 + 200.0 * v}});
        }
    if (!run) {
        // instantiate every form; the library is linked but not called
        auto f0 = &poselib_b200::project_points<Camera, Vector3d, Vector2d>;
        auto f1 = &poselib_b200::project_points<Camera, Vector3d, Vector2d, Mat<2, 3>, MatDyn>;
        auto f2 = &poselib_b200::unproject_points<Camera, Vector2d, Vector3d>;
        auto f3 = &poselib_b200::unproject_points<Camera, Vector2d, Vector3d, Mat<3, 2>, MatDyn>;
        expect(f0 && f1 && f2 && f3, "templates instantiate");
        std::printf("adapter camera link ok\n");
        return failures ? 1 : 0;
    }
    std::vector<std::vector<Vector2d>> xp, xq;
    std::vector<std::vector<Mat<2, 3>>> J;
    std::vector<std::vector<MatDyn>> Jp, Mp;
    std::vector<std::vector<Vector3d>> b, d;
    std::vector<std::vector<Mat<3, 2>>> M;
    poselib_b200::project_points(cams, X, &xp);
    poselib_b200::project_points(cams, X, &xq, &J, &Jp);
    poselib_b200::unproject_points(cams, px, &b);
    poselib_b200::unproject_points(cams, px, &d, &M, &Mp);
    for (size_t c = 0; c < 3; ++c) {
        std::vector<double> out, jac, jp;
        direct(PLB_CAMOP_PROJECT, cams[c], &X[c][0].d[0], X[c].size(), out, jac, jp, false);
        expect(same(xp[c], out), "project");
        direct(PLB_CAMOP_PROJECT, cams[c], &X[c][0].d[0], X[c].size(), out, jac, jp, true);
        expect(same(xq[c], out) && same(J[c], jac) && same_dyn(Jp[c], jp, 2), "project_with_jac");
        direct(PLB_CAMOP_UNPROJECT, cams[c], &px[c][0].d[0], px[c].size(), out, jac, jp, false);
        expect(same(b[c], out), "unproject");
        direct(PLB_CAMOP_UNPROJECT, cams[c], &px[c][0].d[0], px[c].size(), out, jac, jp, true);
        expect(same(d[c], out) && same(M[c], jac) && same_dyn(Mp[c], jp, 3), "unproject_with_jac");
    }
    std::printf(failures ? "adapter camera FAILED\n" : "adapter camera ok\n");
    return failures ? 1 : 0;
}
