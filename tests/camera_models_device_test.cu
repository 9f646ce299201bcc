// Device-side check of the camera functions of poselib_b200/csrc/camera.cuh with the fisheye and division models
// (X = true): one kernel evaluates every function on the given pixels and camera-frame points on the GPU, and the same
// functions are evaluated by the host build of the same source, which tests/test_camera_models.py pins bit for bit to
// the reference.  Both are printed as hex doubles ("dev" / "host" lines, the layout of camera_models_host_test.cu's
// "px" / "pt" rows) for tests/test_camera_models.py.
#include "../poselib_b200/csrc/camera.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

using namespace plb;

constexpr int PX_W = 3 + 2 + 3 + 6 + 3 + 6 + 3 * CAM_MAX_PARAMS; // row width of a pixel
constexpr int PT_W = 4 + 6 + 2 * CAM_MAX_PARAMS;                 // row width of a camera-frame point

__host__ __device__ void eval_px(const CamDev &c, double u, double v, double *o) {
    for (int i = 0; i < PX_W; ++i) o[i] = 0.0;
    cam_unproject<true>(c, u, v, o);
    cam_unproject2<true>(c, u, v, o[3], o[4]);
    cam_unproject_with_jac<true>(c, u, v, o + 5, o + 8);
    cam_unproject_with_jac_params<true>(c, u, v, o + 14, o + 17, o + 23);
}
__host__ __device__ void eval_pt(const CamDev &c, double X, double Y, double Z, double *o) {
    for (int i = 0; i < PT_W; ++i) o[i] = 0.0;
    cam_project<true>(c, X, Y, Z, o[0], o[1]);
    cam_project_with_jac<true>(c, X, Y, Z, o[2], o[3], o + 4);
    cam_jac_params<true>(c, X, Y, Z, o + 10);
}
__global__ void k_eval(CamDev c, const double *in, int n, bool px, double *out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    if (px)
        eval_px(c, in[2 * k], in[2 * k + 1], out + (size_t)PX_W * k);
    else
        eval_pt(c, in[3 * k], in[3 * k + 1], in[3 * k + 2], out + (size_t)PT_W * k);
}

static int check(cudaError_t e, const char *what) {
    if (e == cudaSuccess) return 0;
    std::fprintf(stderr, "%s: %s\n", what, cudaGetErrorString(e));
    return 1;
}

int main(int argc, char **argv) {
    // argv: model p0..p7, then "px" u v pairs or "pt" X Y Z triples until the end
    if (argc < 11) return 2;
    CamDev c;
    c.model = std::atoi(argv[1]);
    c.reserved = 0;
    for (int i = 0; i < 8; ++i) c.p[i] = std::strtod(argv[2 + i], nullptr);
    const bool px = std::strcmp(argv[10], "px") == 0;
    const int dim = px ? 2 : 3, w = px ? PX_W : PT_W;
    std::vector<double> in;
    for (int a = 11; a < argc; ++a) in.push_back(std::strtod(argv[a], nullptr));
    const int n = (int)in.size() / dim;
    std::vector<double> dev((size_t)w * n), host((size_t)w * n);
    double *d_in = nullptr, *d_out = nullptr;
    if (check(cudaMalloc(&d_in, sizeof(double) * in.size()), "cudaMalloc") ||
        check(cudaMalloc(&d_out, sizeof(double) * dev.size()), "cudaMalloc") ||
        check(cudaMemcpy(d_in, in.data(), sizeof(double) * in.size(), cudaMemcpyHostToDevice), "cudaMemcpy"))
        return 1;
    k_eval<<<(n + 63) / 64, 64>>>(c, d_in, n, px, d_out);
    if (check(cudaGetLastError(), "launch") ||
        check(cudaMemcpy(dev.data(), d_out, sizeof(double) * dev.size(), cudaMemcpyDeviceToHost), "cudaMemcpy"))
        return 1;
    cudaFree(d_in);
    cudaFree(d_out);
    for (int k = 0; k < n; ++k) {
        if (px)
            eval_px(c, in[2 * k], in[2 * k + 1], host.data() + (size_t)w * k);
        else
            eval_pt(c, in[3 * k], in[3 * k + 1], in[3 * k + 2], host.data() + (size_t)w * k);
    }
    for (int k = 0; k < n; ++k) {
        std::printf("dev");
        for (int i = 0; i < w; ++i) std::printf(" %a", dev[(size_t)w * k + i]);
        std::printf("\nhost");
        for (int i = 0; i < w; ++i) std::printf(" %a", host[(size_t)w * k + i]);
        std::printf("\n");
    }
    return 0;
}
