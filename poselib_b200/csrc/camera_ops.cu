// poselib_b200 — the camera models' project / unproject (and their Jacobians) over many points, for sm_90a (H100):
//   k_camera<OP, JAC, T>   plb_camera_batch[_device]
// A translation unit of its own: the fisheye and division functions of camera.cuh are called, not inlined, and the
// kernels of kernels.cu that call them keep the code they compile to when these callers are not in the same module.
// Compiled with -fmad=false (see device_math.cuh).
#include "kernels.cuh"

namespace plb {

// ---- the camera functions over many points (plb_camera_batch) ------------------------------------------------------
// A persistent 1D grid walks the tiles of the descriptors, each found by binary search on tile0 as in k_score, so neither
// n nor the number of problems is capped by a grid dimension.  Thread 0 loads the tile's camera into shared memory once;
// every point of a tile has that camera, so the model switch does not diverge.  One thread per point calls the camera.cuh
// functions with the fisheye and division models (X):
//   PROJECT        cam_project; JAC: cam_project_with_jac, and cam_jac_params when jac_params is given;
//   UNPROJECT      cam_unproject; JAC: cam_unproject_with_jac, or cam_unproject_with_jac_params when jac_params is given;
//   UNPROJECT_2D   cam_unproject2.
// The functions' row-major matrices go out column-major, as Eigen stores them.  T: the input type, widened exactly.
template <int OP, bool JAC, typename T>
__global__ void __launch_bounds__(CAM_TILE) k_camera(const CamOpDesc *__restrict__ descs, int n_desc, long long n_tiles) {
    constexpr int IN = OP == CAMOP_PROJECT ? 3 : 2, OUT = OP == CAMOP_UNPROJECT ? 3 : 2;
    __shared__ CamDev cam;
    __shared__ const CamOpDesc *item;
    __shared__ long long item_k0;
    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        if (threadIdx.x == 0) {
            int lo = 0, hi = n_desc - 1; // the last descriptor with tile0 <= t
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (descs[mid].tile0 <= t) lo = mid;
                else hi = mid - 1;
            }
            item = descs + lo;
            item_k0 = (t - descs[lo].tile0) * CAM_TILE;
            cam = descs[lo].cam;
        }
        __syncthreads();
        const CamOpDesc &D = *item;
        const long long k = item_k0 + threadIdx.x;
        if (k < D.n) {
            const T *in = static_cast<const T *>(D.in) + k * IN;
            double x[IN];
#pragma unroll
            for (int i = 0; i < IN; ++i) x[i] = (double)in[i];
            double o[OUT];
            if (OP == CAMOP_PROJECT) {
                if (!JAC) {
                    cam_project<true>(cam, x[0], x[1], x[IN - 1], o[0], o[1]);
                } else {
                    double J[6];
                    cam_project_with_jac<true>(cam, x[0], x[1], x[IN - 1], o[0], o[1], J);
                    if (D.jac)
                        for (int r = 0; r < 2; ++r)
                            for (int c = 0; c < 3; ++c) D.jac[6 * k + r + 2 * c] = J[3 * r + c];
                    if (D.jac_params) {
                        double jp[2 * CAM_MAX_PARAMS];
                        cam_jac_params<true>(cam, x[0], x[1], x[IN - 1], jp);
                        const int np = cam_num_params(cam.model);
                        for (int c = 0; c < np; ++c)
                            for (int r = 0; r < 2; ++r) D.jac_params[2 * np * k + r + 2 * c] = jp[CAM_MAX_PARAMS * r + c];
                    }
                }
            } else if (OP == CAMOP_UNPROJECT) {
                if (!JAC) {
                    cam_unproject<true>(cam, x[0], x[1], o);
                } else {
                    double M[6];
                    if (D.jac_params) {
                        double dp[3 * CAM_MAX_PARAMS];
                        cam_unproject_with_jac_params<true>(cam, x[0], x[1], o, M, dp);
                        const int np = cam_num_params(cam.model);
                        for (int c = 0; c < np; ++c)
                            for (int r = 0; r < 3; ++r) D.jac_params[3 * np * k + r + 3 * c] = dp[CAM_MAX_PARAMS * r + c];
                    } else {
                        cam_unproject_with_jac<true>(cam, x[0], x[1], o, M);
                    }
                    if (D.jac)
                        for (int r = 0; r < 3; ++r)
                            for (int c = 0; c < 2; ++c) D.jac[6 * k + r + 3 * c] = M[2 * r + c];
                }
            } else {
                cam_unproject2<true>(cam, x[0], x[1], o[0], o[OUT - 1]);
            }
#pragma unroll
            for (int i = 0; i < OUT; ++i) D.out[OUT * k + i] = o[i];
        }
        __syncthreads(); // the shared item is rewritten for the next tile
    }
}
template <int OP, bool JAC>
static void launch_camera_t(bool f32, const CamOpDesc *descs_dev, int n_desc, long long n_tiles, cudaStream_t stream) {
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        sms = 132;
    const unsigned blocks = (unsigned)(n_tiles < 8LL * sms ? n_tiles : 8LL * sms);
    if (f32)
        k_camera<OP, JAC, float><<<blocks, CAM_TILE, 0, stream>>>(descs_dev, n_desc, n_tiles);
    else
        k_camera<OP, JAC, double><<<blocks, CAM_TILE, 0, stream>>>(descs_dev, n_desc, n_tiles);
}
void launch_camera(int op, bool jac, bool f32, const CamOpDesc *descs_dev, int n_desc, long long n_tiles,
                   cudaStream_t stream) {
    if (n_desc <= 0 || n_tiles <= 0) return;
    if (op == CAMOP_PROJECT && jac) launch_camera_t<CAMOP_PROJECT, true>(f32, descs_dev, n_desc, n_tiles, stream);
    else if (op == CAMOP_PROJECT) launch_camera_t<CAMOP_PROJECT, false>(f32, descs_dev, n_desc, n_tiles, stream);
    else if (op == CAMOP_UNPROJECT && jac) launch_camera_t<CAMOP_UNPROJECT, true>(f32, descs_dev, n_desc, n_tiles, stream);
    else if (op == CAMOP_UNPROJECT) launch_camera_t<CAMOP_UNPROJECT, false>(f32, descs_dev, n_desc, n_tiles, stream);
    else launch_camera_t<CAMOP_UNPROJECT_2D, false>(f32, descs_dev, n_desc, n_tiles, stream);
}

} // namespace plb
