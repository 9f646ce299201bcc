// Device-side check of the degree-10 Sturm root finder of poselib_b200/csrc/solvers.cuh.  Two kernels run on the same
// polynomials:
//   k_warp    mirrors k5_roots of kernels.cu (64-thread CTAs, one lane per polynomial, lanes past the end of the list
//             take part with zero coefficients and has_poly = false) and calls sturm_bisect10_warp;
//   k_serial  one thread per polynomial, calling the serial sturm_bisect10.
// The real k5_roots runs through the library's 5-point solver surface; tests/test_solver_degenerate.py checks that
// separately.  Input (stdin): lists of polynomials, each "n" followed by 11 * n ascending coefficients as hex doubles.
// Output: for every list, one "L n" line, then per polynomial a "w count roots..." and an "s count roots..." line, the
// roots printed with %a.
#include "../poselib_b200/csrc/solvers.cuh"
#include <cstdio>
#include <cstdlib>
#include <vector>

using namespace plb;

constexpr int THREADS = 64;

__global__ void __launch_bounds__(THREADS) k_warp(int n, const double *cpoly, int *nroots, double *roots_out) {
    __shared__ RootsShared S[THREADS / 32];
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    const bool has = g < n;
    double c[11], roots[10];
#pragma unroll
    for (int k = 0; k < 11; ++k) c[k] = has ? cpoly[(size_t)k * n + g] : 0.0;
    const int nr = sturm_bisect10_warp(c, has, roots, &S[threadIdx.x >> 5], threadIdx.x & 31);
    if (has) {
        nroots[g] = nr;
        double *o = roots_out + (size_t)g * 10;
        for (int k = 0; k < nr; ++k) o[k] = roots[k];
    }
}

__global__ void k_serial(int n, const double *cpoly, int *nroots, double *roots_out) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n) return;
    double c[11], roots[10];
    for (int k = 0; k < 11; ++k) c[k] = cpoly[(size_t)k * n + g];
    SturmWork w;
    const int nr = sturm_bisect10(c, roots, &w);
    nroots[g] = nr;
    for (int k = 0; k < nr; ++k) roots_out[(size_t)g * 10 + k] = roots[k];
}

static int check(cudaError_t e, const char *what) {
    if (e == cudaSuccess) return 0;
    std::fprintf(stderr, "%s: %s\n", what, cudaGetErrorString(e));
    return 1;
}

static void print_row(const char *tag, const std::vector<int> &nr, const std::vector<double> &r, int g) {
    std::printf("%s %d", tag, nr[g]);
    for (int k = 0; k < nr[g] && k < 10; ++k) std::printf(" %a", r[(size_t)g * 10 + k]);
    std::printf("\n");
}

int main() {
    char tok[64];
    int n;
    while (std::scanf("%d", &n) == 1) {
        if (n <= 0) return 2;
        std::vector<double> cp((size_t)11 * n); // coefficient-major, the layout of HypOut::s5_cpoly
        for (int g = 0; g < n; ++g)
            for (int k = 0; k < 11; ++k) {
                if (std::scanf("%63s", tok) != 1) return 2;
                cp[(size_t)k * n + g] = std::strtod(tok, nullptr);
            }
        double *d_c = nullptr, *d_rw = nullptr, *d_rs = nullptr;
        int *d_nw = nullptr, *d_ns = nullptr;
        const size_t rb = sizeof(double) * 10 * n;
        if (check(cudaMalloc(&d_c, sizeof(double) * cp.size()), "cudaMalloc") ||
            check(cudaMalloc(&d_rw, rb), "cudaMalloc") || check(cudaMalloc(&d_rs, rb), "cudaMalloc") ||
            check(cudaMalloc(&d_nw, sizeof(int) * n), "cudaMalloc") ||
            check(cudaMalloc(&d_ns, sizeof(int) * n), "cudaMalloc") ||
            check(cudaMemcpy(d_c, cp.data(), sizeof(double) * cp.size(), cudaMemcpyHostToDevice), "cudaMemcpy") ||
            check(cudaMemset(d_rw, 0, rb), "cudaMemset") || check(cudaMemset(d_rs, 0, rb), "cudaMemset"))
            return 1;
        const int blocks = (n + THREADS - 1) / THREADS;
        k_warp<<<blocks, THREADS>>>(n, d_c, d_nw, d_rw);
        if (check(cudaGetLastError(), "launch k_warp")) return 1;
        k_serial<<<blocks, THREADS>>>(n, d_c, d_ns, d_rs);
        if (check(cudaGetLastError(), "launch k_serial")) return 1;
        std::vector<int> nw(n), ns(n);
        std::vector<double> rw((size_t)10 * n), rs((size_t)10 * n);
        if (check(cudaMemcpy(nw.data(), d_nw, sizeof(int) * n, cudaMemcpyDeviceToHost), "cudaMemcpy") ||
            check(cudaMemcpy(ns.data(), d_ns, sizeof(int) * n, cudaMemcpyDeviceToHost), "cudaMemcpy") ||
            check(cudaMemcpy(rw.data(), d_rw, rb, cudaMemcpyDeviceToHost), "cudaMemcpy") ||
            check(cudaMemcpy(rs.data(), d_rs, rb, cudaMemcpyDeviceToHost), "cudaMemcpy"))
            return 1;
        cudaFree(d_c);
        cudaFree(d_rw);
        cudaFree(d_rs);
        cudaFree(d_nw);
        cudaFree(d_ns);
        std::printf("L %d\n", n);
        for (int g = 0; g < n; ++g) {
            print_row("w", nw, rw, g);
            print_row("s", ns, rs, g);
        }
    }
    return 0;
}
