// Cycles and accuracy of the 32 x 32 diagonal-block factorisations in lvb_chol.cuh (one warp), and of the panel-row solve.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o diag_probe diag_probe.cu
#include <cstdio>
#include <cmath>
#include <vector>
#include <cuda_runtime.h>
#include "../lvio_fusion_b200/csrc/lvb_chol.cuh"
template <int V> __global__ void probe(const double* A, double* L, double* invd_out, long long* cyc, int* bad_out) {
    __shared__ __align__(16) double Dt[32 * 34];
    __shared__ double invd[32];
    const int lane = threadIdx.x;
    long long best = 1ll << 60; int bad = 0;
    for (int rep = 0; rep < 4; ++rep) {
        double a[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) a[j] = (j <= lane) ? A[lane * 32 + j] : ((j == lane) ? 1.0 : 0.0);
        __syncwarp();
        const long long t0 = clock64();
        bad = V == 0 ? chol_diag32(a, lane, Dt, invd) : chol_diag32_pair(a, lane, Dt, invd);
        const long long t1 = clock64();
        best = min(best, t1 - t0);
    }
    for (int j = 0; j < 32; ++j) L[lane * 32 + j] = Dt[j * 34 + lane];
    invd_out[lane] = invd[lane];
    if (lane == 0) { *cyc = best; *bad_out = bad; }
}
__global__ void panel_probe(const double* A, long long* cyc, double* out) {
    __shared__ __align__(16) double Dt[32 * 34];
    __shared__ double invd[32];
    const int lane = threadIdx.x;
    for (int j = 0; j < 32; ++j) { Dt[j * 34 + lane] = A[lane * 32 + j] * 0.01 + (j == lane); } invd[lane] = 1.0;
    __syncwarp();
    double a[32];
    for (int j = 0; j < 32; ++j) a[j] = A[lane * 32 + j];
    long long best = 1ll << 60;
    for (int rep = 0; rep < 4; ++rep) {
        const long long t0 = clock64();
        chol_panel_row(a, Dt, invd);
        const long long t1 = clock64();
        best = min(best, t1 - t0);
    }
    double s = 0; for (int j = 0; j < 32; ++j) s += a[j];
    out[lane] = s;
    if (lane == 0) *cyc = best;
}
int main() {
    const int n = 32;
    std::vector<double> B(n * n), A(n * n, 0.0), Lref(n * n, 0.0);
    unsigned long long st = 12345;
    auto rnd = [&]() { st = st * 6364136223846793005ull + 1442695040888963407ull; return (double)(st >> 11) / (double)(1ull << 53) - 0.5; };
    for (auto& v : B) v = rnd();
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) { double s = 0; for (int k = 0; k < n; ++k) s += B[i * n + k] * B[j * n + k]; A[i * n + j] = s * (1.0 + 1e3 * (i % 3 == 0) * (j % 3 == 0)) + (i == j) * 1e-3; }
    for (int j = 0; j < n; ++j) {
        double d = A[j * n + j]; for (int k = 0; k < j; ++k) d -= Lref[j * n + k] * Lref[j * n + k];
        Lref[j * n + j] = sqrt(d);
        for (int i = j + 1; i < n; ++i) { double s = A[i * n + j]; for (int k = 0; k < j; ++k) s -= Lref[i * n + k] * Lref[j * n + k]; Lref[i * n + j] = s / Lref[j * n + j]; }
    }
    double *dA, *dL, *dI; long long* dc; int* db;
    cudaMalloc(&dA, n * n * 8); cudaMalloc(&dL, n * n * 8); cudaMalloc(&dI, n * 8); cudaMalloc(&dc, 8); cudaMalloc(&db, 4);
    cudaMemcpy(dA, A.data(), n * n * 8, cudaMemcpyHostToDevice);
    for (int v = 0; v < 2; ++v) {
        if (v == 0) probe<0><<<1, 32>>>(dA, dL, dI, dc, db); else probe<1><<<1, 32>>>(dA, dL, dI, dc, db);
        std::vector<double> L(n * n), I(n); long long c; int bad;
        cudaMemcpy(L.data(), dL, n * n * 8, cudaMemcpyDeviceToHost); cudaMemcpy(I.data(), dI, n * 8, cudaMemcpyDeviceToHost);
        cudaMemcpy(&c, dc, 8, cudaMemcpyDeviceToHost); cudaMemcpy(&bad, db, 4, cudaMemcpyDeviceToHost);
        double err = 0, ierr = 0, scale = 0;
        for (int i = 0; i < n; ++i) for (int j = 0; j <= i; ++j) { err = fmax(err, fabs(L[i * n + j] - Lref[i * n + j])); scale = fmax(scale, fabs(Lref[i * n + j])); }
        for (int j = 0; j < n; ++j) ierr = fmax(ierr, fabs(I[j] * Lref[j * n + j] - 1.0));
        printf("%-28s %6lld cycles (%.0f per column)  max |L - Lref| / max|L| = %.2e   max |invd * Ljj - 1| = %.2e   bad=%d\n",
               v == 0 ? "chol_diag32 (1 column/step)" : "chol_diag32_pair (2/step)", c, c / 32.0, err / scale, ierr, bad);
    }
    double* dout; cudaMalloc(&dout, 256);
    panel_probe<<<1, 32>>>(dA, dc, dout);
    long long c; cudaMemcpy(&c, dc, 8, cudaMemcpyDeviceToHost);
    printf("chol_panel_row, one warp: %lld cycles\n", c);
    cudaError_t e = cudaDeviceSynchronize(); if (e) printf("error %s\n", cudaGetErrorString(e));
    return 0;
}
