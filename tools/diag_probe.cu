// Cycles and accuracy of the 32 x 32 diagonal-block factorisation (one warp): the shipped chol_diag32_pair of lvb_chol.cuh against the
// one-column-per-step chol_diag32 below; and of the panel-row solve.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o diag_probe diag_probe.cu
#include <cstdio>
#include <cmath>
#include <vector>
#include <cuda_runtime.h>
#include "../lvio_fusion_b200/csrc/lvb_chol.cuh"

// 1 / sqrt(x) for a positive normal x without the library routine's special-case branch: a single warp is an in-order machine, and
// that branch (plus the call behind it) fences the scheduler, so nothing independent could be interleaved into the pivot chain's
// latency.  MUFU.RSQ64H seed (rsqrt.approx.ftz.f64, ~2^-20) + two coupled Newton (Goldschmidt) steps: 2^-40, then below 2^-52.
__device__ __forceinline__ double rsqrt_pos(double x) {
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    double g = x * y, h = 0.5 * y;
    double r = fma(-g, h, 0.5);
    g = fma(g, r, g); h = fma(h, r, h);
    r = fma(-g, h, 0.5);
    h = fma(h, r, h);
    return h + h;
}

// The one-column-per-step baseline of chol_diag32_pair (same contract).  One warp, lane = row of the block, a[r] = entry (lane, c0 + r)
// of the block (lower triangle valid).
// The 32 columns go in 4 groups of 8.  Inside a group a finished column is applied at once only to the group's own columns: its
// entries L[c0 + r][j] come from the owning lanes by shuffle (no shared-memory round trip, no warp barrier in the chain); the
// columns right of the group receive the group's rank-8 update in one sweep afterwards, operands broadcast from Dt as LDS.128.
// Per column the dependent chain is mul -> shuffle -> FMA -> shuffle -> rsqrt (~110 cycles); everything else is independent work
// the scheduler can place into its shadow because the loop body is branch-free.  Entries above the diagonal are don't-care and are
// updated without per-lane predicates (garbage stays garbage, nothing valid ever reads it), and nothing is stored to global memory
// here -- the caller copies the finished block (Dt, invd) to its place with all threads at the start of the next panel phase.
__device__ __forceinline__ int chol_diag32(double (&a)[32], const int lane, double* __restrict__ Dt, double* __restrict__ invd) {
    int bad = 0;
    double d0 = __shfl_sync(0xffffffffu, a[0], 0);
    if (!(d0 > 0.0)) { bad = 1; d0 = 1.0; }
    double inv = rsqrt_pos(d0);
#pragma unroll 1
    for (int c0 = 0; c0 < 32; c0 += 8) {
        const int rel = lane - c0;                    // register index of this lane's diagonal entry
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const int j = c0 + jj;
            a[jj] *= inv;                             // l_ij for lanes >= j (lane j: sqrt(d_jj)); don't-care above the diagonal
            Dt[j * 34 + lane] = a[jj];
            if (rel == jj) invd[j] = inv;
#pragma unroll
            for (int r = jj + 1; r < 8; ++r) {        // r = jj + 1 first: it completes the next pivot
                const double v = __shfl_sync(0xffffffffu, a[jj], c0 + r);
                a[r] -= a[jj] * v;
                if (r == jj + 1) {
                    double dn = __shfl_sync(0xffffffffu, a[jj + 1], j + 1);
                    if (!(dn > 0.0)) { bad = 1; dn = 1.0; }
                    inv = rsqrt_pos(dn);
                }
            }
        }
        if (c0 < 24) {
            __syncwarp();                             // the group's columns are in Dt
            // rank-8 update of the columns right of the group: a[r] -= sum_k L[lane][c0 + k] * L[c0 + r][c0 + k].  Register 8 (the next
            // pivot's column) first, so that its shuffle + rsqrt overlap the rest of the sweep.
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const double2 v = *reinterpret_cast<const double2*>(Dt + (c0 + k) * 34 + c0 + 8);
                a[8] -= a[k] * v.x; a[9] -= a[k] * v.y;
            }
            double dn = __shfl_sync(0xffffffffu, a[8], c0 + 8);
            if (!(dn > 0.0)) { bad = 1; dn = 1.0; }
            inv = rsqrt_pos(dn);
#pragma unroll
            for (int r = 10; r < 32; r += 2) {
                if (c0 + r < 32) {                    // warp-uniform
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const double2 v = *reinterpret_cast<const double2*>(Dt + (c0 + k) * 34 + c0 + r);
                        a[r] -= a[k] * v.x; a[r + 1] -= a[k] * v.y;
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < 24; ++r) a[r] = a[r + 8];
#pragma unroll
        for (int r = 24; r < 32; ++r) a[r] = 0.0;
    }
    __syncwarp();
    return bad;
}

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
