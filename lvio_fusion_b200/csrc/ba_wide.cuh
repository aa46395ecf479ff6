// ba_wide.cuh -- reduced-system solve for envelopes that fit neither the one-CTA kernel's shared-memory panel nor a separator tree:
// a loop closure couples keyframes far apart along the trajectory, so some block columns of S reach over thousands of rows
// (Relocator / global BA after a loop: the reference hands that to SuiteSparse behind SPARSE_SCHUR, backend.cpp:207).
//
// Same right-looking blocked (32) algorithm and the same building blocks (lvb_chol.cuh) as ba_cholesky_kernel, but the panel stays
// in S (global memory / L2) and each phase of a 32-column step is its own grid over all SMs:
//   diag   (1 warp)       factor diagonal block kb in registers, write L and 1/diag back
//   panel  (rows / 128)   x L^T = a for every row below inside the envelope + the rhs row, in place
//   update (tiles / 4)    A22 -= P P^T, one warp per 32 x 32 tile, the two 32-row operand strips staged in shared memory
// then one small grid per block, last block first, for the backward substitution.  4 launches per 32 unknowns: a fallback for the
// rare wide solve (a few milliseconds at 3 000 unknowns), not a fast path.
#pragma once

__global__ void __launch_bounds__(32) ba_wide_diag_kernel(double* __restrict__ S, int n, long long srow, long long soff, int kb,
                                                          double* __restrict__ invd_g, LmState* st, int run_control_pre) {
    if (run_control_pre) { if (threadIdx.x == 0) lm_control_pre(*st); __syncwarp(); }
    if (st->done) return;
    __shared__ __align__(16) double Dt[32 * 34];
    __shared__ double invd[32];
    const CholGlobal G{S, srow, soff};
    const int lane = threadIdx.x, bs = min(32, n - kb);
    double a[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) a[j] = (lane < bs && j <= lane) ? *G.at(kb + lane, kb + j) : ((j == lane) ? 1.0 : 0.0);
    const int bad = chol_diag32_pair(a, lane, Dt, invd);
    if (bad && lane == 0) st->solve_fail = 1;
#pragma unroll
    for (int j = 0; j < 32; ++j) if (lane < bs && j <= lane) *G.at(kb + lane, kb + j) = Dt[j * 34 + lane];
    if (lane < bs) invd_g[kb + lane] = invd[lane];
}

// rows kb+bs .. rmax (S rows) and the rhs row (index m - 1)
__global__ void __launch_bounds__(128) ba_wide_panel_kernel(double* __restrict__ S, double* __restrict__ rhs, int n, long long srow, long long soff, int kb,
                                                            const double* __restrict__ invd_g, const LmState* st, const int* __restrict__ env_rmax) {
    if (st->done) return;
    __shared__ __align__(16) double Dt[32 * 34];
    __shared__ double invd[32];
    const CholGlobal G{S, srow, soff};
    const int bs = min(32, n - kb);
    for (int e = threadIdx.x; e < 32 * 32; e += blockDim.x) { const int k = e >> 5, j = e & 31; Dt[j * 34 + k] = (j <= k && k < bs) ? *G.at(kb + k, kb + j) : ((j == k) ? 1.0 : 0.0); }
    if (threadIdx.x < 32) invd[threadIdx.x] = threadIdx.x < bs ? invd_g[kb + threadIdx.x] : 1.0;
    __syncthreads();
    const int m = env_rmax[kb >> 5] - (kb + bs) + 1 + 1;
    const int rr = blockIdx.x * blockDim.x + threadIdx.x;
    if (rr >= m) return;
    double* src = (rr == m - 1) ? (rhs + kb) : G.at(kb + bs + rr, kb);
    double a[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) a[j] = (j < bs) ? src[j] : 0.0;
    chol_panel_row(a, Dt, invd);
#pragma unroll
    for (int j = 0; j < 32; ++j) if (j < bs) src[j] = a[j];
}

enum { WIDE_WARPS = 4 };
__global__ void __launch_bounds__(WIDE_WARPS * 32) ba_wide_update_kernel(double* __restrict__ S, double* __restrict__ rhs, int n, long long srow, long long soff, int kb,
                                                                         const LmState* st, const int* __restrict__ env_rmax) {
    if (st->done) return;
    extern __shared__ __align__(16) double wsm[];
    const CholGlobal G{S, srow, soff};
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int bs = min(32, n - kb);
    const int m = env_rmax[kb >> 5] - (kb + bs) + 1 + 1;
    const int ntile = (m + 31) >> 5;
    const int total = (m > 1) ? ntile * (ntile + 1) / 2 : 0;
    const int t = blockIdx.x * WIDE_WARPS + warp;
    if (t >= total) return;
    int ti, tj;
    chol_tile_index(t, ti, tj);
    // the two operand strips (rows of tile row ti, rows of tile row tj) of the panel: 2 x 32 rows x 32 columns, from S / rhs
    double* Pr = wsm + (size_t)warp * 2 * 32 * 34;
    double* Pc = Pr + 32 * 34;
    for (int r = 0; r < 32; ++r) {
        const int ir = ti * 32 + r, ic = tj * 32 + r;
        double vr = 0.0, vc = 0.0;
        if (lane < bs) {
            if (ir < m) vr = (ir == m - 1) ? rhs[kb + lane] : *G.at(kb + bs + ir, kb + lane);
            if (ic < m) vc = (ic == m - 1) ? rhs[kb + lane] : *G.at(kb + bs + ic, kb + lane);
        }
        Pr[r * 34 + lane] = vr; Pc[r * 34 + lane] = vc;
    }
    __syncwarp();
    const int ry = lane >> 2, cx = lane & 3;
    double acc[4][8] = {};
    const double2* rp[4]; const double2* cp[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) rp[i] = reinterpret_cast<const double2*>(Pr + (ry + 8 * i) * 34);
#pragma unroll
    for (int j = 0; j < 8; ++j) cp[j] = reinterpret_cast<const double2*>(Pc + (cx + 4 * j) * 34);
    chol_tile_product(acc, rp, cp);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int ip = ti * 32 + ry + 8 * i;
        if (ip >= m) continue;
        double* dst = (ip == m - 1) ? (rhs + kb + bs) : G.at(kb + bs + ip, kb + bs);
#pragma unroll
        for (int j = 0; j < 8; ++j) { const int jp = tj * 32 + cx + 4 * j; if (jp < m - 1 && jp <= ip) dst[jp] -= acc[i][j]; }
    }
}

// one block of the backward substitution  L^T x = y  (x overwrites rhs): GEMV over the rows below, then the 32-step substitution
__global__ void __launch_bounds__(256) ba_wide_backward_kernel(const double* __restrict__ S, double* __restrict__ rhs, int n, long long srow, long long soff, int kb,
                                                               const double* __restrict__ invd_g, const LmState* st, const int* __restrict__ env_rmax) {
    if (st->done) return;
    __shared__ double part[8 * 32];
    const CholGlobal G{S, srow, soff};
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int bs = min(32, n - kb), rend = env_rmax[kb >> 5];
    double acc = 0.0;
    if (lane < bs) for (int r = kb + bs + warp; r <= rend; r += nw) acc += *G.at(r, kb + lane) * rhs[r];
    part[warp * 32 + lane] = acc;
    __syncthreads();
    if (warp != 0) return;
    double col[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) col[i] = (i < bs && lane < bs && i >= lane) ? *G.at(kb + i, kb + lane) : 0.0;
    double t = lane < bs ? rhs[kb + lane] : 0.0;
    const double my_inv = lane < bs ? invd_g[kb + lane] : 1.0;
    for (int w = 0; w < nw; ++w) t -= part[w * 32 + lane];
    t = chol_back_block(t, my_inv, col, lane);
    if (lane < bs) rhs[kb + lane] = t;
}
