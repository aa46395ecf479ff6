// lvb_chol.cuh -- the pieces the blocked (32-column, right-looking) Cholesky kernels of the reduced camera system share
// (ba_cholesky_kernel, the separator tree's ba_front_* and the wide solver's ba_wide_* kernels, all in ba_solve.cu): the element
// accessors of S, the 32 x 32 diagonal-block factorisation by one warp, the per-row panel solve, the register micro-tile of the
// trailing update and the 32-step back-substitution of one block.
//
// Shared-memory operand: Dt[j * 34 + k] = L[k][j] (the block's factor, column-major with a 16-byte aligned stride), invd[j] = 1 / L[j][j].
#pragma once

// Element (i, j), i >= j, of S in global memory: lower triangle, row-major at i * srow + j + soff (dense: srow = n, soff = 0;
// banded of half bandwidth B: srow = soff = B).  T = const double for the kernels that only read S.
template <class T> struct CholGlobal {
    T* S; long long srow, soff;
    __device__ __forceinline__ T* at(int i, int j) const { return S + ((size_t)i * (size_t)srow + (size_t)j + (size_t)soff); }
};
template <class T> CholGlobal(T*, long long, long long) -> CholGlobal<T>;

// Element (i, j) of block column k = j / 32 in shared memory: rows kb .. rmax[k], row stride 34, block column k at col + boff[k]
// (chol_resident_columns, ba_plan.h).
struct CholResident {
    double* col; const int* boff;
    __device__ __forceinline__ double* at(int i, int j) const { const int k = j >> 5; return col + boff[k] + (i - (k << 5)) * 34 + (j & 31); }
};

// 1 / sqrt(x), seed + ONE third-order step  y (1 + e/2 + 3 e^2/8),  e = 1 - x y^2: the seed is good to ~2^-20 (tools/lat_probe.cu prints
// the measured worst case), the truncation term 5/16 e^3 is then below 2^-58, and the dependent chain is MUFU + 4 FP64 operations
// instead of MUFU + 6 for two Goldschmidt steps (tools/diag_probe.cu compares both).
__device__ __forceinline__ double rsqrt_pos3(double x) {
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    const double t = x * y;
    const double e = fma(-t, y, 1.0);
    const double p = fma(e, 0.375, 0.5), ye = y * e;
    return fma(ye, p, y);
}

// One warp, lane = row of the block, a[r] = entry (lane, r) of the block (lower triangle valid; rows past the block's end are
// identity rows, whose unit pivots leave the valid rows alone); returns 1 on a non-positive pivot.  Two columns per pivot step:
// the 2 x 2 pivot block [[p, q], [q, c]] is factored in closed form:
// L11 = sqrt(p), L21 = q / L11, L22 = sqrt(det / p) with det = p c - q^2, so the two reciprocal square roots 1 / sqrt(p) and 1 / sqrt(det)
// are independent and run side by side -- one MUFU + refinement latency per TWO columns -- and the broadcast / update round trip
// (shuffle -> FMA -> shuffle) is also paid once per pair.  The 32 columns go in 4 groups of 8: a finished pair is applied at once only
// to the group's own columns, by shuffle; the columns right of the group receive the group's rank-8 update in one sweep afterwards,
// operands broadcast from Dt as LDS.128.  Entries above the diagonal are don't-care and are updated without per-lane predicates, and
// nothing is stored to global memory here -- the caller copies the finished block (Dt, invd) to its place.
__device__ __forceinline__ int chol_diag32_pair(double (&a)[32], const int lane, double* __restrict__ Dt, double* __restrict__ invd) {
    int bad = 0;
#pragma unroll 1
    for (int c0 = 0; c0 < 32; c0 += 8) {
#pragma unroll
        for (int jj = 0; jj < 8; jj += 2) {
            const int j = c0 + jj;
            double p = __shfl_sync(0xffffffffu, a[jj], j);
            const double q = __shfl_sync(0xffffffffu, a[jj], j + 1);
            const double c = __shfl_sync(0xffffffffu, a[jj + 1], j + 1);
            double det = fma(p, c, -q * q);
            if (!(p > 0.0) || !(det > 0.0)) { bad = 1; p = 1.0; det = 1.0; }
            const double i1 = rsqrt_pos3(p), id = rsqrt_pos3(det);
            const double l11 = p * i1, l21 = q * i1;
            const double i2 = id * l11;
            const double l1 = a[jj] * i1;
            const double l2 = fma(-l1, l21, a[jj + 1]) * i2;
            a[jj] = l1; a[jj + 1] = l2;
            Dt[j * 34 + lane] = l1; Dt[(j + 1) * 34 + lane] = l2;
            if (lane == j) { invd[j] = i1; invd[j + 1] = i2; }
#pragma unroll
            for (int r = jj + 2; r < 8; ++r) {
                const double v1 = __shfl_sync(0xffffffffu, l1, c0 + r), v2 = __shfl_sync(0xffffffffu, l2, c0 + r);
                a[r] = fma(-l2, v2, fma(-l1, v1, a[r]));
            }
        }
        if (c0 < 24) {
            __syncwarp();                             // the group's columns are in Dt
            // rank-8 update of the columns right of the group; registers 8 and 9 (the next pivot pair) first
#pragma unroll
            for (int r = 8; r < 32; r += 2) {
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

// One panel row: x L^T = a for the 32 columns of the block (right-looking, no divisions), operands broadcast from Dt as LDS.128.
__device__ __forceinline__ void chol_panel_row(double (&a)[32], const double* __restrict__ Dt, const double* __restrict__ invd) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        a[j] *= invd[j];
        const double2* bp = reinterpret_cast<const double2*>(Dt + j * 34);
#pragma unroll
        for (int p = 0; p < 16; ++p) {
            if (2 * p + 1 > j) {
                const double2 v = bp[p];
                if (2 * p > j) a[2 * p] -= a[j] * v.x;
                a[2 * p + 1] -= a[j] * v.y;
            }
        }
    }
}

// Tile t of the lower triangle of a grid of 32 x 32 tiles, row by row: t -> (ti, tj), tj <= ti.
__device__ __forceinline__ void chol_tile_index(const int t, int& ti, int& tj) {
    ti = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
    while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
    while (ti * (ti + 1) / 2 > t) --ti;
    tj = t - ti * (ti + 1) / 2;
}

// One lane's RI x CJ register micro-tile of a tile of P P^T: acc[i][j] += (row rp[i]) . (row cp[j]) over 32 columns, rows read
// as double2, every entry accumulated in the same order (k = 0..15, .x then .y) whatever the micro-tile's shape.  The trailing
// updates use 4 x 8 and give lane the rows ry + 8 i and the columns cx + 4 j (ry = lane / 4, cx = lane % 4): consecutive lanes
// touch consecutive panel rows, so the LDS.128 operand loads are bank-conflict free and every loaded value feeds 4 or 8 DFMAs.
// The callers zero acc before they set up rp and cp: zeroing it here instead makes the compiler schedule ba_front_factor_kernel
// differently.
template <int RI, int CJ>
__device__ __forceinline__ void chol_tile_product(double (&acc)[RI][CJ], const double2* const (&rp)[RI], const double2* const (&cp)[CJ]) {
#pragma unroll 2
    for (int k = 0; k < 16; ++k) {
        double2 rv[RI], cv[CJ];
#pragma unroll
        for (int i = 0; i < RI; ++i) rv[i] = rp[i][k];
#pragma unroll
        for (int j = 0; j < CJ; ++j) cv[j] = cp[j][k];
#pragma unroll
        for (int i = 0; i < RI; ++i)
#pragma unroll
            for (int j = 0; j < CJ; ++j) { acc[i][j] += rv[i].x * cv[j].x; acc[i][j] += rv[i].y * cv[j].y; }
    }
}

// L^T x = t for one diagonal block, one warp: lane i holds t_i, 1 / L[i][i] and col[j] = L[j][i] (j >= i, zero elsewhere); returns x_i.
__device__ __forceinline__ double chol_back_block(double t, const double my_inv, const double (&col)[32], const int lane) {
#pragma unroll
    for (int j = 31; j >= 0; --j) {
        const double xj = __shfl_sync(0xffffffffu, t * my_inv, j);     // lane j's t is final here
        if (lane == j) t = xj;
        else if (lane < j) t -= col[j] * xj;
    }
    return t;
}
