// ba_tree.cuh -- multifrontal (nested-dissection) Cholesky of the banded reduced camera system: many SMs instead of one.
//
// What it replaces: SuiteSparse's supernodal Cholesky behind SPARSE_SCHUR (/root/reference/src/lvio_fusion/src/backend.cpp:207).
// The reduced system of a trajectory is block-banded (keyframe-interleaved ordering, half bandwidth B): a single CTA walking the
// band is a chain of dimc dependent pivots (42 ms at 75 000 unknowns).  Any w >= B consecutive unknowns separate the chain, so
// the unknowns are split by a complete binary tree of separators:
//
//      [ leaf 0 | s | leaf 1 | S | leaf 2 | s | leaf 3 ]          s: level-1 separators, S: root
//
// Every tree node owns a *front*: its own unknowns (leaf: a banded segment, internal node: a dense separator block) followed by
// the <= 2 ancestor separators that bound its subtree (the border) and the right-hand side as one more row.  A front is
// eliminated by ONE CTA with a partial Cholesky over its own columns -- the blocked right-looking kernel of ba_cholesky_kernel
// with the border rows riding along in every panel -- which leaves  L_own,  W = L_own^-1 A_own,border  (in the border rows),
// y = L_own^-1 b_own  and the update  -W^T W  of the border x border block.  All fronts of a level run concurrently (grid = number
// of fronts), a child adds its update into its parent's front when it is done (extend-add); log2(P) + 1 launches factor the system and
// the same number of launches, root first, back-substitute.  Own x own blocks are factored in place in the banded storage of S
// (a separator of width w = B fits inside the band), border rows live in a pool.
#pragma once
#include "ba_plan.h"        // struct Front, CHOL_T; the tree itself is built there (build_front_tree)

// Panel row p of a front's 32-column step: the own rows r1 + p inside the band (p < nr1), then the active border rows, then the rhs
// row.  base(p)[c] is the row's entry in own column c (c >= n: border column c - n); col(p) is the own column of its diagonal entry.
struct FrontRows {
    CholGlobal<double> G; double* Bd; int o0, r1, nr1, nbp, nb, n, ld;
    __device__ __forceinline__ int border(int p) const { return (p - nr1 < nbp) ? p - nr1 : nb; }
    __device__ __forceinline__ double* base(int p) const { return (p < nr1) ? G.at(o0 + r1 + p, o0) : Bd + (size_t)border(p) * ld; }
    __device__ __forceinline__ int col(int p) const { return (p < nr1) ? r1 + p : n + border(p); }
};

// Every front's border array before the factorisation starts.  Leaves: zeros, the couplings with the bounding separators
// gathered out of the band (the left one transposed: in the front the separator comes after the segment) and the right-hand
// side.  Internal fronts: zeros and their own part of the right-hand side -- their children add the rest (extend-add at the end of
// ba_front_factor_kernel).  Grid-wide, HBM-bound.
__global__ void __launch_bounds__(256) ba_front_init_kernel(const Front* __restrict__ fr, int n_fronts, const double* __restrict__ S, const double* __restrict__ rhs,
                                                             double* __restrict__ pool, long long srow, long long soff, int band, const LmState* st) {
    if (st->done) return;
    const CholGlobal G{S, srow, soff};
    for (int f = blockIdx.y; f < n_fronts; f += gridDim.y) {
        const Front F = fr[f];
        double* Bd = pool + F.bd;
        const size_t total = (size_t)(F.nb + 1) * F.ld;
        const bool leaf = F.child0 < 0;
        for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
            const int q = (int)(e / F.ld), c = (int)(e - (size_t)q * F.ld);
            double v = 0.0;
            if (c < F.m) {
                if (q == F.nb) v = rhs[F.o0 + c];
                else if (leaf) {
                    if (q < F.wL) { const int gi = F.o0 + c, gj = F.bL0 + q; if (gi - gj <= band) v = *G.at(gi, gj); }
                    else { const int gi = F.bR0 + (q - F.wL), gj = F.o0 + c; if (gi - gj <= band) v = *G.at(gi, gj); }
                }
            }
            Bd[e] = v;
        }
    }
}

// One CTA per front of a level.  Shared memory (front_factor_smem, ba_plan.h): Dt (32 x 34), invd (32), P (panel rows x 34).
__global__ void __launch_bounds__(CHOL_T) ba_front_factor_kernel(const Front* __restrict__ fr, int first, double* __restrict__ S, const double* __restrict__ rhs,
                                                                  double* __restrict__ pool, long long srow, long long soff, int band,
                                                                  double* __restrict__ invd_g, LmState* st) {
    if (st->done) return;
    extern __shared__ __align__(16) double sm[];
    double* Dt = sm;                   // 32 x 34   diagonal block of L, column-major: Dt[j * 34 + k] = L[k][j] (lvb_chol.cuh)
    double* invd = sm + 32 * 34;       // 32        reciprocals of diag(L) of the current block
    double* P = sm + FRONT_PANEL;      // rows x 34 panel (16 B aligned rows for broadcast double2 loads)
    __shared__ int fail;
    const CholGlobal G{S, srow, soff};
    const Front F = fr[first + blockIdx.x];
    const int n = F.m, nb = F.nb, ld = F.ld;
    double* Bd = pool + F.bd;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    if (tid == 0) fail = 0;
    __syncthreads();
    // Software-pipelined over the 32-column block steps with look-ahead (see ba_cholesky_kernel): while warps 1.. finish the
    // trailing update of step kb, warp 0 updates the next diagonal block first (tile 0) and factors it.
    for (int kb = -32; kb < n; kb += 32) {
        const int bs = min(32, n - kb);
        if (kb >= 0) {
            // ---- panel rows: own rows below the block inside the band | active border rows | rhs row
            const int r1 = kb + bs;
            const int nr1 = max(0, min(n - 1, kb + band) - r1 + 1);
            const int nbp = F.wL + ((r1 > F.actR) ? F.wR : 0);
            const int m = nr1 + nbp + 1;
            const FrontRows rows{G, Bd, F.o0, r1, nr1, nbp, nb, n, ld};
            // the diagonal block factored during the previous step's look-ahead goes to its place in S (all threads, row by row)
            for (int e = tid; e < 32 * 32; e += nt) { const int k = e >> 5, j = e & 31; if (j <= k && k < bs) *G.at(F.o0 + kb + k, F.o0 + kb + j) = Dt[j * 34 + k]; }
            if (tid < bs) invd_g[F.o0 + kb + tid] = invd[tid];
            for (int rr = tid; rr < m; rr += nt) {
                double* src = rows.base(rr) + kb;
                double a[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) a[j] = (j < bs) ? src[j] : 0.0;
                chol_panel_row(a, Dt, invd);
#pragma unroll
                for (int j = 0; j < 32; ++j) { P[rr * 34 + j] = a[j]; if (j < bs) src[j] = a[j]; }
            }
            __syncthreads();
            // ---- trailing update A22 -= P P^T on the lower triangle: one warp per 32 x 32 tile, 4 x 8 register micro-tiles
            const int ntile = (m + 31) >> 5;
            const int total = ntile * (ntile + 1) / 2;
            for (int t = (warp == 0) ? 0 : warp; t < total; t += (warp == 0) ? total : (nw - 1)) {
                int ti, tj;
                chol_tile_index(t, ti, tj);
                const int ry = lane >> 2, cx = lane & 3;
                const int r0 = ti * 32 + ry, c0 = tj * 32 + cx;
                double acc[4][8] = {};
                const double2* rp[4]; const double2* cp[8];
#pragma unroll
                for (int i = 0; i < 4; ++i) rp[i] = reinterpret_cast<const double2*>(P + (size_t)min(r0 + 8 * i, m - 1) * 34);
#pragma unroll
                for (int j = 0; j < 8; ++j) cp[j] = reinterpret_cast<const double2*>(P + (size_t)min(c0 + 4 * j, m - 1) * 34);
                chol_tile_product(acc, rp, cp);
                int colx[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) { const int jp = min(c0 + 4 * j, m - 1); colx[j] = rows.col(jp); }
                double cur[4][8];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int ip = min(r0 + 8 * i, m - 1);
                    const double* src = rows.base(ip);
#pragma unroll
                    for (int j = 0; j < 8; ++j) { const int jp = c0 + 4 * j; cur[i][j] = (r0 + 8 * i < m && jp < m - 1 && jp <= ip) ? src[colx[j]] : 0.0; }
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int ip = r0 + 8 * i;
                    if (ip >= m) continue;
                    double* dst = rows.base(ip);
#pragma unroll
                    for (int j = 0; j < 8; ++j) { const int jp = c0 + 4 * j; if (jp < m - 1 && jp <= ip) dst[colx[j]] = cur[i][j] - acc[i][j]; }
                }
            }
        }
        const int kn = kb + 32, bn = min(32, n - kn);
        // ---- diagonal block kn: warp 0 holds one row per lane in registers and factors it with shuffles (4 groups of 8 columns)
        if (kn < n) {
            __syncwarp();
            if (warp == 0) {
                double a[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) a[j] = (lane < bn && j <= lane) ? *G.at(F.o0 + kn + lane, F.o0 + kn + j) : ((j == lane) ? 1.0 : 0.0);
                const int bad = chol_diag32_pair(a, lane, Dt, invd);
                if (bad && lane == 0) fail = 1;
            }
        }
        __syncthreads();
    }
    if (tid == 0 && fail) st->solve_fail = 1;
    // ---- extend-add: this front's update matrix (border x border block + the rhs row's border part) goes into its parent's front.
    // Done here, by the child, with fire-and-forget reductions: as a prologue of the parent it was a chain of dependent
    // load -> read-modify-write round trips on a single CTA (150 of the 180 us of every internal level).  The sibling adds into the
    // same own x own block and rhs entries of the parent concurrently, hence the atomics; the parent's array was initialised by
    // ba_front_init_kernel, and the parent level's launch comes after this one in stream order.
    if (F.parent >= 0) {
        const Front Pf = fr[F.parent];
        double* Bp = pool + Pf.bd;
        const int pn = Pf.m, pld = Pf.ld, pnb = Pf.nb;
        // my border id t -> parent front: left child: [0, wL) = parent's left border, the rest = parent's own unknowns;
        //                                right child: [0, wL) = parent's own unknowns, the rest = parent's right border
        const int total = (nb + 1) * nb;
        for (int e0 = tid; e0 < total; e0 += 4 * nt) {
            double u[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) { const int e = e0 + k * nt; const int r = e / nb, c = e - r * nb; u[k] = (e < total && c <= r) ? Bd[(size_t)r * ld + n + c] : 0.0; }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (u[k] == 0.0) continue;
                const int e = e0 + k * nt; const int r = e / nb, c = e - r * nb;
                bool c_own; int c_idx;
                if (F.side == 0) { c_own = c >= F.wL; c_idx = c_own ? c - F.wL : c; } else { c_own = c < F.wL; c_idx = c_own ? c : Pf.wL + (c - F.wL); }
                if (r == nb) { atomicAdd(&Bp[(size_t)pnb * pld + (c_own ? c_idx : pn + c_idx)], u[k]); continue; }
                bool r_own; int r_idx;
                if (F.side == 0) { r_own = r >= F.wL; r_idx = r_own ? r - F.wL : r; } else { r_own = r < F.wL; r_idx = r_own ? r : Pf.wL + (r - F.wL); }
                if (r_own && c_own) atomicAdd(G.at(Pf.o0 + r_idx, Pf.o0 + c_idx), u[k]);          // r_idx >= c_idx: the maps are monotone
                else if (r_own) atomicAdd(&Bp[(size_t)c_idx * pld + r_idx], u[k]);                 // A(own, left border): stored transposed
                else if (c_own) atomicAdd(&Bp[(size_t)r_idx * pld + c_idx], u[k]);                 // A(right border, own)
                else atomicAdd(&Bp[(size_t)r_idx * pld + pn + c_idx], u[k]);                       // border x border
            }
        }
    }
}

// Back-substitution of one level (root level first): x_own = L_own^-T (y - W x_border), x in place in `x` (the rhs vector).
// Shared memory: xb (nb) + part (warps x 32).
__global__ void __launch_bounds__(CHOL_T) ba_front_backward_kernel(const Front* __restrict__ fr, int first, const double* __restrict__ S, double* __restrict__ x,
                                                                    const double* __restrict__ pool, long long srow, long long soff, int band,
                                                                    const double* __restrict__ invd_g, const LmState* st) {
    if (st->done) return;
    extern __shared__ __align__(16) double sm[];
    const CholGlobal G{S, srow, soff};
    const Front F = fr[first + blockIdx.x];
    const int n = F.m, nb = F.nb, ld = F.ld;
    const double* Bd = pool + F.bd;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    double* xb = sm;
    double* part = sm + ((nb + 1) & ~1);
    for (int q = tid; q < nb; q += nt) xb[q] = x[q < F.wL ? F.bL0 + q : F.bR0 + (q - F.wL)];
    __syncthreads();
    const int last = ((n - 1) / 32) * 32;
    for (int kb = last; kb >= 0; kb -= 32) {
        const int bs = min(32, n - kb);
        const int rend = min(n - 1, kb + band);
        const int nbq = (kb + bs > F.actR) ? nb : F.wL;          // right-border rows are zero left of actR
        double col[32];
        double t = 0.0, my_inv = 1.0;
        if (warp == 0) {
#pragma unroll
            for (int i = 0; i < 32; ++i) col[i] = (i < bs && lane < bs && i >= lane) ? *G.at(F.o0 + kb + i, F.o0 + kb + lane) : 0.0;
            if (lane < bs) { t = Bd[(size_t)nb * ld + kb + lane]; my_inv = invd_g[F.o0 + kb + lane]; }
        }
        double acc = 0.0;
        if (lane < bs) {
            for (int r0 = kb + bs + warp; r0 <= rend; r0 += 16 * nw) {
                double lv[16], xv[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) { const int r = r0 + u * nw; const bool ok = r <= rend; lv[u] = ok ? *G.at(F.o0 + r, F.o0 + kb + lane) : 0.0; xv[u] = ok ? x[F.o0 + r] : 0.0; }
#pragma unroll
                for (int u = 0; u < 16; ++u) acc += lv[u] * xv[u];
            }
            for (int q0 = warp; q0 < nbq; q0 += 16 * nw) {
                double lv[16], xv[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) { const int q = q0 + u * nw; const bool ok = q < nbq; lv[u] = ok ? Bd[(size_t)q * ld + kb + lane] : 0.0; xv[u] = ok ? xb[q] : 0.0; }
#pragma unroll
                for (int u = 0; u < 16; ++u) acc += lv[u] * xv[u];
            }
        }
        part[warp * 32 + lane] = acc;
        __syncthreads();
        if (warp == 0) {
            for (int w = 0; w < nw; ++w) t -= part[w * 32 + lane];
            t = chol_back_block(t, my_inv, col, lane);
            if (lane < bs) x[F.o0 + kb + lane] = t;
        }
        __syncthreads();
    }
}
