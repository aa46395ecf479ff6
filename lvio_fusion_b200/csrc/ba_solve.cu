// ba_solve.cu -- the solve of the reduced camera system (ba_solve.h): the single-CTA kernel, the separator tree (ba_tree.cuh) and the
// wide solver (ba_wide.cuh), the one place that sets their launch attributes, and the solver's own debug entry points.
#include <stdlib.h>
#include <string.h>
#include "ba_solve.h"
#include "lvb_chol.cuh"

using namespace lvb;

namespace lvb {

__global__ void lm_control_pre_kernel(LmState* st) { lm_control_pre(*st); }

bool no_tree_switch() { static const bool on = getenv("LVB_NO_TREE") && getenv("LVB_NO_TREE")[0] == '1'; return on; }
bool tree_sep_band_switch() { static const bool on = getenv("LVB_TREE_SEP_BAND") && getenv("LVB_TREE_SEP_BAND")[0] == '1'; return on; }

}  // namespace lvb

namespace {

// accumulated SM clocks per Cholesky phase as thread 0 sees them: the diagonal-block factorisations (warp 0), the all-warp panel +
// head block, warp 0's wait for the rest of each step, backward, total, calls; then the resident kernel's load phase (warps 1..7,
// overlapping warp 0's first diagonal block) and its calls
__device__ long long g_chol_dbg[8];

// ------------------------------------------------------------------ single-CTA solve
// Right-looking blocked (32) factorisation of the lower triangle of S (n x n, row-major, in L2/HBM) with
// the right-hand side carried along as an extra row (so the forward substitution is free), then a
// blocked backward substitution.  Result: rhs <- S^-1 rhs.
//
// Schedule of one 32-column step k (look-ahead of depth one: only the factorisation of the next diagonal block is serial, and it
// has a warp to itself):
//   1. all warps : panel solve of every panel row, one row per thread: the 32 "head" rows (= the rows of diagonal block k + 1)
//                  first, then the others, the rhs row last;  the last warp also stores the INVERSE of block k of L to the
//                  block's place in S (for the backward pass)
//   2. warps 0..2: update of the lower triangle of diagonal block k + 1 by the head rows, a 16 x 16 block per warp, staged in the
//                  free (Dt, invd) buffer
//   3. warp 0    : block k + 1 minus that update, factored into the free buffer
//      warps 1..7: trailing update of everything but diagonal block k + 1
// so the pivot chain of block k + 1 overlaps the trailing update of step k instead of following it.  The last step has no next
// block and its trailing update is empty: it ends after the panel (the rhs row).
//
// The schedule runs on one of two storages of S.  kResident = false: S in global memory (in practice L2), each panel copied to the
// shared buffer P.  kResident = true (the windows, whenever plan_reduced_solver finds that the envelope fits): warps 1..7 load the
// envelope into shared memory once (chol_resident_columns, ba_plan.h) while warp 0 factors diagonal block 0 from global memory;
// the panel of step k is then block column k itself, the rhs a shared vector, and only x goes back to global memory.  Nothing reads
// the factor after the solve (S is rebuilt from Hpp on every pass), so the two storages compute the same x with the same arithmetic.
//
// run_pre: thread 0 runs the LM pre-check first.  The single-GPU window pass runs it in the last CTA of its Schur kernel instead;
// then nothing precedes warp 0's loads of diagonal block 0, and every warp only checks `done` (issued next to those loads).
template <bool kResident>
__global__ void __launch_bounds__(CHOL_T) ba_cholesky_kernel(double* __restrict__ S, double* __restrict__ rhs, int n, long long srow, long long soff,
                                                                  LmState* st, const int* __restrict__ env_rmax, int run_pre) {
    if (run_pre) {
        if (threadIdx.x == 0) lm_control_pre(*st);
        __syncthreads();
    }
    extern __shared__ __align__(16) double sm[];
    __shared__ int fail;
    __shared__ int boff[CHOL_RES_STEPS];
    __shared__ long long t_load;
    constexpr int nt = CHOL_T, nw = CHOL_T / 32;       // launched with CHOL_T threads; constants keep registers free
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // global memory: P is the rows x 34 panel (16 B aligned rows for broadcast double2 loads), later the backward partial sums.
    // resident: the partial sums (nw x 32), the rhs, then the block columns.
    double* const part = sm + CHOL_HDR;
    double* const R = kResident ? part + CHOL_T : rhs;
    const CholGlobal G{S, srow, soff};
    const auto W = [&] { if constexpr (kResident) return CholResident{R + ((n + 1) & ~1), boff}; else return G; }();   // chol_resident_rhs
    if (tid == 0) fail = 0;
    // 32-bit SM clocks (a call is far shorter than a wrap): 64-bit timers would be spilled out of the loop-carried registers
    unsigned t_fact = 0, t_panel = 0, t_wait = 0, t0 = clock(), tA;
    const unsigned t_begin = t0;
    // ---- diagonal block 0: warp 0, one row per lane in registers (lvb_chol.cuh), from global memory in both storages
    if (warp == 0) {
        const int b0 = min(32, n);
        double a[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) a[j] = (lane < b0 && j <= lane) ? *G.at(lane, j) : ((j == lane) ? 1.0 : 0.0);
        if (st->done) return;                       // uniform over the CTA, like the check of the other warps
        const int bad = chol_diag32_pair(a, lane, sm, sm + 32 * 34);
        if (bad && lane == 0) fail = 1;
        tA = clock(); t_fact += tA - t0; t0 = tA;
    } else if (st->done) {
        return;
    } else if constexpr (kResident) {
        // ---- load: the rhs and the envelope, all of S the solve touches (upper triangles of the diagonal blocks and columns past n
        // as zeros); batches of 8 independent loads per thread
        const int t1 = tid - 32, n1 = nt - 32;
        for (int i = t1; i < n; i += n1) R[i] = rhs[i];
        int o = 0;
        for (int kb = 0; kb < n; kb += 32) {
            const int cnt = (env_rmax[kb >> 5] - kb + 1) * 32;
            if (t1 == 0) boff[kb >> 5] = o;
            double* dst = W.col + o;
            for (int e0 = t1; e0 < cnt; e0 += 8 * n1) {
                double v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) { const int e = e0 + u * n1, r = e >> 5, c = e & 31; v[u] = (e < cnt && c <= r && kb + c < n) ? *G.at(kb + r, kb + c) : 0.0; }
#pragma unroll
                for (int u = 0; u < 8; ++u) { const int e = e0 + u * n1; if (e < cnt) dst[(e >> 5) * 34 + (e & 31)] = v[u]; }
            }
            o += cnt / 32 * 34;
        }
        if (t1 == 0) t_load = (unsigned)clock() - t0;
    }
    __syncthreads();
    tA = clock(); t_wait += tA - t0; t0 = tA;
    for (int kb = 0; kb < n; kb += 32) {
        const int bs = min(32, n - kb), kn = kb + 32;
        const int hb = max(0, min(32, n - kn));                    // rows of the next diagonal block ("head" rows of the panel)
        double* Dt = sm + ((kb >> 5) & 1) * CHOL_DT;               // block kb of L, column-major: Dt[j * 34 + k] = L[k][j]
        double* invd = Dt + 32 * 34;
        double* Dn = sm + (((kb >> 5) & 1) ^ 1) * CHOL_DT;
        // panel rows: the rows below the block inside the envelope of this block column (S is block-banded by construction) + the rhs row (last)
        const int m = env_rmax[kb >> 5] - (kb + bs) + 1 + 1;
        const int mh = min(hb, m - 1);                             // head rows inside the envelope
        // panel row rr < m - 1 at P + rr * 34, the rhs row at Prhs (resident: the panel is block column k below its diagonal block)
        double* const P = kResident ? W.at(kb + bs, kb) : part;
        double* const Prhs = kResident ? R + kb : P + (m - 1) * 34;
        // the INVERSE of block kb of L goes to the block's place in S: the backward pass then applies a diagonal block as 32 independent
        // FMAs per lane instead of a 32-step substitution chain.  Column c of L^-1 is the panel solve of the unit row e_c; one warp
        // (the last one, which has the fewest panel rows) does it while the others are in the panel.
        if (warp == nw - 1) {
            double e[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) e[j] = (j == lane) ? 1.0 : 0.0;
            chol_panel_row(e, Dt, invd);
#pragma unroll
            for (int j = 0; j < 32; ++j) if (j >= lane && j < bs) W.at(kb + j, kb)[lane] = e[j];
        }
        // ---- panel, one row per thread:  x L^T = a, right-looking, no divisions.  Rows 0 .. mh - 1 are the head rows.
        for (int rr = tid; rr < m; rr += nt) {
            const bool is_rhs = (rr == m - 1);
            double* src = is_rhs ? (R + kb) : W.at(kb + bs + rr, kb);
            double a[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) a[j] = (j < bs) ? src[j] : 0.0;
            chol_panel_row(a, Dt, invd);
#pragma unroll
            for (int j = 0; j < 32; ++j) { if (!kResident) P[rr * 34 + j] = a[j]; if (j < bs) src[j] = a[j]; }
        }
        __syncthreads();
        if (hb == 0) {                         // the last step: nothing right of the block (env_rmax <= n - 1, so m == 1)
            tA = clock(); t_panel += tA - t0; t0 = tA;
            break;
        }
        // ---- head block: diagonal block kn -= (head rows)(head rows)^T on its lower triangle, staged in the free diagonal-block
        // buffer for warp 0's row-per-lane layout.  Warps 0..2 each form one of the 16 x 16 blocks (0, 0), (16, 0), (16, 16), lane
        // (ry, cx) a 2 x 4 micro-tile (chol_tile_product: each entry summed as the trailing update sums it).  The block (0, 16) lies
        // above the diagonal, which chol_diag32_pair never lets into the lower triangle, so it is not formed: this phase is bound by
        // the product's shared-memory loads, not by its DFMAs.  Head rows outside the envelope are structurally zero and have no
        // panel row.
        if (mh > 0 && warp < 3) {
            const int R0 = warp ? 16 : 0, C0 = warp == 2 ? 16 : 0, ry = lane >> 2, cx = lane & 3;
            double acc[2][4] = {};
            const double2* rp[2]; const double2* cp[4];
#pragma unroll
            for (int i = 0; i < 2; ++i) rp[i] = reinterpret_cast<const double2*>(P + (size_t)min(R0 + ry + 8 * i, mh - 1) * 34);
#pragma unroll
            for (int j = 0; j < 4; ++j) cp[j] = reinterpret_cast<const double2*>(P + (size_t)min(C0 + cx + 4 * j, mh - 1) * 34);
            chol_tile_product(acc, rp, cp);
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int r = R0 + ry + 8 * i, c = C0 + cx + 4 * j;
                    Dn[r * 34 + c] = (r < mh && c < mh) ? acc[i][j] : 0.0;
                }
        }
        __syncthreads();
        tA = clock(); t_panel += tA - t0; t0 = tA;
        if (warp == 0) {
            // ---- factorisation of block kn into the free buffer (loading the block earlier, to overlap the head block, spills)
            double a[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) a[j] = (lane < hb && j <= lane) ? W.at(kn + lane, kn)[j] : ((j == lane) ? 1.0 : 0.0);
            if (mh > 0) {
#pragma unroll
                for (int j = 0; j < 32; ++j) a[j] -= Dn[lane * 34 + j];
                __syncwarp();
            }
            const int bad = chol_diag32_pair(a, lane, Dn, Dn + 32 * 34);
            if (bad && lane == 0) fail = 1;
            tA = clock(); t_fact += tA - t0; t0 = tA;
        } else {
            // ---- trailing update A22 -= P P^T on the lower triangle but diagonal block kn: one warp per 32x32 tile, each lane a 4x8
            // register micro-tile (chol_tile_product)
            const int wid = warp - 1, nwk = nw - 1;
            const int ntile = (m + 31) >> 5;
            const int total = (m > 1) ? ntile * (ntile + 1) / 2 : 0;
            for (int t = wid; t < total; t += nwk) {
                if (t == 0 && mh >= min(32, m)) continue;
                int ti, tj;
                chol_tile_index(t, ti, tj);
                const int row_lo = (t == 0) ? mh : 0;
                const int ry = lane >> 2, cx = lane & 3;
                const int r0 = ti * 32 + ry, c0 = tj * 32 + cx;
                double acc[4][8] = {};
                // rows / columns beyond the panel read row 0 (valid memory) and are masked at the store
                const double2* rp[4]; const double2* cp[8];
    #pragma unroll
                for (int i = 0; i < 4; ++i) { const int ri = min(r0 + 8 * i, m - 1); rp[i] = reinterpret_cast<const double2*>(ri == m - 1 ? Prhs : P + (size_t)ri * 34); }
    #pragma unroll
                for (int j = 0; j < 8; ++j) { const int ci = min(c0 + 4 * j, m - 1); cp[j] = reinterpret_cast<const double2*>(ci == m - 1 ? Prhs : P + (size_t)ci * 34); }
                chol_tile_product(acc, rp, cp);
                // read-modify-write of the tile: all loads first (one round trip), then the stores.  src / dst point at the tile's
                // first column (tj * 32 past the panel): the tile lies in one block column of the resident storage.
                double cur[4][8];
                const int tc = kb + bs + tj * 32;
    #pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int ip = min(r0 + 8 * i, m - 1);
                    const double* src = (ip == m - 1) ? (R + tc) : W.at(kb + bs + ip, tc);
    #pragma unroll
                    for (int j = 0; j < 8; ++j) { const int jp = c0 + 4 * j; cur[i][j] = (r0 + 8 * i < m && r0 + 8 * i >= row_lo && jp < m - 1 && jp <= ip) ? src[cx + 4 * j] : 0.0; }
                }
    #pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int ip = r0 + 8 * i;
                    if (ip >= m || ip < row_lo) continue;
                    double* dst = (ip == m - 1) ? (R + tc) : W.at(kb + bs + ip, tc);
    #pragma unroll
                    for (int j = 0; j < 8; ++j) { const int jp = c0 + 4 * j; if (jp < m - 1 && jp <= ip) dst[cx + 4 * j] = cur[i][j] - acc[i][j]; }
                }
            }
        }
        __syncthreads();
        tA = clock(); t_wait += tA - t0; t0 = tA;
    }
    // ---- backward substitution  L^T x = y  (y is in rhs), left-looking per 32-column block:
    //   x_k = D_k^-T (y_k - sum_{r below} L[r][k-block]^T x_r),  D_k^-1 stored in place of D_k by the factorisation
    // the sum is a GEMV over the envelope rows spread over all warps (independent coalesced loads, one L2 round trip per
    // batch), then warp 0 applies the inverse diagonal block: 32 independent FMAs per lane, no substitution chain.  x overwrites rhs.
    const int last = ((n - 1) / 32) * 32;
    for (int kb = last; kb >= 0; kb -= 32) {
        const int bs = min(32, n - kb);
        const int rend = env_rmax[kb >> 5];
        double col[32];                               // warp 0: column `lane` of the inverse diagonal block, col[i] = Linv[kb+i][kb+lane], i >= lane
        double t = 0.0;
        if (warp == 0) {
#pragma unroll
            for (int i = 0; i < 32; ++i) col[i] = (i < bs && lane < bs && i >= lane) ? W.at(kb + i, kb)[lane] : 0.0;
            if (lane < bs) t = R[kb + lane];
        }
        double acc = 0.0;
        if (lane < bs) {
            for (int r0 = kb + bs + warp; r0 <= rend; r0 += 16 * nw) {
                double lv[16], xv[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) { const int r = r0 + u * nw; const bool ok = r <= rend; lv[u] = ok ? W.at(r, kb)[lane] : 0.0; xv[u] = ok ? R[r] : 0.0; }
#pragma unroll
                for (int u = 0; u < 16; ++u) acc += lv[u] * xv[u];
            }
        }
        part[warp * 32 + lane] = acc;
        __syncthreads();
        if (warp == 0) {
            for (int w = 0; w < nw; ++w) t -= part[w * 32 + lane];
            // x = D^-T t with the stored inverse: x_lane = sum_{j >= lane} Linv[j][lane] t_j
            double y0 = 0.0, y1 = 0.0, y2 = 0.0, y3 = 0.0;
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                y0 = fma(col[j], __shfl_sync(0xffffffffu, t, j), y0);
                y1 = fma(col[j + 1], __shfl_sync(0xffffffffu, t, j + 1), y1);
                y2 = fma(col[j + 2], __shfl_sync(0xffffffffu, t, j + 2), y2);
                y3 = fma(col[j + 3], __shfl_sync(0xffffffffu, t, j + 3), y3);
            }
            t = (y0 + y1) + (y2 + y3);
            if (lane < bs) R[kb + lane] = t;
        }
        __syncthreads();
    }
    if (kResident) for (int i = tid; i < n; i += nt) rhs[i] = R[i];
    if (tid == 0 && fail) st->solve_fail = 1;
    if (tid == 0) {
        tA = clock(); g_chol_dbg[0] += t_fact; g_chol_dbg[1] += t_panel; g_chol_dbg[2] += t_wait; g_chol_dbg[3] += tA - t0; g_chol_dbg[4] += tA - t_begin; g_chol_dbg[5] += 1;
        if (kResident) { g_chol_dbg[6] += t_load; g_chol_dbg[7] += 1; }
    }
}

#include "ba_tree.cuh"
#include "ba_wide.cuh"

}  // namespace

static int set_solver_attributes() {
    static bool done = false;
    if (done) return LVB_OK;
    LVB_CUDA(cudaFuncSetAttribute(ba_cholesky_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_CTA_SMEM));
    LVB_CUDA(cudaFuncSetAttribute(ba_cholesky_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_CTA_SMEM));
    LVB_CUDA(cudaFuncSetAttribute(ba_front_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_CTA_SMEM));
    LVB_CUDA(cudaFuncSetAttribute(ba_front_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    LVB_CUDA(cudaFuncSetAttribute(ba_wide_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WIDE_WARPS * 2 * 32 * 34 * 8));
    done = true;
    return LVB_OK;
}

namespace lvb {

int ReducedSolver::upload(lvb_ctx* ctx, const SolverPlan& sp, const std::vector<int>& env_rmax, int n) {
    LVB_TRY(set_solver_attributes());
    cudaStream_t s = ctx->stream;
    plan = sp;
    rmax = env_rmax;
    LVB_TRY(rmax_d.upload(rmax.data(), rmax.size(), s));
    LVB_TRY(invd.ensure((size_t)n + 32));
    if (plan.tree_levels > 0) { LVB_TRY(fronts.upload(plan.fronts.data(), plan.fronts.size(), s)); LVB_TRY(pool.ensure(plan.pool_doubles)); }
    return LVB_OK;
}

int ReducedSolver::launch(lvb_ctx* ctx, double* S, double* rhs, int n, long long srow, long long soff, int band, LmState* st, bool pre_done) const {
    const SolverPlan& sp = plan;
    const int run_pre = pre_done ? 0 : 1;
    if (sp.tree_levels > 0) {
        // multifrontal tree: leaves (all SMs) -> ... -> root, then the back-substitution root -> leaves; 2 (levels + 1) launches
        if (run_pre) LAUNCH(ctx, lm_control_pre_kernel, 1, 1, 0, st);
        const int n_fronts = sp.level_first[sp.tree_levels - 1] + sp.level_count[sp.tree_levels - 1];
        ba_front_init_kernel<<<dim3(16, n_fronts), 256, 0, ctx->stream>>>(fronts.p, n_fronts, S, rhs, pool.p, srow, soff, band, st);
        ctx->launches++; timing_mark(ctx->stream, "ba_front_init_kernel");
        for (int l = 0; l < sp.tree_levels; ++l)
            LAUNCH(ctx, ba_front_factor_kernel, sp.level_count[l], CHOL_T, sp.tree_factor_smem, fronts.p, sp.level_first[l], S, rhs, pool.p, srow, soff, band, invd.p, st);
        for (int l = sp.tree_levels - 1; l >= 0; --l)
            LAUNCH(ctx, ba_front_backward_kernel, sp.level_count[l], CHOL_T, sp.tree_back_smem, fronts.p, sp.level_first[l], S, rhs, pool.p, srow, soff, band, invd.p, st);
    } else if (sp.wide) {
        // one grid per phase of every 32-column step, then one per block of the backward substitution (ba_wide.cuh)
        for (int kb = 0; kb < n; kb += 32) {
            const int bs = std::min(32, n - kb);
            const int m = rmax[kb >> 5] - (kb + bs) + 2;
            const int ntile = (m + 31) / 32, total = m > 1 ? ntile * (ntile + 1) / 2 : 0;
            LAUNCH(ctx, ba_wide_diag_kernel, 1, 32, 0, S, n, srow, soff, kb, invd.p, st, kb == 0 ? run_pre : 0);
            LAUNCH(ctx, ba_wide_panel_kernel, (m + 127) / 128, 128, 0, S, rhs, n, srow, soff, kb, invd.p, st, rmax_d.p);
            LAUNCH(ctx, ba_wide_update_kernel, (total + WIDE_WARPS - 1) / WIDE_WARPS, WIDE_WARPS * 32, (size_t)WIDE_WARPS * 2 * 32 * 34 * 8, S, rhs, n, srow, soff, kb, st, rmax_d.p);
        }
        for (int kb = ((n - 1) / 32) * 32; kb >= 0; kb -= 32)
            LAUNCH(ctx, ba_wide_backward_kernel, 1, 256, 0, S, rhs, n, srow, soff, kb, invd.p, st, rmax_d.p);
    } else if (sp.resident) {
        LAUNCH_AS(ctx, "ba_cholesky_kernel", ba_cholesky_kernel<true>, 1, CHOL_T, sp.resident_smem, S, rhs, n, srow, soff, st, rmax_d.p, run_pre);
    } else {
        LAUNCH_AS(ctx, "ba_cholesky_kernel", ba_cholesky_kernel<false>, 1, CHOL_T, sp.chol_smem, S, rhs, n, srow, soff, st, rmax_d.p, run_pre);
    }
    return LVB_OK;
}

}  // namespace lvb

extern "C" {

LVB_API int lvb_debug_cholesky_clocks(long long out[8], int reset) {
    LVB_CUDA(cudaMemcpyFromSymbol(out, g_chol_dbg, 8 * sizeof(long long)));
    if (reset) { long long z[8] = {0}; LVB_CUDA(cudaMemcpyToSymbol(g_chol_dbg, z, sizeof(z))); }
    return LVB_OK;
}

// Direct access to the reduced-system solver for its own parity test (tests/test_gpu_band_solver.py): solves S x = b for a
// symmetric positive definite band matrix given as n rows of (band + 1) entries (row i: columns i - band .. i; the true half
// bandwidth must be <= band - 31, the block-granular slack the envelope kernel needs).  use_tree = 0 forces the single-CTA kernel.
LVB_API int lvb_debug_band_solve(lvb_ctx* ctx, int n, int band, const double* S_band, const double* b, double* x, int use_tree, int* levels_out) {
    if (!ctx || n <= 0 || band < 31 || !S_band || !b || !x) { set_error("bad arguments"); return LVB_ERR_INVALID; }
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    cudaStream_t s = ctx->stream;
    const size_t nS = (size_t)n * (band + 1);
    DevBuf<double> Sb;                  // S in banded storage (srow = soff = band), then the rhs
    DevBuf<LmState> st;
    LVB_TRY(Sb.ensure(nS + n));
    LVB_CUDA(cudaMemcpyAsync(Sb.p, S_band, nS * sizeof(double), cudaMemcpyHostToDevice, s));
    LVB_CUDA(cudaMemcpyAsync(Sb.p + nS, b, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, s));
    LVB_TRY(st.ensure(1));
    lvb_solve_options opt; lvb_default_options(&opt);
    LmState h; lm_init(h, opt);
    const double one = 1.0; memcpy(&h.grad_max_bits, &one, sizeof(double));        // not converged: the pre-check lets the solve run
    LVB_CUDA(cudaMemcpyAsync(st.p, &h, sizeof(h), cudaMemcpyHostToDevice, s));
    std::vector<int> rmax, cmin;
    uniform_band_envelope(n, band, rmax, cmin);
    ReducedSolver solver;
    LVB_TRY(solver.upload(ctx, plan_reduced_solver(n, band, tree_sep_band_switch() ? band : band - 31, rmax, ctx->sm_count, !use_tree), rmax, n));
    if (levels_out) *levels_out = solver.plan.tree_levels;
    LVB_TRY(solver.launch(ctx, Sb.p, Sb.p + nS, n, band, band, band, st.p));
    LVB_TRY(check_launch("band solve"));
    LVB_CUDA(cudaMemcpyAsync(x, Sb.p + nS, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, s));
    LVB_CUDA(cudaMemcpyAsync(&h, st.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    LVB_TRY(lvb::host_sync(ctx, s));
    if (h.solve_fail) { set_error("band solve: non-positive pivot"); return LVB_ERR_NUMERIC; }
    return LVB_OK;
}

}  // extern "C"
