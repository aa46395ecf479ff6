// ba_solve.h -- the solve of the reduced camera system, rhs <- S^-1 rhs, by the solver plan_reduced_solver (ba_plan.h) picked: the
// single-CTA kernel (S resident in shared memory or in global memory), the separator tree (ba_tree.cuh) or the wide solver
// (ba_wide.cuh).  Kernels and launches live in ba_solve.cu.
#pragma once
#include "ba_plan.h"
#include "lvb_internal.cuh"

namespace lvb {

// The solver's device state for one system: built from the plan and the envelope by upload(), then launched once per LM pass.
struct ReducedSolver {
    SolverPlan plan;                    // which solver, its shared memory and the tree's levels
    std::vector<int> rmax;              // envelope: last row of S per 32-column step (the wide solver sizes its grids by it)
    DevBuf<int> rmax_d;
    DevBuf<double> invd;                // 1 / diag(L)
    DevBuf<Front> fronts; DevBuf<double> pool;      // separator tree: the fronts and their border arrays
    // n unknowns; allocates on the context's stream and sets the solver kernels' shared-memory limits on first use
    int upload(lvb_ctx* ctx, const SolverPlan& sp, const std::vector<int>& env_rmax, int n);
    // rhs <- S^-1 rhs for S (n x n, element (i, j) at i * srow + j + soff, half bandwidth `band` for the tree), after lm_control_pre
    // (run by the solver's first kernel unless pre_done: an earlier kernel of the pass ran it);
    // a non-positive pivot sets st->solve_fail, a finished solve (st->done) makes every kernel return at once
    int launch(lvb_ctx* ctx, double* S, double* rhs, int n, long long srow, long long soff, int band, LmState* st, bool pre_done = false) const;
};

// The plan-shaping A/B switches LVB_NO_TREE and LVB_TREE_SEP_BAND, read once per process.
bool no_tree_switch();
bool tree_sep_band_switch();

// The LM pre-check (lm_control_pre) on its own, for passes whose solver does not run it in its first kernel.
__global__ void lm_control_pre_kernel(LmState* st);

}  // namespace lvb
