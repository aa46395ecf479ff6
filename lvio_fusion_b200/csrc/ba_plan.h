// ba_plan.h -- the structure plan of a bundle-adjustment problem: pure host arithmetic on the caller's index arrays that fixes the
// device layout before anything is uploaded (lvb_ba_finalize runs it, then uploads what it produced).  Plain C++17 with no CUDA
// include, so that the planner can be compiled and tested on its own (tests/test_ba_plan.py).
//
// Phases, in order (plan_ba runs them in sequence):
//   validate -> order the unknowns -> order the factors -> landmark CSR -> Schur groups -> envelope of S
//   -> storage and reduced solver -> tensor-core compaction maps
#pragma once
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <algorithm>
#include <functional>
#include <string>
#include <utility>
#include <vector>
#include "../../include/lvio_b200.h"

namespace lvb {

// MAX_CTA_SMEM: the 227 KB of dynamic shared memory one CTA may opt into on sm_90, less 256 B of headroom
// CHOL_RES_STEPS: most 32-column steps of the resident single-CTA solve (its table of block-column offsets)
enum { MAX_DIMC = 736, MAX_TRACK = 16, IMU_RAW = 469, CHOL_T = 256, CHOL_DT = 32 * 34 + 32, CHOL_HDR = 2 * CHOL_DT,      // doubles: (Dt, invd) twice, then the panel
       MAX_CTA_SMEM = 227 * 1024 - 256, CHOL_RES_STEPS = 32 };

// Shared memory of the resident single-CTA solve, in doubles after the (Dt, invd) pair: the backward partial sums (CHOL_T), the rhs
// (n, padded to an even count), then block column k = rows kb .. rmax[k] x 32 columns at a row stride of 34 doubles (16-byte rows, as
// the panel of the global-memory kernel).  rmax is non-decreasing and >= the step's last column, so every trailing tile of step k
// lands inside the stored rows of its block column.  Returns the block-column area's size in doubles.
inline long long chol_resident_columns(int n, const int* rmax) {
    long long d = 0;
    for (int kb = 0; kb < n; kb += 32) d += (long long)(rmax[kb >> 5] - kb + 1) * 34;
    return d;
}
inline int chol_resident_rhs(int n) { return (n + 1) & ~1; }

// per factor kind: doubles of one constant record and int32 indices of one block, as the caller adds them
constexpr int kConstStride[6] = {5, 6, 5, IMU_RAW, 8, 9};
constexpr int kIdxStride[6] = {3, 1, 1, 8, 2, 1};

struct Front {
    int o0, m;              // own unknowns [o0, o0 + m)
    int wL, wR;             // widths of the bounding ancestor separators (0 at the ends of the trajectory)
    int bL0, bR0;           // their first unknowns
    int actR;               // own column from which the right-border rows can be non-zero (leaves: m - band; internal: 0)
    int child0, child1;     // front ids, -1 for leaves
    int parent, side;       // parent front id (-1: root) and which child this is (0: left, 1: right)
    int ld, nb;             // border array: (nb + 1) rows (borders, then the rhs row) x ld (= m own columns + nb border columns)
    long long bd;           // offset of the border array in the pool (doubles)
};

// Shared memory of a front's partial factorisation (ba_front_factor_kernel) for panels of up to `rows` rows, in bytes: the diagonal
// block Dt (32 x 34) and its invd (32), then the panel from FRONT_PANEL on at a row stride of 34, reserved for rows + 2 rows, then
// 96 doubles of slack.  The slack counts in the size that decides whether a tree's fronts fit (MAX_CTA_SMEM).
enum { FRONT_PANEL = 32 * 34 + 32 };
inline size_t front_factor_smem(int rows) { return (size_t)(FRONT_PANEL + (rows + 2) * 34 + 96) * 8; }

// How the reduced camera system is factored: the separator tree when it has levels (ba_tree.cuh), else the single-CTA kernel with
// the whole envelope resident in shared memory when it fits, else the single-CTA kernel on S in global memory when its panel fits,
// else the per-phase grids of ba_wide.cuh.
struct SolverPlan {
    size_t chol_smem = 0;               // single-CTA kernel on S in global memory: two diagonal-block buffers + the panel (>= 34 rows; later the backward partial sums)
    bool resident = false;              // single-CTA kernel with the envelope in shared memory
    size_t resident_smem = 0;           // its dynamic shared memory (chol_resident_layout)
    int tree_levels = 0;                // 0: no separator tree
    std::vector<Front> fronts;
    std::vector<int> level_first, level_count;
    size_t pool_doubles = 0, tree_factor_smem = 0, tree_back_smem = 0;
    bool wide = false;
};

// What the plan reads of a problem: counts, constant flags and the factor records in the caller's order (not owned).
struct BaProblemView {
    int np = 0, nv = 0, nr = 0;
    const uint8_t *pose_const = nullptr, *vec3_const = nullptr, *rho_const = nullptr;
    int n[6] = {0, 0, 0, 0, 0, 0};
    const double* fc[6] = {};
    const int32_t* fi[6] = {};
};

struct PlanBlock { long long key; int type, idx, width; };      // one free parameter block of the camera system (type 0: pose, 1: vec3)

struct BaPlan {
    // unknowns of the reduced camera system, keyframe by keyframe
    int n_pose_free = 0, n_vec3_free = 0, n_rho_free = 0, dimc = 0;
    std::vector<int> pose_off, vec3_off, rho_slot;      // camera-system offset of a pose / vec3 block, slot of an inverse depth (-1: constant)
    std::vector<int> canon;             // internal camera-system offset -> canonical (poses first, then vec3) offset
    std::vector<PlanBlock> blks;        // the free blocks in camera-system order
    std::vector<int> blk_start, blk_of_off;
    bool dense = true;                  // dense lower-triangular storage of Hpp / S (dimc <= MAX_DIMC), else banded
    bool solvable = false;
    const char* unsolvable_why = "the problem has no free camera parameter";
    // factors in device order
    int nd[6] = {0, 0, 0, 0, 0, 0};     // blocks in the device layout (kinds 0/1: sorted by pose key, each key padded to 32)
    std::vector<int> order[6];          // device position -> caller index, -1 - caller index for a padding copy
    // landmark CSR over device positions: TwoFrame i -> i, TwoCamera f -> -(f+1); lm_off: the two free-pose offsets of every entry
    std::vector<int> lm_start, lm_fac, lm_off;
    // Schur groups: landmarks with the same sorted set of free pose offsets share a warp-sized work item
    std::vector<int> tf_slot, sw_group, sw_lm, grp_ns, grp_off;
    int n_schur_warps = 0, schur_cols_max = 0;
    // envelope of S per 32-column block step, and the true half bandwidth
    std::vector<int> chol_rmax, chol_cmin;
    int true_band = 0;
    // storage of Hpp / S: element (i, j), i >= j, at i * srow + j + soff; band: half bandwidth of the banded storage (dense: of the envelope)
    int band = 0;
    long long srow = 0, soff = 0;
    size_t nS = 1;
    SolverPlan solver;
    // tensor-core Schur (schur_mode 1): camera offset -> compact pose dimension (0..127) and back
    bool tc_ok = false;
    std::vector<int> tc_cdim, tc_off;
};

// Sharded problems: the collectives that make the plan the same on every rank.  Each reduces a host array element-wise over the
// ranks in place and returns LVB_OK or an error code (whose message it has set).  Not called when world == 1.
struct PlanHooks {
    std::function<int(std::vector<int>&)> max_reduce;      // the keys of the vec3 blocks
    std::function<int(std::vector<int>&)> min_reduce;      // the first column of every block row of S
    std::function<void(const char*)> phase_done;           // optional: called with the name of each phase when it is done
};

inline int plan_fail(std::string& err, int rc, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    err = buf;
    return rc;
}

// ---- validate indices (the TwoFrame list is the long one: a branch-free pass; the other kinds through the general rule)
inline int plan_validate(const BaProblemView& in, std::string& err) {
    const int np = in.np, nv = in.nv, nr = in.nr;
    const int32_t* ix = in.fi[0];
    int bad = 0;
    for (int f = 0; f < in.n[0]; ++f, ix += 3) bad |= ((unsigned)ix[0] >= (unsigned)nr) | ((unsigned)ix[1] >= (unsigned)np) | ((unsigned)ix[2] >= (unsigned)np);
    for (int k = bad ? 0 : 1; k < 6; ++k) for (int f = 0; f < in.n[k]; ++f) for (int j = 0; j < kIdxStride[k]; ++j) {
        const int v = in.fi[k][(size_t)f * kIdxStride[k] + j];
        int lim = np;
        if ((k == 0 && j == 0) || k == 2) lim = nr;
        if (k == 3 && j != 0 && j != 4) lim = nv;
        if (k == 3 && (j == 6 || j == 7) && v == -1 && in.fc[3][(size_t)f * IMU_RAW + 467] >= 0.0) continue;     // ImuInitError has no j-side bias blocks
        if (v < 0 || v >= lim) return plan_fail(err, LVB_ERR_INVALID, "factor kind %d block %d: index %d out of range [0,%d)", k, f, v, lim);
    }
    return LVB_OK;
}

// ---- slots / offsets.  Unknowns of the reduced camera system are ordered keyframe by keyframe
// (pose_i, then the velocity / bias blocks an ImuError ties to pose_i): co-visibility and the IMU chain only
// couple neighbouring keyframes, so S is block-banded and the Cholesky works inside its envelope.
// `canon` is the caller-visible order (all poses, then all vec3 blocks) used by lvb_ba_reduced_system.
inline int plan_unknowns(const BaProblemView& in, int world, const PlanHooks& hooks, BaPlan& p, std::string& err) {
    const int np = in.np, nv = in.nv, nr = in.nr;
    p.pose_off.assign(np, -1); p.vec3_off.assign(nv, -1); p.rho_slot.assign(nr, 0);
    int npf = 0, nvf = 0, nrf = 0;
    for (int i = 0; i < np; ++i) if (!in.pose_const[i]) ++npf;
    for (int i = 0; i < nv; ++i) if (!in.vec3_const[i]) ++nvf;
    for (int i = 0; i < nr; ++i) p.rho_slot[i] = in.rho_const[i] ? -1 : nrf++;
    p.n_pose_free = npf; p.n_vec3_free = nvf; p.n_rho_free = nrf; p.dimc = 6 * npf + 3 * nvf;
    std::vector<PlanBlock>& blks = p.blks;
    blks.clear();
    {
        std::vector<int> vkey(nv, -1);
        if ((long long)np * 8 >= (1ll << 31)) return plan_fail(err, LVB_ERR_UNSUPPORTED, "too many poses");
        for (int f = 0; f < in.n[3]; ++f) {
            const int32_t* ix = &in.fi[3][8 * (size_t)f];
            for (int b = 1; b < 8; ++b) { if (b == 4) continue; const int v = ix[b]; if (v < 0) continue; const int q = ix[b < 4 ? 0 : 4]; if (vkey[v] < 0) vkey[v] = q * 8 + (b & 3); }
        }
        // sharded problems: a rank only sees the IMU factors it owns, but the order of the unknowns (= the layout of the
        // all-reduced system) must be the same on every rank: take the key any rank found (collective, like the envelope)
        if (world > 1 && nv > 0) { if (int rc = hooks.max_reduce(vkey)) return rc; }
        for (int i = 0; i < np; ++i) if (!in.pose_const[i]) blks.push_back({(long long)i * 8, 0, i, 6});
        for (int i = 0; i < nv; ++i) if (!in.vec3_const[i]) blks.push_back({vkey[i] >= 0 ? (long long)vkey[i] : (long long)np * 8 + i, 1, i, 3});
        std::stable_sort(blks.begin(), blks.end(), [](const PlanBlock& a, const PlanBlock& b) { return a.key < b.key; });
    }
    p.blk_of_off.assign(p.dimc, 0); p.blk_start.assign(blks.size() + 1, 0);
    p.canon.assign(p.dimc, 0);
    {
        int off = 0, ps = 0, vs = 0;
        std::vector<int> pslot(np, -1), vslot(nv, -1);
        for (int i = 0; i < np; ++i) if (!in.pose_const[i]) pslot[i] = ps++;
        for (int i = 0; i < nv; ++i) if (!in.vec3_const[i]) vslot[i] = vs++;
        for (size_t b = 0; b < blks.size(); ++b) {
            p.blk_start[b] = off;
            const int c0 = blks[b].type == 0 ? 6 * pslot[blks[b].idx] : 6 * npf + 3 * vslot[blks[b].idx];
            if (blks[b].type == 0) p.pose_off[blks[b].idx] = off; else p.vec3_off[blks[b].idx] = off;
            for (int k = 0; k < blks[b].width; ++k) { p.blk_of_off[off + k] = (int)b; p.canon[off + k] = c0 + k; }
            off += blks[b].width;
        }
        p.blk_start[blks.size()] = off;
    }
    // camera systems up to MAX_DIMC use dense lower-triangular storage, larger ones banded storage
    p.dense = p.dimc <= MAX_DIMC;
    p.solvable = p.dimc > 0;
    return LVB_OK;
}

// ---- device order of the blocks.  TwoFrame blocks sorted by (pose_1, pose_2), PoseOnly blocks by pose, so that
// a warp of the linearize kernel owns one key (or a few key segments) and can reduce its J^T J in shared memory
// before touching HBM.  Dense-layout (window-sized) problems also pad every key run to a multiple of 32 with
// weight-0 copies: one segment per warp.  Large problems stay unpadded (their runs are short, padding would
// inflate the block arrays).
inline void plan_factor_order(const BaProblemView& in, BaPlan& p) {
    const int np = in.np;
    for (int k = 0; k < 6; ++k) {
        std::vector<int>& ord = p.order[k];
        ord.clear();
        const int n = in.n[k];
        if (p.solvable && (k == 0 || k == 1) && n > 0) {
            // stable order by key: counting sort when the key space is small (window-sized problems), else a pair sort
            std::vector<long long> keys(n);
            const long long key_space = (k == 0) ? (long long)np * np : (long long)np;
            for (int f = 0; f < n; ++f) keys[f] = (k == 0) ? (long long)in.fi[0][3 * (size_t)f + 1] * np + in.fi[0][3 * (size_t)f + 2] : (long long)in.fi[1][f];
            std::vector<int> ids(n);
            if (key_space <= (1 << 16)) {
                std::vector<int> start((size_t)key_space + 1, 0);
                for (int f = 0; f < n; ++f) start[keys[f] + 1]++;
                for (long long c = 0; c < key_space; ++c) start[c + 1] += start[c];
                for (int f = 0; f < n; ++f) ids[start[keys[f]]++] = f;
            } else {
                std::vector<std::pair<long long, int>> kv(n);
                for (int f = 0; f < n; ++f) kv[f] = {keys[f], f};
                std::sort(kv.begin(), kv.end());
                for (int f = 0; f < n; ++f) ids[f] = kv[f].second;
            }
            ord.reserve((size_t)n + 32 * 64);
            for (int i = 0; i < n;) {
                int j = i; while (j < n && keys[ids[j]] == keys[ids[i]]) ++j;
                for (int t = i; t < j; ++t) ord.push_back(ids[t]);
                while (p.dense && ord.size() % 32) ord.push_back(-1 - ids[i]);     // padding: encoded source block
                i = j;
            }
        } else { ord.resize(n); for (int f = 0; f < n; ++f) ord[f] = f; }
        p.nd[k] = (int)ord.size();
    }
}

// ---- landmark CSR.  The count runs over the caller's order (sequential); the fill has to follow the device order, so its gather
// is prefetched, and it also notes the two free-pose offsets of every entry (lm_off) so that the grouping never goes back to the
// factor records.
inline void plan_landmark_csr(const BaProblemView& in, BaPlan& p) {
    const int nr = in.nr, n_tf = p.nd[0];
    std::vector<int>& lm_start = p.lm_start;
    lm_start.assign(nr + 1, 0);
    {
        const int32_t* ix = in.fi[0];
        for (int f = 0; f < in.n[0]; ++f) lm_start[ix[3 * (size_t)f] + 1]++;
    }
    for (int f = 0; f < in.n[2]; ++f) lm_start[in.fi[2][f] + 1]++;
    for (int i = 0; i < nr; ++i) lm_start[i + 1] += lm_start[i];
    p.lm_fac.assign(std::max(1, lm_start[nr]), 0); p.lm_off.assign(2 * (size_t)std::max(1, lm_start[nr]), -1);
    std::vector<int> fill(lm_start.begin(), lm_start.end() - 1);
    {
        const int32_t* hi = in.fi[0];
        const int* ord = p.order[0].data();
        for (int i = 0; i < n_tf; ++i) {
            if (i + 16 < n_tf && ord[i + 16] >= 0) __builtin_prefetch(hi + 3 * (size_t)ord[i + 16]);
            if (ord[i] < 0) continue;
            const int32_t* ix = hi + 3 * (size_t)ord[i];
            const int pos = fill[ix[0]]++;
            p.lm_fac[pos] = i; p.lm_off[2 * (size_t)pos] = p.pose_off[ix[1]]; p.lm_off[2 * (size_t)pos + 1] = p.pose_off[ix[2]];
        }
    }
    for (int f = 0; f < in.n[2]; ++f) p.lm_fac[fill[in.fi[2][f]]++] = -(f + 1);
}

// ---- Schur groups.  signature = sorted set of free pose offsets of a landmark; groups found through an open-addressing hash table
// over the signatures (no per-landmark heap traffic), numbered in order of first appearance
inline int plan_schur_groups(int nr, BaPlan& p, std::string& err) {
    const int n_tf = p.nd[0];
    const std::vector<int>& lm_start = p.lm_start;
    const std::vector<int>& lm_fac = p.lm_fac;
    const std::vector<int>& lm_off = p.lm_off;
    std::vector<int>& tf_slot = p.tf_slot;
    std::vector<int>& sw_group = p.sw_group;
    std::vector<int>& sw_lm = p.sw_lm;
    std::vector<int>& grp_ns = p.grp_ns;
    std::vector<int>& grp_off = p.grp_off;
    tf_slot.assign((size_t)std::max(1, n_tf) * 2, -1); sw_group.clear(); sw_lm.clear(); grp_ns.clear(); grp_off.clear();
    int cols_max = 0;
    std::vector<std::vector<int>> members;
    size_t tsize = 64; while (tsize < 4 * (size_t)std::max(1, p.n_rho_free)) tsize <<= 1;
    if (tsize > ((size_t)1 << 20)) tsize = (size_t)1 << 20;
    std::vector<int> table(tsize, -1);
    for (int l = 0; l < nr; ++l) {
        if (p.rho_slot[l] < 0) continue;
        int sig[MAX_TRACK + 1], ns = 0;
        for (int e = lm_start[l]; e < lm_start[l + 1]; ++e) {
            if (lm_fac[e] < 0) continue;
            for (int side = 1; side <= 2; ++side) {
                const int off = lm_off[2 * (size_t)e + side - 1];
                if (off < 0) continue;
                int q = 0; while (q < ns && sig[q] < off) ++q;
                if (q < ns && sig[q] == off) continue;
                if (ns == MAX_TRACK) return plan_fail(err, LVB_ERR_UNSUPPORTED, "landmark %d is observed from more than %d keyframes", l, (int)MAX_TRACK);
                for (int t = ns; t > q; --t) sig[t] = sig[t - 1];
                sig[q] = off; ++ns;
            }
        }
        unsigned long long h = 1469598103934665603ull ^ (unsigned long long)ns;
        for (int q = 0; q < ns; ++q) { h ^= (unsigned long long)(unsigned)sig[q]; h *= 1099511628211ull; }
        size_t slot = (size_t)(h ^ (h >> 29)) & (tsize - 1);
        int g = -1;
        for (;;) {
            const int cand = table[slot];
            if (cand < 0) break;
            if (grp_ns[cand] == ns) {
                bool same = true;
                for (int q = 0; q < ns && same; ++q) same = grp_off[(size_t)cand * MAX_TRACK + q] == sig[q];
                if (same) { g = cand; break; }
            }
            slot = (slot + 1) & (tsize - 1);
        }
        if (g < 0) {
            g = (int)members.size();
            if ((size_t)g * 2 >= tsize) {      // keep the load factor below 1/2: rebuild a larger table
                tsize <<= 1; table.assign(tsize, -1);
                for (int c = 0; c < g; ++c) {
                    unsigned long long hc = 1469598103934665603ull ^ (unsigned long long)grp_ns[c];
                    for (int q = 0; q < grp_ns[c]; ++q) { hc ^= (unsigned long long)(unsigned)grp_off[(size_t)c * MAX_TRACK + q]; hc *= 1099511628211ull; }
                    size_t sc = (size_t)(hc ^ (hc >> 29)) & (tsize - 1);
                    while (table[sc] >= 0) sc = (sc + 1) & (tsize - 1);
                    table[sc] = c;
                }
                slot = (size_t)(h ^ (h >> 29)) & (tsize - 1);
                while (table[slot] >= 0) slot = (slot + 1) & (tsize - 1);
            }
            table[slot] = g;
            members.emplace_back(); grp_ns.push_back(ns);
            for (int k2 = 0; k2 < MAX_TRACK; ++k2) grp_off.push_back(k2 < ns ? sig[k2] : -1);
        }
        members[g].push_back(l);
        for (int e = lm_start[l]; e < lm_start[l + 1]; ++e) {
            const int i = lm_fac[e]; if (i < 0) continue;
            for (int side = 1; side <= 2; ++side) {
                const int off = lm_off[2 * (size_t)e + side - 1];
                if (off < 0) continue;
                int q = 0; while (sig[q] != off) ++q;
                tf_slot[(size_t)(side - 1) * n_tf + i] = q;
            }
        }
    }
    for (size_t g = 0; g < members.size(); ++g) {
        cols_max = std::max(cols_max, 6 * grp_ns[g] + 1);
        for (size_t i = 0; i < members[g].size(); i += 32) {
            sw_group.push_back((int)g);
            for (size_t t = i; t < i + 32; ++t) sw_lm.push_back(t < members[g].size() ? members[g][t] : -1);
        }
    }
    p.n_schur_warps = (int)sw_group.size(); p.schur_cols_max = cols_max;
    // never empty on the device
    if (sw_group.empty()) { sw_group.push_back(0); sw_lm.assign(32, -1); }
    if (grp_ns.empty()) { grp_ns.push_back(0); grp_off.assign(MAX_TRACK, -1); }
    return LVB_OK;
}

// ---- envelope of S: first structurally non-zero column per row, from every coupling the assembly can create
inline int plan_envelope(const BaProblemView& in, int world, const PlanHooks& hooks, BaPlan& p) {
    const int dimc = p.dimc;
    const std::vector<int>& blk_of_off = p.blk_of_off;
    const std::vector<int>& blk_start = p.blk_start;
    const std::vector<int>& pose_off = p.pose_off;
    p.chol_rmax.assign(dimc / 32 + 2, 0); p.chol_cmin.assign(dimc / 32 + 2, 0);
    int band = 0, true_band = 0;
    if (p.solvable) {
        std::vector<int> first(dimc);
        std::vector<int> fb(p.blks.size());
        for (size_t b = 0; b < p.blks.size(); ++b) fb[b] = blk_start[b];
        auto couple = [&](int offA, int offB) {
            if (offA < 0 || offB < 0) return;
            const int a = blk_of_off[offA], b = blk_of_off[offB];
            const int lo = std::min(a, b), hi = std::max(a, b);
            fb[hi] = std::min(fb[hi], blk_start[lo]);
        };
        for (size_t g = 0; g < p.grp_ns.size(); ++g) for (int a = 0; a < p.grp_ns[g]; ++a) for (int b = 0; b < a; ++b) couple(p.grp_off[g * MAX_TRACK + a], p.grp_off[g * MAX_TRACK + b]);
        for (int f = 0; f < in.n[0]; ++f) couple(pose_off[in.fi[0][3 * (size_t)f + 1]], pose_off[in.fi[0][3 * (size_t)f + 2]]);
        for (int f = 0; f < in.n[3]; ++f) {
            const int32_t* ix = &in.fi[3][8 * (size_t)f];
            int offs[8];
            for (int b = 0; b < 8; ++b) offs[b] = ix[b] < 0 ? -1 : ((b == 0 || b == 4) ? pose_off[ix[b]] : p.vec3_off[ix[b]]);
            for (int a = 0; a < 8; ++a) for (int b = 0; b < a; ++b) couple(offs[a], offs[b]);
        }
        for (int f = 0; f < in.n[4]; ++f) couple(pose_off[in.fi[4][2 * (size_t)f]], pose_off[in.fi[4][2 * (size_t)f + 1]]);
        // sharded problems: the other ranks' couplings arrive with the all-reduce, so the envelope must be the global one
        if (world > 1) { if (int rc = hooks.min_reduce(fb)) return rc; }
        for (int r = 0; r < dimc; ++r) { first[r] = fb[blk_of_off[r]]; true_band = std::max(true_band, r - first[r]); }
        // rmax per 32-column step by a backward sweep: rows whose first column lies left of the end of the step
        const int nstep = (dimc + 31) / 32;
        std::vector<int> last_row_of_col(dimc, 0);      // largest row r with first[r] <= c, via prefix max over c
        for (int c = 0; c < dimc; ++c) last_row_of_col[c] = c;
        for (int r = 0; r < dimc; ++r) last_row_of_col[first[r]] = std::max(last_row_of_col[first[r]], r);
        for (int c = 1; c < dimc; ++c) last_row_of_col[c] = std::max(last_row_of_col[c], last_row_of_col[c - 1]);
        for (int step = 0; step < nstep; ++step) {
            const int kb = step * 32, bs = std::min(32, dimc - kb);
            int cmin = kb;
            for (int r = kb; r < kb + bs; ++r) cmin = std::min(cmin, first[r]);
            const int rmax = std::max(kb + bs - 1, last_row_of_col[kb + bs - 1]);
            p.chol_rmax[step] = rmax; p.chol_cmin[step] = cmin;
            band = std::max(band, std::max(rmax - kb, kb + bs - 1 - cmin));
        }
    }
    p.band = band; p.true_band = true_band;
    return LVB_OK;
}

// Separator tree of the banded reduced system (see ba_tree.cuh): complete binary tree with 2^D leaves, separators of width
// w = min(sep, band), the true half bandwidth being enough to separate (the storage band carries up to 31 columns of block-step
// slack; a front's cost grows with the cube of w).  Leaves keep >= 2w unknowns so that a separator is coupled to nothing beyond its
// two neighbouring subtrees.
inline int build_front_tree(int n, int band, int sep, int max_leaves, std::vector<Front>& out, std::vector<int>& level_first, std::vector<int>& level_count,
                            size_t& pool_doubles, int& max_panel_rows, int& max_nb) {
    out.clear(); level_first.clear(); level_count.clear(); pool_doubles = 0; max_panel_rows = 0; max_nb = 0;
    const int w = std::max(1, std::min(sep, band));
    int D = 0;
    while ((1 << (D + 1)) <= max_leaves) {
        const long long P = 1ll << (D + 1);
        const long long leaf = ((long long)n - (P - 1) * w) / P;
        if (leaf < 2ll * w || leaf < 64) break;
        ++D;
    }
    if (D == 0) return 0;
    struct Node { int o0, m, bL0, wL, bR0, wR, c0, c1, h; };
    std::vector<Node> nodes;
    std::function<int(int, int, int, int, int, int, int)> rec = [&](int a, int b, int depth, int bL0, int wL, int bR0, int wR) -> int {
        if (depth == D) { nodes.push_back({a, b - a, bL0, wL, bR0, wR, -1, -1, 0}); return (int)nodes.size() - 1; }
        const int s0 = a + (b - a - w) / 2;
        const int c0 = rec(a, s0, depth + 1, bL0, wL, s0, w);
        const int c1 = rec(s0 + w, b, depth + 1, s0, w, bR0, wR);
        nodes.push_back({s0, w, bL0, wL, bR0, wR, c0, c1, D - depth});
        return (int)nodes.size() - 1;
    };
    rec(0, n, 0, 0, 0, 0, 0);
    std::vector<int> ids(nodes.size()), new_id(nodes.size());
    for (size_t i = 0; i < ids.size(); ++i) ids[i] = (int)i;
    std::stable_sort(ids.begin(), ids.end(), [&](int a, int b) { return nodes[a].h != nodes[b].h ? nodes[a].h < nodes[b].h : nodes[a].o0 < nodes[b].o0; });
    for (size_t i = 0; i < ids.size(); ++i) new_id[ids[i]] = (int)i;
    level_first.assign(D + 1, 0); level_count.assign(D + 1, 0);
    for (size_t i = 0; i < ids.size(); ++i) {
        const Node& nd = nodes[ids[i]];
        Front F;
        F.o0 = nd.o0; F.m = nd.m; F.wL = nd.wL; F.wR = nd.wR; F.bL0 = nd.bL0; F.bR0 = nd.bR0;
        F.actR = nd.h == 0 ? std::max(0, nd.m - band) : 0;
        F.child0 = nd.c0 < 0 ? -1 : new_id[nd.c0]; F.child1 = nd.c1 < 0 ? -1 : new_id[nd.c1];
        F.parent = -1; F.side = 0;
        F.nb = nd.wL + nd.wR; F.ld = (nd.m + F.nb + 1) & ~1;
        F.bd = (long long)pool_doubles;
        pool_doubles += ((size_t)(F.nb + 1) * F.ld + 1) & ~(size_t)1;
        if (level_count[nd.h] == 0) level_first[nd.h] = (int)i;
        level_count[nd.h]++;
        max_nb = std::max(max_nb, F.nb);
        max_panel_rows = std::max(max_panel_rows, std::min(nd.m, band) + F.nb + 1);
        out.push_back(F);
    }
    for (size_t i = 0; i < out.size(); ++i) {
        if (out[i].child0 >= 0) { out[out[i].child0].parent = (int)i; out[out[i].child0].side = 0; }
        if (out[i].child1 >= 0) { out[out[i].child1].parent = (int)i; out[out[i].child1].side = 1; }
    }
    return D + 1;
}

// The one rule that picks the solver of an n x n system in banded storage of half bandwidth `band` with the envelope rmax (last
// row per 32-column step): the single-CTA kernel's shared memory, then -- unless no_tree -- a separator tree with separators of
// width `sep` when it has at least two leaves and its fronts and pool fit; without a tree, the resident single-CTA solve when the
// whole envelope fits in shared memory, the single-CTA solve on S in global memory when its panel fits, else the wide solver.
inline SolverPlan plan_reduced_solver(int n, int band, int sep, const std::vector<int>& rmax, int sm_count, bool no_tree) {
    SolverPlan s;
    int panel_rows = 2;
    const int nstep = (n + 31) / 32;
    for (int step = 0; step < nstep; ++step) {
        const int kb = step * 32, bs = std::min(32, n - kb);
        panel_rows = std::max(panel_rows, rmax[step] - (kb + bs) + 2);
    }
    s.chol_smem = (size_t)(CHOL_HDR + std::max(panel_rows + 2, 34) * 34) * 8;
    s.resident_smem = (size_t)(CHOL_HDR + CHOL_T + chol_resident_rhs(n) + chol_resident_columns(n, rmax.data())) * 8;
    if (!no_tree) {
        int rows = 0, mnb = 0, max_leaves = 1;
        while (max_leaves * 2 <= std::max(2, sm_count)) max_leaves *= 2;
        const int lv = build_front_tree(n, band, sep, max_leaves, s.fronts, s.level_first, s.level_count, s.pool_doubles, rows, mnb);
        const size_t fs = front_factor_smem(rows), bs = (size_t)(((mnb + 1) & ~1) + (CHOL_T / 32) * 32) * 8;
        if (lv > 0 && fs <= MAX_CTA_SMEM && s.pool_doubles < ((size_t)1 << 31)) { s.tree_levels = lv; s.tree_factor_smem = fs; s.tree_back_smem = bs; }
    }
    s.resident = s.tree_levels == 0 && nstep <= CHOL_RES_STEPS && s.resident_smem <= MAX_CTA_SMEM;
    s.wide = s.tree_levels == 0 && !s.resident && s.chol_smem > MAX_CTA_SMEM;
    return s;
}

// Envelope of a full band of half bandwidth `band` (every row reaches `band` columns left of the diagonal).
inline void uniform_band_envelope(int n, int band, std::vector<int>& rmax, std::vector<int>& cmin) {
    const int nstep = (n + 31) / 32;
    rmax.assign(nstep + 2, 0); cmin.assign(nstep + 2, 0);
    for (int st = 0; st < nstep; ++st) {
        const int kb = st * 32, bs = std::min(32, n - kb);
        rmax[st] = std::min(n - 1, kb + band); cmin[st] = std::max(0, kb + bs - 1 - band);
    }
}

// ---- storage of Hpp / S and the reduced solver.  The envelope is the one of GLOBAL 32-column steps; the fronts of the separator
// tree step through 32 columns from their own first unknown, and for an arbitrary start a block column needs rows up to
// true_band + 31 below its first column.  Banded systems are split by a separator tree when the band leaves room for at least two
// leaves (ba_tree.cuh).
inline void plan_storage_and_solver(int sm_count, bool no_tree, bool sep_is_band, BaPlan& p) {
    int band = p.band;
    if (!p.dense) band = std::max(band, p.true_band + 31);
    band = std::min(std::max(band, 31), std::max(31, p.dimc - 1));
    if (p.dense) { p.srow = p.dimc; p.soff = 0; p.nS = (size_t)p.dimc * p.dimc; }
    else         { p.srow = band; p.soff = band; p.nS = (size_t)p.dimc * (size_t)(band + 1); }
    p.band = band;
    p.solver = plan_reduced_solver(p.dimc, band, sep_is_band ? band : p.true_band, p.chol_rmax, sm_count, no_tree || p.dense || !p.solvable);
    if (p.solvable && p.nS > ((size_t)3 << 30)) { p.solvable = false; p.unsolvable_why = "the banded reduced camera system exceeds 24 GB"; }
    if (!p.solvable) p.nS = 1;
}

// ---- tensor-core Schur operands: compact pose dimensions (<= 128)
inline void plan_tensor_core_maps(int world, BaPlan& p) {
    p.tc_ok = p.solvable && p.dense && 6 * p.n_pose_free <= 128 && p.n_pose_free > 0 && world == 1;
    p.tc_cdim.assign(std::max(1, p.dimc), -1); p.tc_off.assign(128, -1);
    int c = 0;
    for (size_t b = 0; b < p.blks.size(); ++b) if (p.blks[b].type == 0 && c + 6 <= 128) { for (int k = 0; k < 6; ++k) { p.tc_cdim[p.blk_start[b] + k] = c + k; p.tc_off[c + k] = p.blk_start[b] + k; } c += 6; }
}

// All phases in order.  no_tree: never split the banded system by a separator tree; sep_is_band: separators as wide as the storage
// band instead of the true half bandwidth.  On failure returns the error code with its message in `err` (empty when a hook failed).
inline int plan_ba(const BaProblemView& in, int sm_count, int world, bool no_tree, bool sep_is_band, const PlanHooks& hooks, BaPlan& p, std::string& err) {
    auto done = [&](const char* name) { if (hooks.phase_done) hooks.phase_done(name); };
    if (int rc = plan_validate(in, err)) return rc;
    done("validate");
    if (int rc = plan_unknowns(in, world, hooks, p, err)) return rc;
    done("block order");
    plan_factor_order(in, p);
    done("factor sort + pad");
    plan_landmark_csr(in, p);
    done("landmark CSR");
    if (int rc = plan_schur_groups(in.nr, p, err)) return rc;
    done("schur groups");
    if (int rc = plan_envelope(in, world, hooks, p)) return rc;
    plan_storage_and_solver(sm_count, no_tree, sep_is_band, p);
    plan_tensor_core_maps(world, p);
    done("envelope");
    return LVB_OK;
}

}  // namespace lvb
