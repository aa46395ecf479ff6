// ba.cu -- sliding-window bundle adjustment on the device: the kernels behind
// adapt::Problem / ceres::Solve for the factor mix of Backend::BuildProblem
// (/root/reference/src/lvio_fusion/src/backend.cpp:96-183,192-211).
//
// Data layout in HBM (all FP64 unless noted):
//   parameter blocks   poses[n][7] (AoS, 56 B), vec3[n][3], rho[n]           + candidate copies
//   factor constants   SoA planes per kind: plane k of kind K at fc[K] + k*n[K]  (coalesced reads)
//   factor indices     SoA int32 planes fi[K] + k*n[K]
//   IMU constants      AoS per factor, 287 doubles: 17 scalars, five 3x3 sub-blocks, U (15x15)
//   accumulators       Hpp (dimc x dimc, lower), gc, Hll, gl, per-TwoFrame-factor W rows (one 96 B record per factor)
//   reduction arena    [ S | rhs | gc | diag(Hpp) | 16 scalars ]  -- the one buffer all-reduced per iteration
//
// Kernels (K-numbers of SURVEY.md section 2):
//   K1  ba_eval_*            residual + ambient Jacobian materialised (parity / roofline entry)
//   K1-K4 ba_linearize       fused evaluate + robustify + J^T J / J^T r assembly (atomics on the lower triangle)
//   K5  ba_schur             eliminate the 1-dim inverse-depth blocks into S
//   K6  ba_cholesky + ba_update + lm control   reduced solve, back-substitution, (+) update, LM decisions
#include <math.h>
#include <algorithm>
#include <chrono>
#include <functional>
#include <map>
#include <string.h>
#include <cuda_bf16.h>
#include "lvb_internal.cuh"
#include "lvb_math.cuh"
#include "lvb_imu_warp.cuh"
#include "lvb_chol.cuh"
#include "lvb_p2p.cuh"

using namespace lvb;

namespace {

enum { TPB = 128, IMU_STRIDE = 17 + 45 + 225 + 1, IMU_RAW = 469, MAX_DIMC = 736, MAX_STAGE_POSES = 512, MAX_TRACK = 16, CHOL_T = 256, SYRK_ROWS = 64, SYRK_LD = 14 };

__device__ long long g_chol_dbg[8];     // accumulated SM clocks per Cholesky phase (diag, panel, trailing, backward, total)
__device__ unsigned char c_tri_a[465];   // lower-triangle enumeration e -> (a, b), a >= b; global (not __constant__):
__device__ unsigned char c_tri_b[465];   // the index differs per lane and would serialise on the constant cache

struct BaDev {
    int n_poses, n_vec3, n_rho, dimc, n_pose_free;
    // lower-triangular storage of Hpp and S: element (i, j), i >= j, lives at i * srow + j + soff.
    // dense: srow = dimc, soff = 0 ; banded (half bandwidth B, dimc > MAX_DIMC): srow = B, soff = B (row-major n x (B+1)).
    long long srow, soff; size_t nS;
    double *poses, *vec3, *rho, *c_poses, *c_vec3, *c_rho;
    const int *pose_off, *vec3_off, *rho_slot;
    int n[6];
    const double* fc[6];
    const int* fi[6];
    double huber[6];
    const int *lm_start, *lm_fac;
    const int *tf_slot;                 // 2 planes: slot of pose_1 / pose_2 inside the landmark's Schur group (-1: constant pose)
    const int *sw_group, *sw_lm, *grp_ns, *grp_off;   // Schur warps: group id, 32 landmark ids (-1 pad); per group: #slots, offsets
    int n_schur_warps, warp_syrk;
    int tc_mode;                        // 1: Schur contraction on the tensor cores (wgmma, split bf16), FP64 rhs only here
    unsigned short* tc_u;               // packed U^T: [chunk of 16 landmarks][3 splits][128 x 16 bf16 K-major core-matrix tile]
    const int* tc_cdim;                 // camera offset -> compact pose dimension (0..127) or -1
    const int* tc_off;                  // compact pose dimension -> camera offset
    int tc_ndim;                        // 6 * free poses (<= 128)
    double *Hpp, *gc, *Hll, *gl, *tf_w;
    double *S, *rhs, *gcr, *diagH, *scal;      // inside the arena
    double *scale_c, *scale_l, *lam_c, *lam_l;
    LmState* st;
    int rank0, rank, world;
    int stage_poses;
    int imu_cta;                        // 1: one CTA per IMU factor (window-sized problems: latency), 0: one warp per factor (map scale)
    Cams cams;
};

#define SIDX(d_, i_, j_) ((size_t)(i_) * (size_t)(d_).srow + (size_t)(j_) + (size_t)(d_).soff)
struct BlockRanges { int b[7]; };   // cumulative block starts per kind, b[6] = total

// ------------------------------------------------------------------ small device helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    // TMA 1-D bulk copy global -> shared, completion counted on the mbarrier (SASS: UBLKCP)
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
    uint32_t ok = 0;
    do {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(phase) : "memory");
    } while (!ok);
}

// Stage the pose array into shared memory (TMA bulk copy when enabled) and return the pointer
// the block should read poses from.
__device__ __forceinline__ const double* stage_poses(const BaDev& d, const double* src, double* s_poses, uint64_t* bar) {
    if (!d.stage_poses) return src;
    const uint32_t bytes = ((uint32_t)d.n_poses * 56u + 15u) & ~15u;
    if (d.stage_poses == 2) {
        if (threadIdx.x == 0) mbar_init(bar, 1);
        __syncthreads();
        if (threadIdx.x == 0) { mbar_expect_tx(bar, bytes); bulk_load_1d(s_poses, src, bytes, bar); }
        mbar_wait(bar, 0);
    } else {
        for (int i = threadIdx.x; i < d.n_poses * 7; i += blockDim.x) s_poses[i] = src[i];
        __syncthreads();
    }
    return s_poses;
}

__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ void block_add(double v, double* target, double* s_red /*>= blockDim/32*/) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        double t = (lane < (int)(blockDim.x >> 5)) ? s_red[lane] : 0.0;
        t = warp_sum(t);
        if (lane == 0 && t != 0.0) atomicAdd(target, t);
    }
    __syncthreads();
}

// H(lower) += JA^T JB for two distinct blocks; offsets are global camera-system offsets (>= 0)
__device__ __forceinline__ void add_cross(double* H, const BaDev& d, int offA, const double* JA, int wa, int offB, const double* JB, int wb, int rows) {
    for (int i = 0; i < wa; ++i) for (int j = 0; j < wb; ++j) {
        double s = 0; for (int k = 0; k < rows; ++k) s += JA[k * wa + i] * JB[k * wb + j];
        const int ra = offA + i, cb = offB + j;
        if (ra > cb) atomicAdd(&H[SIDX(d, ra, cb)], s); else atomicAdd(&H[SIDX(d, cb, ra)], s);
    }
}
__device__ __forceinline__ void add_diag(double* H, double* g, const BaDev& d, int off, const double* J, int w, int rows, const double* r) {
    for (int i = 0; i < w; ++i) {
        double gi = 0; for (int k = 0; k < rows; ++k) gi += J[k * w + i] * r[k];
        atomicAdd(&g[off + i], gi);
        for (int j = 0; j <= i; ++j) {
            double s = 0; for (int k = 0; k < rows; ++k) s += J[k * w + i] * J[k * w + j];
            atomicAdd(&H[SIDX(d, off + i, off + j)], s);
        }
    }
}

__device__ __forceinline__ ImuConst load_imu_const(const double* c) {
    ImuConst k;
    k.dp = v3(c[0], c[1], c[2]); k.dq = q4(c[3], c[4], c[5], c[6]); k.dv = v3(c[7], c[8], c[9]);
    k.lin_ba = v3(c[10], c[11], c[12]); k.lin_bg = v3(c[13], c[14], c[15]); k.sum_dt = c[16];
    const double* m = c + 17;
    for (int i = 0; i < 9; ++i) { k.dp_dba.m[i] = m[i]; k.dp_dbg.m[i] = m[9 + i]; k.dq_dbg.m[i] = m[18 + i]; k.dv_dba.m[i] = m[27 + i]; k.dv_dbg.m[i] = m[36 + i]; }
    return k;
}

// ------------------------------------------------------------------ IMU prepare (once per finalize)
// raw 467 -> packed 287 (scalars, five sub-blocks, U); status[f] != 0 when the covariance is singular or a pivot is NaN
// One warp per factor.  Same arithmetic per element as lvb_math.cuh::sqrt_information (partial-pivot LU inverse, then
// Cholesky; the oracle's order), with the independent elements of every step spread over the lanes.
__global__ void __launch_bounds__(128) imu_prepare_kernel(const double* raw, double* packed, int n, int* status) {
    __shared__ double s_work[4][450];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int f = blockIdx.x * 4 + warp;
    if (f >= n) return;
    const double* c = raw + (size_t)f * IMU_RAW;
    double* o = packed + (size_t)f * IMU_STRIDE;
    if (lane < 17) o[lane] = c[lane];
    const double* jac = c + 17;
    for (int e = lane; e < 45; e += 32) {
        const int br[5] = {0, 0, 3, 6, 6}, bc[5] = {9, 12, 12, 9, 12};
        const int b = e / 9, i = (e % 9) / 3, j = e % 3;
        o[17 + e] = jac[(br[b] + i) * 15 + bc[b] + j];
    }
    const int st = sqrt_information_warp(c + 242, o + 62, s_work[warp], s_work[warp] + 225, c[467], c[468]);
    if (lane == 0) { status[f] = st; o[287] = (c[467] >= 0.0 && c[468] >= 0.0) ? 1.0 : 0.0; }     // ImuInitError variant
}

// ------------------------------------------------------------------ K1 eval kernels (parity / roofline)
// TwoFrame: 308 algorithmic bytes per block (40 const + 12 idx + 16 r + 240 J); output staged through
// shared memory so that the 240 B Jacobian record leaves the SM as full 128 B lines.
template <int STAGE, int MINB>
__global__ void __launch_bounds__(TPB, MINB) ba_eval_two_frame_kernel(BaDev d, double* __restrict__ r_out, double* __restrict__ J_out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* s_J = reinterpret_cast<double*>(smem_raw);          // TPB x 31 (STAGE) -- the 240 B record leaves the SM as full lines
    double* s_poses = s_J + (STAGE ? TPB * 31 : 0);              // TPB*31*8 = 31744 B, a multiple of 16
    __shared__ __align__(8) uint64_t bar;
    const double* poses = stage_poses(d, d.poses, s_poses, &bar);
    const int n = d.n[0];
    const int f = blockIdx.x * TPB + threadIdx.x;
    if (f < n) {
        const double* c = d.fc[0];
        const int* ix = d.fi[0];
        const double fo_x = c[f], fo_y = c[n + f], ob_x = c[2 * n + f], ob_y = c[3 * n + f], w = c[4 * n + f];
        const int il = ix[f], i1 = ix[n + f], i2 = ix[2 * n + f];
        TwoFrameLin o; UQ u1, u2;
        two_frame_lin(d.cams, fo_x, fo_y, ob_x, ob_y, w, d.rho[il], poses + 7 * i1, poses + 7 * i2, o, &u1, &u2);
        if (r_out) reinterpret_cast<double2*>(r_out)[f] = make_double2(o.r[0], o.r[1]);
        if (STAGE) {
            double* row = s_J + threadIdx.x * 31;
            row[0] = o.Jrho[0]; row[15] = o.Jrho[1];
            pose_block_to_ambient(u1, o.J1, 2, row + 1, 15);
            pose_block_to_ambient(u2, o.J2, 2, row + 8, 15);
        } else if (J_out) {
            double row[30];
            row[0] = o.Jrho[0]; row[15] = o.Jrho[1];
            pose_block_to_ambient(u1, o.J1, 2, row + 1, 15);
            pose_block_to_ambient(u2, o.J2, 2, row + 8, 15);
            double2* out = reinterpret_cast<double2*>(J_out + (size_t)f * 30);
#pragma unroll
            for (int k = 0; k < 15; ++k) out[k] = make_double2(row[2 * k], row[2 * k + 1]);
        }
    }
    if (STAGE) {
        __syncthreads();
        if (J_out) {
            const int first = blockIdx.x * TPB;
            const int cnt = min(TPB, n - first) * 15;                // double2 elements
            double2* out = reinterpret_cast<double2*>(J_out + (size_t)first * 30);
            for (int e = threadIdx.x; e < cnt; e += TPB) {
                const int t = e / 15, k = (e - t * 15) * 2;
                out[e] = make_double2(s_J[t * 31 + k], s_J[t * 31 + k + 1]);
            }
        }
    }
}

__global__ void __launch_bounds__(TPB) ba_eval_pose_only_kernel(BaDev d, double* __restrict__ r_out, double* __restrict__ J_out) {
    const int n = d.n[1];
    const int f = blockIdx.x * TPB + threadIdx.x;
    if (f >= n) return;
    const double* c = d.fc[1];
    const int ip = d.fi[1][f];
    PoseOnlyLin o; UQ u;
    pose_only_lin(d.cams, c[f], c[n + f], v3(c[2 * n + f], c[3 * n + f], c[4 * n + f]), c[5 * n + f], d.poses + 7 * ip, o, &u);
    if (r_out) { r_out[2 * f] = o.r[0]; r_out[2 * f + 1] = o.r[1]; }
    if (J_out) { double Ja[14]; pose_block_to_ambient(u, o.J, 2, Ja, 7); for (int k = 0; k < 14; ++k) J_out[(size_t)f * 14 + k] = Ja[k]; }
}

__global__ void __launch_bounds__(TPB) ba_eval_two_camera_kernel(BaDev d, double* __restrict__ r_out, double* __restrict__ J_out) {
    const int n = d.n[2];
    const int f = blockIdx.x * TPB + threadIdx.x;
    if (f >= n) return;
    const double* c = d.fc[2];
    TwoCameraLin o;
    two_camera_lin(d.cams, c[f], c[n + f], c[2 * n + f], c[3 * n + f], c[4 * n + f], d.rho[d.fi[2][f]], o);
    if (r_out) { r_out[2 * f] = o.r[0]; r_out[2 * f + 1] = o.r[1]; }
    if (J_out) { J_out[2 * f] = o.Jrho[0]; J_out[2 * f + 1] = o.Jrho[1]; }
}

// IMU: one warp per factor.  Fills s_r (whitened residual, 15) and s_Jw (whitened ambient Jacobian 15x32).
__device__ void imu_warp_eval(const BaDev& d, int f, const double* P, const double* V, double* s_raw /*480*/, double* s_Jw /*480*/, double* s_r /*32: raw 0..14, whitened 16..30*/, bool with_jac = true) {
    const int lane = threadIdx.x & 31;
    const double* c = d.fc[3] + (size_t)f * IMU_STRIDE;
    const int n = d.n[3];
    const int* ix = d.fi[3];
    for (int e = lane; e < 480; e += 32) s_raw[e] = 0.0;
    __syncwarp();
    if (lane < 9) {   // lanes 0..7: one Jacobian block each (disjoint columns), lane 8: the residual
        const ImuConst k = load_imu_const(c);
        const double* Ti = P + 7 * ix[f]; const double* Vi = V + 3 * ix[n + f]; const double* Bai = V + 3 * ix[2 * n + f]; const double* Bgi = V + 3 * ix[3 * n + f];
        const double zero3[3] = {0.0, 0.0, 0.0};         // ImuInitError: Baj = Bgj = 0 (imu_error.hpp:141-142), idx = -1
        const int i6 = ix[6 * n + f], i7 = ix[7 * n + f];
        const double* Tj = P + 7 * ix[4 * n + f]; const double* Vj = V + 3 * ix[5 * n + f]; const double* Baj = i6 < 0 ? zero3 : V + 3 * i6; const double* Bgj = i7 < 0 ? zero3 : V + 3 * i7;
        if (lane == 8) imu_raw_residual(k, Ti, Vi, Bai, Bgi, Tj, Vj, Baj, Bgj, s_r);
        else if (with_jac && !(lane >= 6 && c[287] != 0.0)) imu_raw_jacobian_block(k, lane, Ti, Vi, Bgi, Tj, Vj, s_raw);
    }
    __syncwarp();
    const double* U = c + 62;
    if (lane < 15) { double s = 0; for (int k = 0; k < 15; ++k) s += U[15 * lane + k] * s_r[k]; s_r[16 + lane] = s; }
    if (with_jac) for (int e = lane; e < 480; e += 32) {
        const int i = e >> 5, j = e & 31;
        double s = 0; for (int k = i; k < 15; ++k) s += U[15 * i + k] * s_raw[32 * k + j];     // U is upper triangular
        s_Jw[e] = s;
    }
    __syncwarp();
}

__global__ void __launch_bounds__(TPB) ba_eval_imu_kernel(BaDev d, double* __restrict__ r_out, double* __restrict__ J_out) {
    __shared__ double s_raw[4][480], s_Jw[4][480], s_r[4][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int f = blockIdx.x * 4 + warp;
    if (f >= d.n[3]) return;
    imu_warp_eval(d, f, d.poses, d.vec3, s_raw[warp], s_Jw[warp], s_r[warp]);
    if (r_out && lane < 15) r_out[(size_t)f * 15 + lane] = s_r[warp][16 + lane];
    if (J_out) for (int e = lane; e < 480; e += 32) J_out[(size_t)f * 480 + e] = s_Jw[warp][e];
}

__global__ void ba_eval_prior_kernel(BaDev d, int kind, double* __restrict__ r_out, double* __restrict__ J_out) {
    const int n = d.n[kind];
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    const int stride = kind == 4 ? 8 : 9;
    double c[9];
    for (int k = 0; k < stride; ++k) c[k] = d.fc[kind][(size_t)k * n + f];
    double r[6], J[84];
    if (kind == 4) pose_graph_eval(c, d.poses + 7 * d.fi[4][f], d.poses + 7 * d.fi[4][n + f], r, J);
    else pose_prior_eval(c, d.poses + 7 * d.fi[5][f], r, J);
    const int cols = kind == 4 ? 14 : 7;
    if (r_out) for (int k = 0; k < 6; ++k) r_out[(size_t)f * 6 + k] = r[k];
    if (J_out) for (int k = 0; k < 6 * cols; ++k) J_out[(size_t)f * 6 * cols + k] = J[k];
}

// ------------------------------------------------------------------ fused linearize / cost kernel
// MODE 0: at x      -> Hpp, gc, Hll, gl, tf_w, st->cost_acc      (skipped unless st->need_linearize)
// MODE 1: at cand   -> st->cand_cost_acc only
// Warp-level SYRK: the 32 blocks of a warp share their pose key (finalize() sorts and pads), so the warp
// writes its Jacobian rows [2 x ncol per lane] to shared memory, each lane then owns a few entries of the
// lower triangle of A^T A (A = [J_1 | J_2 | r] or [J | r]) and issues ONE red.global per entry instead of 32.
__device__ __forceinline__ void warp_syrk_flush(const BaDev& d, const double* A /*64 x SYRK_LD*/, int ncol, int off1, int off2) {
    const int lane = threadIdx.x & 31;
    const int nent = ncol * (ncol + 1) / 2;
    for (int e = lane; e < nent; e += 32) {
        const int a = c_tri_a[e], b = c_tri_b[e];                 // a >= b, both < ncol <= 13
        if (a == ncol - 1 && b == ncol - 1) continue;             // r.r : the cost goes through block_add
        double v = 0.0;
#pragma unroll 8
        for (int r = 0; r < SYRK_ROWS; ++r) v += A[r * SYRK_LD + a] * A[r * SYRK_LD + b];
        if (v == 0.0) continue;
        const int gb = (ncol == 13) ? (b < 6 ? (off1 < 0 ? -1 : off1 + b) : (off2 < 0 ? -1 : off2 + b - 6)) : (off1 < 0 ? -1 : off1 + b);
        if (gb < 0) continue;
        if (a == ncol - 1) { atomicAdd(&d.gc[gb], v); continue; }
        const int ga = (ncol == 13) ? (a < 6 ? (off1 < 0 ? -1 : off1 + a) : (off2 < 0 ? -1 : off2 + a - 6)) : (off1 < 0 ? -1 : off1 + a);
        if (ga < 0) continue;
        if (ga >= gb) atomicAdd(&d.Hpp[SIDX(d, ga, gb)], v); else atomicAdd(&d.Hpp[SIDX(d, gb, ga)], v);
    }
}

template <int MODE>
__device__ __forceinline__ void linearize_visual_body(const BaDev& d, const BlockRanges& R, const int b) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t bar;
    __shared__ double s_red[TPB / 32];
    const LmState* st = d.st;
    if (st->done) return;
    if (MODE == 0 && !st->need_linearize) return;
    const double* Psrc = MODE == 0 ? d.poses : d.c_poses;
    const double* Rho = MODE == 0 ? d.rho : d.c_rho;
    double* cost_target = MODE == 0 ? &d.st->cost_acc : &d.st->cand_cost_acc;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double cost = 0.0;
    const size_t pose_bytes = d.stage_poses ? (((size_t)d.n_poses * 56 + 16 + 15) & ~(size_t)15) : 0;
    double* A = reinterpret_cast<double*>(smem_raw + pose_bytes) + (size_t)warp * SYRK_ROWS * SYRK_LD;
    const double* P = stage_poses(d, Psrc, reinterpret_cast<double*>(smem_raw), &bar);
    if (b < R.b[1]) {            // ---- a1 TwoFrameReprojectionError
        const int n = d.n[0];
        const int f = (b - R.b[0]) * TPB + threadIdx.x;
        const bool valid = f < n;
        const double* c = d.fc[0]; const int* ix = d.fi[0];
        int il = 0, i1 = -1, i2 = -1, off1 = -1, off2 = -1;
        TwoFrameLin o;
        bool lfree = false;
        if (valid) {
            il = ix[f]; i1 = ix[n + f]; i2 = ix[2 * n + f];
            two_frame_lin(d.cams, c[f], c[n + f], c[2 * n + f], c[3 * n + f], c[4 * n + f], Rho[il], P + 7 * i1, P + 7 * i2, o, nullptr, nullptr);
            double rho_v, sr;
            huber(d.huber[0], o.r[0] * o.r[0] + o.r[1] * o.r[1], &rho_v, &sr);
            cost = 0.5 * rho_v;
            if (MODE == 0) {
                o.r[0] *= sr; o.r[1] *= sr; o.Jrho[0] *= sr; o.Jrho[1] *= sr;
                for (int k = 0; k < 12; ++k) { o.J1[k] *= sr; o.J2[k] *= sr; }
                off1 = d.pose_off[i1]; off2 = d.pose_off[i2];
                if (i1 == i2) { for (int k = 0; k < 12; ++k) o.J1[k] += o.J2[k]; off2 = -1; }
                lfree = d.rho_slot[il] >= 0;
                double* w = d.tf_w;
                if (lfree) {
                    const double h = o.Jrho[0] * o.Jrho[0] + o.Jrho[1] * o.Jrho[1], g = o.Jrho[0] * o.r[0] + o.Jrho[1] * o.r[1];
                    if (h != 0.0) atomicAdd(&d.Hll[il], h);
                    if (g != 0.0) atomicAdd(&d.gl[il], g);
                }
                // coupling rows W = J_rho^T [J_1 | J_2], one 96-byte record per factor (the Schur and back-substitution kernels gather
                // them per landmark: a record is 3 sectors, the former 12 planes were 12)
                double wv[12];
                for (int k = 0; k < 6; ++k) {
                    wv[k] = (lfree && off1 >= 0) ? o.Jrho[0] * o.J1[k] + o.Jrho[1] * o.J1[6 + k] : 0.0;
                    wv[6 + k] = (lfree && off2 >= 0) ? o.Jrho[0] * o.J2[k] + o.Jrho[1] * o.J2[6 + k] : 0.0;
                }
                double2* wr = reinterpret_cast<double2*>(w + (size_t)f * 12);
#pragma unroll
                for (int k = 0; k < 6; ++k) wr[k] = make_double2(wv[2 * k], wv[2 * k + 1]);
            }
        }
        if (MODE == 0) {
            // blocks are sorted by (pose_1, pose_2): a warp holds one key (padded layout) or a few key segments
            unsigned todo = d.warp_syrk ? __ballot_sync(0xffffffffu, valid && i1 != i2) : 0u;
            const bool direct = valid && (!d.warp_syrk || i1 == i2);
            while (todo) {
                const int leader = __ffs(todo) - 1;
                const int k1 = __shfl_sync(0xffffffffu, i1, leader), k2 = __shfl_sync(0xffffffffu, i2, leader);
                const int o1 = __shfl_sync(0xffffffffu, off1, leader), o2 = __shfl_sync(0xffffffffu, off2, leader);
                const bool mine = valid && i1 == k1 && i2 == k2;
                double* row0 = A + (2 * lane) * SYRK_LD; double* row1 = row0 + SYRK_LD;
                if (mine) {
                    for (int k = 0; k < 6; ++k) { row0[k] = o.J1[k]; row1[k] = o.J1[6 + k]; row0[6 + k] = o.J2[k]; row1[6 + k] = o.J2[6 + k]; }
                    row0[12] = o.r[0]; row1[12] = o.r[1];
                } else for (int k = 0; k < 13; ++k) { row0[k] = 0.0; row1[k] = 0.0; }
                __syncwarp();
                warp_syrk_flush(d, A, 13, o1, o2);
                __syncwarp();
                todo &= ~__ballot_sync(0xffffffffu, mine);
            }
            if (direct) {
                if (off1 >= 0) add_diag(d.Hpp, d.gc, d, off1, o.J1, 6, 2, o.r);
                if (off2 >= 0) add_diag(d.Hpp, d.gc, d, off2, o.J2, 6, 2, o.r);
                if (off1 >= 0 && off2 >= 0) add_cross(d.Hpp, d, off1, o.J1, 6, off2, o.J2, 6, 2);
            }
        }
    } else if (b < R.b[2]) {     // ---- a2 PoseOnlyReprojectionError
        const int n = d.n[1];
        const int f = (b - R.b[1]) * TPB + threadIdx.x;
        const bool valid = f < n;
        const double* c = d.fc[1];
        int ip = -1, off = -1;
        PoseOnlyLin o;
        if (valid) {
            ip = d.fi[1][f];
            pose_only_lin(d.cams, c[f], c[n + f], v3(c[2 * n + f], c[3 * n + f], c[4 * n + f]), c[5 * n + f], P + 7 * ip, o, nullptr);
            double rho_v, sr;
            huber(d.huber[1], o.r[0] * o.r[0] + o.r[1] * o.r[1], &rho_v, &sr);
            cost = 0.5 * rho_v;
            if (MODE == 0) { off = d.pose_off[ip]; o.r[0] *= sr; o.r[1] *= sr; for (int k = 0; k < 12; ++k) o.J[k] *= sr; }
        }
        if (MODE == 0) {
            unsigned todo = d.warp_syrk ? __ballot_sync(0xffffffffu, valid) : 0u;
            while (todo) {
                const int leader = __ffs(todo) - 1;
                const int k1 = __shfl_sync(0xffffffffu, ip, leader), o1 = __shfl_sync(0xffffffffu, off, leader);
                const bool mine = valid && ip == k1;
                double* row0 = A + (2 * lane) * SYRK_LD; double* row1 = row0 + SYRK_LD;
                if (mine) {
                    for (int k = 0; k < 6; ++k) { row0[k] = o.J[k]; row1[k] = o.J[6 + k]; }
                    row0[6] = o.r[0]; row1[6] = o.r[1];
                } else for (int k = 0; k < 7; ++k) { row0[k] = 0.0; row1[k] = 0.0; }
                __syncwarp();
                warp_syrk_flush(d, A, 7, o1, -1);
                __syncwarp();
                todo &= ~__ballot_sync(0xffffffffu, mine);
            }
            if (!d.warp_syrk && valid && off >= 0) add_diag(d.Hpp, d.gc, d, off, o.J, 6, 2, o.r);
        }
    } else {                     // ---- a3 TwoCameraReprojectionError
        const int n = d.n[2];
        const int f = (b - R.b[2]) * TPB + threadIdx.x;
        if (f < n) {
            const double* c = d.fc[2];
            const int il = d.fi[2][f];
            TwoCameraLin o;
            two_camera_lin(d.cams, c[f], c[n + f], c[2 * n + f], c[3 * n + f], c[4 * n + f], Rho[il], o);
            double rho_v, sr;
            huber(d.huber[2], o.r[0] * o.r[0] + o.r[1] * o.r[1], &rho_v, &sr);
            cost = 0.5 * rho_v;
            if (MODE == 0 && d.rho_slot[il] >= 0) {
                const double j0 = o.Jrho[0] * sr, j1 = o.Jrho[1] * sr;
                atomicAdd(&d.Hll[il], j0 * j0 + j1 * j1);
                atomicAdd(&d.gl[il], j0 * o.r[0] * sr + j1 * o.r[1] * sr);
            }
        }
    }
    block_add(cost, cost_target, s_red);
}

template <int MODE>
__global__ void __launch_bounds__(TPB) ba_linearize_kernel(BaDev d, BlockRanges R) { linearize_visual_body<MODE>(d, R, blockIdx.x); }

// IMU (one warp per factor) and the two prior kinds: rare, register-hungry blocks kept out of the visual kernel at map scale
template <int MODE>
__device__ __forceinline__ void linearize_other_body(const BaDev& d, const BlockRanges& R, const int b /* absolute block index >= R.b[3] */) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ double s_red[TPB / 32];
    const LmState* st = d.st;
    if (st->done) return;
    if (MODE == 0 && !st->need_linearize) return;
    const double* Psrc = MODE == 0 ? d.poses : d.c_poses;
    const double* V = MODE == 0 ? d.vec3 : d.c_vec3;
    double* cost_target = MODE == 0 ? &d.st->cost_acc : &d.st->cand_cost_acc;
    double cost = 0.0;
    if (b < R.b[4] && d.imu_cta) {   // ---- IMU, window size: one CTA (4 warps) per factor
        // The eight Jacobian blocks and the residual are nine different scalar programs: as nine lanes of one warp they ran one
        // after the other (divergence), which made this factor kind a ~15 us single-warp chain.  Here they are spread over the four
        // warps (lane 0 each, heavy blocks on different warps), the constants and U come from shared memory, and the whitening and
        // the J^T J accumulation use all 128 threads.
        double* s_raw = reinterpret_cast<double*>(smem_raw);     // 480: raw ambient Jacobian 15 x 32, later the tangent Jacobian 15 x 30
        double* s_Jw = s_raw + 480;                              // 480: whitened ambient Jacobian
        double* s_r = s_Jw + 480;                                // 32 : raw residual 0..14, whitened 16..30
        double* s_c = s_r + 32;                                  // 288: the factor's constants (17 scalars, five 3x3 blocks, U, init flag)
        int* s_gidx = reinterpret_cast<int*>(s_c + IMU_STRIDE);  // 32
        const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
        const int f = b - R.b[3];
        const int n = d.n[3];
        const int* ix = d.fi[3];
        {
            const double* c = d.fc[3] + (size_t)f * IMU_STRIDE;
            for (int e = tid; e < IMU_STRIDE; e += TPB) s_c[e] = c[e];
            for (int e = tid; e < 480; e += TPB) s_raw[e] = 0.0;
        }
        __syncthreads();
        if (lane == 0) {
            const ImuConst k = load_imu_const(s_c);
            const double* Ti = Psrc + 7 * ix[f]; const double* Vi = V + 3 * ix[n + f]; const double* Bai = V + 3 * ix[2 * n + f]; const double* Bgi = V + 3 * ix[3 * n + f];
            const double zero3[3] = {0.0, 0.0, 0.0};         // ImuInitError: Baj = Bgj = 0 (imu_error.hpp:141-142), idx = -1
            const int i6 = ix[6 * n + f], i7 = ix[7 * n + f];
            const double* Tj = Psrc + 7 * ix[4 * n + f]; const double* Vj = V + 3 * ix[5 * n + f]; const double* Baj = i6 < 0 ? zero3 : V + 3 * i6; const double* Bgj = i7 < 0 ? zero3 : V + 3 * i7;
            // tasks 0..7 = Jacobian blocks (pose_i v_i ba_i bg_i pose_j v_j ba_j bg_j), 8 = residual; heavy ones: 0, 3, 4, 8
            const int tasks[4][3] = {{0, -1, -1}, {3, 1, 5}, {4, 2, 6}, {8, 7, -1}};
            for (int t = 0; t < 3; ++t) {
                const int task = tasks[warp][t];
                if (task < 0) continue;
                if (task == 8) imu_raw_residual(k, Ti, Vi, Bai, Bgi, Tj, Vj, Baj, Bgj, s_r);
                else if (MODE == 0 && !(task >= 6 && s_c[287] != 0.0)) imu_raw_jacobian_block(k, task, Ti, Vi, Bgi, Tj, Vj, s_raw);
            }
        }
        __syncthreads();
        const double* U = s_c + 62;
        if (tid < 15) { double sacc = 0; for (int k = 0; k < 15; ++k) sacc += U[15 * tid + k] * s_r[k]; s_r[16 + tid] = sacc; }
        if (MODE == 0) for (int e = tid; e < 480; e += TPB) {
            const int i = e >> 5, j = e & 31;
            double sacc = 0; for (int k = i; k < 15; ++k) sacc += U[15 * i + k] * s_raw[32 * k + j];     // U is upper triangular
            s_Jw[e] = sacc;
        }
        __syncthreads();
        double s = 0.0;
        for (int i = 0; i < 15; ++i) s += s_r[16 + i] * s_r[16 + i];
        double rho_v, sr;
        huber(d.huber[3], s, &rho_v, &sr);
        if (tid == 0) cost = 0.5 * rho_v;
        if (MODE == 0) {
            // tangent Jacobian Jt[15][30] into s_raw (cols: pose_i 6 | v ba bg 9 | pose_j 6 | v ba bg 9)
            __syncthreads();                                      // every thread has read the whitened residual
            if (tid < 15) {
                const double* a = s_Jw + 32 * tid;
                double* t = s_raw + 30 * tid;
                double t6[6];
                ambient_row_to_tangent(Psrc + 7 * ix[f], a, t6);
                for (int k = 0; k < 6; ++k) t[k] = t6[k] * sr;
                for (int k = 0; k < 9; ++k) t[6 + k] = a[7 + k] * sr;
                ambient_row_to_tangent(Psrc + 7 * ix[4 * n + f], a + 16, t6);
                for (int k = 0; k < 6; ++k) t[15 + k] = t6[k] * sr;
                for (int k = 0; k < 9; ++k) t[21 + k] = a[23 + k] * sr;
                s_r[16 + tid] *= sr;
            } else if (tid >= 32 && tid < 62) {
                const int l = tid - 32;
                int blk, loc;
                if (l < 6) { blk = 0; loc = l; } else if (l < 15) { blk = 1 + (l - 6) / 3; loc = (l - 6) % 3; }
                else if (l < 21) { blk = 4; loc = l - 15; } else { blk = 5 + (l - 21) / 3; loc = (l - 21) % 3; }
                const int id = ix[(size_t)blk * n + f];
                const int off = id < 0 ? -1 : ((blk == 0 || blk == 4) ? d.pose_off[id] : d.vec3_off[id]);
                s_gidx[l] = off < 0 ? -1 : off + loc;
            }
            __syncthreads();
            if (tid < 30 && s_gidx[tid] >= 0) {
                double g = 0; for (int i = 0; i < 15; ++i) g += s_raw[30 * i + tid] * s_r[16 + i];
                atomicAdd(&d.gc[s_gidx[tid]], g);
            }
            for (int e = tid; e < 465; e += TPB) {
                const int a = c_tri_a[e], bb = c_tri_b[e];
                const int ga = s_gidx[a], gb = s_gidx[bb];
                if (ga < 0 || gb < 0) continue;
                double h = 0; for (int i = 0; i < 15; ++i) h += s_raw[30 * i + a] * s_raw[30 * i + bb];
                if (ga >= gb) atomicAdd(&d.Hpp[SIDX(d, ga, gb)], h); else atomicAdd(&d.Hpp[SIDX(d, gb, ga)], h);
            }
        }
    } else if (b < R.b[4]) {   // ---- IMU, map scale: one warp per factor, four factors per CTA (throughput: thousands of factors)
        double* s_raw = reinterpret_cast<double*>(smem_raw);     // 4 x 480
        double* s_Jw = s_raw + 4 * 480;                          // 4 x 480
        double* s_r = s_Jw + 4 * 480;                            // 4 x 32
        int* s_gidx = reinterpret_cast<int*>(s_r + 4 * 32);      // 4 x 32
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const int f = (b - R.b[3]) * 4 + warp;
        const int n = d.n[3];
        if (f < n) {
            double* raw = s_raw + warp * 480; double* Jw = s_Jw + warp * 480; double* rr = s_r + warp * 32; int* gidx = s_gidx + warp * 32;
            imu_warp_eval(d, f, Psrc, V, raw, Jw, rr, MODE == 0);
            double s = (lane < 15) ? rr[16 + lane] * rr[16 + lane] : 0.0;
            s = warp_sum(s);
            double rho_v, sr;
            huber(d.huber[3], s, &rho_v, &sr);
            if (lane == 0) cost = 0.5 * rho_v;
            if (MODE == 0) {
                const int* ix = d.fi[3];
                // tangent Jacobian Jt[15][30] into `raw` (cols: pose_i 6 | v ba bg 9 | pose_j 6 | v ba bg 9)
                if (lane < 15) {
                    const double* a = Jw + 32 * lane;
                    double* t = raw + 30 * lane;
                    double t6[6];
                    ambient_row_to_tangent(Psrc + 7 * ix[f], a, t6);
                    for (int k = 0; k < 6; ++k) t[k] = t6[k] * sr;
                    for (int k = 0; k < 9; ++k) t[6 + k] = a[7 + k] * sr;
                    ambient_row_to_tangent(Psrc + 7 * ix[4 * n + f], a + 16, t6);
                    for (int k = 0; k < 6; ++k) t[15 + k] = t6[k] * sr;
                    for (int k = 0; k < 9; ++k) t[21 + k] = a[23 + k] * sr;
                    rr[16 + lane] *= sr;
                }
                if (lane < 30) {
                    int blk, loc;
                    if (lane < 6) { blk = 0; loc = lane; } else if (lane < 15) { blk = 1 + (lane - 6) / 3; loc = (lane - 6) % 3; }
                    else if (lane < 21) { blk = 4; loc = lane - 15; } else { blk = 5 + (lane - 21) / 3; loc = (lane - 21) % 3; }
                    const int id = ix[(size_t)blk * n + f];
                    const int off = id < 0 ? -1 : ((blk == 0 || blk == 4) ? d.pose_off[id] : d.vec3_off[id]);
                    gidx[lane] = off < 0 ? -1 : off + loc;
                }
                __syncwarp();
                if (lane < 30 && gidx[lane] >= 0) {
                    double g = 0; for (int i = 0; i < 15; ++i) g += raw[30 * i + lane] * rr[16 + i];
                    atomicAdd(&d.gc[gidx[lane]], g);
                }
                for (int e = lane; e < 465; e += 32) {
                    const int a = c_tri_a[e], bb = c_tri_b[e];
                    const int ga = gidx[a], gb = gidx[bb];
                    if (ga < 0 || gb < 0) continue;
                    double h = 0; for (int i = 0; i < 15; ++i) h += raw[30 * i + a] * raw[30 * i + bb];
                    if (ga >= gb) atomicAdd(&d.Hpp[SIDX(d, ga, gb)], h); else atomicAdd(&d.Hpp[SIDX(d, gb, ga)], h);
                }
            }
        }
    } else {   // ---- PoseGraphError / PoseError priors: one thread per block
        const int kind = b < R.b[5] ? 4 : 5;
        const int n = d.n[kind];
        const int f = (b - R.b[kind]) * TPB + threadIdx.x;
        if (f < n) {
            const int stride = kind == 4 ? 8 : 9;
            double c[9];
            for (int k = 0; k < stride; ++k) c[k] = d.fc[kind][(size_t)k * n + f];
            double r[6], J[84];
            const int i1 = d.fi[kind][f];
            const int i2 = kind == 4 ? d.fi[kind][n + f] : -1;
            if (kind == 4) pose_graph_eval(c, Psrc + 7 * i1, Psrc + 7 * i2, r, MODE == 0 ? J : nullptr);
            else pose_prior_eval(c, Psrc + 7 * i1, r, MODE == 0 ? J : nullptr);
            double s = 0; for (int k = 0; k < 6; ++k) s += r[k] * r[k];
            double rho_v, sr;
            huber(d.huber[kind], s, &rho_v, &sr);
            cost = 0.5 * rho_v;
            if (MODE == 0) {
                const int cols = kind == 4 ? 14 : 7;
                double J1[36], J2[36];
                for (int k = 0; k < 36; ++k) J2[k] = 0.0;
                for (int k = 0; k < 6; ++k) {
                    r[k] *= sr;
                    ambient_row_to_tangent(Psrc + 7 * i1, J + cols * k, J1 + 6 * k);
                    if (kind == 4) ambient_row_to_tangent(Psrc + 7 * i2, J + cols * k + 7, J2 + 6 * k);
                }
                for (int k = 0; k < 36; ++k) { J1[k] *= sr; J2[k] *= sr; }
                const int off1 = d.pose_off[i1], off2 = kind == 4 ? d.pose_off[i2] : -1;
                if (off1 >= 0) add_diag(d.Hpp, d.gc, d, off1, J1, 6, 6, r);
                if (off2 >= 0) add_diag(d.Hpp, d.gc, d, off2, J2, 6, 6, r);
                if (off1 >= 0 && off2 >= 0 && off1 != off2) add_cross(d.Hpp, d, off1, J1, 6, off2, J2, 6, 6);
            }
        }
    }
    block_add(cost, cost_target, s_red);
}

template <int MODE>
__global__ void __launch_bounds__(TPB) ba_linearize_other_kernel(BaDev d, BlockRanges R) { linearize_other_body<MODE>(d, R, blockIdx.x + R.b[3]); }

// Window-sized problems: ONE launch for all factor kinds.  The IMU blocks are a long single-warp dependency chain (~20 us) and the
// visual blocks a short wide one; in one grid -- IMU and priors first so they start at once -- they overlap instead of running
// back to back, and a launch is saved.  (At map scale the visual kernel's occupancy matters and the kernels stay separate.)
template <int MODE>
__global__ void __launch_bounds__(TPB) ba_linearize_all_kernel(BaDev d, BlockRanges R) {
    const int n_other = R.b[6] - R.b[3];
    if ((int)blockIdx.x < n_other) linearize_other_body<MODE>(d, R, (int)blockIdx.x + R.b[3]);
    else linearize_visual_body<MODE>(d, R, (int)blockIdx.x - n_other);
}

// ------------------------------------------------------------------ per-iteration system assembly
__global__ void ba_zero_kernel(BaDev d) {
    const LmState* st = d.st;
    if (st->done || !st->need_linearize) return;
    const size_t nH = d.nS;
    const size_t total = nH + d.dimc + 2 * (size_t)d.n_rho;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        if (i < nH) d.Hpp[i] = 0.0;
        else if (i < nH + d.dimc) d.gc[i - nH] = 0.0;
        else if (i < nH + d.dimc + d.n_rho) d.Hll[i - nH - d.dimc] = 0.0;
        else d.gl[i - nH - d.dimc - d.n_rho] = 0.0;
    }
}

__device__ __forceinline__ void atomic_max_nonneg(unsigned long long* p, double v) {
    if (v == v) atomicMax(p, (unsigned long long)__double_as_longlong(fabs(v)));
    else atomicMax(p, 0x7ff0000000000000ull);   // NaN -> +inf so the tolerance test fails
}


// K5: eliminate the inverse depths.  One warp per 32 landmarks that share their set of pose offsets
// (finalize() groups and pads them).  Lane l writes u_l = sqrt(1/h_l) [w_l | g_l] (its couplings merged by
// pose slot) as a row of a shared-memory tile; the warp then forms the lower triangle of U^T U and subtracts
// it from S / adds the last column to rhs with one red.global per entry:  S -= sum_l w_l^T w_l / h_l.
__global__ void __launch_bounds__(TPB) ba_schur_kernel(BaDev d, int cols_max) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    if (d.st->done) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int w = blockIdx.x * (TPB / 32) + warp;
    if (w >= d.n_schur_warps) return;
    const int g = d.sw_group[w];
    const int ns = d.grp_ns[g];
    const int ncol = 6 * ns + 1;
    double* U = reinterpret_cast<double*>(smem_raw) + (size_t)warp * 32 * cols_max;
    double* row = U + (size_t)lane * ncol;
    for (int k = 0; k < ncol; ++k) row[k] = 0.0;
    const int l = d.sw_lm[(size_t)w * 32 + lane];
    unsigned long long gmax_bits = 0ull;          // |gradient| of this lane's inverse depth as ordered bits (NaN -> +inf)
    if (l >= 0) {
        // Jacobi scale (first pass), LM damping and gradient max-norm of this inverse depth
        LmState* st = d.st;
        const double h = d.Hll[l];
        if (!st->scale_valid) d.scale_l[l] = st->jacobi ? 1.0 / (1.0 + sqrt(h)) : 1.0;
        const double sc = d.scale_l[l], sc2 = sc * sc;
        const double lam = fmin(fmax(sc2 * h, st->min_diag), st->max_diag) / (st->radius * sc2);
        d.lam_l[l] = lam;
        if (st->need_linearize && d.lm_start[l + 1] > d.lm_start[l]) { const double gv = d.gl[l]; gmax_bits = (gv == gv) ? (unsigned long long)__double_as_longlong(fabs(gv)) : 0x7ff0000000000000ull; }
        const double hl = h + lam;
        if (hl > 0.0 && ns > 0) {
            const int n = d.n[0];
            // gather the landmark's coupling records four factors at a time: all index loads of a batch are issued before the first
            // use (factor id -> slots -> 96-byte record is a chain of three dependent round trips; one factor at a time made this
            // kernel L2-latency bound, 35 long-scoreboard stall cycles per issue at map scale)
            const int e1 = d.lm_start[l + 1];
            for (int eb = d.lm_start[l]; eb < e1; eb += 4) {
                int f[4], s0[4], s1[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) f[u] = (eb + u < e1) ? d.lm_fac[eb + u] : -1;
#pragma unroll
                for (int u = 0; u < 4; ++u) { const int fc = max(f[u], 0); s0[u] = d.tf_slot[fc]; s1[u] = d.tf_slot[(size_t)n + fc]; }      // unconditional (clamped) loads: no branches between them
                double2 w[4][6];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const double2* src = reinterpret_cast<const double2*>(d.tf_w + (size_t)max(f[u], 0) * 12);
#pragma unroll
                    for (int k = 0; k < 6; ++k) w[u][k] = src[k];
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    if (f[u] < 0) continue;
                    if (s0[u] >= 0) { double* t = row + 6 * s0[u]; t[0] += w[u][0].x; t[1] += w[u][0].y; t[2] += w[u][1].x; t[3] += w[u][1].y; t[4] += w[u][2].x; t[5] += w[u][2].y; }
                    if (s1[u] >= 0) { double* t = row + 6 * s1[u]; t[0] += w[u][3].x; t[1] += w[u][3].y; t[2] += w[u][4].x; t[3] += w[u][4].y; t[4] += w[u][5].x; t[5] += w[u][5].y; }
                }
            }
            const double sh = sqrt(1.0 / hl);
            for (int k = 0; k < ncol - 1; ++k) row[k] *= sh;
            row[ncol - 1] = d.gl[l] * sh;
        }
    }
    __syncwarp();
    // one atomicMax per warp, not per landmark: at map scale 500 000 atomics on the one address serialised in L2 (most of the kernel)
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long v = __shfl_xor_sync(0xffffffffu, gmax_bits, o); gmax_bits = v > gmax_bits ? v : gmax_bits; }
    if (lane == 0 && gmax_bits) atomicMax(&d.st->grad_max_bits, gmax_bits);
    const int* offs = d.grp_off + (size_t)g * MAX_TRACK;
    if (d.tc_mode) {
        // tensor-core mode: this warp only (a) adds its rhs column  sum_l u_l g_l / h_l  in FP64 and (b) writes its 32
        // rows of U as three bf16 planes (x ~ hi + mid + lo, 24 mantissa bits) into the K-major wgmma tiles of its two
        // 16-landmark chunks.  Positions outside the group's pose set were zeroed once at finalize and never change.
        for (int b = lane; b < ncol - 1; b += 32) {
            double v = 0.0;
#pragma unroll 8
            for (int r = 0; r < 32; ++r) v += U[r * ncol + ncol - 1] * U[r * ncol + b];
            if (v != 0.0) atomicAdd(&d.rhs[offs[b / 6] + b % 6], v);
        }
        const size_t chunk = (size_t)w * 2 + (lane >> 4);
        const int k = lane & 15;
        unsigned short* tile = d.tc_u + chunk * (3 * 2048);       // 2048 bf16 = 4096 B per split tile
        for (int b = 0; b < ncol - 1; ++b) {
            const int r = d.tc_cdim[offs[b / 6]] + b % 6;         // compact pose dimension of this column
            const double x = row[b];
            const __nv_bfloat16 hi = __float2bfloat16_rn((float)x);
            const double r1 = x - (double)__bfloat162float(hi);
            const __nv_bfloat16 mid = __float2bfloat16_rn((float)r1);
            const double r2 = r1 - (double)__bfloat162float(mid);
            const __nv_bfloat16 lo = __float2bfloat16_rn((float)r2);
            // canonical no-swizzle K-major tile: 8x16B core matrices, SBO = 256 B between 8-row groups, LBO = 128 B
            const int e = (r >> 3) * 128 + (k >> 3) * 64 + (r & 7) * 8 + (k & 7);
            tile[e] = __bfloat16_as_ushort(hi); tile[2048 + e] = __bfloat16_as_ushort(mid); tile[4096 + e] = __bfloat16_as_ushort(lo);
        }
        return;
    }
    const int nent = ncol * (ncol + 1) / 2 - 1;                   // the (v,v) corner is not needed
    for (int e = lane; e < nent; e += 32) {
        int a = (int)((sqrt(8.0 * e + 1.0) - 1.0) * 0.5);
        while ((a + 1) * (a + 2) / 2 <= e) ++a;
        while (a * (a + 1) / 2 > e) --a;
        const int b = e - a * (a + 1) / 2;
        double v = 0.0;
#pragma unroll 8
        for (int r = 0; r < 32; ++r) v += U[r * ncol + a] * U[r * ncol + b];
        if (v == 0.0) continue;
        const int gb = offs[b / 6] + b % 6;
        if (a == ncol - 1) { atomicAdd(&d.rhs[gb], v); continue; }
        const int ga = offs[a / 6] + a % 6;
        if (ga >= gb) atomicAdd(&d.S[SIDX(d, ga, gb)], -v); else atomicAdd(&d.S[SIDX(d, gb, ga)], -v);
    }
}

// K5 on the tensor cores.  S_pose -= U^T U with U^T staged as bf16 split planes (hi, mid, lo); per 16-landmark chunk six
// products (hi.hi, hi.mid, mid.hi, mid.mid, hi.lo, lo.hi) accumulate in FP32 in registers, which keeps ~2^-23 of each
// product.  One warpgroup issues wgmma.m64n128k16 for the two 64-row halves of the 128 x 128 result in turn (64 accumulator
// registers per thread instead of 128); one CTA owns TC_CHUNKS chunks (a 256-landmark slice of K), so the FP32 accumulation
// stays short and the cross-CTA sum happens in FP64 (red.global.add.f64 on the lower triangle).  The FP64 kernel above
// remains the parity reference; this path is selected with lvb_solve_options.schur_mode = 1 when 6 * (free poses) <= 128.
enum { TC_CHUNKS = 16, TC_TILE_BYTES = 4096, TC_CHUNK_BYTES = 3 * TC_TILE_BYTES };

__device__ __forceinline__ uint64_t gmma_smem_desc(uint32_t smem_addr) {
    // sm_90 matrix descriptor: start >> 4 [0,14) | LBO >> 4 [16,30) | SBO >> 4 [32,46) | base offset 0 [49,52) | layout 0 = no
    // swizzle [62,64).  K-major canonical layout ((8,m),2):((1,SBO),LBO) in 16-byte units: LBO = 128 B between the two 8-wide
    // K core matrices, SBO = 256 B between 8-row groups.
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(256 >> 4) << 32);
}
// D[64 x 128] += A[64 x 16] . B[128 x 16]^T, both operands K-major bf16 in shared memory, D in FP32 registers, overwritten when accumulate == 0 (warpgroup layout:
// thread t holds rows 16 (t / 32) + (t % 32) / 4 + {0, 8}, columns 8 n + 2 (t % 4) + {0, 1} in c[4 n + {0, 1}] / c[4 n + {2, 3}])
__device__ __forceinline__ void wgmma_bf16_m64n128(float (&c)[64], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\nwgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]), "+f"(c[4]), "+f"(c[5]), "+f"(c[6]), "+f"(c[7]), "+f"(c[8]), "+f"(c[9]), "+f"(c[10]), "+f"(c[11]), "+f"(c[12]), "+f"(c[13]), "+f"(c[14]), "+f"(c[15]), "+f"(c[16]), "+f"(c[17]), "+f"(c[18]), "+f"(c[19]), "+f"(c[20]), "+f"(c[21]), "+f"(c[22]), "+f"(c[23]), "+f"(c[24]), "+f"(c[25]), "+f"(c[26]), "+f"(c[27]), "+f"(c[28]), "+f"(c[29]), "+f"(c[30]), "+f"(c[31]), "+f"(c[32]), "+f"(c[33]), "+f"(c[34]), "+f"(c[35]), "+f"(c[36]), "+f"(c[37]), "+f"(c[38]), "+f"(c[39]), "+f"(c[40]), "+f"(c[41]), "+f"(c[42]), "+f"(c[43]), "+f"(c[44]), "+f"(c[45]), "+f"(c[46]), "+f"(c[47]), "+f"(c[48]), "+f"(c[49]), "+f"(c[50]), "+f"(c[51]), "+f"(c[52]), "+f"(c[53]), "+f"(c[54]), "+f"(c[55]), "+f"(c[56]), "+f"(c[57]), "+f"(c[58]), "+f"(c[59]), "+f"(c[60]), "+f"(c[61]), "+f"(c[62]), "+f"(c[63])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate) : "memory");
}

__global__ void __launch_bounds__(128) ba_schur_tc_kernel(BaDev d, int n_chunks) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t bar_load;
    if (d.st->done) return;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int c0 = blockIdx.x * TC_CHUNKS;
    const int nc = min(TC_CHUNKS, n_chunks - c0);
    if (tid == 0) mbar_init(&bar_load, 1);
    __syncthreads();
    if (tid == 0) {
        // TMA 1-D bulk copies of this CTA's chunks (contiguous in HBM), one mbarrier transaction
        mbar_expect_tx(&bar_load, (uint32_t)nc * TC_CHUNK_BYTES);
        const unsigned char* src = reinterpret_cast<const unsigned char*>(d.tc_u) + (size_t)c0 * TC_CHUNK_BYTES;
        for (int c = 0; c < nc; ++c) bulk_load_1d(smem_raw + (size_t)c * TC_CHUNK_BYTES, src + (size_t)c * TC_CHUNK_BYTES, TC_CHUNK_BYTES, &bar_load);
    }
    mbar_wait(&bar_load, 0);
    const uint32_t base = smem_u32(smem_raw);
    const int ndim = d.tc_ndim;
    for (int mh = 0; mh < 2 && 64 * mh < ndim; ++mh) {
        float acc[64];                                  // the first product overwrites it (scale-d = 0)
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        for (int c = 0; c < nc; ++c) {
            const uint32_t cb = base + c * TC_CHUNK_BYTES, ab = cb + mh * 2048;      // rows 64 mh.. of the tile: 8 row groups of 256 B
            const uint64_t a_hi = gmma_smem_desc(ab), a_mid = gmma_smem_desc(ab + TC_TILE_BYTES), a_lo = gmma_smem_desc(ab + 2 * TC_TILE_BYTES);
            const uint64_t b_hi = gmma_smem_desc(cb), b_mid = gmma_smem_desc(cb + TC_TILE_BYTES), b_lo = gmma_smem_desc(cb + 2 * TC_TILE_BYTES);
            wgmma_bf16_m64n128(acc, a_hi, b_hi, c > 0);
            wgmma_bf16_m64n128(acc, a_hi, b_mid, 1); wgmma_bf16_m64n128(acc, a_mid, b_hi, 1);
            wgmma_bf16_m64n128(acc, a_mid, b_mid, 1);
            wgmma_bf16_m64n128(acc, a_hi, b_lo, 1); wgmma_bf16_m64n128(acc, a_lo, b_hi, 1);
        }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        // epilogue: FP32 -> FP64, subtract from the lower triangle of S (compact order)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int a = 64 * mh + 16 * warp + (lane >> 2) + 8 * i;
            if (a >= ndim) continue;
            const int ga = d.tc_off[a];
#pragma unroll
            for (int n = 0; n < 16; ++n) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int b = 8 * n + 2 * (lane & 3) + j;
                    const float f = acc[4 * n + 2 * i + j];
                    if (b > a || b >= ndim || f == 0.0f) continue;
                    const int gb = d.tc_off[b];
                    if (ga >= gb) atomicAdd(&d.S[SIDX(d, ga, gb)], -(double)f); else atomicAdd(&d.S[SIDX(d, gb, ga)], -(double)f);
                }
            }
        }
    }
}

__global__ void ba_pack_scalars_kernel(BaDev d) {
    LmState* st = d.st;
    if (st->done) return;
    d.scal[0] = st->need_linearize ? st->cost_acc : 0.0;
    d.scal[1 + d.rank] = __longlong_as_double((long long)st->grad_max_bits);
}
__global__ void ba_unpack_scalars_kernel(BaDev d) {
    LmState* st = d.st;
    if (st->done) return;
    if (st->need_linearize) st->cost_acc = d.scal[0];
    double m = 0.0;
    for (int r = 0; r < d.world; ++r) m = fmax(m, d.scal[1 + r]);
    st->grad_max_bits = (unsigned long long)__double_as_longlong(m);
}

// camera blocks: Jacobi scale, damping added to diag(S), gradient max-norm ||x - Plus(x,-g)||_inf
// returns the block's gradient max-norm as ordered bits (0: nothing to report); the caller reduces over the warp and issues ONE atomicMax
__device__ __forceinline__ unsigned long long prepare_camera_block(const BaDev& d, int i) {
    LmState* st = d.st;
    const bool is_pose = i < d.n_poses;
    const int off = is_pose ? d.pose_off[i] : d.vec3_off[i - d.n_poses];
    if (off < 0) return 0ull;
    const int w = is_pose ? 6 : 3;
    for (int k = 0; k < w; ++k) {
        const double h = d.diagH[off + k];
        if (!st->scale_valid) d.scale_c[off + k] = st->jacobi ? 1.0 / (1.0 + sqrt(h)) : 1.0;
        const double s = d.scale_c[off + k], s2 = s * s;
        const double lam = fmin(fmax(s2 * h, st->min_diag), st->max_diag) / (st->radius * s2);
        d.lam_c[off + k] = lam;
        d.S[SIDX(d, off + k, off + k)] += lam;
    }
    if (st->need_linearize) {
        double gm = 0.0;
        if (is_pose) {
            double ng[6], out[7];
            for (int k = 0; k < 6; ++k) ng[k] = -d.gcr[off + k];
            const double* x = d.poses + 7 * i;
            pose_plus(x, ng, out);
            for (int k = 0; k < 7; ++k) { const double df = fabs(x[k] - out[k]); gm = (df == df) ? fmax(gm, df) : INFINITY; }
        } else for (int k = 0; k < 3; ++k) { const double df = fabs(d.gcr[off + k]); gm = (df == df) ? fmax(gm, df) : INFINITY; }
        return (gm == gm) ? (unsigned long long)__double_as_longlong(fabs(gm)) : 0x7ff0000000000000ull;
    }
    return 0ull;
}
__device__ __forceinline__ void warp_max_to_state(LmState* st, unsigned long long bits) {
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long v = __shfl_xor_sync(0xffffffffu, bits, o); bits = v > bits ? v : bits; }
    if ((threadIdx.x & 31) == 0 && bits) atomicMax(&st->grad_max_bits, bits);
}

// S <- lower(Hpp), rhs <- -gc, gcr <- gc, diagH <- diag(Hpp), scalars <- 0.
// FUSE_DAMP (single GPU): the camera blocks' Jacobi scale, LM damping and gradient max-norm (prepare_camera_block) ride along: the
// bulk copy skips the diagonal and the thread that owns a block fills that block's rows (diagonal of S, rhs, gcr, diagH) and damps
// them itself, so there is no ordering hazard -- the Schur kernel's `S -= ...` atomics that follow commute with the damping.
// Sharded problems damp after the all-reduce instead (the diagonal must be the global one) and keep ba_prepare_camera_kernel.
template <int FUSE_DAMP>
__global__ void ba_build_S_kernel(BaDev d) {
    if (d.st->done) return;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    if (gid < 16) d.scal[gid] = 0.0;
    const size_t dstep = (size_t)d.srow + 1;                                   // distance between consecutive diagonal entries
    for (size_t i = gid; i < d.nS; i += stride) {
        if (FUSE_DAMP && i >= (size_t)d.soff && (i - (size_t)d.soff) % dstep == 0) continue;
        d.S[i] = d.Hpp[i];          // only the lower triangle / band is ever written
    }
    if (!FUSE_DAMP) {
        for (size_t r = gid; r < (size_t)d.dimc; r += stride) { d.diagH[r] = d.Hpp[SIDX(d, r, r)]; d.rhs[r] = -d.gc[r]; d.gcr[r] = d.gc[r]; }
    } else {
        unsigned long long gbits = 0ull;
        for (size_t i = gid; i < (size_t)(d.n_poses + d.n_vec3); i += stride) {
            const bool is_pose = i < (size_t)d.n_poses;
            const int off = is_pose ? d.pose_off[i] : d.vec3_off[i - d.n_poses];
            if (off < 0) continue;
            const int w = is_pose ? 6 : 3;
            for (int k = 0; k < w; ++k) {
                const int r = off + k;
                const double h = d.Hpp[SIDX(d, r, r)];
                d.diagH[r] = h; d.rhs[r] = -d.gc[r]; d.gcr[r] = d.gc[r]; d.S[SIDX(d, r, r)] = h;
            }
            gbits = max(gbits, prepare_camera_block(d, (int)i));
        }
        warp_max_to_state(d.st, gbits);
    }
}

__global__ void ba_prepare_camera_kernel(BaDev d) {
    if (d.st->done) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    warp_max_to_state(d.st, (i < d.n_poses + d.n_vec3) ? prepare_camera_block(d, i) : 0ull);
}

// Sharded problems, window size: the exchange of the reduced system and everything that only exists because of it, in ONE kernel
// over NVLink peer memory -- the scalars ride in the arena (packed on the fly while the contribution is copied into the exchange
// buffer), the sum over the ranks is formed with loads from the peers' buffers, and the CTA that finishes last unpacks the scalars
// and applies the camera damping, which needs the global diagonal.  (Four launches before: pack, all-reduce, unpack, damping.)
__global__ void __launch_bounds__(256) ba_allreduce_fused_kernel(P2PArgs a, BaDev d, int count) {
    LmState* st = d.st;
    const bool active = !st->done;                      // identical on every rank; the exchange itself always runs
    double* buf = d.S;
    const int i_scal = (int)(d.scal - d.S);
    const int need_lin = st->need_linearize;
    const double my_cost = st->cost_acc;
    const double my_gmax = __longlong_as_double((long long)st->grad_max_bits);
    bool last; unsigned int epoch;
    const bool alive = p2p_allreduce_body(a, buf, count, [&](int i) -> double {
        if (active && i == i_scal) return need_lin ? my_cost : 0.0;
        if (active && i == i_scal + 1 + d.rank) return my_gmax;
        return __ldcg(buf + i);
    }, &last, &epoch);
    if (!alive || !last) return;
    if (active) {
        if (threadIdx.x == 0) {
            if (need_lin) st->cost_acc = __ldcg(d.scal);
            double m = 0.0;
            for (int r = 0; r < d.world; ++r) m = fmax(m, __ldcg(d.scal + 1 + r));
            st->grad_max_bits = (unsigned long long)__double_as_longlong(m);
        }
        __syncthreads();
        unsigned long long gbits = 0ull;
        for (int i = threadIdx.x; i < d.n_poses + d.n_vec3; i += blockDim.x) gbits = max(gbits, prepare_camera_block(d, i));
        warp_max_to_state(st, gbits);
        __syncthreads();
    }
    p2p_finish_epoch(a, epoch);
}

__global__ void lm_control_pre_kernel(LmState* st) { lm_control_pre(*st); }

// ------------------------------------------------------------------ K6 dense Cholesky, one CTA
// Right-looking blocked (32) factorisation of the lower triangle of S (n x n, row-major, in L2/HBM) with
// the right-hand side carried along as an extra row (so the forward substitution is free), then a
// blocked backward substitution.  Result: rhs <- S^-1 rhs.
//
// Schedule of one 32-column step k (look-ahead of depth one, the serial part on its own warp):
//   warp 0     : panel solve of the 32 "head" rows (= the rows of diagonal block k + 1), one row per lane;  update of diagonal block
//                k + 1 by these rows as one 32 x 32 register-tiled product, handed to the row-per-lane layout of the factorisation
//                through shared memory (no trip through global memory);  factorisation of block k + 1 into the OTHER (Dt, invd) buffer
//   warps 1..7 : the INVERSE of block k of L to the block's place in S (for the backward pass);  panel solve of the remaining rows +
//                the rhs row;  named barrier (warp 0 only arrives, once its head rows are in shared memory);  trailing update of
//                everything but diagonal block k + 1
// so the pivot chain of block k + 1 overlaps the panel and the trailing update of step k instead of following them.
#define SA(i_, j_) S[(size_t)(i_) * (size_t)srow + (size_t)(j_) + (size_t)soff]
enum { CHOL_DT = 32 * 34 + 32, CHOL_HDR = 2 * CHOL_DT };        // doubles: (Dt, invd) twice, then the panel
__global__ void __launch_bounds__(CHOL_T) ba_cholesky_kernel(double* __restrict__ S, double* __restrict__ rhs, int n, long long srow, long long soff,
                                                                  double* __restrict__ invd_g, LmState* st, int run_control_pre,
                                                                  const int* __restrict__ env_rmax, const int* __restrict__ env_cmin) {
    if (run_control_pre) { if (threadIdx.x == 0) lm_control_pre(*st); __syncthreads(); }
    if (st->done) return;
    extern __shared__ __align__(16) double sm[];
    double* P = sm + CHOL_HDR;         // rows x 34 panel (16 B aligned rows for broadcast double2 loads)
    __shared__ int fail;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    if (tid == 0) fail = 0;
    long long t_diag = 0, t_panel = 0, t_trail = 0, t0 = clock64(), tA;
    const long long t_begin = t0;
    // ---- diagonal block 0: warp 0, one row per lane in registers (lvb_chol.cuh)
    if (warp == 0) {
        const int b0 = min(32, n);
        double a[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) a[j] = (lane < b0 && j <= lane) ? SA(lane, j) : ((j == lane) ? 1.0 : 0.0);
        const int bad = chol_diag32_pair(a, lane, sm, sm + 32 * 34);
        if (bad && lane == 0) fail = 1;
    }
    __syncthreads();
    tA = clock64(); t_diag += tA - t0; t0 = tA;
    for (int kb = 0; kb < n; kb += 32) {
        const int bs = min(32, n - kb), kn = kb + 32;
        const int hb = max(0, min(32, n - kn));                    // rows of the next diagonal block ("head" rows of the panel)
        double* Dt = sm + ((kb >> 5) & 1) * CHOL_DT;               // block kb of L, column-major: Dt[j * 34 + k] = L[k][j]
        double* invd = Dt + 32 * 34;
        double* Dn = sm + (((kb >> 5) & 1) ^ 1) * CHOL_DT;
        // panel rows: the rows below the block inside the envelope of this block column (S is block-banded by construction) + the rhs row (last)
        const int m = env_rmax[kb >> 5] - (kb + bs) + 1 + 1;
        const int mh = min(hb, m - 1);                             // head rows inside the envelope
        if (warp == 0 && hb > 0) {
            double x[32], a[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) x[j] = (lane < mh && j < bs) ? SA(kn + lane, kb + j) : 0.0;
#pragma unroll
            for (int j = 0; j < 32; ++j) a[j] = (lane < hb && j <= lane) ? SA(kn + lane, kn + j) : ((j == lane) ? 1.0 : 0.0);
            chol_panel_row(x, Dt, invd);
#pragma unroll
            for (int j = 0; j < 32; ++j) if (lane < mh) { P[lane * 34 + j] = x[j]; if (j < bs) SA(kn + lane, kb + j) = x[j]; }
            __syncwarp();
            asm volatile("bar.arrive 1, %0;" :: "r"(nt) : "memory");
            tA = clock64(); t_panel += tA - t0; t0 = tA;
            // diagonal block kn -= (head rows)(head rows)^T: computed as a 32 x 32 tile in the 4 x 8 register micro-tile layout of the
            // trailing update (12 LDS.128 per 64 DFMA; the row-per-lane layout would need one LDS.128 per 2 DFMA and is bound by the
            // shared-memory return path), then passed through the free diagonal-block buffer to the row-per-lane layout of the
            // factorisation.  Head rows outside the envelope are structurally zero and have no panel row.
            if (mh > 0) {
                const int ry = lane >> 2, cx = lane & 3;
                double acc[4][8];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0;
                const double2* rp[4]; const double2* cp[8];
#pragma unroll
                for (int i = 0; i < 4; ++i) rp[i] = reinterpret_cast<const double2*>(P + (size_t)min(ry + 8 * i, mh - 1) * 34);
#pragma unroll
                for (int j = 0; j < 8; ++j) cp[j] = reinterpret_cast<const double2*>(P + (size_t)min(cx + 4 * j, mh - 1) * 34);
#pragma unroll 2
                for (int k = 0; k < 16; ++k) {
                    double2 rv[4], cv[8];
#pragma unroll
                    for (int i = 0; i < 4; ++i) rv[i] = rp[i][k];
#pragma unroll
                    for (int j = 0; j < 8; ++j) cv[j] = cp[j][k];
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 8; ++j) { acc[i][j] += rv[i].x * cv[j].x; acc[i][j] += rv[i].y * cv[j].y; }
                }
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) Dn[(ry + 8 * i) * 34 + cx + 4 * j] = (ry + 8 * i < mh && cx + 4 * j < mh) ? acc[i][j] : 0.0;
                __syncwarp();
#pragma unroll
                for (int j = 0; j < 32; ++j) a[j] -= Dn[lane * 34 + j];
                __syncwarp();
            }
            const int bad = chol_diag32_pair(a, lane, Dn, Dn + 32 * 34);
            if (bad && lane == 0) fail = 1;
            tA = clock64(); t_diag += tA - t0; t0 = tA;
        } else {
            const int wid = hb > 0 ? warp - 1 : warp, nwk = hb > 0 ? nw - 1 : nw;       // the warps doing this part
            const int t2 = wid * 32 + lane, nt2 = nwk * 32;
            // the INVERSE of block kb of L goes to the block's place in S: the backward pass then applies a diagonal block as 32 independent
            // FMAs per lane instead of a 32-step substitution chain.  Column c of L^-1 is the panel solve of the unit row e_c; one warp
            // (the last one, which has the fewest panel rows) does it while the others are in the panel.
            if (wid == nwk - 1) {
                double e[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) e[j] = (j == lane) ? 1.0 : 0.0;
                chol_panel_row(e, Dt, invd);
#pragma unroll
                for (int j = 0; j < 32; ++j) if (j >= lane && j < bs) SA(kb + j, kb + lane) = e[j];
            }
            // ---- panel, the rows warp 0 does not take:  x L^T = a, right-looking, no divisions
            for (int rr = mh + t2; rr < m; rr += nt2) {
                const bool is_rhs = (rr == m - 1);
                double* src = is_rhs ? (rhs + kb) : &SA(kb + bs + rr, kb);
                double a[32];
    #pragma unroll
                for (int j = 0; j < 32; ++j) a[j] = (j < bs) ? src[j] : 0.0;
                chol_panel_row(a, Dt, invd);
    #pragma unroll
                for (int j = 0; j < 32; ++j) { P[rr * 34 + j] = a[j]; if (j < bs) src[j] = a[j]; }
            }
            asm volatile("bar.sync 1, %0;" :: "r"(nt) : "memory");
            // ---- trailing update A22 -= P P^T on the lower triangle.  One warp per 32x32 tile, each lane a 4x8
            // register micro-tile (rows ry+8i, columns cx+4j: consecutive lanes touch consecutive panel rows, so the
            // LDS.128 operand loads are bank-conflict free and every loaded value feeds 4 or 8 DFMAs).  The head rows of
            // tile (0, 0) -- diagonal block kn -- are warp 0's.
            const int ntile = (m + 31) >> 5;
            const int total = (m > 1) ? ntile * (ntile + 1) / 2 : 0;
            for (int t = wid; t < total; t += nwk) {
                if (t == 0 && mh >= min(32, m)) continue;
                int ti = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
                while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
                while (ti * (ti + 1) / 2 > t) --ti;
                const int tj = t - ti * (ti + 1) / 2;
                const int row_lo = (t == 0) ? mh : 0;
                const int ry = lane >> 2, cx = lane & 3;
                const int r0 = ti * 32 + ry, c0 = tj * 32 + cx;
                double acc[4][8];
    #pragma unroll
                for (int i = 0; i < 4; ++i)
    #pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0;
                // rows / columns beyond the panel read row 0 (valid memory) and are masked at the store
                const double2* rp[4]; const double2* cp[8];
    #pragma unroll
                for (int i = 0; i < 4; ++i) rp[i] = reinterpret_cast<const double2*>(P + (size_t)min(r0 + 8 * i, m - 1) * 34);
    #pragma unroll
                for (int j = 0; j < 8; ++j) cp[j] = reinterpret_cast<const double2*>(P + (size_t)min(c0 + 4 * j, m - 1) * 34);
    #pragma unroll 2
                for (int k = 0; k < 16; ++k) {
                    double2 rv[4], cv[8];
    #pragma unroll
                    for (int i = 0; i < 4; ++i) rv[i] = rp[i][k];
    #pragma unroll
                    for (int j = 0; j < 8; ++j) cv[j] = cp[j][k];
    #pragma unroll
                    for (int i = 0; i < 4; ++i)
    #pragma unroll
                        for (int j = 0; j < 8; ++j) { acc[i][j] += rv[i].x * cv[j].x; acc[i][j] += rv[i].y * cv[j].y; }
                }
                // read-modify-write of the tile: all loads first (one round trip), then the stores
                double cur[4][8];
    #pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int ip = min(r0 + 8 * i, m - 1);
                    const double* src = (ip == m - 1) ? (rhs + kb + bs) : &SA(kb + bs + ip, kb + bs);
    #pragma unroll
                    for (int j = 0; j < 8; ++j) { const int jp = c0 + 4 * j; cur[i][j] = (r0 + 8 * i < m && r0 + 8 * i >= row_lo && jp < m - 1 && jp <= ip) ? src[jp] : 0.0; }
                }
    #pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int ip = r0 + 8 * i;
                    if (ip >= m || ip < row_lo) continue;
                    double* dst = (ip == m - 1) ? (rhs + kb + bs) : &SA(kb + bs + ip, kb + bs);
    #pragma unroll
                    for (int j = 0; j < 8; ++j) { const int jp = c0 + 4 * j; if (jp < m - 1 && jp <= ip) dst[jp] = cur[i][j] - acc[i][j]; }
                }
            }
        }
        __syncthreads();
        tA = clock64(); t_trail += tA - t0; t0 = tA;
    }
    // ---- backward substitution  L^T x = y  (y is in rhs), left-looking per 32-column block:
    //   x_k = D_k^-T (y_k - sum_{r below} L[r][k-block]^T x_r),  D_k^-1 stored in place of D_k by the factorisation
    // the sum is a GEMV over the envelope rows spread over all warps (independent coalesced loads, one L2 round trip per
    // batch), then warp 0 applies the inverse diagonal block: 32 independent FMAs per lane, no substitution chain.  x overwrites rhs.
    const int last = ((n - 1) / 32) * 32;
    double* part = P;                                 // nw x 32 partial sums
    for (int kb = last; kb >= 0; kb -= 32) {
        const int bs = min(32, n - kb);
        const int rend = env_rmax[kb >> 5];
        double col[32];                               // warp 0: column `lane` of the inverse diagonal block, col[i] = Linv[kb+i][kb+lane], i >= lane
        double t = 0.0;
        if (warp == 0) {
#pragma unroll
            for (int i = 0; i < 32; ++i) col[i] = (i < bs && lane < bs && i >= lane) ? SA(kb + i, kb + lane) : 0.0;
            if (lane < bs) t = rhs[kb + lane];
        }
        double acc = 0.0;
        if (lane < bs) {
            for (int r0 = kb + bs + warp; r0 <= rend; r0 += 16 * nw) {
                double lv[16], xv[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) { const int r = r0 + u * nw; const bool ok = r <= rend; lv[u] = ok ? SA(r, kb + lane) : 0.0; xv[u] = ok ? rhs[r] : 0.0; }
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
            if (lane < bs) rhs[kb + lane] = t;
        }
        __syncthreads();
    }
    if (tid == 0 && fail) st->solve_fail = 1;
    if (tid == 0) { tA = clock64(); g_chol_dbg[0] += t_diag; g_chol_dbg[1] += t_panel; g_chol_dbg[2] += t_trail; g_chol_dbg[3] += tA - t0; g_chol_dbg[4] += tA - t_begin; g_chol_dbg[5] += 1; }
}

#include "ba_tree.cuh"
#include "ba_wide.cuh"

// ------------------------------------------------------------------ back-substitution + candidate point
__global__ void __launch_bounds__(TPB) ba_update_kernel(BaDev d) {
    __shared__ double s_red[TPB / 32];
    LmState* st = d.st;
    if (st->done) return;
    const double* dc = d.rhs;
    const int i = blockIdx.x * TPB + threadIdx.x;
    double a = 0, b = 0, sn = 0, xn = 0;
    if (i < d.n_poses) {
        const double* x = d.poses + 7 * i; double* c = d.c_poses + 7 * i;
        const int off = d.pose_off[i];
        if (off < 0) { for (int k = 0; k < 7; ++k) c[k] = x[k]; }
        else {
            double dl[6], out[7];
            for (int k = 0; k < 6; ++k) dl[k] = dc[off + k];
            pose_plus(x, dl, out);
            for (int k = 0; k < 7; ++k) { c[k] = out[k]; if (d.rank0) { sn += (x[k] - out[k]) * (x[k] - out[k]); xn += x[k] * x[k]; } }
            if (d.rank0) for (int k = 0; k < 6; ++k) { a += dl[k] * d.lam_c[off + k] * dl[k]; b += d.gcr[off + k] * dl[k]; }
        }
    } else if (i < d.n_poses + d.n_vec3) {
        const int j = i - d.n_poses;
        const double* x = d.vec3 + 3 * j; double* c = d.c_vec3 + 3 * j;
        const int off = d.vec3_off[j];
        for (int k = 0; k < 3; ++k) {
            const double dl = off < 0 ? 0.0 : dc[off + k];
            c[k] = x[k] + dl;
            if (off >= 0 && d.rank0) { sn += dl * dl; xn += x[k] * x[k]; a += dl * d.lam_c[off + k] * dl; b += d.gcr[off + k] * dl; }
        }
    } else if (i < d.n_poses + d.n_vec3 + d.n_rho) {
        const int l = i - d.n_poses - d.n_vec3;
        double dl = 0.0;
        const int e0 = d.lm_start[l], e1 = d.lm_start[l + 1];
        if (d.rho_slot[l] >= 0 && e1 > e0) {
            const int n = d.n[0];
            const int* ix = d.fi[0];
            double s = d.gl[l];
            for (int eb = e0; eb < e1; eb += 4) {      // four factors at a time, loads before uses (see ba_schur_kernel)
                int f[4], o0[4], o1[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) f[u] = (eb + u < e1) ? d.lm_fac[eb + u] : -1;
#pragma unroll
                for (int u = 0; u < 4; ++u) { const int fc = max(f[u], 0); o0[u] = ix[(size_t)n + fc]; o1[u] = ix[(size_t)2 * n + fc]; }      // unconditional (clamped) loads
#pragma unroll
                for (int u = 0; u < 4; ++u) { o0[u] = d.pose_off[o0[u]]; o1[u] = d.pose_off[o1[u]]; }
                double2 w[4][6];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const double2* src = reinterpret_cast<const double2*>(d.tf_w + (size_t)max(f[u], 0) * 12);
#pragma unroll
                    for (int k = 0; k < 6; ++k) w[u][k] = src[k];
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    if (f[u] < 0) continue;
                    if (o0[u] >= 0) { const double* t = dc + o0[u]; s += w[u][0].x * t[0] + w[u][0].y * t[1] + w[u][1].x * t[2] + w[u][1].y * t[3] + w[u][2].x * t[4] + w[u][2].y * t[5]; }
                    if (o1[u] >= 0) { const double* t = dc + o1[u]; s += w[u][3].x * t[0] + w[u][3].y * t[1] + w[u][4].x * t[2] + w[u][4].y * t[3] + w[u][5].x * t[4] + w[u][5].y * t[5]; }
                }
            }
            const double lam = d.lam_l[l];
            dl = -s / (d.Hll[l] + lam);
            sn = dl * dl; xn = d.rho[l] * d.rho[l]; a = dl * lam * dl; b = d.gl[l] * dl;
        }
        d.c_rho[l] = d.rho[l] + dl;
    }
    block_add(a, &st->mcc_a, s_red);
    block_add(b, &st->mcc_b, s_red);
    block_add(sn, &st->step_norm2, s_red);
    block_add(xn, &st->x_norm2, s_red);
}

// One CTA closes the iteration: LM decision (thread 0), then -- if the step was accepted -- candidate -> x and the
// accumulators of the next linearisation are cleared (problems on the dense-solver path are small: < 1 MB).
__global__ void __launch_bounds__(1024) ba_post_kernel(BaDev d, int decide_only) {
    LmState* st = d.st;
    __shared__ int s_accept, s_zero;
    if (threadIdx.x == 0) {
        const int was_done = st->done;
        if (!was_done) { lm_control_post(*st); if (st->accept) st->x_cost = st->cand_cost_acc; }
        s_accept = (!was_done && st->accept) ? 1 : 0;
        s_zero = (!st->done && st->need_linearize) ? 1 : 0;
    }
    __syncthreads();
    if (decide_only) return;
    if (s_accept) {
        const size_t np = (size_t)d.n_poses * 7, nv = (size_t)d.n_vec3 * 3, nr = d.n_rho;
        for (size_t i = threadIdx.x; i < np + nv + nr; i += blockDim.x) {
            if (i < np) d.poses[i] = d.c_poses[i];
            else if (i < np + nv) d.vec3[i - np] = d.c_vec3[i - np];
            else d.rho[i - np - nv] = d.c_rho[i - np - nv];
        }
    }
    if (s_zero) {
        const size_t nH = d.nS;
        double2* H2 = reinterpret_cast<double2*>(d.Hpp);
        for (size_t i = threadIdx.x; i < nH / 2; i += blockDim.x) H2[i] = make_double2(0.0, 0.0);
        if ((nH & 1) && threadIdx.x == 0) d.Hpp[nH - 1] = 0.0;
        for (size_t i = threadIdx.x; i < (size_t)d.dimc; i += blockDim.x) d.gc[i] = 0.0;
        for (size_t i = threadIdx.x; i < (size_t)d.n_rho; i += blockDim.x) { d.Hll[i] = 0.0; d.gl[i] = 0.0; }
    }
}

// Large problems (banded storage): the same accept + clear spread over the whole grid.  `accept` may be stale when the
// solve finished in an earlier pass; the copy is idempotent then (the candidate has not been rewritten).
__global__ void ba_post_wide_kernel(BaDev d) {
    const LmState* st = d.st;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    if (st->accept) {
        const size_t np = (size_t)d.n_poses * 7, nv = (size_t)d.n_vec3 * 3, nr = d.n_rho;
        for (size_t i = gid; i < np + nv + nr; i += stride) {
            if (i < np) d.poses[i] = d.c_poses[i];
            else if (i < np + nv) d.vec3[i - np] = d.c_vec3[i - np];
            else d.rho[i - np - nv] = d.c_rho[i - np - nv];
        }
    }
    if (!st->done && st->need_linearize) {
        const size_t nH = d.nS;
        double2* H2 = reinterpret_cast<double2*>(d.Hpp);
        for (size_t i = gid; i < nH / 2; i += stride) H2[i] = make_double2(0.0, 0.0);
        if ((nH & 1) && gid == 0) d.Hpp[nH - 1] = 0.0;
        for (size_t i = gid; i < (size_t)d.dimc; i += stride) d.gc[i] = 0.0;
        for (size_t i = gid; i < (size_t)d.n_rho; i += stride) { d.Hll[i] = 0.0; d.gl[i] = 0.0; }
    }
}

__global__ void ba_reproj_error_kernel(BaDev d, int n, const double* __restrict__ ob_pw, const int* __restrict__ pose_idx, double* __restrict__ err) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    PoseOnlyLin o;
    const double* e = ob_pw + 5 * (size_t)f;
    pose_only_lin(d.cams, e[0], e[1], v3(e[2], e[3], e[4]), 1.0, d.poses + 7 * pose_idx[f], o, nullptr);
    err[f] = sqrt(o.r[0] * o.r[0] + o.r[1] * o.r[1]);
}

}  // namespace

// ====================================================================================== host side
struct lvb_ba {
    lvb_ctx* ctx = nullptr;
    bool finalized = false, solvable = false;
    const char* unsolvable_why = "the problem has no free camera parameter";
    long long srow = 0, soff = 0; size_t nS = 1, chol_smem = 0; int band = 0, panel_rows = 2;
    DevBuf<double> chol_invd;
    double cam[22];
    bool have_cam = false;
    std::vector<double> h_poses, h_vec3, h_rho;
    std::vector<double> r_params; bool host_fresh = false;      // parameter blocks as last read back (one round trip serves the three getters)
    std::vector<uint8_t> h_pose_const, h_vec3_const, h_rho_const;
    std::vector<double> h_fc[6];
    std::vector<int32_t> h_fi[6];
    int n[6] = {0, 0, 0, 0, 0, 0};      // blocks as added by the caller
    int nd[6] = {0, 0, 0, 0, 0, 0};     // blocks in the device layout (kinds 0/1: sorted by pose key, each key padded to 32)
    std::vector<int> order[6];          // device position -> caller index, -1 for padding
    double huber[6] = {0, 0, 0, 0, 0, 0};
    int dimc = 0, n_pose_free = 0, n_vec3_free = 0, n_rho_free = 0;
    std::vector<int> canon;             // internal camera-system offset -> canonical (poses first, then vec3) offset
    DevBuf<int> chol_rmax, chol_cmin;   // envelope of S per 32-column block step
    // multifrontal tree over the banded system (ba_tree.cuh); tree_levels == 0: single-CTA envelope Cholesky
    DevBuf<Front> fronts; DevBuf<double> front_pool;
    std::vector<int> level_first, level_count;
    int tree_levels = 0; size_t tree_factor_smem = 0, tree_back_smem = 0;
    bool wide_solver = false;           // envelope too wide for the one-CTA panel and no tree: per-phase grids over S in global memory (ba_wide.cuh)
    std::vector<int> h_rmax;            // host copy of the envelope (launch geometry of the wide solver)
    // device
    DevBuf<unsigned char> upload_arena;      // one allocation for everything finalize uploads (the buffers below are views into it)
    DevBuf<double> poses, vec3, rho, c_poses, c_vec3, c_rho;
    DevBuf<int> pose_off, vec3_off, rho_slot, lm_start, lm_fac;
    DevBuf<int> tf_slot, sw_group, sw_lm, grp_ns, grp_off;
    int n_schur_warps = 0, schur_cols_max = 0;
    size_t schur_smem = 0, lin_smem = 0;
    cudaGraphExec_t pass_graph = nullptr;
    bool graph_borrowed = false;        // pass_graph is the context's cached exec (never destroyed from here)
    int pass_launches = 0;
    bool capturing = false;
    bool imu_checked = true;
    // tensor-core Schur (schur_mode 1)
    bool tc_ok = false; int schur_mode = 0, graph_mode = -1, n_tc_chunks = 0;
    DevBuf<unsigned short> tc_u; DevBuf<int> tc_cdim, tc_off;
    int solves_done = 0;
    DevBuf<double> fc[6];
    DevBuf<int> fi[6];
    DevBuf<double> imu_raw;
    DevBuf<int> imu_status;
    DevBuf<double> Hpp, gc, Hll, gl, tf_w, arena, scale_c, scale_l, lam_c, lam_l;
    DevBuf<double> eval_r, eval_J;
    DevBuf<LmState> st;
    BaDev dev;
    BlockRanges ranges;
    size_t pose_smem = 0, imu_smem = 0;
};

// the pass graph is either the problem's own or the context's cached one (borrowed while ctx->graph_owner == ba)
static void drop_graph(lvb_ba* ba) {
    if (!ba->pass_graph) return;
    if (ba->graph_borrowed) { if (ba->ctx->graph_owner == ba) ba->ctx->graph_owner = nullptr; }
    else cudaGraphExecDestroy(ba->pass_graph);
    ba->pass_graph = nullptr; ba->graph_borrowed = false;
}

static const int kConstStride[6] = {5, 6, 5, IMU_RAW, 8, 9};
static const int kIdxStride[6] = {3, 1, 1, 8, 2, 1};
static const int kResDim[6] = {2, 2, 2, 15, 6, 6};
static const int kJacCols[6] = {15, 7, 1, 32, 14, 7};

static bool g_tables_ready = false;
static int init_tables() {
    if (g_tables_ready) return LVB_OK;
    unsigned char a[465], b[465]; int e = 0;
    for (int i = 0; i < 30; ++i) for (int j = 0; j <= i; ++j) { a[e] = (unsigned char)i; b[e] = (unsigned char)j; ++e; }
    LVB_CUDA(cudaMemcpyToSymbol(c_tri_a, a, sizeof(a)));
    LVB_CUDA(cudaMemcpyToSymbol(c_tri_b, b, sizeof(b)));
    LVB_CUDA(cudaFuncSetAttribute(ba_cholesky_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 256));
    LVB_CUDA(cudaFuncSetAttribute(ba_front_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 256));
    LVB_CUDA(cudaFuncSetAttribute(ba_front_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    LVB_CUDA(cudaFuncSetAttribute(ba_eval_two_frame_kernel<1, 5>, cudaFuncAttributeMaxDynamicSharedMemorySize, (TPB * 31 + MAX_STAGE_POSES * 7 + 2) * 8));
    LVB_CUDA(cudaFuncSetAttribute(ba_eval_two_frame_kernel<1, 6>, cudaFuncAttributeMaxDynamicSharedMemorySize, (TPB * 31 + MAX_STAGE_POSES * 7 + 2) * 8));
    LVB_CUDA(cudaFuncSetAttribute(ba_eval_two_frame_kernel<0, 5>, cudaFuncAttributeMaxDynamicSharedMemorySize, (MAX_STAGE_POSES * 7 + 2) * 8));
    LVB_CUDA(cudaFuncSetAttribute(ba_eval_two_frame_kernel<0, 6>, cudaFuncAttributeMaxDynamicSharedMemorySize, (MAX_STAGE_POSES * 7 + 2) * 8));
    LVB_CUDA(cudaFuncSetAttribute(ba_linearize_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    LVB_CUDA(cudaFuncSetAttribute(ba_linearize_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    LVB_CUDA(cudaFuncSetAttribute(ba_linearize_all_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    LVB_CUDA(cudaFuncSetAttribute(ba_linearize_all_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    LVB_CUDA(cudaFuncSetAttribute(ba_schur_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_CHUNKS * TC_CHUNK_BYTES));
    LVB_CUDA(cudaFuncSetAttribute(ba_schur_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (TPB / 32) * 32 * (6 * MAX_TRACK + 1) * 8));
    g_tables_ready = true;
    return LVB_OK;
}

static inline int nblk(size_t n, int per) { return (int)((n + per - 1) / per); }
static void mark(struct lvb_ba* ba, const char* name);
#define LAUNCH_ON(ba, stream_, kernel, grid, block, smem, ...)                             \
    do { if ((grid) > 0) { kernel<<<(grid), (block), (smem), (stream_)>>>(__VA_ARGS__); (ba)->ctx->launches++; } } while (0)
#define LAUNCH(ba, kernel, grid, block, smem, ...)                                        \
    do { if ((grid) > 0) { kernel<<<(grid), (block), (smem), (ba)->ctx->stream>>>(__VA_ARGS__); (ba)->ctx->launches++; mark(ba, #kernel); } } while (0)

// Separator tree of the banded reduced system (see ba_tree.cuh): complete binary tree with 2^D leaves, separators of width
// w = true half bandwidth.  Leaves keep >= 2w unknowns so that a separator is coupled to nothing beyond its two neighbouring subtrees.
static int build_front_tree(int n, int band, int sep, int max_leaves, std::vector<Front>& out, std::vector<int>& level_first, std::vector<int>& level_count,
                            size_t& pool_doubles, int& max_panel_rows, int& max_nb) {
    out.clear(); level_first.clear(); level_count.clear(); pool_doubles = 0; max_panel_rows = 0; max_nb = 0;
    // separator width: the TRUE half bandwidth is enough to separate (the storage band carries up to 31 columns of block-step slack);
    // a front's cost grows with the cube of it
    static const bool sep_is_band = getenv("LVB_TREE_SEP_BAND") && getenv("LVB_TREE_SEP_BAND")[0] == '1';      // A/B switch
    const int w = sep_is_band ? band : std::max(1, std::min(sep, band));
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

static void mark(lvb_ba* ba, const char* name) { lvb::timing_mark(ba->ctx->stream, name); }
#define g_timing lvb::g_timing

static int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("kernel launch failed in %s: %s", what, cudaGetErrorString(e)); return LVB_ERR_CUDA; }
    return LVB_OK;
}

// AoS -> SoA of one factor kind in device order: record i of the output is caller record ord[i] (or a padding copy of record
// -1 - ord[i] with its weight column zeroed).  Compile-time strides for the visual kinds: the generic loop spends its time on the
// loop control of a 5-iteration inner loop.
template <int CS> static void gather_planes(double* __restrict__ out, const double* __restrict__ hc, const int* __restrict__ ord, int n, int wcol) {
    for (int i = 0; i < n; ++i) {
        if (i + 16 < n) { const int g = ord[i + 16] >= 0 ? ord[i + 16] : -1 - ord[i + 16]; __builtin_prefetch(hc + (size_t)g * CS); __builtin_prefetch(hc + (size_t)g * CS + CS - 1); }
        const bool pad = ord[i] < 0;
        const double* src = hc + (size_t)(pad ? -1 - ord[i] : ord[i]) * CS;
#pragma GCC unroll 8
        for (int j = 0; j < CS; ++j) out[(size_t)j * n + i] = src[j];
        if (pad && wcol >= 0) out[(size_t)wcol * n + i] = 0.0;
    }
}
template <int IS> static void gather_index_planes(int* __restrict__ out, const int32_t* __restrict__ hi, const int* __restrict__ ord, int n) {
    for (int i = 0; i < n; ++i) {
        if (i + 16 < n) { const int g = ord[i + 16] >= 0 ? ord[i + 16] : -1 - ord[i + 16]; __builtin_prefetch(hi + (size_t)g * IS); }
        const int32_t* src = hi + (size_t)(ord[i] >= 0 ? ord[i] : -1 - ord[i]) * IS;
#pragma GCC unroll 8
        for (int j = 0; j < IS; ++j) out[(size_t)j * n + i] = src[j];
    }
}

// Assembles the arrays a problem uploads in the context's pinned staging area; commit() sends them to the device with ONE copy into
// ONE allocation and points the DevBufs at their pieces (finalize used to issue ~40 pageable cudaMemcpyAsync calls: 0.29 of its
// 0.53 ms at window size).  A reserve() hands out staging memory to be filled in place (the AoS -> SoA transposition writes its
// planes there directly); the pointer is good until the next reserve / put.  Map-scale problems (more than STAGE_MAX bytes of
// factors) keep the per-array uploads: pinning hundreds of megabytes costs more than it saves.
struct Stager {
    enum : size_t { STAGE_MAX = (size_t)24 << 20 };
    lvb_ctx* ctx; cudaStream_t s; bool staged; size_t used = 0;
    struct Item { void* buf; size_t off, count; void (*bind)(void*, unsigned char*, size_t, size_t); };
    std::vector<Item> items;
    std::vector<unsigned char> scratch;               // direct mode: the memory reserve() hands out
    void* pending_buf = nullptr; size_t pending_count = 0; int (*pending_up)(void*, const void*, size_t, cudaStream_t) = nullptr;
    template <class T> static void bind_fn(void* b, unsigned char* base, size_t off, size_t count) { static_cast<DevBuf<T>*>(b)->set_view(reinterpret_cast<T*>(base + off), count); }
    template <class T> static int up_fn(void* b, const void* src, size_t count, cudaStream_t st) { return static_cast<DevBuf<T>*>(b)->upload(static_cast<const T*>(src), count, st); }
    Stager(lvb_ctx* c, size_t estimate) : ctx(c), s(c->stream), staged(estimate <= STAGE_MAX) {
        static const bool off = getenv("LVB_NO_STAGING") && getenv("LVB_NO_STAGING")[0] == '1';      // A/B switch
        if (off) staged = false;
    }
    int begin() {
        if (!staged) return LVB_OK;
        if (!ctx->stage_ev) LVB_CUDA(cudaEventCreateWithFlags(&ctx->stage_ev, cudaEventDisableTiming));
        if (ctx->stage_busy) { LVB_CUDA(cudaEventSynchronize(ctx->stage_ev)); ctx->stage_busy = false; }      // the previous problem's copy has read it
        return LVB_OK;
    }
    int grow(size_t need) {
        if (need <= ctx->stage_cap) return LVB_OK;
        size_t cap = std::max<size_t>(std::max<size_t>(2 * ctx->stage_cap, need), (size_t)4 << 20);
        unsigned char* q = nullptr;
        LVB_CUDA(cudaHostAlloc((void**)&q, cap, cudaHostAllocDefault));
        if (used) memcpy(q, ctx->stage_h, used);
        if (ctx->stage_h) cudaFreeHost(ctx->stage_h);
        ctx->stage_h = q; ctx->stage_cap = cap;
        return LVB_OK;
    }
    // memory for `count` elements of dst, to be filled by the caller before the next reserve / put; finish() after filling
    template <class T> int reserve(DevBuf<T>& dst, size_t count, T** out) {
        const size_t c = std::max<size_t>(count, 1), bytes = c * sizeof(T);
        if (staged) {
            const size_t off = (used + 255) & ~(size_t)255;
            LVB_TRY(grow(off + bytes + 256));
            if (off > used) memset(ctx->stage_h + used, 0, off - used);
            items.push_back({&dst, off, c, &bind_fn<T>});
            used = off + bytes;
            *out = reinterpret_cast<T*>(ctx->stage_h + off);
        } else {
            scratch.resize(bytes);
            pending_buf = &dst; pending_count = count; pending_up = &up_fn<T>;
            *out = reinterpret_cast<T*>(scratch.data());
        }
        return LVB_OK;
    }
    int finish() {
        if (staged || !pending_buf) return LVB_OK;
        void* b = pending_buf; pending_buf = nullptr;
        return pending_up(b, scratch.data(), pending_count, s);      // pageable source: the call returns once it has been staged by the driver
    }
    template <class T> int put(DevBuf<T>& dst, const T* src, size_t count) {
        if (!staged) return dst.upload(src, count, s);
        T* q = nullptr;
        LVB_TRY(reserve(dst, count, &q));
        if (count) memcpy(q, src, count * sizeof(T));
        return LVB_OK;
    }
    int commit(DevBuf<unsigned char>& arena) {
        if (!staged) return LVB_OK;
        // a fresh allocation every time: the views of an earlier finalize may still be referenced by work in flight on the stream
        arena.release();
        LVB_TRY(arena.ensure(std::max<size_t>(used, 256)));
        LVB_CUDA(cudaMemcpyAsync(arena.p, ctx->stage_h, used, cudaMemcpyHostToDevice, s));
        LVB_CUDA(cudaEventRecord(ctx->stage_ev, s));
        ctx->stage_busy = true;
        for (const Item& it : items) it.bind(it.buf, arena.p, it.off, it.count);
        return LVB_OK;
    }
};

extern "C" {

int lvb_ba_create(lvb_ctx* ctx, lvb_ba** out) {
    if (!ctx || !out) { set_error("null argument"); return LVB_ERR_INVALID; }
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    LVB_TRY(init_tables());
    lvb_ba* b = new lvb_ba();
    b->ctx = ctx;
    *out = b;
    return LVB_OK;
}
void lvb_ba_destroy(lvb_ba* ba) { if (ba) { cudaSetDevice(ba->ctx->device); drop_graph(ba); delete ba; } }

int lvb_ba_set_cameras(lvb_ba* ba, const double cam[22]) { memcpy(ba->cam, cam, sizeof(ba->cam)); ba->have_cam = true; ba->finalized = false; return LVB_OK; }

static void assign_const(std::vector<uint8_t>& dst, const uint8_t* c, int n) { if (c) dst.assign(c, c + n); else dst.assign(n, 0); }
int lvb_ba_set_poses(lvb_ba* ba, int n, const double* v, const uint8_t* c) {
    if (n < 0 || (n && !v)) { set_error("bad poses"); return LVB_ERR_INVALID; }
    ba->h_poses.assign(v, v + (size_t)7 * n); assign_const(ba->h_pose_const, c, n); ba->finalized = false; return LVB_OK;
}
int lvb_ba_set_vec3(lvb_ba* ba, int n, const double* v, const uint8_t* c) {
    if (n < 0 || (n && !v)) { set_error("bad vec3"); return LVB_ERR_INVALID; }
    ba->h_vec3.assign(v, v + (size_t)3 * n); assign_const(ba->h_vec3_const, c, n); ba->finalized = false; return LVB_OK;
}
int lvb_ba_set_inv_depths(lvb_ba* ba, int n, const double* v, const uint8_t* c) {
    if (n < 0 || (n && !v)) { set_error("bad inverse depths"); return LVB_ERR_INVALID; }
    ba->h_rho.assign(v, v + n); assign_const(ba->h_rho_const, c, n); ba->finalized = false; return LVB_OK;
}
int lvb_ba_add_factors(lvb_ba* ba, int kind, int n, const double* consts, const int32_t* idx) {
    if (kind < 0 || kind >= 6 || n < 0 || (n && (!consts || !idx))) { set_error("bad factor arguments"); return LVB_ERR_INVALID; }
    ba->h_fc[kind].insert(ba->h_fc[kind].end(), consts, consts + (size_t)n * kConstStride[kind]);
    ba->h_fi[kind].insert(ba->h_fi[kind].end(), idx, idx + (size_t)n * kIdxStride[kind]);
    ba->n[kind] += n; ba->finalized = false;
    return LVB_OK;
}
int lvb_ba_set_loss(lvb_ba* ba, int kind, double a) {
    if (kind < 0 || kind >= 6) { set_error("bad kind"); return LVB_ERR_INVALID; }
    ba->huber[kind] = a;
    if (ba->finalized) { ba->dev.huber[kind] = a; drop_graph(ba); }
    return LVB_OK;
}

int lvb_ba_finalize(lvb_ba* ba) {
    static const bool prof_on = getenv("LVB_PROFILE") != nullptr;
    auto prof_t = std::chrono::steady_clock::now();
#define PROF(name) do { if (prof_on) { const auto t_ = std::chrono::steady_clock::now(); fprintf(stderr, "[finalize] %-28s %8.1f us\n", name, std::chrono::duration<double, std::micro>(t_ - prof_t).count()); prof_t = t_; } } while (0)
    lvb_ctx* ctx = ba->ctx;
    ba->host_fresh = false;
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    cudaStream_t s = ctx->stream;
    size_t stage_estimate = (ba->h_poses.size() + ba->h_vec3.size() + ba->h_rho.size()) * 24;
    for (int k = 0; k < 6; ++k) stage_estimate += ba->h_fc[k].size() * 8 + ba->h_fi[k].size() * 12;
    Stager stg(ctx, stage_estimate);
    LVB_TRY(stg.begin());
    if (!ba->have_cam) { set_error("cameras not set"); return LVB_ERR_STATE; }
    const int np = (int)ba->h_poses.size() / 7, nv = (int)ba->h_vec3.size() / 3, nr = (int)ba->h_rho.size();
    // validate indices (the TwoFrame list is the long one: a branch-free pass; the other kinds through the general rule)
    {
        const int32_t* ix = ba->h_fi[0].data();
        int bad = 0;
        for (int f = 0; f < ba->n[0]; ++f, ix += 3) bad |= ((unsigned)ix[0] >= (unsigned)nr) | ((unsigned)ix[1] >= (unsigned)np) | ((unsigned)ix[2] >= (unsigned)np);
        for (int k = bad ? 0 : 1; k < 6; ++k) for (int f = 0; f < ba->n[k]; ++f) for (int j = 0; j < kIdxStride[k]; ++j) {
            const int v = ba->h_fi[k][(size_t)f * kIdxStride[k] + j];
            int lim = np;
            if ((k == 0 && j == 0) || k == 2) lim = nr;
            if (k == 3 && j != 0 && j != 4) lim = nv;
            if (k == 3 && (j == 6 || j == 7) && v == -1 && ba->h_fc[3][(size_t)f * IMU_RAW + 467] >= 0.0) continue;     // ImuInitError has no j-side bias blocks
            if (v < 0 || v >= lim) { set_error("factor kind %d block %d: index %d out of range [0,%d)", k, f, v, lim); return LVB_ERR_INVALID; }
        }
    }
    PROF("validate");
    // slots / offsets.  Unknowns of the reduced camera system are ordered keyframe by keyframe
    // (pose_i, then the velocity / bias blocks an ImuError ties to pose_i): co-visibility and the IMU chain only
    // couple neighbouring keyframes, so S is block-banded and the Cholesky works inside its envelope.
    // `canon` is the caller-visible order (all poses, then all vec3 blocks) used by lvb_ba_reduced_system.
    std::vector<int> pose_off(np, -1), vec3_off(nv, -1), rho_slot(nr);
    int npf = 0, nvf = 0, nrf = 0;
    for (int i = 0; i < np; ++i) if (!ba->h_pose_const[i]) ++npf;
    for (int i = 0; i < nv; ++i) if (!ba->h_vec3_const[i]) ++nvf;
    for (int i = 0; i < nr; ++i) rho_slot[i] = ba->h_rho_const[i] ? -1 : nrf++;
    ba->n_pose_free = npf; ba->n_vec3_free = nvf; ba->n_rho_free = nrf; ba->dimc = 6 * npf + 3 * nvf;
    struct Blk { long long key; int type, idx, width; };
    std::vector<Blk> blks;
    {
        std::vector<int> vkey(nv, -1);
        if ((long long)np * 8 >= (1ll << 31)) { set_error("too many poses"); return LVB_ERR_UNSUPPORTED; }
        for (int f = 0; f < ba->n[3]; ++f) {
            const int32_t* ix = &ba->h_fi[3][8 * (size_t)f];
            for (int b = 1; b < 8; ++b) { if (b == 4) continue; const int v = ix[b]; if (v < 0) continue; const int p = ix[b < 4 ? 0 : 4]; if (vkey[v] < 0) vkey[v] = p * 8 + (b & 3); }
        }
        // sharded problems: a rank only sees the IMU factors it owns, but the order of the unknowns (= the layout of the
        // all-reduced system) must be the same on every rank: take the key any rank found (collective, like the envelope)
        if (ctx->world > 1 && nv > 0) {
            DevBuf<int> tmp;
            LVB_TRY(tmp.upload(vkey.data(), vkey.size(), s));
            LVB_TRY(comm_allreduce_max_i32(ctx, tmp.p, vkey.size()));
            LVB_CUDA(cudaMemcpyAsync(vkey.data(), tmp.p, vkey.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
            LVB_CUDA(cudaStreamSynchronize(s));
        }
        for (int i = 0; i < np; ++i) if (!ba->h_pose_const[i]) blks.push_back({(long long)i * 8, 0, i, 6});
        for (int i = 0; i < nv; ++i) if (!ba->h_vec3_const[i]) blks.push_back({vkey[i] >= 0 ? (long long)vkey[i] : (long long)np * 8 + i, 1, i, 3});
        std::stable_sort(blks.begin(), blks.end(), [](const Blk& a, const Blk& b) { return a.key < b.key; });
    }
    std::vector<int> blk_of_off(ba->dimc, 0), blk_start(blks.size() + 1, 0);
    ba->canon.assign(ba->dimc, 0);
    {
        int off = 0, ps = 0, vs = 0;
        std::vector<int> pslot(np, -1), vslot(nv, -1);
        for (int i = 0; i < np; ++i) if (!ba->h_pose_const[i]) pslot[i] = ps++;
        for (int i = 0; i < nv; ++i) if (!ba->h_vec3_const[i]) vslot[i] = vs++;
        for (size_t b = 0; b < blks.size(); ++b) {
            blk_start[b] = off;
            const int c0 = blks[b].type == 0 ? 6 * pslot[blks[b].idx] : 6 * npf + 3 * vslot[blks[b].idx];
            if (blks[b].type == 0) pose_off[blks[b].idx] = off; else vec3_off[blks[b].idx] = off;
            for (int k = 0; k < blks[b].width; ++k) { blk_of_off[off + k] = (int)b; ba->canon[off + k] = c0 + k; }
            off += blks[b].width;
        }
        blk_start[blks.size()] = off;
    }
    PROF("block order");
    // camera systems up to MAX_DIMC use dense lower-triangular storage, larger ones banded storage (decided below)
    const bool dense_layout = ba->dimc <= MAX_DIMC;
    ba->solvable = ba->dimc > 0;
    // ---- device order of the blocks.  TwoFrame blocks sorted by (pose_1, pose_2), PoseOnly blocks by pose, so that
    // a warp of the linearize kernel owns one key (or a few key segments) and can reduce its J^T J in shared memory
    // before touching HBM.  Dense-layout (window-sized) problems also pad every key run to a multiple of 32 with
    // weight-0 copies: one segment per warp.  Large problems stay unpadded (their runs are short, padding would
    // inflate the block arrays).
    for (int k = 0; k < 6; ++k) {
        std::vector<int>& ord = ba->order[k];
        ord.clear();
        const int n = ba->n[k];
        if (ba->solvable && (k == 0 || k == 1) && n > 0) {
            // stable order by key: counting sort when the key space is small (window-sized problems), else a pair sort
            std::vector<long long> keys(n);
            const long long key_space = (k == 0) ? (long long)np * np : (long long)np;
            for (int f = 0; f < n; ++f) keys[f] = (k == 0) ? (long long)ba->h_fi[0][3 * (size_t)f + 1] * np + ba->h_fi[0][3 * (size_t)f + 2] : (long long)ba->h_fi[1][f];
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
                while (dense_layout && ord.size() % 32) ord.push_back(-1 - ids[i]);     // padding: encoded source block
                i = j;
            }
        } else { ord.resize(n); for (int f = 0; f < n; ++f) ord[f] = f; }
        ba->nd[k] = (int)ord.size();
    }
    PROF("factor sort + pad");
    const int n_tf = ba->nd[0];
    // landmark CSR over device positions: TwoFrame i -> i, TwoCamera f -> -(f+1); padding is skipped.  The count runs over the caller's
    // order (sequential); the fill has to follow the device order, so its gather is prefetched, and it also notes the two free-pose
    // offsets of every entry (lm_off) so that the grouping below never goes back to the factor records.
    std::vector<int> lm_start(nr + 1, 0);
    {
        const int32_t* ix = ba->h_fi[0].data();
        for (int f = 0; f < ba->n[0]; ++f) lm_start[ix[3 * (size_t)f] + 1]++;
    }
    for (int f = 0; f < ba->n[2]; ++f) lm_start[ba->h_fi[2][f] + 1]++;
    for (int i = 0; i < nr; ++i) lm_start[i + 1] += lm_start[i];
    std::vector<int> lm_fac(std::max(1, lm_start[nr])), lm_off(2 * (size_t)std::max(1, lm_start[nr]), -1), fill(lm_start.begin(), lm_start.end() - 1);
    {
        const int32_t* hi = ba->h_fi[0].data();
        const int* ord = ba->order[0].data();
        for (int i = 0; i < n_tf; ++i) {
            if (i + 16 < n_tf && ord[i + 16] >= 0) __builtin_prefetch(hi + 3 * (size_t)ord[i + 16]);
            if (ord[i] < 0) continue;
            const int32_t* ix = hi + 3 * (size_t)ord[i];
            const int pos = fill[ix[0]]++;
            lm_fac[pos] = i; lm_off[2 * (size_t)pos] = pose_off[ix[1]]; lm_off[2 * (size_t)pos + 1] = pose_off[ix[2]];
        }
    }
    for (int f = 0; f < ba->n[2]; ++f) lm_fac[fill[ba->h_fi[2][f]]++] = -(f + 1);

    PROF("landmark CSR");
    // ---- Schur groups: landmarks with the same sorted set of free pose offsets share a warp-sized work item
    std::vector<int> tf_slot((size_t)std::max(1, n_tf) * 2, -1), sw_group, sw_lm, grp_ns, grp_off;
    int cols_max = 0;
    {
        // signature = sorted set of free pose offsets of a landmark; groups found through an open-addressing hash table
        // over the signatures (no per-landmark heap traffic), numbered in order of first appearance
        std::vector<std::vector<int>> members;
        size_t tsize = 64; while (tsize < 4 * (size_t)std::max(1, nrf)) tsize <<= 1;
        if (tsize > ((size_t)1 << 20)) tsize = (size_t)1 << 20;
        std::vector<int> table(tsize, -1);
        for (int l = 0; l < nr; ++l) {
            if (rho_slot[l] < 0) continue;
            int sig[MAX_TRACK + 1], ns = 0;
            for (int e = lm_start[l]; e < lm_start[l + 1]; ++e) {
                if (lm_fac[e] < 0) continue;
                for (int side = 1; side <= 2; ++side) {
                    const int off = lm_off[2 * (size_t)e + side - 1];
                    if (off < 0) continue;
                    int p = 0; while (p < ns && sig[p] < off) ++p;
                    if (p < ns && sig[p] == off) continue;
                    if (ns == MAX_TRACK) { set_error("landmark %d is observed from more than %d keyframes", l, (int)MAX_TRACK); return LVB_ERR_UNSUPPORTED; }
                    for (int q = ns; q > p; --q) sig[q] = sig[q - 1];
                    sig[p] = off; ++ns;
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
                    int p = 0; while (sig[p] != off) ++p;
                    tf_slot[(size_t)(side - 1) * n_tf + i] = p;
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
    }
    ba->n_schur_warps = (int)sw_group.size(); ba->schur_cols_max = cols_max;
    PROF("schur groups");
    // ---- envelope of S: first structurally non-zero column per row, from every coupling the assembly can create
    std::vector<int> chol_rmax(ba->dimc / 32 + 2, 0), chol_cmin(ba->dimc / 32 + 2, 0);
    int band = 0, panel_rows = 2, true_band = 0;
    if (ba->solvable) {
        std::vector<int> first(ba->dimc);
        std::vector<int> fb(blks.size());
        for (size_t b = 0; b < blks.size(); ++b) fb[b] = blk_start[b];
        auto couple = [&](int offA, int offB) {
            if (offA < 0 || offB < 0) return;
            const int a = blk_of_off[offA], b = blk_of_off[offB];
            const int lo = std::min(a, b), hi = std::max(a, b);
            fb[hi] = std::min(fb[hi], blk_start[lo]);
        };
        for (size_t g = 0; g < grp_ns.size(); ++g) for (int a = 0; a < grp_ns[g]; ++a) for (int b = 0; b < a; ++b) couple(grp_off[g * MAX_TRACK + a], grp_off[g * MAX_TRACK + b]);
        for (int f = 0; f < ba->n[0]; ++f) couple(pose_off[ba->h_fi[0][3 * (size_t)f + 1]], pose_off[ba->h_fi[0][3 * (size_t)f + 2]]);
        for (int f = 0; f < ba->n[3]; ++f) {
            const int32_t* ix = &ba->h_fi[3][8 * (size_t)f];
            int offs[8];
            for (int b = 0; b < 8; ++b) offs[b] = ix[b] < 0 ? -1 : ((b == 0 || b == 4) ? pose_off[ix[b]] : vec3_off[ix[b]]);
            for (int a = 0; a < 8; ++a) for (int b = 0; b < a; ++b) couple(offs[a], offs[b]);
        }
        for (int f = 0; f < ba->n[4]; ++f) couple(pose_off[ba->h_fi[4][2 * (size_t)f]], pose_off[ba->h_fi[4][2 * (size_t)f + 1]]);
        // sharded problems: the other ranks' couplings arrive with the all-reduce, so the envelope must be the global one
        if (ctx->world > 1) {
            DevBuf<int> tmp;
            LVB_TRY(tmp.upload(fb.data(), fb.size(), s));
            LVB_TRY(comm_allreduce_min_i32(ctx, tmp.p, fb.size()));
            LVB_CUDA(cudaMemcpyAsync(fb.data(), tmp.p, fb.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
            LVB_CUDA(cudaStreamSynchronize(s));
        }
        for (int r = 0; r < ba->dimc; ++r) { first[r] = fb[blk_of_off[r]]; true_band = std::max(true_band, r - first[r]); }
        // rmax per 32-column step by a backward sweep: rows whose first column lies left of the end of the step
        {
            const int nstep = (ba->dimc + 31) / 32;
            std::vector<int> last_row_of_col(ba->dimc, 0);      // largest row r with first[r] <= c, via prefix max over c
            for (int c = 0; c < ba->dimc; ++c) last_row_of_col[c] = c;
            for (int r = 0; r < ba->dimc; ++r) last_row_of_col[first[r]] = std::max(last_row_of_col[first[r]], r);
            for (int c = 1; c < ba->dimc; ++c) last_row_of_col[c] = std::max(last_row_of_col[c], last_row_of_col[c - 1]);
            for (int step = 0; step < nstep; ++step) {
                const int kb = step * 32, bs = std::min(32, ba->dimc - kb);
                int cmin = kb;
                for (int r = kb; r < kb + bs; ++r) cmin = std::min(cmin, first[r]);
                const int rmax = std::max(kb + bs - 1, last_row_of_col[kb + bs - 1]);
                chol_rmax[step] = rmax; chol_cmin[step] = cmin;
                band = std::max(band, std::max(rmax - kb, kb + bs - 1 - cmin));
                panel_rows = std::max(panel_rows, rmax - (kb + bs) + 2);
            }
        }
    }
    // ---- storage of Hpp / S
    // the envelope above is the one of GLOBAL 32-column steps; the fronts of the separator tree step through 32 columns from their
    // own first unknown, and for an arbitrary start a block column needs rows up to true_band + 31 below its first column
    if (!dense_layout) band = std::max(band, true_band + 31);
    band = std::min(std::max(band, 31), std::max(31, ba->dimc - 1));
    if (dense_layout) { ba->srow = ba->dimc; ba->soff = 0; ba->nS = (size_t)ba->dimc * ba->dimc; }
    else              { ba->srow = band; ba->soff = band; ba->nS = (size_t)ba->dimc * (size_t)(band + 1); }
    ba->band = band; ba->panel_rows = panel_rows;
    ba->chol_smem = (size_t)(CHOL_HDR + std::max(panel_rows + 2, 34) * 34) * 8;      // two diagonal-block buffers + the panel (>= 34 rows; later the backward partial sums)
    // banded systems: split the chain by a separator tree when the band leaves room for at least two leaves (ba_tree.cuh)
    ba->tree_levels = 0;
    std::vector<Front> h_fronts;
    size_t pool_doubles = 0;
    {
        static const bool no_tree = getenv("LVB_NO_TREE") && getenv("LVB_NO_TREE")[0] == '1';
        int rows = 0, mnb = 0, max_leaves = 1;
        while (max_leaves * 2 <= std::max(2, ctx->sm_count)) max_leaves *= 2;
        if (ba->solvable && !dense_layout && !no_tree) {
            const int lv = build_front_tree(ba->dimc, band, true_band, max_leaves, h_fronts, ba->level_first, ba->level_count, pool_doubles, rows, mnb);
            const size_t fs = (size_t)(32 * 33 + 32 + 128 + (rows + 2) * 34) * 8, bs_ = (size_t)(((mnb + 1) & ~1) + (CHOL_T / 32) * 32) * 8;
            if (lv > 0 && fs <= 227 * 1024 - 256 && pool_doubles < ((size_t)1 << 31)) { ba->tree_levels = lv; ba->tree_factor_smem = fs; ba->tree_back_smem = bs_; }
        }
    }
    // loop-closure shaped envelopes: neither a tree nor a panel that fits in shared memory -- the per-phase grids of ba_wide.cuh
    ba->wide_solver = ba->solvable && ba->tree_levels == 0 && ba->chol_smem > 227 * 1024 - 256;
    ba->h_rmax = chol_rmax;
    if (ba->solvable && ba->nS > ((size_t)3 << 30)) { ba->solvable = false; ba->unsolvable_why = "the banded reduced camera system exceeds 24 GB"; }
    if (!ba->solvable) ba->nS = 1;
    if (sw_group.empty()) { sw_group.push_back(0); sw_lm.assign(32, -1); }
    if (grp_ns.empty()) { grp_ns.push_back(0); grp_off.assign(MAX_TRACK, -1); }

    PROF("envelope");
    LVB_TRY(stg.put(ba->poses, ba->h_poses.data(), ba->h_poses.size()));
    LVB_TRY(stg.put(ba->vec3, ba->h_vec3.data(), ba->h_vec3.size()));
    LVB_TRY(stg.put(ba->rho, ba->h_rho.data(), ba->h_rho.size()));
    LVB_TRY(stg.put(ba->c_poses, ba->h_poses.data(), ba->h_poses.size()));
    LVB_TRY(stg.put(ba->c_vec3, ba->h_vec3.data(), ba->h_vec3.size()));
    LVB_TRY(stg.put(ba->c_rho, ba->h_rho.data(), ba->h_rho.size()));
    LVB_TRY(stg.put(ba->pose_off, pose_off.data(), np));
    LVB_TRY(stg.put(ba->vec3_off, vec3_off.data(), nv));
    LVB_TRY(stg.put(ba->rho_slot, rho_slot.data(), nr));
    LVB_TRY(stg.put(ba->lm_start, lm_start.data(), nr + 1));
    LVB_TRY(stg.put(ba->lm_fac, lm_fac.data(), lm_fac.size()));
    LVB_TRY(stg.put(ba->tf_slot, tf_slot.data(), tf_slot.size()));
    LVB_TRY(stg.put(ba->sw_group, sw_group.data(), sw_group.size()));
    LVB_TRY(stg.put(ba->sw_lm, sw_lm.data(), sw_lm.size()));
    LVB_TRY(stg.put(ba->grp_ns, grp_ns.data(), grp_ns.size()));
    LVB_TRY(stg.put(ba->grp_off, grp_off.data(), grp_off.size()));
    LVB_TRY(stg.put(ba->chol_rmax, chol_rmax.data(), chol_rmax.size()));
    LVB_TRY(stg.put(ba->chol_cmin, chol_cmin.data(), chol_cmin.size()));
    if (ba->tree_levels > 0) { LVB_TRY(stg.put(ba->fronts, h_fronts.data(), h_fronts.size())); LVB_TRY(ba->front_pool.ensure(pool_doubles)); }
    // tensor-core Schur operands: compact pose dimensions (<= 128) and the zero-initialised split-bf16 U^T tiles
    ba->tc_ok = ba->solvable && dense_layout && 6 * npf <= 128 && npf > 0 && ctx->world == 1;
    {
        std::vector<int> cdim(std::max(1, ba->dimc), -1), coff(128, -1);
        int c = 0;
        for (size_t b = 0; b < blks.size(); ++b) if (blks[b].type == 0 && c + 6 <= 128) { for (int k = 0; k < 6; ++k) { cdim[blk_start[b] + k] = c + k; coff[c + k] = blk_start[b] + k; } c += 6; }
        LVB_TRY(stg.put(ba->tc_cdim, cdim.data(), cdim.size()));
        LVB_TRY(stg.put(ba->tc_off, coff.data(), coff.size()));
        ba->n_tc_chunks = ba->tc_ok ? ((2 * ba->n_schur_warps + TC_CHUNKS - 1) / TC_CHUNKS) * TC_CHUNKS : 0;
        LVB_TRY(ba->tc_u.ensure((size_t)std::max(1, ba->n_tc_chunks) * 3 * 2048));
        LVB_CUDA(cudaMemsetAsync(ba->tc_u.p, 0, (size_t)std::max(1, ba->n_tc_chunks) * 3 * 2048 * sizeof(unsigned short), s));
    }

    PROF("uploads (params, structure)");
    // factor planes in device order (AoS -> SoA transpose on the host, written straight into the staging area; IMU stays AoS and
    // is packed on the device).  The one copy to the device is issued when the last array is in place; the IMU kernel follows it.
    {
        for (int k = 0; k < 6; ++k) {
            const int n = ba->nd[k];
            const std::vector<int>& ord = ba->order[k];
            const int is = kIdxStride[k];
            int* iplanes = nullptr;
            LVB_TRY(stg.reserve(ba->fi[k], (size_t)std::max(1, n) * is, &iplanes));
            if (n == 0) std::fill(iplanes, iplanes + is, 0);
            const int32_t* hi = ba->h_fi[k].data();
            // record-major walk: one contiguous source record per block, `is` / `cs` output streams (the plane-major walk re-read the
            // strided source once per plane); the device order is a permutation of the caller's, so the gather prefetches its records
            if (is == 3) gather_index_planes<3>(iplanes, hi, ord.data(), n);
            else if (is == 1) gather_index_planes<1>(iplanes, hi, ord.data(), n);
            else for (int i = 0; i < n; ++i) { const int f = ord[i] >= 0 ? ord[i] : -1 - ord[i]; const int32_t* src = hi + (size_t)f * is; for (int j = 0; j < is; ++j) iplanes[(size_t)j * n + i] = src[j]; }
            LVB_TRY(stg.finish());
            if (k == 3) continue;
            const int cs = kConstStride[k];
            double* planes = nullptr;
            LVB_TRY(stg.reserve(ba->fc[k], (size_t)std::max(1, n) * cs, &planes));
            if (n == 0) std::fill(planes, planes + cs, 0.0);
            const int wcol = (k == 0) ? 4 : (k == 1 ? 5 : -1);     // weight column, zeroed on padding
            const double* hc = ba->h_fc[k].data();
            if (cs == 5) gather_planes<5>(planes, hc, ord.data(), n, wcol);
            else if (cs == 6) gather_planes<6>(planes, hc, ord.data(), n, wcol);
            else for (int i = 0; i < n; ++i) {
                const bool pad = ord[i] < 0;
                const double* src = hc + (size_t)(pad ? -1 - ord[i] : ord[i]) * cs;
                for (int j = 0; j < cs; ++j) planes[(size_t)j * n + i] = (pad && j == wcol) ? 0.0 : src[j];
            }
            LVB_TRY(stg.finish());
        }
        const int n = ba->nd[3];
        LVB_TRY(stg.put(ba->imu_raw, ba->h_fc[3].data(), ba->h_fc[3].size()));
        LVB_TRY(stg.commit(ba->upload_arena));      // everything uploaded so far: one copy
        LVB_TRY(ba->fc[3].ensure((size_t)std::max(1, n) * IMU_STRIDE));
        LVB_TRY(ba->imu_status.ensure(std::max(1, n)));
        if (n) {
            imu_prepare_kernel<<<nblk(n, 4), 128, 0, s>>>(ba->imu_raw.p, ba->fc[3].p, n, ba->imu_status.p);
            ctx->launches++;
            LVB_TRY(check_launch("imu_prepare"));
            ba->imu_checked = false;      // status is read back with the first solve / eval (no extra round trip here)
        }
    }
    PROF("planes + uploads");

    const size_t nH = ba->nS;
    LVB_TRY(ba->chol_invd.ensure(ba->dimc + 32));
    LVB_TRY(ba->Hpp.ensure(nH)); LVB_TRY(ba->gc.ensure(ba->dimc));
    LVB_TRY(ba->Hll.ensure(std::max(1, nr))); LVB_TRY(ba->gl.ensure(std::max(1, nr)));
    LVB_TRY(ba->tf_w.ensure((size_t)std::max(1, ba->nd[0]) * 12));
    LVB_TRY(ba->arena.ensure(nH + 3 * (size_t)ba->dimc + 16));
    LVB_TRY(ba->scale_c.ensure(ba->dimc)); LVB_TRY(ba->lam_c.ensure(ba->dimc));
    LVB_TRY(ba->scale_l.ensure(std::max(1, nr))); LVB_TRY(ba->lam_l.ensure(std::max(1, nr)));
    LVB_TRY(ba->st.ensure(1));

    PROF("sync + alloc");
    BaDev& d = ba->dev;
    d.n_poses = np; d.n_vec3 = nv; d.n_rho = nr; d.dimc = ba->dimc; d.n_pose_free = npf;
    d.srow = ba->srow; d.soff = ba->soff; d.nS = ba->nS;
    d.poses = ba->poses.p; d.vec3 = ba->vec3.p; d.rho = ba->rho.p; d.c_poses = ba->c_poses.p; d.c_vec3 = ba->c_vec3.p; d.c_rho = ba->c_rho.p;
    d.pose_off = ba->pose_off.p; d.vec3_off = ba->vec3_off.p; d.rho_slot = ba->rho_slot.p;
    for (int k = 0; k < 6; ++k) { d.n[k] = ba->nd[k]; d.fc[k] = ba->fc[k].p; d.fi[k] = ba->fi[k].p; d.huber[k] = ba->huber[k]; }
    d.lm_start = ba->lm_start.p; d.lm_fac = ba->lm_fac.p;
    d.tf_slot = ba->tf_slot.p; d.sw_group = ba->sw_group.p; d.sw_lm = ba->sw_lm.p; d.grp_ns = ba->grp_ns.p; d.grp_off = ba->grp_off.p;
    d.n_schur_warps = ba->n_schur_warps; d.warp_syrk = 1;
    d.tc_mode = 0; d.tc_u = ba->tc_u.p; d.tc_cdim = ba->tc_cdim.p; d.tc_off = ba->tc_off.p; d.tc_ndim = 6 * npf;
    d.Hpp = ba->Hpp.p; d.gc = ba->gc.p; d.Hll = ba->Hll.p; d.gl = ba->gl.p; d.tf_w = ba->tf_w.p;
    d.S = ba->arena.p; d.rhs = d.S + nH; d.gcr = d.rhs + ba->dimc; d.diagH = d.gcr + ba->dimc; d.scal = d.diagH + ba->dimc;
    d.scale_c = ba->scale_c.p; d.scale_l = ba->scale_l.p; d.lam_c = ba->lam_c.p; d.lam_l = ba->lam_l.p;
    d.st = ba->st.p;
    d.rank = ctx->rank; d.world = ctx->world; d.rank0 = (ctx->rank == 0) ? 1 : 0;
    d.stage_poses = (np <= MAX_STAGE_POSES) ? (ctx->use_tma ? 2 : 1) : 0;
    d.cams.c0 = make_cam(ba->cam); d.cams.c1 = make_cam(ba->cam + 11);

    BlockRanges& R = ba->ranges;
    R.b[0] = 0;
    R.b[1] = R.b[0] + nblk(ba->nd[0], TPB);
    R.b[2] = R.b[1] + nblk(ba->nd[1], TPB);
    R.b[3] = R.b[2] + nblk(ba->nd[2], TPB);
    d.imu_cta = dense_layout ? 1 : 0;
    R.b[4] = R.b[3] + (d.imu_cta ? ba->nd[3] : nblk(ba->nd[3], 4));
    R.b[5] = R.b[4] + nblk(ba->nd[4], TPB);
    R.b[6] = R.b[5] + nblk(ba->nd[5], TPB);
    const size_t smem_imu = d.imu_cta ? (size_t)(480 * 2 + 32 + IMU_STRIDE) * 8 + 32 * 4 : (size_t)(4 * 480 * 2 + 4 * 32) * 8 + 4 * 32 * 4;
    const size_t smem_pose = d.stage_poses ? ((size_t)np * 56 + 16) : 0;
    drop_graph(ba);
    ba->pose_smem = smem_pose; ba->imu_smem = smem_imu;
    ba->lin_smem = ((smem_pose + 15) & ~(size_t)15) + (size_t)(TPB / 32) * SYRK_ROWS * SYRK_LD * 8;
    ba->schur_smem = (size_t)(TPB / 32) * 32 * (size_t)std::max(1, cols_max) * 8;
    PROF("tail");
#undef PROF
    ba->finalized = true;
    return LVB_OK;
}

int lvb_ba_dims(lvb_ba* ba, int* dimc, int* nrf, int* rows) {
    if (!ba->finalized) { set_error("finalize first"); return LVB_ERR_STATE; }
    if (dimc) *dimc = ba->dimc;
    if (nrf) *nrf = ba->n_rho_free;
    if (rows) { int r = 0; for (int k = 0; k < 6; ++k) r += ba->n[k] * kResDim[k]; *rows = r; }
    return LVB_OK;
}

int lvb_ba_update_params(lvb_ba* ba, const double* P, const double* V, const double* R) {
    if (!ba->finalized) { set_error("finalize first"); return LVB_ERR_STATE; }
    cudaStream_t s = ba->ctx->stream;
    ba->host_fresh = false;
    LVB_CUDA(cudaSetDevice(ba->ctx->device)); lvb::g_alloc_stream = ba->ctx->stream;
    if (P) { ba->h_poses.assign(P, P + ba->h_poses.size()); LVB_TRY(ba->poses.upload(P, ba->h_poses.size(), s)); }
    if (V) { ba->h_vec3.assign(V, V + ba->h_vec3.size()); LVB_TRY(ba->vec3.upload(V, ba->h_vec3.size(), s)); }
    if (R) { ba->h_rho.assign(R, R + ba->h_rho.size()); LVB_TRY(ba->rho.upload(R, ba->h_rho.size(), s)); }
    LVB_CUDA(cudaStreamSynchronize(s));
    return LVB_OK;
}

static int check_imu_status(lvb_ba* ba) {
    if (ba->imu_checked || ba->nd[3] == 0) { ba->imu_checked = true; return LVB_OK; }
    std::vector<int> status(ba->nd[3]);
    LVB_TRY(ba->imu_status.download(status.data(), status.size(), ba->ctx->stream));
    LVB_CUDA(cudaStreamSynchronize(ba->ctx->stream));
    for (size_t f = 0; f < status.size(); ++f) if (status[f]) { set_error("ImuError %d: covariance is singular or not finite (code %d)", (int)f, status[f]); return LVB_ERR_NUMERIC; }
    ba->imu_checked = true;
    return LVB_OK;
}

static int launch_eval(lvb_ba* ba, int kind, double* r_dev, double* J_dev) {
    const int n = ba->nd[kind];
    if (n == 0) return LVB_OK;
    BaDev& d = ba->dev;
    switch (kind) {
    case 0: {
        const size_t pose_b = d.stage_poses ? (size_t)d.n_poses * 56 + 16 : 0;
        const int v = ba->ctx->eval_variant;       // LVB_EVAL_VARIANT: 0 staged/5 CTAs, 1 staged/6, 2 direct/5, 3 direct/6
        if (v == 1) LAUNCH(ba, (ba_eval_two_frame_kernel<1, 6>), nblk(n, TPB), TPB, (size_t)(TPB * 31) * 8 + pose_b, d, r_dev, J_dev);
        else if (v == 2) LAUNCH(ba, (ba_eval_two_frame_kernel<0, 5>), nblk(n, TPB), TPB, pose_b, d, r_dev, J_dev);
        else if (v == 3) LAUNCH(ba, (ba_eval_two_frame_kernel<0, 6>), nblk(n, TPB), TPB, pose_b, d, r_dev, J_dev);
        else LAUNCH(ba, (ba_eval_two_frame_kernel<1, 5>), nblk(n, TPB), TPB, (size_t)(TPB * 31) * 8 + pose_b, d, r_dev, J_dev);
        break; }
    case 1: LAUNCH(ba, ba_eval_pose_only_kernel, nblk(n, TPB), TPB, 0, d, r_dev, J_dev); break;
    case 2: LAUNCH(ba, ba_eval_two_camera_kernel, nblk(n, TPB), TPB, 0, d, r_dev, J_dev); break;
    case 3: LAUNCH(ba, ba_eval_imu_kernel, nblk(n, 4), TPB, 0, d, r_dev, J_dev); break;
    default: LAUNCH(ba, ba_eval_prior_kernel, nblk(n, 64), 64, 0, d, kind, r_dev, J_dev); break;
    }
    return check_launch("ba_eval");
}

static int ensure_eval_buffers(lvb_ba* ba, int kind) {
    const size_t n = ba->nd[kind];
    LVB_TRY(ba->eval_r.ensure(std::max<size_t>(1, n * kResDim[kind])));
    LVB_TRY(ba->eval_J.ensure(std::max<size_t>(1, n * kResDim[kind] * kJacCols[kind])));
    return LVB_OK;
}

int lvb_ba_eval(lvb_ba* ba, int kind, double* r, double* J) {
    if (!ba->finalized) { set_error("finalize first"); return LVB_ERR_STATE; }
    if (kind < 0 || kind >= 6) { set_error("bad kind"); return LVB_ERR_INVALID; }
    LVB_CUDA(cudaSetDevice(ba->ctx->device)); lvb::g_alloc_stream = ba->ctx->stream;
    LVB_TRY(check_imu_status(ba));
    LVB_TRY(ensure_eval_buffers(ba, kind));
    LVB_TRY(launch_eval(ba, kind, ba->eval_r.p, ba->eval_J.p));
    const size_t nd = ba->nd[kind], rd = kResDim[kind], jd = (size_t)kResDim[kind] * kJacCols[kind];
    const std::vector<int>& ord = ba->order[kind];
    bool identity = (nd == (size_t)ba->n[kind]);
    for (size_t i = 0; identity && i < nd; ++i) identity = (ord[i] == (int)i);
    cudaStream_t s = ba->ctx->stream;
    if (identity) {
        if (r) LVB_TRY(ba->eval_r.download(r, nd * rd, s));
        if (J) LVB_TRY(ba->eval_J.download(J, nd * jd, s));
        LVB_CUDA(cudaStreamSynchronize(s));
        return LVB_OK;
    }
    // the device layout is sorted / padded: hand the rows back in the caller's block order
    std::vector<double> hr(r ? nd * rd : 0), hJ(J ? nd * jd : 0);
    if (r) LVB_TRY(ba->eval_r.download(hr.data(), nd * rd, s));
    if (J) LVB_TRY(ba->eval_J.download(hJ.data(), nd * jd, s));
    LVB_CUDA(cudaStreamSynchronize(s));
    for (size_t i = 0; i < nd; ++i) {
        if (ord[i] < 0) continue;
        if (r) memcpy(r + (size_t)ord[i] * rd, hr.data() + i * rd, rd * sizeof(double));
        if (J) memcpy(J + (size_t)ord[i] * jd, hJ.data() + i * jd, jd * sizeof(double));
    }
    return LVB_OK;
}

int lvb_ba_eval_device(lvb_ba* ba, int kind) {
    if (!ba->finalized) { set_error("finalize first"); return LVB_ERR_STATE; }
    if (kind < 0 || kind >= 6) { set_error("bad kind"); return LVB_ERR_INVALID; }
    lvb::g_alloc_stream = ba->ctx->stream;
    LVB_TRY(ensure_eval_buffers(ba, kind));
    return launch_eval(ba, kind, ba->eval_r.p, ba->eval_J.p);
}

static bool merged_linearize(lvb_ba* ba) {
    static const bool off = getenv("LVB_NO_MERGED_LINEARIZE") && getenv("LVB_NO_MERGED_LINEARIZE")[0] == '1';
    return !off && ba->srow == ba->dimc && ba->soff == 0 && ba->ranges.b[3] > 0 && ba->ranges.b[6] > ba->ranges.b[3];      // dense layout = window-sized
}

static bool use_side_branch(lvb_ba* ba) {
    // not inside a captured graph: replaying a graph with parallel branches was measured to be erratic (0.19 - 0.9 ms per
    // pass on the same build), a linear graph is stable
    return ba->ctx->use_side && ba->ctx->side && !g_timing && !ba->capturing && ba->ranges.b[3] > 0 && ba->ranges.b[6] > ba->ranges.b[3];
}

// one pass = one LM iteration attempt (all decisions on the device), 10 launches (the two linearise kernels and the two
// cost kernels run as parallel branches on a second stream):
//   linearize (visual) | linearize (IMU + priors) | build S | Schur | camera damping | Cholesky (+ LM pre-check)
//   | back-substitution + candidate | cost (visual) | cost (IMU + priors) | LM decision + accept + clear
static int launch_linearize_and_reduce(lvb_ba* ba, bool standalone) {
    BaDev& d = ba->dev;
    lvb_ctx* ctx = ba->ctx;
    const size_t nH = d.nS;
    // the visual and the IMU / prior linearisations are independent (both only add into the accumulators): one grid for both at
    // window size, two kernels (parallel branches when launched directly) at map scale
    const bool one_grid = merged_linearize(ba);
    const bool fork = !one_grid && use_side_branch(ba);
    if (one_grid) LAUNCH(ba, ba_linearize_all_kernel<0>, ba->ranges.b[6], TPB, std::max(ba->lin_smem, ba->imu_smem), d, ba->ranges);
    else {
    if (fork) { LVB_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream)); LVB_CUDA(cudaStreamWaitEvent(ctx->side, ctx->ev_fork, 0)); }
    LAUNCH(ba, ba_linearize_kernel<0>, ba->ranges.b[3], TPB, ba->lin_smem, d, ba->ranges);
    if (fork) {
        LAUNCH_ON(ba, ctx->side, ba_linearize_other_kernel<0>, ba->ranges.b[6] - ba->ranges.b[3], TPB, ba->imu_smem, d, ba->ranges);
        LVB_CUDA(cudaEventRecord(ctx->ev_join, ctx->side)); LVB_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    } else LAUNCH(ba, ba_linearize_other_kernel<0>, ba->ranges.b[6] - ba->ranges.b[3], TPB, ba->imu_smem, d, ba->ranges);
    }
    const bool fuse_damp = ctx->world == 1;
    if (fuse_damp) LAUNCH(ba, ba_build_S_kernel<1>, std::min(1024, nblk(nH, 256)), 256, 0, d);
    else LAUNCH(ba, ba_build_S_kernel<0>, std::min(1024, nblk(nH, 256)), 256, 0, d);
    LAUNCH(ba, ba_schur_kernel, nblk(d.n_schur_warps, TPB / 32), TPB, ba->schur_smem, d, std::max(1, ba->schur_cols_max));
    if (d.tc_mode) LAUNCH(ba, ba_schur_tc_kernel, ba->n_tc_chunks / TC_CHUNKS, 128, (size_t)TC_CHUNKS * TC_CHUNK_BYTES, d, ba->n_tc_chunks);
    const size_t n_arena = nH + 3 * (size_t)d.dimc + 16;
    P2PArgs pa;
    const bool fused_comm = ctx->world > 1 && comm_p2p_args(ctx, n_arena, &pa) && (size_t)(d.n_poses + d.n_vec3) <= 4096;
    if (fused_comm) {
        LAUNCH(ba, ba_allreduce_fused_kernel, (int)std::max<size_t>(1, std::min<size_t>(XB_BLOCKS, (n_arena + 255) / 256)), 256, 0, pa, d, (int)n_arena);
    } else if (ctx->world > 1) {
        LAUNCH(ba, ba_pack_scalars_kernel, 1, 1, 0, d);
        LVB_TRY(comm_allreduce_sum_f64(ctx, d.S, n_arena));
        LAUNCH(ba, ba_unpack_scalars_kernel, 1, 1, 0, d);
    }
    // (fusing this into the Cholesky prologue was measured: it perturbs that kernel's register allocation and is slower)
    if (!fuse_damp && !fused_comm) LAUNCH(ba, ba_prepare_camera_kernel, nblk(d.n_poses + d.n_vec3, 128), 128, 0, d);
    if (standalone) LAUNCH(ba, lm_control_pre_kernel, 1, 1, 0, d.st);
    return check_launch("linearize");
}

// rhs <- S^-1 rhs (+ the LM pre-check): multifrontal tree over the banded system, or the single-CTA envelope Cholesky
static int launch_wide_solve(lvb_ba* ba) {
    BaDev& d = ba->dev;
    const int n = d.dimc;
    static bool attr_set = false;
    if (!attr_set) { LVB_CUDA(cudaFuncSetAttribute(ba_wide_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WIDE_WARPS * 2 * 32 * 34 * 8)); attr_set = true; }
    for (int kb = 0; kb < n; kb += 32) {
        const int bs = std::min(32, n - kb);
        const int m = ba->h_rmax[kb >> 5] - (kb + bs) + 2;
        const int ntile = (m + 31) / 32, total = m > 1 ? ntile * (ntile + 1) / 2 : 0;
        LAUNCH(ba, ba_wide_diag_kernel, 1, 32, 0, d.S, n, d.srow, d.soff, kb, ba->chol_invd.p, d.st, kb == 0 ? 1 : 0);
        LAUNCH(ba, ba_wide_panel_kernel, nblk(m, 128), 128, 0, d.S, d.rhs, n, d.srow, d.soff, kb, ba->chol_invd.p, d.st, ba->chol_rmax.p);
        LAUNCH(ba, ba_wide_update_kernel, nblk(total, WIDE_WARPS), WIDE_WARPS * 32, (size_t)WIDE_WARPS * 2 * 32 * 34 * 8, d.S, d.rhs, n, d.srow, d.soff, kb, d.st, ba->chol_rmax.p);
    }
    for (int kb = ((n - 1) / 32) * 32; kb >= 0; kb -= 32)
        LAUNCH(ba, ba_wide_backward_kernel, 1, 256, 0, d.S, d.rhs, n, d.srow, d.soff, kb, ba->chol_invd.p, d.st, ba->chol_rmax.p);
    return LVB_OK;
}

static int launch_reduced_solve(lvb_ba* ba) {
    BaDev& d = ba->dev;
    lvb_ctx* ctx = ba->ctx;
    if (ba->tree_levels > 0) {
        // multifrontal tree: leaves (all SMs) -> ... -> root, then the back-substitution root -> leaves; 2 (levels + 1) launches
        const Front* fr = ba->fronts.p;
        LAUNCH(ba, lm_control_pre_kernel, 1, 1, 0, d.st);
        const int n_fronts = ba->level_first[ba->tree_levels - 1] + ba->level_count[ba->tree_levels - 1];
        ba_front_init_kernel<<<dim3(16, n_fronts), 256, 0, ctx->stream>>>(fr, n_fronts, d.S, d.rhs, ba->front_pool.p, d.srow, d.soff, ba->band, d.st);
        ctx->launches++; mark(ba, "ba_front_init_kernel");
        for (int l = 0; l < ba->tree_levels; ++l)
            LAUNCH(ba, ba_front_factor_kernel, ba->level_count[l], CHOL_T, ba->tree_factor_smem, fr, ba->level_first[l], d.S, d.rhs, ba->front_pool.p, d.srow, d.soff, ba->band, ba->chol_invd.p, d.st);
        for (int l = ba->tree_levels - 1; l >= 0; --l)
            LAUNCH(ba, ba_front_backward_kernel, ba->level_count[l], CHOL_T, ba->tree_back_smem, fr, ba->level_first[l], d.S, d.rhs, ba->front_pool.p, d.srow, d.soff, ba->band, ba->chol_invd.p, d.st);
    } else if (ba->wide_solver) {
        LVB_TRY(launch_wide_solve(ba));
    } else
    LAUNCH(ba, ba_cholesky_kernel, 1, CHOL_T, ba->chol_smem, d.S, d.rhs, d.dimc, d.srow, d.soff, ba->chol_invd.p, d.st, 1, ba->chol_rmax.p, ba->chol_cmin.p);
    return LVB_OK;
}

static int launch_step(lvb_ba* ba) {
    BaDev& d = ba->dev;
    lvb_ctx* ctx = ba->ctx;
    LVB_TRY(launch_reduced_solve(ba));
    LAUNCH(ba, ba_update_kernel, nblk((size_t)d.n_poses + d.n_vec3 + d.n_rho, TPB), TPB, 0, d);
    const bool one_grid = merged_linearize(ba);
    const bool fork = !one_grid && use_side_branch(ba);
    if (one_grid) LAUNCH(ba, ba_linearize_all_kernel<1>, ba->ranges.b[6], TPB, std::max(ba->lin_smem, ba->imu_smem), d, ba->ranges);
    else {
    if (fork) { LVB_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream)); LVB_CUDA(cudaStreamWaitEvent(ctx->side, ctx->ev_fork, 0)); }
    LAUNCH(ba, ba_linearize_kernel<1>, ba->ranges.b[3], TPB, ba->lin_smem, d, ba->ranges);
    if (fork) {
        LAUNCH_ON(ba, ctx->side, ba_linearize_other_kernel<1>, ba->ranges.b[6] - ba->ranges.b[3], TPB, ba->imu_smem, d, ba->ranges);
        LVB_CUDA(cudaEventRecord(ctx->ev_join, ctx->side)); LVB_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    } else LAUNCH(ba, ba_linearize_other_kernel<1>, ba->ranges.b[6] - ba->ranges.b[3], TPB, ba->imu_smem, d, ba->ranges);
    }
    if (ctx->world > 1) LVB_TRY(comm_allreduce_sum_f64(ctx, &d.st->cand_cost_acc, 5));
    const bool wide = d.nS > ((size_t)1 << 20) || (size_t)d.n_poses * 7 + (size_t)d.n_vec3 * 3 + d.n_rho > ((size_t)1 << 17);
    LAUNCH(ba, ba_post_kernel, 1, wide ? 32 : 1024, 0, d, wide ? 1 : 0);
    if (wide) LAUNCH(ba, ba_post_wide_kernel, 4 * ba->ctx->sm_count, 256, 0, d);
    return check_launch("step");
}

static int launch_clear(lvb_ba* ba) {
    BaDev& d = ba->dev;
    const size_t nH = d.nS;
    LAUNCH(ba, ba_zero_kernel, std::min(1024, nblk(nH + d.dimc + 2 * (size_t)d.n_rho, 256)), 256, 0, d);
    return check_launch("clear");
}

static int upload_state(lvb_ba* ba, const lvb_solve_options* o, double radius_override) {
    lvb_solve_options opt;
    if (o) opt = *o; else lvb_default_options(&opt);
    if (radius_override > 0) opt.initial_trust_region_radius = radius_override;
    LmState h;
    lm_init(h, opt);
    // pageable source of a few hundred bytes: the call returns once the driver has staged it, no synchronisation needed before `h` dies
    LVB_CUDA(cudaMemcpyAsync(ba->st.p, &h, sizeof(h), cudaMemcpyHostToDevice, ba->ctx->stream));
    return LVB_OK;
}

static void apply_schur_mode(lvb_ba* ba, int mode) {
    const int m = (mode == 1 && ba->tc_ok) ? 1 : 0;
    ba->dev.tc_mode = m;
    if (ba->pass_graph && ba->graph_mode != m) drop_graph(ba);
    ba->graph_mode = m;
}

static int require_solvable(lvb_ba* ba) {
    if (!ba->finalized) { set_error("finalize first"); return LVB_ERR_STATE; }
    if (!ba->solvable) { set_error("camera system of dimension %d cannot be solved: %s", ba->dimc, ba->unsolvable_why); return LVB_ERR_UNSUPPORTED; }
    return check_imu_status(ba);
}

int lvb_ba_reduced_system(lvb_ba* ba, double radius, double* S, double* b, double* cost) {
    LVB_TRY(require_solvable(ba));
    LVB_CUDA(cudaSetDevice(ba->ctx->device)); lvb::g_alloc_stream = ba->ctx->stream;
    apply_schur_mode(ba, ba->schur_mode);
    LVB_TRY(upload_state(ba, nullptr, radius));
    LVB_TRY(launch_clear(ba));
    LVB_TRY(launch_linearize_and_reduce(ba, true));
    const int n = ba->dimc;
    if ((size_t)n > 8192) { set_error("lvb_ba_reduced_system: dimension %d is too large for a dense download", n); return LVB_ERR_UNSUPPORTED; }
    std::vector<double> hS(ba->nS);
    const size_t srow = (size_t)ba->srow, soff = (size_t)ba->soff; const int band = (ba->soff == 0) ? n : ba->band;
    auto at = [&](int i, int j) { return (i - j <= band) ? hS[(size_t)i * srow + j + soff] : 0.0; };   // i >= j
    LmState h;
    cudaStream_t s = ba->ctx->stream;
    LVB_CUDA(cudaMemcpyAsync(hS.data(), ba->dev.S, hS.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (b) LVB_CUDA(cudaMemcpyAsync(b, ba->dev.rhs, n * sizeof(double), cudaMemcpyDeviceToHost, s));
    LVB_CUDA(cudaMemcpyAsync(&h, ba->st.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    LVB_CUDA(cudaStreamSynchronize(s));
    // hand the system back in the caller-visible order (all poses, then all vec3 blocks)
    const std::vector<int>& cn = ba->canon;
    if (S) for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) S[(size_t)cn[i] * n + cn[j]] = (j <= i) ? at(i, j) : at(j, i);
    if (b) { std::vector<double> hb(b, b + n); for (int i = 0; i < n; ++i) b[cn[i]] = hb[i]; }
    if (cost) *cost = h.x_cost;
    return LVB_OK;
}

int lvb_ba_solve(lvb_ba* ba, const lvb_solve_options* options, lvb_solve_summary* summary) {
    LVB_TRY(require_solvable(ba));
    ba->host_fresh = false;
    LVB_CUDA(cudaSetDevice(ba->ctx->device)); lvb::g_alloc_stream = ba->ctx->stream;
    const auto t0 = std::chrono::steady_clock::now();
    static const bool prof_on = getenv("LVB_PROFILE") != nullptr;
    auto prof_t = t0;
#define PROF(name) do { if (prof_on) { const auto t_ = std::chrono::steady_clock::now(); fprintf(stderr, "[solve] %-28s %8.1f us\n", name, std::chrono::duration<double, std::micro>(t_ - prof_t).count()); prof_t = t_; } } while (0)
    lvb_solve_options opt;
    if (options) opt = *options; else lvb_default_options(&opt);
    apply_schur_mode(ba, options ? opt.schur_mode : ba->schur_mode);
    LVB_TRY(upload_state(ba, &opt, -1.0));
    PROF("state upload");
    cudaStream_t s = ba->ctx->stream;
    LmState h;
    memset(&h, 0, sizeof(h));
    mark(ba, "begin");
    LVB_TRY(launch_clear(ba));
    // The pass is a fixed sequence of launches whose kernels all read their control flags from the device state,
    // so it is captured once into a CUDA graph and replayed; the host looks at the state only every
    // `check_every` passes (kernels of a finished solve return immediately).
    const bool graph_ok = comm_graph_safe(ba->ctx, ba->nS + 3 * (size_t)ba->dimc + 16) && ba->ctx->use_graph && !g_timing;
    const int check_every = std::max(1, ba->ctx->check_every);
    const bool capped = opt.max_solver_time_in_seconds < 1e8;
    int pass = 0;
    while (pass <= opt.max_num_iterations) {
        int chunk = std::min(check_every, opt.max_num_iterations + 1 - pass);
        if (capped) {      // never overrun the wall-clock budget by more than about one pass (backend.cpp:208)
            // sharded problems: every pass contains collectives, so all ranks must launch the same number of passes -- the decision
            // is taken on the maximum elapsed time over the ranks (one small collective per look at the clock), never on a local clock
            double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            LVB_TRY(comm_max_seconds(ba->ctx, &el));
            if (pass > 0 && el >= opt.max_solver_time_in_seconds) break;
            chunk = pass == 0 ? 1 : std::max(1, std::min(chunk, (int)((opt.max_solver_time_in_seconds - el) / (el / pass))));
        }
        // instantiating a graph costs a few hundred microseconds: only worth it for a long solve or a reused problem
        // a borrowed graph only stays valid while this problem is the one the context's cached exec was last updated for
        if (ba->graph_borrowed && (ba->ctx->graph_owner != ba || ba->ctx->graph_cache != ba->pass_graph)) { ba->pass_graph = nullptr; ba->graph_borrowed = false; }
        // instantiating a graph costs a few hundred microseconds: worth it for a long solve or a reused problem; re-targeting the
        // context's cached exec to a fresh problem (cudaGraphExecUpdate) costs a few tens: worth it from a handful of iterations on
        const bool cache_ok = ba->ctx->use_graph_cache && opt.max_num_iterations >= 3 && ba->solves_done == 0;
        const bool use_graph = graph_ok && (ba->pass_graph || (pass >= 8 && opt.max_num_iterations - pass >= 16) || ba->solves_done >= 1 || cache_ok);
        if (use_graph && !ba->pass_graph) {
            cudaGraph_t g = nullptr;
            const long long before = ba->ctx->launches;
            LVB_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
            ba->capturing = true;
            int rc = launch_linearize_and_reduce(ba, false);
            if (rc == LVB_OK) rc = launch_step(ba);
            ba->capturing = false;
            cudaError_t ce = cudaStreamEndCapture(s, &g);
            if (rc != LVB_OK) { if (g) cudaGraphDestroy(g); return rc; }
            LVB_CUDA(ce);
            lvb_ctx* cx = ba->ctx;
            const bool own = ba->solves_done >= 1 || !cx->use_graph_cache;      // a reused problem keeps a graph of its own
            if (!own && cx->graph_cache) {
                cudaGraphExecUpdateResultInfo info;
                if (cudaGraphExecUpdate(cx->graph_cache, g, &info) == cudaSuccess) { ba->pass_graph = cx->graph_cache; ba->graph_borrowed = true; cx->graph_owner = ba; }
                else { cudaGetLastError(); cudaGraphExecDestroy(cx->graph_cache); cx->graph_cache = nullptr; cx->graph_owner = nullptr; }
            }
            if (!ba->pass_graph) {
                cudaGraphExec_t ex = nullptr;
                ce = cudaGraphInstantiate(&ex, g, 0);
                if (ce != cudaSuccess) { cudaGraphDestroy(g); LVB_CUDA(ce); }
                ba->pass_graph = ex; ba->graph_borrowed = !own;
                if (!own) { cx->graph_cache = ex; cx->graph_owner = ba; }
            }
            cudaGraphDestroy(g);
            ba->pass_launches = (int)(ba->ctx->launches - before);
            ba->ctx->launches = before;                     // capture is not execution
            PROF("capture + exec update");
        }
        for (int c = 0; c < chunk; ++c) {
            if (use_graph) { LVB_CUDA(cudaGraphLaunch(ba->pass_graph, s)); ba->ctx->launches += ba->pass_launches; }
            else { LVB_TRY(launch_linearize_and_reduce(ba, false)); LVB_TRY(launch_step(ba)); }
        }
        pass += chunk;
        LVB_CUDA(cudaMemcpyAsync(&h, ba->st.p, sizeof(h), cudaMemcpyDeviceToHost, s));
        LVB_CUDA(cudaStreamSynchronize(s));
        LVB_TRY(comm_check(ba->ctx));
        PROF("launch + wait");
        if (h.done) break;             // identical on every rank: the state is a function of bitwise-identical all-reduced sums
    }
#undef PROF
    ba->solves_done++;
    if (summary) {
        int nb = 0; for (int k = 0; k < 6; ++k) nb += ba->n[k];
        summary->initial_cost = h.initial_cost; summary->final_cost = h.x_cost;
        summary->num_iterations = h.iter; summary->num_successful_steps = h.num_successful;
        summary->termination_type = h.termination; summary->num_residual_blocks = nb; summary->num_residual_blocks_reduced = nb;
        summary->final_radius = h.radius;
        summary->total_time_in_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    }
    if (h.termination == 2) { set_error("LM failed: %d consecutive invalid steps", h.invalid); }
    return LVB_OK;
}

int lvb_ba_set_schur_mode(lvb_ba* ba, int mode) {
    if (mode != 0 && mode != 1) { set_error("schur_mode must be 0 (FP64) or 1 (tensor cores)"); return LVB_ERR_INVALID; }
    ba->schur_mode = mode;
    return LVB_OK;
}

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
    LVB_TRY(init_tables());
    lvb_ba ba;
    ba.ctx = ctx;
    cudaStream_t s = ctx->stream;
    ba.dimc = n; ba.band = band; ba.srow = band; ba.soff = band; ba.nS = (size_t)n * (band + 1);
    LVB_TRY(ba.arena.ensure(ba.nS + n));
    LVB_CUDA(cudaMemcpyAsync(ba.arena.p, S_band, ba.nS * sizeof(double), cudaMemcpyHostToDevice, s));
    LVB_CUDA(cudaMemcpyAsync(ba.arena.p + ba.nS, b, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, s));
    LVB_TRY(ba.chol_invd.ensure(n + 32));
    LVB_TRY(ba.st.ensure(1));
    lvb_solve_options opt; lvb_default_options(&opt);
    LmState h; lm_init(h, opt);
    const double one = 1.0; memcpy(&h.grad_max_bits, &one, sizeof(double));        // not converged: the pre-check lets the solve run
    LVB_CUDA(cudaMemcpyAsync(ba.st.p, &h, sizeof(h), cudaMemcpyHostToDevice, s));
    const int nstep = (n + 31) / 32;
    std::vector<int> rmax(nstep + 2, 0), cmin(nstep + 2, 0);
    int panel_rows = 2;
    for (int st = 0; st < nstep; ++st) {
        const int kb = st * 32, bs = std::min(32, n - kb);
        rmax[st] = std::min(n - 1, kb + band); cmin[st] = std::max(0, kb + bs - 1 - band);
        panel_rows = std::max(panel_rows, rmax[st] - (kb + bs) + 2);
    }
    LVB_TRY(ba.chol_rmax.upload(rmax.data(), rmax.size(), s)); LVB_TRY(ba.chol_cmin.upload(cmin.data(), cmin.size(), s));
    ba.chol_smem = (size_t)(CHOL_HDR + std::max(panel_rows + 2, 34) * 34) * 8;
    std::vector<Front> fr; size_t pool = 0; int rows = 0, mnb = 0, max_leaves = 1;
    while (max_leaves * 2 <= std::max(2, ctx->sm_count)) max_leaves *= 2;
    ba.tree_levels = 0;
    if (use_tree) {
        const int lv = build_front_tree(n, band, band - 31, max_leaves, fr, ba.level_first, ba.level_count, pool, rows, mnb);
        ba.tree_factor_smem = (size_t)(32 * 33 + 32 + 128 + (rows + 2) * 34) * 8; ba.tree_back_smem = (size_t)(((mnb + 1) & ~1) + (CHOL_T / 32) * 32) * 8;
        if (lv > 0 && ba.tree_factor_smem <= 227 * 1024 - 256) { ba.tree_levels = lv; LVB_TRY(ba.fronts.upload(fr.data(), fr.size(), s)); LVB_TRY(ba.front_pool.ensure(pool)); }
    }
    if (levels_out) *levels_out = ba.tree_levels;
    ba.wide_solver = ba.tree_levels == 0 && ba.chol_smem > 227 * 1024 - 256;      // ba_wide.cuh
    ba.h_rmax = rmax;
    BaDev& d = ba.dev;
    memset(&d, 0, sizeof(d));
    d.dimc = n; d.srow = ba.srow; d.soff = ba.soff; d.nS = ba.nS; d.S = ba.arena.p; d.rhs = ba.arena.p + ba.nS; d.st = ba.st.p;
    LVB_TRY(launch_reduced_solve(&ba));
    LVB_TRY(check_launch("band solve"));
    LVB_CUDA(cudaMemcpyAsync(x, d.rhs, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, s));
    LVB_CUDA(cudaMemcpyAsync(&h, ba.st.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    LVB_CUDA(cudaStreamSynchronize(s));
    if (h.solve_fail) { set_error("band solve: non-positive pivot"); return LVB_ERR_NUMERIC; }
    return LVB_OK;
}

// The three getters share one device round trip: the first call after a solve / parameter update brings all parameter blocks back
// (through the context's pinned staging area when it is free), the others copy from that snapshot.
static int fetch_params(lvb_ba* ba) {
    if (!ba->finalized) { set_error("finalize first"); return LVB_ERR_STATE; }
    if (ba->host_fresh) return LVB_OK;
    lvb_ctx* c = ba->ctx;
    LVB_CUDA(cudaSetDevice(c->device)); lvb::g_alloc_stream = c->stream;
    const size_t n0 = ba->h_poses.size(), n1 = ba->h_vec3.size(), n2 = ba->h_rho.size(), total = (n0 + n1 + n2) * sizeof(double);
    ba->r_params.resize(n0 + n1 + n2);
    const bool pinned = c->stage_h && c->stage_cap >= total && (!c->stage_busy || cudaEventQuery(c->stage_ev) == cudaSuccess);
    double* dst = pinned ? reinterpret_cast<double*>(c->stage_h) : ba->r_params.data();
    cudaStream_t s = c->stream;
    LVB_TRY(ba->poses.download(dst, n0, s)); LVB_TRY(ba->vec3.download(dst + n0, n1, s)); LVB_TRY(ba->rho.download(dst + n0 + n1, n2, s));
    LVB_CUDA(cudaStreamSynchronize(s));
    if (pinned) { memcpy(ba->r_params.data(), dst, total); c->stage_busy = false; }
    ba->host_fresh = true;
    return LVB_OK;
}
int lvb_ba_get_poses(lvb_ba* ba, double* out) {
    LVB_TRY(fetch_params(ba)); memcpy(out, ba->r_params.data(), ba->h_poses.size() * sizeof(double)); return LVB_OK;
}
int lvb_ba_get_vec3(lvb_ba* ba, double* out) {
    LVB_TRY(fetch_params(ba)); memcpy(out, ba->r_params.data() + ba->h_poses.size(), ba->h_vec3.size() * sizeof(double)); return LVB_OK;
}
int lvb_ba_get_inv_depths(lvb_ba* ba, double* out) {
    LVB_TRY(fetch_params(ba)); memcpy(out, ba->r_params.data() + ba->h_poses.size() + ba->h_vec3.size(), ba->h_rho.size() * sizeof(double)); return LVB_OK;
}

int lvb_ba_reprojection_errors(lvb_ba* ba, int n, const double* ob_pw, const int32_t* pose_idx, double* err) {
    if (!ba->finalized) { set_error("finalize first"); return LVB_ERR_STATE; }
    if (n <= 0) return LVB_OK;
    LVB_CUDA(cudaSetDevice(ba->ctx->device)); lvb::g_alloc_stream = ba->ctx->stream;
    const int np = (int)ba->h_poses.size() / 7;
    for (int i = 0; i < n; ++i) if (pose_idx[i] < 0 || pose_idx[i] >= np) { set_error("pose index out of range"); return LVB_ERR_INVALID; }
    DevBuf<double> d_in, d_err; DevBuf<int> d_idx;
    cudaStream_t s = ba->ctx->stream;
    LVB_TRY(d_in.upload(ob_pw, (size_t)5 * n, s)); LVB_TRY(d_idx.upload(pose_idx, n, s)); LVB_TRY(d_err.ensure(n));
    LAUNCH(ba, ba_reproj_error_kernel, nblk(n, 128), 128, 0, ba->dev, n, d_in.p, d_idx.p, d_err.p);
    LVB_TRY(check_launch("reproj"));
    LVB_TRY(d_err.download(err, n, s));
    LVB_CUDA(cudaStreamSynchronize(s));
    return LVB_OK;
}

}  // extern "C"
