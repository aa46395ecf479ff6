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
//   K6  reduced solve (ba_solve.cu) + ba_update + lm control   back-substitution, (+) update, LM decisions
#include <math.h>
#include <algorithm>
#include <chrono>
#include <map>
#include <string.h>
#include <cuda_bf16.h>
#include "ba_plan.h"
#include "lvb_internal.cuh"
#include "lvb_math.cuh"
#include "lvb_imu_warp.cuh"
#include "ba_solve.h"
#include "lvb_p2p.cuh"

using namespace lvb;

namespace {

enum { TPB = 128, IMU_STRIDE = 17 + 45 + 225 + 1, MAX_STAGE_POSES = 512, SYRK_ROWS = 64, SYRK_LD = 14 };

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
    int n_schur_warps;
    int tc_mode;                        // 1: Schur contraction on the tensor cores (wgmma, split bf16), FP64 rhs only here
    unsigned short* tc_u;               // packed U^T: [chunk of 16 landmarks][3 splits][128 x 16 bf16 K-major core-matrix tile]
    const int* tc_cdim;                 // camera offset -> compact pose dimension (0..127) or -1
    const int* tc_off;                  // compact pose dimension -> camera offset
    int tc_ndim;                        // 6 * free poses (<= 128)
    double *Hpp, *gc, *Hll, *gl, *tf_w;
    double *S, *rhs, *gcr, *diagH, *scal;      // inside the arena
    double *scale_c, *scale_l, *lam_c, *lam_l;
    LmState* st;
    unsigned int* cta_done;             // last-CTA-done counters: [0] ba_schur_kernel, [1] ba_linearize_all_kernel<1> (zero between launches)
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

// Last-CTA-done (as in lvb_p2p.cuh): every CTA of the grid arrives once, after its global writes; the CTA that arrives last sees
// all of them and resets the counter for the next launch.  True in every thread of that CTA.
__device__ __forceinline__ bool arrive_last(unsigned int* counter) {
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const int last = atomicAdd(counter, 1u) == gridDim.x - 1;
        if (last) { *counter = 0u; __threadfence(); }
        s_last = last;
    }
    __syncthreads();
    return s_last != 0;
}

// The LM state as a block-wide copy in shared memory: every field loaded at once from L2 (the accumulators were written with
// atomics), the decision then runs on shared memory instead of a chain of dependent L2 round trips, and the copy goes back whole.
// Only for a CTA that no other thread of the grid can race with (the last one to arrive).
static_assert(sizeof(LmState) % 8 == 0 && sizeof(LmState) / 8 <= TPB, "LmState is copied as 8-byte words, one per thread");
__device__ __forceinline__ void lm_state_load(LmState* s, const LmState* g) {
    if (threadIdx.x < sizeof(LmState) / 8) reinterpret_cast<unsigned long long*>(s)[threadIdx.x] = __ldcg(reinterpret_cast<const unsigned long long*>(g) + threadIdx.x);
    __syncthreads();
}
__device__ __forceinline__ void lm_state_store(LmState* g, const LmState* s) {
    __syncthreads();
    if (threadIdx.x < sizeof(LmState) / 8) reinterpret_cast<unsigned long long*>(g)[threadIdx.x] = reinterpret_cast<const unsigned long long*>(s)[threadIdx.x];
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

// An IMU factor is worked on by a thread group of NT threads: one warp (NT = 32) or one 128-thread CTA (window-sized problems).
template <int NT> __device__ __forceinline__ void group_sync() { if (NT == 32) __syncwarp(); else __syncthreads(); }

// Whitening by the square-root information U (upper triangular): s_r[16..30] = U r, s_Jw = U J (ambient, 15 x 32).
template <int NT>
__device__ __forceinline__ void imu_whiten(const double* U, const double* s_raw, double* s_Jw, double* s_r, bool with_jac) {
    const int t = NT == 32 ? threadIdx.x & 31 : threadIdx.x;
    if (t < 15) { double s = 0; for (int k = 0; k < 15; ++k) s += U[15 * t + k] * s_r[k]; s_r[16 + t] = s; }
    if (with_jac) for (int e = t; e < 480; e += NT) {
        const int i = e >> 5, j = e & 31;
        double s = 0; for (int k = i; k < 15; ++k) s += U[15 * i + k] * s_raw[32 * k + j];
        s_Jw[e] = s;
    }
    group_sync<NT>();
}

// The linearised IMU factor into the system, once the whitened residual and Jacobian are in s_r / s_Jw and every thread of the
// group has read the whitened residual: the tangent Jacobian Jt[15][30] scaled by the robust weight sr goes into s_raw (cols:
// pose_i 6 | v ba bg 9 | pose_j 6 | v ba bg 9), the residual is scaled likewise, s_gidx gets the 30 global camera-system indices
// (-1: constant block), then gc += Jt^T r and lower(Hpp) += Jt^T Jt.  In a CTA, warp 0 forms the tangent rows while warp 1
// builds the index table.
template <int NT>
__device__ __forceinline__ void imu_accumulate(const BaDev& d, const int* ix, int n, int f, const double* P, double sr, const double* s_Jw, double* s_raw, double* s_r, int* s_gidx) {
    const int t = NT == 32 ? threadIdx.x & 31 : threadIdx.x;
    if (t < 15) {
        const double* a = s_Jw + 32 * t;
        double* row = s_raw + 30 * t;
        double t6[6];
        ambient_row_to_tangent(P + 7 * ix[f], a, t6);
        for (int k = 0; k < 6; ++k) row[k] = t6[k] * sr;
        for (int k = 0; k < 9; ++k) row[6 + k] = a[7 + k] * sr;
        ambient_row_to_tangent(P + 7 * ix[4 * n + f], a + 16, t6);
        for (int k = 0; k < 6; ++k) row[15 + k] = t6[k] * sr;
        for (int k = 0; k < 9; ++k) row[21 + k] = a[23 + k] * sr;
        s_r[16 + t] *= sr;
    }
    const int l = NT == 32 ? t : t - 32;
    if (l >= 0 && l < 30) {
        int blk, loc;
        if (l < 6) { blk = 0; loc = l; } else if (l < 15) { blk = 1 + (l - 6) / 3; loc = (l - 6) % 3; }
        else if (l < 21) { blk = 4; loc = l - 15; } else { blk = 5 + (l - 21) / 3; loc = (l - 21) % 3; }
        const int id = ix[(size_t)blk * n + f];
        const int off = id < 0 ? -1 : ((blk == 0 || blk == 4) ? d.pose_off[id] : d.vec3_off[id]);
        s_gidx[l] = off < 0 ? -1 : off + loc;
    }
    group_sync<NT>();
    if (t < 30 && s_gidx[t] >= 0) {
        double g = 0; for (int i = 0; i < 15; ++i) g += s_raw[30 * i + t] * s_r[16 + i];
        atomicAdd(&d.gc[s_gidx[t]], g);
    }
    for (int e = t; e < 465; e += NT) {
        const int a = c_tri_a[e], b = c_tri_b[e];
        const int ga = s_gidx[a], gb = s_gidx[b];
        if (ga < 0 || gb < 0) continue;
        double h = 0; for (int i = 0; i < 15; ++i) h += s_raw[30 * i + a] * s_raw[30 * i + b];
        if (ga >= gb) atomicAdd(&d.Hpp[SIDX(d, ga, gb)], h); else atomicAdd(&d.Hpp[SIDX(d, gb, ga)], h);
    }
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
    imu_whiten<32>(c + 62, s_raw, s_Jw, s_r, with_jac);
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
__device__ __forceinline__ void syrk_flush(const BaDev& d, const double* A /*64 x SYRK_LD*/, int ncol, int off1, int off2) {
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
// The SYRK loop of one warp: while lanes with `take` remain, the first one's key (key1, key2) and camera offsets lead, the lanes
// holding that key write their two rows (rows(row0, row1), NCOL entries each), the others zeros, and the warp flushes A^T A.
// TWO_POSES: 13 columns [J_1 | J_2 | r], and key2 / off2 are exchanged too; one pose: 7 columns [J | r], key2 / off2 constants.
template <bool TWO_POSES, class Rows>
__device__ __forceinline__ void syrk_loop(const BaDev& d, double* A, bool take, int key1, int key2, int off1, int off2, Rows rows) {
    constexpr int NCOL = TWO_POSES ? 13 : 7;
    const int lane = threadIdx.x & 31;
    unsigned todo = __ballot_sync(0xffffffffu, take);
    while (todo) {
        const int leader = __ffs(todo) - 1;
        const int k1 = __shfl_sync(0xffffffffu, key1, leader), o1 = __shfl_sync(0xffffffffu, off1, leader);
        const int k2 = TWO_POSES ? __shfl_sync(0xffffffffu, key2, leader) : key2;
        const int o2 = TWO_POSES ? __shfl_sync(0xffffffffu, off2, leader) : off2;
        const bool mine = take && key1 == k1 && key2 == k2;
        double* row0 = A + (2 * lane) * SYRK_LD; double* row1 = row0 + SYRK_LD;
        if (mine) rows(row0, row1);
        else for (int k = 0; k < NCOL; ++k) { row0[k] = 0.0; row1[k] = 0.0; }
        __syncwarp();
        syrk_flush(d, A, NCOL, o1, o2);
        __syncwarp();
        todo &= ~__ballot_sync(0xffffffffu, mine);
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
    const int warp = threadIdx.x >> 5;
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
            syrk_loop<true>(d, A, valid && i1 != i2, i1, i2, off1, off2, [&](double* row0, double* row1) {
                for (int k = 0; k < 6; ++k) { row0[k] = o.J1[k]; row1[k] = o.J1[6 + k]; row0[6 + k] = o.J2[k]; row1[6 + k] = o.J2[6 + k]; }
                row0[12] = o.r[0]; row1[12] = o.r[1];
            });
            if (valid && i1 == i2) {
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
            syrk_loop<false>(d, A, valid, ip, 0, off, -1, [&](double* row0, double* row1) {
                for (int k = 0; k < 6; ++k) { row0[k] = o.J[k]; row1[k] = o.J[6 + k]; }
                row0[6] = o.r[0]; row1[6] = o.r[1];
            });
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
        imu_whiten<TPB>(s_c + 62, s_raw, s_Jw, s_r, MODE == 0);
        double s = 0.0;
        for (int i = 0; i < 15; ++i) s += s_r[16 + i] * s_r[16 + i];
        double rho_v, sr;
        huber(d.huber[3], s, &rho_v, &sr);
        if (tid == 0) cost = 0.5 * rho_v;
        if (MODE == 0) {
            __syncthreads();                                      // every thread has read the whitened residual
            imu_accumulate<TPB>(d, ix, n, f, Psrc, sr, s_Jw, s_raw, s_r, s_gidx);
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
            if (MODE == 0) imu_accumulate<32>(d, d.fi[3], n, f, Psrc, sr, Jw, raw, rr, gidx);     // each lane has read only its own residual entry
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

// The LM decision of a single-GPU window pass, in the last CTA of the cost kernel (the candidate cost is complete).  What the
// decision implies -- candidate -> x, clearing the accumulators -- is left to ba_post_wide_kernel over a whole grid: on the one CTA
// it took longer than the kernel it would save (window of 10 keyframes: 10 us in this CTA, 20 keyframes: 24 us).
__device__ __forceinline__ void decide_step_last_cta(const BaDev& d) {
    __shared__ LmState s;
    lm_state_load(&s, d.st);
    if (threadIdx.x == 0) { lm_control_post(s); if (s.accept) s.x_cost = s.cand_cost_acc; }
    lm_state_store(d.st, &s);
}

// Window-sized problems: ONE launch for all factor kinds.  The IMU blocks are a long single-warp dependency chain (~20 us) and the
// visual blocks a short wide one; in one grid -- IMU and priors first so they start at once -- they overlap instead of running
// back to back, and a launch is saved.  (At map scale the visual kernel's occupancy matters and the kernels stay separate.)
// decide (MODE 1, single GPU): the kernel also closes the pass.  Every CTA clears its share of S and rhs, which the next pass's
// ba_schur_kernel assembles into from zero whatever the decision; the last CTA to finish decides the step (decide_step_last_cta).
template <int MODE>
__global__ void __launch_bounds__(TPB) ba_linearize_all_kernel(BaDev d, BlockRanges R, int decide) {
    if (MODE == 1 && d.st->done) return;            // uniform: only the last CTA below writes `done`
    const int n_other = R.b[6] - R.b[3];
    if ((int)blockIdx.x < n_other) linearize_other_body<MODE>(d, R, (int)blockIdx.x + R.b[3]);
    else linearize_visual_body<MODE>(d, R, (int)blockIdx.x - n_other);
    if (MODE == 1 && decide) {
        const size_t n = d.nS + (size_t)d.dimc;     // S, then rhs: adjacent in the arena
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) d.S[i] = 0.0;
        if (arrive_last(d.cta_done + 1)) decide_step_last_cta(d);
    }
}

// ------------------------------------------------------------------ per-iteration system assembly
// zero_S: the pass assembles S and rhs from zero (ba_schur_kernel with `assemble`); later passes get them cleared by the cost kernel
__global__ void ba_zero_kernel(BaDev d, int zero_S) {
    const LmState* st = d.st;
    if (st->done || !st->need_linearize) return;
    const size_t nH = d.nS;
    const size_t total = nH + d.dimc + 2 * (size_t)d.n_rho, nA = zero_S ? nH + d.dimc : 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total + nA; i += (size_t)gridDim.x * blockDim.x) {
        if (i < nH) d.Hpp[i] = 0.0;
        else if (i < nH + d.dimc) d.gc[i - nH] = 0.0;
        else if (i < nH + d.dimc + d.n_rho) d.Hll[i - nH - d.dimc] = 0.0;
        else if (i < total) d.gl[i - nH - d.dimc - d.n_rho] = 0.0;
        else d.S[i - total] = 0.0;              // S, then rhs
    }
}

__device__ __forceinline__ void atomic_max_nonneg(unsigned long long* p, double v) {
    if (v == v) atomicMax(p, (unsigned long long)__double_as_longlong(fabs(v)));
    else atomicMax(p, 0x7ff0000000000000ull);   // NaN -> +inf so the tolerance test fails
}


// Four factors of a landmark's track at once, every load issued before the first use: factor id -> pose slots -> 96-byte coupling
// record is a chain of dependent round trips, and one factor at a time made the Schur kernel L2-latency bound (35 long-scoreboard
// stall cycles per issue at map scale).  f[u] = lm_fac[eb + u], -1 past e1; slots() issues the caller's index loads (unconditional,
// at max(f, 0): no branches between them); w[u] is factor f[u]'s record (factor 0's when f[u] < 0).
template <class Slots>
__device__ __forceinline__ void gather_couplings(const BaDev& d, int eb, int e1, int (&f)[4], double2 (&w)[4][6], Slots slots) {
#pragma unroll
    for (int u = 0; u < 4; ++u) f[u] = (eb + u < e1) ? d.lm_fac[eb + u] : -1;
    slots();
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const double2* src = reinterpret_cast<const double2*>(d.tf_w + (size_t)max(f[u], 0) * 12);
#pragma unroll
        for (int k = 0; k < 6; ++k) w[u][k] = src[k];
    }
}

// K5: eliminate the inverse depths.  One warp per 32 landmarks that share their set of pose offsets
// (finalize() groups and pads them).  Lane l writes u_l = sqrt(1/h_l) [w_l | g_l] (its couplings merged by
// pose slot) as a row of a shared-memory tile; the warp then forms the lower triangle of U^T U and subtracts
// it from S / adds the last column to rhs with one red.global per entry:  S -= sum_l w_l^T w_l / h_l.
__device__ __forceinline__ void schur_warp(const BaDev& d, int cols_max, int w) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
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
            const int e1 = d.lm_start[l + 1];
            for (int eb = d.lm_start[l]; eb < e1; eb += 4) {      // the landmark's coupling records, merged by pose slot
                int f[4], s0[4], s1[4];
                double2 w[4][6];
                gather_couplings(d, eb, e1, f, w, [&] {
#pragma unroll
                    for (int u = 0; u < 4; ++u) { const int fc = max(f[u], 0); s0[u] = d.tf_slot[fc]; s1[u] = d.tf_slot[(size_t)n + fc]; }
                });
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

__device__ __forceinline__ void warp_max_to_state(LmState* st, unsigned long long bits) {
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long v = __shfl_xor_sync(0xffffffffu, bits, o); bits = v > bits ? v : bits; }
    if ((threadIdx.x & 31) == 0 && bits) atomicMax(&st->grad_max_bits, bits);
}

// Row r of a camera block: its Hessian diagonal, gradient and (once valid) Jacobi scale; zeros and a scale of one when !in
__device__ __forceinline__ void camera_row_load(const BaDev& d, bool reduced, int r, bool in, int scale_valid, double& h, double& g, double& sc) {
    h = in ? (reduced ? d.diagH[r] : d.Hpp[SIDX(d, r, r)]) : 0.0;
    g = in ? (reduced ? d.gcr : d.gc)[r] : 0.0;
    sc = (in && scale_valid) ? d.scale_c[r] : 1.0;
}

// The LM step of camera block i (a pose, or a vec3 at i - n_poses), from the Hessian diagonal h_k and the gradient g_k of its rows r
// (Hpp's diagonal and gc, or with `reduced` the all-reduced diagH and gcr): the Jacobi scale (written on the first pass), the
// damping lambda_k = clamp(s^2 h_k, min_diag, max_diag) / (radius s^2), then damp(r, h_k, g_k, lambda_k) -- the caller's rows of
// the system.  Returns the gradient max-norm ||x - Plus(x, -g)||_inf as ordered bits (0: nothing to report); the caller reduces it
// over the warp and issues ONE atomicMax.
// LOAD_FIRST (the window pass, where this is on the critical path) issues every load -- the LM state's fields, the block's h, g,
// scale and x -- before the first use.  Otherwise each row is loaded as it is used, and the state's fields, x and g are read again
// where needed (the stores to scale_c / lam_c may alias the state): holding them would raise the wider kernels' register counts.
template <bool LOAD_FIRST, class Damp>
__device__ __forceinline__ unsigned long long camera_block_step(const BaDev& d, int i, bool reduced, Damp damp) {
    LmState held;
    if (LOAD_FIRST) {
        const LmState* src = d.st;
        held.scale_valid = src->scale_valid; held.jacobi = src->jacobi; held.need_linearize = src->need_linearize;
        held.min_diag = src->min_diag; held.max_diag = src->max_diag; held.radius = src->radius;
    }
    const LmState* st = LOAD_FIRST ? &held : d.st;
    const bool is_pose = i < d.n_poses;
    const int off = is_pose ? d.pose_off[i] : d.vec3_off[i - d.n_poses];
    if (off < 0) return 0ull;
    const int w = is_pose ? 6 : 3;
    const double* grad = reduced ? d.gcr : d.gc;
    double h[6], g[6], sc[6], x[7];
    if (LOAD_FIRST) {
#pragma unroll
        for (int k = 0; k < 6; ++k) camera_row_load(d, reduced, off + k, k < w, st->scale_valid, h[k], g[k], sc[k]);
#pragma unroll
        for (int k = 0; k < 7; ++k) x[k] = (is_pose && st->need_linearize) ? d.poses[7 * i + k] : 0.0;
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        if (k >= w) break;
        if (!LOAD_FIRST) camera_row_load(d, reduced, off + k, true, st->scale_valid, h[k], g[k], sc[k]);
        const int r = off + k;
        const double s = st->scale_valid ? sc[k] : (st->jacobi ? 1.0 / (1.0 + sqrt(h[k])) : 1.0), s2 = s * s;
        if (!st->scale_valid) d.scale_c[r] = s;
        const double lam = fmin(fmax(s2 * h[k], st->min_diag), st->max_diag) / (st->radius * s2);
        d.lam_c[r] = lam;
        damp(r, h[k], g[k], lam);
    }
    if (!st->need_linearize) return 0ull;
    const double* xp = LOAD_FIRST ? x : d.poses + 7 * i;
    const double* gp = LOAD_FIRST ? g : grad + off;
    double gm = 0.0;
    if (is_pose) {
        double ng[6], out[7];
        for (int k = 0; k < 6; ++k) ng[k] = -gp[k];
        pose_plus(xp, ng, out);
        for (int k = 0; k < 7; ++k) { const double df = fabs(xp[k] - out[k]); gm = (df == df) ? fmax(gm, df) : INFINITY; }
    } else for (int k = 0; k < 3; ++k) { const double df = fabs(gp[k]); gm = (df == df) ? fmax(gm, df) : INFINITY; }
    return (gm == gm) ? (unsigned long long)__double_as_longlong(fabs(gm)) : 0x7ff0000000000000ull;
}

// Single-GPU pass: S = lower(Hpp) + damping and rhs = -gc, added over the whole grid into the S / rhs the previous pass (or
// ba_zero_kernel) cleared.  The adds commute with the Schur warps' `S -= U^T U` and `rhs += sum u g` atomics: no ordering between
// the two and no grid barrier.  Dense storage (the only one on this path): one warp per row of the strict lower triangle.
__device__ __forceinline__ void assemble_system(const BaDev& d) {
    const int gid = blockIdx.x * blockDim.x + threadIdx.x, nthr = gridDim.x * blockDim.x, lane = threadIdx.x & 31;
    if (gid < 16) d.scal[gid] = 0.0;
    unsigned long long gbits = 0ull;
    for (int i = gid; i < d.n_poses + d.n_vec3; i += nthr)       // the block's rows: S[diag] += H_kk + lambda_k, rhs += -g_k
        gbits = max(gbits, camera_block_step<true>(d, i, false, [&](int r, double h, double g, double lam) {
            d.diagH[r] = h; d.gcr[r] = g;
            atomicAdd(&d.S[SIDX(d, r, r)], h + lam);
            atomicAdd(&d.rhs[r], -g);
        }));
    warp_max_to_state(d.st, gbits);
    for (int r = gid >> 5; r < d.dimc; r += nthr >> 5) {
        const double* src = d.Hpp + SIDX(d, r, 0);
        double* dst = d.S + SIDX(d, r, 0);
        for (int j0 = lane; j0 < r; j0 += 4 * 32) {
            double v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = (j0 + 32 * u < r) ? __ldg(src + j0 + 32 * u) : 0.0;
#pragma unroll
            for (int u = 0; u < 4; ++u) if (v[u] != 0.0) atomicAdd(dst + j0 + 32 * u, v[u]);
        }
    }
}

// assemble (single GPU): S and rhs arrive as zeros; the kernel adds the rest of the system (assemble_system) next to the
// elimination, and the last CTA to finish -- every gradient contribution and the cost are final then -- runs the LM pre-check
// (lm_control_pre), so the Cholesky that follows only reads `done`.
__global__ void __launch_bounds__(TPB) ba_schur_kernel(BaDev d, int cols_max, int assemble) {
    if (d.st->done) return;                         // uniform: only the last CTA below writes `done`
    if (assemble) assemble_system(d);
    const int w = blockIdx.x * (TPB / 32) + (threadIdx.x >> 5);
    if (w < d.n_schur_warps) schur_warp(d, cols_max, w);
    if (assemble && arrive_last(d.cta_done)) {
        __shared__ LmState s;
        lm_state_load(&s, d.st);
        if (threadIdx.x == 0) lm_control_pre(s);
        lm_state_store(d.st, &s);
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
// Cost and the max over the ranks of the gradient norm from the all-reduced scalars (read past L1: other CTAs or peers summed them)
__device__ __forceinline__ void unpack_scalars(const BaDev& d, LmState* st, int need_lin) {
    if (need_lin) st->cost_acc = __ldcg(d.scal);
    double m = 0.0;
    for (int r = 0; r < d.world; ++r) m = fmax(m, __ldcg(d.scal + 1 + r));
    st->grad_max_bits = (unsigned long long)__double_as_longlong(m);
}
__global__ void ba_unpack_scalars_kernel(BaDev d) {
    LmState* st = d.st;
    if (st->done) return;
    unpack_scalars(d, st, st->need_linearize);
}

// Sharded problems: the damping of camera block i once diagH and gcr hold the global sums, S[diag] += lambda_k
__device__ __forceinline__ unsigned long long damp_reduced_camera_block(const BaDev& d, int i) {
    return camera_block_step<false>(d, i, true, [&](int r, double, double, double lam) { d.S[SIDX(d, r, r)] += lam; });
}

// S <- lower(Hpp), rhs <- -gc, gcr <- gc, diagH <- diag(Hpp), scalars <- 0.
// Not launched for the single-GPU window, whose Schur kernel assembles S itself (assemble_system).
// FUSE_DAMP (single GPU): the camera blocks' Jacobi scale, LM damping and gradient max-norm (camera_block_step) ride along: the
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
        for (size_t i = gid; i < (size_t)(d.n_poses + d.n_vec3); i += stride)
            gbits = max(gbits, camera_block_step<false>(d, (int)i, false, [&](int r, double h, double g, double lam) {
                d.diagH[r] = h; d.rhs[r] = -g; d.gcr[r] = g; d.S[SIDX(d, r, r)] = h + lam;
            }));
        warp_max_to_state(d.st, gbits);
    }
}

__global__ void ba_prepare_camera_kernel(BaDev d) {
    if (d.st->done) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    warp_max_to_state(d.st, (i < d.n_poses + d.n_vec3) ? damp_reduced_camera_block(d, i) : 0ull);
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
        if (threadIdx.x == 0) unpack_scalars(d, st, need_lin);
        __syncthreads();
        unsigned long long gbits = 0ull;
        for (int i = threadIdx.x; i < d.n_poses + d.n_vec3; i += blockDim.x) gbits = max(gbits, damp_reduced_camera_block(d, i));
        warp_max_to_state(st, gbits);
        __syncthreads();
    }
    p2p_finish_epoch(a, epoch);
}

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
            for (int eb = e0; eb < e1; eb += 4) {
                int f[4], o0[4], o1[4];
                double2 w[4][6];
                gather_couplings(d, eb, e1, f, w, [&] {
#pragma unroll
                    for (int u = 0; u < 4; ++u) { const int fc = max(f[u], 0); o0[u] = ix[(size_t)n + fc]; o1[u] = ix[(size_t)2 * n + fc]; }
#pragma unroll
                    for (int u = 0; u < 4; ++u) { o0[u] = d.pose_off[o0[u]]; o1[u] = d.pose_off[o1[u]]; }
                });
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

// What an LM decision implies: candidate -> x when `accept`, the accumulators of the next linearisation cleared when `clear`.
// The calling threads take elements first, first + stride, ...
__device__ __forceinline__ void accept_and_clear(const BaDev& d, bool accept, bool clear, size_t first, size_t stride) {
    if (accept) {
        const size_t np = (size_t)d.n_poses * 7, nv = (size_t)d.n_vec3 * 3, nr = d.n_rho;
        for (size_t i = first; i < np + nv + nr; i += stride) {
            if (i < np) d.poses[i] = d.c_poses[i];
            else if (i < np + nv) d.vec3[i - np] = d.c_vec3[i - np];
            else d.rho[i - np - nv] = d.c_rho[i - np - nv];
        }
    }
    if (clear) {
        const size_t nH = d.nS;
        double2* H2 = reinterpret_cast<double2*>(d.Hpp);
        for (size_t i = first; i < nH / 2; i += stride) H2[i] = make_double2(0.0, 0.0);
        if ((nH & 1) && first == 0) d.Hpp[nH - 1] = 0.0;
        for (size_t i = first; i < (size_t)d.dimc; i += stride) d.gc[i] = 0.0;
        for (size_t i = first; i < (size_t)d.n_rho; i += stride) { d.Hll[i] = 0.0; d.gl[i] = 0.0; }
    }
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
    accept_and_clear(d, s_accept, s_zero, threadIdx.x, blockDim.x);
}

// Large problems (banded storage) and the single-GPU window pass: the same accept + clear spread over the whole grid.  `accept` may
// be stale when the solve finished in an earlier pass; the copy is idempotent then (the candidate has not been rewritten).
__global__ void ba_post_wide_kernel(BaDev d) {
    const LmState* st = d.st;
    accept_and_clear(d, st->accept, !st->done && st->need_linearize, (size_t)blockIdx.x * blockDim.x + threadIdx.x, (size_t)gridDim.x * blockDim.x);
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
    bool finalized = false;
    double cam[22];
    bool have_cam = false;
    std::vector<double> h_poses, h_vec3, h_rho;
    std::vector<double> r_params; bool host_fresh = false;      // parameter blocks as last read back (one round trip serves the three getters)
    std::vector<uint8_t> h_pose_const, h_vec3_const, h_rho_const;
    std::vector<double> h_fc[6];
    std::vector<int32_t> h_fi[6];
    int n[6] = {0, 0, 0, 0, 0, 0};      // blocks as added by the caller
    double huber[6] = {0, 0, 0, 0, 0, 0};
    BaPlan plan;                        // structure, device order, storage and solver of the last finalize (ba_plan.h)
    ReducedSolver solver;               // the reduced camera system's solver for plan.solver (ba_solve.h)
    // device
    DevBuf<unsigned char> upload_arena;      // one allocation for everything finalize uploads (the buffers below are views into it)
    DevBuf<double> poses, vec3, rho, c_poses, c_vec3, c_rho;
    DevBuf<int> pose_off, vec3_off, rho_slot, lm_start, lm_fac;
    DevBuf<int> tf_slot, sw_group, sw_lm, grp_ns, grp_off;
    size_t schur_smem = 0, lin_smem = 0;
    cudaGraphExec_t pass_graph = nullptr;
    bool graph_borrowed = false;        // pass_graph is the context's cached exec (never destroyed from here)
    int pass_launches = 0;
    bool capturing = false;
    bool imu_checked = true;
    // tensor-core Schur (schur_mode 1)
    int schur_mode = 0, graph_mode = -1, n_tc_chunks = 0;
    DevBuf<unsigned short> tc_u; DevBuf<int> tc_cdim, tc_off;
    int solves_done = 0;
    DevBuf<double> fc[6];
    DevBuf<int> fi[6];
    DevBuf<double> imu_raw;
    DevBuf<int> imu_status;
    DevBuf<double> Hpp, gc, Hll, gl, tf_w, arena, scale_c, scale_l, lam_c, lam_l;
    DevBuf<double> eval_r, eval_J;
    DevBuf<LmState> st;
    DevBuf<unsigned int> cta_done;
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

static const int kResDim[6] = {2, 2, 2, 15, 6, 6};
static const int kJacCols[6] = {15, 7, 1, 32, 14, 7};

static bool g_tables_ready = false;
static int init_tables() {
    if (g_tables_ready) return LVB_OK;
    unsigned char a[465], b[465]; int e = 0;
    for (int i = 0; i < 30; ++i) for (int j = 0; j <= i; ++j) { a[e] = (unsigned char)i; b[e] = (unsigned char)j; ++e; }
    LVB_CUDA(cudaMemcpyToSymbol(c_tri_a, a, sizeof(a)));
    LVB_CUDA(cudaMemcpyToSymbol(c_tri_b, b, sizeof(b)));
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
#define g_timing lvb::g_timing

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
    int begin() { return staged ? lvb::stage_wait(ctx) : LVB_OK; }      // the previous problem's copy has read it
    int grow(size_t need) { return lvb::stage_grow(ctx, need, used); }
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
        LVB_TRY(lvb::stage_mark_busy(ctx, s));
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

// element-wise collective over a host array of a sharded problem: through the device, like every all-reduce
static int allreduce_host_i32(lvb_ctx* ctx, std::vector<int>& v, int (*op)(lvb_ctx*, int*, size_t)) {
    cudaStream_t s = ctx->stream;
    DevBuf<int> tmp;
    LVB_TRY(tmp.upload(v.data(), v.size(), s));
    LVB_TRY(op(ctx, tmp.p, v.size()));
    LVB_CUDA(cudaMemcpyAsync(v.data(), tmp.p, v.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    LVB_TRY(lvb::host_sync(ctx, s));
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
    if (!ba->have_cam) { set_error("cameras not set"); return LVB_ERR_STATE; }
    const int np = (int)ba->h_poses.size() / 7, nv = (int)ba->h_vec3.size() / 3, nr = (int)ba->h_rho.size();
    // ---- plan (ba_plan.h): host arithmetic on the index arrays
    BaProblemView in;
    in.np = np; in.nv = nv; in.nr = nr;
    in.pose_const = ba->h_pose_const.data(); in.vec3_const = ba->h_vec3_const.data(); in.rho_const = ba->h_rho_const.data();
    for (int k = 0; k < 6; ++k) { in.n[k] = ba->n[k]; in.fc[k] = ba->h_fc[k].data(); in.fi[k] = ba->h_fi[k].data(); }
    PlanHooks hooks;
    hooks.max_reduce = [ctx](std::vector<int>& v) { return allreduce_host_i32(ctx, v, comm_allreduce_max_i32); };
    hooks.min_reduce = [ctx](std::vector<int>& v) { return allreduce_host_i32(ctx, v, comm_allreduce_min_i32); };
    hooks.phase_done = [&](const char* name) { PROF(name); };
    BaPlan& P = ba->plan;
    std::string err;
    if (int rc = plan_ba(in, ctx->sm_count, ctx->world, no_tree_switch(), tree_sep_band_switch(), hooks, P, err)) {
        if (!err.empty()) set_error("%s", err.c_str());
        return rc;
    }
    const int npf = P.n_pose_free;

    // ---- upload
    size_t stage_estimate = (ba->h_poses.size() + ba->h_vec3.size() + ba->h_rho.size()) * 24;
    for (int k = 0; k < 6; ++k) stage_estimate += ba->h_fc[k].size() * 8 + ba->h_fi[k].size() * 12;
    Stager stg(ctx, stage_estimate);
    LVB_TRY(stg.begin());
    LVB_TRY(stg.put(ba->poses, ba->h_poses.data(), ba->h_poses.size()));
    LVB_TRY(stg.put(ba->vec3, ba->h_vec3.data(), ba->h_vec3.size()));
    LVB_TRY(stg.put(ba->rho, ba->h_rho.data(), ba->h_rho.size()));
    LVB_TRY(stg.put(ba->c_poses, ba->h_poses.data(), ba->h_poses.size()));
    LVB_TRY(stg.put(ba->c_vec3, ba->h_vec3.data(), ba->h_vec3.size()));
    LVB_TRY(stg.put(ba->c_rho, ba->h_rho.data(), ba->h_rho.size()));
    LVB_TRY(stg.put(ba->pose_off, P.pose_off.data(), np));
    LVB_TRY(stg.put(ba->vec3_off, P.vec3_off.data(), nv));
    LVB_TRY(stg.put(ba->rho_slot, P.rho_slot.data(), nr));
    LVB_TRY(stg.put(ba->lm_start, P.lm_start.data(), nr + 1));
    LVB_TRY(stg.put(ba->lm_fac, P.lm_fac.data(), P.lm_fac.size()));
    LVB_TRY(stg.put(ba->tf_slot, P.tf_slot.data(), P.tf_slot.size()));
    LVB_TRY(stg.put(ba->sw_group, P.sw_group.data(), P.sw_group.size()));
    LVB_TRY(stg.put(ba->sw_lm, P.sw_lm.data(), P.sw_lm.size()));
    LVB_TRY(stg.put(ba->grp_ns, P.grp_ns.data(), P.grp_ns.size()));
    LVB_TRY(stg.put(ba->grp_off, P.grp_off.data(), P.grp_off.size()));
    // tensor-core Schur operands: the compaction maps and the zero-initialised split-bf16 U^T tiles
    LVB_TRY(stg.put(ba->tc_cdim, P.tc_cdim.data(), P.tc_cdim.size()));
    LVB_TRY(stg.put(ba->tc_off, P.tc_off.data(), P.tc_off.size()));
    ba->n_tc_chunks = P.tc_ok ? ((2 * P.n_schur_warps + TC_CHUNKS - 1) / TC_CHUNKS) * TC_CHUNKS : 0;
    LVB_TRY(ba->tc_u.ensure((size_t)std::max(1, ba->n_tc_chunks) * 3 * 2048));
    LVB_CUDA(cudaMemsetAsync(ba->tc_u.p, 0, (size_t)std::max(1, ba->n_tc_chunks) * 3 * 2048 * sizeof(unsigned short), s));

    PROF("uploads (params, structure)");
    // factor planes in device order (AoS -> SoA transpose on the host, written straight into the staging area; IMU stays AoS and
    // is packed on the device).  The one copy to the device is issued when the last array is in place; the IMU kernel follows it.
    {
        for (int k = 0; k < 6; ++k) {
            const int n = P.nd[k];
            const std::vector<int>& ord = P.order[k];
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
        const int n = P.nd[3];
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

    const size_t nH = P.nS;
    LVB_TRY(ba->solver.upload(ctx, P.solver, P.chol_rmax, P.dimc));
    LVB_TRY(ba->Hpp.ensure(nH)); LVB_TRY(ba->gc.ensure(P.dimc));
    LVB_TRY(ba->Hll.ensure(std::max(1, nr))); LVB_TRY(ba->gl.ensure(std::max(1, nr)));
    LVB_TRY(ba->tf_w.ensure((size_t)std::max(1, P.nd[0]) * 12));
    LVB_TRY(ba->arena.ensure(nH + 3 * (size_t)P.dimc + 16));
    LVB_TRY(ba->scale_c.ensure(P.dimc)); LVB_TRY(ba->lam_c.ensure(P.dimc));
    LVB_TRY(ba->scale_l.ensure(std::max(1, nr))); LVB_TRY(ba->lam_l.ensure(std::max(1, nr)));
    LVB_TRY(ba->st.ensure(1));
    if (!ba->cta_done.p) { LVB_TRY(ba->cta_done.ensure(2)); LVB_TRY(ba->cta_done.zero(s)); }     // each kernel leaves its counter at zero

    PROF("sync + alloc");
    BaDev& d = ba->dev;
    d.n_poses = np; d.n_vec3 = nv; d.n_rho = nr; d.dimc = P.dimc; d.n_pose_free = npf;
    d.srow = P.srow; d.soff = P.soff; d.nS = P.nS;
    d.poses = ba->poses.p; d.vec3 = ba->vec3.p; d.rho = ba->rho.p; d.c_poses = ba->c_poses.p; d.c_vec3 = ba->c_vec3.p; d.c_rho = ba->c_rho.p;
    d.pose_off = ba->pose_off.p; d.vec3_off = ba->vec3_off.p; d.rho_slot = ba->rho_slot.p;
    for (int k = 0; k < 6; ++k) { d.n[k] = P.nd[k]; d.fc[k] = ba->fc[k].p; d.fi[k] = ba->fi[k].p; d.huber[k] = ba->huber[k]; }
    d.lm_start = ba->lm_start.p; d.lm_fac = ba->lm_fac.p;
    d.tf_slot = ba->tf_slot.p; d.sw_group = ba->sw_group.p; d.sw_lm = ba->sw_lm.p; d.grp_ns = ba->grp_ns.p; d.grp_off = ba->grp_off.p;
    d.n_schur_warps = P.n_schur_warps;
    d.tc_mode = 0; d.tc_u = ba->tc_u.p; d.tc_cdim = ba->tc_cdim.p; d.tc_off = ba->tc_off.p; d.tc_ndim = 6 * npf;
    d.Hpp = ba->Hpp.p; d.gc = ba->gc.p; d.Hll = ba->Hll.p; d.gl = ba->gl.p; d.tf_w = ba->tf_w.p;
    d.S = ba->arena.p; d.rhs = d.S + nH; d.gcr = d.rhs + P.dimc; d.diagH = d.gcr + P.dimc; d.scal = d.diagH + P.dimc;
    d.scale_c = ba->scale_c.p; d.scale_l = ba->scale_l.p; d.lam_c = ba->lam_c.p; d.lam_l = ba->lam_l.p;
    d.st = ba->st.p; d.cta_done = ba->cta_done.p;
    d.rank = ctx->rank; d.world = ctx->world; d.rank0 = (ctx->rank == 0) ? 1 : 0;
    d.stage_poses = (np <= MAX_STAGE_POSES) ? (ctx->use_tma ? 2 : 1) : 0;
    d.cams.c0 = make_cam(ba->cam); d.cams.c1 = make_cam(ba->cam + 11);

    BlockRanges& R = ba->ranges;
    R.b[0] = 0;
    R.b[1] = R.b[0] + nblk(P.nd[0], TPB);
    R.b[2] = R.b[1] + nblk(P.nd[1], TPB);
    R.b[3] = R.b[2] + nblk(P.nd[2], TPB);
    d.imu_cta = P.dense ? 1 : 0;
    R.b[4] = R.b[3] + (d.imu_cta ? P.nd[3] : nblk(P.nd[3], 4));
    R.b[5] = R.b[4] + nblk(P.nd[4], TPB);
    R.b[6] = R.b[5] + nblk(P.nd[5], TPB);
    const size_t smem_imu = d.imu_cta ? (size_t)(480 * 2 + 32 + IMU_STRIDE) * 8 + 32 * 4 : (size_t)(4 * 480 * 2 + 4 * 32) * 8 + 4 * 32 * 4;
    const size_t smem_pose = d.stage_poses ? ((size_t)np * 56 + 16) : 0;
    drop_graph(ba);
    ba->pose_smem = smem_pose; ba->imu_smem = smem_imu;
    ba->lin_smem = ((smem_pose + 15) & ~(size_t)15) + (size_t)(TPB / 32) * SYRK_ROWS * SYRK_LD * 8;
    ba->schur_smem = (size_t)(TPB / 32) * 32 * (size_t)std::max(1, P.schur_cols_max) * 8;
    PROF("tail");
#undef PROF
    ba->finalized = true;
    return LVB_OK;
}

int lvb_ba_dims(lvb_ba* ba, int* dimc, int* nrf, int* rows) {
    if (!ba->finalized) { set_error("finalize first"); return LVB_ERR_STATE; }
    if (dimc) *dimc = ba->plan.dimc;
    if (nrf) *nrf = ba->plan.n_rho_free;
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
    LVB_TRY(lvb::host_sync(ba->ctx, s));
    return LVB_OK;
}

static int check_imu_status(lvb_ba* ba) {
    if (ba->imu_checked || ba->plan.nd[3] == 0) { ba->imu_checked = true; return LVB_OK; }
    std::vector<int> status(ba->plan.nd[3]);
    LVB_TRY(ba->imu_status.download(status.data(), status.size(), ba->ctx->stream));
    LVB_TRY(lvb::host_sync(ba->ctx, ba->ctx->stream));
    for (size_t f = 0; f < status.size(); ++f) if (status[f]) { set_error("ImuError %d: covariance is singular or not finite (code %d)", (int)f, status[f]); return LVB_ERR_NUMERIC; }
    ba->imu_checked = true;
    return LVB_OK;
}

static int launch_eval(lvb_ba* ba, int kind, double* r_dev, double* J_dev) {
    const int n = ba->plan.nd[kind];
    if (n == 0) return LVB_OK;
    BaDev& d = ba->dev;
    switch (kind) {
    case 0: {
        const size_t pose_b = d.stage_poses ? (size_t)d.n_poses * 56 + 16 : 0;
        const int v = ba->ctx->eval_variant;       // LVB_EVAL_VARIANT: 0 staged/5 CTAs, 1 staged/6, 2 direct/5, 3 direct/6
        if (v == 1) LAUNCH(ba->ctx, (ba_eval_two_frame_kernel<1, 6>), nblk(n, TPB), TPB, (size_t)(TPB * 31) * 8 + pose_b, d, r_dev, J_dev);
        else if (v == 2) LAUNCH(ba->ctx, (ba_eval_two_frame_kernel<0, 5>), nblk(n, TPB), TPB, pose_b, d, r_dev, J_dev);
        else if (v == 3) LAUNCH(ba->ctx, (ba_eval_two_frame_kernel<0, 6>), nblk(n, TPB), TPB, pose_b, d, r_dev, J_dev);
        else LAUNCH(ba->ctx, (ba_eval_two_frame_kernel<1, 5>), nblk(n, TPB), TPB, (size_t)(TPB * 31) * 8 + pose_b, d, r_dev, J_dev);
        break; }
    case 1: LAUNCH(ba->ctx, ba_eval_pose_only_kernel, nblk(n, TPB), TPB, 0, d, r_dev, J_dev); break;
    case 2: LAUNCH(ba->ctx, ba_eval_two_camera_kernel, nblk(n, TPB), TPB, 0, d, r_dev, J_dev); break;
    case 3: LAUNCH(ba->ctx, ba_eval_imu_kernel, nblk(n, 4), TPB, 0, d, r_dev, J_dev); break;
    default: LAUNCH(ba->ctx, ba_eval_prior_kernel, nblk(n, 64), 64, 0, d, kind, r_dev, J_dev); break;
    }
    return check_launch("ba_eval");
}

static int ensure_eval_buffers(lvb_ba* ba, int kind) {
    const size_t n = ba->plan.nd[kind];
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
    const size_t nd = ba->plan.nd[kind], rd = kResDim[kind], jd = (size_t)kResDim[kind] * kJacCols[kind];
    const std::vector<int>& ord = ba->plan.order[kind];
    bool identity = (nd == (size_t)ba->n[kind]);
    for (size_t i = 0; identity && i < nd; ++i) identity = (ord[i] == (int)i);
    cudaStream_t s = ba->ctx->stream;
    if (identity) {
        if (r) LVB_TRY(ba->eval_r.download(r, nd * rd, s));
        if (J) LVB_TRY(ba->eval_J.download(J, nd * jd, s));
        LVB_TRY(lvb::host_sync(ba->ctx, s));
        return LVB_OK;
    }
    // the device layout is sorted / padded: hand the rows back in the caller's block order
    std::vector<double> hr(r ? nd * rd : 0), hJ(J ? nd * jd : 0);
    if (r) LVB_TRY(ba->eval_r.download(hr.data(), nd * rd, s));
    if (J) LVB_TRY(ba->eval_J.download(hJ.data(), nd * jd, s));
    LVB_TRY(lvb::host_sync(ba->ctx, s));
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
    return !off && ba->plan.srow == ba->plan.dimc && ba->plan.soff == 0 && ba->ranges.b[3] > 0 && ba->ranges.b[6] > ba->ranges.b[3];      // dense layout = window-sized
}

// accept + clear spread over a whole grid (ba_post_wide_kernel): the arrays are too large for one CTA
static bool wide_post(const lvb_ba* ba) {
    const BaDev& d = ba->dev;
    return d.nS > ((size_t)1 << 20) || (size_t)d.n_poses * 7 + (size_t)d.n_vec3 * 3 + d.n_rho > ((size_t)1 << 17);
}

// The single-GPU window pass (six kernels): S is assembled inside the Schur kernel, whose last CTA runs the LM pre-check, and the
// step is decided in the last CTA of the cost kernel.  Sharded problems need the all-reduce between those stages, and map-scale
// ones keep their own kernels (zeroing a banded S each pass would cost more than the copy it replaces).
static bool fused_pass(lvb_ba* ba) { return ba->ctx->world == 1 && merged_linearize(ba) && !wide_post(ba); }

static bool use_side_branch(lvb_ba* ba) {
    // not inside a captured graph: replaying a graph with parallel branches was measured to be erratic (0.19 - 0.9 ms per
    // pass on the same build), a linear graph is stable
    return ba->ctx->use_side && ba->ctx->side && !g_timing && !ba->capturing && ba->ranges.b[3] > 0 && ba->ranges.b[6] > ba->ranges.b[3];
}

// The visual and the IMU / prior linearisations, MODE 0 at the current parameters (start of a pass), MODE 1 at the candidate (after
// the update).  They are independent (both only add into the accumulators): one grid for both at window size, two kernels (parallel
// branches when launched directly) at map scale.  The timing marks keep the names of the instantiations.
extern "C++" {
template <int MODE> static int launch_linearize(lvb_ba* ba) {
    static const char* const kName[2][3] = {{"ba_linearize_all_kernel<0>", "ba_linearize_kernel<0>", "ba_linearize_other_kernel<0>"},
                                            {"ba_linearize_all_kernel<1>", "ba_linearize_kernel<1>", "ba_linearize_other_kernel<1>"}};
    BaDev& d = ba->dev;
    lvb_ctx* ctx = ba->ctx;
    const bool one_grid = merged_linearize(ba);
    const bool fork = !one_grid && use_side_branch(ba);
    const int decide = (MODE == 1 && fused_pass(ba)) ? 1 : 0;
    if (one_grid) LAUNCH_AS(ba->ctx, kName[MODE][0], ba_linearize_all_kernel<MODE>, ba->ranges.b[6], TPB, std::max(ba->lin_smem, ba->imu_smem), d, ba->ranges, decide);
    else {
    if (fork) { LVB_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream)); LVB_CUDA(cudaStreamWaitEvent(ctx->side, ctx->ev_fork, 0)); }
    LAUNCH_AS(ba->ctx, kName[MODE][1], ba_linearize_kernel<MODE>, ba->ranges.b[3], TPB, ba->lin_smem, d, ba->ranges);
    if (fork) {
        LAUNCH_ON(ba->ctx, ctx->side, ba_linearize_other_kernel<MODE>, ba->ranges.b[6] - ba->ranges.b[3], TPB, ba->imu_smem, d, ba->ranges);
        LVB_CUDA(cudaEventRecord(ctx->ev_join, ctx->side)); LVB_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    } else LAUNCH_AS(ba->ctx, kName[MODE][2], ba_linearize_other_kernel<MODE>, ba->ranges.b[6] - ba->ranges.b[3], TPB, ba->imu_smem, d, ba->ranges);
    }
    return LVB_OK;
}
}  // extern "C++"

// one pass = one LM iteration attempt (all decisions on the device).  The single-GPU window (fused_pass) is six launches:
//   linearize (all factor kinds) | Schur (+ S = lower(Hpp) + damping, rhs, LM pre-check in the last CTA) | Cholesky
//   | back-substitution + candidate | cost (+ clear S / rhs, LM decision in the last CTA) | accept + clear (whole grid)
// Every other problem keeps up to 10 (the two linearise kernels and the two cost kernels run as parallel branches on a second
// stream at map scale):
//   linearize (visual) | linearize (IMU + priors) | build S | Schur | [all-reduce] | camera damping | Cholesky (+ LM pre-check)
//   | back-substitution + candidate | cost (visual) | cost (IMU + priors) | [all-reduce] | LM decision + accept + clear
static int launch_linearize_and_reduce(lvb_ba* ba, bool standalone) {
    BaDev& d = ba->dev;
    lvb_ctx* ctx = ba->ctx;
    const size_t nH = d.nS;
    const bool fused = fused_pass(ba);
    LVB_TRY(launch_linearize<0>(ba));
    const bool fuse_damp = ctx->world == 1;
    if (!fused) {
        if (fuse_damp) LAUNCH(ba->ctx, ba_build_S_kernel<1>, std::min(1024, nblk(nH, 256)), 256, 0, d);
        else LAUNCH(ba->ctx, ba_build_S_kernel<0>, std::min(1024, nblk(nH, 256)), 256, 0, d);
    }
    // the fused pass launches the Schur kernel even without landmarks: it assembles S
    LAUNCH(ba->ctx, ba_schur_kernel, std::max(fused ? 1 : 0, nblk(d.n_schur_warps, TPB / 32)), TPB, ba->schur_smem, d, std::max(1, ba->plan.schur_cols_max), fused ? 1 : 0);
    if (d.tc_mode) LAUNCH(ba->ctx, ba_schur_tc_kernel, ba->n_tc_chunks / TC_CHUNKS, 128, (size_t)TC_CHUNKS * TC_CHUNK_BYTES, d, ba->n_tc_chunks);
    const size_t n_arena = nH + 3 * (size_t)d.dimc + 16;
    P2PArgs pa;
    const bool fused_comm = ctx->world > 1 && comm_p2p_args(ctx, n_arena, &pa) && (size_t)(d.n_poses + d.n_vec3) <= 4096;
    if (fused_comm) {
        LAUNCH(ba->ctx, ba_allreduce_fused_kernel, (int)std::max<size_t>(1, std::min<size_t>(XB_BLOCKS, (n_arena + 255) / 256)), 256, 0, pa, d, (int)n_arena);
    } else if (ctx->world > 1) {
        LAUNCH(ba->ctx, ba_pack_scalars_kernel, 1, 1, 0, d);
        LVB_TRY(comm_allreduce_sum_f64(ctx, d.S, n_arena));
        LAUNCH(ba->ctx, ba_unpack_scalars_kernel, 1, 1, 0, d);
    }
    // (fusing this into the Cholesky prologue was measured: it perturbs that kernel's register allocation and is slower)
    if (!fuse_damp && !fused_comm) LAUNCH(ba->ctx, ba_prepare_camera_kernel, nblk(d.n_poses + d.n_vec3, 128), 128, 0, d);
    if (standalone && !fused) LAUNCH(ba->ctx, lm_control_pre_kernel, 1, 1, 0, d.st);
    return check_launch("linearize");
}

static int launch_step(lvb_ba* ba) {
    BaDev& d = ba->dev;
    lvb_ctx* ctx = ba->ctx;
    const bool fused = fused_pass(ba);
    LVB_TRY(ba->solver.launch(ctx, d.S, d.rhs, d.dimc, d.srow, d.soff, ba->plan.band, d.st, fused));
    LAUNCH(ba->ctx, ba_update_kernel, nblk((size_t)d.n_poses + d.n_vec3 + d.n_rho, TPB), TPB, 0, d);
    LVB_TRY(launch_linearize<1>(ba));
    if (fused) {      // the decision is taken; accept + clear over a grid sized to the larger of the two jobs
        const size_t work = std::max(d.nS / 2, (size_t)d.n_poses * 7 + (size_t)d.n_vec3 * 3 + d.n_rho);
        LAUNCH(ba->ctx, ba_post_wide_kernel, std::min(4 * ba->ctx->sm_count, nblk(work, 256)), 256, 0, d);
        return check_launch("step");
    }
    if (ctx->world > 1) LVB_TRY(comm_allreduce_sum_f64(ctx, &d.st->cand_cost_acc, 5));
    const bool wide = wide_post(ba);
    LAUNCH(ba->ctx, ba_post_kernel, 1, wide ? 32 : 1024, 0, d, wide ? 1 : 0);
    if (wide) LAUNCH(ba->ctx, ba_post_wide_kernel, 4 * ba->ctx->sm_count, 256, 0, d);
    return check_launch("step");
}

static int launch_clear(lvb_ba* ba) {
    BaDev& d = ba->dev;
    const bool zero_S = fused_pass(ba);
    const size_t n = d.nS + d.dimc + 2 * (size_t)d.n_rho + (zero_S ? d.nS + d.dimc : 0);
    LAUNCH(ba->ctx, ba_zero_kernel, std::min(1024, nblk(n, 256)), 256, 0, d, zero_S ? 1 : 0);
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
    const int m = (mode == 1 && ba->plan.tc_ok) ? 1 : 0;
    ba->dev.tc_mode = m;
    if (ba->pass_graph && ba->graph_mode != m) drop_graph(ba);
    ba->graph_mode = m;
}

static int require_solvable(lvb_ba* ba) {
    if (!ba->finalized) { set_error("finalize first"); return LVB_ERR_STATE; }
    if (!ba->plan.solvable) { set_error("camera system of dimension %d cannot be solved: %s", ba->plan.dimc, ba->plan.unsolvable_why); return LVB_ERR_UNSUPPORTED; }
    return check_imu_status(ba);
}

int lvb_ba_reduced_system(lvb_ba* ba, double radius, double* S, double* b, double* cost) {
    LVB_TRY(require_solvable(ba));
    LVB_CUDA(cudaSetDevice(ba->ctx->device)); lvb::g_alloc_stream = ba->ctx->stream;
    apply_schur_mode(ba, ba->schur_mode);
    LVB_TRY(upload_state(ba, nullptr, radius));
    LVB_TRY(launch_clear(ba));
    LVB_TRY(launch_linearize_and_reduce(ba, true));
    const int n = ba->plan.dimc;
    if ((size_t)n > 8192) { set_error("lvb_ba_reduced_system: dimension %d is too large for a dense download", n); return LVB_ERR_UNSUPPORTED; }
    std::vector<double> hS(ba->plan.nS);
    const size_t srow = (size_t)ba->plan.srow, soff = (size_t)ba->plan.soff; const int band = (ba->plan.soff == 0) ? n : ba->plan.band;
    auto at = [&](int i, int j) { return (i - j <= band) ? hS[(size_t)i * srow + j + soff] : 0.0; };   // i >= j
    LmState h;
    cudaStream_t s = ba->ctx->stream;
    LVB_CUDA(cudaMemcpyAsync(hS.data(), ba->dev.S, hS.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (b) LVB_CUDA(cudaMemcpyAsync(b, ba->dev.rhs, n * sizeof(double), cudaMemcpyDeviceToHost, s));
    LVB_CUDA(cudaMemcpyAsync(&h, ba->st.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    LVB_TRY(lvb::host_sync(ba->ctx, s));
    // hand the system back in the caller-visible order (all poses, then all vec3 blocks)
    const std::vector<int>& cn = ba->plan.canon;
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
    lvb::timing_mark(s, "begin");
    LVB_TRY(launch_clear(ba));
    // The pass is a fixed sequence of launches whose kernels all read their control flags from the device state,
    // so it is captured once into a CUDA graph and replayed; the host looks at the state only every
    // `check_every` passes (kernels of a finished solve return immediately).
    const bool graph_ok = comm_graph_safe(ba->ctx, ba->plan.nS + 3 * (size_t)ba->plan.dimc + 16) && ba->ctx->use_graph && !g_timing;
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
                if (cudaGraphExecUpdate(cx->graph_cache, g, &info) == cudaSuccess) {
                    ba->pass_graph = cx->graph_cache; ba->graph_borrowed = true; cx->graph_owner = ba;
                    if (prof_on) fprintf(stderr, "[solve] cached graph re-targeted\n");
                }
                else { cudaGetLastError(); cudaGraphExecDestroy(cx->graph_cache); cx->graph_cache = nullptr; cx->graph_owner = nullptr; }
            }
            if (!ba->pass_graph) {
                cudaGraphExec_t ex = nullptr;
                // no cudaGraphInstantiateFlagUseNodePriority: every node of a replay, the side-stream branches included, runs at the
                // priority of the stream the graph is launched into, i.e. the context's (lvb_ctx_create_with_priority), and a cached
                // graph re-targeted to another problem of the context keeps doing so
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
        LVB_TRY(lvb::host_sync(ba->ctx, s));
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
    LVB_TRY(lvb::host_sync(c, s));
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
    LAUNCH(ba->ctx, ba_reproj_error_kernel, nblk(n, 128), 128, 0, ba->dev, n, d_in.p, d_idx.p, d_err.p);
    LVB_TRY(check_launch("reproj"));
    LVB_TRY(d_err.download(err, n, s));
    LVB_TRY(lvb::host_sync(ba->ctx, s));
    return LVB_OK;
}

}  // extern "C"
