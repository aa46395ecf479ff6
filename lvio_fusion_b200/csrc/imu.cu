// imu.cu -- batched IMU preintegration on the device (SURVEY 8(f).3: the step before the ImuError factor).
//
// Replaces, for a whole window / map of keyframe intervals at once,
//   Preintegration::Append + Propagate + MidPointIntegration   (imu/preintegration.h:27-40, src/preintegration.cpp:30-127)
//   Preintegration::Repropagate                                 (src/preintegration.cpp:129-142): the same call with new biases
// and emits the LVB_IMU constant records (469 doubles) that lvb_ba_add_factors(LVB_IMU, ...) consumes.
//
// One warp per interval: the 15x15 Jacobian / covariance chains live in shared memory, lane 0 integrates the
// state and fills the few 3x3 blocks of F and V that change, all lanes do the three 15x15 products.
#include <algorithm>
#include <cstring>
#include <vector>

#include "lvb_internal.cuh"
#include "lvb_math.cuh"

namespace {

using namespace lvb;

enum { IMU_OUT = 469, WARPS = 4, WS = 225 * 4 + 15 * 18 };   // per-warp shared doubles: jac, cov, F, tmp, V

__device__ __forceinline__ void put_block(double* A, int ld, int r, int c, const M3& b, double s) {
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) A[(r + i) * ld + c + j] = s * b.m[3 * i + j];
}
__device__ __forceinline__ M3 add(const M3& a, const M3& b) { M3 r; for (int i = 0; i < 9; ++i) r.m[i] = a.m[i] + b.m[i]; return r; }
__device__ __forceinline__ M3 ident_minus(const M3& a, double s) { M3 r; for (int i = 0; i < 9; ++i) r.m[i] = ((i % 4 == 0) ? 1.0 : 0.0) - a.m[i] * s; return r; }

__global__ void __launch_bounds__(32 * WARPS) imu_preintegrate_kernel(int n, const int* __restrict__ first, const double* __restrict__ samples,
                                                                      const double* __restrict__ acc0, const double* __restrict__ gyr0,
                                                                      const double* __restrict__ ba, const double* __restrict__ bg,
                                                                      double na2, double ng2, double nwa2, double nwg2, double* __restrict__ out) {
    extern __shared__ __align__(16) double sm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = blockIdx.x * WARPS + warp;
    if (f >= n) return;
    double* jac = sm + (size_t)warp * WS;
    double* cov = jac + 225;
    double* F = cov + 225;
    double* tmp = F + 225;
    double* V = tmp + 225;
    for (int e = lane; e < 225; e += 32) { const int i = e / 15, j = e - 15 * i; jac[e] = (i == j) ? 1.0 : 0.0; cov[e] = 0.0; F[e] = (i == j) ? 1.0 : 0.0; }
    for (int e = lane; e < 270; e += 32) V[e] = 0.0;
    __syncwarp();
    // state (lane 0)
    V3 dp = v3(0, 0, 0), dv = v3(0, 0, 0), a0 = v3(0, 0, 0), g0 = v3(0, 0, 0);
    Q4 dq = q4(0, 0, 0, 1);
    double sum_dt = 0.0;
    const V3 lba = v3(ba[3 * f], ba[3 * f + 1], ba[3 * f + 2]), lbg = v3(bg[3 * f], bg[3 * f + 1], bg[3 * f + 2]);
    if (lane == 0) { a0 = v3(acc0[3 * f], acc0[3 * f + 1], acc0[3 * f + 2]); g0 = v3(gyr0[3 * f], gyr0[3 * f + 1], gyr0[3 * f + 2]); }
    const double nz[6] = {na2, ng2, na2, ng2, nwa2, nwg2};       // per 3-column group of V (preintegration.cpp:15-28)
    for (int s = first[f]; s < first[f + 1]; ++s) {
        if (lane == 0) {
            const double* r = samples + 7 * (size_t)s;
            const double dt = r[0];
            const V3 a1 = v3(r[1], r[2], r[3]), g1 = v3(r[4], r[5], r[6]);
            // midpoint integration (preintegration.cpp:40-48)
            const V3 ua0 = a0 - lba, ua1 = a1 - lba;
            const V3 w = (g0 + g1) * 0.5 - lbg;
            const Q4 rq = qmul(dq, q4(w.x * dt / 2, w.y * dt / 2, w.z * dt / 2, 1.0));
            const V3 un_acc = (qrot(dq, ua0) + qrot(rq, ua1)) * 0.5;
            const V3 ndp = dp + dv * dt + un_acc * (0.5 * dt * dt);
            const V3 ndv = dv + un_acc * dt;
            // F and V blocks (preintegration.cpp:50-98)
            const M3 Rd = qmat(dq), Rr = qmat(rq);
            const M3 RdA0 = mul(Rd, skew(ua0)), RrA1 = mul(Rr, skew(ua1));
            const M3 ImW = ident_minus(skew(w), dt);
            const M3 RrA1W = mul(RrA1, ImW);
            const M3 RdRr = add(Rd, Rr);
            M3 I; for (int i = 0; i < 9; ++i) I.m[i] = (i % 4 == 0) ? 1.0 : 0.0;
            const double q = 0.25 * dt * dt, h = 0.5 * dt;
            M3 f03, f63;
            for (int i = 0; i < 9; ++i) { f03.m[i] = RdA0.m[i] * -q + RrA1W.m[i] * -q; f63.m[i] = RdA0.m[i] * -h + RrA1W.m[i] * -h; }
            put_block(F, 15, 0, 3, f03, 1.0);
            put_block(F, 15, 0, 6, I, dt);
            put_block(F, 15, 0, 9, RdRr, -q);
            put_block(F, 15, 0, 12, RrA1, -q * -dt);
            put_block(F, 15, 3, 3, ImW, 1.0);
            put_block(F, 15, 3, 12, I, -dt);
            put_block(F, 15, 6, 3, f63, 1.0);
            put_block(F, 15, 6, 9, RdRr, -h);
            put_block(F, 15, 6, 12, RrA1, -h * -dt);
            put_block(V, 18, 0, 0, Rd, q);
            put_block(V, 18, 0, 3, RrA1, -q * 0.5 * dt);
            put_block(V, 18, 0, 6, Rr, q);
            put_block(V, 18, 0, 9, RrA1, -q * 0.5 * dt);
            put_block(V, 18, 3, 3, I, h);
            put_block(V, 18, 3, 9, I, h);
            put_block(V, 18, 6, 0, Rd, h);
            put_block(V, 18, 6, 3, RrA1, -h * 0.5 * dt);
            put_block(V, 18, 6, 6, Rr, h);
            put_block(V, 18, 6, 9, RrA1, -h * 0.5 * dt);
            put_block(V, 18, 9, 12, I, dt);
            put_block(V, 18, 12, 15, I, dt);
            // commit, normalise, advance (:117-126)
            dp = ndp; dv = ndv;
            const double nrm = sqrt(rq.x * rq.x + rq.y * rq.y + rq.z * rq.z + rq.w * rq.w);
            dq = q4(rq.x / nrm, rq.y / nrm, rq.z / nrm, rq.w / nrm);
            sum_dt += dt;
            a0 = a1; g0 = g1;
        }
        __syncwarp();
        // jacobian = F jacobian ; covariance = F cov F^T + V N V^T   (:100-101)
        for (int e = lane; e < 225; e += 32) {
            const int i = e / 15, j = e - 15 * i;
            double a = 0.0;
            for (int k = 0; k < 15; ++k) a += F[i * 15 + k] * jac[k * 15 + j];
            tmp[e] = a;
        }
        __syncwarp();
        for (int e = lane; e < 225; e += 32) jac[e] = tmp[e];
        __syncwarp();
        for (int e = lane; e < 225; e += 32) {
            const int i = e / 15, j = e - 15 * i;
            double a = 0.0;
            for (int k = 0; k < 15; ++k) a += F[i * 15 + k] * cov[k * 15 + j];
            tmp[e] = a;
        }
        __syncwarp();
        for (int e = lane; e < 225; e += 32) {
            const int i = e / 15, j = e - 15 * i;
            double a = 0.0, b = 0.0;
            for (int k = 0; k < 15; ++k) a += tmp[i * 15 + k] * F[j * 15 + k];
            for (int k = 0; k < 18; ++k) b += V[i * 18 + k] * nz[k / 3] * V[j * 18 + k];
            cov[e] = a + b;
        }
        __syncwarp();
    }
    double* o = out + (size_t)f * IMU_OUT;
    if (lane == 0) {
        o[0] = dp.x; o[1] = dp.y; o[2] = dp.z; o[3] = dq.x; o[4] = dq.y; o[5] = dq.z; o[6] = dq.w;
        o[7] = dv.x; o[8] = dv.y; o[9] = dv.z; o[10] = lba.x; o[11] = lba.y; o[12] = lba.z; o[13] = lbg.x; o[14] = lbg.y; o[15] = lbg.z;
        o[16] = sum_dt; o[467] = -1.0; o[468] = -1.0;
    }
    for (int e = lane; e < 225; e += 32) { o[17 + e] = jac[e]; o[17 + 225 + e] = cov[e]; }
}

}  // namespace

extern "C" int lvb_imu_preintegrate(lvb_ctx* ctx, int n, const int32_t* first, const double* samples, const double* acc0, const double* gyr0,
                                    const double* ba, const double* bg, const double noise[4], double* consts) {
    if (!ctx || n < 0 || (n && (!first || !acc0 || !gyr0 || !ba || !bg || !noise || !consts))) { lvb::set_error("lvb_imu_preintegrate: bad arguments"); return LVB_ERR_INVALID; }
    if (n == 0) return LVB_OK;
    if (first[0] != 0) { lvb::set_error("lvb_imu_preintegrate: first[0] must be 0"); return LVB_ERR_INVALID; }
    for (int i = 0; i < n; ++i) if (first[i + 1] < first[i]) { lvb::set_error("lvb_imu_preintegrate: first[] must be non-decreasing"); return LVB_ERR_INVALID; }
    const int ns = first[n];
    if (ns && !samples) { lvb::set_error("lvb_imu_preintegrate: samples missing"); return LVB_ERR_INVALID; }
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    cudaStream_t s = ctx->stream;
    lvb::DevBuf<int> d_first; lvb::DevBuf<double> d_samples, d_vec, d_out;
    LVB_TRY(d_first.upload(first, (size_t)n + 1, s));
    LVB_TRY(d_samples.upload(samples, (size_t)ns * 7, s));
    std::vector<double> pack((size_t)12 * n);
    memcpy(pack.data(), acc0, sizeof(double) * 3 * n); memcpy(pack.data() + 3 * (size_t)n, gyr0, sizeof(double) * 3 * n);
    memcpy(pack.data() + 6 * (size_t)n, ba, sizeof(double) * 3 * n); memcpy(pack.data() + 9 * (size_t)n, bg, sizeof(double) * 3 * n);
    LVB_TRY(d_vec.upload(pack.data(), pack.size(), s));
    LVB_TRY(d_out.ensure((size_t)n * IMU_OUT));
    static bool attr = false;
    const size_t smem = (size_t)WARPS * WS * sizeof(double);
    if (!attr) { LVB_CUDA(cudaFuncSetAttribute(imu_preintegrate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
    imu_preintegrate_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS, smem, s>>>(n, d_first.p, d_samples.p, d_vec.p, d_vec.p + 3 * (size_t)n, d_vec.p + 6 * (size_t)n,
                                                                               d_vec.p + 9 * (size_t)n, noise[0] * noise[0], noise[1] * noise[1], noise[2] * noise[2], noise[3] * noise[3], d_out.p);
    ctx->launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { lvb::set_error("imu_preintegrate launch failed: %s", cudaGetErrorString(e)); return LVB_ERR_CUDA; }
    LVB_TRY(d_out.download(consts, (size_t)n * IMU_OUT, s));
    LVB_TRY(lvb::host_sync(ctx, s));
    return LVB_OK;
}
