// Dependent-issue latencies of the instructions in the pivot chain of the diagonal-block Cholesky (one warp, sm_90a).
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o lat_probe lat_probe.cu ; run on the GPU box
#include <cstdio>
#include <cmath>
#include <cuda_runtime.h>
__device__ __forceinline__ double rsqrt_seed(double x) { double y; asm volatile("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x)); return y; }
__device__ __forceinline__ double rcp_seed(double x) { double y; asm volatile("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x)); return y; }
__device__ __forceinline__ double rsqrt_pos(double x) {
    double y = rsqrt_seed(x);
    double g = x * y, h = 0.5 * y;
    double r = fma(-g, h, 0.5);
    g = fma(g, r, g); h = fma(h, r, h);
    r = fma(-g, h, 0.5);
    h = fma(h, r, h);
    return h + h;
}
__device__ __forceinline__ double rsqrt_cubic(double x) {      // seed + one third-order step
    double y = rsqrt_seed(x);
    double t = x * y;
    double e = fma(-t, y, 1.0);
    double p = fma(e, 0.375, 0.5), ye = y * e;
    return fma(ye, p, y);
}
// worst relative error of the seed and of the two refinements over a sweep of mantissas and exponents
__global__ void accuracy(double* out) {
    double ws = 0, wg = 0, wc = 0;
    for (int i = threadIdx.x; i < (1 << 20); i += blockDim.x) {
        const double m = 1.0 + (double)i / (double)(1 << 20) * 3.0 + 1e-7 * (i % 977);
        for (int ex = -40; ex <= 40; ex += 20) {
            const double x = ldexp(m, ex);
            const double ref = 1.0 / sqrt(x);
            ws = fmax(ws, fabs(rsqrt_seed(x) - ref) / ref);
            wg = fmax(wg, fabs(rsqrt_pos(x) - ref) / ref);
            wc = fmax(wc, fabs(rsqrt_cubic(x) - ref) / ref);
        }
    }
    for (int o = 16; o; o >>= 1) { ws = fmax(ws, __shfl_xor_sync(~0u, ws, o)); wg = fmax(wg, __shfl_xor_sync(~0u, wg, o)); wc = fmax(wc, __shfl_xor_sync(~0u, wc, o)); }
    __shared__ double sh[3][32];
    if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = ws; sh[1][threadIdx.x >> 5] = wg; sh[2][threadIdx.x >> 5] = wc; }
    __syncthreads();
    if (threadIdx.x == 0) { for (int k = 0; k < 3; ++k) { double w = 0; for (int i = 0; i < (int)blockDim.x / 32; ++i) w = fmax(w, sh[k][i]); out[k] = w; } }
}
template <int OP> __global__ void probe(double* out, long long* cyc, double seed, double b) {
    double x = seed + threadIdx.x * 1e-9;
    const int lane = threadIdx.x & 31;
    long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < 64; ++it) {
#pragma unroll
        for (int u = 0; u < 16; ++u) {
            if (OP == 0) x = fma(x, b, 1e-30);
            if (OP == 1) x = x * b;
            if (OP == 2) x = __shfl_sync(0xffffffffu, x, (lane + 1) & 31);
            if (OP == 3) x = rsqrt_seed(x) + 1.0;                // seed + one DADD (keeps it in range)
            if (OP == 4) x = rsqrt_pos(x) + 1.0;
            if (OP == 5) x = 1.0 / sqrt(x) + 1.0;
            if (OP == 6) x = rcp_seed(x) + 1.0;
            if (OP == 7) x = x + b;
            if (OP == 8) { float f = __double2float_rn(x); f = rsqrtf(f); x = (double)f + 1.0; }
            if (OP == 9) { x = __shfl_sync(0xffffffffu, x * b, (lane + 1) & 31); x = fma(x, b, 1e-30); }    // mul -> shfl -> fma
            if (OP == 10) { float f = __double2float_rn(x); x = (double)f; }
            if (OP == 12) x = rsqrt_cubic(x) + 1.0;
            if (OP == 11) { float f = __double2float_rn(x); f = fmaf(f, 1.0000001f, 1e-30f); x = (double)f; }
        }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) *cyc = t1 - t0;
    out[threadIdx.x] = x;
}
template <int OP> static void run(const char* name, int dadd) {
    double* out; long long* cyc; cudaMalloc(&out, 256); cudaMalloc(&cyc, 8);
    for (int w = 0; w < 2; ++w) probe<OP><<<1, 32>>>(out, cyc, 1.5, 1.0000001);
    long long h; cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    printf("%-44s %7.1f cycles per op%s\n", name, h / 1024.0, dadd ? "  (includes one dependent DADD)" : "");
    cudaFree(out); cudaFree(cyc);
}
int main() {
    run<0>("DFMA dependent", 0); run<1>("DMUL dependent", 0); run<7>("DADD dependent", 0); run<2>("SHFL.IDX 64-bit dependent", 0);
    run<3>("MUFU.RSQ64H seed", 1); run<6>("MUFU.RCP64H seed", 1); run<4>("rsqrt_pos (seed + 2 Goldschmidt)", 1); run<5>("1.0 / sqrt(x) library", 1);
    run<8>("F2F + MUFU.RSQ f32 + F2F", 1); run<9>("DMUL -> SHFL -> DFMA", 0); run<10>("F2F.F32.F64 + F2F.F64.F32 round trip", 0); run<11>("F2F + FFMA + F2F", 0);
    run<12>("rsqrt cubic (seed + one 3rd-order step)", 1);
    double* acc; cudaMalloc(&acc, 24); accuracy<<<1, 1024>>>(acc); double h[3]; cudaMemcpy(h, acc, 24, cudaMemcpyDeviceToHost);
    printf("max relative error: seed %.3e (2^%.1f)   Goldschmidt x2 %.3e   cubic %.3e\n", h[0], log2(h[0]), h[1], h[2]);
    cudaError_t e = cudaDeviceSynchronize(); if (e) printf("error %s\n", cudaGetErrorString(e));
    return 0;
}
