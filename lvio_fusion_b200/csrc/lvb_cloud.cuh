// lvb_cloud.cuh -- point-cloud device helpers shared by icp.cu (scan-to-map) and lidar.cu (feature pipeline):
// order-preserving float <-> int mapping for atomic min/max, the bit-reproducible float32 SE3 transform, and a
// three-kernel exclusive scan (1024 elements per block).  Everything has internal linkage (one copy per TU).
#pragma once
#include <cuda_runtime.h>
#include <string.h>

namespace {

// ---- float ordering helpers for atomic min / max
__device__ __forceinline__ int f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__host__ __device__ inline float ord2f(int i) { int j = i >= 0 ? i : i ^ 0x7fffffff; float f; memcpy(&f, &j, 4); return f; }

// association.cpp:287-294: ceres::SE3TransformPoint<float> with the float-cast pose.  Operation order of
// ceres::QuaternionRotatePoint / UnitQuaternionRotatePoint [upstream], every product and sum rounded
// separately (no FMA contraction) so that the CPU oracle reproduces the bits.
__device__ __forceinline__ float3 transform_f32(const float* tf, float3 p) {
    const float qx = tf[0], qy = tf[1], qz = tf[2], qw = tf[3];
    const float n2 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(qw, qw), __fmul_rn(qx, qx)), __fmul_rn(qy, qy)), __fmul_rn(qz, qz));
    const float scale = __fdiv_rn(1.0f, __fsqrt_rn(n2));
    const float ux = __fmul_rn(scale, qx), uy = __fmul_rn(scale, qy), uz = __fmul_rn(scale, qz), uw = __fmul_rn(scale, qw);
    float uv0 = __fsub_rn(__fmul_rn(uy, p.z), __fmul_rn(uz, p.y));
    float uv1 = __fsub_rn(__fmul_rn(uz, p.x), __fmul_rn(ux, p.z));
    float uv2 = __fsub_rn(__fmul_rn(ux, p.y), __fmul_rn(uy, p.x));
    uv0 = __fadd_rn(uv0, uv0); uv1 = __fadd_rn(uv1, uv1); uv2 = __fadd_rn(uv2, uv2);
    float rx = __fadd_rn(p.x, __fmul_rn(uw, uv0));
    float ry = __fadd_rn(p.y, __fmul_rn(uw, uv1));
    float rz = __fadd_rn(p.z, __fmul_rn(uw, uv2));
    rx = __fadd_rn(rx, __fsub_rn(__fmul_rn(uy, uv2), __fmul_rn(uz, uv1)));
    ry = __fadd_rn(ry, __fsub_rn(__fmul_rn(uz, uv0), __fmul_rn(ux, uv2)));
    rz = __fadd_rn(rz, __fsub_rn(__fmul_rn(ux, uv1), __fmul_rn(uy, uv0)));
    return make_float3(__fadd_rn(rx, tf[4]), __fadd_rn(ry, tf[5]), __fadd_rn(rz, tf[6]));
}

// exclusive scan, 1024 elements per block: (1) per-block scan + block totals, (2) scan of totals, (3) add.  The bodies are shared with
// icp.cu's variants that read the element count from device memory.
__device__ __forceinline__ void scan_block(const int* in, int* out, int n, int* block_sums) {
    __shared__ int s[1024];
    const int i = blockIdx.x * 1024 + threadIdx.x;
    const int v = i < n ? in[i] : 0;
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const int t = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
        __syncthreads();
        s[threadIdx.x] += t;
        __syncthreads();
    }
    if (i < n) out[i] = s[threadIdx.x] - v;
    if (threadIdx.x == 1023) block_sums[blockIdx.x] = s[1023];
}
__device__ __forceinline__ void scan_sums(int* block_sums, int nb, int* total_out) {
    __shared__ int s[1024];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nb; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < nb ? block_sums[i] : 0;
        s[threadIdx.x] = v;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {
            const int t = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
            __syncthreads();
            s[threadIdx.x] += t;
            __syncthreads();
        }
        if (i < nb) block_sums[i] = carry + s[threadIdx.x] - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry += s[1023];
        __syncthreads();
    }
    if (threadIdx.x == 0) *total_out = carry;
}
__device__ __forceinline__ void scan_add(int* out, int n, const int* block_sums, int* last, const int* total) {
    const int i = blockIdx.x * 1024 + threadIdx.x;
    if (i < n) out[i] += block_sums[blockIdx.x];
    if (i == 0) *last = *total;
}
__global__ void scan_block_kernel(const int* in, int* out, int n, int* block_sums) { scan_block(in, out, n, block_sums); }
__global__ void scan_sums_kernel(int* block_sums, int nb, int* total_out) { scan_sums(block_sums, nb, total_out); }
__global__ void scan_add_kernel(int* out, int n, const int* block_sums, int* last /*out[n] = total*/, const int* total) { scan_add(out, n, block_sums, last, total); }

}  // namespace
