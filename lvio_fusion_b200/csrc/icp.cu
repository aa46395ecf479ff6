// icp.cu -- lidar scan-to-map registration on the device: the kernels behind
// pcl::KdTreeFLANN + FeatureAssociation::ScanToMapWith{Ground,Segmented} + the two DENSE_QR solves
// of Mapping::Optimize (/root/reference/src/lvio_fusion/src/association.cpp:270-384,
// src/mapping.cpp:139-191).
//
//   K7  voxel hash build : key = ix + gx*(iy + gy*iz) over the cloud's bounding box (the PCL VoxelGrid
//       keying), counting sort (histogram -> exclusive scan -> scatter) = one radix pass with radix #cells
//   K8  transform + exact 3-NN + gate : float32, no fused multiply-add (__f*_rn), ascending (d2, index)
//   K9  point-to-plane residual/Jacobian + 3x3 normal equations reduce + LM on three scalars
//
// HBM layout: map cloud re-packed as float4 (x, y, z, original index bits) sorted by voxel key (16 B/pt);
// cell_start int32[#cells+1]; scan cloud read in place from the caller's record stride after upload;
// per-query association: accepted u8, pa float[3][K], normal double[3][K] (SoA planes).
#include <float.h>
#include <math.h>
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <stdlib.h>
#include <string.h>
#include <unordered_map>
#include <unordered_set>
#include <vector>
#include "lvb_internal.cuh"
#include "lvb_math.cuh"
#include "lvb_cloud.cuh"

using namespace lvb;

namespace {

enum { ITPB = 128, MAX_CELLS = 1 << 26 };

struct Grid {
    float minx, miny, minz, inv_cell, cell;   // cell = voxel edge = (search radius * 1.0001) / ring
    int gx, gy, gz;
    int ring;                                 // voxels per search radius: neighbours within the radius lie within `ring` voxels
    int cbx, cby, cbz;                        // the coarse occupancy grid: blocks of 4 x 4 x 4 voxels
};

struct IcpState {
    LmState lm;
    int mode;
    double Twc1[7];
    double rpyxyz[6];
    double x[3], cand[3], delta[3], lam[3], scale[3], grad[3];
    double prior_w, prior_target[3], huber_a, weight;
    double acc[16];      // consumed system: H (9, row-major), g (3), cost, n_accepted
    double part[16];     // per-pass partial sums written by the linearize kernels (all-reduced when world > 1): [0..13] as acc, [14] candidate cost
};

// A map frame: its voxel grid and the sizes that follow from it, decided on the device by icp_map_grid_kernel from the cloud's bounding
// box and read by every kernel that looks at the map.  The host keeps the copy it reads back after the build.
struct MapDesc {
    Grid g;
    int P;                       // map points; 0: an empty map frame (SegmentGround kept no point), which accepts no query
    int ncell, ncb;              // gx * gy * gz; cbx * cby * cbz
    int shift, cgx, cgy, cgz, nc;           // query visiting order (bind_scan): key granularity and its grid
    int err;                     // 0, 1: no finite bounding box, 2: more than MAX_CELLS voxels at ring 1
    int bbox[6];                 // the cloud's bounding box (ordered ints, icp_bbox_kernel's layout), uploaded with its seed values
};

struct IcpDev {
    const float4* map;           // sorted by cell
    const int* cell_start;
    const int* coarse;           // occupancy of the coarse blocks of the map grid (1: holds points)
    const MapDesc* m;            // the map frame's grid (device)
    const float* tf;             // float[7]: the frame pose cast to float (association.cpp:287), in device memory
    const unsigned char* scan;   // device copy of the caller's records
    int K, stride;
    float max_d2;
    double thr;
    unsigned char* accepted;
    float* pa;                   // 3 planes
    double* nrm;                 // 3 planes
    IcpState* st;
    const int* order;            // query visiting order (spatially sorted) or nullptr
};

__device__ __forceinline__ float3 load_xyz(const unsigned char* base, int i, int stride) {
    const float* f = reinterpret_cast<const float*>(base + (size_t)i * stride);
    return make_float3(f[0], f[1], f[2]);
}

// warp min / max of the per-thread boxes, merged into bbox[6] (min xyz, max xyz as ordered ints) by one lane per warp
__device__ __forceinline__ void bbox_merge(float* mn, float* mx, int* bbox) {
    for (int a = 0; a < 3; ++a) {
        for (int o = 16; o > 0; o >>= 1) { mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o)); mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o)); }
        if ((threadIdx.x & 31) == 0) { atomicMin(&bbox[a], f2ord(mn[a])); atomicMax(&bbox[3 + a], f2ord(mx[a])); }
    }
}
// the bounding box of the map frame's m->P points into m->bbox (uploaded with its seed values)
__global__ void icp_bbox_kernel(const unsigned char* pts, int stride, MapDesc* m) {
    const int n = m->P;
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float3 p = load_xyz(pts, i, stride);
        mn[0] = fminf(mn[0], p.x); mn[1] = fminf(mn[1], p.y); mn[2] = fminf(mn[2], p.z);
        mx[0] = fmaxf(mx[0], p.x); mx[1] = fmaxf(mx[1], p.y); mx[2] = fmaxf(mx[2], p.z);
    }
    bbox_merge(mn, mx, m->bbox);
}

__device__ __forceinline__ int cell_coord(float v, float mn, float inv_cell) { return (int)floorf((v - mn) * inv_cell); }
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__global__ void icp_count_kernel(const unsigned char* pts, int stride, const MapDesc* m, int* cell_of, int* counts, int* coarse) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m->P) return;
    const Grid& g = m->g;
    const float3 p = load_xyz(pts, i, stride);
    const int ix = clampi(cell_coord(p.x, g.minx, g.inv_cell), 0, g.gx - 1);
    const int iy = clampi(cell_coord(p.y, g.miny, g.inv_cell), 0, g.gy - 1);
    const int iz = clampi(cell_coord(p.z, g.minz, g.inv_cell), 0, g.gz - 1);
    const int c = ix + g.gx * (iy + g.gy * iz);
    cell_of[i] = c;
    atomicAdd(&counts[c], 1);
    coarse[(ix >> 2) + g.cbx * ((iy >> 2) + g.cby * (iz >> 2))] = 1;       // benign race: every writer stores 1
}

__global__ void icp_scatter_kernel(const unsigned char* pts, int stride, const MapDesc* m, const int* cell_of, const int* cell_start, int* fill, float4* sorted) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m->P) return;
    const float3 p = load_xyz(pts, i, stride);
    const int c = cell_of[i];
    const int pos = cell_start[c] + atomicAdd(&fill[c], 1);
    sorted[pos] = make_float4(p.x, p.y, p.z, __int_as_float(i));
}

// zero a[0..*n) (and b[0..*n) unless null): counters sized on the host by an upper bound, used up to the size the device decided
__global__ void icp_zero_map_kernel(int* a, int* b, const int* n) {
    const int cnt = *n;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += gridDim.x * blockDim.x) { a[i] = 0; if (b) b[i] = 0; }
}
// the exclusive scan of lvb_cloud.cuh over the first *n entries (a count the device decided; blocks launched for it or an upper bound)
__global__ void scan_block_map_kernel(const int* in, int* out, const int* n, int* block_sums) {
    const int cnt = *n;
    if ((int)blockIdx.x * 1024 >= cnt) return;
    scan_block(in, out, cnt, block_sums);
}
__global__ void scan_sums_map_kernel(int* block_sums, const int* n, int* total_out) { scan_sums(block_sums, (*n + 1023) / 1024, total_out); }
__global__ void scan_add_map_kernel(int* out, const int* n, const int* block_sums, const int* total) {
    const int cnt = *n;
    if ((int)blockIdx.x * 1024 >= cnt) return;
    scan_add(out, cnt, block_sums, out + cnt, total);
}

// Mapping::MergeScan (mapping.cpp:193-203): world cloud = float32 SE3 transform of the robot-frame cloud; the other
// fields of each record (intensity, padding) are carried over unchanged.
__global__ void icp_transform_cloud_kernel(const unsigned char* __restrict__ in, unsigned char* __restrict__ out, int n, int stride, const float* __restrict__ tf7) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float tf[7];
    for (int k = 0; k < 7; ++k) tf[k] = tf7[k];
    const float* src = reinterpret_cast<const float*>(in + (size_t)i * stride);
    float* dst = reinterpret_cast<float*>(out + (size_t)i * stride);
    const float3 q = transform_f32(tf, make_float3(src[0], src[1], src[2]));
    dst[0] = q.x; dst[1] = q.y; dst[2] = q.z;
    for (int k = 3; k < stride / 4; ++k) dst[k] = src[k];
}

// Mapping::ToWorld (mapping.cpp:205-220) into the resident store: records of any stride -> packed (x, y, z, intensity) in the world
// frame, and the same records untransformed into `robot` (lvb_icp_map_to_world re-anchors from them); with bbox, also the bounding
// box of the stored cloud into bbox[6] (icp_bbox_kernel's min / max: equal to what it finds on `out`)
__global__ void icp_to_world_kernel(const unsigned char* __restrict__ in, float4* __restrict__ out, float4* __restrict__ robot, int n, int stride,
                                    const float* __restrict__ tf7, int* bbox) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    if (i < n) {
        float tf[7];
        for (int k = 0; k < 7; ++k) tf[k] = tf7[k];
        const float* src = reinterpret_cast<const float*>(in + (size_t)i * stride);
        const float w = stride >= 16 ? src[3] : 0.0f;
        const float3 q = transform_f32(tf, make_float3(src[0], src[1], src[2]));
        out[i] = make_float4(q.x, q.y, q.z, w);
        if (robot) robot[i] = make_float4(src[0], src[1], src[2], w);
        mn[0] = fminf(mn[0], q.x); mn[1] = fminf(mn[1], q.y); mn[2] = fminf(mn[2], q.z);
        mx[0] = fmaxf(mx[0], q.x); mx[1] = fmaxf(mx[1], q.y); mx[2] = fmaxf(mx[2], q.z);
    }
    if (bbox) bbox_merge(mn, mx, bbox);
}

// Mapping::ToWorld(start) (mapping.cpp:222-229) on resident clouds: one entry per (handle, keyframe) re-anchored by lvb_icp_map_to_world
struct TwSeg {
    const float4* robot;         // the keyframe's robot-frame records, as icp_to_world_kernel stored them
    float4* world;               // its world cloud, overwritten in place
    float tf[7];                 // the new pose.cast<float>()
    int n;
};
enum { TW_TPB = 256, TW_PER = 4 };      // threads per block, points per thread: a block re-anchors 1 024 points of one cloud
// Every point of every listed cloud: block b belongs to the last entry whose first block is <= b (first[]: the exclusive prefix of
// ceil(n / 1024) over the entries; an empty cloud owns no block).  The transform is icp_to_world_kernel's, so the result is what
// lvb_icp_map_append of the same records stores, bit for bit; the box of each cloud goes to boxes[6 * entry] (icp_bbox_kernel's values).
__global__ void __launch_bounds__(TW_TPB) icp_map_to_world_kernel(const TwSeg* __restrict__ segs, const int* __restrict__ first, int n_segs,
                                                                  int* __restrict__ boxes) {
    const int b = blockIdx.x;
    int lo = 0, hi = n_segs - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (__ldg(&first[mid]) <= b) lo = mid; else hi = mid - 1; }
    const TwSeg& sg = segs[lo];
    float tf[7];
    for (int k = 0; k < 7; ++k) tf[k] = sg.tf[k];
    const int n = sg.n;
    const float4* __restrict__ in = sg.robot;
    float4* __restrict__ out = sg.world;
    const int base = (b - __ldg(&first[lo])) * (TW_TPB * TW_PER) + threadIdx.x;
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
#pragma unroll
    for (int j = 0; j < TW_PER; ++j) {
        const int i = base + j * TW_TPB;
        if (i < n) {
            const float4 r = __ldg(&in[i]);
            const float3 q = transform_f32(tf, make_float3(r.x, r.y, r.z));
            out[i] = make_float4(q.x, q.y, q.z, r.w);
            mn[0] = fminf(mn[0], q.x); mn[1] = fminf(mn[1], q.y); mn[2] = fminf(mn[2], q.z);
            mx[0] = fmaxf(mx[0], q.x); mx[1] = fmaxf(mx[1], q.y); mx[2] = fmaxf(mx[2], q.z);
        }
    }
    bbox_merge(mn, mx, boxes + 6 * (size_t)lo);
}

struct Best3 { float d[3]; int i[3]; int p[3]; };   // d2, original index, position in the sorted array
__device__ __forceinline__ void best_insert(Best3& b, float d, int i, int p) {
    if (d > b.d[2] || (d == b.d[2] && i > b.i[2])) return;
    if (d < b.d[1] || (d == b.d[1] && i < b.i[1])) {
        b.d[2] = b.d[1]; b.i[2] = b.i[1]; b.p[2] = b.p[1];
        if (d < b.d[0] || (d == b.d[0] && i < b.i[0])) { b.d[1] = b.d[0]; b.i[1] = b.i[0]; b.p[1] = b.p[0]; b.d[0] = d; b.i[0] = i; b.p[0] = p; }
        else { b.d[1] = d; b.i[1] = i; b.p[1] = p; }
    } else { b.d[2] = d; b.i[2] = i; b.p[2] = p; }
}

// exact 3-NN of q among map points with d2 <= max_d2 (max_d2 <= radius^2).  Voxels are visited in Chebyshev
// rings around the query's voxel; a ring r >= 1 cannot hold a point closer than (r-1)*cell, so the search stops
// as soon as the third-best distance is strictly below that bound (strict: ties are broken by index).
struct Occ { unsigned mask; int bx, by, bz; };        // occupancy bits of the 3 x 3 x 3 coarse blocks around the query's block (bx, by, bz)
__device__ __forceinline__ void scan_voxel(const IcpDev& d, const Grid& g, float3 q, int ix, int iy, int iz, Best3& b, const Occ& occ) {
    // an empty coarse block holds no points: skip without touching memory.  A query without neighbours otherwise walks all 729 voxels
    // of the radius at two dependent L2 round trips each (~0.5 ms for ONE thread), and the kernel lasts as long as its slowest thread.
    const int bit = ((iz >> 2) - occ.bz + 1) * 9 + ((iy >> 2) - occ.by + 1) * 3 + ((ix >> 2) - occ.bx + 1);
    if (!((occ.mask >> bit) & 1u)) return;
    if (ix < 0 || iy < 0 || iz < 0 || ix >= g.gx || iy >= g.gy || iz >= g.gz) return;
    const int c = ix + g.gx * (iy + g.gy * iz);
    const int s = d.cell_start[c], e = d.cell_start[c + 1];
    if (s == e) return;
    const float bx0 = g.minx + ix * g.cell, by0 = g.miny + iy * g.cell, bz0 = g.minz + iz * g.cell;
    const float ex = fmaxf(fmaxf(bx0 - q.x, q.x - (bx0 + g.cell)), 0.0f);
    const float ey = fmaxf(fmaxf(by0 - q.y, q.y - (by0 + g.cell)), 0.0f);
    const float ez = fmaxf(fmaxf(bz0 - q.z, q.z - (bz0 + g.cell)), 0.0f);
    const float bd = (ex * ex + ey * ey + ez * ez) * 0.99f - 1e-6f;     // conservative box distance
    if (bd > b.d[2] || bd > d.max_d2) return;
    for (int j = s; j < e; ++j) {
        const float4 m = __ldg(&d.map[j]);
        const float dx = __fsub_rn(m.x, q.x), dy = __fsub_rn(m.y, q.y), dz = __fsub_rn(m.z, q.z);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        best_insert(b, d2, __float_as_int(m.w), j);
    }
}

// g: the map frame's grid, loaded from its MapDesc once per thread
__device__ __forceinline__ Best3 knn3_query(const IcpDev& d, const Grid& g, float3 q) {
    Best3 b;
    b.d[0] = b.d[1] = b.d[2] = INFINITY; b.i[0] = b.i[1] = b.i[2] = 0x7fffffff; b.p[0] = b.p[1] = b.p[2] = -1;
    const int cx = cell_coord(q.x, g.minx, g.inv_cell), cy = cell_coord(q.y, g.miny, g.inv_cell), cz = cell_coord(q.z, g.minz, g.inv_cell);
    Occ occ; occ.mask = 0u; occ.bx = cx >> 2; occ.by = cy >> 2; occ.bz = cz >> 2;       // (ring <= 4 voxels: every probed voxel lies in these 27 blocks)
#pragma unroll
    for (int k = 0; k < 27; ++k) {                  // 27 independent loads, one round trip
        const int x = occ.bx + k % 3 - 1, y = occ.by + (k / 3) % 3 - 1, z = occ.bz + k / 9 - 1;
        const bool in = x >= 0 && y >= 0 && z >= 0 && x < g.cbx && y < g.cby && z < g.cbz;
        if (in && __ldg(&d.coarse[x + g.cbx * (y + g.cby * z)])) occ.mask |= 1u << k;
    }
    scan_voxel(d, g, q, cx, cy, cz, b, occ);
    for (int r = 1; r <= g.ring; ++r) {
        const float lb = (r - 1) * g.cell;
        const float lb2 = lb * lb * 0.99f;
        if (b.d[2] < lb2 || lb2 > d.max_d2) break;
        // the six faces of the ring-r shell, each voxel exactly once
        for (int dz = -r; dz <= r; ++dz) {
            const bool zface = (dz == -r || dz == r);
            for (int dy = -r; dy <= r; ++dy) {
                const bool yface = (dy == -r || dy == r);
                if (zface || yface) { for (int dx = -r; dx <= r; ++dx) scan_voxel(d, g, q, cx + dx, cy + dy, cz + dz, b, occ); }
                else { scan_voxel(d, g, q, cx - r, cy + dy, cz + dz, b, occ); scan_voxel(d, g, q, cx + r, cy + dy, cz + dz, b, occ); }
            }
        }
    }
    for (int j = 0; j < 3; ++j) if (!(b.d[j] <= d.max_d2)) { b.d[j] = INFINITY; b.i[j] = -1; b.p[j] = -1; }
    return b;
}

// Coarse spatial key of a query (blocks of 4x4x4 voxels) so that the lanes of a warp walk the same voxel lists and
// their 16-byte map loads hit the same L1 lines instead of 32 different L2 sectors.
// Measured alternatives that lost against this per-query ring walk (round 2, 120 k queries vs 1 M points, 0.50 ms): scanning
// x-major voxel ROWS as contiguous runs (fewer probes, but no per-voxel culling: 0.78 ms); staging a coarse block's 3 x 3 x 3
// neighbourhood in shared memory per CTA and searching there (ring search on the staged copy 1.4 - 1.8 ms, brute force 4.4 ms):
// a block holds ~25 queries that look at ~50 points each, while its neighbourhood is ~3 000 points -- the staging reads 60x more
// map than the queries need; four lanes per query (a ring's voxel rows dealt round-robin, butterfly merge of the best three after
// every ring): 0.57 ms -- the lanes prune with their own looser bounds and scan more voxels than the chain they shorten; runs only for
// the face rows of the outer rings (r >= 2): 0.57 ms.  The kernel takes ~0.47 - 0.50 ms whether a rank holds 120 k, 60 k or 30 k of
// the queries (round-2 runs at 1 / 2 / 4 GPUs): its duration is set by its slowest warps, not by the query count.
__device__ __forceinline__ float3 query_point(const IcpDev& d, int i) {
    float tf[7];
    for (int k = 0; k < 7; ++k) tf[k] = d.tf[k];
    return transform_f32(tf, load_xyz(d.scan, i, d.stride));
}
__global__ void icp_query_key_kernel(IcpDev d, int* __restrict__ key, int* __restrict__ counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d.K) return;
    const float3 q = query_point(d, i);
    const MapDesc* m = d.m;
    const Grid g = m->g;
    const int shift = m->shift;
    const int ix = clampi(cell_coord(q.x, g.minx, g.inv_cell), 0, g.gx - 1) >> shift;
    const int iy = clampi(cell_coord(q.y, g.miny, g.inv_cell), 0, g.gy - 1) >> shift;
    const int iz = clampi(cell_coord(q.z, g.minz, g.inv_cell), 0, g.gz - 1) >> shift;
    const int c = ix + m->cgx * (iy + m->cgy * iz);
    key[i] = c;
    atomicAdd(&counts[c], 1);
}
__global__ void icp_query_scatter_kernel(int n, const int* __restrict__ key, const int* __restrict__ start, int* __restrict__ fill, int* __restrict__ order) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c = key[i];
    order[start[c] + atomicAdd(&fill[c], 1)] = i;
}

__global__ void __launch_bounds__(ITPB) icp_knn_kernel(IcpDev d, int* __restrict__ idx_out, float* __restrict__ d2_out) {
    const int t = blockIdx.x * ITPB + threadIdx.x;
    if (t >= d.K) return;
    const int i = d.order ? d.order[t] : t;
    const float3 q = query_point(d, i);
    const Grid g = d.m->g;               // loaded after the transform: not held across its division and square root
    const Best3 b = knn3_query(d, g, q);
    for (int j = 0; j < 3; ++j) { idx_out[3 * i + j] = b.i[j]; d2_out[3 * i + j] = b.d[j]; }
}

// K8: transform + 3-NN + gate (association.cpp:296-300) + plane constants (lidar_error.hpp:13-18).  An empty map frame (P = 0:
// SegmentGround kept no point) accepts no query.
__global__ void __launch_bounds__(ITPB) icp_associate_kernel(IcpDev d) {
    const int t = blockIdx.x * ITPB + threadIdx.x;
    if (t >= d.K) return;
    const int i = d.order ? d.order[t] : t;
    const float3 q = query_point(d, i);
    const int P = d.m->P;
    if (P == 0) { d.accepted[i] = 0; return; }
    const Grid g = d.m->g;
    const Best3 b = knn3_query(d, g, q);
    int ok = 1;
    for (int j = 0; j < 3; ++j) if (!(b.i[j] >= 0 && b.i[j] < P && (double)b.d[j] < d.thr)) ok = 0;
    d.accepted[i] = (unsigned char)ok;
    if (!ok) return;
    const float4 a = d.map[b.p[0]], bb = d.map[b.p[1]], c = d.map[b.p[2]];
    const V3 n = plane_normal(v3(a.x, a.y, a.z), v3(bb.x, bb.y, bb.z), v3(c.x, c.y, c.z));
    d.pa[i] = a.x; d.pa[d.K + i] = a.y; d.pa[2 * d.K + i] = a.z;
    d.nrm[i] = n.x; d.nrm[d.K + i] = n.y; d.nrm[2 * (size_t)d.K + i] = n.z;
}

// What a map frame's grid may use: voxels, coarse blocks and query-sort counters.  kGridLimits is what every map frame gets whose
// buffers are sized from exact boxes (2^26 voxels, coarse blocks unbounded, 8 M counters); lvb_icp_map_optimize_keyframes passes the
// capacities it allocated for a map frame whose box the host could only estimate.
struct GridCap { double cells, coarse, qsort; };
__device__ __forceinline__ bool grid_fits(double dx, double dy, double dz, const GridCap& cap) {
    const double cb = __dmul_rn(__dmul_rn(floor(__dmul_rn(__dadd_rn(dx, 3.0), 0.25)), floor(__dmul_rn(__dadd_rn(dy, 3.0), 0.25))),
                                floor(__dmul_rn(__dadd_rn(dz, 3.0), 0.25)));
    return __dmul_rn(__dmul_rn(dx, dy), dz) <= cap.cells && cb <= cap.coarse;
}

// The voxel grid of a map frame and the key granularity of its queries' visiting order, on one thread, from the bounding box in
// m->bbox.  Every float / double operation is rounded on its own (no contraction), so the grid does not depend on how this file is
// compiled.  An empty or failed map frame gets a one-voxel grid and P = 0, which every kernel treats as "nothing to do".
__global__ void icp_map_grid_kernel(MapDesc* m, float cell_size, GridCap cap) {
    Grid g;
    int P = m->P, err = 0;
    double dx = 1, dy = 1, dz = 1;
    g.ring = 1;
    if (P > 0) {
        g.minx = ord2f(m->bbox[0]); g.miny = ord2f(m->bbox[1]); g.minz = ord2f(m->bbox[2]);
        const float mx = ord2f(m->bbox[3]), my = ord2f(m->bbox[4]), mz = ord2f(m->bbox[5]);
        const float wx = __fsub_rn(mx, g.minx), wy = __fsub_rn(my, g.miny), wz = __fsub_rn(mz, g.minz);
        if (!(mx >= g.minx) || !(my >= g.miny) || !(mz >= g.minz) || !isfinite(wx) || !isfinite(wy) || !isfinite(wz)) err = 1;
        else {
            // The voxel edge is (radius * 1.0001) / ring: the hair of slack guarantees that float rounding of the voxel coordinate
            // never separates two points closer than the radius by more than `ring` voxels.  ring = 4 unless the bounding box would
            // need more voxels (or coarse blocks) than `cap` allows; every ring finds the same exact 3-NN.
            int ring = 4;
            for (;; ring >>= 1) {
                g.cell = __fdiv_rn(__fmul_rn(cell_size, 1.0001f), (float)ring); g.inv_cell = __fdiv_rn(1.0f, g.cell);
                dx = __dadd_rn(floor(__dmul_rn((double)wx, (double)g.inv_cell)), 1.0);
                dy = __dadd_rn(floor(__dmul_rn((double)wy, (double)g.inv_cell)), 1.0);
                dz = __dadd_rn(floor(__dmul_rn((double)wz, (double)g.inv_cell)), 1.0);
                if (grid_fits(dx, dy, dz, cap) || ring == 1) break;
            }
            if (!grid_fits(dx, dy, dz, cap)) err = 2;
            g.ring = ring;
        }
    }
    if (P <= 0 || err) {
        P = 0; dx = dy = dz = 1;
        g.minx = g.miny = g.minz = 0.0f; g.cell = g.inv_cell = 1.0f; g.ring = 1;
    }
    g.gx = (int)dx; g.gy = (int)dy; g.gz = (int)dz;
    g.cbx = (g.gx + 3) >> 2; g.cby = (g.gy + 3) >> 2; g.cbz = (g.gz + 3) >> 2;
    m->g = g; m->P = P; m->err = err;
    m->ncell = g.gx * g.gy * g.gz;
    m->ncb = g.cbx * g.cby * g.cbz;
    // key granularity of the query visiting order: blocks of 2 x 2 x 2 voxels (measured on configs[2], association kernel: 4 x 4 x 4
    // blocks 0.51 ms, 2 x 2 x 2 0.44 ms, single voxels 0.50 ms plus a slower sort) -- coarser only when the grid would need more
    // than cap.qsort (8 M) counters
    int shift = 1;
    while (__dmul_rn(__dmul_rn((double)((g.gx >> shift) + 1), (double)((g.gy >> shift) + 1)), (double)((g.gz >> shift) + 1)) > cap.qsort) ++shift;
    const int rnd = (1 << shift) - 1;
    m->shift = shift;
    m->cgx = (g.gx + rnd) >> shift; m->cgy = (g.gy + rnd) >> shift; m->cgz = (g.gz + rnd) >> shift;
    m->nc = m->cgx * m->cgy * m->cgz;
}

__device__ __forceinline__ void icp_substitute(const IcpState& s, const double* x, double* e) {
    for (int k = 0; k < 6; ++k) e[k] = s.rpyxyz[k];
    if (s.mode == 0) { e[1] = x[0]; e[2] = x[1]; e[5] = x[2]; } else { e[0] = x[0]; e[3] = x[1]; e[4] = x[2]; }
}

// parity entry: raw residual / Jacobian per scan point at st->x
__global__ void __launch_bounds__(ITPB) icp_eval_kernel(IcpDev d, double* __restrict__ r_out, double* __restrict__ J_out) {
    __shared__ IcpFrame s_f;
    if (threadIdx.x == 0) { double e[6]; icp_substitute(*d.st, d.st->x, e); s_f = icp_frame(d.st->mode, d.st->Twc1, e); }
    __syncthreads();
    const int i = blockIdx.x * ITPB + threadIdx.x;
    if (i >= d.K) return;
    double r = 0.0, J[3] = {0, 0, 0};
    if (d.accepted[i]) {
        const float3 p = load_xyz(d.scan, i, d.stride);
        r = icp_point(s_f, v3(p.x, p.y, p.z), v3(d.pa[i], d.pa[d.K + i], d.pa[2 * d.K + i]),
                      v3(d.nrm[i], d.nrm[d.K + i], d.nrm[2 * (size_t)d.K + i]), d.st->weight, J);
    }
    r_out[i] = r; J_out[3 * i] = J[0]; J_out[3 * i + 1] = J[1]; J_out[3 * i + 2] = J[2];
}

// K9: residual / Jacobian per accepted point, Huber corrector, block reduce of J^T J (3x3), J^T r, cost.
// MODE 0: at x (skipped unless need_linearize) ; MODE 1: cost at the candidate only.
template <int MODE>
__global__ void __launch_bounds__(ITPB) icp_linearize_kernel(IcpDev d) {
    __shared__ IcpFrame s_f;
    __shared__ double s_red[ITPB / 32][12];
    IcpState* st = d.st;
    if (st->lm.done) return;
    if (MODE == 0 && !st->lm.need_linearize) return;
    if (threadIdx.x == 0) { double e[6]; icp_substitute(*st, MODE == 0 ? st->x : st->cand, e); s_f = icp_frame(st->mode, st->Twc1, e); }
    __syncthreads();
    double a[11];
    for (int k = 0; k < 11; ++k) a[k] = 0.0;     // H00 H10 H11 H20 H21 H22 g0 g1 g2 cost count
    for (int i = blockIdx.x * ITPB + threadIdx.x; i < d.K; i += gridDim.x * ITPB) {
        if (!d.accepted[i]) continue;
        const float3 p = load_xyz(d.scan, i, d.stride);
        double J[3];
        double r = icp_point(s_f, v3(p.x, p.y, p.z), v3(d.pa[i], d.pa[d.K + i], d.pa[2 * d.K + i]),
                             v3(d.nrm[i], d.nrm[d.K + i], d.nrm[2 * (size_t)d.K + i]), st->weight, MODE == 0 ? J : nullptr);
        double rho_v, sr;
        huber(st->huber_a, r * r, &rho_v, &sr);
        a[9] += 0.5 * rho_v; a[10] += 1.0;
        if (MODE == 0) {
            r *= sr; J[0] *= sr; J[1] *= sr; J[2] *= sr;
            a[0] += J[0] * J[0]; a[1] += J[1] * J[0]; a[2] += J[1] * J[1]; a[3] += J[2] * J[0]; a[4] += J[2] * J[1]; a[5] += J[2] * J[2];
            a[6] += J[0] * r; a[7] += J[1] * r; a[8] += J[2] * r;
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = 0; k < 11; ++k) { double v = a[k]; for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o); if (lane == 0) s_red[warp][k] = v; }
    __syncthreads();
    if (threadIdx.x < 11) {
        double v = 0.0; for (int w = 0; w < ITPB / 32; ++w) v += s_red[w][threadIdx.x];
        if (MODE == 0) {
            static const int map[11] = {0, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13};
            if (v != 0.0) atomicAdd(&st->part[map[threadIdx.x]], v);
        } else if (threadIdx.x == 9 && v != 0.0) atomicAdd(&st->part[14], v);
    }
}

// one thread: prior, Jacobi scale, damping, gradient check, 3x3 Cholesky, candidate, model cost change
__global__ void icp_solve_kernel(IcpState* st) {
    LmState& s = st->lm;
    if (s.done) return;
    double* H = st->acc;   // 0 1 2 / 3 4 5 / 6 7 8 row-major (lower filled), g 9..11, cost 12, count 13, cand cost 14
    if (s.need_linearize) {
        for (int k = 0; k < 14; ++k) H[k] = st->part[k];
        H[1] = H[3]; H[2] = H[6]; H[5] = H[7];
        if (st->prior_w >= 0.0) {
            // PoseErrorRPZ (pose_error.hpp:147-154, residual order roll pitch z) / PoseErrorYXY (:176-183):
            // both are weight * (x_k - target_k) up to a row permutation, so J^T J = w^2 I, J^T r = w^2 (x - t)
            const double w2 = st->prior_w * st->prior_w;
            for (int k = 0; k < 3; ++k) { const double e = st->x[k] - st->prior_target[k]; H[4 * k] += w2; H[9 + k] += w2 * e; H[12] += 0.5 * w2 * e * e; }
        }
        s.cost_acc = H[12];
        s.n_accepted = (int)(H[13] + 0.5);
        double gm = 0.0;
        for (int k = 0; k < 3; ++k) { st->grad[k] = H[9 + k]; const double g = fabs(H[9 + k]); gm = (g == g) ? fmax(gm, g) : INFINITY; }
        s.grad_max_bits = (unsigned long long)__double_as_longlong(gm);
        if (!s.scale_valid) for (int k = 0; k < 3; ++k) st->scale[k] = s.jacobi ? 1.0 / (1.0 + sqrt(H[4 * k])) : 1.0;
    }
    for (int k = 0; k < 15; ++k) st->part[k] = 0.0;
    lm_control_pre(s);
    if (s.done) return;
    double A[9];
    for (int k = 0; k < 9; ++k) A[k] = H[k];
    for (int k = 0; k < 3; ++k) {
        const double s2 = st->scale[k] * st->scale[k];
        st->lam[k] = fmin(fmax(s2 * H[4 * k], s.min_diag), s.max_diag) / (s.radius * s2);
        A[4 * k] += st->lam[k];
    }
    // Cholesky 3x3
    double L[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    bool ok = true;
    for (int j = 0; j < 3 && ok; ++j) {
        double dgn = A[4 * j]; for (int k = 0; k < j; ++k) dgn -= L[3 * j + k] * L[3 * j + k];
        if (!(dgn > 0.0)) { ok = false; break; }
        L[4 * j] = sqrt(dgn);
        for (int i = j + 1; i < 3; ++i) { double v = A[3 * i + j]; for (int k = 0; k < j; ++k) v -= L[3 * i + k] * L[3 * j + k]; L[3 * i + j] = v / L[4 * j]; }
    }
    double y[3], dx[3] = {0, 0, 0};
    if (ok) {
        for (int i = 0; i < 3; ++i) { double v = -st->grad[i]; for (int k = 0; k < i; ++k) v -= L[3 * i + k] * y[k]; y[i] = v / L[4 * i]; }
        for (int i = 2; i >= 0; --i) { double v = y[i]; for (int k = i + 1; k < 3; ++k) v -= L[3 * k + i] * dx[k]; dx[i] = v / L[4 * i]; }
    } else s.solve_fail = 1;
    double xn = 0, sn = 0, ma = 0, mb = 0;
    for (int k = 0; k < 3; ++k) {
        st->delta[k] = dx[k]; st->cand[k] = st->x[k] + dx[k];
        xn += st->x[k] * st->x[k]; sn += dx[k] * dx[k]; ma += dx[k] * st->lam[k] * dx[k]; mb += st->grad[k] * dx[k];
    }
    s.x_norm2 = xn; s.step_norm2 = sn; s.mcc_a = ma; s.mcc_b = mb;
}

__global__ void icp_post_kernel(IcpState* st) {
    LmState& s = st->lm;
    if (s.done) return;
    double cand = st->part[14];
    st->part[14] = 0.0;
    if (st->prior_w >= 0.0) { const double w2 = st->prior_w * st->prior_w; for (int k = 0; k < 3; ++k) { const double e = st->cand[k] - st->prior_target[k]; cand += 0.5 * w2 * e * e; } }
    s.cand_cost_acc = cand;
    lm_control_post(s);
    if (s.accept) {
        s.x_cost = cand;
        for (int k = 0; k < 3; ++k) st->x[k] = st->cand[k];
    }
}

// ---- Mapping::Optimize for one keyframe on the device (lvb_icp_map_optimize_keyframe, lvb_icp_map_build_optimize_keyframe): the
// pose arithmetic between the two registrations.  FP64 on one thread; every product and sum is rounded on its own (__dmul_rn /
// __dadd_rn / __dsub_rn: no FMA contraction), in the operation order of the host formulas cited at each function.  Poses are
// [qx qy qz qw tx ty tz].
struct KfBlock {             // the call's device state, uploaded and read back with one copy each
    IcpState st[2];          // [0] ground (mode 0), [1] surf (mode 1)
    double map_pose[7];      // map_frame->pose                                   (uploaded)
    double pose[7];          // frame->pose: the incoming one, then after each registration
    double rpyxyz[6];
    float tf[8];             // pose.cast<float>(): the query transform of the next association, then of ToWorld
    MapDesc map[2];          // [0] ground, [1] surf map frame: the handles' (uploaded), or built in the call; P = 0: no registration
    int out_bbox[2][6];      // bounding boxes of the two clouds ToWorld stores (lvb_icp_map_build_optimize_keyframe)
    // lvb_icp_map_relocate (Mapping::Relocate, mapping.cpp:251-300)
    double old_pose[7];      // last_frame->pose                                  (uploaded)
    double rel[7];           // relative_o_c: the caller's guess (uploaded), then old_pose^-1 * pose after the last round
    double score[2];         // score_ground, score_surf of the last round
};
struct KfSeed {              // what ScanToMapWith* put in each problem (association.cpp:270-384) and the solver options
    lvb_solve_options o;
    double weight[2], huber_a[2], prior_w;
};
__constant__ int c_free[2][3] = {{1, 2, 5}, {0, 3, 4}};     // rpyxyz entries a registration solves for: pitch roll z / yaw x y

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }

// Sophus::SO3 construction from a quaternion (so3.hpp): coeffs /= norm(), squared norm summed x, y, z, w
__device__ void kf_normalize(double* q) {
    const double n = __dsqrt_rn(da(da(da(dm(q[0], q[0]), dm(q[1], q[1])), dm(q[2], q[2])), dm(q[3], q[3])));
    for (int k = 0; k < 4; ++k) q[k] = __ddiv_rn(q[k], n);
}
// SO3 * point = Eigen QuaternionBase::_transformVector: uv = 2 (q.vec x p); p + w uv + q.vec x uv
__device__ void kf_rotate(const double* q, const double* p, double* out) {
    double uv[3] = {ds(dm(q[1], p[2]), dm(q[2], p[1])), ds(dm(q[2], p[0]), dm(q[0], p[2])), ds(dm(q[0], p[1]), dm(q[1], p[0]))};
    for (int k = 0; k < 3; ++k) uv[k] = da(uv[k], uv[k]);
    const double c[3] = {ds(dm(q[1], uv[2]), dm(q[2], uv[1])), ds(dm(q[2], uv[0]), dm(q[0], uv[2])), ds(dm(q[0], uv[1]), dm(q[1], uv[0]))};
    for (int k = 0; k < 3; ++k) out[k] = da(da(p[k], dm(q[3], uv[k])), c[k]);
}
// SE3 * SE3 (Sophus se3.hpp): q = qa qb (Eigen's quaternion product), renormalised by 2 / (1 + |q|^2) when |q|^2 != 1 (so3.hpp
// SO3Base::operator*); t = ta + qa tb
__device__ void kf_se3_mul(const double* a, const double* b, double* c) {
    const double aw = a[3], ax = a[0], ay = a[1], az = a[2], bw = b[3], bx = b[0], by = b[1], bz = b[2];
    double q[4];
    q[3] = ds(ds(ds(dm(aw, bw), dm(ax, bx)), dm(ay, by)), dm(az, bz));
    q[0] = ds(da(da(dm(aw, bx), dm(ax, bw)), dm(ay, bz)), dm(az, by));
    q[1] = ds(da(da(dm(aw, by), dm(ay, bw)), dm(az, bx)), dm(ax, bz));
    q[2] = ds(da(da(dm(aw, bz), dm(az, bw)), dm(ax, by)), dm(ay, bx));
    const double n2 = da(da(da(dm(q[0], q[0]), dm(q[1], q[1])), dm(q[2], q[2])), dm(q[3], q[3]));
    if (n2 != 1.0) { const double s = __ddiv_rn(2.0, da(1.0, n2)); for (int k = 0; k < 4; ++k) q[k] = dm(q[k], s); }
    double t[3];
    kf_rotate(a, b + 4, t);
    for (int k = 0; k < 4; ++k) c[k] = q[k];
    for (int k = 0; k < 3; ++k) c[4 + k] = da(a[4 + k], t[k]);
}
// SE3::inverse (se3.hpp): R^-1 = SO3(conjugate), t^-1 = R^-1 (-t)
__device__ void kf_se3_inv(const double* a, double* c) {
    c[0] = -a[0]; c[1] = -a[1]; c[2] = -a[2]; c[3] = a[3];
    kf_normalize(c);
    const double mt[3] = {-a[4], -a[5], -a[6]};
    kf_rotate(c, mt, c + 4);
}
// se32rpyxyz (utility.cpp:27-33): ceres::EigenQuaternionToRPY (ceres/base.hpp:95-108), then the translation
__device__ void kf_se32rpyxyz(const double* T, double* e) {
    const double q0 = T[3], q1 = T[0], q2 = T[1], q3 = T[2];
    e[0] = atan2(dm(2.0, da(dm(q1, q2), dm(q0, q3))), ds(1.0, dm(2.0, da(dm(q2, q2), dm(q3, q3)))));
    e[1] = asin(dm(2.0, ds(dm(q0, q2), dm(q1, q3))));
    e[2] = atan2(dm(2.0, da(dm(q2, q3), dm(q0, q1))), ds(1.0, dm(2.0, da(dm(q1, q1), dm(q2, q2)))));
    e[3] = T[4]; e[4] = T[5]; e[5] = T[6];
}
// rpyxyz2se3 (utility.cpp:35-40): ceres::RPYToEigenQuaternion (ceres/base.hpp:110-132), SE3d(Quaterniond(q), t) normalises q
__device__ void kf_rpyxyz2se3(const double* e, double* T) {
    const double z = __ddiv_rn(e[0], 2.0), y = __ddiv_rn(e[1], 2.0), x = __ddiv_rn(e[2], 2.0);
    const double cz = cos(z), sz = sin(z), cy = cos(y), sy = sin(y), cx = cos(x), sx = sin(x);
    T[3] = da(dm(dm(cz, cy), cx), dm(dm(sz, sy), sx));
    T[0] = ds(dm(dm(cz, cy), sx), dm(dm(sz, sy), cx));
    T[1] = da(dm(dm(cz, sy), cx), dm(dm(sz, cy), sx));
    T[2] = ds(dm(dm(sz, cy), cx), dm(dm(cz, sy), sx));
    kf_normalize(T);
    T[4] = e[3]; T[5] = e[4]; T[6] = e[5];
}

// One step of mapping.cpp:147-185 on one thread.
//   from < 0  : rpyxyz = se32rpyxyz(map_pose^-1 * pose)                                   (mapping.cpp:154)
//   from = m  : registration m is solved: its free scalars go back into rpyxyz, pose = map_pose * rpyxyz2se3(rpyxyz)  (:165, :177)
//   then      : tf = pose.cast<float>() (association.cpp:287, mapping.cpp:195), and with seed = m the IcpState of registration m
//               is set up from rpyxyz as lvb_icp_scan_to_map's init_state does on the host
__device__ __forceinline__ void kf_pose_update(KfBlock* b, int from) {
    if (from < 0) {
        double inv[7], rel[7];
        kf_se3_inv(b->map_pose, inv);
        kf_se3_mul(inv, b->pose, rel);
        kf_se32rpyxyz(rel, b->rpyxyz);
    } else {
        for (int k = 0; k < 3; ++k) b->rpyxyz[c_free[from][k]] = b->st[from].x[k];
        double rel[7];
        kf_rpyxyz2se3(b->rpyxyz, rel);
        kf_se3_mul(b->map_pose, rel, b->pose);
    }
}
__device__ __forceinline__ void kf_seed(KfBlock* b, int seed, const KfSeed& p) {
    IcpState& s = b->st[seed];
    memset(&s, 0, sizeof(s));
    lm_init(s.lm, p.o);
    s.mode = seed;
    for (int k = 0; k < 7; ++k) s.Twc1[k] = b->map_pose[k];
    for (int k = 0; k < 6; ++k) s.rpyxyz[k] = b->rpyxyz[k];
    for (int k = 0; k < 3; ++k) { s.x[k] = b->rpyxyz[c_free[seed][k]]; s.cand[k] = s.x[k]; s.prior_target[k] = s.x[k]; }
    s.prior_w = p.prior_w; s.huber_a = p.huber_a[seed]; s.weight = p.weight[seed];
}
// lvb_icp_map_optimize_keyframes: what ties keyframe k of the call to the earlier ones.  The blocks and links of a call lie in two
// arrays, link k beside block k.
struct KfLink {
    double T[7];                 // new_k * old_k^-1 (mapping.cpp:181-182), rewritten by every pose kernel of keyframe k
    double old[7];               // old_k: the incoming pose after the earlier keyframes' ForwardUpdates
    MapDesc kept[2];             // the map frame the keyframe's build slot holds after icp_map_keep_kernel
    int k;                       // the keyframe's index in the call
    int map_from;                // the keyframe of the call whose optimised pose is the map pose (the newest map key), or -1
};
// Before keyframe k's registrations: PoseGraph::ForwardUpdate(T_j, t_j + epsilon) of every earlier keyframe j, in order
// (pose_graph.cpp:245-252: pose = T_j * pose), and the map pose of an in-call newest map key
__device__ void kf_chain_in(KfBlock* b, KfLink* l) {
    const KfLink* l0 = l - l->k;
    for (int j = 0; j < l->k; ++j) {
        double t[7];
        kf_se3_mul(l0[j].T, b->pose, t);
        for (int i = 0; i < 7; ++i) b->pose[i] = t[i];
    }
    if (l->map_from >= 0) { const KfBlock* src = b - (l->k - l->map_from); for (int i = 0; i < 7; ++i) b->map_pose[i] = src->pose[i]; }
    for (int i = 0; i < 7; ++i) l->old[i] = b->pose[i];
}

// A registration whose map frame is empty (map[m].P == 0: SegmentGround kept no point in the in-call build) is not solved -- its LM
// passes return at once -- and leaves rpyxyz and the pose as they were, as BuildMapFrame's failure on that side does in the
// step-by-step path.  link (lvb_icp_map_optimize_keyframes only): the incoming pose is chained before the first step, and the
// keyframe's transform is formed after each.
__global__ void icp_kf_pose_kernel(KfBlock* b, int from, int seed, KfSeed p, KfLink* link) {
    if (link && from < 0) kf_chain_in(b, link);
    if (from < 0 || b->map[from].P > 0) kf_pose_update(b, from);
    for (int k = 0; k < 7; ++k) b->tf[k] = __double2float_rn(b->pose[k]);
    if (link) { double inv[7]; kf_se3_inv(link->old, inv); kf_se3_mul(b->pose, inv, link->T); }
    if (seed < 0) return;
    kf_seed(b, seed, p);
    if (b->map[seed].P == 0) b->st[seed].lm.done = 1;
}

// Mapping::Relocate's pose arithmetic around its rounds, on one thread with the rounding rules above:
//   stage 0: clone pose = old_pose * relative_o_c (mapping.cpp:256)
//   stage 1: relative_o_c = old_pose^-1 * pose (:298), and the scores of the last round (:281-282, :294-295):
//            min(n / 10, cap) - 2 final_cost / n with n = num_residual_blocks_reduced (no prior: the accepted points), cap 20 for
//            the ground registration and 30 for the surf one; NaN for a registration that did not run and for n = 0
__global__ void icp_reloc_pose_kernel(KfBlock* b, int stage) {
    if (stage == 0) { kf_se3_mul(b->old_pose, b->rel, b->pose); return; }
    double inv[7];
    kf_se3_inv(b->old_pose, inv);
    kf_se3_mul(inv, b->pose, b->rel);
    for (int m = 0; m < 2; ++m) {
        const double n = (double)b->st[m].lm.n_accepted;
        b->score[m] = b->map[m].P > 0 && n > 0.0
                          ? ds(fmin(__ddiv_rn(n, 10.0), m ? 30.0 : 20.0), __ddiv_rn(dm(2.0, b->st[m].lm.x_cost), n))
                          : __longlong_as_double(0x7ff8000000000000LL);
    }
}

// lvb_icp_map_optimize_keyframes builds the map frames of one side into two slots in turn.  After a build into `dst` whose map frame
// came out empty (SegmentGround kept no point, or it failed), the slot takes over the previous build's map frame from `src` (whose
// descriptor is *prev), so that every slot holds the newest map frame with points: the one the step-by-step loop leaves the handle
// with, as a failed lvb_icp_map_build keeps the map frame before it.  *kept: the descriptor of what dst holds afterwards.
__global__ void icp_map_keep_kernel(const MapDesc* built, const MapDesc* prev, MapDesc* kept, const float4* src_sorted, const int* src_start,
                                    const int* src_coarse, float4* dst_sorted, int* dst_start, int* dst_coarse) {
    const bool take = built->P == 0 && prev->P > 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) *kept = take ? *prev : *built;
    if (!take) return;
    const int P = prev->P, nc = prev->ncell + 1, nb = prev->ncb;
    const int t0 = blockIdx.x * blockDim.x + threadIdx.x, step = gridDim.x * blockDim.x;
    for (int i = t0; i < P; i += step) dst_sorted[i] = src_sorted[i];
    for (int i = t0; i < nc; i += step) dst_start[i] = src_start[i];
    for (int i = t0; i < nb; i += step) dst_coarse[i] = src_coarse[i];
}

}  // namespace

// ====================================================================================== host side
// A resident cloud buffer, held by the store's table and by the calls that read it.  It is freed with cudaFreeAsync on the stream of
// the call that drops the last reference (lvb::g_alloc_stream), not on the allocating handle's, whose context may be gone by then:
// every holder drops its reference after its own synchronisation, or behind its own queued reads of the buffer.
using Cloud = std::shared_ptr<DevBuf<float4>>;
static Cloud new_cloud() {
    return Cloud(new DevBuf<float4>(), [](DevBuf<float4>* b) { b->s = lvb::g_alloc_stream; delete b; });
}
struct IcpStore;

struct lvb_icp {
    lvb_ctx* ctx = nullptr;
    bool have_map = false;
    float cell_size = 0;
    MapDesc map;                 // the current map frame's descriptor, as read back after its build
    // What the kernels of a set_map / lvb_icp_map_build build, and of a knn3 / eval / scan_to_map call, read on the device: the
    // descriptor (the build's working copy, then `map` uploaded with each call's scan) and the query transform
    struct Frame { MapDesc map; float tf[8]; };
    DevBuf<Frame> frame;
    DevBuf<unsigned char> map_raw, scan_raw, accepted;
    DevBuf<float4> map_sorted;
    DevBuf<int> cell_of, counts, cell_start, fill, block_sums, total, coarse;
    DevBuf<float> pa;
    DevBuf<double> nrm, eval_r, eval_J;
    DevBuf<int> knn_idx;
    DevBuf<float> knn_d2;
    DevBuf<IcpState> st;
    DevBuf<int> q_key, q_counts, q_start, q_fill, q_sums, q_total, q_order;
    // device-resident world clouds per keyframe (Mapping::pointclouds_surf / _ground, mapping.cpp:208-219) and the merged map frame
    // robot: the same records in the robot frame (x, y, z, intensity), kept so that lvb_icp_map_to_world can re-anchor the cloud
    // lo / hi: the cloud's bounding box (icp_bbox_kernel's), recorded by the calls that build map frames (kf_chain) and by
    // lvb_icp_map_to_world for the clouds they write, and computed by the former once for the others (has_bbox false)
    // They live in the handle's store (IcpStore), which lvb_icp_share hands to other handles.
    struct Segment {
        long long key; Cloud pts, robot; int n; bool has_bbox = false; float lo[3], hi[3];
        void release() { pts.reset(); robot.reset(); }
    };
    std::shared_ptr<IcpStore> store;
    DevBuf<float4> merged, merged2;
    struct MapBufs { DevBuf<float4> sorted; DevBuf<int> cell_start, coarse; };      // a map frame's sorted cloud and voxel hash
    MapBufs nx;          // every build writes its map frame here; it is swapped in only when the build succeeded
    MapBufs reloc;       // lvb_icp_map_relocate's old map frame: reused by every relocation, never swapped in
    MapBufs chain;       // lvb_icp_map_optimize_keyframes builds its map frames into nx and this slot in turn
    int scan_n = 0, scan_stride = 0;          // the scan of the last upload_scan (reusable by lvb_icp_map_append)
    const unsigned char* scan_dev = nullptr;  // where that scan lies: scan_raw, this handle's part of kf_arena, or scan_cloud
    Cloud scan_cloud;                         // the stored robot-frame cloud of a by-key keyframe when the scan is that cloud
    // the keyframe calls' upload (kf_upload: blocks, links, scans) in one allocation, held by both handles of the call
    // so that either one's scan stays valid for lvb_icp_map_append(NULL) until that handle uploads another scan
    std::shared_ptr<DevBuf<unsigned char>> kf_arena;
    // lvb_icp_map_extract_keyframe's robot-frame feature cloud of a keyframe not yet stored (pending features): packed (x, y, z,
    // intensity) records and their bounding box.  The keyframe calls register it by key and store it as the keyframe's robot cloud.
    struct Pending { long long key; Cloud pts; int n; float lo[3], hi[3]; };
    ~lvb_icp();
};

// The resident keyframe clouds and the pending features, shared by the handles lvb_icp_share makes from one lvb_icp_create.  `mu`
// guards the two tables and their metadata (references, counts, boxes) and is never held across device work or a synchronisation:
// a call that reads clouds copies the entries it needs (taking references to the buffers) and unlocks; a call that writes publishes
// its entries after its synchronisation, so that a reader only ever sees clouds whose device writes are complete.
struct IcpStore {
    std::mutex mu;
    std::vector<lvb_icp::Segment> segments;
    std::vector<lvb_icp::Pending> pending;
    int handles = 0;                 // the handles on this store
    // lvb_icp_map_to_world overwrites the world clouds of an unshared store in place; lvb_icp_share waits until it has committed
    // (`cv`), so that no handle can read a cloud while it is being overwritten
    bool in_place = false;
    std::condition_variable cv;
};
lvb_icp::~lvb_icp() {
    if (!store) return;
    std::lock_guard<std::mutex> lk(store->mu);
    --store->handles;
}

// The store mutexes of a call's handles (either may be NULL; two handles on one store lock it once), taken together
struct StoreLock {
    std::unique_lock<std::mutex> a, b;
    StoreLock(const lvb_icp* g, const lvb_icp* s) {
        IcpStore* x = g ? g->store.get() : nullptr;
        IcpStore* y = s ? s->store.get() : nullptr;
        if (x == y || !x) { x = x ? x : y; y = nullptr; }
        if (x && y) {
            a = std::unique_lock<std::mutex>(x->mu, std::defer_lock); b = std::unique_lock<std::mutex>(y->mu, std::defer_lock);
            std::lock(a, b);
        } else if (x) a = std::unique_lock<std::mutex>(x->mu);
    }
};
// the entry of `key` (the store's mutex held), or NULL
static lvb_icp::Segment* find_segment(IcpStore& st, long long key) {
    for (auto& sg : st.segments) if (sg.key == key) return &sg;
    return nullptr;
}

#define ILAUNCH(h, kernel, grid, block, ...)                                              \
    do { if ((grid) > 0) { kernel<<<(grid), (block), 0, (h)->ctx->stream>>>(__VA_ARGS__); (h)->ctx->launches++; lvb::timing_mark((h)->ctx->stream, #kernel); } } while (0)

static inline int inblk(size_t n, int per) { return (int)((n + per - 1) / per); }
static int icheck(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("kernel launch failed in %s: %s", what, cudaGetErrorString(e)); return LVB_ERR_CUDA; }
    return LVB_OK;
}
// exchange two buffers' ownership (DevBuf has no move operations)
template <class T> static void swap_buf(DevBuf<T>& a, DevBuf<T>& b) { std::swap(a.p, b.p); std::swap(a.n, b.n); std::swap(a.s, b.s); std::swap(a.view, b.view); }

static void bbox_seed(int* b) {       // icp_bbox_kernel's starting values: min = FLT_MAX, max = -FLT_MAX as ordered ints
    float big = FLT_MAX, small = -FLT_MAX; int bi, si; memcpy(&bi, &big, 4); memcpy(&si, &small, 4);
    const int so = si >= 0 ? si : si ^ 0x7fffffff;
    b[0] = b[1] = b[2] = bi; b[3] = b[4] = b[5] = so;
}
// a map frame's descriptor as uploaded before its build: P points (or 0 when an earlier kernel writes the count) and the box seeds
static MapDesc desc_seed(int P) {
    MapDesc m;
    memset(&m, 0, sizeof(m));
    m.P = P;
    bbox_seed(m.bbox);
    return m;
}
static const GridCap kGridLimits = {(double)MAX_CELLS, (double)INFINITY, 8.0e6};
// the failure icp_map_grid_kernel reported in a map frame's descriptor
static int grid_error(const MapDesc& m, const char* fn, const char* side) {
    if (m.err == 1) { set_error("%s: map cloud has no finite bounding box", fn); return LVB_ERR_INVALID; }
    if (m.err) { set_error("%s: voxel grid of the %smap frame exceeds %d cells; increase cell_size or crop the map", fn, side, (int)MAX_CELLS); return LVB_ERR_UNSUPPORTED; }
    return LVB_OK;
}

// The association buffers and the visiting order of the n queries at d_scan (device, stride bytes each), against the map frame whose
// descriptor lies at m and with the query transform at tf (both device); d.map, d.cell_start and d.coarse are the caller's.  The nc
// counters of the sort are cleared with cudaMemsetAsync when nc is the map frame's own count (exact), and by a kernel up to m->nc when
// nc only bounds it (a map frame built in the same call).
static int bind_scan(lvb_icp* h, const unsigned char* d_scan, int n, int stride, const MapDesc* m, const float* tf, float max_d2, double thr,
                     size_t nc, bool exact, IcpDev& d) {
    cudaStream_t s = h->ctx->stream;
    h->scan_n = n; h->scan_stride = stride; h->scan_dev = d_scan;
    LVB_TRY(h->accepted.ensure(std::max(1, n)));
    LVB_TRY(h->pa.ensure((size_t)std::max(1, n) * 3));
    LVB_TRY(h->nrm.ensure((size_t)std::max(1, n) * 3));
    LVB_TRY(h->st.ensure(1));
    d.m = m; d.tf = tf;
    d.scan = d_scan; d.K = n; d.stride = stride;
    d.max_d2 = max_d2; d.thr = thr;
    d.accepted = h->accepted.p; d.pa = h->pa.p; d.nrm = h->nrm.p; d.st = h->st.p;
    d.order = nullptr;
    if (n >= 4096) {       // spatial visiting order: counting sort of the queries by coarse voxel block
        const int nb = inblk(nc, 1024);
        LVB_TRY(h->q_key.ensure(n)); LVB_TRY(h->q_order.ensure(n)); LVB_TRY(h->q_counts.ensure(nc)); LVB_TRY(h->q_fill.ensure(nc));
        LVB_TRY(h->q_start.ensure(nc + 1)); LVB_TRY(h->q_sums.ensure(nb)); LVB_TRY(h->q_total.ensure(1));
        if (exact) {
            LVB_CUDA(cudaMemsetAsync(h->q_counts.p, 0, nc * sizeof(int), s));
            LVB_CUDA(cudaMemsetAsync(h->q_fill.p, 0, nc * sizeof(int), s));
        } else ILAUNCH(h, icp_zero_map_kernel, std::min(inblk(nc, 256), 8 * h->ctx->sm_count), 256, h->q_counts.p, h->q_fill.p, &m->nc);
        ILAUNCH(h, icp_query_key_kernel, inblk(n, 256), 256, d, h->q_key.p, h->q_counts.p);
        ILAUNCH(h, scan_block_map_kernel, nb, 1024, h->q_counts.p, h->q_start.p, &m->nc, h->q_sums.p);
        ILAUNCH(h, scan_sums_map_kernel, 1, 1024, h->q_sums.p, &m->nc, h->q_total.p);
        ILAUNCH(h, scan_add_map_kernel, nb, 1024, h->q_start.p, &m->nc, h->q_sums.p, h->q_total.p);
        ILAUNCH(h, icp_query_scatter_kernel, inblk(n, 256), 256, n, h->q_key.p, h->q_start.p, h->q_fill.p, h->q_order.p);
        d.order = h->q_order.p;
    }
    return LVB_OK;
}

// knn3 / eval / scan_to_map: the scan, the current map frame's descriptor and the frame pose cast to float go to the device on the
// context's stream
static int upload_scan(lvb_icp* h, const void* scan, int n, int stride, const double* frame_pose, float max_d2, double thr, IcpDev& d) {
    if (!h->have_map) { set_error("set_map first"); return LVB_ERR_STATE; }
    if (n < 0 || stride < 12 || (stride & 3) || (n && !scan)) { set_error("bad scan arguments"); return LVB_ERR_INVALID; }
    cudaStream_t s = h->ctx->stream;
    LVB_TRY(h->scan_raw.upload((const unsigned char*)scan, (size_t)n * stride, s));
    h->kf_arena.reset(); h->scan_cloud.reset();
    lvb_icp::Frame f;
    f.map = h->map;
    for (int i = 0; i < 7; ++i) f.tf[i] = (float)frame_pose[i];
    f.tf[7] = 0.0f;
    LVB_TRY(h->frame.upload(&f, 1, s));
    d.map = h->map_sorted.p; d.cell_start = h->cell_start.p; d.coarse = h->coarse.p;
    return bind_scan(h, h->scan_raw.p, n, stride, &h->frame.p->map, h->frame.p->tf, max_d2, thr, h->map.nc, true, d);
}

// one LM pass on d.st: linearise at x, solve, the cost at the candidate, accept or reject (the partial sums all-reduced over the ranks)
static int enqueue_pass(lvb_icp* h, const IcpDev& d) {
    lvb_ctx* ctx = h->ctx;
    const int lin_blocks = std::max(1, std::min(inblk(d.K, ITPB), 4 * ctx->sm_count));
    ILAUNCH(h, icp_linearize_kernel<0>, lin_blocks, ITPB, d);
    if (ctx->world > 1) LVB_TRY(comm_allreduce_sum_f64(ctx, d.st->part, 14));
    ILAUNCH(h, icp_solve_kernel, 1, 1, d.st);
    ILAUNCH(h, icp_linearize_kernel<1>, lin_blocks, ITPB, d);
    if (ctx->world > 1) LVB_TRY(comm_allreduce_sum_f64(ctx, d.st->part + 14, 1));
    ILAUNCH(h, icp_post_kernel, 1, 1, d.st);
    return LVB_OK;
}

// The counting sort by voxel key of the map frame at m (device; icp_map_grid_kernel has decided its grid): its m->P records (stride
// bytes each, at most n) at d_points into `out`.  The cells / coarse counters are cleared with cudaMemsetAsync when they are the map
// frame's own counts (exact), and by kernels up to m->ncell / m->ncb when they only bound them (map_bound).
static int enqueue_hash(lvb_icp* h, const unsigned char* d_points, int n, int stride, const MapDesc* m, size_t cells, size_t coarse, bool exact,
                        lvb_icp::MapBufs& out) {
    lvb_ctx* ctx = h->ctx;
    cudaStream_t s = ctx->stream;
    const int nb = inblk(cells, 1024);
    LVB_TRY(h->cell_of.ensure(n)); LVB_TRY(h->counts.ensure(cells)); LVB_TRY(h->fill.ensure(cells));
    LVB_TRY(out.cell_start.ensure(cells + 1)); LVB_TRY(out.sorted.ensure(n)); LVB_TRY(out.coarse.ensure(coarse));
    LVB_TRY(h->block_sums.ensure(nb)); LVB_TRY(h->total.ensure(1));
    if (exact) {
        LVB_CUDA(cudaMemsetAsync(h->counts.p, 0, cells * sizeof(int), s));
        LVB_CUDA(cudaMemsetAsync(h->fill.p, 0, cells * sizeof(int), s));
        LVB_CUDA(cudaMemsetAsync(out.coarse.p, 0, coarse * sizeof(int), s));
    } else {
        ILAUNCH(h, icp_zero_map_kernel, std::min(inblk(cells, 256), 8 * ctx->sm_count), 256, h->counts.p, h->fill.p, &m->ncell);
        ILAUNCH(h, icp_zero_map_kernel, std::min(inblk(coarse, 256), 8 * ctx->sm_count), 256, out.coarse.p, (int*)nullptr, &m->ncb);
    }
    ILAUNCH(h, icp_count_kernel, inblk(n, 256), 256, d_points, stride, m, h->cell_of.p, h->counts.p, out.coarse.p);
    ILAUNCH(h, scan_block_map_kernel, nb, 1024, h->counts.p, out.cell_start.p, &m->ncell, h->block_sums.p);
    ILAUNCH(h, scan_sums_map_kernel, 1, 1024, h->block_sums.p, &m->ncell, h->total.p);
    ILAUNCH(h, scan_add_map_kernel, nb, 1024, out.cell_start.p, &m->ncell, h->block_sums.p, h->total.p);
    ILAUNCH(h, icp_scatter_kernel, inblk(n, 256), 256, d_points, stride, m, h->cell_of.p, out.cell_start.p, h->fill.p, out.sorted.p);
    return icheck("map frame build");
}

// set_map / lvb_icp_map_build: upload the descriptor's seed, P points, before the build (P = 0 when SegmentGround writes the count)
static int seed_frame(lvb_icp* h, int P) {
    LVB_TRY(h->frame.ensure(1));
    const MapDesc seed = desc_seed(P);
    LVB_CUDA(cudaMemcpyAsync(&h->frame.p->map, &seed, sizeof(seed), cudaMemcpyHostToDevice, h->ctx->stream));
    return LVB_OK;
}

// Voxel hash of the map frame at d_points (device, stride bytes per record, at most n of them: the count lies in the seeded
// descriptor): bounding box and grid on the device, the descriptor read back (the one synchronisation before the sort), the
// counting sort sized by it, and the new map frame swapped in on success -- a failed build leaves the previous one in place.
static int build_map(lvb_icp* h, const unsigned char* d_points, int n, int stride, float cell_size, const char* fn, int* n_points) {
    lvb_ctx* ctx = h->ctx;
    cudaStream_t s = ctx->stream;
    MapDesc* md = &h->frame.p->map;
    ILAUNCH(h, icp_bbox_kernel, std::min(1024, inblk(n, 256)), 256, d_points, stride, md);
    ILAUNCH(h, icp_map_grid_kernel, 1, 1, md, cell_size, kGridLimits);
    LVB_TRY(icheck("map grid"));
    MapDesc m;
    LVB_CUDA(cudaMemcpyAsync(&m, md, sizeof(m), cudaMemcpyDeviceToHost, s));
    LVB_TRY(host_sync(ctx, s));
    if (m.P == 0 && !m.err) { set_error("%s: the ground plane fit kept no point", fn); return LVB_ERR_NUMERIC; }
    if (n_points) *n_points = m.P;
    LVB_TRY(grid_error(m, fn, ""));
    LVB_TRY(enqueue_hash(h, d_points, m.P, stride, md, m.ncell, m.ncb, true, h->nx));
    LVB_TRY(host_sync(ctx, s));
    swap_buf(h->map_sorted, h->nx.sorted); swap_buf(h->cell_start, h->nx.cell_start); swap_buf(h->coarse, h->nx.coarse);
    h->map = m; h->cell_size = cell_size; h->have_map = true;
    return LVB_OK;
}

// A cloud stored by a by-key keyframe call keeps the pending buffer as its robot-frame records, and the scan lvb_icp_map_append(NULL)
// refers to may be that buffer: it goes with the cloud when h drops it.  The table's references move into `drop`, which the caller
// releases after unlocking the store.
static void release_segment(lvb_icp* h, lvb_icp::Segment& sg, std::vector<lvb_icp::Segment>& drop) {
    if (sg.robot && h->scan_dev == reinterpret_cast<const unsigned char*>(sg.robot->p)) { h->scan_n = 0; h->scan_dev = nullptr; h->scan_cloud.reset(); }
    drop.push_back(sg);
    sg.release();
}
// the pending features of `key` (the store's mutex held), or NULL
static lvb_icp::Pending* find_pending(IcpStore& st, long long key) {
    for (auto& pd : st.pending) if (pd.key == key) return &pd;
    return nullptr;
}
// drop the pending features of `key` (key < 0: all) into `drop` (the store's mutex held)
static void drop_pending(IcpStore& st, long long key, std::vector<lvb_icp::Pending>& drop) {
    size_t w = 0;
    for (size_t i = 0; i < st.pending.size(); ++i) {
        if (key < 0 || st.pending[i].key == key) drop.push_back(st.pending[i]); else st.pending[w++] = st.pending[i];
    }
    st.pending.resize(w);
}

extern "C" {

int lvb_icp_create(lvb_ctx* ctx, lvb_icp** out) {
    if (!ctx || !out) { set_error("null argument"); return LVB_ERR_INVALID; }
    lvb_icp* h = new lvb_icp();
    h->ctx = ctx;
    h->store = std::make_shared<IcpStore>();
    h->store->handles = 1;
    *out = h;
    return LVB_OK;
}

int lvb_icp_share(lvb_ctx* ctx, lvb_icp* owner, lvb_icp** out) {
    if (!ctx || !owner || !out) { set_error("lvb_icp_share: null argument"); return LVB_ERR_INVALID; }
    if (ctx->device != owner->ctx->device) {
        set_error("lvb_icp_share: the context is on device %d, the store on device %d", ctx->device, owner->ctx->device); return LVB_ERR_INVALID; }
    if (ctx->world > 1 || owner->ctx->world > 1) { set_error("lvb_icp_share: sharded contexts keep their stores per rank"); return LVB_ERR_UNSUPPORTED; }
    lvb_icp* h = new lvb_icp();
    h->ctx = ctx;
    h->store = owner->store;
    {
        std::unique_lock<std::mutex> lk(h->store->mu);
        h->store->cv.wait(lk, [&] { return !h->store->in_place; });
        ++h->store->handles;
    }
    *out = h;
    return LVB_OK;
}
// The store outlives the handle while another handle holds it; what this handle drops is freed on its context's stream.
void lvb_icp_destroy(lvb_icp* icp) {
    if (!icp) return;
    cudaSetDevice(icp->ctx->device);
    const cudaStream_t prev = lvb::g_alloc_stream;
    lvb::g_alloc_stream = icp->ctx->stream;
    delete icp;
    lvb::g_alloc_stream = prev;
}

int lvb_icp_set_map(lvb_icp* h, const void* points, int n, int stride, float cell_size) {
    if (n <= 0 || !points || stride < 12 || (stride & 3) || !(cell_size > 0.0f)) { set_error("bad map arguments"); return LVB_ERR_INVALID; }
    lvb_ctx* ctx = h->ctx;
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    LVB_TRY(h->map_raw.upload((const unsigned char*)points, (size_t)n * stride, ctx->stream));
    LVB_TRY(seed_frame(h, n));
    return build_map(h, h->map_raw.p, n, stride, cell_size, "lvb_icp_set_map", nullptr);
}

// ---- device-resident map (SURVEY 8(f).2): the per-keyframe world clouds stay in HBM, the map frame is merged and hashed there
int lvb_icp_map_append(lvb_icp* h, long long key, const void* robot_points, int n, int stride, const double pose[7]) {
    if (!h || !pose) { set_error("null argument"); return LVB_ERR_INVALID; }
    lvb_ctx* ctx = h->ctx;
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    cudaStream_t s = ctx->stream;
    const unsigned char* src = nullptr;
    DevBuf<unsigned char> up;
    if (robot_points) {
        if (n < 0 || stride < 12 || (stride & 3)) { set_error("bad cloud arguments"); return LVB_ERR_INVALID; }
        LVB_TRY(up.upload((const unsigned char*)robot_points, (size_t)n * stride, s));
        src = up.p;
    } else {      // the scan the last scan_to_map / knn3 / eval call uploaded: Mapping::Optimize followed by ToWorld of the same frame
        if (h->scan_n <= 0) { set_error("lvb_icp_map_append: no scan on the device"); return LVB_ERR_STATE; }
        n = h->scan_n; stride = h->scan_stride; src = h->scan_dev;
    }
    {
        std::lock_guard<std::mutex> lk(h->store->mu);
        if (find_segment(*h->store, key)) { set_error("lvb_icp_map_append: key %lld exists", key); return LVB_ERR_INVALID; }
    }
    lvb_icp::Segment sg; sg.key = key; sg.n = n; sg.pts = new_cloud(); sg.robot = new_cloud();
    int rc = sg.pts->ensure(std::max(1, n));
    if (rc == LVB_OK) rc = sg.robot->ensure(std::max(1, n));
    DevBuf<float> d_tf;
    float tf[7]; for (int i = 0; i < 7; ++i) tf[i] = (float)pose[i];      // Twc.cast<float>() (mapping.cpp:195)
    if (rc == LVB_OK) rc = d_tf.upload(tf, 7, s);
    if (rc != LVB_OK) { sg.release(); return rc; }
    ILAUNCH(h, icp_to_world_kernel, inblk(n, 256), 256, src, sg.pts->p, sg.robot->p, n, stride, d_tf.p, (int*)nullptr);
    rc = icheck("map_append");
    if (rc != LVB_OK) { sg.release(); return rc; }
    LVB_TRY(host_sync(h->ctx, s));
    std::lock_guard<std::mutex> lk(h->store->mu);
    h->store->segments.push_back(sg);
    return LVB_OK;
}

int lvb_icp_map_evict(lvb_icp* h, long long key) {
    if (!h) { set_error("null argument"); return LVB_ERR_INVALID; }
    LVB_CUDA(cudaSetDevice(h->ctx->device)); lvb::g_alloc_stream = h->ctx->stream;
    std::vector<lvb_icp::Segment> drop;           // released after the store is unlocked
    std::vector<lvb_icp::Pending> drop_pd;
    std::lock_guard<std::mutex> lk(h->store->mu);
    auto& segs = h->store->segments;
    size_t w = 0;
    for (size_t i = 0; i < segs.size(); ++i) {
        if (key < 0 || segs[i].key == key) release_segment(h, segs[i], drop); else segs[w++] = segs[i];
    }
    segs.resize(w);
    drop_pending(*h->store, key, drop_pd);
    return LVB_OK;
}

int lvb_icp_map_build(lvb_icp* h, const long long* keys, int n_keys, float cell_size, double ground_threshold, int* n_points) {
    if (!h || n_keys <= 0 || !keys || !(cell_size > 0.0f)) { set_error("bad arguments"); return LVB_ERR_INVALID; }
    lvb_ctx* ctx = h->ctx;
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    cudaStream_t s = ctx->stream;
    size_t total = 0;
    std::vector<lvb_icp::Segment> pick;           // the call's snapshot: references to the clouds it merges
    {
        std::lock_guard<std::mutex> lk(h->store->mu);
        for (int k = 0; k < n_keys; ++k) {
            const lvb_icp::Segment* f = find_segment(*h->store, keys[k]);
            if (!f) { set_error("lvb_icp_map_build: key %lld is not resident", keys[k]); return LVB_ERR_INVALID; }
            pick.push_back(*f); total += f->n;
        }
    }
    if (total == 0 || total > 0x7fffffffull) { set_error("lvb_icp_map_build: %zu points", total); return LVB_ERR_INVALID; }
    // points_*_merged += pointclouds_*[time] in key order (mapping.cpp:121-125): the position in the merged cloud is the point's index
    LVB_TRY(h->merged.ensure(total));
    size_t off = 0;
    for (auto& f : pick) { if (f.n) LVB_CUDA(cudaMemcpyAsync(h->merged.p + off, f.pts->p, (size_t)f.n * sizeof(float4), cudaMemcpyDeviceToDevice, s)); off += f.n; }
    const float4* cloud = h->merged.p;
    const int n = (int)total;
    const bool ransac = ground_threshold > 0.0;
    LVB_TRY(seed_frame(h, ransac ? 0 : n));
    if (ransac) {      // association_->SegmentGround(points_ground_merged) (mapping.cpp:126): the inlier count stays on the device
        LVB_TRY(h->merged2.ensure(total));
        LVB_TRY(lidar_segment_ground_device_async(ctx, h->merged.p, n, ground_threshold, h->merged2.p, &h->frame.p->map.P));
        lvb::g_alloc_stream = ctx->stream;
        cloud = h->merged2.p;
    }
    return build_map(h, reinterpret_cast<const unsigned char*>(cloud), n, 16, cell_size, "lvb_icp_map_build", n_points);
}

int lvb_icp_map_download(lvb_icp* h, float* xyzi, int capacity, int* n_out) {
    if (!h || !h->have_map) { set_error("no map"); return LVB_ERR_STATE; }
    LVB_CUDA(cudaSetDevice(h->ctx->device));
    const int P = h->map.P;
    if (n_out) *n_out = P;
    if (!xyzi) return LVB_OK;
    if (capacity < P) { set_error("capacity %d < %d map points", capacity, P); return LVB_ERR_INVALID; }
    // hand the cloud back in its original (merge) order: map_sorted carries the original index in .w
    std::vector<float4> tmp(P);
    LVB_CUDA(cudaMemcpyAsync(tmp.data(), h->map_sorted.p, (size_t)P * sizeof(float4), cudaMemcpyDeviceToHost, h->ctx->stream));
    LVB_TRY(host_sync(h->ctx, h->ctx->stream));
    for (int j = 0; j < P; ++j) { int i; memcpy(&i, &tmp[j].w, 4); if (i < 0 || i >= P) { set_error("corrupt index"); return LVB_ERR_NUMERIC; } xyzi[4 * (size_t)i] = tmp[j].x; xyzi[4 * (size_t)i + 1] = tmp[j].y; xyzi[4 * (size_t)i + 2] = tmp[j].z; xyzi[4 * (size_t)i + 3] = 0.0f; }
    return LVB_OK;
}

int lvb_icp_transform_cloud(lvb_icp* h, const void* points, int n, int stride, const double pose[7], void* out) {
    if (n < 0 || stride < 12 || (stride & 3) || (n && (!points || !out))) { set_error("bad cloud arguments"); return LVB_ERR_INVALID; }
    if (n == 0) return LVB_OK;
    LVB_CUDA(cudaSetDevice(h->ctx->device)); lvb::g_alloc_stream = h->ctx->stream;
    cudaStream_t s = h->ctx->stream;
    DevBuf<unsigned char> d_in, d_out; DevBuf<float> d_tf;
    float tf[7]; for (int i = 0; i < 7; ++i) tf[i] = (float)pose[i];      // Twc.cast<float>()
    LVB_TRY(d_in.upload((const unsigned char*)points, (size_t)n * stride, s)); LVB_TRY(d_out.ensure((size_t)n * stride)); LVB_TRY(d_tf.upload(tf, 7, s));
    ILAUNCH(h, icp_transform_cloud_kernel, inblk(n, 256), 256, d_in.p, d_out.p, n, stride, d_tf.p);
    LVB_TRY(icheck("transform_cloud"));
    LVB_TRY(d_out.download((unsigned char*)out, (size_t)n * stride, s));
    LVB_TRY(host_sync(h->ctx, s));
    return LVB_OK;
}

int lvb_icp_knn3(lvb_icp* h, const void* scan, int n, int stride, const double frame_pose[7], float max_d2, int32_t* idx, float* d2) {
    LVB_CUDA(cudaSetDevice(h->ctx->device)); lvb::g_alloc_stream = h->ctx->stream;
    if (h->have_map && max_d2 > h->cell_size * h->cell_size) { set_error("max_d2 %.6g exceeds cell_size^2 %.6g", max_d2, h->cell_size * h->cell_size); return LVB_ERR_INVALID; }
    IcpDev d;
    LVB_TRY(upload_scan(h, scan, n, stride, frame_pose, max_d2, 0.0, d));
    if (n == 0) return LVB_OK;
    LVB_TRY(h->knn_idx.ensure((size_t)n * 3)); LVB_TRY(h->knn_d2.ensure((size_t)n * 3));
    ILAUNCH(h, icp_knn_kernel, inblk(n, ITPB), ITPB, d, h->knn_idx.p, h->knn_d2.p);
    LVB_TRY(icheck("knn3"));
    LVB_TRY(h->knn_idx.download(idx, (size_t)n * 3, h->ctx->stream));
    LVB_TRY(h->knn_d2.download(d2, (size_t)n * 3, h->ctx->stream));
    LVB_TRY(host_sync(h->ctx, h->ctx->stream));
    return LVB_OK;
}

static int init_state(lvb_icp* h, int mode, const double* map_pose, const double* rpyxyz, double weight, double prior_w, double huber_a,
                      const lvb_solve_options* o) {
    lvb_solve_options opt;
    if (o) opt = *o; else lvb_default_options(&opt);
    IcpState hs;
    memset(&hs, 0, sizeof(hs));
    lm_init(hs.lm, opt);
    hs.mode = mode;
    memcpy(hs.Twc1, map_pose, sizeof(hs.Twc1)); memcpy(hs.rpyxyz, rpyxyz, sizeof(hs.rpyxyz));
    const int fr[2][3] = {{1, 2, 5}, {0, 3, 4}};
    for (int k = 0; k < 3; ++k) { hs.x[k] = rpyxyz[fr[mode][k]]; hs.cand[k] = hs.x[k]; hs.prior_target[k] = hs.x[k]; }
    hs.prior_w = prior_w; hs.huber_a = huber_a; hs.weight = weight;
    LVB_CUDA(cudaMemcpyAsync(h->st.p, &hs, sizeof(hs), cudaMemcpyHostToDevice, h->ctx->stream));
    LVB_TRY(host_sync(h->ctx, h->ctx->stream));
    return LVB_OK;
}

static void fill_summary(const IcpState& hs, double prior_weight, double seconds, lvb_solve_summary* summary) {
    const int nb = hs.lm.n_accepted + (prior_weight >= 0 ? 1 : 0);
    summary->initial_cost = hs.lm.initial_cost; summary->final_cost = hs.lm.x_cost;
    summary->num_iterations = hs.lm.iter; summary->num_successful_steps = hs.lm.num_successful;
    summary->termination_type = hs.lm.termination; summary->num_residual_blocks = nb; summary->num_residual_blocks_reduced = nb;
    summary->final_radius = hs.lm.radius;
    summary->total_time_in_seconds = seconds;
}

int lvb_icp_eval(lvb_icp* h, int mode, const void* scan, int n, int stride, const double frame_pose[7], const double map_pose[7],
                 const double rpyxyz[6], double weight, double dist_thr, uint8_t* accepted, double* r, double* J) {
    if (mode < 0 || mode > 1) { set_error("bad mode"); return LVB_ERR_INVALID; }
    LVB_CUDA(cudaSetDevice(h->ctx->device)); lvb::g_alloc_stream = h->ctx->stream;
    IcpDev d;
    LVB_TRY(upload_scan(h, scan, n, stride, frame_pose, h->cell_size * h->cell_size, dist_thr, d));
    if (n == 0) return LVB_OK;
    LVB_TRY(init_state(h, mode, map_pose, rpyxyz, weight, -1.0, 0.0, nullptr));
    LVB_TRY(h->eval_r.ensure(n)); LVB_TRY(h->eval_J.ensure((size_t)n * 3));
    ILAUNCH(h, icp_associate_kernel, inblk(n, ITPB), ITPB, d);
    ILAUNCH(h, icp_eval_kernel, inblk(n, ITPB), ITPB, d, h->eval_r.p, h->eval_J.p);
    LVB_TRY(icheck("icp_eval"));
    cudaStream_t s = h->ctx->stream;
    if (accepted) LVB_TRY(h->accepted.download(accepted, n, s));
    if (r) LVB_TRY(h->eval_r.download(r, n, s));
    if (J) LVB_TRY(h->eval_J.download(J, (size_t)n * 3, s));
    LVB_TRY(host_sync(h->ctx, s));
    return LVB_OK;
}

int lvb_icp_scan_to_map(lvb_icp* h, int mode, const void* scan, int n, int stride, const double frame_pose[7], const double map_pose[7],
                        double rpyxyz[6], double weight, double prior_weight, double huber_a, double dist_thr,
                        const lvb_solve_options* options, lvb_solve_summary* summary) {
    if (mode < 0 || mode > 1) { set_error("bad mode"); return LVB_ERR_INVALID; }
    LVB_CUDA(cudaSetDevice(h->ctx->device)); lvb::g_alloc_stream = h->ctx->stream;
    const auto t0 = std::chrono::steady_clock::now();
    lvb_solve_options opt;
    if (options) opt = *options; else lvb_default_options(&opt);
    IcpDev d;
    lvb::timing_mark(h->ctx->stream, "begin");
    LVB_TRY(upload_scan(h, scan, n, stride, frame_pose, h->cell_size * h->cell_size, dist_thr, d));
    if ((double)h->cell_size * h->cell_size * (1.0 + 1e-6) < dist_thr) {
        set_error("dist_thr %.6g exceeds the map's cell_size^2 %.6g", dist_thr, (double)h->cell_size * h->cell_size); return LVB_ERR_INVALID; }
    LVB_TRY(init_state(h, mode, map_pose, rpyxyz, weight, prior_weight, huber_a, &opt));
    cudaStream_t s = h->ctx->stream;
    lvb_ctx* ctx = h->ctx;
    ILAUNCH(h, icp_associate_kernel, inblk(n, ITPB), ITPB, d);
    IcpState hs;
    memset(&hs, 0, sizeof(hs));
    for (int pass = 0; pass <= opt.max_num_iterations; ++pass) {
        LVB_TRY(enqueue_pass(h, d));
        LVB_TRY(icheck("icp iteration"));
        LVB_CUDA(cudaMemcpyAsync(&hs, h->st.p, sizeof(hs), cudaMemcpyDeviceToHost, s));
        LVB_TRY(host_sync(h->ctx, s));
        LVB_TRY(comm_check(ctx));
        if (hs.lm.done) break;
        if (opt.max_solver_time_in_seconds < 1e8) {      // collective decision when the queries are sharded (see lvb_ba_solve)
            double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            LVB_TRY(comm_max_seconds(ctx, &el));
            if (el >= opt.max_solver_time_in_seconds) break;
        }
    }
    const int fr[2][3] = {{1, 2, 5}, {0, 3, 4}};
    for (int k = 0; k < 3; ++k) rpyxyz[fr[mode][k]] = hs.x[k];
    if (summary) fill_summary(hs, prior_weight, std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(), summary);
    return LVB_OK;
}

// ---- Mapping::Optimize on the device: lvb_icp_map_optimize_keyframe against the handles' map frames, and the calls that build them
// in the same call (lvb_icp_map_optimize_keyframes, lvb_icp_map_build_optimize_keyframe, lvb_icp_map_relocate)
struct KfUpload {                                     // one keyframe's part of its call's upload
    std::shared_ptr<DevBuf<unsigned char>> arena;     // [KfBlock x n | KfLink x n (lvb_icp_map_optimize_keyframes) | ground, surf scan of each]
    KfBlock* blk;                                     // its KfBlock (device)
    KfBlock* hb;                                      // its KfBlock in the pinned staging area: the upload, then the read-back
    size_t off[2];                                    // where its scans lie in the arena
    KfLink* link = nullptr;                           // its KfLink (device), with links
    KfLink* hl = nullptr;                             // its KfLink in the staging area
    const unsigned char* scan[2];                     // its scans (device): in the arena, or pending features (by_key)
    int stride[2];                                    // their record sizes
    bool by_key[2] = {false, false};
};

// One copy from the pinned staging area for n keyframes: the blocks (zero but for the out_bbox seeds and what fill(k, u[k]) writes
// into keyframe k's: poses, map descriptors), with `links` the links (zero but for fill's), and the scans pts[2 k + m] of ns[2 k + m]
// records -- except those with dev[2 k + m] (dev may be NULL), pending features already on the device, which are not copied.
// u[k]: keyframe k's views; back: the bytes of the blocks and links, which the read-back copies.  The staging area stays busy until
// the caller's read-back.
static int kf_upload(lvb_ctx* ctx, int n, bool links, const void* const* pts, const float4* const* dev, const int* ns, int stride,
                     std::vector<KfUpload>& u, size_t& back, const std::function<void(int, KfUpload&)>& fill) {
    auto on_device = [&](int e) { return dev && dev[e]; };
    const size_t blk_bytes = ((size_t)n * sizeof(KfBlock) + 255) & ~(size_t)255;
    back = blk_bytes + (links ? (size_t)n * sizeof(KfLink) : 0);
    u.assign(n, KfUpload());
    size_t all = (back + 255) & ~(size_t)255;
    for (int k = 0; k < n; ++k)
        for (int m = 0; m < 2; ++m) { u[k].off[m] = all; all = (all + (on_device(2 * k + m) ? 0 : (size_t)ns[2 * k + m] * stride) + 255) & ~(size_t)255; }
    LVB_TRY(lvb::stage_wait(ctx));
    LVB_TRY(lvb::stage_grow(ctx, all, 0));
    KfBlock* hb = reinterpret_cast<KfBlock*>(ctx->stage_h);
    KfLink* hl = reinterpret_cast<KfLink*>(ctx->stage_h + blk_bytes);
    memset(hb, 0, (size_t)n * sizeof(KfBlock));
    if (links) memset(hl, 0, (size_t)n * sizeof(KfLink));
    for (int k = 0; k < n; ++k) {
        u[k].hb = hb + k;
        if (links) u[k].hl = hl + k;
        for (int m = 0; m < 2; ++m) {
            bbox_seed(hb[k].out_bbox[m]);
            const size_t bytes = on_device(2 * k + m) ? 0 : (size_t)ns[2 * k + m] * stride;
            if (bytes) memcpy(ctx->stage_h + u[k].off[m], pts[2 * k + m], bytes);
        }
        fill(k, u[k]);
    }
    auto arena = std::make_shared<DevBuf<unsigned char>>();
    LVB_TRY(arena->ensure(all));
    LVB_CUDA(cudaMemcpyAsync(arena->p, ctx->stage_h, all, cudaMemcpyHostToDevice, ctx->stream));
    LVB_TRY(lvb::stage_mark_busy(ctx, ctx->stream));
    for (int k = 0; k < n; ++k) {
        u[k].arena = arena;
        u[k].blk = reinterpret_cast<KfBlock*>(arena->p) + k;
        if (links) u[k].link = reinterpret_cast<KfLink*>(arena->p + blk_bytes) + k;
        for (int m = 0; m < 2; ++m) {
            const int e = 2 * k + m;
            u[k].by_key[m] = on_device(e);
            u[k].scan[m] = on_device(e) ? reinterpret_cast<const unsigned char*>(dev[e]) : arena->p + u[k].off[m];
            u[k].stride[m] = on_device(e) ? (int)sizeof(float4) : stride;
        }
    }
    return LVB_OK;
}

// What registration m reads of its map frame besides blk->map[m]: the sorted cloud and its hash, the cell size (the kNN radius) and
// the sort counters (nc, exact: see bind_scan).
struct KfMap { const float4* sorted; const int* cell_start; const int* coarse; float cell_size; size_t nc; bool exact; };

// Mapping::Optimize's loop body (mapping.cpp:147-177), and one round of Mapping::Relocate's (:264-296), for the registrations that
// run (run[m]): se32rpyxyz of the pose on the device, ScanToMapWithGround + Solve, the pose hand-off, ScanToMapWithSegmented + Solve,
// the pose hand-off.  Nothing waits for the host: each registration runs max_num_iterations + 1 LM passes (the kernels return at once
// after the solver stopped), and the pose kernels write the query transform the next association reads.
static int kf_register(lvb_icp* const hs[2], const bool run[2], const KfMap maps[2], const KfUpload& u, const int ns[2],
                       const lvb_map_optimize_params* p) {
    KfSeed seed;
    seed.o = p->options; seed.prior_w = p->prior_weight;
    for (int m = 0; m < 2; ++m) { seed.weight[m] = p->weight[m]; seed.huber_a[m] = p->huber_a[m]; }
    const int first = run[0] ? 0 : (run[1] ? 1 : -1);
    ILAUNCH(hs[0] ? hs[0] : hs[1], icp_kf_pose_kernel, 1, 1, u.blk, -1, first, seed, u.link);      // rpyxyz from the incoming pose (:154)
    for (int m = 0; m < 2; ++m) {
        if (!run[m]) continue;
        lvb_icp* h = hs[m];
        const KfMap& km = maps[m];
        IcpDev d;
        d.map = km.sorted; d.cell_start = km.cell_start; d.coarse = km.coarse;
        LVB_TRY(bind_scan(h, u.scan[m], ns[m], u.stride[m], &u.blk->map[m], u.blk->tf, km.cell_size * km.cell_size, p->dist_thr[m],
                          km.nc, km.exact, d));
        h->kf_arena = u.arena;
        d.st = &u.blk->st[m];
        ILAUNCH(h, icp_associate_kernel, inblk(ns[m], ITPB), ITPB, d);
        for (int pass = 0; pass <= p->options.max_num_iterations; ++pass) LVB_TRY(enqueue_pass(h, d));
        // pose = map_pose * rpyxyz2se3(rpyxyz) (:165, :177); after the ground solve it also seeds the surf registration
        ILAUNCH(h, icp_kf_pose_kernel, 1, 1, u.blk, m, m == 0 && run[1] ? 1 : -1, seed, u.link);
    }
    return LVB_OK;
}

// The end of Mapping::Optimize's loop body: ToWorld (:185, :205-220) of the scans of every handle given, transformed by the final
// pose.cast<float>(), into fresh[] with their robot-frame records (not yet stored; with `boxes`, their bounding boxes into
// blk->out_bbox).  A scan of pending features is its own robot-frame record: fresh[m].robot stays NULL until the caller commits.
static int kf_to_world(lvb_icp* const hs[2], const KfUpload& u, const int ns[2], bool boxes, lvb_icp::Segment fresh[2]) {
    for (int m = 0; m < 2; ++m) {
        if (!hs[m]) continue;
        fresh[m].key = -1; fresh[m].n = ns[m]; fresh[m].pts = new_cloud(); fresh[m].robot = u.by_key[m] ? nullptr : new_cloud();
        int rc = fresh[m].pts->ensure(std::max(1, ns[m]));
        if (rc == LVB_OK && fresh[m].robot) rc = fresh[m].robot->ensure(std::max(1, ns[m]));
        if (rc != LVB_OK) { fresh[0].release(); fresh[1].release(); return rc; }
        ILAUNCH(hs[m], icp_to_world_kernel, inblk(ns[m], 256), 256, u.scan[m], fresh[m].pts->p, fresh[m].robot ? fresh[m].robot->p : nullptr, ns[m],
                u.stride[m], u.blk->tf, boxes ? u.blk->out_bbox[m] : nullptr);
    }
    return LVB_OK;
}

// replace the cloud under `key` with sg, or add it (the store's mutex held; the replaced references go to `drop`)
static void store_segment(lvb_icp* h, long long key, lvb_icp::Segment& sg, std::vector<lvb_icp::Segment>& drop) {
    sg.key = key;
    if (lvb_icp::Segment* old = find_segment(*h->store, key)) { release_segment(h, *old, drop); *old = sg; return; }
    h->store->segments.push_back(sg);
}

// Mapping::Optimize for one keyframe (mapping.cpp:147-185, after BuildMapFrame) against the map frames lvb_icp_map_build made, with
// one host synchronisation at the end to read the two solver states and the pose back in one copy.
int lvb_icp_map_optimize_keyframe(lvb_icp* ground, lvb_icp* surf, const double map_pose[7], long long key,
                                  const void* ground_pts, int n_ground, const void* surf_pts, int n_surf, int stride,
                                  const lvb_map_optimize_params* p, double pose[7], double rpyxyz[6], lvb_solve_summary summary[2]) {
    lvb_icp* hs[2] = {ground, surf};
    const void* pts[2] = {ground_pts, surf_pts};
    const int ns[2] = {n_ground, n_surf};
    if ((!ground && !surf) || ground == surf || !map_pose || !p || !pose || !rpyxyz) { set_error("null argument"); return LVB_ERR_INVALID; }
    lvb_icp* h0 = ground ? ground : surf;
    lvb_ctx* ctx = h0->ctx;
    if (ground && surf && ground->ctx != surf->ctx) { set_error("lvb_icp_map_optimize_keyframe: the two handles belong to different contexts"); return LVB_ERR_INVALID; }
    if (ctx->world > 1) { set_error("lvb_icp_map_optimize_keyframe: sharded contexts register through lvb_icp_scan_to_map"); return LVB_ERR_UNSUPPORTED; }
    const lvb_solve_options& opt = p->options;
    if (opt.max_solver_time_in_seconds < 1e8) { set_error("lvb_icp_map_optimize_keyframe: no time limit (Mapping::Optimize sets none)"); return LVB_ERR_INVALID; }
    if (opt.max_num_iterations < 0 || stride < 12 || (stride & 3)) { set_error("bad arguments"); return LVB_ERR_INVALID; }
    for (int m = 0; m < 2; ++m) {
        lvb_icp* h = hs[m];
        if (!h) continue;
        if (!h->have_map) { set_error("lvb_icp_map_optimize_keyframe: build the map frame first"); return LVB_ERR_STATE; }
        if (ns[m] < 0 || (ns[m] && !pts[m])) { set_error("bad scan arguments"); return LVB_ERR_INVALID; }
        if ((double)h->cell_size * h->cell_size * (1.0 + 1e-6) < p->dist_thr[m]) {
            set_error("dist_thr %.6g exceeds the map's cell_size^2 %.6g", p->dist_thr[m], (double)h->cell_size * h->cell_size); return LVB_ERR_INVALID; }
    }
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    const auto t0 = std::chrono::steady_clock::now();
    cudaStream_t s = ctx->stream;
    lvb::timing_mark(s, "begin");
    const bool run[2] = {ground != nullptr, surf != nullptr};
    const int up[2] = {ground ? n_ground : 0, surf ? n_surf : 0};          // the scans of the handles given
    KfMap maps[2];
    for (int m = 0; m < 2; ++m)
        if (hs[m]) maps[m] = {hs[m]->map_sorted.p, hs[m]->cell_start.p, hs[m]->coarse.p, hs[m]->cell_size, (size_t)hs[m]->map.nc, true};
    std::vector<KfUpload> uk;
    size_t back;
    LVB_TRY(kf_upload(ctx, 1, false, pts, nullptr, up, stride, uk, back, [&](int, KfUpload& v) {
        memcpy(v.hb->map_pose, map_pose, sizeof(v.hb->map_pose)); memcpy(v.hb->pose, pose, sizeof(v.hb->pose));
        for (int m = 0; m < 2; ++m) v.hb->map[m] = hs[m] ? hs[m]->map : desc_seed(0);          // P = 0: no registration on that side
    }));
    const KfUpload& u = uk[0];
    lvb_icp::Segment fresh[2];
    LVB_TRY(kf_register(hs, run, maps, u, ns, p));
    LVB_TRY(kf_to_world(hs, u, ns, false, fresh));
    int rc = icheck("map_optimize_keyframe");
    if (rc != LVB_OK) { fresh[0].release(); fresh[1].release(); return rc; }
    // the one read-back: both solver states, rpyxyz and the pose; the clouds are published once it has run
    LVB_CUDA(cudaMemcpyAsync(u.hb, u.blk, back, cudaMemcpyDeviceToHost, s));
    LVB_TRY(host_sync(ctx, s));
    ctx->stage_busy = false;
    {
        std::vector<lvb_icp::Segment> drop;
        StoreLock lk(ground, surf);
        for (int m = 0; m < 2; ++m) if (hs[m]) store_segment(hs[m], key, fresh[m], drop);
    }
    const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    memcpy(pose, u.hb->pose, sizeof(u.hb->pose)); memcpy(rpyxyz, u.hb->rpyxyz, sizeof(u.hb->rpyxyz));
    if (summary) {
        for (int m = 0; m < 2; ++m) {
            if (hs[m]) { fill_summary(u.hb->st[m], p->prior_weight, el, &summary[m]); continue; }
            memset(&summary[m], 0, sizeof(summary[m]));
            summary[m].termination_type = -1;          // registration skipped (mapping.cpp:155,167: empty map cloud)
        }
    }
    return LVB_OK;
}

// ---- Map frames built inside a call: Mapping::BuildMapFrame (lvb_icp_map_optimize_keyframes, lvb_icp_map_build_optimize_keyframe)
// and Mapping::BuildOldMapFrame (lvb_icp_map_relocate)
static void bbox_store(lvb_icp::Segment& sg, const int* b) {
    for (int a = 0; a < 3; ++a) { sg.lo[a] = ord2f(b[a]); sg.hi[a] = ord2f(b[3 + a]); }
    sg.has_bbox = true;
}

// Clouds stored by lvb_icp_map_append / lvb_icp_map_optimize_keyframe carry no bounding box: compute those of `segs` (a call's
// snapshot of clouds of any handle on h's context; segs[i] is an entry of stores[i]) once, all with one host synchronisation, and
// record them in the snapshot and in the stores, for the entries that still hold the same cloud.
static int fill_bboxes(lvb_icp* h, const std::vector<lvb_icp::Segment*>& segs, const std::vector<IcpStore*>& stores) {
    std::vector<lvb_icp::Segment*> todo;
    std::vector<IcpStore*> todo_st;
    for (size_t i = 0; i < segs.size(); ++i) if (!segs[i]->has_bbox) { todo.push_back(segs[i]); todo_st.push_back(stores[i]); }
    if (todo.empty()) return LVB_OK;
    lvb_ctx* ctx = h->ctx;
    cudaStream_t s = ctx->stream;
    const size_t bytes = todo.size() * sizeof(MapDesc);
    LVB_TRY(lvb::stage_wait(ctx));
    LVB_TRY(lvb::stage_grow(ctx, bytes, 0));
    MapDesc* hb = reinterpret_cast<MapDesc*>(ctx->stage_h);
    for (size_t i = 0; i < todo.size(); ++i) hb[i] = desc_seed(todo[i]->n);
    DevBuf<MapDesc> d;
    LVB_TRY(d.ensure(todo.size()));
    LVB_CUDA(cudaMemcpyAsync(d.p, hb, bytes, cudaMemcpyHostToDevice, s));
    for (size_t i = 0; i < todo.size(); ++i)
        ILAUNCH(h, icp_bbox_kernel, std::min(1024, inblk(todo[i]->n, 256)), 256, reinterpret_cast<const unsigned char*>(todo[i]->pts->p), 16, d.p + i);
    LVB_TRY(icheck("map frame bounding boxes"));
    LVB_CUDA(cudaMemcpyAsync(hb, d.p, bytes, cudaMemcpyDeviceToHost, s));
    LVB_TRY(host_sync(ctx, s));
    for (size_t i = 0; i < todo.size(); ++i) {
        bbox_store(*todo[i], hb[i].bbox);
        std::lock_guard<std::mutex> lk(todo_st[i]->mu);
        lvb_icp::Segment* e = find_segment(*todo_st[i], todo[i]->key);
        if (e && e->pts == todo[i]->pts) bbox_store(*e, hb[i].bbox);
    }
    return LVB_OK;
}

// Capacities of a map frame whose cloud lies inside the box lo..hi: icp_map_grid_kernel's ring-4 grid of the box (the voxel counts per
// axis only shrink with a smaller box or a coarser ring), capped at MAX_CELLS -- above it the device picks a coarser ring or fails.
// qcap: the most query-sort counters the grid kernel picks for a grid no larger than the box's at ring 4 (it bounds qsort)
struct MapBound { size_t cells, coarse, qsort, qcap; bool finite; };
static MapBound map_bound(const float* lo, const float* hi, float cell_size) {
    MapBound b;
    const float cell = cell_size * 1.0001f / 4.0f, inv = 1.0f / cell;
    double d[3];
    b.finite = true;
    for (int a = 0; a < 3; ++a) {
        const float w = hi[a] - lo[a];
        if (!(hi[a] >= lo[a]) || !std::isfinite(w)) { b.finite = false; d[a] = 0; } else d[a] = std::floor((double)w * inv) + 1;
    }
    const double cap = (double)MAX_CELLS;
    if (!b.finite) { b.cells = b.coarse = MAX_CELLS; b.qsort = b.qcap = 8000000; return b; }
    auto blocks = [&](int sh) { double v = 1; for (int a = 0; a < 3; ++a) v *= std::ceil(d[a] / (double)(1 << sh)); return v; };
    b.cells = (size_t)std::min(cap, d[0] * d[1] * d[2]);
    b.coarse = (size_t)std::min(cap, blocks(2));
    b.qsort = (size_t)std::min(8.0e6, blocks(1));          // the grid kernel keeps the sort grid at <= 8 M counters
    b.qcap = (size_t)std::min(8.0e6, (std::floor(d[0] / 2) + 1) * (std::floor(d[1] / 2) + 1) * (std::floor(d[2] / 2) + 1));
    return b;
}

// A map key's clouds: the ones keyframe kf of the call stores (kf >= 0), else the ones resident on both handles (seg: entries of the
// call's snapshot)
struct KfSrc { int kf; lvb_icp::Segment* seg[2]; };
// The resident clouds a call reads, per side: copies of the store entries (references to the clouds), taken under the stores' mutexes
// (StoreLock) and kept until the call's synchronisation.  Node-based: the entries do not move.
struct Snapshot { std::unordered_map<long long, lvb_icp::Segment> seg[2]; };
static bool find_resident(lvb_icp* const hs[2], Snapshot& snap, long long key, KfSrc& sr) {
    for (int m = 0; m < 2; ++m) {
        sr.seg[m] = nullptr;
        auto it = snap.seg[m].find(key);
        if (it == snap.seg[m].end()) {
            const lvb_icp::Segment* e = find_segment(*hs[m]->store, key);
            if (!e) continue;
            it = snap.seg[m].emplace(key, *e).first;
        }
        sr.seg[m] = &it->second;
    }
    return sr.seg[0] && sr.seg[1];
}

// One keyframe's map frame (BuildMapFrame, mapping.cpp:114-137; BuildOldMapFrame, :78-112) on both handles: the clouds in merge order,
// the merged sizes, which side is built (an empty merged cloud: BuildMapFrame fails on that side and nothing registers, :155,167), the
// descriptor seeds, the union lo..hi of the resident clouds' boxes and the capacity bounds of the builds.
// cap: the limits the grid kernel keeps to (kGridLimits when the bounds come from exact boxes)
struct KfPlan { std::vector<lvb_icp::Segment*> pick[2]; size_t total[2] = {0, 0}; bool build[2]; MapBound bound[2]; MapDesc seed[2];
                GridCap cap[2] = {kGridLimits, kGridLimits}; float lo[2][3], hi[2][3]; };

// A keyframe of kf_chain: lvb_map_keyframe with the map keys as a pointer and a count
struct KfRec {
    long long key; const long long* map_keys; int n_map_keys;
    const void* pts[2]; int n[2];                 // the robot-frame clouds: ground, surf
    lvb_icp::Pending pend[2];                     // by key: the pending features of `key` on each handle (a copy of the entry), else empty
    const double* map_pose;
    double pose[7];                               // in: frame->pose; out: optimised
    double weight[2], prior_weight;
    double transform[7], rpyxyz[6]; lvb_solve_summary summary[2]; int n_map_points[2];        // out
};

// The plans of the map frames of srcs[k], one per keyframe k.  The clouds keyframe j of the call stores (stage[2 j + m], of
// kfs[j].n[m] points) have no box yet: the bounds are those of the resident clouds, and the caller widens them by the estimates of the
// others (in_call_box).  The missing boxes of the resident clouds are computed with one synchronisation, after the checks that need none.
static int plan_frames(lvb_icp* const hs[2], const std::vector<std::vector<KfSrc>>& srcs, const KfRec* kfs, lvb_icp::Segment* stage,
                       const float cell_size[2], bool ransac, const char* fn, std::vector<KfPlan>& pl) {
    pl.assign(srcs.size(), KfPlan());
    std::vector<lvb_icp::Segment*> res;           // the resident clouds, each once, and their stores
    std::vector<IcpStore*> res_st;
    std::unordered_set<lvb_icp::Segment*> seen;
    for (size_t k = 0; k < srcs.size(); ++k) {
        KfPlan& q = pl[k];
        for (auto& sr : srcs[k]) {
            for (int m = 0; m < 2; ++m) {
                if (sr.kf >= 0) { q.pick[m].push_back(&stage[2 * (size_t)sr.kf + m]); q.total[m] += kfs[sr.kf].n[m]; continue; }
                q.pick[m].push_back(sr.seg[m]); q.total[m] += sr.seg[m]->n;
                if (seen.insert(sr.seg[m]).second) { res.push_back(sr.seg[m]); res_st.push_back(hs[m]->store.get()); }
            }
        }
        for (int m = 0; m < 2; ++m) {
            if (q.total[m] > 0x7fffffffull) { set_error("%s: map frame of more than 2^31 points", fn); return LVB_ERR_INVALID; }
            q.build[m] = q.total[m] > 0;
            q.seed[m] = desc_seed(q.build[m] && !(m == 0 && ransac) ? (int)q.total[m] : 0);      // the ground count comes from SegmentGround
        }
    }
    LVB_TRY(fill_bboxes(hs[0], res, res_st));
    for (size_t k = 0; k < srcs.size(); ++k) {
        KfPlan& q = pl[k];
        for (int m = 0; m < 2; ++m) {
            float* lo = q.lo[m]; float* hi = q.hi[m];
            for (int a = 0; a < 3; ++a) { lo[a] = FLT_MAX; hi[a] = -FLT_MAX; }
            bool resident = false;
            for (auto& sr : srcs[k]) {
                if (sr.kf >= 0) continue;
                for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], sr.seg[m]->lo[a]); hi[a] = std::max(hi[a], sr.seg[m]->hi[a]); }
                resident = true;
            }
            if (!q.build[m]) continue;
            q.bound[m] = map_bound(lo, hi, cell_size[m]);
            // without SegmentGround the map frame's box is the union: the grid kernel's check can be made here (after it, on the device).
            // The estimates of the call's clouds are finite: only the resident ones can make the box infinite.
            if (resident && !q.bound[m].finite && !(m == 0 && ransac)) { set_error("%s: map cloud has no finite bounding box", fn); return LVB_ERR_INVALID; }
        }
    }
    return LVB_OK;
}

// The build of side m of a plan: merge in key order, SegmentGround on the ground side (ground_threshold > 0), voxel hash sized by the
// bound into `out`, grid decided on the device into u.blk->map[m].  map: what registration m reads of it.
static int kf_build(lvb_icp* h, const KfPlan& pl, int m, float cell_size, double ground_threshold, const KfUpload& u,
                    lvb_icp::MapBufs& out, KfMap& map) {
    lvb_ctx* ctx = h->ctx;
    cudaStream_t s = ctx->stream;
    MapDesc* md = &u.blk->map[m];
    const int n = (int)pl.total[m];
    LVB_TRY(h->merged.ensure(n));
    size_t o = 0;
    for (auto* f : pl.pick[m]) { if (f->n) LVB_CUDA(cudaMemcpyAsync(h->merged.p + o, f->pts->p, (size_t)f->n * sizeof(float4), cudaMemcpyDeviceToDevice, s)); o += f->n; }
    const float4* cloud = h->merged.p;
    if (m == 0 && ground_threshold > 0.0) {
        LVB_TRY(h->merged2.ensure(n));
        LVB_TRY(lidar_segment_ground_device_async(ctx, h->merged.p, n, ground_threshold, h->merged2.p, &md->P));
        lvb::g_alloc_stream = ctx->stream;
        cloud = h->merged2.p;
    }
    const unsigned char* cp = reinterpret_cast<const unsigned char*>(cloud);
    ILAUNCH(h, icp_bbox_kernel, std::min(1024, inblk(n, 256)), 256, cp, 16, md);
    ILAUNCH(h, icp_map_grid_kernel, 1, 1, md, cell_size, pl.cap[m]);
    LVB_TRY(enqueue_hash(h, cp, n, 16, md, pl.bound[m].cells, pl.bound[m].coarse, false, out));
    map = {out.sorted.p, out.cell_start.p, out.coarse.p, cell_size, pl.bound[m].qsort, false};
    return LVB_OK;
}

// The scan a handle's lvb_icp_map_append(NULL) refers to (bind_scan moves it to the registration's scan)
struct ScanState {
    int n, stride; const unsigned char* dev; std::shared_ptr<DevBuf<unsigned char>> arena; Cloud cloud;
    void save(const lvb_icp* h) { n = h->scan_n; stride = h->scan_stride; dev = h->scan_dev; arena = h->kf_arena; cloud = h->scan_cloud; }
    void restore(lvb_icp* h) const { h->scan_n = n; h->scan_stride = stride; h->scan_dev = dev; h->kf_arena = arena; h->scan_cloud = cloud; }
};

// The argument checks of the calls that build map frames; they come before any state changes
static int kf_check_args(lvb_icp* const hs[2], const float cell_size[2], const void* const pts[2], const int ns[2], int stride,
                         const lvb_map_optimize_params* p, const char* fn) {
    lvb_ctx* ctx = hs[0]->ctx;
    if (hs[1]->ctx != ctx) { set_error("%s: the two handles belong to different contexts", fn); return LVB_ERR_INVALID; }
    if (ctx->world > 1) { set_error("%s: sharded contexts register through lvb_icp_scan_to_map", fn); return LVB_ERR_UNSUPPORTED; }
    const lvb_solve_options& opt = p->options;
    if (opt.max_solver_time_in_seconds < 1e8) { set_error("%s: no time limit (Mapping::Optimize and Mapping::Relocate set none)", fn); return LVB_ERR_INVALID; }
    if (opt.max_num_iterations < 0 || stride < 12 || (stride & 3)) { set_error("%s: bad arguments", fn); return LVB_ERR_INVALID; }
    for (int m = 0; m < 2; ++m) {
        if (ns[m] < 0 || (ns[m] && !pts[m])) { set_error("%s: bad scan arguments", fn); return LVB_ERR_INVALID; }
        if (!(cell_size[m] > 0.0f)) { set_error("%s: bad cell size", fn); return LVB_ERR_INVALID; }
        if ((double)cell_size[m] * cell_size[m] * (1.0 + 1e-6) < p->dist_thr[m]) {
            set_error("%s: dist_thr %.6g exceeds cell_size^2 %.6g", fn, p->dist_thr[m], (double)cell_size[m] * cell_size[m]); return LVB_ERR_INVALID; }
    }
    return LVB_OK;
}

// ---- Mapping::Optimize(active_kfs) (mapping.cpp:139-191) for every lidar keyframe of a backend pass in one call
// (lvb_icp_map_optimize_keyframes), and for one keyframe (lvb_icp_map_build_optimize_keyframe) as the chain of one.  Keyframe k's map
// frame may merge the clouds earlier keyframes of the call store: their poses are decided on the device, so the host sizes that map
// frame from an estimate of their boxes -- the robot-frame box moved by the incoming pose the caller gave, widened by kInCallMargin --
// and passes the capacity it allocated to the grid kernel as a limit.  A cloud that ends up outside its estimate makes the kernel take a
// coarser ring (each ring is exact); only a grid that does not fit at ring 1 fails.
static const float kInCallMargin = 1.0f;        // metres on every side
// The estimate from the robot-frame box rlo..rhi (FLT_MAX / -FLT_MAX when empty)
static void world_box(const float rlo[3], const float rhi[3], const double* pose, float lo[3], float hi[3]) {
    const double mn[3] = {rlo[0], rlo[1], rlo[2]}, mx[3] = {rhi[0], rhi[1], rhi[2]};
    double wl[3], wh[3];
    bool finite = true;
    for (int a = 0; a < 3; ++a) finite = finite && mn[a] <= mx[a] && std::isfinite(mn[a]) && std::isfinite(mx[a]) && mn[a] > -FLT_MAX && mx[a] < FLT_MAX;
    if (!finite) {                             // no point, or an infinite one: the keyframe's position
        for (int a = 0; a < 3; ++a) wl[a] = wh[a] = pose[4 + a];
    } else {                                   // the world box of the robot-frame box's corners
        const double qn = std::sqrt(pose[0] * pose[0] + pose[1] * pose[1] + pose[2] * pose[2] + pose[3] * pose[3]);
        const double x = pose[0] / qn, y = pose[1] / qn, z = pose[2] / qn, w = pose[3] / qn;
        const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                             2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                             2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
        for (int a = 0; a < 3; ++a) { wl[a] = INFINITY; wh[a] = -INFINITY; }
        for (int c = 0; c < 8; ++c) {
            const double p[3] = {c & 1 ? mx[0] : mn[0], c & 2 ? mx[1] : mn[1], c & 4 ? mx[2] : mn[2]};
            for (int a = 0; a < 3; ++a) {
                const double v = R[3 * a] * p[0] + R[3 * a + 1] * p[1] + R[3 * a + 2] * p[2] + pose[4 + a];
                wl[a] = std::min(wl[a], v); wh[a] = std::max(wh[a], v);
            }
        }
    }
    for (int a = 0; a < 3; ++a) {
        lo[a] = std::nextafter((float)(wl[a] - kInCallMargin), -INFINITY);
        hi[a] = std::nextafter((float)(wh[a] + kInCallMargin), INFINITY);
    }
}
// The estimate of a host cloud.  Pending features carry the box the device computed over their points (all finite), which is this one.
static void in_call_box(const void* pts, int n, int stride, const double* pose, float lo[3], float hi[3]) {
    // compare-and-select: a NaN coordinate never wins; an infinite one leaves the box infinite (the device reports that cloud)
    float l[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, h[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    const unsigned char* base = static_cast<const unsigned char*>(pts);
    for (int i = 0; i < n; ++i) {
        const float* f = reinterpret_cast<const float*>(base + (size_t)i * stride);
        for (int a = 0; a < 3; ++a) { l[a] = f[a] < l[a] ? f[a] : l[a]; h[a] = f[a] > h[a] ? f[a] : h[a]; }
    }
    world_box(l, h, pose, lo, hi);
}

// the call's parameters with keyframe kf's own weights and prior weight (ScanToMapWith* read them from each frame)
static lvb_map_optimize_params kf_params(const lvb_map_optimize_params& p, const KfRec& kf) {
    lvb_map_optimize_params q = p;
    q.weight[0] = kf.weight[0]; q.weight[1] = kf.weight[1]; q.prior_weight = kf.prior_weight;
    return q;
}

// A chain of keyframes, entirely on the device: per keyframe the incoming pose chained through the earlier keyframes' transforms, the
// map frame (resident clouds and clouds of earlier keyframes) built into one of two slots per side, both registrations, the transform
// and ToWorld into staged clouds.  The host knows every size the launches depend on -- the scans, the merged clouds, max_num_iterations
// -- and an upper bound on each map frame's grid; the device decides the grid itself (icp_map_grid_kernel) and every counter is used up
// to that size.  One pinned upload, one read-back, one host synchronisation; the staged clouds and the map frames are committed, and
// the records' outputs written, only when every keyframe succeeded.  The callers have checked the arguments (kf_check_args).
static int kf_chain(lvb_icp* const hs[2], KfRec* kfs, int n_kf, const float cell_size[2], double ground_threshold, int stride,
                    const lvb_map_optimize_params* p, const char* fn) {
    // each map key: the cloud an earlier keyframe of the call stores, else the resident one of both handles (one snapshot for all)
    std::vector<std::vector<KfSrc>> srcs(n_kf);
    Snapshot snap;
    {
        StoreLock lk(hs[0], hs[1]);
        for (int k = 0; k < n_kf; ++k) {
            for (int i = 0; i < kfs[k].n_map_keys; ++i) {
                const long long mk = kfs[k].map_keys[i];
                if (mk == kfs[k].key) { set_error("%s: key %lld is its own map key", fn, mk); return LVB_ERR_INVALID; }
                KfSrc sr = {-1, {nullptr, nullptr}};
                for (int j = 0; j < k; ++j) if (kfs[j].key == mk) sr.kf = j;
                if (sr.kf < 0 && !find_resident(hs, snap, mk, sr)) {
                    set_error("%s: map key %lld of keyframe %d is neither resident nor an earlier keyframe of the call", fn, mk, k); return LVB_ERR_INVALID; }
                srcs[k].push_back(sr);
            }
        }
    }
    lvb_ctx* ctx = hs[0]->ctx;
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    std::vector<lvb_icp::Segment> stage(2 * (size_t)n_kf);          // [2 k + m]: the clouds ToWorld stores for keyframe k
    std::vector<KfPlan> pl;
    LVB_TRY(plan_frames(hs, srcs, kfs, stage.data(), cell_size, ground_threshold > 0.0, fn, pl));
    // which slot each build goes into (nx first, then in turn), and the keyframe whose optimised pose is the map pose
    std::vector<int> map_from(n_kf, -1), slot(2 * (size_t)n_kf, -1);
    int turn[2] = {-1, -1};
    for (int k = 0; k < n_kf; ++k) {
        for (int m = 0; m < 2; ++m) if (pl[k].build[m]) { turn[m] = turn[m] < 0 ? 0 : 1 - turn[m]; slot[2 * k + m] = turn[m]; }
        if (!srcs[k].empty() && srcs[k].back().kf >= 0) map_from[k] = srcs[k].back().kf;
    }
    // The estimated boxes of the call's own clouds, and with them the bounds of the map frames that merge them, are formed just before
    // each keyframe is enqueued, while the device runs the keyframes before it.
    std::vector<float> est(12 * (size_t)n_kf);                      // [12 k + 6 m]: the estimated box of keyframe k's stored cloud
    std::vector<char> have_est(2 * (size_t)n_kf, 0);
    // keyframe k's bounds (the resident clouds' union with the estimates of its in-call clouds) and the grid limits that follow from them
    auto plan_bounds = [&](int k) {
        bool in_call = false;
        for (int m = 0; m < 2; ++m) {
            if (!pl[k].build[m]) continue;
            float lo[3], hi[3];
            for (int a = 0; a < 3; ++a) { lo[a] = pl[k].lo[m][a]; hi[a] = pl[k].hi[m][a]; }
            for (auto& sr : srcs[k]) {
                if (sr.kf < 0) continue;
                const size_t e = 2 * (size_t)sr.kf + m;
                if (!have_est[e]) {
                    const KfRec& src = kfs[sr.kf];
                    if (src.pend[m].pts) world_box(src.pend[m].lo, src.pend[m].hi, src.pose, &est[6 * e], &est[6 * e + 3]);
                    else in_call_box(src.pts[m], src.n[m], stride, src.pose, &est[6 * e], &est[6 * e + 3]);
                    have_est[e] = 1;
                }
                for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], est[6 * e + a]); hi[a] = std::max(hi[a], est[6 * e + 3 + a]); }
                in_call = true;
            }
            pl[k].bound[m] = map_bound(lo, hi, cell_size[m]);
        }
        for (int m = 0; m < 2 && in_call; ++m) {
            if (!pl[k].build[m]) continue;
            MapBound& b = pl[k].bound[m];
            b.qsort = b.qcap;
            pl[k].cap[m] = {(double)b.cells, (double)b.coarse, (double)b.qcap};
        }
    };

    const auto t0 = std::chrono::steady_clock::now();
    cudaStream_t s = ctx->stream;
    lvb::timing_mark(s, "begin");
    std::vector<const void*> pts(2 * (size_t)n_kf);
    std::vector<const float4*> dev(2 * (size_t)n_kf);
    std::vector<int> ns(2 * (size_t)n_kf);
    for (int k = 0; k < n_kf; ++k)
        for (int m = 0; m < 2; ++m) { pts[2 * k + m] = kfs[k].pts[m]; dev[2 * k + m] = kfs[k].pend[m].pts ? kfs[k].pend[m].pts->p : nullptr; ns[2 * k + m] = kfs[k].n[m]; }
    std::vector<KfUpload> u;
    size_t back;
    LVB_TRY(kf_upload(ctx, n_kf, true, pts.data(), dev.data(), ns.data(), stride, u, back, [&](int k, KfUpload& v) {
        memcpy(v.hb->map_pose, kfs[k].map_pose, sizeof(v.hb->map_pose)); memcpy(v.hb->pose, kfs[k].pose, sizeof(v.hb->pose));
        for (int m = 0; m < 2; ++m) v.hb->map[m] = pl[k].seed[m];
        v.hl->k = k; v.hl->map_from = map_from[k];
    }));
    KfBlock* dblk = u[0].blk;
    KfLink* dlink = u[0].link;

    ScanState saved[2];
    for (int m = 0; m < 2; ++m) saved[m].save(hs[m]);
    int first[2] = {-1, -1}, last[2] = {-1, -1};       // per side: the keyframes of the first and the latest build
    // the descriptor of what the latest build's slot holds: its own map frame, or (after icp_map_keep_kernel) the one it kept
    auto kept_desc = [&](const KfBlock* b, const KfLink* l, int m) -> const MapDesc* { return first[m] == last[m] ? &b[last[m]].map[m] : &l[last[m]].kept[m]; };
    // per side and slot: the sizes the slot's buffers hold at least (a slot may take over the other slot's map frame)
    size_t held[2][2][3] = {};
    int rc = LVB_OK;
    for (int k = 0; k < n_kf && rc == LVB_OK; ++k) {
        const lvb_map_optimize_params pk = kf_params(*p, kfs[k]);
        KfMap maps[2];
        plan_bounds(k);
        for (int m = 0; m < 2 && rc == LVB_OK; ++m) {
            const int sl = slot[2 * k + m];
            if (sl < 0) continue;
            lvb_icp* h = hs[m];
            lvb_icp::MapBufs& dst = sl ? h->chain : h->nx;
            size_t* need = held[m][sl];
            need[0] = pl[k].total[m]; need[1] = pl[k].bound[m].cells; need[2] = pl[k].bound[m].coarse;
            if (last[m] >= 0) {
                for (int i = 0; i < 3; ++i) need[i] = std::max(need[i], held[m][1 - sl][i]);
                rc = dst.sorted.ensure(need[0]);
                if (rc == LVB_OK) rc = dst.cell_start.ensure(need[1] + 1);
                if (rc == LVB_OK) rc = dst.coarse.ensure(need[2]);
                if (rc != LVB_OK) break;
            }
            rc = kf_build(h, pl[k], m, cell_size[m], ground_threshold, u[k], dst, maps[m]);
            if (rc == LVB_OK && last[m] >= 0) {
                const lvb_icp::MapBufs& src = sl ? h->nx : h->chain;
                ILAUNCH(h, icp_map_keep_kernel, 2 * ctx->sm_count, 256, &dblk[k].map[m], kept_desc(dblk, dlink, m), &dlink[k].kept[m],
                        src.sorted.p, src.cell_start.p, src.coarse.p, dst.sorted.p, dst.cell_start.p, dst.coarse.p);
            }
            if (first[m] < 0) first[m] = k;
            last[m] = k;
        }
        if (rc == LVB_OK) rc = kf_register(hs, pl[k].build, maps, u[k], kfs[k].n, &pk);
        if (rc == LVB_OK) rc = kf_to_world(hs, u[k], kfs[k].n, true, &stage[2 * (size_t)k]);
    }
    if (rc == LVB_OK) rc = icheck(fn);
    // the one read-back: every keyframe's solver states, poses, map descriptors and stored boxes, and its link (transform, kept frames)
    const KfBlock* hb = u[0].hb;
    const KfLink* hl = u[0].hl;
    if (rc == LVB_OK && cudaMemcpyAsync(u[0].hb, dblk, back, cudaMemcpyDeviceToHost, s) != cudaSuccess) rc = lvb::cuda_fail(cudaGetLastError(), "read-back", __FILE__, __LINE__);
    if (rc == LVB_OK) rc = host_sync(ctx, s);
    if (rc == LVB_OK) ctx->stage_busy = false;
    for (int k = 0; k < n_kf && rc == LVB_OK; ++k) {
        for (int m = 0; m < 2 && rc == LVB_OK; ++m) {
            if (!pl[k].build[m]) continue;
            const MapDesc& md = hb[k].map[m];
            if (md.err == 2 && pl[k].cap[m].cells < (double)MAX_CELLS) {
                set_error("%s: the voxel grid of keyframe %d's %s map frame exceeds, at every ring, the capacity sized from the incoming poses", fn, k,
                          m ? "surf" : "ground");
                rc = LVB_ERR_UNSUPPORTED;
            } else rc = grid_error(md, fn, m ? "surf " : "ground ");
        }
    }
    if (rc != LVB_OK) {        // nothing was committed: the resident clouds, the map frames and the scans are as they were
        for (auto& sg : stage) sg.release();
        for (int m = 0; m < 2; ++m) saved[m].restore(hs[m]);
        return rc;
    }
    const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    for (int m = 0; m < 2; ++m) {
        lvb_icp* h = hs[m];
        if (last[m] >= 0) {    // the newest map frame with points replaces the one before, as the step-by-step loop leaves it
            const MapDesc& kd = *kept_desc(hb, hl, m);
            if (kd.P > 0) {
                lvb_icp::MapBufs& sl = slot[2 * last[m] + m] ? h->chain : h->nx;
                swap_buf(h->map_sorted, sl.sorted); swap_buf(h->cell_start, sl.cell_start); swap_buf(h->coarse, sl.coarse);
                h->map = kd; h->cell_size = cell_size[m]; h->have_map = true;
            }
        }
        const KfUpload& ul = u[n_kf - 1];
        h->scan_n = kfs[n_kf - 1].n[m]; h->scan_stride = ul.stride[m]; h->scan_dev = ul.scan[m]; h->kf_arena = ul.arena;
        h->scan_cloud = kfs[n_kf - 1].pend[m].pts;
    }
    std::vector<lvb_icp::Segment> drop;           // released after the stores are unlocked
    StoreLock lk(hs[0], hs[1]);
    for (int k = 0; k < n_kf; ++k) {
        KfRec& kf = kfs[k];
        for (int m = 0; m < 2; ++m) {
            lvb_icp::Segment& sg = stage[2 * (size_t)k + m];
            if (kf.pend[m].pts) sg.robot = kf.pend[m].pts;          // the pending cloud becomes the robot-frame cloud; its entry goes below
            bbox_store(sg, hb[k].out_bbox[m]);
            store_segment(hs[m], kf.key, sg, drop);
            const MapDesc& md = hb[k].map[m];
            const bool built = pl[k].build[m] && md.P > 0;
            kf.n_map_points[m] = built ? md.P : 0;
            if (built) fill_summary(hb[k].st[m], kf.prior_weight, el, &kf.summary[m]);
            else { memset(&kf.summary[m], 0, sizeof(kf.summary[m])); kf.summary[m].termination_type = -1; }
        }
        memcpy(kf.pose, hb[k].pose, sizeof(kf.pose)); memcpy(kf.rpyxyz, hb[k].rpyxyz, sizeof(kf.rpyxyz));
        memcpy(kf.transform, hl[k].T, sizeof(kf.transform));
    }
    for (int m = 0; m < 2; ++m) {
        auto& pv = hs[m]->store->pending;
        std::unordered_set<const DevBuf<float4>*> used;
        for (int k = 0; k < n_kf; ++k) if (kfs[k].pend[m].pts) used.insert(kfs[k].pend[m].pts.get());
        pv.erase(std::remove_if(pv.begin(), pv.end(), [&](const lvb_icp::Pending& pd) { return used.count(pd.pts.get()) > 0; }), pv.end());
    }
    return LVB_OK;
}

// A record's clouds by key (ground_pts == NULL && n_ground < 0, and the same for surf): the pending features of its key on both
// handles.  One side alone, or a key with nothing pending on a handle, is an error; nothing changes.
static int resolve_by_key(lvb_icp* const hs[2], KfRec& kf, const char* fn) {
    const bool bk[2] = {!kf.pts[0] && kf.n[0] < 0, !kf.pts[1] && kf.n[1] < 0};
    kf.pend[0] = kf.pend[1] = lvb_icp::Pending();
    if (!bk[0] && !bk[1]) return LVB_OK;
    if (!bk[0] || !bk[1]) { set_error("%s: keyframe %lld: give both clouds by key or neither", fn, kf.key); return LVB_ERR_INVALID; }
    lvb_icp::Pending pd[2];
    {
        StoreLock lk(hs[0], hs[1]);
        for (int m = 0; m < 2; ++m) {
            const lvb_icp::Pending* e = find_pending(*hs[m]->store, kf.key);
            if (!e) { set_error("%s: key %lld has no pending features on the %s handle", fn, kf.key, m ? "surf" : "ground"); return LVB_ERR_INVALID; }
            pd[m] = *e;
        }
    }
    for (int m = 0; m < 2; ++m) { kf.pend[m] = pd[m]; kf.pts[m] = pd[m].pts->p; kf.n[m] = pd[m].n; }
    return LVB_OK;
}

// Mapping::BuildMapFrame (mapping.cpp:114-137) + the body of Mapping::Optimize's loop (:147-185) for one keyframe: kf_chain of one
// keyframe with the call's weights and prior weight
int lvb_icp_map_build_optimize_keyframe(lvb_icp* ground, lvb_icp* surf, const long long* keys, int n_keys, const float cell_size[2],
                                        double ground_threshold, const double map_pose[7], long long key, const void* ground_pts, int n_ground,
                                        const void* surf_pts, int n_surf, int stride, const lvb_map_optimize_params* p, double pose[7],
                                        double rpyxyz[6], lvb_solve_summary summary[2], int n_map_points[2]) {
    static const char* fn = "lvb_icp_map_build_optimize_keyframe";
    lvb_icp* hs[2] = {ground, surf};
    if (!ground || !surf || ground == surf || !cell_size || !map_pose || !p || !pose || !rpyxyz || n_keys < 0 || (n_keys && !keys)) {
        set_error("%s: null or bad argument", fn); return LVB_ERR_INVALID; }
    KfRec kf = {key, keys, n_keys, {ground_pts, surf_pts}, {n_ground, n_surf}, {}, map_pose, {}, {p->weight[0], p->weight[1]}, p->prior_weight};
    LVB_TRY(resolve_by_key(hs, kf, fn));
    LVB_TRY(kf_check_args(hs, cell_size, kf.pts, kf.n, stride, p, fn));
    memcpy(kf.pose, pose, sizeof(kf.pose));
    LVB_TRY(kf_chain(hs, &kf, 1, cell_size, ground_threshold, stride, p, fn));
    memcpy(pose, kf.pose, sizeof(kf.pose)); memcpy(rpyxyz, kf.rpyxyz, sizeof(kf.rpyxyz));
    if (summary) memcpy(summary, kf.summary, sizeof(kf.summary));
    if (n_map_points) memcpy(n_map_points, kf.n_map_points, sizeof(kf.n_map_points));
    return LVB_OK;
}

int lvb_icp_map_optimize_keyframes(lvb_icp* ground, lvb_icp* surf, lvb_map_keyframe* kfs, int n_kf, const float cell_size[2],
                                   double ground_threshold, int stride, const lvb_map_optimize_params* p) {
    static const char* fn = "lvb_icp_map_optimize_keyframes";
    lvb_icp* hs[2] = {ground, surf};
    if (!ground || !surf || ground == surf || !cell_size || !p || n_kf < 0 || (n_kf > 0 && !kfs)) { set_error("%s: null or bad argument", fn); return LVB_ERR_INVALID; }
    {
        const void* none[2] = {nullptr, nullptr};
        const int zero[2] = {0, 0};
        LVB_TRY(kf_check_args(hs, cell_size, none, zero, stride, p, fn));
    }
    std::unordered_set<long long> batch;
    std::vector<KfRec> rec(n_kf);
    for (int k = 0; k < n_kf; ++k) {
        const lvb_map_keyframe& kf = kfs[k];
        rec[k] = {kf.key, kf.map_keys, kf.n_map_keys, {kf.ground_pts, kf.surf_pts}, {kf.n_ground, kf.n_surf}, {}, kf.map_pose, {},
                  {kf.weight[0], kf.weight[1]}, kf.prior_weight};
        memcpy(rec[k].pose, kf.pose, sizeof(kf.pose));
        LVB_TRY(resolve_by_key(hs, rec[k], fn));
        LVB_TRY(kf_check_args(hs, cell_size, rec[k].pts, rec[k].n, stride, p, fn));
        if (kf.n_map_keys < 0 || kf.n_map_keys > 3) { set_error("%s: keyframe %d has %d map keys (0 to 3)", fn, k, kf.n_map_keys); return LVB_ERR_INVALID; }
        if (!batch.insert(kf.key).second) { set_error("%s: key %lld is listed twice", fn, kf.key); return LVB_ERR_INVALID; }
    }
    if (n_kf == 0) return LVB_OK;
    LVB_TRY(kf_chain(hs, rec.data(), n_kf, cell_size, ground_threshold, stride, p, fn));
    for (int k = 0; k < n_kf; ++k) {
        lvb_map_keyframe& kf = kfs[k];
        memcpy(kf.pose, rec[k].pose, sizeof(kf.pose)); memcpy(kf.rpyxyz, rec[k].rpyxyz, sizeof(kf.rpyxyz));
        memcpy(kf.transform, rec[k].transform, sizeof(kf.transform));
        memcpy(kf.summary, rec[k].summary, sizeof(kf.summary)); memcpy(kf.n_map_points, rec[k].n_map_points, sizeof(kf.n_map_points));
    }
    return LVB_OK;
}

// ---- Mapping::Relocate for one loop-closure candidate (mapping.cpp:251-300): BuildOldMapFrame (:78-112) into each handle's
// relocation slot, then `rounds` rounds of both registrations without a prior, all on the device.  The map frame is planned as a
// keyframe of kf_chain whose keys are all resident; one pinned upload, one read-back, one host synchronisation.  Nothing is stored and
// the handles' map frames, resident clouds and map_append(NULL) scan stay as they were.
int lvb_icp_map_relocate(lvb_icp* ground, lvb_icp* surf, const long long* keys, int n_keys, const float cell_size[2], double ground_threshold,
                         const double map_pose[7], const double old_pose[7], const double relative_guess[7],
                         const void* ground_pts, int n_ground, const void* surf_pts, int n_surf, int stride,
                         const lvb_map_optimize_params* p, int rounds, double relative_o_c[7], double pose[7],
                         lvb_solve_summary summary[2], double score[2], int n_map_points[2]) {
    static const char* fn = "lvb_icp_map_relocate";
    lvb_icp* hs[2] = {ground, surf};
    const void* pts[2] = {ground_pts, surf_pts};
    const int ns[2] = {n_ground, n_surf};
    if (!ground || !surf || ground == surf || !keys || !cell_size || !map_pose || !old_pose || !relative_guess || !p || !relative_o_c || !pose) {
        set_error("%s: null or bad argument", fn); return LVB_ERR_INVALID; }
    if (n_keys < 1 || n_keys > 3) { set_error("%s: the old map frame has 1 to 3 keyframes, got %d", fn, n_keys); return LVB_ERR_INVALID; }
    if (rounds < 1 || rounds > 16) { set_error("%s: rounds %d outside 1..16", fn, rounds); return LVB_ERR_INVALID; }
    LVB_TRY(kf_check_args(hs, cell_size, pts, ns, stride, p, fn));
    if (!(p->prior_weight < 0.0)) { set_error("%s: prior_weight must be < 0 (ScanToMapWith* with relocate = true add no prior)", fn); return LVB_ERR_INVALID; }
    lvb_ctx* ctx = ground->ctx;
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    std::vector<std::vector<KfSrc>> srcs(1);
    Snapshot snap;
    {
        StoreLock lk(ground, surf);
        for (int k = 0; k < n_keys; ++k) {
            KfSrc sr = {-1, {nullptr, nullptr}};
            if (!find_resident(hs, snap, keys[k], sr)) { set_error("%s: key %lld is not resident", fn, keys[k]); return LVB_ERR_INVALID; }
            srcs[0].push_back(sr);
        }
    }
    std::vector<KfPlan> plans;
    LVB_TRY(plan_frames(hs, srcs, nullptr, nullptr, cell_size, ground_threshold > 0.0, fn, plans));
    const KfPlan& pl = plans[0];
    const auto t0 = std::chrono::steady_clock::now();
    cudaStream_t s = ctx->stream;
    lvb::timing_mark(s, "begin");
    std::vector<KfUpload> uk;
    size_t back;
    LVB_TRY(kf_upload(ctx, 1, false, pts, nullptr, ns, stride, uk, back, [&](int, KfUpload& v) {
        memcpy(v.hb->map_pose, map_pose, sizeof(v.hb->map_pose));
        memcpy(v.hb->pose, old_pose, sizeof(v.hb->pose));          // replaced on the device by old_pose * relative_guess
        memcpy(v.hb->old_pose, old_pose, sizeof(v.hb->old_pose)); memcpy(v.hb->rel, relative_guess, sizeof(v.hb->rel));
        for (int m = 0; m < 2; ++m) v.hb->map[m] = pl.seed[m];
    }));
    const KfUpload& u = uk[0];
    KfMap maps[2];
    for (int m = 0; m < 2; ++m) if (pl.build[m]) LVB_TRY(kf_build(hs[m], pl, m, cell_size[m], ground_threshold, u, hs[m]->reloc, maps[m]));

    ScanState saved[2];
    for (int m = 0; m < 2; ++m) saved[m].save(hs[m]);
    int rc = LVB_OK;
    ILAUNCH(ground, icp_reloc_pose_kernel, 1, 1, u.blk, 0);
    for (int r = 0; r < rounds && rc == LVB_OK; ++r) rc = kf_register(hs, pl.build, maps, u, ns, p);
    if (rc == LVB_OK) ILAUNCH(ground, icp_reloc_pose_kernel, 1, 1, u.blk, 1);
    if (rc == LVB_OK) rc = icheck(fn);
    // the one read-back: solver states, pose, relative_o_c, scores, both map descriptors (grid, point count, failure)
    if (rc == LVB_OK && cudaMemcpyAsync(u.hb, u.blk, back, cudaMemcpyDeviceToHost, s) != cudaSuccess) rc = lvb::cuda_fail(cudaGetLastError(), "read-back", __FILE__, __LINE__);
    if (rc == LVB_OK) rc = host_sync(ctx, s);
    if (rc == LVB_OK) ctx->stage_busy = false;
    for (int m = 0; m < 2; ++m) saved[m].restore(hs[m]);
    for (int m = 0; m < 2 && rc == LVB_OK; ++m) if (pl.build[m]) rc = grid_error(u.hb->map[m], fn, m ? "surf " : "ground ");
    if (rc != LVB_OK) return rc;
    const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    for (int m = 0; m < 2; ++m) {
        const bool built = pl.build[m] && u.hb->map[m].P > 0;
        if (n_map_points) n_map_points[m] = built ? u.hb->map[m].P : 0;
        if (score) score[m] = u.hb->score[m];
        if (summary) {
            if (built) fill_summary(u.hb->st[m], p->prior_weight, el, &summary[m]);
            else { memset(&summary[m], 0, sizeof(summary[m])); summary[m].termination_type = -1; }
        }
    }
    memcpy(pose, u.hb->pose, sizeof(u.hb->pose)); memcpy(relative_o_c, u.hb->rel, sizeof(u.hb->rel));
    return LVB_OK;
}

// ---- Mapping::ToWorld(start) after a GNSS or loop correction (mapping.cpp:222-229; backend.cpp:71-91, relocator.cpp:236-244): the
// world clouds of n_keys resident keyframes on one or both handles re-made from their robot-frame records at new poses.  One pinned
// upload of the table [TwSeg per (handle, key) | first block per entry | boxes], one kernel over every point, the boxes read back with
// one copy, one host synchronisation.  Every check comes before the upload; the clouds are overwritten in place, or on a shared store
// written into new buffers that replace them at the commit.
int lvb_icp_map_to_world(lvb_icp* ground, lvb_icp* surf, const long long* keys, int n_keys, const double* poses) {
    static const char* fn = "lvb_icp_map_to_world";
    lvb_icp* hs[2] = {ground, surf};
    if ((!ground && !surf) || ground == surf || n_keys < 0 || (n_keys > 0 && (!keys || !poses))) {
        set_error("%s: null or bad argument", fn); return LVB_ERR_INVALID; }
    if (ground && surf && ground->ctx != surf->ctx) { set_error("%s: the two handles belong to different contexts", fn); return LVB_ERR_INVALID; }
    if (n_keys == 0) return LVB_OK;
    {
        std::vector<long long> sorted(keys, keys + n_keys);
        std::sort(sorted.begin(), sorted.end());
        const auto dup = std::adjacent_find(sorted.begin(), sorted.end());
        if (dup != sorted.end()) { set_error("%s: key %lld is listed twice", fn, *dup); return LVB_ERR_INVALID; }
    }
    // the call's snapshot of the listed clouds; on a store another handle shares, each gets a new world buffer (copy-on-write): another
    // thread's call may take its snapshot while the kernel runs, and must see the cloud as it was.  An unshared store is overwritten in
    // place, and lvb_icp_share waits for that write to be committed.
    std::vector<lvb_icp::Segment> segs;
    std::vector<int> pose_of, side;           // the row of `poses` each entry takes, and its handle
    bool cow[2] = {false, false};
    struct InPlace {                          // clears the in-place flags on every return
        IcpStore* st[2] = {nullptr, nullptr};
        ~InPlace() { for (IcpStore* x : st) if (x) { { std::lock_guard<std::mutex> lk(x->mu); x->in_place = false; } x->cv.notify_all(); } }
    } in_place;
    {
        StoreLock lk(ground, surf);
        for (int m = 0; m < 2; ++m) {
            if (!hs[m]) continue;
            std::unordered_map<long long, const lvb_icp::Segment*> at;
            for (auto& sg : hs[m]->store->segments) at[sg.key] = &sg;
            for (int k = 0; k < n_keys; ++k) {
                const auto it = at.find(keys[k]);
                if (it == at.end()) { set_error("%s: key %lld is not resident on the %s handle", fn, keys[k], m ? "surf" : "ground"); return LVB_ERR_INVALID; }
                segs.push_back(*it->second); pose_of.push_back(k); side.push_back(m);
            }
            cow[m] = hs[m]->store->handles > 1;
            if (!cow[m]) { hs[m]->store->in_place = true; in_place.st[m] = hs[m]->store.get(); }
        }
    }
    const size_t S = segs.size();
    std::vector<int> first(S);
    size_t blocks = 0;
    for (size_t i = 0; i < S; ++i) {
        first[i] = (int)blocks;
        blocks += inblk(segs[i].n, TW_TPB * TW_PER);
        if (blocks > 0x7fffffffull) { set_error("%s: more than 2^31 blocks of %d points", fn, TW_TPB * TW_PER); return LVB_ERR_INVALID; }
    }
    int seed[6];
    bbox_seed(seed);
    std::vector<Cloud> fresh(S);              // the copy-on-write world buffers (NULL: in place)
    std::vector<lvb_icp::Segment> drop;       // the replaced references, released after the stores are unlocked
    // publish the boxes (boxes + 6 i) and the new buffers of the listed clouds; `commit` is set once the device writes are complete
    auto publish = [&](const int* boxes) {
        StoreLock lk(ground, surf);
        for (size_t i = 0; i < S; ++i) {
            lvb_icp::Segment* e = find_segment(*hs[side[i]]->store, segs[i].key);
            if (!e || e->pts != segs[i].pts) continue;
            if (fresh[i]) { drop.push_back(*e); e->pts = fresh[i]; }
            bbox_store(*e, boxes ? boxes + 6 * i : seed);
        }
    };
    if (blocks == 0) {         // every listed cloud is empty: nothing to write, and their boxes stay the empty seeds
        publish(nullptr);
        return LVB_OK;
    }
    lvb_ctx* ctx = (ground ? ground : surf)->ctx;
    lvb_icp* h0 = ground ? ground : surf;
    LVB_CUDA(cudaSetDevice(ctx->device)); lvb::g_alloc_stream = ctx->stream;
    for (size_t i = 0; i < S; ++i) {
        if (!cow[side[i]]) continue;
        fresh[i] = new_cloud();
        LVB_TRY(fresh[i]->ensure(std::max(1, segs[i].n)));
    }
    cudaStream_t s = ctx->stream;
    const size_t off_first = (S * sizeof(TwSeg) + 255) & ~(size_t)255;
    const size_t off_box = (off_first + S * sizeof(int) + 255) & ~(size_t)255;
    const size_t all = off_box + S * 6 * sizeof(int);
    LVB_TRY(lvb::stage_wait(ctx));
    LVB_TRY(lvb::stage_grow(ctx, all, 0));
    TwSeg* ht = reinterpret_cast<TwSeg*>(ctx->stage_h);
    int* hbox = reinterpret_cast<int*>(ctx->stage_h + off_box);
    for (size_t i = 0; i < S; ++i) {
        ht[i].robot = segs[i].robot->p; ht[i].world = fresh[i] ? fresh[i]->p : segs[i].pts->p; ht[i].n = segs[i].n;
        for (int k = 0; k < 7; ++k) ht[i].tf[k] = (float)poses[7 * (size_t)pose_of[i] + k];      // pose.cast<float>() (mapping.cpp:195)
        memcpy(hbox + 6 * i, seed, sizeof(seed));
    }
    memcpy(ctx->stage_h + off_first, first.data(), S * sizeof(int));
    DevBuf<unsigned char> d;
    LVB_TRY(d.ensure(all));
    LVB_CUDA(cudaMemcpyAsync(d.p, ctx->stage_h, all, cudaMemcpyHostToDevice, s));
    LVB_TRY(lvb::stage_mark_busy(ctx, s));
    int* dbox = reinterpret_cast<int*>(d.p + off_box);
    lvb::timing_mark(s, "begin");        // with per-kernel timing on, the kernel's interval starts after the table's upload
    ILAUNCH(h0, icp_map_to_world_kernel, (int)blocks, TW_TPB, reinterpret_cast<const TwSeg*>(d.p), reinterpret_cast<const int*>(d.p + off_first),
            (int)S, dbox);
    LVB_TRY(icheck(fn));
    LVB_CUDA(cudaMemcpyAsync(hbox, dbox, S * 6 * sizeof(int), cudaMemcpyDeviceToHost, s));
    LVB_TRY(host_sync(ctx, s));
    ctx->stage_busy = false;
    publish(hbox);
    return LVB_OK;
}

// ---- FeatureAssociation::Process (association.cpp:85-109) into the map handles: the keyframe's feature clouds stay on the device as
// the pending features of `key`, which lvb_icp_map_optimize_keyframes / lvb_icp_map_build_optimize_keyframe register and store by key
int lvb_icp_map_extract_keyframe(lvb_icp* ground, lvb_icp* surf, const lvb_lidar_config* cfg, long long key, const void* points, int n, int stride,
                                 int32_t* n_ground, int32_t* n_surf, float* ground_xyzi, float* surf_xyzi) {
    static const char* fn = "lvb_icp_map_extract_keyframe";
    if (!ground || !surf || ground == surf || !n_ground || !n_surf) { set_error("%s: null or bad argument", fn); return LVB_ERR_INVALID; }
    if (ground->ctx != surf->ctx) { set_error("%s: the two handles belong to different contexts", fn); return LVB_ERR_INVALID; }
    DevBuf<float4> feat[2];
    float box[12];
    int32_t counts[2];
    LVB_TRY(lidar_extract_keyframe(ground->ctx, cfg, points, n, stride, fn, feat[0], feat[1], &counts[0], &counts[1], box, ground_xyzi, surf_xyzi));
    // The extraction buffers hold num_scans * horizon_scan records; a pending cloud becomes a resident keyframe's robot-frame cloud, so
    // it keeps exactly its points, as a host cloud stored by the keyframe calls does (stream-ordered copy, no wait)
    lvb_icp::Pending pd[2];
    int rc = LVB_OK;
    for (int m = 0; m < 2; ++m) {
        pd[m].key = key; pd[m].n = counts[m]; pd[m].pts = new_cloud();
        for (int a = 0; a < 3; ++a) { pd[m].lo[a] = box[6 * m + a]; pd[m].hi[a] = box[6 * m + 3 + a]; }
        if (rc == LVB_OK) rc = pd[m].pts->ensure(std::max(1, counts[m]));
        if (rc == LVB_OK && counts[m] &&
            cudaMemcpyAsync(pd[m].pts->p, feat[m].p, (size_t)counts[m] * sizeof(float4), cudaMemcpyDeviceToDevice, ground->ctx->stream) != cudaSuccess)
            rc = lvb::cuda_fail(cudaGetLastError(), "pending copy", __FILE__, __LINE__);
    }
    if (rc != LVB_OK) return rc;
    lvb_icp* hs[2] = {ground, surf};
    bool shared = false;
    {
        StoreLock lk(ground, surf);
        for (int m = 0; m < 2; ++m) shared = shared || hs[m]->store->handles > 1;
    }
    // the copies are stream-ordered on this context: another handle's stream may read the features next, so on a shared store they are
    // waited for before they are published
    if (shared) LVB_TRY(host_sync(ground->ctx, ground->ctx->stream));
    std::vector<lvb_icp::Pending> drop;
    StoreLock lk(ground, surf);
    for (int m = 0; m < 2; ++m) {
        drop_pending(*hs[m]->store, key, drop);          // a second extraction under the same key replaces the first
        hs[m]->store->pending.push_back(pd[m]);
    }
    *n_ground = counts[0]; *n_surf = counts[1];
    return LVB_OK;
}

int lvb_debug_icp_cloud_capacity(lvb_icp* h, long long key, long long cap[3]) {
    if (!h || !cap) { set_error("null argument"); return LVB_ERR_INVALID; }
    cap[0] = cap[1] = cap[2] = -1;
    std::lock_guard<std::mutex> lk(h->store->mu);
    if (const lvb_icp::Segment* sg = find_segment(*h->store, key)) { cap[0] = sg->pts ? (long long)sg->pts->n : -1; cap[1] = sg->robot ? (long long)sg->robot->n : -1; }
    if (const lvb_icp::Pending* pd = find_pending(*h->store, key)) cap[2] = (long long)pd->pts->n;
    return LVB_OK;
}

int lvb_debug_icp_map_grid(lvb_icp* h, int grid[4]) {
    if (!h || !grid) { set_error("null argument"); return LVB_ERR_INVALID; }
    if (!h->have_map) { set_error("no map"); return LVB_ERR_STATE; }
    grid[0] = h->map.g.ring; grid[1] = h->map.g.gx; grid[2] = h->map.g.gy; grid[3] = h->map.g.gz;
    return LVB_OK;
}

}  // extern "C"
