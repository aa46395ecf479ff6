// lvb_internal.cuh -- context, error plumbing, device buffers, LM state shared by ba.cu / icp.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>
#include "../../include/lvio_b200.h"

namespace lvb {

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define LVB_CUDA(expr)                                                              \
    do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) return lvb::cuda_fail(e_, #expr, __FILE__, __LINE__); } while (0)
#define LVB_TRY(expr)                                                               \
    do { int rc_ = (expr); if (rc_ != LVB_OK) return rc_; } while (0)

}  // namespace lvb

struct lvb_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    cudaStream_t side = nullptr;        // second stream: independent kernels of an LM pass run as parallel branches
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    bool use_side = true;               // env LVB_NO_SIDE=1 disables
    long long launches = 0;
    long long syncs = 0;                // host waits on this context's stream (lvb::host_sync, lvb::stage_wait)
    int sm_count = 132;
    bool use_tma = true;          // cp.async.bulk staging of the pose array (env LVB_NO_TMA=1 disables)
    bool use_graph = true;        // replay the LM pass as a CUDA graph (env LVB_NO_GRAPH=1 disables)
    int eval_variant = 0;         // A/B switch of the Jacobian-eval kernel (env LVB_EVAL_VARIANT)
    int check_every = 4;          // LM passes between host looks at the device state (env LVB_CHECK_EVERY)
    // NCCL (resolved at run time through dlopen, see comm.cu)
    void* comm = nullptr;
    int rank = 0, world = 1;
    // peer-memory exchange for the in-kernel all-reduce over NVLink (ctx.cu); peer[rank] == own buffer
    unsigned char* xbuf = nullptr;
    unsigned char* xpeer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    bool p2p_ok = false;
    unsigned long long p2p_timeout_ns = 20000000000ull;   // env LVB_P2P_TIMEOUT_MS; a silent peer becomes LVB_ERR_COMM, not a hang
    int* scratch_i32 = nullptr;                           // device word for small host-driven collectives (comm_max_seconds)
    // One instantiated LM-pass graph per context, re-targeted to each new problem with cudaGraphExecUpdate (a fresh capture costs a
    // few tens of microseconds, an instantiation a few hundred): the reference builds a new problem per keyframe (Backend::Optimize),
    // so without this the first -- usually only -- solve of a problem could never replay a graph.
    cudaGraphExec_t graph_cache = nullptr;
    const void* graph_owner = nullptr;                    // the lvb_ba whose parameters the cached graph currently holds
    bool use_graph_cache = true;                          // env LVB_NO_GRAPH_CACHE=1 disables
    // Pinned staging area for the arrays a problem uploads when it is finalised (ba.cu, Stager): they are assembled here and go to
    // the device in ONE copy instead of ~40 pageable ones.  Grown on demand, reused by every problem of the context; `stage_ev`
    // marks the last copy that read it.
    unsigned char* stage_h = nullptr;
    size_t stage_cap = 0;
    cudaEvent_t stage_ev = nullptr;
    bool stage_busy = false;
};

namespace lvb {

int comm_allreduce_sum_f64(lvb_ctx* ctx, double* buf, size_t count);   // no-op when world == 1
bool comm_graph_safe(const lvb_ctx* ctx, size_t max_count);          // every all-reduce of <= max_count doubles is a capturable kernel
int comm_allreduce_min_i32(lvb_ctx* ctx, int* buf, size_t count);      // device buffer, no-op when world == 1
int comm_allreduce_max_i32(lvb_ctx* ctx, int* buf, size_t count);
// per-kernel timing (lvb_debug_timing): a CUDA event on the launching stream after every kernel, named; off by default
extern bool g_timing;
void timing_mark(cudaStream_t s, const char* name);
// SegmentGround on a device cloud (lidar.cu): the inlier count stays on the device at n_out_dev (0 when n < 3 or no plane is found),
// `out` holds n records; nothing is waited for
int lidar_segment_ground_device_async(lvb_ctx* ctx, const float4* in, int n, double thr, float4* out, int* n_out_dev);
template <class T> struct DevBuf;
// FeatureAssociation::Process of one scan (lidar.cu), with one host synchronisation: the robot-frame feature clouds stay on the device in
// ground / surf (*n_ground / *n_surf records), with box (may be NULL) their bounding boxes {min xyz, max xyz} x {ground, surf} (FLT_MAX /
// -FLT_MAX when empty), and ground_xyzi / surf_xyzi (may be NULL) receive host copies.  Argument errors come before any work; a
// voxel grid above 2^26 voxels is LVB_ERR_UNSUPPORTED after the synchronisation, with ground / surf untouched.  fn names the caller.
int lidar_extract_keyframe(lvb_ctx* ctx, const lvb_lidar_config* cfg, const void* points, int n, int stride, const char* fn,
                           DevBuf<float4>& ground, DevBuf<float4>& surf, int32_t* n_ground, int32_t* n_surf, float box[12],
                           float* ground_xyzi, float* surf_xyzi);
// every host wait on a context's stream goes through here and is counted in ctx->syncs (lvb_sync_count)
int host_sync(lvb_ctx* ctx, cudaStream_t s);
// The context's pinned staging area (lvb_ctx::stage_h), used by ba.cu (Stager) and icp.cu (lvb_icp_map_optimize_keyframe):
//   stage_wait        wait until the last copy that read it has run (then it may be written)
//   stage_grow        at least `need` bytes, the first `keep` bytes carried over (grows to max(2 x capacity, need, 4 MB))
//   stage_mark_busy   a copy reading it has just been enqueued on `s`
int stage_wait(lvb_ctx* ctx);
int stage_grow(lvb_ctx* ctx, size_t need, size_t keep);
int stage_mark_busy(lvb_ctx* ctx, cudaStream_t s);
int comm_check(lvb_ctx* ctx);                                          // LVB_ERR_COMM when an in-kernel exchange timed out
int comm_max_seconds(lvb_ctx* ctx, double* seconds);                   // collective: max over the ranks (no-op when world == 1)

// Kernel launches on a context's stream (LAUNCH_ON: on another stream, unnamed): an empty grid launches nothing, every launch is
// counted in ctx->launches and, with per-kernel timing on, marked with its name.
#define LAUNCH_ON(ctx, stream_, kernel, grid, block, smem, ...)                            \
    do { if ((grid) > 0) { kernel<<<(grid), (block), (smem), (stream_)>>>(__VA_ARGS__); (ctx)->launches++; } } while (0)
#define LAUNCH_AS(ctx, name, kernel, grid, block, smem, ...)                              \
    do { if ((grid) > 0) { kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__); (ctx)->launches++; lvb::timing_mark((ctx)->stream, name); } } while (0)
#define LAUNCH(ctx, kernel, grid, block, smem, ...) LAUNCH_AS(ctx, #kernel, kernel, grid, block, smem, __VA_ARGS__)

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("kernel launch failed in %s: %s", what, cudaGetErrorString(e)); return LVB_ERR_CUDA; }
    return LVB_OK;
}

// Minimal owning device buffer on the stream-ordered allocator: a problem object allocates ~40 arrays, and
// cudaMalloc (a device-wide synchronising call, ~0.1 ms each) would dominate the end-to-end time of a solve that
// itself takes a couple of milliseconds.  lvb_ctx_create raises the pool's release threshold so freed blocks are
// reused by the next problem instead of being returned to the driver.
extern thread_local cudaStream_t g_alloc_stream;    // stream of the handle currently being operated on
template <class T> struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    cudaStream_t s = nullptr;
    bool view = false;               // p points into another allocation (a problem's upload arena): never freed from here
    ~DevBuf() { release(); }
    void release() { if (p && !view) cudaFreeAsync(p, s); p = nullptr; n = 0; view = false; }
    void set_view(T* q, size_t count) { release(); p = q; n = count; view = true; }
    int ensure(size_t count) {
        if (count <= n && p) return LVB_OK;
        release();
        if (count == 0) count = 1;
        // round up so cp.async.bulk sources stay 16-byte sized and padded reads stay inside the allocation
        size_t bytes = (count * sizeof(T) + 255) / 256 * 256;
        s = g_alloc_stream;
        LVB_CUDA(cudaMallocAsync((void**)&p, bytes, s));
        n = count;
        return LVB_OK;
    }
    int upload(const T* h, size_t count, cudaStream_t st) {
        LVB_TRY(ensure(count));
        if (count) LVB_CUDA(cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, st));
        return LVB_OK;
    }
    int download(T* h, size_t count, cudaStream_t st) const {
        if (count) LVB_CUDA(cudaMemcpyAsync(h, p, count * sizeof(T), cudaMemcpyDeviceToHost, st));
        return LVB_OK;
    }
    int zero(cudaStream_t st) { if (p) LVB_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), st)); return LVB_OK; }
};

// Trust-region state kept on the device so that an LM iteration needs no host round trip for
// its decisions.  Semantics: Ceres TrustRegionMinimizer + LevenbergMarquardtStrategy defaults
// [upstream, not vendored in the reference]; see oracle/lm.h for the CPU restatement.
struct LmState {
    // accumulators (zeroed by the kernels named in the comments)
    double cost_acc;        // 1/2 sum rho at x           (linearize)
    double cand_cost_acc;   // 1/2 sum rho at candidate   (cost kernel)
    double mcc_a, mcc_b;    // sum d.L.d , sum g.d        (update kernel)
    double step_norm2, x_norm2;
    unsigned long long grad_max_bits;
    // trust region
    double x_cost, initial_cost;
    double radius, decrease_factor;
    int iter, num_successful, invalid, done, termination, need_linearize, scale_valid, accept, solve_fail, last_successful;
    int n_accepted;         // ICP: accepted correspondences
    // options
    double f_tol, g_tol, p_tol, min_radius, max_radius, min_diag, max_diag, min_rel_dec;
    int jacobi, max_invalid, max_iter;
};

__host__ __device__ inline void lm_init(LmState& s, const lvb_solve_options& o) {
    s.cost_acc = s.cand_cost_acc = s.mcc_a = s.mcc_b = s.step_norm2 = s.x_norm2 = 0.0;
    s.grad_max_bits = 0ull;
    s.x_cost = s.initial_cost = 0.0;
    s.radius = o.initial_trust_region_radius; s.decrease_factor = 2.0;
    s.iter = 0; s.num_successful = 0; s.invalid = 0; s.done = 0; s.termination = 1; s.need_linearize = 1;
    s.scale_valid = 0; s.accept = 0; s.solve_fail = 0; s.last_successful = 0; s.n_accepted = 0;
    s.f_tol = o.function_tolerance; s.g_tol = o.gradient_tolerance; s.p_tol = o.parameter_tolerance;
    s.min_radius = 1e-32; s.max_radius = 1e16; s.min_diag = 1e-6; s.max_diag = 1e32; s.min_rel_dec = 1e-3;
    s.jacobi = o.jacobi_scaling; s.max_invalid = 5; s.max_iter = o.max_num_iterations;
}

#if defined(__CUDACC__)
// Runs once per iteration after the linearisation (and its all-reduce) is complete and before
// the step is computed: FinalizeIterationAndCheckIfMinimizerCanContinue.
__device__ inline void lm_control_pre(LmState& s) {
    if (s.done) return;
    if (s.need_linearize) { s.x_cost = s.cost_acc; if (s.iter == 0 && s.num_successful == 0 && s.scale_valid == 0) s.initial_cost = s.x_cost; }
    s.scale_valid = 1;
    const double gmax = __longlong_as_double((long long)*(volatile unsigned long long*)&s.grad_max_bits);   // written with atomics: read at L2
    // the gradient at the start point is checked before any limit; after a step, Ceres checks the iteration limit first
    // (time, iterations, gradient, radius), so a solve capped on the step that also reaches gradient_tolerance is NO_CONVERGENCE
    if (s.iter == 0 && gmax <= s.g_tol) { s.done = 1; s.termination = 0; return; }
    if (s.iter >= s.max_iter) { s.done = 1; return; }
    if (s.last_successful && gmax <= s.g_tol) { s.done = 1; s.termination = 0; return; }
    if (s.radius <= s.min_radius) { s.done = 1; s.termination = 0; return; }
    s.iter += 1;
    s.last_successful = 0;
    s.mcc_a = s.mcc_b = s.step_norm2 = s.x_norm2 = 0.0;
    s.cand_cost_acc = 0.0;
    s.solve_fail = 0;
    s.accept = 0;
}
// Runs after the candidate cost is known: step validity, tolerances, accept / reject, radius.
__device__ inline void lm_control_post(LmState& s) {
    if (s.done) return;
    s.need_linearize = 0;
    const double model_cost_change = 0.5 * (s.mcc_a - s.mcc_b);
    if (s.solve_fail || !(model_cost_change > 0.0) || !isfinite(model_cost_change)) {
        if (++s.invalid >= s.max_invalid) { s.done = 1; s.termination = 2; return; }
        // LevenbergMarquardtStrategy::StepIsInvalid() is `StepRejected(0.0)` in Ceres 1.x / 2.x (levenberg_marquardt_strategy.cc;
        // the `radius *= 0.5` rule belongs to DoglegStrategy::StepRejected): same shrink as a rejected step  [upstream]
        s.radius = s.radius / s.decrease_factor; s.decrease_factor *= 2.0;
        return;
    }
    s.invalid = 0;
    const double cand = s.cand_cost_acc;
    if (sqrt(s.step_norm2) <= s.p_tol * (sqrt(s.x_norm2) + s.p_tol)) { s.done = 1; s.termination = 0; return; }
    if (fabs(s.x_cost - cand) <= s.f_tol * s.x_cost) { s.done = 1; s.termination = 0; return; }
    const double rel = (s.x_cost - cand) / model_cost_change;
    if (rel > s.min_rel_dec) {
        s.accept = 1; s.need_linearize = 1; s.last_successful = 1; s.num_successful += 1;
        s.cost_acc = 0.0; s.grad_max_bits = 0ull;
        const double t = 2.0 * rel - 1.0;
        s.radius = fmin(s.max_radius, s.radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
        s.decrease_factor = 2.0;
    } else {
        s.radius = s.radius / s.decrease_factor; s.decrease_factor *= 2.0;
    }
}
#endif

}  // namespace lvb
