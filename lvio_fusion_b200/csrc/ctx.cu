// ctx.cu -- context, error text, launch accounting and the NCCL hook of liblvio_b200.so.
//
// NCCL is resolved with dlopen at run time (libnccl.so.2: the copy torch already mapped into
// the process if there is one, else the system library), so the library carries no link-time
// dependency on it and single-GPU use never touches it.
#include <dlfcn.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "lvb_internal.cuh"

namespace lvb {

static thread_local std::string g_last_error;
thread_local cudaStream_t g_alloc_stream = nullptr;

void set_error(const char* fmt, ...) {
    char buf[1024];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    g_last_error = buf;
}
int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
    set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
    return LVB_ERR_CUDA;
}

bool g_timing = false;
static std::vector<std::pair<const char*, cudaEvent_t>> g_marks;
void timing_mark(cudaStream_t s, const char* name) {
    if (!g_timing) return;
    cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, s); g_marks.push_back({name, e});
}

// ---- NCCL through dlopen ---------------------------------------------------------------
struct NcclId { char internal[128]; };
typedef int (*fn_get_unique_id)(NcclId*);
typedef int (*fn_comm_init_rank)(void**, int, NcclId, int);
typedef int (*fn_all_reduce)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef int (*fn_all_gather)(const void*, void*, size_t, int, void*, cudaStream_t);
typedef int (*fn_comm_destroy)(void*);
typedef const char* (*fn_get_error_string)(int);

static struct {
    void* handle = nullptr;
    fn_get_unique_id get_unique_id = nullptr;
    fn_comm_init_rank comm_init_rank = nullptr;
    fn_all_reduce all_reduce = nullptr;
    fn_all_gather all_gather = nullptr;
    fn_comm_destroy comm_destroy = nullptr;
    fn_get_error_string get_error_string = nullptr;
} g_nccl;

static int nccl_load() {
    if (g_nccl.handle) return LVB_OK;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    void* h = nullptr;
    for (const char* n : names) { h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (h) break; }
    if (!h) { set_error("NCCL not found: %s", dlerror()); return LVB_ERR_COMM; }
    g_nccl.get_unique_id = (fn_get_unique_id)dlsym(h, "ncclGetUniqueId");
    g_nccl.comm_init_rank = (fn_comm_init_rank)dlsym(h, "ncclCommInitRank");
    g_nccl.all_reduce = (fn_all_reduce)dlsym(h, "ncclAllReduce");
    g_nccl.all_gather = (fn_all_gather)dlsym(h, "ncclAllGather");
    g_nccl.comm_destroy = (fn_comm_destroy)dlsym(h, "ncclCommDestroy");
    g_nccl.get_error_string = (fn_get_error_string)dlsym(h, "ncclGetErrorString");
    if (!g_nccl.get_unique_id || !g_nccl.comm_init_rank || !g_nccl.all_reduce) { set_error("NCCL symbols missing"); return LVB_ERR_COMM; }
    g_nccl.handle = h;
    return LVB_OK;
}
static int nccl_fail(int rc, const char* what) {
    set_error("NCCL error %d (%s) in %s", rc, g_nccl.get_error_string ? g_nccl.get_error_string(rc) : "?", what);
    return LVB_ERR_COMM;
}

// ---- in-kernel all-reduce over peer memory (NVLink / NVSwitch): protocol and device functions in lvb_p2p.cuh
}  // namespace lvb
#include "lvb_p2p.cuh"
namespace lvb {

__global__ void __launch_bounds__(256) p2p_allreduce_kernel(P2PArgs a, double* __restrict__ buf, int count) {
    bool last; unsigned int epoch;
    if (!p2p_allreduce_body(a, buf, count, [&](int i) { return __ldcg(buf + i); }, &last, &epoch)) return;
    if (last) p2p_finish_epoch(a, epoch);
}

static int p2p_setup(lvb_ctx* ctx) {
    // every step is collective; a failure on any rank disables the path on all of them (min all-reduce of the ok flag)
    int ok = 1;
    const char* off = getenv("LVB_NO_P2P");
    if ((off && off[0] == '1') || ctx->world > 8 || !g_nccl.all_gather) ok = 0;
    cudaIpcMemHandle_t mine; memset(&mine, 0, sizeof(mine));
    if (ok) {
        if (cudaMalloc((void**)&ctx->xbuf, XB_TOTAL) != cudaSuccess) { ok = 0; ctx->xbuf = nullptr; cudaGetLastError(); }
        // zeroed on the context's stream, which is synchronised below before any peer can learn the handle
        else if (cudaMemsetAsync(ctx->xbuf, 0, XB_TOTAL, ctx->stream) != cudaSuccess || cudaIpcGetMemHandle(&mine, ctx->xbuf) != cudaSuccess) { ok = 0; cudaGetLastError(); }
    }
    unsigned char* d_all = nullptr;
    const size_t hb = sizeof(cudaIpcMemHandle_t);
    LVB_CUDA(cudaMalloc((void**)&d_all, hb * ctx->world + 16));
    LVB_CUDA(cudaMemcpy(d_all + hb * ctx->rank, &mine, hb, cudaMemcpyHostToDevice));
    int* d_ok = reinterpret_cast<int*>(d_all + hb * ctx->world);
    if (g_nccl.all_gather) {
        const int rc = g_nccl.all_gather(d_all + hb * ctx->rank, d_all, hb, /*ncclChar*/ 0, ctx->comm, ctx->stream);
        if (rc != 0) { cudaFree(d_all); return nccl_fail(rc, "ncclAllGather"); }
    }
    LVB_CUDA(cudaStreamSynchronize(ctx->stream));
    std::vector<cudaIpcMemHandle_t> all(ctx->world);
    LVB_CUDA(cudaMemcpy(all.data(), d_all, hb * ctx->world, cudaMemcpyDeviceToHost));
    if (ok) {
        for (int r = 0; r < ctx->world && ok; ++r) {
            if (r == ctx->rank) { ctx->xpeer[r] = ctx->xbuf; continue; }
            void* p = nullptr;
            if (cudaIpcOpenMemHandle(&p, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = 0; cudaGetLastError(); }
            ctx->xpeer[r] = (unsigned char*)p;
        }
    }
    LVB_CUDA(cudaMemcpy(d_ok, &ok, sizeof(int), cudaMemcpyHostToDevice));
    const int rc = g_nccl.all_reduce(d_ok, d_ok, 1, /*ncclInt32*/ 2, /*ncclMin*/ 3, ctx->comm, ctx->stream);
    if (rc != 0) { cudaFree(d_all); return nccl_fail(rc, "ncclAllReduce(p2p ok)"); }
    LVB_CUDA(cudaStreamSynchronize(ctx->stream));
    LVB_CUDA(cudaMemcpy(&ok, d_ok, sizeof(int), cudaMemcpyDeviceToHost));
    cudaFree(d_all);
    ctx->p2p_ok = ok != 0;
    return LVB_OK;
}

// peer pointers for a kernel that runs the exchange itself (ba_allreduce_fused_kernel); false when the message must go through NCCL
bool comm_p2p_args(const lvb_ctx* ctx, size_t count, P2PArgs* a) {
    static const bool off = getenv("LVB_NO_FUSED_COMM") && getenv("LVB_NO_FUSED_COMM")[0] == '1';
    if (off || ctx->world <= 1 || !ctx->p2p_ok || count * sizeof(double) > (size_t)XB_DATA) return false;
    for (int r = 0; r < 8; ++r) a->peer[r] = ctx->xpeer[r];
    a->rank = ctx->rank; a->world = ctx->world; a->timeout_ns = ctx->p2p_timeout_ns;
    return true;
}

bool comm_graph_safe(const lvb_ctx* ctx, size_t max_count) {
    return ctx->world <= 1 || (ctx->p2p_ok && max_count * sizeof(double) <= (size_t)XB_DATA);
}

int comm_allreduce_sum_f64(lvb_ctx* ctx, double* buf, size_t count) {
    if (ctx->world <= 1 || !ctx->comm) return LVB_OK;
    if (ctx->p2p_ok && count * sizeof(double) <= (size_t)XB_DATA) {
        P2PArgs a;
        for (int r = 0; r < 8; ++r) a.peer[r] = ctx->xpeer[r];
        a.rank = ctx->rank; a.world = ctx->world; a.timeout_ns = ctx->p2p_timeout_ns;
        const int blocks = (int)std::min<size_t>(XB_BLOCKS, (count + 255) / 256);
        p2p_allreduce_kernel<<<std::max(1, blocks), 256, 0, ctx->stream>>>(a, buf, (int)count);
        ctx->launches++;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { set_error("p2p all-reduce launch failed: %s", cudaGetErrorString(e)); return LVB_ERR_CUDA; }
        timing_mark(ctx->stream, "p2p_allreduce_kernel");
        return LVB_OK;
    }
    const int rc = g_nccl.all_reduce(buf, buf, count, /*ncclDouble*/ 8, /*ncclSum*/ 0, ctx->comm, ctx->stream);
    if (rc != 0) return nccl_fail(rc, "ncclAllReduce");
    timing_mark(ctx->stream, "ncclAllReduce");
    return LVB_OK;
}

// Turns the sticky error word of the in-kernel exchange into LVB_ERR_COMM.  Called where the host looks at device state anyway.
int comm_check(lvb_ctx* ctx) {
    if (ctx->world <= 1 || !ctx->p2p_ok || !ctx->xbuf) return LVB_OK;
    unsigned int word = 0;
    LVB_CUDA(cudaMemcpyAsync(&word, ctx->xbuf + XB_FLAGS + 8, sizeof(word), cudaMemcpyDeviceToHost, ctx->stream));
    LVB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (word) {
        set_error("peer-memory all-reduce on rank %d timed out after %.1f s waiting for rank %u: the ranks issued different collective sequences "
                  "or a peer is gone; this communicator is unusable", ctx->rank, ctx->p2p_timeout_ns * 1e-9, word - 1u);
        return LVB_ERR_COMM;
    }
    return LVB_OK;
}

// max over the ranks of a host double (seconds), so that wall-clock decisions are the same on every rank (collective)
int comm_max_seconds(lvb_ctx* ctx, double* seconds) {
    if (ctx->world <= 1) return LVB_OK;
    if (!ctx->scratch_i32) LVB_CUDA(cudaMalloc((void**)&ctx->scratch_i32, 64));
    int us = (int)std::min(2.0e9, std::max(0.0, *seconds * 1e6));
    LVB_CUDA(cudaMemcpyAsync(ctx->scratch_i32, &us, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    LVB_TRY(comm_allreduce_max_i32(ctx, ctx->scratch_i32, 1));
    LVB_CUDA(cudaMemcpyAsync(&us, ctx->scratch_i32, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    LVB_CUDA(cudaStreamSynchronize(ctx->stream));
    *seconds = us * 1e-6;
    return LVB_OK;
}

int comm_allreduce_max_i32(lvb_ctx* ctx, int* buf, size_t count) {
    if (ctx->world <= 1 || count == 0) return LVB_OK;
    const int rc = g_nccl.all_reduce(buf, buf, count, /*ncclInt32*/ 2, /*ncclMax*/ 2, ctx->comm, ctx->stream);
    if (rc != 0) return nccl_fail(rc, "ncclAllReduce(max)");
    return LVB_OK;
}

int comm_allreduce_min_i32(lvb_ctx* ctx, int* buf, size_t count) {
    if (ctx->world <= 1 || count == 0) return LVB_OK;
    const int rc = g_nccl.all_reduce(buf, buf, count, /*ncclInt32*/ 2, /*ncclMin*/ 3, ctx->comm, ctx->stream);
    if (rc != 0) return nccl_fail(rc, "ncclAllReduce(min)");
    return LVB_OK;
}

}  // namespace lvb

using namespace lvb;

extern "C" {

int lvb_version(void) { return 100; }

void lvb_default_options(lvb_solve_options* o) {
    o->max_num_iterations = 50; o->max_solver_time_in_seconds = 1e9; o->function_tolerance = 1e-6;
    o->gradient_tolerance = 1e-10; o->parameter_tolerance = 1e-8; o->initial_trust_region_radius = 1e4;
    o->jacobi_scaling = 1; o->linear_solver_type = 0; o->num_threads = 1; o->schur_mode = 0;
}

const char* lvb_last_error(void) { return g_last_error.c_str(); }

int lvb_ctx_create(int device, void* cuda_stream, lvb_ctx** out) {
    if (!out) { set_error("out is NULL"); return LVB_ERR_INVALID; }
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        set_error("no CUDA device available (%s); this library has no CPU fallback", cudaGetErrorString(e));
        return LVB_ERR_CUDA;
    }
    if (device < 0 || device >= count) { set_error("device %d out of range (%d devices)", device, count); return LVB_ERR_INVALID; }
    LVB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    LVB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) { set_error("device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor); return LVB_ERR_CUDA; }
    lvb_ctx* c = new lvb_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    if (cuda_stream) { c->stream = (cudaStream_t)cuda_stream; c->own_stream = false; }
    else { LVB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)); c->own_stream = true; }
    {   // keep freed device memory in the stream-ordered pool (see DevBuf)
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) { unsigned long long thr = ~0ull; cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr); }
    }
    LVB_CUDA(cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking));
    LVB_CUDA(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
    LVB_CUDA(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
    const char* no_side = getenv("LVB_NO_SIDE");
    c->use_side = !(no_side && no_side[0] == '1');
    const char* no_tma = getenv("LVB_NO_TMA");
    c->use_tma = !(no_tma && no_tma[0] == '1');
    const char* no_graph = getenv("LVB_NO_GRAPH");
    c->use_graph = !(no_graph && no_graph[0] == '1');
    const char* ev = getenv("LVB_EVAL_VARIANT");
    if (ev) c->eval_variant = atoi(ev);
    const char* ngc = getenv("LVB_NO_GRAPH_CACHE");
    c->use_graph_cache = !(ngc && ngc[0] == '1');
    const char* pt = getenv("LVB_P2P_TIMEOUT_MS");
    if (pt && atof(pt) > 0) c->p2p_timeout_ns = (unsigned long long)(atof(pt) * 1e6);
    const char* ce = getenv("LVB_CHECK_EVERY");
    if (ce && atoi(ce) > 0) c->check_every = atoi(ce);
    *out = c;
    return LVB_OK;
}

void lvb_ctx_destroy(lvb_ctx* ctx) {
    if (!ctx) return;
    for (int r = 0; r < 8; ++r) if (ctx->xpeer[r] && r != ctx->rank) cudaIpcCloseMemHandle(ctx->xpeer[r]);
    if (ctx->xbuf) cudaFree(ctx->xbuf);
    if (ctx->scratch_i32) cudaFree(ctx->scratch_i32);
    if (ctx->graph_cache) cudaGraphExecDestroy(ctx->graph_cache);
    if (ctx->stage_ev) { cudaEventSynchronize(ctx->stage_ev); cudaEventDestroy(ctx->stage_ev); }
    if (ctx->stage_h) cudaFreeHost(ctx->stage_h);
    if (ctx->comm && g_nccl.comm_destroy) g_nccl.comm_destroy(ctx->comm);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    if (ctx->side) cudaStreamDestroy(ctx->side);
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

long long lvb_launch_count(lvb_ctx* ctx) { return ctx ? ctx->launches : 0; }

int lvb_ctx_synchronize(lvb_ctx* ctx) {
    if (!ctx) return LVB_ERR_INVALID;
    LVB_CUDA(cudaStreamSynchronize(ctx->stream));
    return LVB_OK;
}

int lvb_debug_timing(int enable) {
    if (!enable && g_timing) {
        cudaDeviceSynchronize();
        for (size_t i = 1; i < g_marks.size(); ++i) { float ms = 0; cudaEventElapsedTime(&ms, g_marks[i - 1].second, g_marks[i].second); printf("%-40s %8.2f us\n", g_marks[i].first, ms * 1e3); }
        for (auto& m : g_marks) cudaEventDestroy(m.second);
        g_marks.clear();
    }
    g_timing = enable != 0;
    return LVB_OK;
}

// Same as lvb_debug_timing(0), but the per-kernel times ("name microseconds" per line, in launch order) go into `out`
// (bench.py sums them by kernel: CUDA events on the launching stream around every kernel of the pass).
int lvb_debug_timing_report(char* out, int cap) {
    if (!out || cap <= 0) { set_error("bad buffer"); return LVB_ERR_INVALID; }
    cudaDeviceSynchronize();
    int pos = 0; out[0] = 0;
    for (size_t i = 1; i < g_marks.size(); ++i) {
        float ms = 0; cudaEventElapsedTime(&ms, g_marks[i - 1].second, g_marks[i].second);
        const int w = snprintf(out + pos, (size_t)(cap - pos), "%s %.3f\n", g_marks[i].first, ms * 1e3);
        if (w < 0 || w >= cap - pos) break;
        pos += w;
    }
    for (auto& m : g_marks) cudaEventDestroy(m.second);
    g_marks.clear();
    g_timing = false;
    return LVB_OK;
}

int lvb_comm_unique_id(char id[128]) {
    LVB_TRY(nccl_load());
    NcclId u;
    const int rc = g_nccl.get_unique_id(&u);
    if (rc != 0) return nccl_fail(rc, "ncclGetUniqueId");
    memcpy(id, u.internal, 128);
    return LVB_OK;
}

int lvb_comm_init(lvb_ctx* ctx, int rank, int world_size, const char id[128]) {
    if (!ctx || world_size < 1 || rank < 0 || rank >= world_size) { set_error("bad comm arguments"); return LVB_ERR_INVALID; }
    if (world_size == 1) { ctx->rank = 0; ctx->world = 1; return LVB_OK; }
    LVB_TRY(nccl_load());
    LVB_CUDA(cudaSetDevice(ctx->device));
    NcclId u; memcpy(u.internal, id, 128);
    void* comm = nullptr;
    const int rc = g_nccl.comm_init_rank(&comm, world_size, u, rank);
    if (rc != 0) return nccl_fail(rc, "ncclCommInitRank");
    ctx->comm = comm; ctx->rank = rank; ctx->world = world_size;
    return p2p_setup(ctx);
}

}  // extern "C"
