// include/lvio_b200/ceres_shim.h -- header-only C++ host side of the drop-in boundary.
//
// Keeps the subset of the Ceres API that lvio_fusion's hot path is written against (SURVEY.md 8b; closed
// set taken from `grep ceres::` over /root/reference/src/lvio_fusion) and forwards it to the C ABI in
// include/lvio_b200.h.  What the reference does with these calls:
//
//   adapt::Problem : ceres::Problem          include/lvio_fusion/adapt/problem.h:34-81
//   AddParameterBlock(double*, size[, param]) problem.h:49-63, backend.cpp:111,121,150-152
//   AddResidualBlock(cost, loss, x0, xs...)   problem.h:37-47 (<= 8 blocks: ImuError)
//   ceres::Solve(options, &problem, &summary) problem.h:83-88, backend.cpp:204-211, mapping.cpp:159-164
//   HuberLoss / TrivialLoss / ProductParameterization(EigenQuaternion, Identity3)  backend.cpp:98-101
//
// Design: a GPU backend cannot run arbitrary C++ functors, so the cost functions on the hot path are the
// closed set in factors.h (same class names and Create() signatures as include/lvio_fusion/ceres/*.hpp),
// each a lvb::DeviceCost carrying its factor kind and constant record.  Problem records pointers exactly
// like Ceres (pointer identity = block identity, memory owned by the caller's Frame / Landmark objects),
// Solve() packs them into the flat arrays of lvb_ba_*, runs the LM on the device and writes the
// parameters back IN PLACE.  There is no CPU fallback for these: without a device Solve() reports FAILURE.
// Problems made only of generic functors (ceres_autodiff.h: the off-path tiny solves of the reference --
// navsat, section pose graph, relocation; SURVEY 8f-4), optionally with PoseGraphError / PoseError blocks, are
// solved by the small dense host LM in host_solver.h; mixing them with hot-path factor kinds is an error.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>
#include "../lvio_b200.h"

namespace lvb {

// Device context + the stereo rig constants (Camera::Get(0/1) of the reference).
// The reference solves from several host threads at once (Backend::BackendLoop, Backend::GlobalLoop, Relocator::DetectorLoop:
// backend.cpp:19-20, relocator.cpp), so the context -- one CUDA stream, on which an LM pass may be under graph capture -- is per
// host THREAD: kernels of one thread's solve never land in another thread's stream.  The rig is registered once for the process.
struct Runtime {
    lvb_ctx* ctx = nullptr;
    std::string error;
    double (&cameras)[22];
    bool& have_cameras;
    static Runtime& get() { static thread_local Runtime r; return r; }
    bool ensure(int device = 0) {
        if (ctx) return true;
        const int rc = create_with_priority ? create_with_priority(device, priority, &ctx) : lvb_ctx_create(device, nullptr, &ctx);
        if (rc != LVB_OK) { error = lvb_last_error(); ctx = nullptr; return false; }
        return true;
    }
    // The CUDA stream priority of this thread's device work (lvb_ctx_create_with_priority; lower runs earlier, see
    // lvb_device_priority_range), e.g. the greatest for the thread that runs Backend::Optimize, whose pass the frontend waits for.
    // Call it on the thread, before its first device call: the context is made then.  Once it exists this returns false with a
    // message in `error` and leaves the priority as it is.
    bool set_thread_priority(int p) {
        if (ctx) { error = "set_thread_priority: this thread's context already exists; call it before the thread's first device call"; return false; }
        priority = p;
        create_with_priority = &lvb_ctx_create_with_priority;
        return true;
    }
    // cam = { fx fy cx cy  extrinsic[7] } per camera, Camera::Get(0) then Camera::Get(1)
    void set_cameras(const double* cam0_11, const double* cam1_11) {
        std::memcpy(cameras, cam0_11, 11 * sizeof(double)); std::memcpy(cameras + 11, cam1_11, 11 * sizeof(double)); have_cameras = true;
    }
    // (never destroyed: the solver threads of the reference live as long as the process, and tearing a context down from a
    // thread_local destructor at process exit would call into a CUDA runtime that is already unloading)
private:
    int priority = 0;
    // set by set_thread_priority, so that only a program that sets a priority references the entry point (a C ABI server without
    // stream priorities, such as the CPU oracle, still serves the others)
    int (*create_with_priority)(int, int, lvb_ctx**) = nullptr;
    struct Rig { double c[22] = {0}; bool have = false; };
    static Rig& rig() { static Rig r; return r; }
    Runtime() : cameras(rig().c), have_cameras(rig().have) {}
};

}  // namespace lvb

namespace ceres {

enum LinearSolverType { DENSE_QR = 2, SPARSE_NORMAL_CHOLESKY = 1, SPARSE_SCHUR = 0, DENSE_SCHUR = 3 };
enum TerminationType { CONVERGENCE = 0, NO_CONVERGENCE = 1, FAILURE = 2 };
enum Ownership { DO_NOT_TAKE_OWNERSHIP, TAKE_OWNERSHIP };

class CostFunction {
public:
    virtual ~CostFunction() {}
    // Ceres contract: jacobians == nullptr or jacobians[i] == nullptr means "skip".
    virtual bool Evaluate(double const* const* parameters, double* residuals, double** jacobians) const = 0;
    const std::vector<int32_t>& parameter_block_sizes() const { return sizes_; }
    int num_residuals() const { return num_residuals_; }
protected:
    std::vector<int32_t>* mutable_parameter_block_sizes() { return &sizes_; }
    void set_num_residuals(int n) { num_residuals_ = n; }
private:
    std::vector<int32_t> sizes_;
    int num_residuals_ = 0;
};

template <int kNumResiduals, int... Ns>
class SizedCostFunction : public CostFunction {
public:
    SizedCostFunction() { set_num_residuals(kNumResiduals); *mutable_parameter_block_sizes() = std::vector<int32_t>{Ns...}; }
};

class LossFunction { public: virtual ~LossFunction() {} virtual double huber_a() const { return 0.0; } };
class TrivialLoss : public LossFunction {};
class HuberLoss : public LossFunction { public: explicit HuberLoss(double a) : a_(a) {} double huber_a() const override { return a_; } private: double a_; };

// Plus / ComputeJacobian are only exercised by the host solver of the off-path small solves (host_solver.h); on the device
// path the 7-double pose block always carries the quaternion (x) identity product (backend.cpp:99-101).
class LocalParameterization {
public:
    virtual ~LocalParameterization() {}
    virtual int GlobalSize() const = 0;
    virtual int LocalSize() const = 0;
    virtual bool Plus(const double* x, const double* delta, double* x_plus_delta) const = 0;
    virtual bool ComputeJacobian(const double* x, double* jacobian /* GlobalSize x LocalSize, row-major */) const = 0;
};
// [upstream] ceres::EigenQuaternionParameterization: storage x y z w, q' = q_delta (x) q with q_delta = (sin|d|/|d| d, cos|d|)
class EigenQuaternionParameterization : public LocalParameterization {
public:
    int GlobalSize() const override { return 4; }
    int LocalSize() const override { return 3; }
    bool Plus(const double* x, const double* d, double* out) const override {
        const double n = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        if (n == 0.0) { for (int i = 0; i < 4; ++i) out[i] = x[i]; return true; }
        const double k = std::sin(n) / n, qx = k * d[0], qy = k * d[1], qz = k * d[2], qw = std::cos(n);
        out[0] = qw * x[0] + qx * x[3] + qy * x[2] - qz * x[1];
        out[1] = qw * x[1] - qx * x[2] + qy * x[3] + qz * x[0];
        out[2] = qw * x[2] + qx * x[1] - qy * x[0] + qz * x[3];
        out[3] = qw * x[3] - qx * x[0] - qy * x[1] - qz * x[2];
        return true;
    }
    bool ComputeJacobian(const double* x, double* j) const override {
        j[0] = x[3]; j[1] = x[2]; j[2] = -x[1];
        j[3] = -x[2]; j[4] = x[3]; j[5] = x[0];
        j[6] = x[1]; j[7] = -x[0]; j[8] = x[3];
        j[9] = -x[0]; j[10] = -x[1]; j[11] = -x[2];
        return true;
    }
};
class IdentityParameterization : public LocalParameterization {
public:
    explicit IdentityParameterization(int n) : n_(n) {}
    int GlobalSize() const override { return n_; }
    int LocalSize() const override { return n_; }
    bool Plus(const double* x, const double* d, double* out) const override { for (int i = 0; i < n_; ++i) out[i] = x[i] + d[i]; return true; }
    bool ComputeJacobian(const double*, double* j) const override { for (int i = 0; i < n_ * n_; ++i) j[i] = 0.0; for (int i = 0; i < n_; ++i) j[i * n_ + i] = 1.0; return true; }
private:
    int n_;
};
class ProductParameterization : public LocalParameterization {
public:
    ProductParameterization(LocalParameterization* a, LocalParameterization* b) : a_(a), b_(b) {}
    int GlobalSize() const override { return a_->GlobalSize() + b_->GlobalSize(); }
    int LocalSize() const override { return a_->LocalSize() + b_->LocalSize(); }
    bool Plus(const double* x, const double* d, double* out) const override {
        return a_->Plus(x, d, out) && b_->Plus(x + a_->GlobalSize(), d + a_->LocalSize(), out + a_->GlobalSize());
    }
    bool ComputeJacobian(const double* x, double* j) const override {
        const int ga = a_->GlobalSize(), la = a_->LocalSize(), gb = b_->GlobalSize(), lb = b_->LocalSize(), l = la + lb;
        std::vector<double> ja((size_t)ga * la), jb((size_t)gb * lb);
        if (!a_->ComputeJacobian(x, ja.data()) || !b_->ComputeJacobian(x + ga, jb.data())) return false;
        for (int i = 0; i < (ga + gb) * l; ++i) j[i] = 0.0;
        for (int r = 0; r < ga; ++r) for (int c = 0; c < la; ++c) j[r * l + c] = ja[(size_t)r * la + c];
        for (int r = 0; r < gb; ++r) for (int c = 0; c < lb; ++c) j[(ga + r) * l + la + c] = jb[(size_t)r * lb + c];
        return true;
    }
private:
    std::unique_ptr<LocalParameterization> a_, b_;
};

struct ResidualBlock { CostFunction* cost; LossFunction* loss; std::vector<double*> blocks; };
typedef ResidualBlock* ResidualBlockId;

}  // namespace ceres

namespace lvb {

// A cost function the device knows: factor kind + constant record (lvb_factor_kind, include/lvio_b200.h).
class DeviceCost : public ceres::CostFunction {
public:
    DeviceCost(int kind, int num_residuals, std::vector<int32_t> sizes, std::vector<double> consts) : kind_(kind), consts_(std::move(consts)) {
        set_num_residuals(num_residuals); *mutable_parameter_block_sizes() = std::move(sizes);
    }
    int kind() const { return kind_; }
    const std::vector<double>& consts() const { return consts_; }
    // Host-side single-block evaluation is not part of the device path; callers that need residuals of many
    // blocks use lvb_ba_eval / lvb_ba_reprojection_errors (compute_reprojection_error, backend.cpp:185-190).
    // Kinds that also occur in the off-path host solves (PoseGraphError / PoseError in navsat.cpp:294-301,
    // pose_graph.cpp) carry a host evaluator (factors.h attaches it); the hot-path kinds do not.
    bool Evaluate(double const* const* p, double* r, double** j) const override { return host_ ? host_->Evaluate(p, r, j) : false; }
    void set_host_evaluator(ceres::CostFunction* f) { host_.reset(f); }
    bool has_host_evaluator() const { return (bool)host_; }
private:
    int kind_;
    std::vector<double> consts_;
    std::unique_ptr<ceres::CostFunction> host_;
};

// One whole ScanToMapWith{Ground,Segmented} association expressed as a single residual "block group":
// the per-point LidarPlaneErrorRPZ/YXY factors are created on the device (association.cpp:291-317).
struct ScanToMapCost : public ceres::CostFunction {
    int mode = 0;                       // 0 ground (RPZ), 1 segmented (YXY)
    lvb_icp* icp = nullptr;             // map already set
    const void* scan = nullptr; int n = 0, stride = 0;
    double frame_pose[7], map_pose[7];
    double* rpyxyz = nullptr;           // the live array (lidar_error.hpp:74,109)
    double weight = 1, dist_thr = 0;
    bool Evaluate(double const* const*, double*, double**) const override { return false; }
};
// PoseErrorRPZ / PoseErrorYXY prior (pose_error.hpp:135-190): folded into the scan-to-map solve.
struct IcpPriorCost : public ceres::CostFunction {
    int mode = 0; double weight = 0;
    bool Evaluate(double const* const*, double*, double**) const override { return false; }
};

}  // namespace lvb

namespace ceres {

class Solver {
public:
    struct Options {
        LinearSolverType linear_solver_type = SPARSE_NORMAL_CHOLESKY;
        int max_num_iterations = 50;
        double max_solver_time_in_seconds = 1e9;
        int num_threads = 1;
        double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
        double initial_trust_region_radius = 1e4;
        bool jacobi_scaling = true;
        bool minimizer_progress_to_stdout = false;
    };
    struct Summary {
        double initial_cost = 0, final_cost = 0, total_time_in_seconds = 0;
        int num_successful_steps = 0, num_unsuccessful_steps = 0;
        int num_residual_blocks = 0, num_residual_blocks_reduced = 0;
        TerminationType termination_type = NO_CONVERGENCE;
        std::string message;
        std::string BriefReport() const { return "lvio_b200: cost " + std::to_string(initial_cost) + " -> " + std::to_string(final_cost) + " (" + message + ")"; }
        bool IsSolutionUsable() const { return termination_type != FAILURE; }
    };
};

class Problem {
public:
    Problem() {}
    ~Problem() {
        // default ceres::Problem::Options: the problem owns cost / loss / parameterization objects; a pointer
        // shared by many blocks (backend.cpp:98-101) is freed once.
        std::set<CostFunction*> costs; std::set<LossFunction*> losses;
        for (auto& rb : residuals_) { costs.insert(rb->cost); if (rb->loss) losses.insert(rb->loss); }
        for (auto* c : costs) delete c;
        for (auto* l : losses) delete l;
        for (auto* p : params_owned_) delete p;
    }
    Problem(const Problem&) = delete;
    Problem& operator=(const Problem&) = delete;

    void AddParameterBlock(double* values, int size) { add_block(values, size); }
    void AddParameterBlock(double* values, int size, LocalParameterization* p) { add_block(values, size); if (p) { params_owned_.insert(p); param_of_[values] = p; } }

    template <typename... Ts>
    ResidualBlockId AddResidualBlock(CostFunction* cost, LossFunction* loss, double* x0, Ts*... xs) {
        std::unique_ptr<ResidualBlock> rb(new ResidualBlock{cost, loss, {x0, xs...}});
        const std::vector<int32_t>& sz = cost->parameter_block_sizes();
        for (size_t i = 0; i < rb->blocks.size(); ++i) add_block(rb->blocks[i], i < sz.size() ? sz[i] : 0);
        for (double* b : rb->blocks) by_block_[b].push_back(rb.get());
        residuals_.push_back(std::move(rb));
        return residuals_.back().get();
    }
    void SetParameterBlockConstant(double* v) { constant_.insert(v); }
    void SetParameterBlockVariable(double* v) { constant_.erase(v); }
    bool IsParameterBlockConstant(double* v) const { return constant_.count(v) != 0; }
    void GetResidualBlocksForParameterBlock(const double* v, std::vector<ResidualBlockId>* out) const {
        out->clear(); auto it = by_block_.find(const_cast<double*>(v)); if (it != by_block_.end()) *out = it->second;
    }
    // navsat.cpp:245-246 (only honoured by the host solver; the device path has no bounded blocks)
    void SetParameterLowerBound(double* v, int i, double b) { bound(lower_, v, -std::numeric_limits<double>::infinity())[i] = b; }
    void SetParameterUpperBound(double* v, int i, double b) { bound(upper_, v, std::numeric_limits<double>::infinity())[i] = b; }
    const LocalParameterization* parameterization_of(double* v) const { auto it = param_of_.find(v); return it == param_of_.end() ? nullptr : it->second; }
    const double* lower_bounds_of(double* v) const { auto it = lower_.find(v); return it == lower_.end() ? nullptr : it->second.data(); }
    const double* upper_bounds_of(double* v) const { auto it = upper_.find(v); return it == upper_.end() ? nullptr : it->second.data(); }
    int NumResidualBlocks() const { return (int)residuals_.size(); }
    int NumParameterBlocks() const { return (int)blocks_.size(); }

    // ---- used by Solve()
    const std::vector<std::unique_ptr<ResidualBlock>>& residual_blocks() const { return residuals_; }
    const std::vector<std::pair<double*, int>>& parameter_blocks() const { return blocks_; }

private:
    void add_block(double* v, int size) { if (index_.emplace(v, (int)blocks_.size()).second) blocks_.push_back({v, size}); }   // idempotent re-add (tools.cpp:107,151)
    std::vector<std::pair<double*, int>> blocks_;
    std::unordered_map<double*, int> index_;
    std::vector<std::unique_ptr<ResidualBlock>> residuals_;
    std::unordered_map<double*, std::vector<ResidualBlockId>> by_block_;
    std::set<double*> constant_;
    std::set<LocalParameterization*> params_owned_;
    std::unordered_map<double*, LocalParameterization*> param_of_;
    std::unordered_map<double*, std::vector<double>> lower_, upper_;
    std::vector<double>& bound(std::unordered_map<double*, std::vector<double>>& m, double* v, double init) {
        auto it = m.find(v);
        if (it == m.end()) { int size = 1; auto ix = index_.find(v); if (ix != index_.end()) size = blocks_[ix->second].second; it = m.emplace(v, std::vector<double>((size_t)size, init)).first; }
        return it->second;
    }
};

}  // namespace ceres

namespace lvb { namespace host { inline void solve(const ceres::Solver::Options&, ceres::Problem*, ceres::Solver::Summary*); } }   // host_solver.h

namespace ceres {

inline void fill_options(const Solver::Options& o, lvb_solve_options* out) {
    lvb_default_options(out);
    out->max_num_iterations = o.max_num_iterations; out->max_solver_time_in_seconds = o.max_solver_time_in_seconds;
    out->function_tolerance = o.function_tolerance; out->gradient_tolerance = o.gradient_tolerance; out->parameter_tolerance = o.parameter_tolerance;
    out->initial_trust_region_radius = o.initial_trust_region_radius; out->jacobi_scaling = o.jacobi_scaling ? 1 : 0;
    out->linear_solver_type = (int)o.linear_solver_type; out->num_threads = o.num_threads;
}
inline void fill_summary(const lvb_solve_summary& s, Solver::Summary* out) {
    out->initial_cost = s.initial_cost; out->final_cost = s.final_cost; out->total_time_in_seconds = s.total_time_in_seconds;
    out->num_successful_steps = s.num_successful_steps; out->num_unsuccessful_steps = s.num_iterations - s.num_successful_steps;
    out->num_residual_blocks = s.num_residual_blocks; out->num_residual_blocks_reduced = s.num_residual_blocks_reduced;
    out->termination_type = (TerminationType)s.termination_type;
}

// ceres::Solve: never throws; failure is reported through the Summary (which the reference ignores except in
// Mapping::Relocate, mapping.cpp:279-280,293-294).
inline void Solve(const Solver::Options& options, Problem* problem, Solver::Summary* summary) {
    Solver::Summary local; if (!summary) summary = &local;
    *summary = Solver::Summary();
    lvb::Runtime& rt = lvb::Runtime::get();
    auto fail = [&](const std::string& m) { summary->termination_type = FAILURE; summary->message = m; };

    // ---- scan-to-map problems (Mapping::Optimize): one ScanToMapCost (+ optional IcpPriorCost)
    const lvb::ScanToMapCost* scan = nullptr; const lvb::IcpPriorCost* prior = nullptr; const LossFunction* scan_loss = nullptr;
    bool has_device = false, has_other = false, has_hostable = false;
    for (auto& rb : problem->residual_blocks()) {
        if (auto* s = dynamic_cast<const lvb::ScanToMapCost*>(rb->cost)) { scan = s; scan_loss = rb->loss; }
        else if (auto* p = dynamic_cast<const lvb::IcpPriorCost*>(rb->cost)) prior = p;
        else if (auto* dc = dynamic_cast<const lvb::DeviceCost*>(rb->cost)) { if (dc->has_host_evaluator()) has_hostable = true; else has_device = true; }
        else has_other = true;
    }
    // Off-path small solves (navsat, section pose graph, relocation: generic AutoDiff functors, possibly together with
    // PoseGraphError / PoseError): dense LM on the host, host_solver.h.  A problem with any reprojection / IMU / scan-to-map
    // block never goes there.
    if (has_other) {
        if (has_device || scan) return fail("generic cost functions cannot be mixed with the device factor kinds of the CUDA path");
        return lvb::host::solve(options, problem, summary);
    }
    (void)has_hostable;
    if (!rt.ensure()) return fail("no device: " + rt.error);
    lvb_solve_options opt; fill_options(options, &opt);
    lvb_solve_summary sum; std::memset(&sum, 0, sizeof(sum));
    if (scan) {
        if (has_device) return fail("scan-to-map blocks cannot be mixed with BA blocks");
        const double huber = scan_loss ? scan_loss->huber_a() : 0.0;
        const int rc = lvb_icp_scan_to_map(scan->icp, scan->mode, scan->scan, scan->n, scan->stride, scan->frame_pose, scan->map_pose, scan->rpyxyz,
                                           scan->weight, prior ? prior->weight : -1.0, huber, scan->dist_thr, &opt, &sum);
        if (rc != LVB_OK) return fail(lvb_last_error());
        fill_summary(sum, summary); summary->message = "scan-to-map on device";
        return;
    }
    if (!rt.have_cameras) return fail("lvb::Runtime::set_cameras was not called");

    // ---- bundle adjustment: pack pointers into the flat arrays of the C ABI
    std::vector<double*> pose_ptr, vec3_ptr, rho_ptr;
    std::unordered_map<double*, int> index;
    for (auto& pb : problem->parameter_blocks()) {
        std::vector<double*>* dst = pb.second == 7 ? &pose_ptr : (pb.second == 3 ? &vec3_ptr : (pb.second == 1 ? &rho_ptr : nullptr));
        if (!dst) return fail("parameter block of size " + std::to_string(pb.second) + " is not pose(7)/vec3(3)/inverse depth(1)");
        index[pb.first] = (int)dst->size(); dst->push_back(pb.first);
    }
    auto gather = [&](const std::vector<double*>& ptrs, int w, std::vector<double>& vals, std::vector<uint8_t>& cst) {
        vals.resize(ptrs.size() * w); cst.resize(ptrs.size());
        for (size_t i = 0; i < ptrs.size(); ++i) { std::memcpy(&vals[i * w], ptrs[i], w * sizeof(double)); cst[i] = problem->IsParameterBlockConstant(ptrs[i]) ? 1 : 0; }
    };
    std::vector<double> poses, vec3, rho; std::vector<uint8_t> pc, vc, rc_;
    gather(pose_ptr, 7, poses, pc); gather(vec3_ptr, 3, vec3, vc); gather(rho_ptr, 1, rho, rc_);
    std::vector<double> consts[LVB_NUM_KINDS]; std::vector<int32_t> idx[LVB_NUM_KINDS]; double huber[LVB_NUM_KINDS]; bool loss_set[LVB_NUM_KINDS] = {false};
    for (int k = 0; k < LVB_NUM_KINDS; ++k) huber[k] = 0.0;
    for (auto& rb : problem->residual_blocks()) {
        const lvb::DeviceCost* dc = static_cast<const lvb::DeviceCost*>(rb->cost);
        const int k = dc->kind();
        consts[k].insert(consts[k].end(), dc->consts().begin(), dc->consts().end());
        static const int nidx_k[LVB_NUM_KINDS] = {3, 1, 1, 8, 2, 1};
        int added = 0;
        for (double* b : rb->blocks) { idx[k].push_back(index[b]); ++added; }
        for (; added < nidx_k[k]; ++added) idx[k].push_back(-1);     // ImuInitError has no ba_j / bg_j blocks
        const double a = rb->loss ? rb->loss->huber_a() : 0.0;
        if (loss_set[k] && a != huber[k]) return fail("blocks of one factor kind must share their loss function on the device path");
        huber[k] = a; loss_set[k] = true;
    }
    lvb_ba* ba = nullptr;
    if (lvb_ba_create(rt.ctx, &ba) != LVB_OK) return fail(lvb_last_error());
    struct Guard { lvb_ba* p; ~Guard() { lvb_ba_destroy(p); } } guard{ba};
    int rc = lvb_ba_set_cameras(ba, rt.cameras);
    if (rc == LVB_OK) rc = lvb_ba_set_poses(ba, (int)pose_ptr.size(), poses.data(), pc.data());
    if (rc == LVB_OK) rc = lvb_ba_set_vec3(ba, (int)vec3_ptr.size(), vec3.data(), vc.data());
    if (rc == LVB_OK) rc = lvb_ba_set_inv_depths(ba, (int)rho_ptr.size(), rho.data(), rc_.data());
    static const int nidx[LVB_NUM_KINDS] = {3, 1, 1, 8, 2, 1};
    for (int k = 0; k < LVB_NUM_KINDS && rc == LVB_OK; ++k) {
        const int n = (int)idx[k].size() / nidx[k];
        if (n) rc = lvb_ba_add_factors(ba, k, n, consts[k].data(), idx[k].data());
        if (rc == LVB_OK) rc = lvb_ba_set_loss(ba, k, huber[k]);
    }
    if (rc == LVB_OK) rc = lvb_ba_finalize(ba);
    if (rc == LVB_OK) rc = lvb_ba_solve(ba, &opt, &sum);
    if (rc == LVB_OK && !poses.empty()) rc = lvb_ba_get_poses(ba, poses.data());
    if (rc == LVB_OK && !vec3.empty()) rc = lvb_ba_get_vec3(ba, vec3.data());
    if (rc == LVB_OK && !rho.empty()) rc = lvb_ba_get_inv_depths(ba, rho.data());
    if (rc != LVB_OK) return fail(lvb_last_error());
    // the solver updates the caller's memory in place (frame->pose.data(), &landmark->inv_depth, ...)
    for (size_t i = 0; i < pose_ptr.size(); ++i) if (!pc[i]) std::memcpy(pose_ptr[i], &poses[7 * i], 7 * sizeof(double));
    for (size_t i = 0; i < vec3_ptr.size(); ++i) if (!vc[i]) std::memcpy(vec3_ptr[i], &vec3[3 * i], 3 * sizeof(double));
    for (size_t i = 0; i < rho_ptr.size(); ++i) if (!rc_[i]) *rho_ptr[i] = rho[i];
    fill_summary(sum, summary); summary->message = "bundle adjustment on device";
}

}  // namespace ceres

#include "host_solver.h"
