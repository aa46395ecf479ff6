// include/lvio_b200/host_solver.h -- dense Levenberg-Marquardt on the host for the reference's OFF-PATH small solves
// (SURVEY 8(f).4): navsat alignment (navsat.cpp:104-129,199-263,273-306: 1-6 scalars or a short pose chain), the section
// pose graph (pose_graph.cpp:163-224: O(#sections) poses), relocation (relocator.cpp:247-282).  Their cost functions are
// generic AutoDiff functors, not the device factor records of the two hot loops.
//
// This is NOT a fallback of the device path: ceres::Solve (ceres_shim.h) routes a problem here only if it holds no
// reprojection / IMU / scan-to-map block at all, and refuses anything larger than kMaxResiduals x kMaxUnknowns.  Bundle
// adjustment and scan-to-map keep failing loudly without a GPU.
//
// Trust-region semantics: the same published Ceres defaults the device path follows (DESIGN.md section 4): radius 1e4,
// min/max LM diagonal 1e-6 / 1e32, Jacobi scaling fixed at the first linearisation, step quality rho against
// min_relative_decrease 1e-3, radius /= max(1/3, 1 - (2 rho - 1)^3) on success, /= decrease_factor (2, doubling) otherwise,
// function / gradient / parameter tolerances, 5 consecutive invalid steps -> FAILURE.  Loss: Huber through the Corrector's
// sqrt(rho') scaling.  Bounds (navsat.cpp:245-246) by projecting the candidate onto the box [simplification of Ceres'
// projected line search].
#pragma once
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <limits>
#include <string>
#include <unordered_map>
#include <vector>
#include "ceres_shim.h"

namespace lvb {
namespace host {

enum { kMaxResiduals = 200000, kMaxUnknowns = 3000 };

// ---- SE3 helpers on a generic scalar (Sophus storage [qx qy qz qw tx ty tz]); the operations of
// ceres/base.hpp:26-141 restated: normalising rotate, conjugate inverse, Hamilton product, ZYX Euler extraction
using std::asin; using std::atan2; using std::sqrt;
template <class T> inline void rotate(const T* q, const T* p, T* out) {
    const T s = T(1) / sqrt(q[3] * q[3] + q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    const T x = q[0] * s, y = q[1] * s, z = q[2] * s, w = q[3] * s;
    T u0 = y * p[2] - z * p[1], u1 = z * p[0] - x * p[2], u2 = x * p[1] - y * p[0];
    u0 = u0 + u0; u1 = u1 + u1; u2 = u2 + u2;
    out[0] = p[0] + w * u0 + (y * u2 - z * u1); out[1] = p[1] + w * u1 + (z * u0 - x * u2); out[2] = p[2] + w * u2 + (x * u1 - y * u0);
}
template <class T> inline void se3_inverse(const T* a, T* out) {
    out[0] = -a[0]; out[1] = -a[1]; out[2] = -a[2]; out[3] = a[3];
    const T nt[3] = {-a[4], -a[5], -a[6]};
    rotate(out, nt, out + 4);
}
template <class T> inline void se3_product(const T* a, const T* b, T* out) {
    const T zw = a[3], zx = a[0], zy = a[1], zz = a[2], ww = b[3], wx = b[0], wy = b[1], wz = b[2];
    out[3] = zw * ww - zx * wx - zy * wy - zz * wz;
    out[0] = zw * wx + zx * ww + zy * wz - zz * wy;
    out[1] = zw * wy - zx * wz + zy * ww + zz * wx;
    out[2] = zw * wz + zx * wy - zy * wx + zz * ww;
    T t[3]; rotate(a, b + 4, t);
    out[4] = t[0] + a[4]; out[5] = t[1] + a[5]; out[6] = t[2] + a[6];
}
template <class T> inline void se3_to_rpyxyz(const T* a, T* e) {
    const T q0 = a[3], q1 = a[0], q2 = a[1], q3 = a[2];
    e[0] = atan2(T(2) * (q1 * q2 + q0 * q3), T(1) - T(2) * (q2 * q2 + q3 * q3));
    e[1] = asin(T(2) * (q0 * q2 - q1 * q3));
    e[2] = atan2(T(2) * (q2 * q3 + q0 * q1), T(1) - T(2) * (q1 * q1 + q2 * q2));
    e[3] = a[4]; e[4] = a[5]; e[5] = a[6];
}

// pose_error.hpp:10-53 (weights v w, v w, v w, w, 10 w, 10 w) and :55-86 (v w x3, w x3) as functors over T
struct PoseGraphFunctor {
    double e[6], w, v;
    template <class T> bool operator()(const T* T1, const T* T2, T* r) const {
        T inv[7], rel[7], c[6];
        se3_inverse(T1, inv); se3_product(inv, T2, rel); se3_to_rpyxyz(rel, c);
        const double k[6] = {v * w, v * w, v * w, w, 10 * w, 10 * w};
        for (int i = 0; i < 6; ++i) r[i] = T(k[i]) * (T(e[i]) - c[i]);
        return true;
    }
};
struct PoseFunctor {
    double pose[7], w, v;
    template <class T> bool operator()(const T* x, T* r) const {
        T origin[7], inv[7], rel[7], c[6];
        for (int i = 0; i < 7; ++i) origin[i] = T(pose[i]);
        se3_inverse(origin, inv); se3_product(inv, x, rel); se3_to_rpyxyz(rel, c);
        const double k[6] = {v * w, v * w, v * w, w, w, w};
        for (int i = 0; i < 6; ++i) r[i] = T(k[i]) * c[i];
        return true;
    }
};

struct Block { double* user; int gsize, lsize, off; bool constant; const ceres::LocalParameterization* param; const double* lower; const double* upper; std::vector<double> x, cand; };

// dense Cholesky solve of (H + diag(lam)) d = -g ; returns false when not positive definite
inline bool solve_damped(const std::vector<double>& H, const std::vector<double>& lam, const std::vector<double>& g, int n, std::vector<double>& L, std::vector<double>& d) {
    L = H;
    for (int i = 0; i < n; ++i) L[(size_t)i * n + i] += lam[i];
    for (int j = 0; j < n; ++j) {
        double s = L[(size_t)j * n + j];
        for (int k = 0; k < j; ++k) s -= L[(size_t)j * n + k] * L[(size_t)j * n + k];
        if (!(s > 0.0) || !std::isfinite(s)) return false;
        const double ljj = std::sqrt(s);
        L[(size_t)j * n + j] = ljj;
        for (int i = j + 1; i < n; ++i) {
            double t = L[(size_t)i * n + j];
            for (int k = 0; k < j; ++k) t -= L[(size_t)i * n + k] * L[(size_t)j * n + k];
            L[(size_t)i * n + j] = t / ljj;
        }
    }
    for (int i = 0; i < n; ++i) { double t = -g[i]; for (int k = 0; k < i; ++k) t -= L[(size_t)i * n + k] * d[k]; d[i] = t / L[(size_t)i * n + i]; }
    for (int i = n - 1; i >= 0; --i) { double t = d[i]; for (int k = i + 1; k < n; ++k) t -= L[(size_t)k * n + i] * d[k]; d[i] = t / L[(size_t)i * n + i]; }
    return true;
}

inline void solve(const ceres::Solver::Options& options, ceres::Problem* problem, ceres::Solver::Summary* summary) {
    const auto t0 = std::chrono::steady_clock::now();
    auto elapsed = [&]() { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); };
    auto fail = [&](const std::string& m) { summary->termination_type = ceres::FAILURE; summary->message = m; };
    // ---- parameter blocks
    std::vector<Block> blocks;
    std::unordered_map<const double*, int> index;
    int n = 0;
    for (auto& pb : problem->parameter_blocks()) {
        Block b;
        b.user = pb.first; b.gsize = pb.second; b.constant = problem->IsParameterBlockConstant(pb.first);
        b.param = problem->parameterization_of(pb.first);
        if (b.param && b.param->GlobalSize() != b.gsize) return fail("local parameterization size does not match its block");
        b.lsize = b.param ? b.param->LocalSize() : b.gsize;
        b.lower = problem->lower_bounds_of(pb.first); b.upper = problem->upper_bounds_of(pb.first);
        b.off = -1;
        b.x.assign(pb.first, pb.first + pb.second); b.cand = b.x;
        index[pb.first] = (int)blocks.size();
        blocks.push_back(std::move(b));
    }
    // only blocks that appear in a residual are unknowns
    std::vector<char> used(blocks.size(), 0);
    int total_res = 0;
    for (auto& rb : problem->residual_blocks()) { total_res += rb->cost->num_residuals(); for (double* p : rb->blocks) used[index[p]] = 1; }
    for (size_t i = 0; i < blocks.size(); ++i) if (used[i] && !blocks[i].constant) { blocks[i].off = n; n += blocks[i].lsize; }
    summary->num_residual_blocks = summary->num_residual_blocks_reduced = (int)problem->residual_blocks().size();
    if (total_res > kMaxResiduals || n > kMaxUnknowns) return fail("problem too large for the host solver (it only serves the off-path small solves)");

    int max_g = 1, max_r = 1;
    for (auto& b : blocks) max_g = std::max(max_g, b.gsize);
    for (auto& rb : problem->residual_blocks()) max_r = std::max(max_r, rb->cost->num_residuals());
    std::vector<double> H((size_t)n * n), g(n), hdiag(n), scale(n, 1.0), lam(n), delta(n), L;
    std::vector<double> r(max_r);
    std::vector<std::vector<double>> Jg, Jl;          // per argument: global / local Jacobians of one residual block
    std::vector<double> P((size_t)max_g * max_g);

    // cost (and optionally the normal equations) at x or at the candidate
    auto evaluate = [&](bool at_candidate, bool linearize, double* cost_out) -> bool {
        double cost = 0.0;
        if (linearize) { std::fill(H.begin(), H.end(), 0.0); std::fill(g.begin(), g.end(), 0.0); }
        for (auto& rb : problem->residual_blocks()) {
            const int nr = rb->cost->num_residuals(), na = (int)rb->blocks.size();
            std::vector<const double*> args(na); std::vector<double*> jac(na, nullptr);
            if ((int)Jg.size() < na) { Jg.resize(na); Jl.resize(na); }
            for (int a = 0; a < na; ++a) {
                Block& b = blocks[index[rb->blocks[a]]];
                args[a] = at_candidate ? b.cand.data() : b.x.data();
                if (linearize && b.off >= 0) { Jg[a].assign((size_t)nr * b.gsize, 0.0); jac[a] = Jg[a].data(); }
            }
            if (!rb->cost->Evaluate(args.data(), r.data(), linearize ? jac.data() : nullptr)) return false;
            double s = 0.0; for (int i = 0; i < nr; ++i) s += r[i] * r[i];
            double rho = s, sq = 1.0;
            const double a_h = rb->loss ? rb->loss->huber_a() : 0.0;
            if (a_h > 0.0 && s > a_h * a_h) { const double root = std::sqrt(s); rho = 2.0 * a_h * root - a_h * a_h; sq = std::sqrt(a_h / root); }
            cost += 0.5 * rho;
            if (!std::isfinite(cost)) return false;
            if (!linearize) continue;
            for (int i = 0; i < nr; ++i) r[i] *= sq;
            for (int a = 0; a < na; ++a) {
                Block& b = blocks[index[rb->blocks[a]]];
                if (b.off < 0) continue;
                if (b.param) {       // J_local = J_global * dPlus/ddelta
                    b.param->ComputeJacobian(at_candidate ? b.cand.data() : b.x.data(), P.data());
                    Jl[a].assign((size_t)nr * b.lsize, 0.0);
                    for (int i = 0; i < nr; ++i) for (int k = 0; k < b.gsize; ++k) { const double v = Jg[a][(size_t)i * b.gsize + k] * sq; if (v != 0.0) for (int c = 0; c < b.lsize; ++c) Jl[a][(size_t)i * b.lsize + c] += v * P[(size_t)k * b.lsize + c]; }
                } else { Jl[a] = Jg[a]; for (double& v : Jl[a]) v *= sq; }
            }
            for (int a = 0; a < na; ++a) {
                const Block& ba = blocks[index[rb->blocks[a]]];
                if (ba.off < 0) continue;
                for (int c = 0; c < ba.lsize; ++c) { double t = 0.0; for (int i = 0; i < nr; ++i) t += Jl[a][(size_t)i * ba.lsize + c] * r[i]; g[ba.off + c] += t; }
                for (int b2 = 0; b2 < na; ++b2) {
                    const Block& bb = blocks[index[rb->blocks[b2]]];
                    if (bb.off < 0) continue;
                    for (int c = 0; c < ba.lsize; ++c) for (int e = 0; e < bb.lsize; ++e) {
                        double t = 0.0; for (int i = 0; i < nr; ++i) t += Jl[a][(size_t)i * ba.lsize + c] * Jl[b2][(size_t)i * bb.lsize + e];
                        H[(size_t)(ba.off + c) * n + bb.off + e] += t;
                    }
                }
            }
        }
        *cost_out = cost;
        return true;
    };
    auto plus_all = [&](const std::vector<double>& d) {       // cand = Plus(x, d), projected onto the bounds
        for (Block& b : blocks) {
            if (b.off < 0) { b.cand = b.x; continue; }
            if (b.param) b.param->Plus(b.x.data(), d.data() + b.off, b.cand.data());
            else for (int k = 0; k < b.gsize; ++k) b.cand[k] = b.x[k] + d[b.off + k];
            if (b.lower) for (int k = 0; k < b.gsize; ++k) b.cand[k] = std::max(b.cand[k], b.lower[k]);
            if (b.upper) for (int k = 0; k < b.gsize; ++k) b.cand[k] = std::min(b.cand[k], b.upper[k]);
        }
    };
    auto gradient_max_norm = [&]() {                            // ||x - Plus(x, -g)||_inf
        std::vector<double> neg(n); for (int i = 0; i < n; ++i) neg[i] = -g[i];
        plus_all(neg);
        double m = 0.0;
        for (Block& b : blocks) if (b.off >= 0) for (int k = 0; k < b.gsize; ++k) m = std::max(m, std::fabs(b.x[k] - b.cand[k]));
        return m;
    };
    auto write_back = [&]() { for (Block& b : blocks) if (b.off >= 0) std::memcpy(b.user, b.x.data(), sizeof(double) * b.gsize); };

    double x_cost = 0.0;
    if (!evaluate(false, true, &x_cost)) return fail("cost function evaluation failed at the initial point");
    summary->initial_cost = summary->final_cost = x_cost;
    summary->termination_type = ceres::NO_CONVERGENCE;
    summary->message = "host LM (off-path small solve)";
    if (n == 0) { summary->termination_type = ceres::CONVERGENCE; return; }
    for (int i = 0; i < n; ++i) hdiag[i] = H[(size_t)i * n + i];
    if (options.jacobi_scaling) for (int i = 0; i < n; ++i) scale[i] = 1.0 / (1.0 + std::sqrt(hdiag[i]));
    double radius = options.initial_trust_region_radius, decrease_factor = 2.0;
    int invalid = 0, iter = 0;
    bool last_successful = false;
    if (gradient_max_norm() <= options.gradient_tolerance) { summary->termination_type = ceres::CONVERGENCE; return; }
    while (true) {
        if (elapsed() >= options.max_solver_time_in_seconds) break;
        if (iter >= options.max_num_iterations) break;        // before the gradient rule, as in Ceres and the device loop
        if (iter > 0 && last_successful && gradient_max_norm() <= options.gradient_tolerance) { summary->termination_type = ceres::CONVERGENCE; break; }
        if (radius <= 1e-32) { summary->termination_type = ceres::CONVERGENCE; break; }
        ++iter;
        last_successful = false;
        for (int i = 0; i < n; ++i) { const double s2 = scale[i] * scale[i]; lam[i] = std::min(std::max(s2 * hdiag[i], 1e-6), 1e32) / (radius * s2); }
        bool ok = solve_damped(H, lam, g, n, L, delta);
        double model_change = 0.0;
        if (ok) { for (int i = 0; i < n; ++i) model_change += delta[i] * lam[i] * delta[i] - g[i] * delta[i]; model_change *= 0.5; ok = model_change > 0.0 && std::isfinite(model_change); }
        if (!ok) {
            if (++invalid >= 5) { fail("host LM: 5 consecutive invalid steps"); break; }
            radius /= decrease_factor; decrease_factor *= 2.0; ++summary->num_unsuccessful_steps;
            continue;
        }
        invalid = 0;
        plus_all(delta);
        double step2 = 0.0, x2 = 0.0;
        for (Block& b : blocks) if (b.off >= 0) for (int k = 0; k < b.gsize; ++k) { step2 += (b.cand[k] - b.x[k]) * (b.cand[k] - b.x[k]); x2 += b.x[k] * b.x[k]; }
        if (std::sqrt(step2) <= options.parameter_tolerance * (std::sqrt(x2) + options.parameter_tolerance)) { summary->termination_type = ceres::CONVERGENCE; break; }
        double cand_cost = 0.0;
        const bool evaluated = evaluate(true, false, &cand_cost);
        // FunctionToleranceReached is tested on the candidate before the step is judged (Ceres' order; the step is not taken)
        if (evaluated && std::fabs(x_cost - cand_cost) <= options.function_tolerance * x_cost) { summary->termination_type = ceres::CONVERGENCE; break; }
        const double rho = evaluated ? (x_cost - cand_cost) / model_change : -1.0;
        if (evaluated && rho > 1e-3) {
            for (Block& b : blocks) if (b.off >= 0) b.x = b.cand;
            radius = std::min(1e16, radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rho - 1.0, 3)));
            decrease_factor = 2.0;
            last_successful = true; ++summary->num_successful_steps;
            if (!evaluate(false, true, &x_cost)) { fail("cost function evaluation failed"); break; }
            for (int i = 0; i < n; ++i) hdiag[i] = H[(size_t)i * n + i];
        } else {
            radius /= decrease_factor; decrease_factor *= 2.0; ++summary->num_unsuccessful_steps;
        }
    }
    write_back();
    summary->final_cost = x_cost;
    summary->total_time_in_seconds = elapsed();
}

// sqrt_info = LLT(cov^-1 with the bias blocks overwritten by the priors).matrixL()^T  (imu_error.hpp:147-150,254-257), row-major
// 15 x 15, for the host-evaluated ImuInitGError.  Same restatement as the device path's (lvio_fusion_b200/csrc/lvb_math.cuh ::
// sqrt_information, oracle/imu.h): partial-pivot LU inverse, then the unblocked lower Cholesky with Eigen's early return on a
// non-positive pivot (from that column on matrixL() shows the untouched lower triangle of the input).  False: singular / NaN.
inline bool imu_sqrt_information(const double* cov, double prior_a, double prior_g, double* U) {
    const int n = 15;
    double a[225], inv[225], L[225];
    int piv[15];
    for (int i = 0; i < 225; ++i) a[i] = cov[i];
    for (int i = 0; i < n; ++i) piv[i] = i;
    for (int k = 0; k < n; ++k) {
        int best = k; double bv = std::fabs(a[k * n + k]);
        for (int i = k + 1; i < n; ++i) if (std::fabs(a[i * n + k]) > bv) { bv = std::fabs(a[i * n + k]); best = i; }
        if (bv == 0.0) return false;
        if (best != k) { for (int j = 0; j < n; ++j) std::swap(a[k * n + j], a[best * n + j]); std::swap(piv[k], piv[best]); }
        for (int i = k + 1; i < n; ++i) { a[i * n + k] /= a[k * n + k]; const double f = a[i * n + k]; for (int j = k + 1; j < n; ++j) a[i * n + j] -= f * a[k * n + j]; }
    }
    for (int c = 0; c < n; ++c) {
        double y[15];
        for (int i = 0; i < n; ++i) { double s = (piv[i] == c) ? 1.0 : 0.0; for (int k = 0; k < i; ++k) s -= a[i * n + k] * y[k]; y[i] = s; }
        for (int i = n - 1; i >= 0; --i) { double s = y[i]; for (int k = i + 1; k < n; ++k) s -= a[i * n + k] * inv[k * n + c]; inv[i * n + c] = s / a[i * n + i]; }
    }
    if (prior_a >= 0.0 && prior_g >= 0.0)
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { inv[(9 + i) * n + 9 + j] = (i == j) ? prior_a : 0.0; inv[(12 + i) * n + 12 + j] = (i == j) ? prior_g : 0.0; }
    for (int i = 0; i < 225; ++i) L[i] = 0.0;
    for (int j = 0; j < n; ++j) {
        double d = inv[j * n + j];
        for (int k = 0; k < j; ++k) d -= L[j * n + k] * L[j * n + k];
        if (d != d) return false;
        if (d <= 0.0) { for (int c = j; c < n; ++c) for (int i = c; i < n; ++i) L[i * n + c] = inv[i * n + c]; break; }
        L[j * n + j] = std::sqrt(d);
        for (int i = j + 1; i < n; ++i) { double s = inv[i * n + j]; for (int k = 0; k < j; ++k) s -= L[i * n + k] * L[j * n + k]; L[i * n + j] = s / L[j * n + j]; }
    }
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) U[i * n + j] = L[j * n + i];
    return true;
}

}  // namespace host
}  // namespace lvb
