// tests/cpp/relocate_shim.cpp -- Mapping::Relocate for one loop-closure candidate (mapping.cpp:251-300) two ways through the C++ shim
// (include/lvio_b200/association.h): the reference's own sequence -- four rounds of ScanToMapWithGround / ScanToMapWithSegmented with
// relocate = true and ceres::Solve (DENSE_QR, 4 iterations) against host map clouds, the poses composed on the host -- and
// RelocateKeyframe against the keyframe clouds kept on the device by AppendKeyframe.  Compiled as C++14 against liblvio_b200.so by
// tests/test_gpu_map_relocate.py.
//   in.bin : int32 K, then per keyframe: double pose[7], cloud ground, cloud surf (robot frame)
//            int32 n_keys, int64 keys[n_keys], double map_pose[7], old_pose[7], relative_guess[7], ground_threshold
//            the current frame: cloud ground, cloud surf (robot frame); the old map frame: cloud ground, cloud surf (world frame)
//            cloud = int32 n, float n x 4 (x y z intensity)
//   out.bin: double relative_o_c[7], score of the reference's sequence; relative_o_c[7], score of RelocateKeyframe
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>
#include "lvio_b200/association.h"

struct Pt { float x, y, z, intensity; };
struct Pose { double d[7]; double* data() { return d; } const double* data() const { return d; } };
struct LidarFeature { std::vector<Pt> points_ground, points_surf; };
struct Weights { double visual = 0, lidar_ground = 1, lidar_surf = 0.01; };         // frame.cpp:13-15
struct Frame { Pose pose; std::shared_ptr<LidarFeature> feature_lidar; Weights weights; std::vector<int> features_left; };

template <class T> static bool rd(FILE* f, T* p, size_t n) { return std::fread(p, sizeof(T), n, f) == n; }
static bool rd_cloud(FILE* f, std::vector<Pt>& c) { int n = 0; if (!rd(f, &n, 1)) return false; c.resize(n); return rd(f, c.data(), n); }

// Sophus SE3 arithmetic in the layout [qx qy qz qw tx ty tz], and utility.cpp's se32rpyxyz / rpyxyz2se3
static void rotate(const double* q, const double* p, double* out) {
    const double uv[3] = {2 * (q[1] * p[2] - q[2] * p[1]), 2 * (q[2] * p[0] - q[0] * p[2]), 2 * (q[0] * p[1] - q[1] * p[0])};
    const double c[3] = {q[1] * uv[2] - q[2] * uv[1], q[2] * uv[0] - q[0] * uv[2], q[0] * uv[1] - q[1] * uv[0]};
    for (int k = 0; k < 3; ++k) out[k] = p[k] + q[3] * uv[k] + c[k];
}
static Pose mul(const Pose& A, const Pose& B) {
    const double* a = A.d; const double* b = B.d;
    Pose c;
    c.d[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    c.d[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    c.d[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    c.d[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
    const double n = std::sqrt(c.d[0] * c.d[0] + c.d[1] * c.d[1] + c.d[2] * c.d[2] + c.d[3] * c.d[3]);
    for (int k = 0; k < 4; ++k) c.d[k] /= n;
    double t[3];
    rotate(a, b + 4, t);
    for (int k = 0; k < 3; ++k) c.d[4 + k] = a[4 + k] + t[k];
    return c;
}
static Pose inv(const Pose& A) {
    Pose c;
    c.d[0] = -A.d[0]; c.d[1] = -A.d[1]; c.d[2] = -A.d[2]; c.d[3] = A.d[3];
    const double mt[3] = {-A.d[4], -A.d[5], -A.d[6]};
    rotate(c.d, mt, c.d + 4);
    return c;
}
static void se32rpyxyz(const Pose& T, double* e) {
    const double q0 = T.d[3], q1 = T.d[0], q2 = T.d[1], q3 = T.d[2];
    e[0] = std::atan2(2 * (q1 * q2 + q0 * q3), 1 - 2 * (q2 * q2 + q3 * q3));
    e[1] = std::asin(2 * (q0 * q2 - q1 * q3));
    e[2] = std::atan2(2 * (q2 * q3 + q0 * q1), 1 - 2 * (q1 * q1 + q2 * q2));
    e[3] = T.d[4]; e[4] = T.d[5]; e[5] = T.d[6];
}
static Pose rpyxyz2se3(const double* e) {
    const double cz = std::cos(e[0] / 2), sz = std::sin(e[0] / 2), cy = std::cos(e[1] / 2), sy = std::sin(e[1] / 2);
    const double cx = std::cos(e[2] / 2), sx = std::sin(e[2] / 2);
    Pose T;
    T.d[3] = cz * cy * cx + sz * sy * sx; T.d[0] = cz * cy * sx - sz * sy * cx;
    T.d[1] = cz * sy * cx + sz * cy * sx; T.d[2] = sz * cy * cx - cz * sy * sx;
    const double n = std::sqrt(T.d[0] * T.d[0] + T.d[1] * T.d[1] + T.d[2] * T.d[2] + T.d[3] * T.d[3]);
    for (int k = 0; k < 4; ++k) T.d[k] /= n;
    T.d[4] = e[3]; T.d[5] = e[4]; T.d[6] = e[5];
    return T;
}

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: relocate_shim in.bin out.bin\n"); return 1; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 1;
    int K = 0;
    if (!rd(f, &K, 1)) return 1;
    std::vector<std::shared_ptr<Frame>> kfs;
    for (int k = 0; k < K; ++k) {
        auto fr = std::make_shared<Frame>();
        fr->feature_lidar = std::make_shared<LidarFeature>();
        if (!rd(f, fr->pose.d, 7) || !rd_cloud(f, fr->feature_lidar->points_ground) || !rd_cloud(f, fr->feature_lidar->points_surf)) return 1;
        kfs.push_back(fr);
    }
    int n_keys = 0;
    long long keys[3];
    Pose map_pose, old_pose, guess;
    double thr = 0;
    auto cur = std::make_shared<Frame>();
    cur->feature_lidar = std::make_shared<LidarFeature>();
    auto map_frame = std::make_shared<Frame>();
    map_frame->feature_lidar = std::make_shared<LidarFeature>();
    if (!rd(f, &n_keys, 1) || n_keys < 1 || n_keys > 3 || !rd(f, keys, n_keys) || !rd(f, map_pose.d, 7) || !rd(f, old_pose.d, 7) ||
        !rd(f, guess.d, 7) || !rd(f, &thr, 1) || !rd_cloud(f, cur->feature_lidar->points_ground) || !rd_cloud(f, cur->feature_lidar->points_surf) ||
        !rd_cloud(f, map_frame->feature_lidar->points_ground) || !rd_cloud(f, map_frame->feature_lidar->points_surf)) return 1;
    std::fclose(f);
    map_frame->pose = map_pose;

    // mapping.cpp:251-300 as the reference writes it, the shim serving ScanToMapWith* and ceres::Solve
    lvio_fusion::FeatureAssociation per_call(0.2);           // kitti.yaml:45
    auto clone = std::make_shared<Frame>(*cur);
    clone->pose = mul(old_pose, guess);
    double score_ground = NAN, score_surf = NAN;
    for (int i = 0; i < 4; ++i) {
        double rpyxyz[6];
        se32rpyxyz(mul(inv(map_frame->pose), clone->pose), rpyxyz);
        ceres::Solver::Options options;
        options.linear_solver_type = ceres::DENSE_QR;
        options.max_num_iterations = 4;
        if (!map_frame->feature_lidar->points_ground.empty()) {
            ceres::Problem problem;
            if (!per_call.ScanToMapWithGround(clone, map_frame, rpyxyz, problem, true)) { std::fprintf(stderr, "ground: %s\n", lvb_last_error()); return 2; }
            ceres::Solver::Summary summary;
            ceres::Solve(options, &problem, &summary);
            clone->pose = mul(map_frame->pose, rpyxyz2se3(rpyxyz));
            score_ground = std::min((double)summary.num_residual_blocks_reduced / 10, 20.0);
            score_ground -= 2 * summary.final_cost / summary.num_residual_blocks_reduced;
        }
        if (!map_frame->feature_lidar->points_surf.empty()) {
            ceres::Problem problem;
            if (!per_call.ScanToMapWithSegmented(clone, map_frame, rpyxyz, problem, true)) { std::fprintf(stderr, "surf: %s\n", lvb_last_error()); return 2; }
            ceres::Solver::Summary summary;
            ceres::Solve(options, &problem, &summary);
            clone->pose = mul(map_frame->pose, rpyxyz2se3(rpyxyz));
            score_surf = std::min((double)summary.num_residual_blocks_reduced / 10, 30.0);
            score_surf -= 2 * summary.final_cost / summary.num_residual_blocks_reduced;
        }
    }
    const Pose rel_ref = mul(inv(old_pose), clone->pose);
    const double sum = score_ground + score_surf;
    const int score_ref = std::isfinite(sum) ? (int)sum : 0;            // RelocateKeyframe's documented reading of a missing score

    // the resident path: the keyframes' clouds on the device, one call
    lvio_fusion::FeatureAssociation resident(0.2);
    for (int k = 0; k < K; ++k)
        if (!resident.AppendKeyframe(k, kfs[k]->feature_lidar->points_ground, kfs[k]->feature_lidar->points_surf, kfs[k]->pose.d)) {
            std::fprintf(stderr, "append %d: %s\n", k, lvb_last_error()); return 2; }
    Pose rel = guess;
    const int score = resident.RelocateKeyframe(cur, keys, n_keys, map_pose.data(), old_pose.data(), rel, thr);

    std::vector<double> out(rel_ref.d, rel_ref.d + 7);
    out.push_back(score_ref);
    out.insert(out.end(), rel.d, rel.d + 7);
    out.push_back(score);
    f = std::fopen(argv[2], "wb");
    if (!f) return 1;
    std::fwrite(out.data(), sizeof(double), out.size(), f);
    std::fclose(f);
    return 0;
}
