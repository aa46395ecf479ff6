// tests/cpp/map_to_world_shim.cpp -- Mapping::ToWorld(double start) after a correction (mapping.cpp:222-229, called from
// Backend::GlobalLoop and Relocator::CorrectLoop) through the C++ shim (include/lvio_b200/association.h), two ways: mode 0 re-stores
// every lidar keyframe with AppendKeyframe, as the reference's per-frame ToWorld does; mode 1 hands all of them to ToWorldKeyframes
// (one device call for the keyframes already stored).  The run around it: keyframes through OptimizeKeyframe(frame, keys, ...), a
// correction applied to every pose from some keyframe on (as PoseGraph::ForwardUpdate does), the re-anchoring over a range that holds
// a lidar keyframe never stored and a frame without lidar, further keyframes, then RelocateKeyframe.  Compiled as C++14 against
// liblvio_b200.so by tests/test_gpu_map_to_world.py.
//   in.bin : int32 K, double visual weight, int32 features_left
//            per frame: double pose[7], int32 has_lidar, cloud ground, cloud surf (robot frame); cloud = int32 n, float n x 4
//            int32 n_first (frames 0 .. n_first-1 are registered before the correction), int32 from (the correction moves frames
//            from .. n_first), double correction[7] (pose = correction * pose)
//            int32 n_keys, int64 keys[n_keys], int32 old (the old keyframe), double guess[7] (the world pose the relocation starts
//            from), double ground_threshold; the last frame is the relocated one
//   out.bin: double pose[7] per frame, the relocation's score, its relative_o_c[7], the host synchronisations of the re-anchoring
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
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

// Sophus SE3 product and inverse in the layout [qx qy qz qw tx ty tz]
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

typedef std::shared_ptr<Frame> FramePtr;

// Mapping::Optimize's loop body for frame k (mapping.cpp:114-185): the map frame of the last (up to) three lidar keyframes before it
static bool optimize(lvio_fusion::FeatureAssociation& fa, const std::vector<FramePtr>& frames, int k, double thr) {
    if (!frames[k]->feature_lidar) return true;                  // mapping.cpp: `if (!pair.second->feature_lidar) continue;`
    long long keys[3]; int n = 0;
    for (int j = k - 1; j >= 0 && n < 3; --j) if (frames[j]->feature_lidar) keys[n++] = j;
    std::reverse(keys, keys + n);                                 // merge order: oldest first
    Pose map_pose = {{0, 0, 0, 1, 0, 0, 0}};
    if (n) map_pose = frames[keys[n - 1]]->pose;
    if (!fa.OptimizeKeyframe(frames[k], keys, n, map_pose.data(), k, thr)) { std::fprintf(stderr, "keyframe %d: %s\n", k, lvb_last_error()); return false; }
    return true;
}

int main(int argc, char** argv) {
    if (argc != 4) { std::fprintf(stderr, "usage: map_to_world_shim in.bin out.bin mode\n"); return 1; }
    const int mode = std::atoi(argv[3]);
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 1;
    int K = 0, n_feat = 0; double visual = 0;
    if (!rd(f, &K, 1) || !rd(f, &visual, 1) || !rd(f, &n_feat, 1)) return 1;
    std::vector<FramePtr> frames;
    for (int k = 0; k < K; ++k) {
        auto fr = std::make_shared<Frame>();
        fr->weights.visual = visual; fr->features_left.resize(n_feat);
        auto lf = std::make_shared<LidarFeature>();
        int has_lidar = 0;
        if (!rd(f, fr->pose.d, 7) || !rd(f, &has_lidar, 1) || !rd_cloud(f, lf->points_ground) || !rd_cloud(f, lf->points_surf)) return 1;
        if (has_lidar) fr->feature_lidar = lf;
        frames.push_back(fr);
    }
    int n_first = 0, from = 0, n_keys = 0, old = 0;
    Pose correction, guess;
    long long rkeys[3];
    double thr = 0;
    if (!rd(f, &n_first, 1) || !rd(f, &from, 1) || !rd(f, correction.d, 7) || !rd(f, &n_keys, 1) || n_keys < 1 || n_keys > 3 ||
        !rd(f, rkeys, n_keys) || !rd(f, &old, 1) || !rd(f, guess.d, 7) || !rd(f, &thr, 1)) return 1;
    std::fclose(f);
    if (n_first >= K - 1 || from > n_first) return 1;

    lvio_fusion::FeatureAssociation fa(0.2);                     // kitti.yaml:45
    for (int k = 0; k < n_first; ++k) if (!optimize(fa, frames, k, thr)) return 2;
    // the correction, as PoseGraph::ForwardUpdate applies it to every frame after a time
    for (int k = from; k <= n_first; ++k) frames[k]->pose = mul(correction, frames[k]->pose);
    // Mapping::ToWorld(start): frames from .. n_first, frame n_first a lidar keyframe not stored yet
    lvb_ctx* ctx = lvb::Runtime::get().ctx;
    const long long s0 = lvb_sync_count(ctx);
    if (mode == 0) {
        for (int k = from; k <= n_first; ++k) {
            if (!frames[k]->feature_lidar) continue;
            if (!fa.AppendKeyframe(k, frames[k]->feature_lidar->points_ground, frames[k]->feature_lidar->points_surf, frames[k]->pose.d)) {
                std::fprintf(stderr, "append %d: %s\n", k, lvb_last_error()); return 2; }
        }
    } else {
        std::vector<long long> keys;
        std::vector<FramePtr> which;
        for (int k = n_first; k >= from; --k) { keys.push_back(k); which.push_back(frames[k]); }      // any order
        if (!fa.ToWorldKeyframes(keys.data(), which.data(), (int)keys.size())) { std::fprintf(stderr, "to_world: %s\n", lvb_last_error()); return 2; }
    }
    const long long syncs = lvb_sync_count(ctx) - s0;
    for (int k = n_first; k < K - 1; ++k) if (!optimize(fa, frames, k, thr)) return 2;
    Pose rel = mul(inv(frames[old]->pose), guess);
    const int score = fa.RelocateKeyframe(frames[K - 1], rkeys, n_keys, frames[rkeys[0]]->pose.data(), frames[old]->pose.data(), rel, thr);

    std::vector<double> out;
    for (auto& fr : frames) out.insert(out.end(), fr->pose.d, fr->pose.d + 7);
    out.push_back(score);
    out.insert(out.end(), rel.d, rel.d + 7);
    out.push_back((double)syncs);
    f = std::fopen(argv[2], "wb");
    if (!f) return 1;
    std::fwrite(out.data(), sizeof(double), out.size(), f);
    std::fclose(f);
    return 0;
}
