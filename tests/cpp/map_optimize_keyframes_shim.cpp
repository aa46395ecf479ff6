// tests/cpp/map_optimize_keyframes_shim.cpp -- a Mapping::Optimize(active_kfs)-shaped pass (mapping.cpp:139-191) through the C++ shim
// (include/lvio_b200/association.h) two ways on the same frames: per keyframe OptimizeKeyframe(frame, keys, ...) with
// PoseGraph::ForwardUpdate replayed on the host after each, and one OptimizeKeyframes call followed by the ForwardUpdate replay and the
// optimised poses written last (INTEGRATION.md 3a).  Every frame is a lidar keyframe of the pass; its map frame is the (up to) three
// keyframes before it, and each frame has its own feature count and lidar weights (so its own prior weight).  Writes both paths' poses
// (2 x K x 7 doubles) and prints SAME CLOUDS when a probe registration against the last three stored keyframes gives the same pose
// (to 1e-11) on both.  Input file as tests/cpp/map_build_optimize_shim.cpp's; compiled as C++14
// against liblvio_b200.so by tests/test_gpu_map_optimize_keyframes.py.
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>
#include "lvio_b200/association.h"
#include "lvio_b200/se3.h"

struct Pt { float x, y, z, intensity; };
struct Pose { double d[7]; double* data() { return d; } const double* data() const { return d; } };
struct LidarFeature { std::vector<Pt> points_ground, points_surf; };
struct Weights { double visual = 0, lidar_ground = 1, lidar_surf = 0.01; };         // frame.cpp:13-15
struct Frame { Pose pose; std::shared_ptr<LidarFeature> feature_lidar; Weights weights; std::vector<int> features_left; };
typedef std::shared_ptr<Frame> FramePtr;

template <class T> static bool rd(FILE* f, T* p, size_t n) { return std::fread(p, sizeof(T), n, f) == n; }

// PoseGraph::ForwardUpdate(T, t_k + epsilon): every frame after k, pose = T * pose
static void forward_update(std::vector<FramePtr>& frames, int k, const double* T) {
    for (size_t j = k + 1; j < frames.size(); ++j) { double p[7]; lvb::se3::mul(T, frames[j]->pose.d, p); std::memcpy(frames[j]->pose.d, p, sizeof(p)); }
}

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: map_optimize_keyframes_shim in.bin out.bin\n"); return 1; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 1;
    int K = 0, n_feat = 0; double visual = 0;
    if (!rd(f, &K, 1) || !rd(f, &visual, 1) || !rd(f, &n_feat, 1)) return 1;
    std::vector<FramePtr> a, b;
    for (int k = 0; k < K; ++k) {
        auto fr = std::make_shared<Frame>();
        fr->feature_lidar = std::make_shared<LidarFeature>();
        // each keyframe its own prior weight (features_left.size() * weights.visual) and lidar weights, as real keyframes have
        fr->weights.visual = visual; fr->features_left.resize(n_feat + 37 * k);
        fr->weights.lidar_ground = 1.0 + 0.25 * k; fr->weights.lidar_surf = 0.01 * (1.0 + 0.5 * (k % 3));
        int n = 0;
        if (!rd(f, fr->pose.d, 7) || !rd(f, &n, 1)) return 1;
        fr->feature_lidar->points_ground.resize(n);
        if (!rd(f, fr->feature_lidar->points_ground.data(), n) || !rd(f, &n, 1)) return 1;
        fr->feature_lidar->points_surf.resize(n);
        if (!rd(f, fr->feature_lidar->points_surf.data(), n)) return 1;
        a.push_back(fr);
        auto copy = std::make_shared<Frame>(*fr);
        b.push_back(copy);
    }
    std::fclose(f);
    std::vector<long long> keys(K), map_keys(3 * K);
    std::vector<int> n_map(K);
    for (int k = 0; k < K; ++k) {
        keys[k] = k;
        for (int j = k - 3; j < k; ++j) if (j >= 0) map_keys[3 * k + n_map[k]++] = j;
    }
    lvio_fusion::FeatureAssociation fa(0.2), fb(0.2);               // kitti.yaml:45
    // per keyframe: build + optimise, then ForwardUpdate of the later frames
    for (int k = 0; k < K; ++k) {
        const double old[7] = {a[k]->pose.d[0], a[k]->pose.d[1], a[k]->pose.d[2], a[k]->pose.d[3], a[k]->pose.d[4], a[k]->pose.d[5], a[k]->pose.d[6]};
        Pose map_pose = {{0, 0, 0, 1, 0, 0, 0}};
        if (n_map[k]) map_pose = a[map_keys[3 * k + n_map[k] - 1]]->pose;
        if (!fa.OptimizeKeyframe(a[k], &map_keys[3 * k], n_map[k], map_pose.data(), keys[k], -1.0)) { std::fprintf(stderr, "keyframe %d: %s\n", k, lvb_last_error()); return 2; }
        double inv[7], T[7];
        lvb::se3::inv(old, inv);
        lvb::se3::mul(a[k]->pose.d, inv, T);
        forward_update(a, k, T);
    }
    // one call: map poses of resident keys only (none here), then the replay and the optimised poses written last
    std::vector<double> map_poses(7 * K, 0.0), poses(7 * K), Ts(7 * K);
    for (int k = 0; k < K; ++k) map_poses[7 * k + 3] = 1.0;
    if (!fb.OptimizeKeyframes(b.data(), keys.data(), map_keys.data(), n_map.data(), map_poses.data(), K, -1.0, poses.data(), Ts.data())) {
        std::fprintf(stderr, "chain: %s\n", lvb_last_error()); return 2; }
    for (int k = 0; k < K; ++k) forward_update(b, k, &Ts[7 * k]);
    for (int k = 0; k < K; ++k) std::memcpy(b[k]->pose.d, &poses[7 * k], 7 * sizeof(double));
    // a probe registration against the last three stored keyframes of each path
    Frame pa = *a[K - 1], pb = *b[K - 1];
    FramePtr qa = std::make_shared<Frame>(pa), qb = std::make_shared<Frame>(pb);
    std::memcpy(qb->pose.d, qa->pose.d, sizeof(qa->pose.d));
    const long long last3[3] = {K - 3, K - 2, K - 1};
    if (!fa.OptimizeKeyframe(qa, last3, 3, a[K - 1]->pose.data(), 1000, -1.0) ||
        !fb.OptimizeKeyframe(qb, last3, 3, a[K - 1]->pose.data(), 1000, -1.0)) { std::fprintf(stderr, "probe: %s\n", lvb_last_error()); return 2; }
    std::vector<double> out;
    for (auto* v : {&a, &b}) for (auto& fr : *v) out.insert(out.end(), fr->pose.d, fr->pose.d + 7);
    f = std::fopen(argv[2], "wb");
    if (!f) return 1;
    std::fwrite(out.data(), sizeof(double), out.size(), f);
    std::fclose(f);
    double d = 0;
    for (int i = 0; i < 7; ++i) d = std::max(d, std::fabs(qa->pose.d[i] - qb->pose.d[i]));
    std::printf("probe pose difference %.3g\n", d);
    if (d < 1e-11) std::printf("SAME CLOUDS\n");
    return 0;
}
