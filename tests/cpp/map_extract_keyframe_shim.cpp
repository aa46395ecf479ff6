// tests/cpp/map_extract_keyframe_shim.cpp -- FeatureAssociation::AddScan -> Process -> Mapping::Optimize through the C++ shim
// (include/lvio_b200/association.h, lidar_features.h) two ways on the same raw scans: the features extracted to the host
// (LidarFeatureExtractor::Process) and registered from frame->feature_lidar, and the features extracted into the resident map
// (FeatureAssociation::ExtractKeyframe) and registered by key.  Both ways run once as one OptimizeKeyframes pass and once as the
// per-keyframe OptimizeKeyframe(frame, keys, ...) loop with PoseGraph::ForwardUpdate replayed on the host.  Every keyframe's map frame
// is the (up to) three keyframes before it.  Writes the poses (4 x K x 7 doubles: pass host, pass by key, loop host, loop by key) and
// prints SAME FEATURES when ExtractKeyframe filled frame->feature_lidar with what Process returns.
// Input: K, visual weight, n_features_left, then per keyframe its incoming pose (7 doubles), n and n x (x y z intensity) float32.
// Compiled as C++14 against liblvio_b200.so by tests/test_gpu_map_extract_keyframe.py.
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>
#include "lvio_b200/association.h"
#include "lvio_b200/lidar_features.h"
#include "lvio_b200/se3.h"

struct Pt { float x, y, z, intensity; };
struct Pose { double d[7]; double* data() { return d; } const double* data() const { return d; } };
struct LidarFeature { std::vector<Pt> points_ground, points_surf; };
struct Weights { double visual = 0, lidar_ground = 1, lidar_surf = 0.01; };         // frame.cpp:13-15
struct Frame { Pose pose; std::shared_ptr<LidarFeature> feature_lidar; Weights weights; std::vector<int> features_left; };
typedef std::shared_ptr<Frame> FramePtr;

template <class T> static bool rd(FILE* f, T* p, size_t n) { return std::fread(p, sizeof(T), n, f) == n; }

static void forward_update(std::vector<FramePtr>& frames, int k, const double* T) {
    for (size_t j = k + 1; j < frames.size(); ++j) { double p[7]; lvb::se3::mul(T, frames[j]->pose.d, p); std::memcpy(frames[j]->pose.d, p, sizeof(p)); }
}
static bool same(const std::vector<Pt>& a, const std::vector<Pt>& b) {
    return a.size() == b.size() && (a.empty() || std::memcmp(a.data(), b.data(), a.size() * sizeof(Pt)) == 0);
}

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: map_extract_keyframe_shim in.bin out.bin\n"); return 1; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 1;
    int K = 0, n_feat = 0; double visual = 0;
    if (!rd(f, &K, 1) || !rd(f, &visual, 1) || !rd(f, &n_feat, 1)) return 1;
    std::vector<std::vector<Pt>> scans(K);
    std::vector<FramePtr> frames[4];                  // pass host, pass by key, loop host, loop by key
    for (int k = 0; k < K; ++k) {
        auto fr = std::make_shared<Frame>();
        fr->weights.visual = visual; fr->features_left.resize(n_feat + 37 * k);
        fr->weights.lidar_ground = 1.0 + 0.25 * k; fr->weights.lidar_surf = 0.01 * (1.0 + 0.5 * (k % 3));
        int n = 0;
        if (!rd(f, fr->pose.d, 7) || !rd(f, &n, 1)) return 1;
        scans[k].resize(n);
        if (!rd(f, scans[k].data(), n)) return 1;
        for (auto& v : frames) { auto c = std::make_shared<Frame>(*fr); c->feature_lidar = std::make_shared<LidarFeature>(); v.push_back(c); }
    }
    std::fclose(f);
    std::vector<long long> keys(K), map_keys(3 * K);
    std::vector<int> n_map(K);
    for (int k = 0; k < K; ++k) {
        keys[k] = k;
        for (int j = k - 3; j < k; ++j) if (j >= 0) map_keys[3 * k + n_map[k]++] = j;
    }
    lvb::LidarFeatureExtractor ex(64, 1800, 0.427, 24.9, 60, 0.1036, 5, 30, 0.2);      // kitti.yaml:35-45
    lvio_fusion::FeatureAssociation fa[4] = {lvio_fusion::FeatureAssociation(0.2), lvio_fusion::FeatureAssociation(0.2),
                                             lvio_fusion::FeatureAssociation(0.2), lvio_fusion::FeatureAssociation(0.2)};
    bool same_features = true;
    for (int v = 0; v < 4; ++v) {
        fa[v].SetLidarConfig(ex.config());
        for (int k = 0; k < K; ++k) {
            LidarFeature& lf = *frames[v][k]->feature_lidar;
            const bool ok = (v & 1) ? fa[v].ExtractKeyframe(keys[k], scans[k], frames[v][k]) : ex.Process(scans[k], lf.points_ground, lf.points_surf);
            if (!ok) { std::fprintf(stderr, "extract %d/%d: %s\n", v, k, lvb_last_error()); return 2; }
            if (!(v & 1)) continue;
            const LidarFeature& host = *frames[v - 1][k]->feature_lidar;
            if (!same(lf.points_ground, host.points_ground) || !same(lf.points_surf, host.points_surf)) {
                same_features = false;
                std::printf("features differ: way %d keyframe %d: ground %zu / %zu, surf %zu / %zu points\n", v, k, lf.points_ground.size(),
                            host.points_ground.size(), lf.points_surf.size(), host.points_surf.size());
            }
        }
    }
    // one pass per way: no resident map keys, so every map pose comes from the call
    std::vector<double> map_poses(7 * K, 0.0), poses(7 * K), Ts(7 * K);
    for (int k = 0; k < K; ++k) map_poses[7 * k + 3] = 1.0;
    for (int v = 0; v < 2; ++v) {
        if (!fa[v].OptimizeKeyframes(frames[v].data(), keys.data(), map_keys.data(), n_map.data(), map_poses.data(), K, 0.05, poses.data(), Ts.data())) {
            std::fprintf(stderr, "pass %d: %s\n", v, lvb_last_error()); return 2; }
        for (int k = 0; k < K; ++k) forward_update(frames[v], k, &Ts[7 * k]);
        for (int k = 0; k < K; ++k) std::memcpy(frames[v][k]->pose.d, &poses[7 * k], 7 * sizeof(double));
    }
    // the per-keyframe loop per way
    for (int v = 2; v < 4; ++v) {
        std::vector<FramePtr>& fr = frames[v];
        for (int k = 0; k < K; ++k) {
            double old[7];
            std::memcpy(old, fr[k]->pose.d, sizeof(old));
            Pose map_pose = {{0, 0, 0, 1, 0, 0, 0}};
            if (n_map[k]) map_pose = fr[map_keys[3 * k + n_map[k] - 1]]->pose;
            if (!fa[v].OptimizeKeyframe(fr[k], &map_keys[3 * k], n_map[k], map_pose.data(), keys[k], 0.05)) {
                std::fprintf(stderr, "loop %d keyframe %d: %s\n", v, k, lvb_last_error()); return 2; }
            double inv[7], T[7];
            lvb::se3::inv(old, inv);
            lvb::se3::mul(fr[k]->pose.d, inv, T);
            forward_update(fr, k, T);
        }
    }
    std::vector<double> out;
    for (auto& v : frames) for (auto& fr : v) out.insert(out.end(), fr->pose.d, fr->pose.d + 7);
    f = std::fopen(argv[2], "wb");
    if (!f) return 1;
    std::fwrite(out.data(), sizeof(double), out.size(), f);
    std::fclose(f);
    if (same_features) std::printf("SAME FEATURES\n");
    return 0;
}
