// tests/cpp/map_build_optimize_shim.cpp -- Mapping::Optimize's loop (mapping.cpp:139-191) through the C++ shim's one-call member
// (include/lvio_b200/association.h, OptimizeKeyframe(frame, keys, n_keys, ...)): per keyframe the map frame of the last (up to) three
// keyframes -- none for the first -- is built and registered against in one call, then the keyframe that left the window is evicted.
// Same input and output files as tests/cpp/map_optimize_shim.cpp, which runs the BuildMapFrame + OptimizeKeyframe loop; compiled as
// C++14 against liblvio_b200.so by tests/test_gpu_map_build_keyframe.py.
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

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: map_build_optimize_shim in.bin out.bin\n"); return 1; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 1;
    int K = 0, n_feat = 0; double visual = 0;
    if (!rd(f, &K, 1) || !rd(f, &visual, 1) || !rd(f, &n_feat, 1)) return 1;
    std::vector<std::shared_ptr<Frame>> frames;
    for (int k = 0; k < K; ++k) {
        auto fr = std::make_shared<Frame>();
        fr->feature_lidar = std::make_shared<LidarFeature>();
        fr->weights.visual = visual; fr->features_left.resize(n_feat);
        int n = 0;
        if (!rd(f, fr->pose.d, 7) || !rd(f, &n, 1)) return 1;
        fr->feature_lidar->points_ground.resize(n);
        if (!rd(f, fr->feature_lidar->points_ground.data(), n) || !rd(f, &n, 1)) return 1;
        fr->feature_lidar->points_surf.resize(n);
        if (!rd(f, fr->feature_lidar->points_surf.data(), n)) return 1;
        frames.push_back(fr);
    }
    std::fclose(f);
    lvio_fusion::FeatureAssociation fa(0.2);                 // kitti.yaml:45
    std::vector<double> out;
    for (int k = 0; k < K; ++k) {
        long long keys[3]; int n = 0;
        for (int j = k - 3; j < k; ++j) if (j >= 0) keys[n++] = j;
        Pose map_pose = {{0, 0, 0, 1, 0, 0, 0}};             // map_frame->pose = the newest merged keyframe's (mapping.cpp:131-133)
        if (n) map_pose = frames[keys[n - 1]]->pose;
        lvb_solve_summary sums[2];
        if (!fa.OptimizeKeyframe(frames[k], keys, n, map_pose.data(), k, -1.0, sums)) { std::fprintf(stderr, "keyframe %d: %s\n", k, lvb_last_error()); return 2; }
        if (k >= 3 && !fa.EvictKeyframe(k - 3)) return 2;
        out.insert(out.end(), frames[k]->pose.d, frames[k]->pose.d + 7);
        out.push_back(sums[0].termination_type); out.push_back(sums[1].termination_type);
    }
    f = std::fopen(argv[2], "wb");
    if (!f) return 1;
    std::fwrite(out.data(), sizeof(double), out.size(), f);
    std::fclose(f);
    return 0;
}
