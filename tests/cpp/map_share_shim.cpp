// tests/cpp/map_share_shim.cpp -- the three threads of the reference that reach the resident keyframe clouds, through the C++ shim
// (include/lvio_b200/association.h) on one FeatureAssociation: the mapping thread (Mapping::Optimize -> OptimizeKeyframes), the
// Relocator (Mapping::Relocate -> RelocateKeyframe, once per candidate) and the lidar callback (FeatureAssociation::Process ->
// ExtractKeyframe), each a std::thread with its own context.  Mode "free" runs them without a lock, as the reference does; mode "locked"
// runs every call under one mutex (in whichever order the threads take it); mode "after" starts the Relocator's and the lidar thread's
// calls once the mapping pass has returned.  All must give the same poses, relative poses, integer scores and feature counts.  The
// mapping thread keeps the resident pair and its context, so it stays alive until the other threads are done, as the reference's
// mapping thread outlives the Relocator's and the lidar callback's calls.  Compiled as C++14 against liblvio_b200.so by
// tests/test_gpu_map_share_shim.py.
//   in.bin : int32 K, then per resident keyframe: double pose[7], cloud ground, cloud surf (robot frame)
//            int32 M, then per keyframe of the mapping pass: double pose[7], cloud ground, cloud surf (robot frame)
//            double old_pose[7], relative_guess[7]; the candidate: cloud ground, cloud surf (robot frame); the lidar scan: cloud
//            cloud = int32 n, float n x 4 (x y z intensity)
//   out.bin: M x 7 optimised poses; R x (7 relative_o_c + 1 score); E x 2 feature counts
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include "lvio_b200/association.h"

struct Pt { float x, y, z, intensity; };
struct Pose { double d[7]; double* data() { return d; } const double* data() const { return d; } };
struct LidarFeature { std::vector<Pt> points_ground, points_surf; };
struct Weights { double visual = 0, lidar_ground = 1, lidar_surf = 0.01; };         // frame.cpp:13-15
struct Frame { Pose pose; std::shared_ptr<LidarFeature> feature_lidar; Weights weights; std::vector<int> features_left; };

template <class T> static bool rd(FILE* f, T* p, size_t n) { return std::fread(p, sizeof(T), n, f) == n; }
static bool rd_cloud(FILE* f, std::vector<Pt>& c) { int n = 0; if (!rd(f, &n, 1)) return false; c.resize(n); return rd(f, c.data(), n); }
static bool rd_frames(FILE* f, std::vector<std::shared_ptr<Frame>>& out) {
    int n = 0;
    if (!rd(f, &n, 1)) return false;
    for (int k = 0; k < n; ++k) {
        auto fr = std::make_shared<Frame>();
        fr->feature_lidar = std::make_shared<LidarFeature>();
        if (!rd(f, fr->pose.d, 7) || !rd_cloud(f, fr->feature_lidar->points_ground) || !rd_cloud(f, fr->feature_lidar->points_surf)) return false;
        out.push_back(fr);
    }
    return true;
}

enum { RELOCS = 8, EXTRACTS = 4 };

int main(int argc, char** argv) {
    if (argc != 4) { std::fprintf(stderr, "usage: map_share_shim free|locked|after in.bin out.bin\n"); return 1; }
    const std::string mode = argv[1];
    if (mode != "free" && mode != "locked" && mode != "after") { std::fprintf(stderr, "unknown mode %s\n", argv[1]); return 1; }
    const bool locked = mode == "locked";
    FILE* f = std::fopen(argv[2], "rb");
    if (!f) return 1;
    std::vector<std::shared_ptr<Frame>> res, pass;
    Pose old_pose, guess;
    auto cur = std::make_shared<Frame>();
    cur->feature_lidar = std::make_shared<LidarFeature>();
    std::vector<Pt> scan;
    if (!rd_frames(f, res) || !rd_frames(f, pass) || !rd(f, old_pose.d, 7) || !rd(f, guess.d, 7) ||
        !rd_cloud(f, cur->feature_lidar->points_ground) || !rd_cloud(f, cur->feature_lidar->points_surf) || !rd_cloud(f, scan)) return 1;
    std::fclose(f);
    const int K = (int)res.size(), M = (int)pass.size();

    lvio_fusion::FeatureAssociation assoc(0.2);                 // kitti.yaml:45
    std::mutex big;                                             // mode "locked": every call under it
    auto guard = [&]() { return locked ? std::unique_lock<std::mutex>(big) : std::unique_lock<std::mutex>(); };
    std::vector<double> poses(7 * (size_t)M), relocs(8 * (size_t)RELOCS), counts(2 * (size_t)EXTRACTS);
    std::string err;
    std::mutex err_mu;
    auto fail = [&](const char* what) { std::lock_guard<std::mutex> lk(err_mu); err += std::string(what) + ": " + lvb_last_error() + "\n"; };
    // the mapping thread stores the resident keyframes first (it keeps them); the others start once it has (mode "after": once its pass
    // has returned), and it returns once they are done
    std::mutex state_mu;
    std::condition_variable state_cv;
    int stage = 0;                              // 1: keyframes stored, 2: pass returned
    int finished = 0;                           // Relocator and lidar threads done
    auto wait_for = [&](const std::function<bool()>& cond) { std::unique_lock<std::mutex> lk(state_mu); state_cv.wait(lk, cond); };
    auto update = [&](const std::function<void()>& fn) { { std::lock_guard<std::mutex> lk(state_mu); fn(); } state_cv.notify_all(); };
    auto wait_ready = [&]() { wait_for([&] { return stage >= (mode == "after" ? 2 : 1); }); };

    std::thread mapping([&]() {
        for (int k = 0; k < K; ++k)
            if (!assoc.AppendKeyframe(k, res[k]->feature_lidar->points_ground, res[k]->feature_lidar->points_surf, res[k]->pose.d)) fail("append");
        update([&] { stage = 1; });
        // Mapping::Optimize(active_kfs): keyframe K + j merges the three keyframes before it
        std::vector<long long> keys(M), map_keys(3 * (size_t)M);
        std::vector<int> n_map(M, 3);
        std::vector<double> map_poses(7 * (size_t)M);
        for (int j = 0; j < M; ++j) {
            keys[j] = K + j;
            for (int i = 0; i < 3; ++i) map_keys[3 * j + i] = K + j - 3 + i;
            std::memcpy(&map_poses[7 * j], res[K - 1]->pose.d, sizeof(res[K - 1]->pose.d));
        }
        {
            auto lk = guard();
            if (!assoc.OptimizeKeyframes(pass.data(), keys.data(), map_keys.data(), n_map.data(), map_poses.data(), M, 0.05, poses.data(), nullptr)) fail("optimize");
        }
        update([&] { stage = 2; });
        wait_for([&] { return finished == 2; });
    });
    std::thread relocator([&]() {
        wait_ready();
        const long long keys[3] = {0, 1, 2};
        for (int r = 0; r < RELOCS; ++r) {
            Pose rel = guess;
            auto lk = guard();
            const int score = assoc.RelocateKeyframe(cur, keys, 3, res[0]->pose.d, old_pose.d, rel, 0.05);
            if (!std::memcmp(rel.d, guess.d, sizeof(rel.d))) fail("relocate");          // a failed call leaves relative_o_c as it was
            std::memcpy(&relocs[8 * r], rel.d, sizeof(rel.d));
            relocs[8 * r + 7] = score;
        }
        update([&] { ++finished; });
    });
    std::thread lidar([&]() {
        wait_ready();
        for (int e = 0; e < EXTRACTS; ++e) {
            auto fr = std::make_shared<Frame>();
            fr->feature_lidar = std::make_shared<LidarFeature>();
            auto lk = guard();
            if (!assoc.ExtractKeyframe(1000 + e, scan, fr)) fail("extract");
            counts[2 * e] = (double)fr->feature_lidar->points_ground.size();
            counts[2 * e + 1] = (double)fr->feature_lidar->points_surf.size();
        }
        update([&] { ++finished; });
    });
    mapping.join(); relocator.join(); lidar.join();
    if (!err.empty()) { std::fprintf(stderr, "%s", err.c_str()); return 2; }
    f = std::fopen(argv[3], "wb");
    if (!f) return 1;
    std::fwrite(poses.data(), sizeof(double), poses.size(), f);
    std::fwrite(relocs.data(), sizeof(double), relocs.size(), f);
    std::fwrite(counts.data(), sizeof(double), counts.size(), f);
    std::fclose(f);
    return 0;
}
