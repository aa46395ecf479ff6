// tests/cpp/ctx_priority_shim.cpp -- the mapping, Relocator and lidar threads of the reference through the C++ shim
// (include/lvio_b200/association.h) on one FeatureAssociation, each thread setting its device priority first with
// lvb::Runtime::set_thread_priority, as an integration does where the thread starts: the mapping thread (Backend::BackendLoop ->
// Mapping::Optimize -> OptimizeKeyframes) at the greatest priority, the lidar callback (FeatureAssociation::Process -> ExtractKeyframe)
// one step lower, the Relocator (Mapping::Relocate -> RelocateKeyframe) at the default.  Mode "priority" runs them without a lock;
// mode "locked" runs every call under one mutex (in whichever order the threads take it).  Both must give the same poses, relative
// poses, integer scores and feature counts.  Each thread also checks, after its first device call, that its context runs at the
// priority it asked for (as CUDA clamps it) and that a second set_thread_priority is refused.  Compiled as C++14 against
// liblvio_b200.so by tests/test_gpu_ctx_priority.py.
//   in.bin : int32 K, then per resident keyframe: double pose[7], cloud ground, cloud surf (robot frame)
//            int32 M, then per keyframe of the mapping pass: double pose[7], cloud ground, cloud surf (robot frame)
//            double old_pose[7], relative_guess[7]; the candidate: cloud ground, cloud surf (robot frame); the lidar scan: cloud
//            cloud = int32 n, float n x 4 (x y z intensity)
//   out.bin: M x 7 optimised poses; R x (7 relative_o_c + 1 score); E x 2 feature counts
#include <algorithm>
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
    if (argc != 4) { std::fprintf(stderr, "usage: ctx_priority_shim priority|locked in.bin out.bin\n"); return 1; }
    const std::string mode = argv[1];
    if (mode != "priority" && mode != "locked") { std::fprintf(stderr, "unknown mode %s\n", argv[1]); return 1; }
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
    int least = 0, greatest = 0;
    if (lvb_device_priority_range(0, &least, &greatest) != LVB_OK) { std::fprintf(stderr, "range: %s\n", lvb_last_error()); return 2; }
    const int p_mapping = greatest, p_lidar = std::min(greatest + 1, least), p_relocator = 0;

    lvio_fusion::FeatureAssociation assoc(0.2);                 // kitti.yaml:45
    std::mutex big;                                             // mode "locked": every call under it
    auto guard = [&]() { return locked ? std::unique_lock<std::mutex>(big) : std::unique_lock<std::mutex>(); };
    std::vector<double> poses(7 * (size_t)M), relocs(8 * (size_t)RELOCS), counts(2 * (size_t)EXTRACTS);
    std::string err;
    std::mutex err_mu;
    auto fail = [&](const std::string& what) { std::lock_guard<std::mutex> lk(err_mu); err += what + ": " + lvb_last_error() + "\n"; };
    // the thread's priority, set where the thread starts
    auto start = [&](int p, const char* who) { if (!lvb::Runtime::get().set_thread_priority(p)) fail(std::string(who) + " set_thread_priority"); };
    // after the thread's first device call: its context runs at the priority it asked for, and a second request is refused
    auto check = [&](int want, const char* who) {
        lvb::Runtime& rt = lvb::Runtime::get();
        int got = 1 << 30;
        if (!rt.ctx || lvb_ctx_priority(rt.ctx, &got) != LVB_OK || got != want) fail(std::string(who) + " priority " + std::to_string(got));
        if (rt.set_thread_priority(least)) fail(std::string(who) + " late set_thread_priority accepted");
        else if (rt.error.find("already exists") == std::string::npos) fail(std::string(who) + " late set_thread_priority message: " + rt.error);
    };
    // the mapping thread stores the resident keyframes first (it keeps them); the others start once it has, and it returns once they
    // are done
    std::mutex state_mu;
    std::condition_variable state_cv;
    int stage = 0;                              // 1: keyframes stored
    int finished = 0;                           // Relocator and lidar threads done
    auto wait_for = [&](const std::function<bool()>& cond) { std::unique_lock<std::mutex> lk(state_mu); state_cv.wait(lk, cond); };
    auto update = [&](const std::function<void()>& fn) { { std::lock_guard<std::mutex> lk(state_mu); fn(); } state_cv.notify_all(); };

    std::thread mapping([&]() {
        start(p_mapping, "mapping");
        for (int k = 0; k < K; ++k)
            if (!assoc.AppendKeyframe(k, res[k]->feature_lidar->points_ground, res[k]->feature_lidar->points_surf, res[k]->pose.d)) fail("append");
        check(p_mapping, "mapping");
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
        wait_for([&] { return finished == 2; });
    });
    std::thread relocator([&]() {
        start(p_relocator, "relocator");
        wait_for([&] { return stage >= 1; });
        const long long keys[3] = {0, 1, 2};
        for (int r = 0; r < RELOCS; ++r) {
            Pose rel = guess;
            {
                auto lk = guard();
                const int score = assoc.RelocateKeyframe(cur, keys, 3, res[0]->pose.d, old_pose.d, rel, 0.05);
                if (!std::memcmp(rel.d, guess.d, sizeof(rel.d))) fail("relocate");          // a failed call leaves relative_o_c as it was
                std::memcpy(&relocs[8 * r], rel.d, sizeof(rel.d));
                relocs[8 * r + 7] = score;
            }
            if (r == 0) check(p_relocator, "relocator");
        }
        update([&] { ++finished; });
    });
    std::thread lidar([&]() {
        start(p_lidar, "lidar");
        wait_for([&] { return stage >= 1; });
        for (int e = 0; e < EXTRACTS; ++e) {
            auto fr = std::make_shared<Frame>();
            fr->feature_lidar = std::make_shared<LidarFeature>();
            {
                auto lk = guard();
                if (!assoc.ExtractKeyframe(1000 + e, scan, fr)) fail("extract");
                counts[2 * e] = (double)fr->feature_lidar->points_ground.size();
                counts[2 * e + 1] = (double)fr->feature_lidar->points_surf.size();
            }
            if (e == 0) check(p_lidar, "lidar");
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
