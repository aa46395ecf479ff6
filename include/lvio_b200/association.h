// include/lvio_b200/association.h -- scan-to-map registration with the call shape of
// lvio_fusion::FeatureAssociation::ScanToMapWithGround / ScanToMapWithSegmented
// (/root/reference/src/lvio_fusion/include/lvio_fusion/lidar/association.h:30-32, src/association.cpp:270-384).
//
// In the reference each call builds a pcl::KdTreeFLANN on the map cloud, searches 3 neighbours per scan point on
// the host and adds one LidarPlaneErrorRPZ/YXY residual block per accepted point; the caller then runs
// adapt::Solve (mapping.cpp:159-177).  Here the call uploads the map cloud once per call into the voxel hash,
// and adds ONE lvb::ScanToMapCost describing the whole association; ceres::Solve (ceres_shim.h) runs
// association + LM on the device and updates para[] in place.  Frame types are duck-typed:
//   frame->pose.data()                       Sophus::SE3d layout [qx qy qz qw tx ty tz]
//   frame->feature_lidar->points_ground / points_surf : contiguous clouds of 32-byte pcl::PointXYZI
//       (anything with .size() and .data() whose records start with float x, y, z)
//   frame->weights.lidar_ground / lidar_surf / visual,  frame->features_left.size()
#pragma once
#include <algorithm>
#include <atomic>
#include <cmath>
#include <mutex>
#include <type_traits>
#include <unordered_map>
#include <unordered_set>
#include <vector>
#include "ceres_shim.h"

// Inside the reference tree the class of the same name already exists (it also owns the feature extraction):
// compile with -DLVB_ASSOCIATION_CLASS=ScanToMapDevice and forward the two members to it (INTEGRATION.md section 3).
#ifndef LVB_ASSOCIATION_CLASS
#define LVB_ASSOCIATION_CLASS FeatureAssociation
#endif

namespace lvio_fusion {

namespace assoc_detail {
// first record of a cloud: pcl::PointCloud keeps its records in the public vector `points` (every PCL version; PCL >= 1.11
// also has data()); plain containers have data()
template <class Cloud> inline auto cloud_data(const Cloud& c, int) -> decltype(c.points.data()) { return c.points.data(); }
template <class Cloud> inline auto cloud_data(const Cloud& c, long) -> decltype(c.data()) { return c.data(); }
// adapt::Problem (adapt/problem.h:37-47) hides ceres::Problem::AddResidualBlock behind an overload that takes the block's
// ProblemType first and keeps a census of them; a plain ceres::Problem has no such census.  Use whichever the caller has:
// `lidar` selects ProblemType::LidarError, otherwise ProblemType::Other (association.cpp:318,324).
template <class P>
inline auto add_block(P& p, int, bool lidar, ceres::CostFunction* c, ceres::LossFunction* l, double* x0, double* x1, double* x2) -> decltype(p.num_types, void()) {
    typedef typename std::decay<decltype(p.num_types.begin()->first)>::type Type;
    p.AddResidualBlock(lidar ? Type::LidarError : Type::Other, c, l, x0, x1, x2);
}
template <class P>
inline void add_block(P& p, long, bool, ceres::CostFunction* c, ceres::LossFunction* l, double* x0, double* x1, double* x2) { p.AddResidualBlock(c, l, x0, x1, x2); }
}  // namespace assoc_detail

class LVB_ASSOCIATION_CLASS {
public:
    explicit LVB_ASSOCIATION_CLASS(double lidar_resolution = 0.2) : resolution_(lidar_resolution) {
        lvb_lidar_default_config(&lidar_cfg_);
        lidar_cfg_.resolution = lidar_resolution;
    }
    // the lidar configuration ExtractKeyframe uses (FeatureAssociation's constructor arguments, association.h:21-26; by default
    // kitti.yaml's with this object's resolution and an identity extrinsic), e.g. lvb::LidarFeatureExtractor::config()
    void SetLidarConfig(const lvb_lidar_config& cfg) { lidar_cfg_ = cfg; }

    // FeatureAssociation::AddScan -> Process (association.cpp:85-109) straight into the resident map (lvb_icp_map_extract_keyframe):
    // the scan's two feature clouds stay on the device as the pending features of `key`, and frame->feature_lidar->points_ground /
    // points_surf (which the caller has created; the Relocator and ToWorldKeyframes read them) receive the host copies.
    // OptimizeKeyframe(frame, keys, ...) and OptimizeKeyframes then register a pending key by key, with no upload; the other
    // OptimizeKeyframe overload uses the host copies and drops the pending features first.  Threading: it runs on the calling thread's
    // own handles over the resident store (StoreView), with no lock: the lidar callback extracts while the mapping thread registers
    // and the Relocator relocates (INTEGRATION.md 3a).  Before the mapping thread has stored a keyframe the features go to the calling
    // thread's own handles, and a keyframe call on other handles uses the host copies.  false: the call failed and changed nothing
    // (lvb_last_error()).
    template <class Cloud, class FramePtr>
    bool ExtractKeyframe(long long key, const Cloud& points, FramePtr frame) {
        StoreView h;
        if (!store_view(h)) return false;
        const size_t cap = (size_t)lidar_cfg_.num_scans * (size_t)lidar_cfg_.horizon_scan;
        extract_ground_.resize(cap); extract_surf_.resize(cap);
        int32_t ng = 0, ns = 0;
        const int stride = (int)sizeof(assoc_detail::cloud_data(points, 0)[0]);
        if (lvb_icp_map_extract_keyframe(h.ground, h.surf, &lidar_cfg_, key, assoc_detail::cloud_data(points, 0), (int)points.size(), stride, &ng, &ns,
                                         &extract_ground_[0].x, &extract_surf_[0].x) != LVB_OK)
            return false;
        unpack(extract_ground_, ng, frame->feature_lidar->points_ground);
        unpack(extract_surf_, ns, frame->feature_lidar->points_surf);
        std::lock_guard<std::mutex> lk(meta_);
        h.meta->pending.insert(key);
        return true;
    }
    ~LVB_ASSOCIATION_CLASS() {                      // the calling thread's handles; another thread's go with that thread's context
        for (auto* m : {&handles_of_thread(), &shared_of_thread()}) {
            auto it = m->find(this);
            if (it != m->end()) { if (it->second.ground) lvb_icp_destroy(it->second.ground); if (it->second.surf) lvb_icp_destroy(it->second.surf); m->erase(it); }
        }
    }

    // association.cpp:270-326 : pitch/roll/z = para+1,+2,+5 ; gate d2 < 100 res^2 ; TrivialLoss ; PoseErrorRPZ prior
    template <class FramePtr, class Problem>
    bool ScanToMapWithGround(FramePtr frame, FramePtr map_frame, double* para, Problem& problem, bool relocate = false) {
        return add(0, frame, map_frame, frame->feature_lidar->points_ground, map_frame->feature_lidar->points_ground, para, problem, relocate,
                   resolution_ * resolution_ * 100, frame->weights.lidar_ground, new ceres::TrivialLoss(), handles_of_thread()[this].ground);
    }
    // association.cpp:328-384 : yaw/x/y = para+0,+3,+4 ; gate d2 < 25 res^2 ; HuberLoss(0.1) ; PoseErrorYXY prior
    template <class FramePtr, class Problem>
    bool ScanToMapWithSegmented(FramePtr frame, FramePtr map_frame, double* para, Problem& problem, bool relocate = false) {
        return add(1, frame, map_frame, frame->feature_lidar->points_surf, map_frame->feature_lidar->points_surf, para, problem, relocate,
                   resolution_ * resolution_ * 25, frame->weights.lidar_surf, new ceres::HuberLoss(0.1), handles_of_thread()[this].surf);
    }

    // ---- device-resident map (INTEGRATION.md 3a).  Mapping::ToWorld (mapping.cpp:205-220) -> AppendKeyframe: the keyframe's two
    // robot-frame feature clouds go to the device once and stay there in the world frame; Mapping::BuildMapFrame (:114-137) ->
    // BuildMapFrame: merge of the given keyframes in order, SegmentGround on the merged ground cloud, voxel hash -- all on the
    // device.  After a BuildMapFrame the two ScanToMapWith* members register against that resident map frame and no longer upload
    // map_frame's clouds; UsePerCallMap() goes back to the per-call behaviour (Relocator::RelocateByPoints hands over its own map).
    template <class Cloud>
    bool AppendKeyframe(long long key, const Cloud& ground_robot, const Cloud& surf_robot, const double* pose7) {
        Handles& h = handles_of_thread()[this];
        if (!ensure_handles(h)) return false;
        resident_ = &h;
        return store_keyframe(h.ground, h.surf, h, key, ground_robot, surf_robot, pose7);
    }
    bool EvictKeyframe(long long key) {
        Handles& h = handles_of_thread()[this];
        if (!ensure_handles(h)) return false;
        {
            std::lock_guard<std::mutex> lk(meta_);
            if (key < 0) h.keys.clear(); else h.keys.erase(key);
        }
        return lvb_icp_map_evict(h.ground, key) == LVB_OK && lvb_icp_map_evict(h.surf, key) == LVB_OK;
    }

    // Mapping::ToWorld(double start) (mapping.cpp:222-229) and Relocator::CorrectLoop's ToWorld loop over the keyframes since old_time
    // (relocator.cpp:236-244), after a GNSS or loop correction moved their poses: keys[i] / frames[i], n of them, in any order.  The
    // keyframes this class has stored are re-anchored at frame->pose with ONE device call (lvb_icp_map_to_world: their robot-frame
    // clouds stay on the device, one host synchronisation for all of them); a lidar keyframe it has not stored (ToWorld(start) also
    // writes the window's keyframes) goes through AppendKeyframe; a frame without feature_lidar is skipped -- the reference stores
    // empty clouds for it, which no map frame ever merges.  A key listed twice is re-anchored once.  Like RelocateKeyframe this runs on
    // the calling thread's own handles over the resident store; it writes, so the caller holds backend_->mutex, which serialises it
    // with the mapping thread's keyframe calls (INTEGRATION.md 3a).  false: a library call failed (lvb_last_error()).
    template <class FramePtr>
    bool ToWorldKeyframes(const long long* keys, const FramePtr* frames, int n) {
        StoreView h;
        if (!store_view(h)) return false;
        std::vector<long long> moved;
        std::vector<double> poses;
        std::unordered_set<long long> seen;
        bool ok = true;
        for (int i = 0; i < n; ++i) {
            const FramePtr& f = frames[i];
            if (!f->feature_lidar || !seen.insert(keys[i]).second) continue;
            bool held;
            {
                std::lock_guard<std::mutex> lk(meta_);
                held = h.meta->keys.count(keys[i]) > 0;
            }
            if (held) {
                moved.push_back(keys[i]);
                poses.insert(poses.end(), f->pose.data(), f->pose.data() + 7);
            } else if (!store_keyframe(h.ground, h.surf, *h.meta, keys[i], f->feature_lidar->points_ground, f->feature_lidar->points_surf, f->pose.data())) {
                ok = false;
            }
        }
        return lvb_icp_map_to_world(h.ground, h.surf, moved.data(), (int)moved.size(), poses.data()) == LVB_OK && ok;
    }
    bool BuildMapFrame(const long long* keys, int n_keys, double ground_ransac_threshold) {
        Handles& h = handles_of_thread()[this];
        if (!ensure_handles(h)) return false;
        // each side is built on its own: OptimizeKeyframe registers whichever side has a map frame cloud (mapping.cpp:155,167)
        h.ground_map = lvb_icp_map_build(h.ground, keys, n_keys, cell_of(resolution_ * resolution_ * 100), ground_ransac_threshold, nullptr) == LVB_OK;
        h.surf_map = lvb_icp_map_build(h.surf, keys, n_keys, cell_of(resolution_ * resolution_ * 25), -1.0, nullptr) == LVB_OK;
        h.resident = h.ground_map && h.surf_map;
        return h.resident;
    }
    void UsePerCallMap() { Handles& h = handles_of_thread()[this]; h.resident = h.ground_map = h.surf_map = false; }

    // What ScanToMapWithGround / ScanToMapWithSegmented put into their problems for `frame` (association.cpp:270-384: weights, the
    // PoseErrorRPZ / YXY prior unless relocating, TrivialLoss / HuberLoss(0.1), the two gates) and the options of the two Solve
    // calls of Mapping::Optimize (mapping.cpp:159-162, 171-174), as lvb_icp_map_optimize_keyframe takes them.
    template <class FramePtr>
    lvb_map_optimize_params MapOptimizeParams(FramePtr frame, bool relocate = false) const {
        lvb_map_optimize_params p;
        p.weight[0] = frame->weights.lidar_ground; p.weight[1] = frame->weights.lidar_surf;
        p.prior_weight = relocate ? -1.0 : (double)frame->features_left.size() * frame->weights.visual;
        p.huber_a[0] = 0.0; p.huber_a[1] = 0.1;
        p.dist_thr[0] = resolution_ * resolution_ * 100; p.dist_thr[1] = resolution_ * resolution_ * 25;
        lvb_default_options(&p.options);
        p.options.linear_solver_type = 2;            // DENSE_QR
        p.options.max_num_iterations = 4;
        return p;
    }
    // The body of Mapping::Optimize's loop after BuildMapFrame (mapping.cpp:152-185 without PoseGraph::ForwardUpdate): the
    // registrations against the map frame BuildMapFrame just made, frame->pose updated in place, then ToWorld of the keyframe's two
    // robot-frame clouds under `key` -- one device call, one host synchronisation.  As in the reference, a side whose map frame
    // cloud could not be built (BuildMapFrame with no keys: the first lidar keyframe, mapping.cpp:118-119; an empty merged cloud,
    // :155,167) is not registered, and ToWorld stores both clouds whatever ran (:185).  summary: 2 entries (ground, surf) or NULL;
    // a registration that did not run has termination_type = -1.  false: a library call failed (lvb_last_error()).
    template <class FramePtr>
    bool OptimizeKeyframe(FramePtr frame, const double* map_pose7, long long key, lvb_solve_summary* summary = nullptr) {
        Handles& h = handles_of_thread()[this];
        if (!ensure_handles(h)) return false;
        resident_ = &h;
        const auto& g = frame->feature_lidar->points_ground;
        const auto& s = frame->feature_lidar->points_surf;
        const int stride = (int)sizeof(assoc_detail::cloud_data(g, 0)[0]);
        lvb_icp* reg_g = h.ground_map ? h.ground : nullptr;
        lvb_icp* reg_s = h.surf_map ? h.surf : nullptr;
        lvb_solve_summary sums[2];
        lvb_solve_summary* out = summary ? summary : sums;
        bool was_pending;
        {
            std::lock_guard<std::mutex> lk(meta_);
            was_pending = h.pending.erase(key) > 0;
        }
        if (was_pending) {                          // this call stores the host copies: the pending features (and key's clouds) go first
            if (lvb_icp_map_evict(h.ground, key) != LVB_OK || lvb_icp_map_evict(h.surf, key) != LVB_OK) return false;
            std::lock_guard<std::mutex> lk(meta_);
            h.keys.erase(key);
        }
        if (reg_g || reg_s) {
            const lvb_map_optimize_params p = MapOptimizeParams(frame);
            double rpyxyz[6];
            if (lvb_icp_map_optimize_keyframe(reg_g, reg_s, map_pose7, key, assoc_detail::cloud_data(g, 0), (int)g.size(),
                                              assoc_detail::cloud_data(s, 0), (int)s.size(), stride, &p, frame->pose.data(), rpyxyz, out) != LVB_OK)
                return false;
        } else {
            for (int m = 0; m < 2; ++m) { std::memset(&out[m], 0, sizeof(out[m])); out[m].termination_type = -1; }
        }
        // ToWorld of a side that was not registered: the call above stores only the clouds of the handles it was given
        const double* pose = frame->pose.data();
        {
            std::lock_guard<std::mutex> lk(meta_);
            h.keys.erase(key);                       // until both sides hold the keyframe's clouds again
        }
        if (!reg_g && !(lvb_icp_map_evict(h.ground, key) == LVB_OK &&
                        lvb_icp_map_append(h.ground, key, assoc_detail::cloud_data(g, 0), (int)g.size(), stride, pose) == LVB_OK)) return false;
        if (!reg_s && !(lvb_icp_map_evict(h.surf, key) == LVB_OK &&
                        lvb_icp_map_append(h.surf, key, assoc_detail::cloud_data(s, 0), (int)s.size(), stride, pose) == LVB_OK)) return false;
        std::lock_guard<std::mutex> lk(meta_);
        h.keys.insert(key);
        return true;
    }

    // Mapping::BuildMapFrame + the same body of Mapping::Optimize's loop (mapping.cpp:114-185 without PoseGraph::ForwardUpdate) in ONE
    // device call with one host synchronisation (lvb_icp_map_build_optimize_keyframe): the map frame of `keys` (in merge order; none
    // for the first lidar keyframe, :118-119) is merged, SegmentGround'ed (ground_ransac_threshold > 0) and hashed with the cell sizes
    // BuildMapFrame uses, each side with a non-empty map frame is registered, frame->pose is updated in place and both robot-frame
    // clouds are stored under `key`.  Afterwards the map frames it built are the resident ones, as after BuildMapFrame.
    // summary: 2 entries (ground, surf) or NULL; a side that was not registered has termination_type = -1.  false: the call failed
    // (lvb_last_error()).
    template <class FramePtr>
    bool OptimizeKeyframe(FramePtr frame, const long long* keys, int n_keys, const double* map_pose7, long long key,
                          double ground_ransac_threshold, lvb_solve_summary* summary = nullptr) {
        Handles& h = handles_of_thread()[this];
        if (!ensure_handles(h)) return false;
        const auto& g = frame->feature_lidar->points_ground;
        const auto& s = frame->feature_lidar->points_surf;
        const int stride = (int)sizeof(assoc_detail::cloud_data(g, 0)[0]);
        const lvb_map_optimize_params p = MapOptimizeParams(frame);
        const float cells[2] = {cell_of(resolution_ * resolution_ * 100), cell_of(resolution_ * resolution_ * 25)};
        lvb_solve_summary sums[2];
        double rpyxyz[6];
        int n_map[2];
        bool by_key;                                           // ExtractKeyframe left the clouds on the device: NULL clouds, -1 points
        {
            std::lock_guard<std::mutex> lk(meta_);
            by_key = h.pending.count(key) > 0;
        }
        if (lvb_icp_map_build_optimize_keyframe(h.ground, h.surf, keys, n_keys, cells, ground_ransac_threshold, map_pose7, key,
                                                by_key ? nullptr : assoc_detail::cloud_data(g, 0), by_key ? -1 : (int)g.size(),
                                                by_key ? nullptr : assoc_detail::cloud_data(s, 0), by_key ? -1 : (int)s.size(), stride,
                                                &p, frame->pose.data(), rpyxyz, summary ? summary : sums, n_map) != LVB_OK)
            return false;
        {
            std::lock_guard<std::mutex> lk(meta_);
            h.pending.erase(key);
            h.keys.insert(key);
        }
        h.ground_map = n_map[0] > 0; h.surf_map = n_map[1] > 0;
        h.resident = h.ground_map && h.surf_map;
        resident_ = &h;
        return true;
    }

    // Mapping::Optimize(active_kfs) (mapping.cpp:139-191) for its n lidar keyframes, in time order, in ONE device call with one host
    // synchronisation (lvb_icp_map_optimize_keyframes): frames[k] is keyframe keys[k]; its map frame is map_keys[3 k .. 3 k +
    // n_map_keys[k]) (get_lidar_frames(0, t_k, 3), merge order), resident or keys of earlier frames of the call; map_poses7[7 k]: the
    // newest map key's pose when it is resident.  frame->pose goes in as the caller holds it -- before the earlier keyframes'
    // ForwardUpdates, which the device chains -- and comes back optimised, also copied to poses7 (n x 7).  transforms7 (n x 7): T_k =
    // new_k * old_k^-1, in order; the caller replays PoseGraph::ForwardUpdate(T_k, t_k + epsilon) and then writes poses7 back to the
    // frames of the call (INTEGRATION.md 3a).  Each keyframe registers with its own MapOptimizeParams weights and prior weight, as
    // ScanToMapWith* would.  summary: 2 per keyframe or NULL.  false: the call failed and changed nothing (the
    // per-keyframe OptimizeKeyframe loop is the fallback; lvb_last_error() says why).
    template <class FramePtr>
    bool OptimizeKeyframes(const FramePtr* frames, const long long* keys, const long long* map_keys, const int* n_map_keys, const double* map_poses7,
                           int n, double ground_ransac_threshold, double* poses7, double* transforms7, lvb_solve_summary* summary = nullptr) {
        Handles& h = handles_of_thread()[this];
        if (!ensure_handles(h)) return false;
        if (n <= 0) return true;
        std::vector<lvb_map_keyframe> recs(n);
        int stride = 0;
        std::unique_lock<std::mutex> meta_lock(meta_);
        for (int k = 0; k < n; ++k) {
            const auto& g = frames[k]->feature_lidar->points_ground;
            const auto& s = frames[k]->feature_lidar->points_surf;
            stride = (int)sizeof(assoc_detail::cloud_data(g, 0)[0]);
            lvb_map_keyframe& r = recs[k];
            std::memset(&r, 0, sizeof(r));
            r.key = keys[k]; r.n_map_keys = n_map_keys[k];
            for (int i = 0; i < n_map_keys[k] && i < 3; ++i) r.map_keys[i] = map_keys[3 * k + i];
            if (h.pending.count(keys[k])) { r.ground_pts = r.surf_pts = nullptr; r.n_ground = r.n_surf = -1; }      // by key (ExtractKeyframe)
            else {
                r.ground_pts = assoc_detail::cloud_data(g, 0); r.n_ground = (int)g.size();
                r.surf_pts = assoc_detail::cloud_data(s, 0); r.n_surf = (int)s.size();
            }
            std::memcpy(r.map_pose, map_poses7 + 7 * k, sizeof(r.map_pose)); std::memcpy(r.pose, frames[k]->pose.data(), sizeof(r.pose));
            const lvb_map_optimize_params pk = MapOptimizeParams(frames[k]);      // each keyframe's own weights and prior weight
            r.weight[0] = pk.weight[0]; r.weight[1] = pk.weight[1]; r.prior_weight = pk.prior_weight;
        }
        meta_lock.unlock();
        const lvb_map_optimize_params p = MapOptimizeParams(frames[0]);          // the options, gates and losses every keyframe shares
        const float cells[2] = {cell_of(resolution_ * resolution_ * 100), cell_of(resolution_ * resolution_ * 25)};
        if (lvb_icp_map_optimize_keyframes(h.ground, h.surf, recs.data(), n, cells, ground_ransac_threshold, stride, &p) != LVB_OK) return false;
        meta_lock.lock();
        for (int k = 0; k < n; ++k) {
            const lvb_map_keyframe& r = recs[k];
            std::memcpy(frames[k]->pose.data(), r.pose, sizeof(r.pose));
            if (poses7) std::memcpy(poses7 + 7 * k, r.pose, sizeof(r.pose));
            if (transforms7) std::memcpy(transforms7 + 7 * k, r.transform, sizeof(r.transform));
            if (summary) { summary[2 * k] = r.summary[0]; summary[2 * k + 1] = r.summary[1]; }
            h.keys.insert(keys[k]);
            h.pending.erase(keys[k]);
        }
        meta_lock.unlock();
        // as OptimizeKeyframe(frame, keys, ...) leaves them after the last keyframe: that keyframe's map frames
        h.ground_map = recs[n - 1].n_map_points[0] > 0; h.surf_map = recs[n - 1].n_map_points[1] > 0;
        h.resident = h.ground_map && h.surf_map;
        resident_ = &h;
        return true;
    }

    // Mapping::Relocate for one loop-closure candidate (mapping.cpp:78-112, 251-300) in ONE device call with one host synchronisation
    // (lvb_icp_map_relocate): BuildOldMapFrame of `keys` (1 to 3 resident keyframes in time order: the lidar keyframe before the old
    // one, the old one if it has lidar, the one after it; map_pose7 = the earliest one's pose) with BuildMapFrame's cell sizes and
    // SegmentGround threshold, then the reference's four rounds of ScanToMapWithGround / ScanToMapWithSegmented with relocate = true,
    // from old_pose7 * relative_o_c.  relative_o_c (anything with .data() in the Sophus layout; frame->loop_closure->relative_o_c in
    // the reference) is the guess on entry and old_pose^-1 * the final pose on return; frame->pose is not touched, nothing is stored
    // and the resident map frames stay as they were.  Returns (int)(score_ground + score_surf) as mapping.cpp:299 does.
    // Deviation: where the reference adds a score that was never set (a side whose map frame cloud is empty is skipped in every round)
    // or that is NaN (no accepted point), this returns 0 -- a rejected candidate -- so that `score - 20` (relocator.cpp:178) cannot
    // overflow; a sum below -1e9 is returned as -1e9 (the truncation of a larger one is undefined).  A failed library call also
    // returns 0 and leaves relative_o_c as it was (lvb_last_error() says why).
    // The call runs on the calling thread's own handles over the resident store (StoreView), read-only and with no lock: the Relocator
    // relocates its candidates while the mapping thread registers, as the reference does (INTEGRATION.md 3a).
    template <class FramePtr, class Pose>
    int RelocateKeyframe(FramePtr frame, const long long* keys, int n_keys, const double* map_pose7, const double* old_pose7, Pose& relative_o_c,
                         double ground_ransac_threshold, lvb_solve_summary* summary = nullptr) {
        StoreView h;
        if (!store_view(h)) return 0;
        const auto& g = frame->feature_lidar->points_ground;
        const auto& s = frame->feature_lidar->points_surf;
        const int stride = (int)sizeof(assoc_detail::cloud_data(g, 0)[0]);
        const lvb_map_optimize_params p = MapOptimizeParams(frame, true);
        const float cells[2] = {cell_of(resolution_ * resolution_ * 100), cell_of(resolution_ * resolution_ * 25)};
        double rel[7], pose[7], score[2];
        if (lvb_icp_map_relocate(h.ground, h.surf, keys, n_keys, cells, ground_ransac_threshold, map_pose7, old_pose7, relative_o_c.data(),
                                 assoc_detail::cloud_data(g, 0), (int)g.size(), assoc_detail::cloud_data(s, 0), (int)s.size(), stride, &p, 4,
                                 rel, pose, summary, score, nullptr) != LVB_OK)
            return 0;
        std::memcpy(relative_o_c.data(), rel, sizeof(rel));
        const double sum = score[0] + score[1];
        if (!std::isfinite(sum)) return 0;
        return (int)std::max(sum, -1e9);
    }

private:
    static float cell_of(double thr) { return std::nextafter((float)std::sqrt(thr), 1e30f) * 1.0001f; }
    template <class FramePtr, class Cloud, class Problem>
    bool add(int mode, FramePtr frame, FramePtr map_frame, const Cloud& scan, const Cloud& map, double* para, Problem& problem, bool relocate,
             double thr, double weight, ceres::LossFunction* loss, lvb_icp*& icp) {
        lvb::Runtime& rt = lvb::Runtime::get();
        if (!rt.ensure()) { delete loss; return false; }
        if (!icp && lvb_icp_create(rt.ctx, &icp) != LVB_OK) { delete loss; return false; }
        const int stride = (int)sizeof(assoc_detail::cloud_data(scan, 0)[0]);
        Handles& h = handles_of_thread()[this];
        if (!h.resident) {
            (mode == 0 ? h.ground_map : h.surf_map) = false;          // the per-call map replaces this side's map frame
            if (lvb_icp_set_map(icp, assoc_detail::cloud_data(map, 0), (int)map.size(), stride, cell_of(thr)) != LVB_OK) { delete loss; return false; }
        }
        if (mode == 0) { problem.AddParameterBlock(para + 1, 1); problem.AddParameterBlock(para + 2, 1); problem.AddParameterBlock(para + 5, 1); }
        else { problem.AddParameterBlock(para + 0, 1); problem.AddParameterBlock(para + 3, 1); problem.AddParameterBlock(para + 4, 1); }
        double* x0 = mode == 0 ? para + 1 : para + 0; double* x1 = mode == 0 ? para + 2 : para + 3; double* x2 = mode == 0 ? para + 5 : para + 4;
        lvb::ScanToMapCost* c = new lvb::ScanToMapCost();
        c->mode = mode; c->icp = icp; c->scan = assoc_detail::cloud_data(scan, 0); c->n = (int)scan.size(); c->stride = stride;
        std::memcpy(c->frame_pose, frame->pose.data(), sizeof(c->frame_pose)); std::memcpy(c->map_pose, map_frame->pose.data(), sizeof(c->map_pose));
        c->rpyxyz = para; c->weight = weight; c->dist_thr = thr;
        assoc_detail::add_block(problem, 0, true, c, loss, x0, x1, x2);
        if (!relocate) {
            lvb::IcpPriorCost* p = new lvb::IcpPriorCost();
            p->mode = mode; p->weight = (double)frame->features_left.size() * frame->weights.visual;   // association.cpp:323,381
            assoc_detail::add_block(problem, 0, false, p, nullptr, x0, x1, x2);
        }
        return true;
    }
    // lvb_icp handles (voxel hash + scratch on one context's stream) are single-threaded and the context is per host thread
    // (ceres_shim.h): Mapping::Optimize and Relocator::RelocateByPoints reach the same object from two threads without a lock
    // (mapping.cpp:155-177, relocator.cpp:188-206), so every thread gets its own pair.
    // resident: both map frames built (ScanToMapWith* use them); ground_map / surf_map: that side's map frame is the last BuildMapFrame's;
    // keys: the keyframes whose clouds both handles hold (ToWorldKeyframes re-anchors those on the device); pending: the keys whose
    // features ExtractKeyframe left on these handles
    struct Handles {
        lvb_icp* ground = nullptr; lvb_icp* surf = nullptr; bool resident = false, ground_map = false, surf_map = false;
        std::unordered_set<long long> keys, pending;
    };
    struct Packed { float x, y, z, intensity; };     // the records lvb_icp_map_extract_keyframe returns
    template <class CloudOut>
    static void unpack(const std::vector<Packed>& src, int n, CloudOut& dst) {
        dst.resize((size_t)n);
        for (int i = 0; i < n; ++i) { auto& q = dst[(size_t)i]; q.x = src[i].x; q.y = src[i].y; q.z = src[i].z; q.intensity = src[i].intensity; }
    }
    // ToWorld of one keyframe into the store of ground / surf, whose keys `meta` lists: its two robot-frame clouds replace whatever the
    // store held under `key`
    template <class Cloud>
    bool store_keyframe(lvb_icp* ground, lvb_icp* surf, Handles& meta, long long key, const Cloud& ground_robot, const Cloud& surf_robot,
                        const double* pose7) {
        const int stride = (int)sizeof(assoc_detail::cloud_data(ground_robot, 0)[0]);
        {
            std::lock_guard<std::mutex> lk(meta_);
            meta.keys.erase(key); meta.pending.erase(key);
        }
        lvb_icp_map_evict(ground, key); lvb_icp_map_evict(surf, key);                // re-registering a keyframe (ToWorld(start)) replaces its clouds
        if (lvb_icp_map_append(ground, key, assoc_detail::cloud_data(ground_robot, 0), (int)ground_robot.size(), stride, pose7) != LVB_OK ||
            lvb_icp_map_append(surf, key, assoc_detail::cloud_data(surf_robot, 0), (int)surf_robot.size(), stride, pose7) != LVB_OK)
            return false;
        std::lock_guard<std::mutex> lk(meta_);
        meta.keys.insert(key);
        return true;
    }
    // The handles a call on the resident store makes from the calling thread: on the thread that keeps the resident pair (or before
    // there is one) the thread's own pair; on any other thread a pair lvb_icp_share made once for that thread, on its own context, from
    // the resident pair.  meta: the Handles whose key sets describe that store (read and written under meta_).  The resident pair and
    // its context belong to the thread that keeps it (thread_local), so that thread must outlive the other threads' calls, as the
    // reference's mapping thread does; the shared pairs keep the clouds themselves alive.  Every pair, own or shared, is made on the
    // calling thread's Runtime::get().ctx, so its calls run at the priority that thread chose with Runtime::set_thread_priority.
    struct StoreView { lvb_icp* ground; lvb_icp* surf; Handles* meta; };
    bool store_view(StoreView& v) {
        Handles& own = handles_of_thread()[this];
        Handles* r = resident_.load();
        if (!r || r == &own) {
            if (!ensure_handles(own)) return false;
            v.ground = own.ground; v.surf = own.surf; v.meta = &own;
            return true;
        }
        lvb::Runtime& rt = lvb::Runtime::get();
        if (!rt.ensure()) return false;
        Handles& sh = shared_of_thread()[this];
        if (!sh.ground && lvb_icp_share(rt.ctx, r->ground, &sh.ground) != LVB_OK) return false;
        if (!sh.surf && lvb_icp_share(rt.ctx, r->surf, &sh.surf) != LVB_OK) return false;
        v.ground = sh.ground; v.surf = sh.surf; v.meta = r;
        return true;
    }
    static bool ensure_handles(Handles& h) {
        lvb::Runtime& rt = lvb::Runtime::get();
        if (!rt.ensure()) return false;
        return (h.ground || lvb_icp_create(rt.ctx, &h.ground) == LVB_OK) && (h.surf || lvb_icp_create(rt.ctx, &h.surf) == LVB_OK);
    }
    static std::unordered_map<const void*, Handles>& handles_of_thread() { static thread_local std::unordered_map<const void*, Handles> m; return m; }
    // the calling thread's handles shared from the resident pair (store_view); only their ground / surf members are used
    static std::unordered_map<const void*, Handles>& shared_of_thread() { static thread_local std::unordered_map<const void*, Handles> m; return m; }
    double resolution_;
    lvb_lidar_config lidar_cfg_;
    std::vector<Packed> extract_ground_, extract_surf_;      // ExtractKeyframe's host copies, num_scans * horizon_scan records each
    // the class stays copyable: a copy takes the resident pointer and gets a mutex of its own
    struct ResidentPtr {
        std::atomic<Handles*> p{nullptr};
        ResidentPtr() = default;
        ResidentPtr(const ResidentPtr& o) : p(o.p.load()) {}
        ResidentPtr& operator=(const ResidentPtr& o) { p = o.p.load(); return *this; }
        ResidentPtr& operator=(Handles* h) { p = h; return *this; }
        Handles* load() const { return p.load(); }
    };
    struct Mutex : std::mutex {
        Mutex() = default;
        Mutex(const Mutex&) : std::mutex() {}
        Mutex& operator=(const Mutex&) { return *this; }
    };
    ResidentPtr resident_;             // the handles that keep the resident keyframe clouds (StoreView); map nodes do not move
    Mutex meta_;                       // guards the key sets (keys, pending) of every Handles: other threads' calls read and write the resident one's
};

}  // namespace lvio_fusion
