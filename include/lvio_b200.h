/* lvio_b200.h -- C ABI of the H100-native optimisation backend for lvio_fusion.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  The reference has no FFI layer: its
 * hot path calls the C++ APIs of Ceres (ceres::Problem / ceres::Solve) and PCL
 * (pcl::KdTreeFLANN) directly.  The C++ shim in include/lvio_b200/ keeps those call shapes
 * and forwards to the functions below; each entry point names the reference interface it
 * stands behind (paths relative to /root/reference/src/lvio_fusion/).
 *
 * Conventions: extern "C", int return (LVB_OK or a negative LVB_ERR_*; text via
 * lvb_last_error), no exceptions or STL across the boundary, the caller owns every host
 * buffer, the library owns the device buffers tied to a handle.  Threads: a context (lvb_ctx:
 * one CUDA stream, on which an LM pass may be under thread-local graph capture) and the handles
 * created from it belong to ONE host thread at a time; use one context per solving thread
 * (Backend thread, global thread, Relocator thread: backend.cpp:19-20, relocator.cpp:188-206) --
 * the C++ shim does (lvb::Runtime is thread_local).  There is NO CPU fallback: every compute entry point fails with
 * LVB_ERR_CUDA when no sm_90 device is usable.
 *
 * Layouts: pose = Sophus::SE3d::data() = [qx qy qz qw tx ty tz] (include/lvio_fusion/ceres/
 * base.hpp:27-38), T_world_body.  All BA arithmetic is FP64.  Jacobians handed back by the
 * *_eval entry points are row-major [n_res x sum(block sizes)] with the parameter blocks in
 * AddResidualBlock order, i.e. the per-block arrays Ceres fills, concatenated.
 */
#ifndef LVIO_B200_H_
#define LVIO_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define LVB_API __attribute__((visibility("default")))
#else
#define LVB_API
#endif

#define LVB_OK 0
#define LVB_ERR_INVALID (-1)     /* bad argument / index out of range */
#define LVB_ERR_CUDA (-2)        /* no usable device, launch or runtime failure */
#define LVB_ERR_STATE (-3)       /* call order violated (e.g. solve before finalize) */
#define LVB_ERR_NUMERIC (-4)     /* non-SPD system, NaN */
#define LVB_ERR_UNSUPPORTED (-5) /* size outside what this build handles */
#define LVB_ERR_COMM (-6)        /* NCCL failure */

typedef struct lvb_ctx lvb_ctx;
typedef struct lvb_ba lvb_ba;
typedef struct lvb_icp lvb_icp;

/* Factor kinds: the closed set of cost functions on the hot path (SURVEY 8a). */
enum lvb_factor_kind {
    LVB_TWO_FRAME = 0,  /* TwoFrameReprojectionError  ceres/visual_error.hpp:78-107  <2,1,7,7>
                           consts[5] = first_ob.xy ob.xy weight ; idx[3] = inv_depth, pose(first kf), pose(kf) */
    LVB_POSE_ONLY = 1,  /* PoseOnlyReprojectionError  ceres/visual_error.hpp:48-76   <2,7>
                           consts[6] = ob.xy pw.xyz weight ; idx[1] = pose */
    LVB_TWO_CAMERA = 2, /* TwoCameraReprojectionError ceres/visual_error.hpp:109-137 <2,1>
                           consts[5] = left_ob.xy right_ob.xy weight ; idx[1] = inv_depth */
    LVB_IMU = 3,        /* ImuError                   ceres/imu_error.hpp:12-122     <15,7,3,3,3,7,3,3,3>
                           consts[469] = delta_p[3] delta_q[4 xyzw] delta_v[3] linearized_ba[3]
                           linearized_bg[3] sum_dt jacobian[15x15 rm] covariance[15x15 rm]
                           (imu/preintegration.h:66-80) prior_a prior_g ;
                           prior_a = prior_g = -1 : ImuError.  Both >= 0 : ImuInitError (ceres/imu_error.hpp:124-229,
                           <15,7,3,3,3,7,3>, imu::FullBA tools.cpp:138-162): idx[6] = idx[7] = -1, Baj = Bgj = 0, the
                           bias blocks of cov^-1 are replaced by prior * I before the LLT ;
                           idx[8] = pose_i v_i ba_i bg_i pose_j v_j ba_j bg_j (v/ba/bg index the vec3 blocks) */
    LVB_POSE_GRAPH = 4, /* PoseGraphError             ceres/pose_error.hpp:10-53     <6,7,7>
                           consts[8] = rpyxyz_[6] weight v ; idx[2] = pose_1 pose_2 */
    LVB_POSE_PRIOR = 5, /* PoseError                  ceres/pose_error.hpp:55-86     <6,7>
                           consts[9] = pose_[7] weight v ; idx[1] = pose */
    LVB_NUM_KINDS = 6
};

/* ceres::Solver::Options subset the reference sets (backend.cpp:205-209, mapping.cpp:159-163,
 * backend.cpp:262-266) plus the Ceres defaults it relies on. */
typedef struct lvb_solve_options {
    int max_num_iterations;             /* 50 ; 4 in Mapping::Optimize ; 1 in UpdateFrontend */
    double max_solver_time_in_seconds;  /* 1e9 ; (end-start)/n_kfs in Backend::Optimize */
    double function_tolerance;          /* 1e-6 */
    double gradient_tolerance;          /* 1e-10 */
    double parameter_tolerance;         /* 1e-8 */
    double initial_trust_region_radius; /* 1e4 */
    int jacobi_scaling;                 /* 1 */
    int linear_solver_type;             /* 0 SPARSE_SCHUR, 1 SPARSE_NORMAL_CHOLESKY, 2 DENSE_QR (informational:
                                           the device always eliminates inverse depths exactly) */
    int num_threads;                    /* ignored on the device */
    int schur_mode;                     /* 0 = FP64 CUDA-core Schur (parity reference), 1 = tensor-core (wgmma) split-precision */
} lvb_solve_options;

/* ceres::Solver::Summary fields the reference reads (mapping.cpp:279-280,293-294) + diagnostics. */
typedef struct lvb_solve_summary {
    double initial_cost;
    double final_cost;
    int num_iterations;        /* LM steps attempted */
    int num_successful_steps;
    int termination_type;      /* 0 CONVERGENCE, 1 NO_CONVERGENCE, 2 FAILURE */
    int num_residual_blocks;
    int num_residual_blocks_reduced;
    double final_radius;
    double total_time_in_seconds;
} lvb_solve_summary;

LVB_API int lvb_version(void);
LVB_API void lvb_default_options(lvb_solve_options* o);

/* ---- context ------------------------------------------------------------------------- */
/* cuda_stream: a cudaStream_t to launch on (e.g. torch.cuda.current_stream().cuda_stream),
 * or NULL to let the context create its own non-blocking stream.  The context's second stream (the parallel branches of an LM pass)
 * gets the priority of the stream it launches on: the default one with NULL. */
LVB_API int lvb_ctx_create(int device, void* cuda_stream, lvb_ctx** out);
/* Scheduling priority of all of a context's device work.  As lvb_ctx_create(device, NULL, out), but both of the context's streams are
 * made with cudaStreamCreateWithPriority(..., cudaStreamNonBlocking, priority).  CUDA's convention: a lower number runs earlier (its
 * pending CTAs are dispatched first; running CTAs are not pre-empted), and CUDA clamps the value to the device's range
 * (lvb_device_priority_range).  Results, launches and synchronisations are those of a default-priority context.  A thread whose calls
 * others wait on -- the one that runs the window solve and the mapping pass -- can put its work first this way. */
LVB_API int lvb_ctx_create_with_priority(int device, int priority, lvb_ctx** out);
/* the priority the context's stream actually has (after clamping, or the caller's stream's) */
LVB_API int lvb_ctx_priority(lvb_ctx* ctx, int* priority);
/* cudaDeviceGetStreamPriorityRange of `device`: *greatest <= *least; the default priority is 0.  The calling thread's current device
 * is left as it was. */
LVB_API int lvb_device_priority_range(int device, int* least, int* greatest);
LVB_API void lvb_ctx_destroy(lvb_ctx* ctx);
LVB_API const char* lvb_last_error(void);            /* thread-local text of the last failure */
LVB_API long long lvb_launch_count(lvb_ctx* ctx);    /* kernels launched through this context so far */
LVB_API long long lvb_sync_count(lvb_ctx* ctx);      /* host synchronisations the library has made on this context's stream so far */
LVB_API int lvb_ctx_synchronize(lvb_ctx* ctx);

/* Multi-GPU (SURVEY 8e): one process per GPU; the id is produced on rank 0 and shipped to
 * the other ranks by the caller (torch.distributed broadcast in bench.py). After init every
 * lvb_ba_solve / lvb_icp_scan_to_map on this context all-reduces its reduced normal
 * equations once per LM iteration: messages up to 1 MB through an in-kernel all-reduce over NVLink peer
 * memory (CUDA IPC exchange buffers set up here; LVB_NO_P2P=1 disables), larger ones through
 * ncclAllReduce(sum, f64).  lvb_comm_init is collective, and so are lvb_ba_finalize / lvb_ba_solve /
 * lvb_ba_reduced_system / lvb_icp_scan_to_map on a context with world_size > 1: every rank must make the
 * same calls in the same order. */
LVB_API int lvb_comm_unique_id(char id[128]);
LVB_API int lvb_comm_init(lvb_ctx* ctx, int rank, int world_size, const char id[128]);

/* ---- bundle adjustment: stands behind adapt::Problem + ceres::Solve -------------------
 * (adapt/problem.h:34-88, backend.cpp:96-183,192-211)                                   */
LVB_API int lvb_ba_create(lvb_ctx* ctx, lvb_ba** out);
LVB_API void lvb_ba_destroy(lvb_ba* ba);
/* cam[22] = 2 x { fx fy cx cy  extrinsic[7] (T_body_cam) } : Camera::Get(0), Camera::Get(1)
 * (visual/camera.h:79-80, sensor.h:21-24) */
LVB_API int lvb_ba_set_cameras(lvb_ba* ba, const double cam[22]);
/* Problem::AddParameterBlock(double*, size[, parameterization]) + SetParameterBlockConstant
 * (adapt/problem.h:49-63): poses use ProductParameterization(EigenQuaternion, Identity3)
 * (backend.cpp:99-101); vec3 blocks (Vw, linearized_ba, linearized_bg, backend.cpp:147-152)
 * and inverse depths (backend.cpp:121) are Euclidean.  is_const may be NULL. */
LVB_API int lvb_ba_set_poses(lvb_ba* ba, int n, const double* poses7, const uint8_t* is_const);
LVB_API int lvb_ba_set_vec3(lvb_ba* ba, int n, const double* v3, const uint8_t* is_const);
LVB_API int lvb_ba_set_inv_depths(lvb_ba* ba, int n, const double* rho, const uint8_t* is_const);
/* Problem::AddResidualBlock(cost, loss, x0, xs...) in bulk (adapt/problem.h:37-47):
 * consts is n x stride(kind) (AoS, one record per block), idx is n x nidx(kind). Appends. */
LVB_API int lvb_ba_add_factors(lvb_ba* ba, int kind, int n, const double* consts, const int32_t* idx);
/* ceres::HuberLoss(a) for every block of `kind` (backend.cpp:98 uses 1.0 on the visual kinds);
 * a <= 0 means NULL / TrivialLoss. */
LVB_API int lvb_ba_set_loss(lvb_ba* ba, int kind, double huber_a);
/* Freeze the structure, sort/transpose to the device layout, upload (window-sized problems: assembled in the context's pinned
 * staging area and sent with one copy).  Collective when world_size > 1 (the order of the unknowns and the envelope of the
 * reduced system are agreed on across the ranks).  The reduced camera system is solved by the one-CTA kernel (<= 736 unknowns or
 * a panel that fits in shared memory), the multifrontal separator tree (banded map-scale systems) or, for loop-closure shaped
 * envelopes, per-phase grids over global memory; LVB_ERR_UNSUPPORTED (at solve) only when its banded storage exceeds 24 GB. */
LVB_API int lvb_ba_finalize(lvb_ba* ba);
LVB_API int lvb_ba_dims(lvb_ba* ba, int* dim_camera, int* n_inv_depth_free, int* n_residual_rows);
/* Re-upload parameter values only (same structure) -- used between solves / by the bench. */
LVB_API int lvb_ba_update_params(lvb_ba* ba, const double* poses7, const double* v3, const double* rho);

/* CostFunction::Evaluate for every block of `kind` at the current parameters (parity entry):
 * r is n x n_res, J is n x n_res x cols(kind) with cols = 15, 7, 1, 32, 14, 7.  Raw values:
 * no loss correction, ambient (not tangent) Jacobians, as Ceres' Evaluate returns them.
 * r or J may be NULL.  The *_device variant runs the same kernel without the copy back
 * (bench roofline entry). */
LVB_API int lvb_ba_eval(lvb_ba* ba, int kind, double* r, double* J);
LVB_API int lvb_ba_eval_device(lvb_ba* ba, int kind);

/* The Schur-reduced, LM-damped camera system of the first trust-region step at the current
 * parameters with the given radius (Jacobi scaling taken at this point): S is
 * dim_camera x dim_camera row-major, b the right-hand side (S dx = b), cost = 1/2 sum rho.
 * Parity entry for kernels K4/K5. */
LVB_API int lvb_ba_reduced_system(lvb_ba* ba, double radius, double* S, double* b, double* cost);

/* ceres::Solve(options, &problem, &summary) (adapt/problem.h:83-88). Parameters are updated
 * on the device; fetch them with the getters (the shim writes them back in place). */
/* Default Schur mode of the handle (used by lvb_ba_reduced_system and by lvb_ba_solve(options == NULL)): 0 = FP64
 * CUDA-core elimination (parity reference), 1 = wgmma split-bf16 contraction with FP32 accumulation in registers, taken
 * only when 6 x (free poses) <= 128 on a single GPU, else the handle silently stays on mode 0. */
LVB_API int lvb_ba_set_schur_mode(lvb_ba* ba, int mode);
LVB_API int lvb_ba_solve(lvb_ba* ba, const lvb_solve_options* options, lvb_solve_summary* summary);
/* The three getters share one device round trip: the first call after a solve / lvb_ba_update_params reads all parameter blocks
 * back, the others copy from that snapshot. */
LVB_API int lvb_ba_get_poses(lvb_ba* ba, double* poses7);
LVB_API int lvb_ba_get_vec3(lvb_ba* ba, double* v3);
LVB_API int lvb_ba_get_inv_depths(lvb_ba* ba, double* rho);
/* compute_reprojection_error over all LVB_POSE_ONLY-shaped (ob, pw, pose) triples
 * (backend.cpp:185-190, outlier pass :229-245): err[i] = |pi(pw_i, pose_i) - ob_i|, weight 1. */
LVB_API int lvb_ba_reprojection_errors(lvb_ba* ba, int n, const double* ob_pw /* n x 5 */, const int32_t* pose_idx, double* err);

/* ---- IMU preintegration, the producer of the LVB_IMU constants (SURVEY 8(f).3).
 * Stands behind Preintegration::Append / Propagate / MidPointIntegration (imu/preintegration.h:27-40,
 * src/preintegration.cpp:30-127) for a batch of n keyframe intervals, and behind Preintegration::Repropagate
 * (src/preintegration.cpp:129-142, called from tools.cpp:87 when the biases move): the same call with the new biases.
 * Interval i owns the samples first[i] .. first[i+1]-1, each `dt acc[3] gyr[3]`; acc0/gyr0 seed the midpoint rule
 * (the measurement at the first keyframe); noise = {ACC_N, GYR_N, ACC_W, GYR_W} (imu/imu.h, kitti.yaml:48-51).
 * consts receives n records of 469 doubles in the LVB_IMU layout (prior_a = prior_g = -1: plain ImuError). */
LVB_API int lvb_imu_preintegrate(lvb_ctx* ctx, int n, const int32_t* first /* n+1 */, const double* samples /* first[n] x 7 */,
                                 const double* acc0 /* n x 3 */, const double* gyr0 /* n x 3 */,
                                 const double* ba /* n x 3 */, const double* bg /* n x 3 */, const double noise[4],
                                 double* consts /* n x 469 */);

/* ---- lidar scan-to-map: stands behind pcl::KdTreeFLANN + FeatureAssociation::ScanToMapWith*
 * (association.cpp:270-384) and the two Solve calls of Mapping::Optimize (mapping.cpp:139-191) */
LVB_API int lvb_icp_create(lvb_ctx* ctx, lvb_icp** out);
/* A handle on ctx that shares `owner`'s resident keyframe clouds and pending features (its store); its map frames, relocation
 * slot and scratch are its own.  ctx: any context on owner's device (typically another host thread's).  Sharing a shared handle
 * shares the same store; lvb_icp_destroy of any handle, the owner included, leaves the store alive for the others (what a handle
 * drops last is freed on its own context's stream).  lvb_icp_create makes a fresh, unshared store.
 * Errors, before anything is created: LVB_ERR_INVALID for NULL arguments or a context on another device; LVB_ERR_UNSUPPORTED on a
 * context with world_size > 1 (sharded stores stay per rank).
 * Concurrency on one store, each handle on its own thread's context:
 *   - read-only calls run concurrently from any thread's handles: lvb_icp_map_build, lvb_icp_map_relocate and the map keys of the
 *     keyframe calls;
 *   - lvb_icp_map_extract_keyframe runs concurrently too: it writes only the pending entry of its own key;
 *   - calls that store, re-anchor or evict a key (the keyframe calls, lvb_icp_map_append, lvb_icp_map_to_world, lvb_icp_map_evict)
 *     are serialised by the caller among themselves, as the reference's backend_->mutex does for Mapping::Optimize and ToWorld;
 *   - each call sees every cloud as committed when it took its snapshot of the store (a writer commits after its synchronisation),
 *     and the results are those of some serial order of the calls.  A by-key keyframe call sees the pending features committed
 *     before it started, and otherwise fails with LVB_ERR_INVALID.
 * On a shared store lvb_icp_map_to_world writes each re-anchored cloud into a new buffer and publishes it at its commit (a
 * concurrent reader keeps the old one until it returns), and lvb_icp_map_extract_keyframe waits for its pending copies before it
 * publishes them (one more host synchronisation).  An unshared store behaves as if sharing did not exist. */
LVB_API int lvb_icp_share(lvb_ctx* ctx, lvb_icp* owner, lvb_icp** out);
LVB_API void lvb_icp_destroy(lvb_icp* icp);
/* KdTreeFLANN::setInputCloud (association.cpp:278-279,336-337).  points: n records of
 * stride_bytes (>= 12) whose first three floats are x,y,z -- 32 for pcl::PointXYZI, 16 for a
 * packed float4.  cell_size: edge of the voxel grid the cloud is hashed into; queries are
 * exact within that radius. */
LVB_API int lvb_icp_set_map(lvb_icp* icp, const void* points, int n, int stride_bytes, float cell_size);
/* ---- device-resident map (SURVEY 8(f).2).  The reference keeps one world-frame cloud per keyframe
 * (Mapping::pointclouds_surf / pointclouds_ground, filled by Mapping::ToWorld -> MergeScan, src/mapping.cpp:193-220), merges the
 * last three into the map frame for every new keyframe and re-runs SegmentGround on the merged ground cloud
 * (Mapping::BuildMapFrame, src/mapping.cpp:114-137), then rebuilds a kd-tree on it per ScanToMap call (association.cpp:278-279).
 * Here the per-keyframe clouds stay in HBM: only the new keyframe's feature cloud is ever uploaded.
 *   lvb_icp_map_append  ToWorld of one keyframe: float32 transform by `pose` (Twc.cast<float>()), stored under `key`.
 *                       robot_points == NULL: the scan the last lvb_icp_scan_to_map / knn3 / eval call left on the device.
 *   lvb_icp_map_evict   drop a keyframe's cloud (key < 0: all).
 *   lvb_icp_map_build   BuildMapFrame: merged = cloud[keys[0]] += cloud[keys[1]] ... in that order (a point's index = its position in
 *                       the merged cloud, as in the per-call path); ground_threshold > 0 runs SegmentGround (plane RANSAC, that
 *                       distance threshold) on the merged cloud first; then the voxel hash -- all on the device.
 *   lvb_icp_map_download the merged map cloud (x y z 0) in merge order, for checks and visualisation. */
LVB_API int lvb_icp_map_append(lvb_icp* icp, long long key, const void* robot_points, int n, int stride_bytes, const double pose[7]);
LVB_API int lvb_icp_map_evict(lvb_icp* icp, long long key);
LVB_API int lvb_icp_map_build(lvb_icp* icp, const long long* keys, int n_keys, float cell_size, double ground_threshold, int* n_points);
LVB_API int lvb_icp_map_download(lvb_icp* icp, float* xyzi, int capacity, int* n_points);
/* Batched KdTreeFLANN::nearestKSearch(point, 3, idx, d2) for every scan point after the
 * float32 SE3 transform of association.cpp:287-294.  Exact 3-NN among map points with
 * d2 <= max_d2 (max_d2 <= cell_size^2), ascending by (d2, index); missing neighbours are
 * idx = -1, d2 = +inf.  idx, d2 are n x 3. */
LVB_API int lvb_icp_knn3(lvb_icp* icp, const void* scan, int n, int stride_bytes, const double frame_pose[7],
                 float max_d2, int32_t* idx, float* d2);
/* Mapping::MergeScan / ToWorld (mapping.cpp:193-220): out[i].xyz = float32 SE3 transform of points[i].xyz with
 * pose.cast<float>() (same arithmetic as the query transform of association.cpp:294); the remaining bytes of each
 * record (intensity, padding) are copied.  points and out are n records of stride_bytes. */
LVB_API int lvb_icp_transform_cloud(lvb_icp* icp, const void* points, int n, int stride_bytes, const double pose[7], void* out);
/* Per scan point: the gate of association.cpp:296-300 and, for accepted points, the raw
 * LidarPlaneErrorRPZ (mode 0) / LidarPlaneErrorYXY (mode 1) residual and 1x3 Jacobian
 * (ceres/lidar_error.hpp:42-110) at rpyxyz.  Rejected rows are zero.  Parity entry. */
LVB_API int lvb_icp_eval(lvb_icp* icp, int mode, const void* scan, int n, int stride_bytes,
                 const double frame_pose[7], const double map_pose[7], const double rpyxyz[6],
                 double weight, double dist_thr, uint8_t* accepted, double* r, double* J);
/* ScanToMapWithGround (mode 0) / ScanToMapWithSegmented (mode 1) followed by adapt::Solve:
 * associates, then runs the LM on the three free scalars of rpyxyz (updated in place).
 * prior_weight < 0 omits the PoseErrorRPZ/YXY prior (relocate = true); huber_a <= 0 is
 * TrivialLoss (association.cpp:272), 0.1 for the segmented cloud (:330).
 * summary->num_residual_blocks = accepted correspondences (+1 with the prior). */
LVB_API int lvb_icp_scan_to_map(lvb_icp* icp, int mode, const void* scan, int n, int stride_bytes,
                        const double frame_pose[7], const double map_pose[7], double rpyxyz[6],
                        double weight, double prior_weight, double huber_a, double dist_thr,
                        const lvb_solve_options* options, lvb_solve_summary* summary);
/* Mapping::Optimize for one keyframe (mapping.cpp:147-185) against the map frame lvb_icp_map_build made on each handle:
 *   rpyxyz = se32rpyxyz(map_pose^-1 * pose)                                        (computed once, from the incoming pose)
 *   ground: ScanToMapWithGround + Solve, pose = map_pose * rpyxyz2se3(rpyxyz)
 *   surf:   ScanToMapWithSegmented + Solve from that rpyxyz, queries transformed by the pose the ground solve produced; pose again
 *   ToWorld: each robot-frame cloud, transformed by pose.cast<float>(), is stored under `key` in its handle, replacing what `key`
 *            held; lvb_icp_map_append(NULL) on a handle afterwards refers to this call's cloud.
 * All on the device with one host synchronisation, at the end.  Index [0] of weight / huber_a / dist_thr / summary is the ground
 * registration, [1] the surf one, with the meaning lvb_icp_scan_to_map gives them; prior_weight < 0 omits both priors.
 * A NULL handle skips that registration and its ToWorld (mapping.cpp:155,167 skip a registration whose map cloud is empty); its
 * summary is zero with termination_type = -1.  ToWorld still stores that keyframe's cloud in the reference (mapping.cpp:215-216):
 * the caller does it with lvb_icp_map_evict(key) + lvb_icp_map_append(key, cloud, returned pose) on that side's handle
 * (lvio_b200/association.h, OptimizeKeyframe, does).  Both handles belong to one context.  total_time_in_seconds is the whole call's.
 * LVB_ERR_STATE when a handle has no map; LVB_ERR_INVALID when options.max_solver_time_in_seconds is set (< 1e8: Mapping::Optimize
 * sets no limit, and the call decides nothing on the host); LVB_ERR_UNSUPPORTED on a context with world_size > 1 (sharded
 * registration: lvb_icp_scan_to_map).  Errors are reported before any state changes. */
typedef struct lvb_map_optimize_params {
    double weight[2], prior_weight, huber_a[2], dist_thr[2];   /* association.cpp:270-384 */
    lvb_solve_options options;                                 /* mapping.cpp:159-162: DENSE_QR, max_num_iterations = 4 */
} lvb_map_optimize_params;
LVB_API int lvb_icp_map_optimize_keyframe(lvb_icp* ground, lvb_icp* surf, const double map_pose[7], long long key,
                                          const void* ground_pts, int n_ground, const void* surf_pts, int n_surf, int stride_bytes,
                                          const lvb_map_optimize_params* p, double pose[7] /* in: frame->pose, out: optimised */,
                                          double rpyxyz[6] /* out */, lvb_solve_summary summary[2]);
/* Mapping::BuildMapFrame + the body of Mapping::Optimize's loop for one keyframe (mapping.cpp:114-137, 147-185): the two
 * lvb_icp_map_build calls and lvb_icp_map_optimize_keyframe in one call, with one host synchronisation.
 * It runs as the chain of one: lvb_icp_map_optimize_keyframes' implementation with this keyframe and p's weights and prior weight.
 *   keys / n_keys  the map frame's keyframes in merge order, as for lvb_icp_map_build, resident on both handles; `key` may not be one
 *                  of them.  n_keys == 0 is the first lidar keyframe (BuildMapFrame returns early, :118-119): nothing is registered
 *                  and both clouds are stored at the incoming pose.
 *   cell_size[2], ground_threshold  what the two lvb_icp_map_build calls take: SegmentGround (plane RANSAC, ground_threshold > 0) on
 *                  the merged cloud of handle `ground`, none on `surf`.
 *   Both handles are required: ToWorld stores both clouds under `key` (:185), replacing what `key` held.  A side is not registered
 *   -- its summary is zero with termination_type = -1 -- when its merged cloud is empty (:155,167) or SegmentGround keeps no point;
 *   its cloud is still stored, with the pose the other registration produced, and its previous map frame stays.  The registrations,
 *   weights, gates and pose hand-off are lvb_icp_map_optimize_keyframe's.  rpyxyz = se32rpyxyz(map_pose^-1 * pose) of the incoming
 *   pose, then updated by each registration that ran.  n_map_points (may be NULL): each map frame's size (0 = not built).
 * Afterwards each handle is in the state lvb_icp_map_build + lvb_icp_map_optimize_keyframe leave it in (knn3, scan_to_map,
 * map_download, map_append(NULL) work on it).  The map frame's voxel grid is decided on the device; the host sizes its buffers from
 * the bounding boxes of the resident clouds, recorded when this call stores a cloud.  A resident cloud stored by another entry point
 * has none: the first call that merges it computes it, at the cost of one more host synchronisation, and keeps it.
 * Errors as lvb_icp_map_optimize_keyframe, plus LVB_ERR_INVALID for an unknown key or `key` among `keys`.  Failures found on the
 * device -- a map frame with no finite bounding box (LVB_ERR_INVALID), a grid above 2^26 voxels at the coarsest ring
 * (LVB_ERR_UNSUPPORTED) -- are reported after the synchronisation and leave every resident cloud and map frame as they were. */
LVB_API int lvb_icp_map_build_optimize_keyframe(lvb_icp* ground, lvb_icp* surf, const long long* keys, int n_keys,
                                                const float cell_size[2], double ground_threshold, const double map_pose[7], long long key,
                                                const void* ground_pts, int n_ground, const void* surf_pts, int n_surf, int stride_bytes,
                                                const lvb_map_optimize_params* p, double pose[7] /* in: frame->pose, out: optimised */,
                                                double rpyxyz[6] /* out */, lvb_solve_summary summary[2], int n_map_points[2]);
/* Mapping::Optimize(active_kfs) (mapping.cpp:139-191) for the n_kf lidar keyframes of a backend pass, in time order, in one call with
 * one host synchronisation: for k = 0 .. n_kf-1, on the device,
 *   incoming pose  pose_k = T_{k-1} * ( ... (T_0 * pose)), pose as the caller holds it: the PoseGraph::ForwardUpdate(T_j, t_j + eps)
 *                  of every earlier keyframe of the call, in order (pose_graph.cpp:245-252)
 *   map frame      map_keys (0 to 3, merge order: get_lidar_frames(0, t_k, 3)), each a cloud resident on both handles before the call or
 *                  the key of an earlier keyframe of the call (then the clouds this call stored for it); built as
 *                  lvb_icp_map_build_optimize_keyframe builds it.  map_pose: that of the newest map key -- the optimised pose of that
 *                  keyframe when it is in the call, the record's map_pose otherwise.
 *   registrations  as lvb_icp_map_build_optimize_keyframe: both sides, the pose hand-off, a side with an empty merged cloud or whose
 *                  SegmentGround keeps no point is not registered, no map keys register nothing
 *   transform      T_k = pose_k(optimised) * pose_k(incoming)^-1 (mapping.cpp:181-182)
 *   ToWorld        both clouds stored under `key`, replacing what it held; later keyframes of the call merge them from there.
 * Every SE3 product and inverse rounds each double operation on its own: lvio_fusion_b200/se3.py restates them bit for bit, and
 * replaying ForwardUpdate(transform, t_k + eps) with Sophus on the host moves the frames after each keyframe as the reference does.
 * The records are read (inputs) and written (outputs, only when the call succeeds).  Each record's weight[2] and prior_weight are that
 * keyframe's (ScanToMapWith* take them from each frame: the lidar weights and features_left.size() * weights.visual, association.cpp:
 * 318-323, 376-381) and replace p's; the rest of p, cell_size[2], ground_threshold and stride_bytes are
 * lvb_icp_map_build_optimize_keyframe's and apply to every keyframe.  Each summary's total_time_in_seconds is the whole call's.  Keys of the call are distinct.  The launch sequence depends
 * only on the sizes and the options.  n_kf == 1 is lvb_icp_map_build_optimize_keyframe, bit for bit, with the same launches and
 * synchronisations; n_kf == 0 launches and waits for nothing.
 * Afterwards each handle is as the step-by-step loop leaves it: its map frame is the newest one built with points, map_append(NULL)
 * refers to the last keyframe's scan.  A map frame that merges clouds of the call is sized from their robot-frame boxes at the
 * incoming poses the caller gave, widened by 1 m; a cloud that ends up outside makes that grid coarser (the 3-NN stays exact), and
 * only a grid that does not fit at ring 1 fails (LVB_ERR_UNSUPPORTED).
 * Errors, all before any state changes: as lvb_icp_map_build_optimize_keyframe (time limit set, sharded context, handles of different
 * contexts, bad cell size or gate), and LVB_ERR_INVALID for a map key that is neither resident nor an earlier keyframe of the call, a
 * key listed twice, a key among its own map keys, or n_map_keys outside 0..3.  Failures found on the device in any keyframe (no finite
 * bounding box, grid overflow) are reported after the synchronisation and commit nothing: every resident cloud, map frame and the
 * map_append(NULL) scan stay as they were. */
typedef struct lvb_map_keyframe {
    long long key;                          /* in: the keyframe's time key */
    long long map_keys[3];                  /* in: its map frame's keys, merge order */
    int n_map_keys;                         /* in: 0 to 3 */
    int n_ground, n_surf;                   /* in: robot-frame cloud sizes (< 0 with NULL clouds: by key, lvb_icp_map_extract_keyframe) */
    const void* ground_pts;                 /* in: n_ground records of stride_bytes */
    const void* surf_pts;                   /* in: n_surf records */
    double map_pose[7];                     /* in: the newest map key's pose (unused when it is a keyframe of the call) */
    double pose[7];                         /* in: frame->pose; out: optimised */
    double weight[2];                       /* in: ground, surf registration weight of this keyframe */
    double prior_weight;                    /* in: this keyframe's prior weight (< 0: no prior) */
    double transform[7];                    /* out: T_k */
    double rpyxyz[6];                       /* out */
    lvb_solve_summary summary[2];           /* out: ground, surf; termination_type -1 when not registered */
    int n_map_points[2];                    /* out: each map frame's size (0 = not built) */
} lvb_map_keyframe;
LVB_API int lvb_icp_map_optimize_keyframes(lvb_icp* ground, lvb_icp* surf, lvb_map_keyframe* kfs, int n_kf, const float cell_size[2],
                                           double ground_threshold, int stride_bytes, const lvb_map_optimize_params* p);
/* Mapping::Relocate for one loop-closure candidate (mapping.cpp:78-112, 251-300), with one host synchronisation:
 *   pose = old_pose * relative_guess                                 (clone_frame->pose, :256)
 *   BuildOldMapFrame: the map frame of keys / n_keys (1 to 3: the lidar keyframe before the old one, the old one if it has lidar, the
 *                  one after it, in time order), resident on both handles, merged in that order, SegmentGround (ground_threshold > 0)
 *                  on the ground side, hashed with cell_size[2] -- into a relocation slot of each handle, reused by every call and never
 *                  made the handle's map frame.  map_pose: the pose of the EARLIEST of the keys (old_frames.begin(), :106-108).
 *   `rounds` rounds (the reference runs 4; 1 to 16): rpyxyz = se32rpyxyz(map_pose^-1 * pose), ScanToMapWithGround + Solve, pose =
 *                  map_pose * rpyxyz2se3(rpyxyz), ScanToMapWithSegmented + Solve, pose again -- as in lvb_icp_map_optimize_keyframe,
 *                  and always without the prior: p->prior_weight must be < 0 (relocate = true).
 *   relative_o_c = old_pose^-1 * pose (:298); pose: the final clone pose.
 *   score[m] = min(n / 10, cap) - 2 final_cost / n of the last round's registration m (:281-282, :294-295; n =
 *                  num_residual_blocks_reduced, cap 20 ground / 30 surf), in FP64; NaN when that side did not run or n == 0.  The
 *                  reference returns (int)(score[0] + score[1]).
 * summary[2] is the last round's (may be NULL, as may score and n_map_points).  A side whose merged cloud is empty or whose
 * SegmentGround keeps no point is skipped in every round: summary zero with termination_type = -1, score NaN, n_map_points 0.
 * Nothing is stored: knn3, map_download, scan_to_map and map_append(NULL) on either handle behave afterwards as before the call, and
 * every resident cloud is unchanged.  The launch sequence depends only on the sizes and options, not on when a solver stops or how
 * many points SegmentGround keeps.  A resident cloud without a recorded bounding box costs one more synchronisation, once.
 * Errors, all before any state changes: as lvb_icp_map_build_optimize_keyframe (unknown key, time limit set, sharded context), and
 * LVB_ERR_INVALID for n_keys outside 1..3, rounds outside 1..16 or prior_weight >= 0; failures found on the device (no finite bounding
 * box, grid overflow) leave every cloud and map frame as they were.  Threading: read-only on the store; it may run on handles
 * lvb_icp_share made (another thread's context) concurrently with any call on the same store (see lvb_icp_share). */
LVB_API int lvb_icp_map_relocate(lvb_icp* ground, lvb_icp* surf, const long long* keys, int n_keys, const float cell_size[2],
                                 double ground_threshold, const double map_pose[7], const double old_pose[7], const double relative_guess[7],
                                 const void* ground_pts, int n_ground, const void* surf_pts, int n_surf, int stride_bytes,
                                 const lvb_map_optimize_params* p, int rounds, double relative_o_c[7] /* out */, double pose[7] /* out */,
                                 lvb_solve_summary summary[2], double score[2], int n_map_points[2]);
/* Mapping::ToWorld for n_keys resident keyframes at once (src/mapping.cpp:206-229; called by Mapping::ToWorld(start) after a
 * GNSS or loop correction, backend.cpp:71-91, relocator.cpp:236-244): the world cloud under keys[i] becomes the float32 SE3
 * transform of that keyframe's robot-frame cloud (kept on the device since it was stored) by poses[i].cast<float>().
 *   Each re-anchored cloud is bit for bit what lvb_icp_map_evict(key) + lvb_icp_map_append(key, robot cloud, poses[i]) stores, whichever
 *   entry point stored it first: the result depends on the robot-frame cloud and poses[i] only, so repeated calls accumulate no error
 *   and re-anchoring at the pose a cloud was stored with changes nothing.
 *   ground / surf: one may be NULL; every key must be resident on every handle given; the two must belong to one context.
 *   keys may come in any order; poses: n_keys x 7 doubles, [qx qy qz qw tx ty tz].
 * One pinned upload, one kernel over every point of every listed cloud, one host synchronisation, whatever n_keys is; n_keys == 0
 * launches and waits for nothing.  The bounding boxes of the new clouds are recorded, so the next lvb_icp_map_build_optimize_keyframe
 * or lvb_icp_map_relocate that merges them pays no extra synchronisation for them.
 * The world clouds are overwritten in place (on a shared store: replaced by new buffers, see lvb_icp_share); nothing else changes: the handles' map frames (copies made by their builds), the
 * relocation slots, the scan lvb_icp_map_append(NULL) refers to and every cloud not listed stay as they were.  Nothing is exchanged
 * between ranks: the call is not collective on a sharded context.
 * Errors, all before any state changes: LVB_ERR_INVALID for an unknown or duplicated key, NULL keys / poses with n_keys > 0,
 * n_keys < 0, both handles NULL or equal, handles of different contexts. */
LVB_API int lvb_icp_map_to_world(lvb_icp* ground, lvb_icp* surf, const long long* keys, int n_keys, const double* poses /* n_keys x 7 */);

/* ---- lidar feature pipeline, the producer of the scan-to-map inputs (SURVEY 8(f).2).
 * Stands behind FeatureAssociation::Process (association.cpp:88-268: Preprocess, AdjustDistortion, CalculateSmoothness,
 * ExtractFeatures, SegmentGround, Sensor2Robot) and ImageProjection::Process (projection.cpp:26-320: range-image
 * projection, ground removal, segmentation), plus the three PCL filters they call (VoxelGrid, RadiusOutlierRemoval,
 * SACSegmentation plane RANSAC).  Clouds are arrays of `x y z intensity` float32 (pcl::PointXYZI without padding) unless
 * a stride is given. */
typedef struct lvb_lidar_config {
    int32_t num_scans, horizon_scan;         /* kitti.yaml:35-36 */
    double ang_res_y, ang_bottom;            /* :37-38 */
    int32_t ground_rows, reserved;           /* :39 */
    double cycle_time, min_range, max_range; /* :40-42 */
    double resolution;                       /* :45, Lidar::resolution */
    double extrinsic[7];                     /* T_body_lidar, Sophus layout (estimator.cpp:133-141) */
} lvb_lidar_config;
LVB_API void lvb_lidar_default_config(lvb_lidar_config* cfg);   /* the kitti.yaml values, identity extrinsic */
/* Preprocess + ImageProjection::Process + AdjustDistortion + CalculateSmoothness.  Outputs have capacity
 * num_scans * horizon_scan; orientation = {start, end, diff}; any output pointer may be NULL. */
LVB_API int lvb_lidar_segment(lvb_ctx* ctx, const lvb_lidar_config* cfg, const void* points, int n, int stride_bytes,
                              float* seg_xyzi, float* seg_range, uint8_t* seg_ground, int32_t* seg_col, float* seg_curvature,
                              int32_t* start_ring /* num_scans */, int32_t* end_ring /* num_scans */, float orientation[3], int32_t* n_seg);
/* pcl::VoxelGrid (cubic leaf, all fields averaged, output ordered by voxel index); out capacity n */
LVB_API int lvb_lidar_voxel_grid(lvb_ctx* ctx, const float* xyzi, int n, float leaf, float* out_xyzi, int32_t* n_out);
/* pcl::RadiusOutlierRemoval: keeps points with >= min_neighbors points (itself included) closer than radius */
LVB_API int lvb_lidar_radius_outlier_removal(lvb_ctx* ctx, const float* xyzi, int n, double radius, int min_neighbors, float* out_xyzi, int32_t* n_out);
/* FeatureAssociation::SegmentGround (association.cpp:254-268): inliers of the RANSAC plane (100 iterations, p = 0.99) */
LVB_API int lvb_lidar_segment_ground(lvb_ctx* ctx, const float* xyzi, int n, double distance_threshold, float* out_xyzi, int32_t* n_out);
/* FeatureAssociation::Process: raw scan -> frame->feature_lidar {points_ground, points_surf} in the robot frame.
 * Output capacity num_scans * horizon_scan points each.  One host synchronisation: every stage keeps its count on the device. */
LVB_API int lvb_lidar_extract_features(lvb_ctx* ctx, const lvb_lidar_config* cfg, const void* points, int n, int stride_bytes,
                                       float* ground_xyzi, int32_t* n_ground, float* surf_xyzi, int32_t* n_surf);

/* FeatureAssociation::Process into the resident map (association.cpp:85-109: AddScan -> Process fills frame->feature_lidar, which
 * Mapping::Optimize registers and stores through ToWorld, mapping.cpp:139-220): lvb_lidar_extract_features on the handles' context, and
 * the two robot-frame feature clouds stay on the device as the PENDING FEATURES of `key` -- the ground cloud on `ground`, the surf cloud
 * on `surf`, as packed 16-byte (x, y, z, intensity) records with their robot-frame bounding boxes.  One host synchronisation brings back
 * the counts (always) and the host copies (ground_xyzi / surf_xyzi may be NULL; capacity num_scans * horizon_scan points each) -- the
 * same points, in the same order, as lvb_lidar_extract_features.
 *   Registering by key: an lvb_map_keyframe record (or lvb_icp_map_build_optimize_keyframe's arguments) with ground_pts == NULL &&
 *   n_ground < 0 and surf_pts == NULL && n_surf < 0 takes the pending features of its key as its two clouds: nothing is uploaded for
 *   them, and they are read as their own 16-byte records (stride_bytes must still be valid: >= 12, a multiple of 4).  Both sides by
 *   key or neither; a by-key record without pending features on both handles is LVB_ERR_INVALID before any state changes.  Each
 *   pending cloud is kept in a buffer of exactly its points; on success it becomes the stored keyframe's robot-frame cloud as it is
 *   (no copy) and the pending entry is gone; on any failure it stays.  The launches and synchronisations are those of the same call fed
 *   with the host copies (stride 16).
 *   Pending features are not resident: lvb_icp_map_build, lvb_icp_map_relocate, lvb_icp_map_to_world and the map keys of the keyframe
 *   calls do not know a pending-only key.  lvb_icp_map_evict(key) drops them (key < 0: all); another extraction under the same key
 *   replaces them.
 * Errors, all before any state changes: LVB_ERR_INVALID for a bad configuration or cloud arguments (lvb_lidar_extract_features'),
 * NULL or equal handles, NULL n_ground / n_surf, handles of different contexts; a feature voxel grid above 2^26 voxels is
 * LVB_ERR_UNSUPPORTED, found on the device and reported after the synchronisation, storing nothing.  Not collective: allowed on a
 * sharded context.  Threading: it may run on handles lvb_icp_share made (another thread's context) concurrently with the keyframe
 * calls and relocations on the same store (see lvb_icp_share). */
LVB_API int lvb_icp_map_extract_keyframe(lvb_icp* ground, lvb_icp* surf, const lvb_lidar_config* cfg, long long key,
                                         const void* points, int n, int stride_bytes,
                                         int32_t* n_ground, int32_t* n_surf,              /* out, always */
                                         float* ground_xyzi, float* surf_xyzi);           /* out, may be NULL */

/* ---- profiling hooks (used by tools/kernel_timing*.py; not part of the drop-in surface) */
/* enable != 0: record a CUDA event after every kernel of the BA pass (disables the graph); 0: print the per-kernel times */
LVB_API int lvb_debug_timing(int enable);
/* as lvb_debug_timing(0), but writes "kernel_name microseconds" lines (launch order) into out instead of printing them */
LVB_API int lvb_debug_timing_report(char* out, int cap);
/* priority[0]: the priority of the context's stream, priority[1]: that of its side stream */
LVB_API int lvb_debug_ctx_stream_priorities(lvb_ctx* ctx, int priority[2]);
/* the capacities, in 16-byte records, of the buffers the handle keeps for `key`: cap[0] its resident world cloud, cap[1] its
 * robot-frame cloud, cap[2] its pending features (-1: none) */
LVB_API int lvb_debug_icp_cloud_capacity(lvb_icp* icp, long long key, long long cap[3]);
/* the voxel grid of the handle's current map frame: grid[0] = ring (voxels per search radius: 4, 2 or 1), grid[1..3] = voxels per
 * axis.  LVB_ERR_STATE without a map frame. */
LVB_API int lvb_debug_icp_map_grid(lvb_icp* icp, int grid[4]);
/* the reduced-system solver alone (parity test of the multifrontal tree, ba_tree.cuh): S x = b for an SPD band matrix stored as
 * n rows of band + 1 entries (row i = columns i - band .. i), true half bandwidth <= band - 31; use_tree 0 forces the single-CTA
 * envelope kernel (or, when its panel does not fit in shared memory, the per-phase grids of ba_wide.cuh); *levels_out = tree levels
 * used (0: no tree) */
LVB_API int lvb_debug_band_solve(lvb_ctx* ctx, int n, int band, const double* S_band, const double* b, double* x, int use_tree, int* levels_out);
/* SM clock counters of ba_cholesky_kernel summed over calls, as seen by the warp that carries the pivot chain:
 * {diagonal tile + factorisation, its panel rows, wait for the other warps, backward pass, total, calls, -, -} */
LVB_API int lvb_debug_cholesky_clocks(long long out[8], int reset);

#ifdef __cplusplus
}
#endif
#endif /* LVIO_B200_H_ */
