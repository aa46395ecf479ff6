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
 * or NULL to let the context create its own non-blocking stream. */
LVB_API int lvb_ctx_create(int device, void* cuda_stream, lvb_ctx** out);
LVB_API void lvb_ctx_destroy(lvb_ctx* ctx);
LVB_API const char* lvb_last_error(void);            /* thread-local text of the last failure */
LVB_API long long lvb_launch_count(lvb_ctx* ctx);    /* kernels launched through this context so far */
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
 * Output capacity num_scans * horizon_scan points each. */
LVB_API int lvb_lidar_extract_features(lvb_ctx* ctx, const lvb_lidar_config* cfg, const void* points, int n, int stride_bytes,
                                       float* ground_xyzi, int32_t* n_ground, float* surf_xyzi, int32_t* n_surf);

/* ---- profiling hooks (used by tools/kernel_timing*.py; not part of the drop-in surface) */
/* enable != 0: record a CUDA event after every kernel of the BA pass (disables the graph); 0: print the per-kernel times */
LVB_API int lvb_debug_timing(int enable);
/* as lvb_debug_timing(0), but writes "kernel_name microseconds" lines (launch order) into out instead of printing them */
LVB_API int lvb_debug_timing_report(char* out, int cap);
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
