"""ctypes binding of the C ABI in include/lvio_b200.h.

The product library is ``lvio_fusion_b200/csrc/liblvio_b200.so`` (CUDA, sm_90a).  There is
no CPU fallback: if the library is missing or no device is usable the calls raise.

The signature table is prefix-agnostic so that ``oracle/binding.py`` (test infrastructure)
can bind the CPU oracle's ``orc_*`` mirror of the same ABI for parity checks.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "liblvio_b200.so")

c_double_p = C.POINTER(C.c_double)
c_int32_p = C.POINTER(C.c_int32)
c_uint8_p = C.POINTER(C.c_uint8)
c_float_p = C.POINTER(C.c_float)
c_int_p = C.POINTER(C.c_int)


class SolveOptions(C.Structure):
    """lvb_solve_options -- ceres::Solver::Options subset (include/lvio_b200.h)."""
    _fields_ = [
        ("max_num_iterations", C.c_int),
        ("max_solver_time_in_seconds", C.c_double),
        ("function_tolerance", C.c_double),
        ("gradient_tolerance", C.c_double),
        ("parameter_tolerance", C.c_double),
        ("initial_trust_region_radius", C.c_double),
        ("jacobi_scaling", C.c_int),
        ("linear_solver_type", C.c_int),
        ("num_threads", C.c_int),
        ("schur_mode", C.c_int),
    ]


class SolveSummary(C.Structure):
    """lvb_solve_summary -- ceres::Solver::Summary subset."""
    _fields_ = [
        ("initial_cost", C.c_double),
        ("final_cost", C.c_double),
        ("num_iterations", C.c_int),
        ("num_successful_steps", C.c_int),
        ("termination_type", C.c_int),
        ("num_residual_blocks", C.c_int),
        ("num_residual_blocks_reduced", C.c_int),
        ("final_radius", C.c_double),
        ("total_time_in_seconds", C.c_double),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class LidarConfig(C.Structure):
    """lvb_lidar_config (include/lvio_b200.h): kitti.yaml:35-45 + the lidar extrinsic."""
    _fields_ = [
        ("num_scans", C.c_int32), ("horizon_scan", C.c_int32),
        ("ang_res_y", C.c_double), ("ang_bottom", C.c_double),
        ("ground_rows", C.c_int32), ("reserved", C.c_int32),
        ("cycle_time", C.c_double), ("min_range", C.c_double), ("max_range", C.c_double),
        ("resolution", C.c_double),
        ("extrinsic", C.c_double * 7),
    ]


class MapOptimizeParams(C.Structure):
    """lvb_map_optimize_params (include/lvio_b200.h): [0] ground registration, [1] surf registration."""
    _fields_ = [
        ("weight", C.c_double * 2),
        ("prior_weight", C.c_double),
        ("huber_a", C.c_double * 2),
        ("dist_thr", C.c_double * 2),
        ("options", SolveOptions),
    ]


class MapKeyframe(C.Structure):
    """lvb_map_keyframe (include/lvio_b200.h): one keyframe of lvb_icp_map_optimize_keyframes, inputs and outputs."""
    _fields_ = [
        ("key", C.c_longlong),
        ("map_keys", C.c_longlong * 3),
        ("n_map_keys", C.c_int),
        ("n_ground", C.c_int),
        ("n_surf", C.c_int),
        ("ground_pts", C.c_void_p),
        ("surf_pts", C.c_void_p),
        ("map_pose", C.c_double * 7),
        ("pose", C.c_double * 7),
        ("weight", C.c_double * 2),
        ("prior_weight", C.c_double),
        ("transform", C.c_double * 7),
        ("rpyxyz", C.c_double * 6),
        ("summary", SolveSummary * 2),
        ("n_map_points", C.c_int * 2),
    ]


VP = C.c_void_p
_SIGS = {
    "version": (C.c_int, []),
    "default_options": (None, [C.POINTER(SolveOptions)]),
    "ctx_create": (C.c_int, [C.c_int, VP, C.POINTER(VP)]),
    "ctx_destroy": (None, [VP]),
    "last_error": (C.c_char_p, []),
    "launch_count": (C.c_longlong, [VP]),
    "ctx_synchronize": (C.c_int, [VP]),
    "ba_create": (C.c_int, [VP, C.POINTER(VP)]),
    "ba_destroy": (None, [VP]),
    "ba_set_cameras": (C.c_int, [VP, c_double_p]),
    "ba_set_poses": (C.c_int, [VP, C.c_int, c_double_p, c_uint8_p]),
    "ba_set_vec3": (C.c_int, [VP, C.c_int, c_double_p, c_uint8_p]),
    "ba_set_inv_depths": (C.c_int, [VP, C.c_int, c_double_p, c_uint8_p]),
    "ba_add_factors": (C.c_int, [VP, C.c_int, C.c_int, c_double_p, c_int32_p]),
    "ba_set_loss": (C.c_int, [VP, C.c_int, C.c_double]),
    "ba_finalize": (C.c_int, [VP]),
    "ba_dims": (C.c_int, [VP, c_int_p, c_int_p, c_int_p]),
    "ba_update_params": (C.c_int, [VP, c_double_p, c_double_p, c_double_p]),
    "ba_eval": (C.c_int, [VP, C.c_int, c_double_p, c_double_p]),
    "ba_eval_device": (C.c_int, [VP, C.c_int]),
    "ba_reduced_system": (C.c_int, [VP, C.c_double, c_double_p, c_double_p, c_double_p]),
    "ba_solve": (C.c_int, [VP, C.POINTER(SolveOptions), C.POINTER(SolveSummary)]),
    "ba_get_poses": (C.c_int, [VP, c_double_p]),
    "ba_get_vec3": (C.c_int, [VP, c_double_p]),
    "ba_get_inv_depths": (C.c_int, [VP, c_double_p]),
    "ba_reprojection_errors": (C.c_int, [VP, C.c_int, c_double_p, c_int32_p, c_double_p]),
    "imu_preintegrate": (C.c_int, [VP, C.c_int, c_int32_p, c_double_p, c_double_p, c_double_p, c_double_p, c_double_p, c_double_p, c_double_p]),
    "lidar_default_config": (None, [C.POINTER(LidarConfig)]),
    "lidar_segment": (C.c_int, [VP, C.POINTER(LidarConfig), VP, C.c_int, C.c_int, c_float_p, c_float_p, c_uint8_p, c_int32_p, c_float_p,
                                c_int32_p, c_int32_p, c_float_p, c_int32_p]),
    "lidar_voxel_grid": (C.c_int, [VP, c_float_p, C.c_int, C.c_float, c_float_p, c_int32_p]),
    "lidar_radius_outlier_removal": (C.c_int, [VP, c_float_p, C.c_int, C.c_double, C.c_int, c_float_p, c_int32_p]),
    "lidar_segment_ground": (C.c_int, [VP, c_float_p, C.c_int, C.c_double, c_float_p, c_int32_p]),
    "lidar_extract_features": (C.c_int, [VP, C.POINTER(LidarConfig), VP, C.c_int, C.c_int, c_float_p, c_int32_p, c_float_p, c_int32_p]),
    "icp_create": (C.c_int, [VP, C.POINTER(VP)]),
    "icp_destroy": (None, [VP]),
    "icp_set_map": (C.c_int, [VP, VP, C.c_int, C.c_int, C.c_float]),
    "icp_transform_cloud": (C.c_int, [VP, VP, C.c_int, C.c_int, c_double_p, VP]),
    "icp_knn3": (C.c_int, [VP, VP, C.c_int, C.c_int, c_double_p, C.c_float, c_int32_p, c_float_p]),
    "icp_eval": (C.c_int, [VP, C.c_int, VP, C.c_int, C.c_int, c_double_p, c_double_p, c_double_p,
                           C.c_double, C.c_double, c_uint8_p, c_double_p, c_double_p]),
    "icp_scan_to_map": (C.c_int, [VP, C.c_int, VP, C.c_int, C.c_int, c_double_p, c_double_p, c_double_p,
                                  C.c_double, C.c_double, C.c_double, C.c_double,
                                  C.POINTER(SolveOptions), C.POINTER(SolveSummary)]),
}
# entry points only the CUDA library exports
_LVB_ONLY = {
    "comm_unique_id": (C.c_int, [C.c_char_p]),
    # stream priorities: the CPU oracle has no streams to schedule
    "ctx_create_with_priority": (C.c_int, [C.c_int, C.c_int, C.POINTER(VP)]),
    "ctx_priority": (C.c_int, [VP, c_int_p]),
    "device_priority_range": (C.c_int, [C.c_int, c_int_p, c_int_p]),
    "comm_init": (C.c_int, [VP, C.c_int, C.c_int, C.c_char_p]),
    "ba_set_schur_mode": (C.c_int, [VP, C.c_int]),
    "icp_share": (C.c_int, [VP, VP, C.POINTER(VP)]),
    "icp_map_append": (C.c_int, [VP, C.c_longlong, VP, C.c_int, C.c_int, c_double_p]),
    "icp_map_evict": (C.c_int, [VP, C.c_longlong]),
    "icp_map_build": (C.c_int, [VP, C.POINTER(C.c_longlong), C.c_int, C.c_float, C.c_double, c_int_p]),
    "icp_map_download": (C.c_int, [VP, c_float_p, C.c_int, c_int_p]),
    "icp_map_optimize_keyframe": (C.c_int, [VP, VP, c_double_p, C.c_longlong, VP, C.c_int, VP, C.c_int, C.c_int,
                                            C.POINTER(MapOptimizeParams), c_double_p, c_double_p, C.POINTER(SolveSummary)]),
    "icp_map_build_optimize_keyframe": (C.c_int, [VP, VP, C.POINTER(C.c_longlong), C.c_int, c_float_p, C.c_double, c_double_p, C.c_longlong,
                                                  VP, C.c_int, VP, C.c_int, C.c_int, C.POINTER(MapOptimizeParams), c_double_p, c_double_p,
                                                  C.POINTER(SolveSummary), c_int_p]),
    "icp_map_relocate": (C.c_int, [VP, VP, C.POINTER(C.c_longlong), C.c_int, c_float_p, C.c_double, c_double_p, c_double_p, c_double_p,
                                   VP, C.c_int, VP, C.c_int, C.c_int, C.POINTER(MapOptimizeParams), C.c_int, c_double_p, c_double_p,
                                   C.POINTER(SolveSummary), c_double_p, c_int_p]),
    "icp_map_to_world": (C.c_int, [VP, VP, C.POINTER(C.c_longlong), C.c_int, c_double_p]),
    "icp_map_optimize_keyframes": (C.c_int, [VP, VP, C.POINTER(MapKeyframe), C.c_int, c_float_p, C.c_double, C.c_int,
                                             C.POINTER(MapOptimizeParams)]),
    "icp_map_extract_keyframe": (C.c_int, [VP, VP, C.POINTER(LidarConfig), C.c_longlong, VP, C.c_int, C.c_int, c_int32_p, c_int32_p,
                                           c_float_p, c_float_p]),
    "sync_count": (C.c_longlong, [VP]),
    "debug_timing": (C.c_int, [C.c_int]),
    "debug_cholesky_clocks": (C.c_int, [C.POINTER(C.c_longlong), C.c_int]),
    "debug_timing_report": (C.c_int, [C.c_char_p, C.c_int]),
    "debug_ctx_stream_priorities": (C.c_int, [VP, c_int_p]),
    "debug_icp_map_grid": (C.c_int, [VP, c_int_p]),
    "debug_icp_cloud_capacity": (C.c_int, [VP, C.c_longlong, C.POINTER(C.c_longlong)]),
    "debug_band_solve": (C.c_int, [VP, C.c_int, C.c_int, c_double_p, c_double_p, c_double_p, C.c_int, c_int_p]),
}

EXPORTED_SYMBOLS = ["lvb_" + k for k in list(_SIGS) + list(_LVB_ONLY)]


class Api:
    """Function table bound to one shared library with one prefix."""

    def __init__(self, lib, prefix, extra=None):
        self.lib = lib
        self.prefix = prefix
        table = dict(_SIGS)
        if extra:
            table.update(extra)
        for name, (res, args) in table.items():
            fn = getattr(lib, prefix + "_" + name)
            fn.restype = res
            fn.argtypes = args
            setattr(self, name, fn)

    def check(self, code, what=""):
        if code != 0:
            msg = self.last_error()
            raise RuntimeError("%s_%s failed (%d): %s" % (self.prefix, what, code, (msg or b"").decode()))


_api = None


def load():
    """Load the CUDA library.  Raises if it has not been built (run __graft_entry__.build())."""
    global _api
    if _api is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("liblvio_b200.so not built: %s missing (python -c 'import __graft_entry__ as g; g.build()')" % LIB_PATH)
        _api = Api(C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL), "lvb", _LVB_ONLY)
    return _api
