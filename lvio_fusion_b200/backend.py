"""Host-side Python mirror of the reference interfaces on the hot path.

The reference is C++ (its host side is mirrored in C++ under include/lvio_b200/); this module
is the thin Python driver over the same C ABI that the tests and bench.py use.  Names follow
the reference:

* ``Problem``  <- ``adapt::Problem`` + ``adapt::Solve``
  (/root/reference/src/lvio_fusion/include/lvio_fusion/adapt/problem.h:34-88) holding the
  factor mix ``Backend::BuildProblem`` creates (src/backend.cpp:96-183).
* ``FeatureAssociation`` <- ``FeatureAssociation::ScanToMapWithGround/Segmented``
  (src/association.cpp:270-384) + the two solves of ``Mapping::Optimize`` (src/mapping.cpp:139-191).

Every class takes an ``api`` (``lvio_fusion_b200._capi.load()`` for the CUDA library; the tests
also pass the oracle's table, which has the same shape).
"""
import ctypes as C

import numpy as np

from . import _capi
from ._capi import SolveOptions, SolveSummary

TWO_FRAME, POSE_ONLY, TWO_CAMERA, IMU, POSE_GRAPH, POSE_PRIOR = range(6)
KIND_NAMES = ["TwoFrameReprojectionError", "PoseOnlyReprojectionError", "TwoCameraReprojectionError",
              "ImuError", "PoseGraphError", "PoseError"]
CONST_STRIDE = [5, 6, 5, 469, 8, 9]
IDX_STRIDE = [3, 1, 1, 8, 2, 1]
RES_DIM = [2, 2, 2, 15, 6, 6]
JAC_COLS = [15, 7, 1, 32, 14, 7]

SPARSE_SCHUR, SPARSE_NORMAL_CHOLESKY, DENSE_QR = 0, 1, 2


def _dp(a):
    return None if a is None else a.ctypes.data_as(_capi.c_double_p)


def _ip(a):
    return None if a is None else a.ctypes.data_as(_capi.c_int32_p)


def _bp(a):
    return None if a is None else a.ctypes.data_as(_capi.c_uint8_p)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class Context:
    """lvb_ctx: one device + stream."""

    def __init__(self, api=None, device=0, stream=None):
        self.api = api or _capi.load()
        h = C.c_void_p()
        self.api.check(self.api.ctx_create(int(device), C.c_void_p(stream) if stream else None, C.byref(h)), "ctx_create")
        self.h = h

    def launch_count(self):
        return int(self.api.launch_count(self.h))

    def synchronize(self):
        self.api.check(self.api.ctx_synchronize(self.h), "ctx_synchronize")

    def comm_init(self, rank, world, uid):
        self.api.check(self.api.comm_init(self.h, rank, world, uid), "comm_init")

    def close(self):
        if self.h:
            self.api.ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def default_options(api, **kw):
    o = SolveOptions()
    api.default_options(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def preintegrate(ctx, first, samples, acc0, gyr0, ba, bg, noise4):
    """Batched Preintegration::Append/Propagate (preintegration.cpp:30-127); re-running it with new biases is
    Repropagate (:129-142).  Interval i owns samples[first[i]:first[i+1]] (rows `dt acc[3] gyr[3]`).
    Returns the LVB_IMU constant records [n, 469]."""
    first = np.ascontiguousarray(first, dtype=np.int32)
    n = len(first) - 1
    samples, acc0, gyr0, ba, bg, noise4 = (_f64(a) for a in (samples, acc0, gyr0, ba, bg, noise4))
    assert samples.shape == (int(first[-1]), 7) and acc0.shape == gyr0.shape == ba.shape == bg.shape == (n, 3) and noise4.shape == (4,)
    out = np.empty((n, CONST_STRIDE[IMU]), dtype=np.float64)
    ctx.api.check(ctx.api.imu_preintegrate(ctx.h, n, _ip(first), _dp(samples), _dp(acc0), _dp(gyr0), _dp(ba), _dp(bg), _dp(noise4), _dp(out)), "imu_preintegrate")
    return out


class Problem:
    """adapt::Problem analogue: parameter blocks by index, residual blocks by kind."""

    def __init__(self, ctx):
        self.ctx = ctx
        self.api = ctx.api
        h = C.c_void_p()
        self.api.check(self.api.ba_create(ctx.h, C.byref(h)), "ba_create")
        self.h = h
        self.n_poses = self.n_vec3 = self.n_rho = 0
        self.n_factors = [0] * 6

    def close(self):
        if self.h:
            self.api.ba_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_cameras(self, cam22):
        cam22 = _f64(cam22).reshape(22)
        self.api.check(self.api.ba_set_cameras(self.h, _dp(cam22)), "ba_set_cameras")

    def set_poses(self, poses, const=None):
        poses = _f64(poses).reshape(-1, 7)
        c = None if const is None else np.ascontiguousarray(const, dtype=np.uint8)
        self.n_poses = len(poses)
        self.api.check(self.api.ba_set_poses(self.h, len(poses), _dp(poses), _bp(c)), "ba_set_poses")

    def set_vec3(self, v, const=None):
        v = _f64(v).reshape(-1, 3)
        c = None if const is None else np.ascontiguousarray(const, dtype=np.uint8)
        self.n_vec3 = len(v)
        self.api.check(self.api.ba_set_vec3(self.h, len(v), _dp(v), _bp(c)), "ba_set_vec3")

    def set_inv_depths(self, rho, const=None):
        rho = _f64(rho).reshape(-1)
        c = None if const is None else np.ascontiguousarray(const, dtype=np.uint8)
        self.n_rho = len(rho)
        self.api.check(self.api.ba_set_inv_depths(self.h, len(rho), _dp(rho), _bp(c)), "ba_set_inv_depths")

    def add_factors(self, kind, consts, idx):
        consts = _f64(consts).reshape(-1, CONST_STRIDE[kind])
        idx = np.ascontiguousarray(idx, dtype=np.int32).reshape(-1, IDX_STRIDE[kind])
        assert len(consts) == len(idx)
        if len(consts) == 0:
            return
        self.n_factors[kind] += len(consts)
        self.api.check(self.api.ba_add_factors(self.h, kind, len(consts), _dp(consts), _ip(idx)), "ba_add_factors")

    def set_loss(self, kind, huber_a):
        self.api.check(self.api.ba_set_loss(self.h, kind, float(huber_a)), "ba_set_loss")

    def set_schur_mode(self, mode):
        """0 = FP64 Schur (parity reference), 1 = wgmma split-bf16 tensor-core Schur (CUDA library only)."""
        self.api.check(self.api.ba_set_schur_mode(self.h, int(mode)), "ba_set_schur_mode")

    def finalize(self):
        self.api.check(self.api.ba_finalize(self.h), "ba_finalize")

    def dims(self):
        a, b, c = C.c_int(), C.c_int(), C.c_int()
        self.api.check(self.api.ba_dims(self.h, C.byref(a), C.byref(b), C.byref(c)), "ba_dims")
        return a.value, b.value, c.value

    def update_params(self, poses=None, vec3=None, rho=None):
        p = None if poses is None else _f64(poses)
        v = None if vec3 is None else _f64(vec3)
        r = None if rho is None else _f64(rho)
        self.api.check(self.api.ba_update_params(self.h, _dp(p), _dp(v), _dp(r)), "ba_update_params")

    def evaluate(self, kind, jacobians=True):
        n = self.n_factors[kind]
        r = np.zeros((n, RES_DIM[kind]))
        J = np.zeros((n, RES_DIM[kind], JAC_COLS[kind])) if jacobians else None
        self.api.check(self.api.ba_eval(self.h, kind, _dp(r), _dp(J)), "ba_eval")
        return r, J

    def evaluate_device(self, kind):
        self.api.check(self.api.ba_eval_device(self.h, kind), "ba_eval_device")

    def reduced_system(self, radius=1e4):
        dimc, _, _ = self.dims()
        S = np.zeros((dimc, dimc))
        b = np.zeros(dimc)
        cost = C.c_double()
        self.api.check(self.api.ba_reduced_system(self.h, float(radius), _dp(S), _dp(b), C.byref(cost)), "ba_reduced_system")
        return S, b, cost.value

    def solve(self, options=None, **kw):
        o = options or default_options(self.api, **kw)
        s = SolveSummary()
        self.api.check(self.api.ba_solve(self.h, C.byref(o), C.byref(s)), "ba_solve")
        return s

    def poses(self):
        out = np.zeros((self.n_poses, 7))
        self.api.check(self.api.ba_get_poses(self.h, _dp(out)), "ba_get_poses")
        return out

    def vec3(self):
        out = np.zeros((self.n_vec3, 3))
        if self.n_vec3:
            self.api.check(self.api.ba_get_vec3(self.h, _dp(out)), "ba_get_vec3")
        return out

    def inv_depths(self):
        out = np.zeros(self.n_rho)
        if self.n_rho:
            self.api.check(self.api.ba_get_inv_depths(self.h, _dp(out)), "ba_get_inv_depths")
        return out

    def reprojection_errors(self, ob_pw, pose_idx):
        ob_pw = _f64(ob_pw).reshape(-1, 5)
        pose_idx = np.ascontiguousarray(pose_idx, dtype=np.int32)
        err = np.zeros(len(ob_pw))
        self.api.check(self.api.ba_reprojection_errors(self.h, len(ob_pw), _dp(ob_pw), _ip(pose_idx), _dp(err)), "ba_reprojection_errors")
        return err

    @classmethod
    def from_dict(cls, ctx, d):
        """Build from a synth.make_ba_problem() dictionary."""
        p = cls(ctx)
        p.set_cameras(d["cameras"])
        p.set_poses(d["poses"], d.get("pose_const"))
        p.set_vec3(d["vec3"], d.get("vec3_const"))
        p.set_inv_depths(d["rho"], d.get("rho_const"))
        for kind in range(6):
            f = d["factors"].get(kind)
            if f is not None and len(f[0]):
                p.add_factors(kind, f[0], f[1])
        for kind, a in d.get("loss", {}).items():
            p.set_loss(kind, a)
        p.finalize()
        return p


class FeatureAssociation:
    """Scan-to-map matcher: kd-tree replacement + the two ICP solves."""

    GROUND, SEGMENTED = 0, 1

    def __init__(self, ctx):
        self.ctx = ctx
        self.api = ctx.api
        h = C.c_void_p()
        self.api.check(self.api.icp_create(ctx.h, C.byref(h)), "icp_create")
        self.h = h

    def close(self):
        if self.h:
            self.api.icp_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _cloud(points):
        pts = np.ascontiguousarray(points, dtype=np.float32)
        assert pts.ndim == 2 and pts.shape[1] >= 3
        return pts, pts.shape[0], pts.shape[1] * 4

    def set_map(self, points, cell_size):
        """KdTreeFLANN::setInputCloud analogue (association.cpp:278-279)."""
        pts, n, stride = self._cloud(points)
        self._map_keepalive = pts
        self.api.check(self.api.icp_set_map(self.h, pts.ctypes.data_as(C.c_void_p), n, stride, float(cell_size)), "icp_set_map")

    # ---- device-resident map (CUDA library only): Mapping::ToWorld / BuildMapFrame without the per-keyframe map upload
    def map_append(self, key, points, pose):
        """Mapping::ToWorld of one keyframe (mapping.cpp:205-220): its robot-frame feature cloud goes to the device once, is
        transformed to the world frame there and kept under `key`.  points=None: the scan of the last scan_to_map call."""
        p = _f64(pose).reshape(7)
        if points is None:
            self.api.check(self.api.icp_map_append(self.h, int(key), None, 0, 0, _dp(p)), "icp_map_append")
            return
        pts, n, stride = self._cloud(points)
        self.api.check(self.api.icp_map_append(self.h, int(key), pts.ctypes.data_as(C.c_void_p), n, stride, _dp(p)), "icp_map_append")

    def map_evict(self, key=-1):
        self.api.check(self.api.icp_map_evict(self.h, int(key)), "icp_map_evict")

    def map_build(self, keys, cell_size, ground_threshold=-1.0):
        """Mapping::BuildMapFrame (mapping.cpp:114-137): merge the resident clouds of `keys` in order (+ SegmentGround when
        ground_threshold > 0) and hash the result, all on the device.  Returns the number of map points."""
        k = (C.c_longlong * len(keys))(*[int(x) for x in keys])
        n = C.c_int()
        self.api.check(self.api.icp_map_build(self.h, k, len(keys), float(cell_size), float(ground_threshold), C.byref(n)), "icp_map_build")
        return n.value

    def map_download(self):
        n = C.c_int()
        self.api.check(self.api.icp_map_download(self.h, None, 0, C.byref(n)), "icp_map_download")
        out = np.zeros((n.value, 4), dtype=np.float32)
        self.api.check(self.api.icp_map_download(self.h, out.ctypes.data_as(_capi.c_float_p), n.value, C.byref(n)), "icp_map_download")
        return out

    def transform_cloud(self, points, pose):
        """Mapping::MergeScan (mapping.cpp:193-203): float32 SE3 transform of a cloud, other fields carried over."""
        pts, n, stride = self._cloud(points)
        out = np.empty_like(pts)
        p = _f64(pose).reshape(7)
        self.api.check(self.api.icp_transform_cloud(self.h, pts.ctypes.data_as(C.c_void_p), n, stride, _dp(p), out.ctypes.data_as(C.c_void_p)), "icp_transform_cloud")
        return out

    def knn3(self, scan, frame_pose, max_d2):
        pts, n, stride = self._cloud(scan)
        pose = _f64(frame_pose).reshape(7)
        idx = np.zeros((n, 3), dtype=np.int32)
        d2 = np.zeros((n, 3), dtype=np.float32)
        self.api.check(self.api.icp_knn3(self.h, pts.ctypes.data_as(C.c_void_p), n, stride, _dp(pose), float(max_d2),
                                         _ip(idx), d2.ctypes.data_as(_capi.c_float_p)), "icp_knn3")
        return idx, d2

    def evaluate(self, mode, scan, frame_pose, map_pose, rpyxyz, weight, dist_thr):
        pts, n, stride = self._cloud(scan)
        fp, mp, e = _f64(frame_pose).reshape(7), _f64(map_pose).reshape(7), _f64(rpyxyz).reshape(6)
        acc = np.zeros(n, dtype=np.uint8)
        r = np.zeros(n)
        J = np.zeros((n, 3))
        self.api.check(self.api.icp_eval(self.h, mode, pts.ctypes.data_as(C.c_void_p), n, stride, _dp(fp), _dp(mp), _dp(e),
                                         float(weight), float(dist_thr), _bp(acc), _dp(r), _dp(J)), "icp_eval")
        return acc, r, J

    def scan_to_map(self, mode, scan, frame_pose, map_pose, rpyxyz, weight, prior_weight, huber_a, dist_thr, options=None, **kw):
        """ScanToMapWithGround / ScanToMapWithSegmented + adapt::Solve; returns (rpyxyz, summary)."""
        pts, n, stride = self._cloud(scan)
        fp, mp = _f64(frame_pose).reshape(7), _f64(map_pose).reshape(7)
        e = _f64(rpyxyz).reshape(6).copy()
        o = options or default_options(self.api, max_num_iterations=4, linear_solver_type=DENSE_QR, **kw)
        s = SolveSummary()
        self.api.check(self.api.icp_scan_to_map(self.h, mode, pts.ctypes.data_as(C.c_void_p), n, stride, _dp(fp), _dp(mp), _dp(e),
                                                float(weight), float(prior_weight), float(huber_a), float(dist_thr),
                                                C.byref(o), C.byref(s)), "icp_scan_to_map")
        return e, s


def _fp(a):
    return None if a is None else a.ctypes.data_as(_capi.c_float_p)


class LidarFeatures:
    """Lidar feature pipeline (FeatureAssociation::Process + ImageProjection::Process, association.cpp:88-268,
    projection.cpp:26-320): raw scan -> ground / surf feature clouds.  Clouds are float32 [n, 4] (x, y, z, intensity)."""

    def __init__(self, ctx, **overrides):
        self.ctx = ctx
        self.cfg = _capi.LidarConfig()
        ctx.api.lidar_default_config(C.byref(self.cfg))
        for k, v in overrides.items():
            if k == "extrinsic":
                for i in range(7):
                    self.cfg.extrinsic[i] = float(v[i])
            else:
                setattr(self.cfg, k, v)

    @property
    def capacity(self):
        return int(self.cfg.num_scans) * int(self.cfg.horizon_scan)

    @staticmethod
    def _raw(points):
        pts = np.ascontiguousarray(points, dtype=np.float32)
        assert pts.ndim == 2 and pts.shape[1] >= 3
        return pts, pts.shape[0], pts.shape[1] * 4

    def segment(self, points):
        """Preprocess + range-image projection + ground removal + segmentation + relative time + smoothness."""
        pts, n, stride = self._raw(points)
        cap, R = self.capacity, int(self.cfg.num_scans)
        seg = np.empty((cap, 4), np.float32); rng = np.empty(cap, np.float32); gnd = np.empty(cap, np.uint8)
        col = np.empty(cap, np.int32); curv = np.empty(cap, np.float32)
        sr = np.empty(R, np.int32); er = np.empty(R, np.int32); ori = np.empty(3, np.float32); m = np.zeros(1, np.int32)
        a = self.ctx.api
        a.check(a.lidar_segment(self.ctx.h, C.byref(self.cfg), pts.ctypes.data_as(C.c_void_p), n, stride, _fp(seg), _fp(rng), _bp(gnd), _ip(col), _fp(curv),
                                _ip(sr), _ip(er), _fp(ori), _ip(m)), "lidar_segment")
        k = int(m[0])
        return {"points": seg[:k].copy(), "range": rng[:k].copy(), "ground": gnd[:k].copy(), "col": col[:k].copy(), "curvature": curv[:k].copy(),
                "start_ring": sr, "end_ring": er, "orientation": ori}

    def _filter(self, fn, name, cloud, *args):
        cloud = np.ascontiguousarray(cloud, dtype=np.float32).reshape(-1, 4)
        out = np.empty_like(cloud) if len(cloud) else np.empty((1, 4), np.float32)
        m = np.zeros(1, np.int32)
        self.ctx.api.check(fn(self.ctx.h, _fp(cloud), len(cloud), *args, _fp(out), _ip(m)), name)
        return out[:int(m[0])].copy()

    def voxel_grid(self, cloud, leaf):
        return self._filter(self.ctx.api.lidar_voxel_grid, "lidar_voxel_grid", cloud, C.c_float(leaf))

    def radius_outlier_removal(self, cloud, radius, min_neighbors):
        return self._filter(self.ctx.api.lidar_radius_outlier_removal, "lidar_radius_outlier_removal", cloud, C.c_double(radius), int(min_neighbors))

    def segment_ground(self, cloud, threshold):
        return self._filter(self.ctx.api.lidar_segment_ground, "lidar_segment_ground", cloud, C.c_double(threshold))

    def extract(self, points):
        """FeatureAssociation::Process: returns (points_ground, points_surf) in the robot frame."""
        pts, n, stride = self._raw(points)
        cap = self.capacity
        g = np.empty((cap, 4), np.float32); s = np.empty((cap, 4), np.float32); ng = np.zeros(1, np.int32); ns = np.zeros(1, np.int32)
        a = self.ctx.api
        a.check(a.lidar_extract_features(self.ctx.h, C.byref(self.cfg), pts.ctypes.data_as(C.c_void_p), n, stride, _fp(g), _ip(ng), _fp(s), _ip(ns)), "lidar_extract_features")
        return g[:int(ng[0])].copy(), s[:int(ns[0])].copy()
