"""FeatureAssociation::Process into the resident map (lvb_icp_map_extract_keyframe, association.cpp:85-109): the feature clouds of a
lidar keyframe extracted with one host synchronisation and kept on the device as the pending features of its key, then registered
and stored by key by the keyframe calls (Mapping::Optimize, mapping.cpp:139-220) without leaving the device.

Extraction is float32 / integer work and is compared bit for bit with lvb_lidar_extract_features and the CPU oracle.  A chain fed by
key is compared with the same chain fed with the host copies of the same clouds: stored clouds, map frames and 3-NN bit for bit, the
launch and synchronisation counts exactly, and the poses to 1e-11 (the linearisation adds its block sums atomically, as in the other
keyframe tests)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from lvio_fusion_b200 import backend, synth
from test_gpu_map_optimize import _same_result, make_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GT = 0.05
# (LidarFeatures overrides, make_lidar_scan arguments): kitti (64 rings), kaist (16 rings, max_range 50), bupt (32 rings, resolution 0.5)
SENSORS = {
    "kitti": ({}, {}),
    "kaist": (dict(num_scans=16, ang_res_y=2.0, ang_bottom=15.1, ground_rows=7, max_range=50.0),
              dict(num_scans=16, ang_res_y=2.0, ang_bottom=15.1)),
    "bupt": (dict(num_scans=32, ang_res_y=1.33, ang_bottom=30.67, ground_rows=20, resolution=0.5),
             dict(num_scans=32, ang_res_y=1.33, ang_bottom=30.67)),
}


@pytest.fixture(scope="module")
def scene():
    return make_scene(200, 200)


def _pair(ctx):
    return backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)


def _code(fn):
    """the library's error code of fn (0: success); ValueError: rejected by the Python argument checks"""
    try:
        fn()
    except RuntimeError as e:
        return int(str(e).split("failed (")[1].split(")")[0])
    except ValueError:
        return "ValueError"
    return 0


@pytest.mark.parametrize("sensor", sorted(SENSORS))
def test_extraction_parity(lvb_ctx, orc_ctx, sensor):
    cfg, scan_kw = SENSORS[sensor]
    g, o = backend.LidarFeatures(lvb_ctx, **cfg), backend.LidarFeatures(orc_ctx, **cfg)
    ga, sa = _pair(lvb_ctx)
    scan = synth.make_lidar_scan(seed=41, **scan_kw)
    wide = np.zeros((len(scan), 8), np.float32); wide[:, :4] = scan; wide[:, 5] = 3.0          # 32-byte pcl::PointXYZI records
    want = o.extract(scan)
    assert len(want[0]) > 50 and len(want[1]) > 50
    for cloud in (scan, wide):
        for got in (g.extract(cloud), g.extract_into(ga, sa, 7, cloud)):
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert g.extract_into(ga, sa, 7, scan, copies=False) == (len(want[0]), len(want[1]))


def test_extraction_edge_cases(lvb_ctx, orc_ctx):
    g, o = backend.LidarFeatures(lvb_ctx), backend.LidarFeatures(orc_ctx)
    ga, sa = _pair(lvb_ctx)
    rng = np.random.default_rng(5)
    empty = np.zeros((0, 4), np.float32)
    nan = np.full((100, 4), np.nan, np.float32)
    near = np.tile(np.array([[1.0, 0.5, 0.1, 0.0]], np.float32), (50, 1))         # inside min_range
    sparse = rng.normal(0, 8, (300, 4)).astype(np.float32)                          # a handful of features: RANSAC on < 3 points
    for cloud in (empty, nan, near, sparse):
        want = o.extract(cloud)
        for got in (g.extract(cloud), g.extract_into(ga, sa, 1, cloud)):
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    for cloud in (empty, nan, near):
        assert g.extract_into(ga, sa, 1, cloud, copies=False) == (0, 0)


def test_one_synchronisation(lvb_ctx):
    g = backend.LidarFeatures(lvb_ctx)
    ga, sa = _pair(lvb_ctx)
    scan = synth.make_lidar_scan(seed=42)
    other = scan + np.float32(0.01) * np.random.default_rng(1).standard_normal(scan.shape).astype(np.float32)
    g.extract(scan)                       # the staging area is free from here on
    counts = []
    for fn in (lambda c: g.extract(c), lambda c: g.extract_into(ga, sa, 3, c), lambda c: g.extract_into(ga, sa, 3, c, copies=False)):
        for cloud in (scan, other):
            s0, l0 = lvb_ctx.sync_count(), lvb_ctx.launch_count()
            fn(cloud)
            counts.append((lvb_ctx.sync_count() - s0, lvb_ctx.launch_count() - l0))
    assert all(s == 1 for s, _ in counts), counts
    assert counts[0][1] == counts[1][1] and counts[2][1] == counts[3][1] == counts[4][1] == counts[5][1], counts


def _capacity(fa, key):
    """(resident world cloud, robot-frame cloud, pending features) buffer capacities of `key` on a handle, in records; -1: none"""
    cap = (C.c_longlong * 3)()
    fa.api.check(fa.api.debug_icp_cloud_capacity(fa.h, int(key), cap), "debug_icp_cloud_capacity")
    return tuple(int(x) for x in cap)


def _same_robot_clouds(a, b, key, sc, pose):
    """the robot-frame clouds two handle pairs keep for `key` are equal: both re-anchored at one pose and compared"""
    for h in (a, b):
        backend.map_to_world(h[0], h[1], [key], [pose])
    for fa, fb, cell in ((a[0], b[0], sc["g"]["cell_size"]), (a[1], b[1], sc["s"]["cell_size"])):
        fa.map_build([key], cell); fb.map_build([key], cell)
        assert np.array_equal(fa.map_download(), fb.map_download()), key


def test_overflow_stores_nothing(lvb_ctx, scene):
    lf = backend.LidarFeatures(lvb_ctx)
    g = backend.LidarFeatures(lvb_ctx, resolution=1e-4)           # leaf 2e-4 m: the feature voxel grids need far more than 2^26 voxels
    ga, sa = _pair(lvb_ctx)
    pose = np.array([0, 0, 0, 1, 0, 0, 0.0])
    first = lf.extract_into(ga, sa, 9, synth.make_lidar_scan(seed=44))
    scan = synth.make_lidar_scan(seed=43)
    assert _code(lambda: g.extract(scan)) == -5
    assert _code(lambda: g.extract_into(ga, sa, 9, scan)) == -5
    assert _code(lambda: g.extract_into(ga, sa, 10, scan)) == -5
    # key 9 still holds the first extraction's features, key 10 nothing
    assert _capacity(ga, 9)[2] == len(first[0]) and _capacity(sa, 9)[2] == len(first[1])
    assert _capacity(ga, 10) == (-1, -1, -1)
    assert _code(lambda: _chain(ga, sa, scene, [(10, [], pose, None, None)])) == -1
    _chain(ga, sa, scene, [(9, [], pose, None, None)])
    ref = _pair(lvb_ctx)
    _chain(ref[0], ref[1], scene, [(9, [], pose, first[0], first[1])])
    _same_robot_clouds((ga, sa), ref, 9, scene, pose)


def test_stored_clouds_keep_exactly_their_points(lvb_ctx, scene):
    """a pending cloud, and the robot-frame cloud it becomes, hold exactly the keyframe's points, as a host cloud stored by key does"""
    lf = backend.LidarFeatures(lvb_ctx)
    a, b = _pair(lvb_ctx), _pair(lvb_ctx)
    pose = np.array([0, 0, 0, 1, 0, 0, 0.0])
    ng, ns = lf.extract_into(a[0], a[1], 5, synth.make_lidar_scan(seed=45), copies=False)
    host = lf.extract(synth.make_lidar_scan(seed=45))
    assert (ng, ns) == (len(host[0]), len(host[1])) and ng < lf.capacity // 4
    assert _capacity(a[0], 5) == (-1, -1, ng) and _capacity(a[1], 5) == (-1, -1, ns)
    _chain(a[0], a[1], scene, [(5, [], pose, None, None)])
    _chain(b[0], b[1], scene, [(5, [], pose, host[0], host[1])])
    assert _capacity(a[0], 5) == _capacity(b[0], 5) == (ng, ng, -1)
    assert _capacity(a[1], 5) == _capacity(b[1], 5) == (ns, ns, -1)


def _poses(n):
    return [np.array([0, 0, np.sin(0.01 * k), np.cos(0.01 * k), 0.4 * k, 0.05 * k, 0.0]) for k in range(n)]


def _chain(ga, sa, sc, kfs, **kw):
    """kfs: (key, map_keys, pose, ground, surf); the map pose is that of the newest map key (in the call)."""
    g, s = sc["g"], sc["s"]
    full = [(key, mk, pose, pose, cg, cs) for key, mk, pose, cg, cs in kfs]
    return backend.build_and_optimize_keyframes(ga, sa, full, (g["cell_size"], s["cell_size"]), GT, (g["weight"], s["weight"]), sc["pw"],
                                                (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]), **kw)


def _single(ga, sa, sc, keys, key, map_pose, pose, cg, cs):
    g, s = sc["g"], sc["s"]
    return backend.build_and_optimize_keyframe(ga, sa, keys, (g["cell_size"], s["cell_size"]), GT, key, map_pose, pose, cg, cs,
                                               (g["weight"], s["weight"]), sc["pw"], (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]))


def _counted(ctx, fn):
    s0, l0 = ctx.sync_count(), ctx.launch_count()
    out = fn()
    return out, (ctx.sync_count() - s0, ctx.launch_count() - l0)


def _same_stored(a, b, keys, sc, poses):
    """the stored world clouds, a map_to_world round trip and the 3-NN against each handle's map frame agree bit for bit"""
    for fa, fb, cell in ((a[0], b[0], sc["g"]["cell_size"]), (a[1], b[1], sc["s"]["cell_size"])):
        for key in keys:
            fa.map_build([key], cell); fb.map_build([key], cell)
            assert np.array_equal(fa.map_download(), fb.map_download()), key
        fa.map_build(keys[-3:], cell); fb.map_build(keys[-3:], cell)
        q = fa.map_download()
        ia, da = fa.knn3(q, poses[0], cell * cell)
        ib, db = fb.knn3(q, poses[0], cell * cell)
        assert np.array_equal(ia, ib) and np.array_equal(da, db)
    moved = [p.copy() for p in poses]
    for p in moved:
        p[4] += 1.5
    for h in (a, b):
        backend.map_to_world(h[0], h[1], keys, moved)
    for fa, fb, cell in ((a[0], b[0], sc["g"]["cell_size"]), (a[1], b[1], sc["s"]["cell_size"])):
        for key in keys:
            fa.map_build([key], cell); fb.map_build([key], cell)
            assert np.array_equal(fa.map_download(), fb.map_download()), key


def test_chain_by_key_matches_host_clouds(lvb_ctx, scene):
    lf = backend.LidarFeatures(lvb_ctx)
    a, b = _pair(lvb_ctx), _pair(lvb_ctx)
    poses = _poses(5)
    keys = list(range(100, 105))
    host = [lf.extract_into(a[0], a[1], key, synth.make_lidar_scan(seed=50 + i)) for i, key in enumerate(keys)]
    kf_key = [(key, keys[max(0, i - 3):i], poses[i], None, None) for i, key in enumerate(keys)]
    kf_host = [(key, keys[max(0, i - 3):i], poses[i], host[i][0], host[i][1]) for i, key in enumerate(keys)]
    by_key, ck = _counted(lvb_ctx, lambda: _chain(a[0], a[1], scene, kf_key))
    by_host, ch = _counted(lvb_ctx, lambda: _chain(b[0], b[1], scene, kf_host))
    assert ck == ch, (ck, ch)
    for x, y in zip(by_key, by_host):
        _same_result((x[0], x[2], x[3]), (y[0], y[2], y[3]))
        assert np.max(np.abs(x[1] - y[1])) < 1e-11 and x[4] == y[4]
    assert all(r[4][0] > 0 and r[4][1] > 0 for r in by_key[1:])
    _same_stored(a, b, keys, scene, [r[0] for r in by_key])
    # the pending features went into the stored clouds: the keys are no longer pending
    assert _code(lambda: _chain(a[0], a[1], scene, [(200, keys[-3:], poses[0], None, None)])) == -1
    assert _code(lambda: _chain(a[0], a[1], scene, [(keys[0], keys[1:4], poses[0], None, None)])) == -1


def test_single_by_key_matches_host_clouds(lvb_ctx, scene):
    lf = backend.LidarFeatures(lvb_ctx)
    a, b = _pair(lvb_ctx), _pair(lvb_ctx)
    poses = _poses(3)
    clouds = [lf.extract_into(a[0], a[1], k, synth.make_lidar_scan(seed=60 + k)) for k in range(3)]
    out = []
    for h, by_key in ((a, True), (b, False)):
        res = []
        for k in range(3):
            cg, cs = (None, None) if by_key else clouds[k]
            mk = list(range(k))
            res.append(_counted(lvb_ctx, lambda: _single(h[0], h[1], scene, mk, k, poses[max(0, k - 1)], poses[k], cg, cs)))
        out.append(res)
    for (x, cx), (y, cy) in zip(*out):
        assert cx == cy
        _same_result((x[0], x[1], x[2]), (y[0], y[1], y[2]))
        assert x[3] == y[3]
    _same_stored(a, b, [0, 1, 2], scene, poses)


def test_state_rules(lvb_ctx, scene):
    lf = backend.LidarFeatures(lvb_ctx)
    ga, sa = _pair(lvb_ctx)
    pose = np.array([0, 0, 0, 1, 0, 0, 0.0])
    first = lf.extract_into(ga, sa, 1, synth.make_lidar_scan(seed=70))
    _chain(ga, sa, scene, [(1, [], pose, None, None)])              # key 1 resident
    lf.extract_into(ga, sa, 2, synth.make_lidar_scan(seed=71))
    # a pending-only key is not a map key, nor resident for map_build / map_to_world
    assert _code(lambda: _chain(ga, sa, scene, [(3, [2], pose, first[0], first[1])])) == -1
    assert _code(lambda: ga.map_build([2], scene["g"]["cell_size"])) == -1
    assert _code(lambda: backend.map_to_world(ga, sa, [2], [pose])) == -1
    # by key on one side only, or with nothing pending
    assert _code(lambda: _chain(ga, sa, scene, [(2, [1], pose, None, first[1])])) == "ValueError"
    assert _code(lambda: _chain(ga, sa, scene, [(4, [1], pose, None, None)])) == -1
    # a failed chain keeps the pending features: key 2's map key 5 is unknown (found on the host), and a map frame whose voxel grid
    # does not fit at any ring (found on the device, after the read-back)
    assert _code(lambda: _chain(ga, sa, scene, [(2, [5], pose, None, None)])) == -1
    held = (_capacity(ga, 2), _capacity(sa, 2))
    assert held[0][2] > 0 and held[1][2] > 0
    s0 = lvb_ctx.sync_count()
    assert _code(lambda: backend.build_and_optimize_keyframes(ga, sa, [(2, [1], pose, pose, None, None)], (1e-3, 1e-3), GT, (1.0, 1.0), 1.0,
                                                              (0.0, 0.1), (1e-7, 1e-7))) == -5
    assert lvb_ctx.sync_count() > s0 and (_capacity(ga, 2), _capacity(sa, 2)) == held
    # evict drops them, re-extraction replaces them
    ga.map_evict(2)
    assert _code(lambda: _chain(ga, sa, scene, [(2, [1], pose, None, None)])) == -1
    sa.map_evict(2)
    second = lf.extract_into(ga, sa, 2, synth.make_lidar_scan(seed=72))
    third = lf.extract_into(ga, sa, 2, synth.make_lidar_scan(seed=73))
    assert len(second[0]) != len(third[0]) or not np.array_equal(second[0], third[0])
    _chain(ga, sa, scene, [(2, [1], pose, None, None)])
    ref = _pair(lvb_ctx)
    _chain(ref[0], ref[1], scene, [(2, [], pose, third[0], third[1])])
    _same_robot_clouds((ga, sa), ref, 2, scene, pose)          # the third extraction's clouds were stored
    # used once: the second by-key registration of the same key finds nothing pending
    assert _code(lambda: _chain(ga, sa, scene, [(2, [1], pose, None, None)])) == -1
    # evict(-1) drops every pending entry
    lf.extract_into(ga, sa, 8, synth.make_lidar_scan(seed=74))
    ga.map_evict(-1); sa.map_evict(-1)
    assert _code(lambda: _chain(ga, sa, scene, [(8, [], pose, None, None)])) == -1


def test_shim_extract_keyframe_matches_host_clouds(lvb_ctx, tmp_path):
    """include/lvio_b200/association.h: ExtractKeyframe + OptimizeKeyframes / OptimizeKeyframe by key against LidarFeatureExtractor::Process
    + the same calls from frame->feature_lidar, on the same raw scans: the same features and the same poses."""
    K = 5
    poses = _poses(K)
    with open(tmp_path / "in.bin", "wb") as f:
        np.array([K], np.int32).tofile(f)
        np.array([synth.W_VISUAL], np.float64).tofile(f)
        np.array([120], np.int32).tofile(f)
        for k in range(K):
            scan = np.ascontiguousarray(synth.make_lidar_scan(seed=80 + k)[:, :4], np.float32)
            np.asarray(poses[k], np.float64).tofile(f)
            np.array([len(scan)], np.int32).tofile(f)
            scan.tofile(f)
    lib_dir = os.path.join(ROOT, "lvio_fusion_b200", "csrc")
    exe = str(tmp_path / "shim")
    subprocess.check_call(["g++", "-O2", "-std=c++14", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "map_extract_keyframe_shim.cpp"), "-L" + lib_dir, "-llvio_b200",
                           "-Wl,-rpath," + lib_dir])
    p = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr + p.stdout
    assert "SAME FEATURES" in p.stdout, p.stdout
    out = np.fromfile(tmp_path / "out.bin").reshape(4, K, 7)
    assert np.max(np.abs(out[0] - out[1])) < 1e-11          # OptimizeKeyframes: host clouds / by key
    assert np.max(np.abs(out[2] - out[3])) < 1e-11          # per-keyframe OptimizeKeyframe: host clouds / by key
    assert np.max(np.abs(out[0, 1:] - np.array(poses[1:]))) > 0        # the registrations moved the poses
