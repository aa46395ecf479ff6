"""Mapping::BuildMapFrame + Mapping::Optimize for one keyframe in one device call (lvb_icp_map_build_optimize_keyframe,
mapping.cpp:114-137, 147-185): the merge of the map frame's resident clouds, SegmentGround on the ground side, both voxel hashes, both
scan-to-map solves, the pose hand-off and ToWorld, with one host synchronisation.  Checked against the step-by-step path of the shim
(lvb_icp_map_build on each side -- a side whose build fails is not registered -- then lvb_icp_map_optimize_keyframe, and ToWorld of an
unregistered side with map_evict + map_append) and against the CPU oracle."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from lvio_fusion_b200 import _capi, backend, synth
from test_gpu_map_optimize import _same_result, _to_robot, _sliding_inputs, _stored, make_scene, one_call

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GT = 0.05           # SegmentGround distance threshold of the ground map frame


@pytest.fixture(scope="module")
def scene():
    return make_scene(6000, 5000)


def _frames(sc, n_extra):
    """The scene's three keyframes, then n_extra registrations of its scans: (pose guess, robot-frame ground, robot-frame surf)."""
    g, s = sc["g"], sc["s"]
    return list(sc["kfs"]) + [(guess, g["scan"], s["scan"]) for guess in _sliding_inputs(sc, n_extra)]


def _pair(ctx):
    return backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)


def new_call(gb, sb, sc, keys, key, map_pose, pose, cg, cs, thr=GT, **kw):
    g, s = sc["g"], sc["s"]
    return backend.build_and_optimize_keyframe(gb, sb, keys, (g["cell_size"], s["cell_size"]), thr, key, map_pose, pose, cg, cs,
                                               (g["weight"], s["weight"]), sc["pw"], (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]), **kw)


def shim_step(ga, sa, sc, keys, key, map_pose, pose, cg, cs, thr=GT, **kw):
    """association.h's BuildMapFrame + OptimizeKeyframe through the C ABI.  Returns (pose, rpyxyz, summaries, map points)."""
    g, s = sc["g"], sc["s"]
    built, nmap = [None, None], [0, 0]
    for m, (fa, cell, t) in enumerate(((ga, g["cell_size"], thr), (sa, s["cell_size"], -1.0))):
        if keys:
            try:
                nmap[m] = fa.map_build(keys, cell, t)
                built[m] = fa
            except RuntimeError:
                pass
    if built[0] or built[1]:
        p, e, sums = one_call(built[0], built[1], sc, key, map_pose, pose, cg if built[0] else None, cs if built[1] else None, **kw)
    else:
        p, e, sums = np.asarray(pose, np.float64).copy(), synth.relative_rpyxyz(map_pose, pose), (None, None)
    sums = tuple(x if built[m] else None for m, x in enumerate(sums))
    for m, (fa, c) in enumerate(((ga, cg), (sa, cs))):
        if built[m] is None:
            fa.map_evict(key)
            fa.map_append(key, c, p)
    return p, e, sums, nmap


def _check_skipped(call, nmap):
    for m in range(2):
        if nmap[m] == 0:
            x = call[2][m]
            assert x.termination_type == -1 and x.num_iterations == 0 and x.num_residual_blocks == 0


def _same_handles(fa, fb, scan, pose, cell):
    """map_download of the map frames and knn3 against them: bit for bit."""
    assert np.array_equal(fa.map_download().view(np.uint32), fb.map_download().view(np.uint32))
    ia, da = fa.knn3(scan, pose, 0.9 * cell * cell)
    ib, db = fb.knn3(scan, pose, 0.9 * cell * cell)
    assert np.array_equal(ia, ib) and np.array_equal(da.view(np.uint32), db.view(np.uint32))


def test_sliding_run_from_the_first_keyframe_equals_step_by_step(lvb_ctx, scene):
    """n_keys 0, 1, 2, 3, 3, 3: the first keyframe (no map frame), then growing and sliding windows."""
    sc = scene
    g, s = sc["g"], sc["s"]
    ga, sa = _pair(lvb_ctx)
    gb, sb = _pair(lvb_ctx)
    poses, syncs_step, syncs_call = {}, [], []
    for k, (guess, cg, cs) in enumerate(_frames(sc, 3)):
        keys = [j for j in range(k - 3, k) if j >= 0]
        map_pose = poses[keys[-1]] if keys else np.array([0, 0, 0, 1, 0, 0, 0.0])
        n0 = lvb_ctx.sync_count()
        step = shim_step(ga, sa, sc, keys, k, map_pose, guess, cg, cs)
        n1 = lvb_ctx.sync_count()
        call = new_call(gb, sb, sc, keys, k, map_pose, guess, cg, cs)
        syncs_step.append(n1 - n0)
        syncs_call.append(lvb_ctx.sync_count() - n1)
        _same_result(step[:3], call[:3])
        assert list(call[3]) == step[3], k
        _check_skipped(call, step[3])
        if keys:
            assert min(call[3]) > 0 and call[3][0] < sum(len(_frames(sc, 3)[j][1]) for j in keys)     # SegmentGround dropped points
            assert all(x.num_iterations > 0 for x in call[2])
            _same_handles(ga, gb, cg, call[0], g["cell_size"])
            _same_handles(sa, sb, cs, call[0], s["cell_size"])
        else:
            assert np.array_equal(call[0], np.asarray(guess, np.float64)) and list(call[3]) == [0, 0]
        for fa, fb, cell in ((ga, gb, g["cell_size"]), (sa, sb, s["cell_size"])):       # ToWorld, bit for bit
            assert np.array_equal(_stored(fa, k, cell).view(np.uint32), _stored(fb, k, cell).view(np.uint32))
        poses[k] = call[0]
        if k >= 3:
            for fa in (ga, sa, gb, sb):
                fa.map_evict(k - 3)
    print("host synchronisations per keyframe: one call %s, step by step %s" % (syncs_call, syncs_step))
    assert syncs_call == [1] * len(syncs_call)
    assert min(syncs_step[1:]) > 1


def test_sliding_run_against_the_oracle(lvb_ctx, orc_ctx, scene):
    """The same run through the oracle: CPU merge of the world clouds, SegmentGround, orc_icp_scan_to_map, poses composed on the host."""
    sc = scene
    g, s = sc["g"], sc["s"]
    gb, sb = _pair(lvb_ctx)
    og, os_ = _pair(orc_ctx)
    lidar = backend.LidarFeatures(orc_ctx)
    world, poses = {}, {}
    for k, (guess, cg, cs) in enumerate(_frames(sc, 3)):
        keys = [j for j in range(k - 3, k) if j >= 0]
        map_pose = poses[keys[-1]] if keys else np.array([0, 0, 0, 1, 0, 0, 0.0])
        p = np.asarray(guess, np.float64)
        if keys:
            og.set_map(lidar.segment_ground(np.concatenate([world[j][0] for j in keys]), GT), g["cell_size"])
            os_.set_map(np.concatenate([world[j][1] for j in keys]), s["cell_size"])
            e = synth.relative_rpyxyz(map_pose, p)
            e, _ = og.scan_to_map(0, cg, p, map_pose, e, g["weight"], sc["pw"], g["huber_a"], g["thr"])
            p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
            e, _ = os_.scan_to_map(1, cs, p, map_pose, e, s["weight"], sc["pw"], s["huber_a"], s["thr"])
            p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
        world[k] = (og.transform_cloud(cg, p), os_.transform_cloud(cs, p))
        pc, ec, _, _ = new_call(gb, sb, sc, keys, k, map_pose, guess, cg, cs)
        assert np.max(np.abs(pc - p)) < 1e-7, k
        if keys:
            assert np.max(np.abs(ec - e)) < 1e-7, k
        poses[k] = pc


def _three_keyframes(ctx, sc, ground=None, surf=None):
    """Two handle pairs holding the scene's keyframes 0..2, the robot-frame clouds replaced by `ground` / `surf` when given."""
    pairs = [_pair(ctx), _pair(ctx)]
    for k, (pose, cg, cs) in enumerate(sc["kfs"]):
        for fa, fs in pairs:
            fa.map_append(k, cg if ground is None else ground, pose)
            fs.map_append(k, cs if surf is None else surf, pose)
    return pairs


@pytest.mark.parametrize("side", ["ground", "surf"])
def test_skipped_side_equals_the_shim_skip_path(lvb_ctx, scene, side):
    """ground: SegmentGround keeps no point (a merged cloud of fewer than 3 points); surf: an empty merged cloud.  That side is not
    registered, the other one is, and both clouds are stored."""
    sc = scene
    g, s = sc["g"], sc["s"]
    one = sc["kfs"][0][1][:1]
    (ga, sa), (gb, sb) = _three_keyframes(lvb_ctx, sc, ground=one if side == "ground" else None,
                                          surf=np.zeros((0, 4), np.float32) if side == "surf" else None)
    keys, key, map_pose = [0, 1], 3, sc["kfs"][1][0]
    step = shim_step(ga, sa, sc, keys, key, map_pose, g["frame_pose"], g["scan"], s["scan"])
    call = new_call(gb, sb, sc, keys, key, map_pose, g["frame_pose"], g["scan"], s["scan"])
    _same_result(step[:3], call[:3])
    m = 0 if side == "ground" else 1
    assert call[3][m] == 0 and step[3][m] == 0 and call[3][1 - m] > 0
    _check_skipped(call, call[3])
    assert call[2][1 - m].num_iterations > 0
    if side == "ground":      # the surf registration starts from the incoming pose, as the shim's path does without a ground map
        e0 = synth.relative_rpyxyz(map_pose, g["frame_pose"])
        assert np.max(np.abs(call[1][[1, 2, 5]] - e0[[1, 2, 5]])) < 1e-12
    for fa, fb, cell in ((ga, gb, g["cell_size"]), (sa, sb, s["cell_size"])):
        assert np.array_equal(_stored(fa, key, cell).view(np.uint32), _stored(fb, key, cell).view(np.uint32))


def test_syncs_of_keys_stored_by_other_entry_points(lvb_ctx, scene):
    """A resident cloud stored by map_append has no recorded bounding box: the first call that merges it computes it (one more
    synchronisation), later calls do not."""
    sc = scene
    g, s = sc["g"], sc["s"]
    (gb, sb), _ = _three_keyframes(lvb_ctx, sc)
    deltas = []
    for _ in range(3):
        n0 = lvb_ctx.sync_count()
        new_call(gb, sb, sc, [0, 1, 2], 3, sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"])
        deltas.append(lvb_ctx.sync_count() - n0)
    assert deltas == [2, 1, 1]


def _expected_launches(iters, n_scan, ransac):
    n = 1
    for m in range(2):
        n += (8 if m == 0 and ransac else 0) + 9                                 # SegmentGround (RANSAC 4, scan 3, gather), bbox .. scatter
        n += (6 if n_scan[m] >= 4096 else 0) + (1 if n_scan[m] > 0 else 0) + 4 * (iters + 1) + 1
        n += 1 if n_scan[m] > 0 else 0                                           # ToWorld
    return n


@pytest.mark.parametrize("iters", [1, 4])
def test_launch_count_is_fixed(lvb_ctx, iters):
    """The launch sequence depends on the scan sizes, the merged sizes and max_num_iterations only: not on how many points
    SegmentGround keeps, nor on when the solvers stop."""
    sc = make_scene(6000, 3000, n_map=30000, seed=5)
    g, s = sc["g"], sc["s"]
    (gb, sb), _ = _three_keyframes(lvb_ctx, sc)
    args = ([0, 1, 2], 3, sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"])
    new_call(gb, sb, sc, *args)                        # records the boxes of the map_append clouds
    counts, kept, stops = [], [], []
    for thr, gtol in ((0.02, 1e-10), (0.3, 1e-10), (0.02, 1e30)):
        opt = backend.default_options(lvb_ctx.api, max_num_iterations=iters, linear_solver_type=backend.DENSE_QR, gradient_tolerance=gtol)
        n0 = lvb_ctx.launch_count()
        _, _, sums, nm = new_call(gb, sb, sc, *args, thr=thr, options=opt)
        counts.append(lvb_ctx.launch_count() - n0)
        kept.append(nm[0])
        stops.append([x.num_iterations for x in sums])
    assert counts[0] == counts[1] == counts[2] == _expected_launches(iters, (len(g["scan"]), len(s["scan"])), True)
    assert kept[0] != kept[1]
    assert min(stops[0]) > 0 and stops[2] == [0, 0]


def test_errors_change_no_state(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    (gb, sb), _ = _three_keyframes(lvb_ctx, sc)
    args = (sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"])
    new_call(gb, sb, sc, [0, 1, 2], 3, *args)
    # key 7: a surf cloud with an infinite point; key 8: a ground plane too wide for the voxel grid at any ring (found on the device,
    # after SegmentGround).  Both stored by the call itself, so their boxes are known.
    bad = s["scan"].copy()
    bad[5, 0] = np.inf
    rng = np.random.default_rng(3)
    wide = np.zeros((4000, 4), np.float32)           # the world's ground plane z = 0, 100 km across, in the robot frame
    wide[:, :2] = rng.uniform(-5e4, 5e4, (4000, 2))
    wide = _to_robot(wide, args[1])
    new_call(gb, sb, sc, [], 7, *args[:3], bad)
    new_call(gb, sb, sc, [], 8, args[0], args[1], wide, s["scan"])
    snap = [fa.map_download() for fa in (gb, sb)]
    stored = [_stored(fa, 3, cell) for fa, cell in ((gb, g["cell_size"]), (sb, s["cell_size"]))]
    new_call(gb, sb, sc, [0, 1, 2], 3, *args)           # the map frames of the snapshot again
    n0 = lvb_ctx.launch_count()
    capped = backend.default_options(lvb_ctx.api, max_num_iterations=4, linear_solver_type=backend.DENSE_QR, max_solver_time_in_seconds=1.0)
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        new_call(gb, sb, sc, [0, 1, 2], 9, *args, options=capped)
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        new_call(gb, sb, sc, [0, 1, 2], 1, *args)                       # key among keys
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        new_call(gb, sb, sc, [0, 42], 9, *args)                         # not resident
    with pytest.raises(RuntimeError, match=r"failed \(-1\).*finite"):
        new_call(gb, sb, sc, [0, 7], 9, *args)
    api = lvb_ctx.api
    prm = _capi.MapOptimizeParams()
    api.default_options(C.byref(prm.options))
    k = (C.c_longlong * 1)(0)
    cs = np.array([g["cell_size"], s["cell_size"]], np.float32)
    pose, e, nm = np.array(args[1], np.float64), np.zeros(6), np.zeros(2, np.int32)
    assert api.icp_map_build_optimize_keyframe(None, sb.h, k, 1, cs.ctypes.data_as(_capi.c_float_p), GT, backend._dp(np.array(args[0])), 9,
                                               None, 0, None, 0, 16, C.byref(prm), backend._dp(pose), backend._dp(e), None,
                                               nm.ctypes.data_as(_capi.c_int_p)) == -1
    assert lvb_ctx.launch_count() == n0
    with pytest.raises(RuntimeError, match=r"failed \(-5\)"):
        new_call(gb, sb, sc, [0, 8], 9, *args)                          # found on the device
    for fa, before in zip((gb, sb), snap):
        assert np.array_equal(fa.map_download().view(np.uint32), before.view(np.uint32))
        with pytest.raises(RuntimeError):
            fa.map_build([9], 1.0)                                      # nothing was stored
    for fa, cell, before in ((gb, g["cell_size"], stored[0]), (sb, s["cell_size"], stored[1])):
        assert np.array_equal(_stored(fa, 3, cell).view(np.uint32), before.view(np.uint32))
    _, _, sums, _ = new_call(gb, sb, sc, [0, 1, 2], 9, *args)         # and the next call runs
    assert sums[0].num_iterations > 0 and sums[1].num_iterations > 0


def test_shim_one_call_loop_equals_build_then_optimize_loop(lvb_ctx, scene, tmp_path):
    """include/lvio_b200/association.h: the OptimizeKeyframe(frame, keys, ...) loop from the first keyframe on against the
    BuildMapFrame + OptimizeKeyframe loop of tests/cpp/map_optimize_shim.cpp, on the same frames."""
    sc = scene
    frames = _frames(sc, 2)
    with open(tmp_path / "in.bin", "wb") as f:
        np.array([len(frames)], np.int32).tofile(f)
        np.array([synth.W_VISUAL], np.float64).tofile(f)
        np.array([sc["g"]["n_features_left"]], np.int32).tofile(f)
        for pose, cg, cs in frames:
            np.asarray(pose, np.float64).tofile(f)
            for c in (cg, cs):
                np.array([len(c)], np.int32).tofile(f)
                np.ascontiguousarray(c[:, :4], np.float32).tofile(f)
    lib_dir = os.path.join(ROOT, "lvio_fusion_b200", "csrc")
    outs = []
    for name in ("map_optimize_shim", "map_build_optimize_shim"):
        exe = str(tmp_path / name)
        subprocess.check_call(["g++", "-O2", "-std=c++14", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                               os.path.join(ROOT, "tests", "cpp", name + ".cpp"), "-L" + lib_dir, "-llvio_b200", "-Wl,-rpath," + lib_dir])
        p = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / (name + ".bin"))], capture_output=True, text=True)
        assert p.returncode == 0, p.stderr
        outs.append(np.fromfile(tmp_path / (name + ".bin")).reshape(len(frames), 9))
    step, call = outs
    assert np.max(np.abs(call[:, :7] - step[:, :7])) < 1e-11
    assert np.array_equal(call[:, 7:], step[:, 7:])
    assert list(call[0, 7:]) == [-1, -1] and (call[1:, 7:] >= 0).all()


def test_sharded_context_is_unsupported():
    """world_size > 1 reports LVB_ERR_UNSUPPORTED and stores nothing (2 ranks; skipped on a single-GPU box)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29521", os.path.join(ROOT, "tests", "map_build_keyframe_multigpu_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert "MAP BUILD KEYFRAME MULTIGPU OK" in p.stdout


def test_python_argument_checks(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    (gb, sb), _ = _three_keyframes(lvb_ctx, sc)
    args = (sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"])
    with pytest.raises(ValueError):
        new_call(gb, None, sc, [0, 1, 2], 3, *args)
    wide = np.zeros((len(s["scan"]), 8), np.float32)
    wide[:, :4] = s["scan"]
    with pytest.raises(ValueError):
        new_call(gb, sb, sc, [0, 1, 2], 3, *args[:3], wide)
    opt = backend.default_options(lvb_ctx.api, max_num_iterations=4, linear_solver_type=backend.DENSE_QR)
    _, _, sums, _ = new_call(gb, sb, sc, [0, 1, 2], 3, *args, options=opt, gradient_tolerance=1e30)
    assert [x.num_iterations for x in sums] == [0, 0] and opt.gradient_tolerance == 1e-10
