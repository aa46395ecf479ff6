"""Mapping::Relocate for one loop-closure candidate in one device call (lvb_icp_map_relocate, mapping.cpp:78-112, 251-300):
BuildOldMapFrame into each handle's relocation slot, then four rounds of both registrations without a prior, with one host
synchronisation.  Checked against the step-by-step path (map_build of the old map frame on a second pair of handles, then per round
scan_to_map ground, the pose composed on the host, scan_to_map surf, the scores computed on the host), against the CPU oracle, and
for leaving the mapping state alone."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from lvio_fusion_b200 import _capi, backend, synth
from test_gpu_map_build_keyframe import GT, _pair, _same_handles, _three_keyframes, new_call
from test_gpu_map_optimize import _perturbed, _same_result, _same_summary, _stored, _to_robot, make_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPS = (20.0, 30.0)


@pytest.fixture(scope="module")
def scene():
    return make_scene(6000, 5000)


# the old keyframe at the start (no predecessor), in the middle and at the end (no successor) of the resident run 0, 1, 2:
# BuildOldMapFrame's keys in time order, the old keyframe
PLACES = {"start": ([0, 1], 0), "middle": ([0, 1, 2], 1), "end": ([1, 2], 2)}


def _candidate(sc, old, seed=11):
    """old_pose and a relative guess that puts the clone near the scans' true pose."""
    old_pose = sc["kfs"][old][0]
    guess = _perturbed(sc["g"]["frame_pose"], np.random.default_rng(seed), 0.05, 0.002)
    return old_pose, synth.se3_mul(synth.se3_inv(old_pose), guess)


def reloc_call(gb, sb, sc, keys, old_pose, rel, cg=None, cs=None, thr=GT, **kw):
    g, s = sc["g"], sc["s"]
    return backend.relocate(gb, sb, keys, (g["cell_size"], s["cell_size"]), thr, sc["kfs"][keys[0]][0], old_pose, rel,
                            g["scan"] if cg is None else cg, s["scan"] if cs is None else cs, (g["weight"], s["weight"]),
                            (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]), **kw)


def _score(summary, cap):
    n = summary.num_residual_blocks_reduced
    with np.errstate(divide="ignore", invalid="ignore"):
        return min(np.float64(n) / 10, cap) - 2 * np.float64(summary.final_cost) / n if n else float("nan")


def step_by_step(ga, sa, sc, keys, old_pose, rel, cg=None, cs=None, thr=GT, rounds=4):
    """Mapping::Relocate through the per-registration entry points: map_build of the old map frame on each side (a side whose build
    fails is skipped), then per round se32rpyxyz, scan_to_map ground, rpyxyz2se3, scan_to_map surf, rpyxyz2se3 on the host."""
    g, s = sc["g"], sc["s"]
    cg = g["scan"] if cg is None else cg
    cs = s["scan"] if cs is None else cs
    map_pose = sc["kfs"][keys[0]][0]
    nmap = [0, 0]
    for m, (fa, cell, t) in enumerate(((ga, g["cell_size"], thr), (sa, s["cell_size"], -1.0))):
        try:
            nmap[m] = fa.map_build(keys, cell, t)
        except RuntimeError:
            pass
    pose = synth.se3_mul(old_pose, rel)
    sums = [None, None]
    for _ in range(rounds):
        e = synth.relative_rpyxyz(map_pose, pose)
        if nmap[0]:
            e, sums[0] = ga.scan_to_map(0, cg, pose, map_pose, e, g["weight"], -1.0, g["huber_a"], g["thr"])
            pose = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
        if nmap[1]:
            e, sums[1] = sa.scan_to_map(1, cs, pose, map_pose, e, s["weight"], -1.0, s["huber_a"], s["thr"])
            pose = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
    scores = [_score(x, c) if x is not None else float("nan") for x, c in zip(sums, CAPS)]
    return synth.se3_mul(synth.se3_inv(old_pose), pose), pose, sums, scores, nmap


def _same_as_step(step, call):
    rs, ps, ss, scs, nms = step
    rc, pc, sc_, scc, nmc = call
    assert np.max(np.abs(pc - ps)) < 1e-11 and np.max(np.abs(rc - rs)) < 1e-11
    assert list(nmc) == nms
    for m in range(2):
        if ss[m] is None:
            assert sc_[m].termination_type == -1 and sc_[m].num_iterations == 0 and sc_[m].num_residual_blocks == 0
            assert np.isnan(scc[m])
        else:
            _same_summary(sc_[m], ss[m])
            assert abs(scc[m] - scs[m]) < 1e-9


@pytest.mark.parametrize("place", sorted(PLACES))
def test_equals_step_by_step(lvb_ctx, scene, place):
    sc = scene
    g, s = sc["g"], sc["s"]
    keys, old = PLACES[place]
    (ga, sa), (gb, sb) = _three_keyframes(lvb_ctx, sc)
    old_pose, rel = _candidate(sc, old)
    step = step_by_step(ga, sa, sc, keys, old_pose, rel)
    # gb / sb hold a map frame of their own, which the relocation must leave as it is
    gb.map_build([2], g["cell_size"], GT)
    sb.map_build([2], s["cell_size"])
    before = [(fa.map_download(), fa.knn3(c, g["frame_pose"], 0.9 * cell * cell)) for fa, c, cell in
              ((gb, g["scan"], g["cell_size"]), (sb, s["scan"], s["cell_size"]))]
    n0 = lvb_ctx.sync_count()
    call = reloc_call(gb, sb, sc, keys, old_pose, rel)
    assert lvb_ctx.sync_count() - n0 == 2          # the first use of clouds stored by map_append computes their boxes
    _same_as_step(step, call)
    assert min(call[4]) > 0 and all(x.num_iterations > 0 for x in call[2]) and all(np.isfinite(call[3]))
    assert call[4][0] < sum(len(sc["kfs"][k][1]) for k in keys)          # SegmentGround dropped points
    for (fa, c, cell), (mp, (idx, d2)) in zip(((gb, g["scan"], g["cell_size"]), (sb, s["scan"], s["cell_size"])), before):
        assert np.array_equal(fa.map_download().view(np.uint32), mp.view(np.uint32))
        i2, e2 = fa.knn3(c, g["frame_pose"], 0.9 * cell * cell)
        assert np.array_equal(i2, idx) and np.array_equal(e2.view(np.uint32), d2.view(np.uint32))
    # a second relocation reuses the slot and the recorded boxes
    n0 = lvb_ctx.sync_count()
    again = reloc_call(gb, sb, sc, keys, old_pose, rel)
    assert lvb_ctx.sync_count() - n0 == 1
    _same_as_step(step, again)


def test_against_the_oracle(lvb_ctx, orc_ctx, scene):
    """The same sequence through the oracle: CPU merge of the world clouds, SegmentGround, orc_icp_scan_to_map without a prior."""
    sc = scene
    g, s = sc["g"], sc["s"]
    (gb, sb), _ = _three_keyframes(lvb_ctx, sc)
    og, os_ = _pair(orc_ctx)
    lidar = backend.LidarFeatures(orc_ctx)
    world = {k: (og.transform_cloud(cg, p), os_.transform_cloud(cs, p)) for k, (p, cg, cs) in enumerate(sc["kfs"])}
    for place in sorted(PLACES):
        keys, old = PLACES[place]
        old_pose, rel = _candidate(sc, old)
        map_pose = sc["kfs"][keys[0]][0]
        og.set_map(lidar.segment_ground(np.concatenate([world[j][0] for j in keys]), GT), g["cell_size"])
        os_.set_map(np.concatenate([world[j][1] for j in keys]), s["cell_size"])
        p = synth.se3_mul(old_pose, rel)
        for _ in range(4):
            e = synth.relative_rpyxyz(map_pose, p)
            e, _ = og.scan_to_map(0, g["scan"], p, map_pose, e, g["weight"], -1.0, g["huber_a"], g["thr"])
            p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
            e, _ = os_.scan_to_map(1, s["scan"], p, map_pose, e, s["weight"], -1.0, s["huber_a"], s["thr"])
            p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
        rc, pc, sums, scores, _ = reloc_call(gb, sb, sc, keys, old_pose, rel)
        assert np.max(np.abs(pc - p)) < 1e-7, place
        assert np.max(np.abs(rc - synth.se3_mul(synth.se3_inv(old_pose), p))) < 1e-7, place
        assert sums[0].num_residual_blocks_reduced > 1000 and sums[1].num_residual_blocks_reduced > 1000


def test_leaves_the_mapping_state_alone(lvb_ctx, scene):
    """A relocation between two keyframes of the mapping loop: the map frames, 3-NN, the stored clouds and map_append(NULL) are bit
    for bit those of a run without it, and so is the next keyframe's result (to the step-by-step tolerance of the keyframe tests)."""
    sc = scene
    g, s = sc["g"], sc["s"]
    (ga, sa), (gb, sb) = _three_keyframes(lvb_ctx, sc)
    guess = _perturbed(g["frame_pose"], np.random.default_rng(5), 0.05, 0.002)
    first = [new_call(fa, fs, sc, [0, 1, 2], 3, sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"]) for fa, fs in ((ga, sa), (gb, sb))]
    old_pose, rel = _candidate(sc, 1)
    reloc_call(ga, sa, sc, [0, 1, 2], old_pose, rel)
    for fa, fb, c, cell in ((ga, gb, g["scan"], g["cell_size"]), (sa, sb, s["scan"], s["cell_size"])):
        _same_handles(fa, fb, c, first[0][0], cell)
        fa.map_append(50, None, first[0][0])          # the keyframe call's scan is still the one map_append(NULL) stores
        fb.map_append(50, None, first[0][0])
    nxt = [new_call(fa, fs, sc, [1, 2, 3], 4, first[0][0], guess, g["scan"], s["scan"]) for fa, fs in ((ga, sa), (gb, sb))]
    _same_result(nxt[1][:3], nxt[0][:3])
    assert nxt[0][3] == nxt[1][3]
    for fa, fb, c, cell in ((ga, gb, g["scan"], g["cell_size"]), (sa, sb, s["scan"], s["cell_size"])):
        _same_handles(fa, fb, c, nxt[0][0], cell)
        for key in (0, 1, 2, 3, 4, 50):
            assert np.array_equal(_stored(fa, key, cell).view(np.uint32), _stored(fb, key, cell).view(np.uint32)), key


@pytest.mark.parametrize("side", ["ground", "surf"])
def test_skipped_side(lvb_ctx, scene, side):
    """ground: SegmentGround keeps no point (a merged cloud of fewer than 3 points); surf: an empty merged cloud.  That side is
    skipped in every round (termination_type -1, NaN score); the other side equals the step-by-step path."""
    sc = scene
    one = sc["kfs"][0][1][:1]
    (ga, sa), (gb, sb) = _three_keyframes(lvb_ctx, sc, ground=one if side == "ground" else None,
                                          surf=np.zeros((0, 4), np.float32) if side == "surf" else None)
    old_pose, rel = _candidate(sc, 0)
    step = step_by_step(ga, sa, sc, [0, 1], old_pose, rel)
    call = reloc_call(gb, sb, sc, [0, 1], old_pose, rel)
    m = 0 if side == "ground" else 1
    assert step[4][m] == 0 and step[4][1 - m] > 0
    _same_as_step(step, call)
    assert np.isnan(call[3][m]) and np.isfinite(call[3][1 - m]) and call[2][1 - m].num_iterations > 0


def _expected_launches(iters, n_scan, rounds, ransac=True):
    n = 2                                                                        # clone pose, relative_o_c and scores
    for m in range(2):
        n += (8 if m == 0 and ransac else 0) + 9                                 # SegmentGround (RANSAC 4, scan 3, gather), bbox .. scatter
    n += rounds * (1 + sum((6 if k >= 4096 else 0) + (1 if k > 0 else 0) + 4 * (iters + 1) + 1 for k in n_scan))
    return n


@pytest.mark.parametrize("rounds", [1, 4])
def test_counts(lvb_ctx, rounds):
    """One synchronisation per call (two on the first use of clouds stored by map_append); the launch sequence depends on the sizes,
    the options and `rounds` only: not on how many points SegmentGround keeps, nor on when the solvers stop."""
    sc = make_scene(6000, 3000, n_map=30000, seed=5)
    g, s = sc["g"], sc["s"]
    (gb, sb), _ = _three_keyframes(lvb_ctx, sc)
    old_pose, rel = _candidate(sc, 1)
    syncs, counts, kept, stops = [], [], [], []
    for thr, gtol in ((0.02, 1e-10), (0.02, 1e-10), (0.3, 1e-10), (0.02, 1e30)):
        opt = backend.default_options(lvb_ctx.api, max_num_iterations=4, linear_solver_type=backend.DENSE_QR, gradient_tolerance=gtol)
        n0, l0 = lvb_ctx.sync_count(), lvb_ctx.launch_count()
        _, _, sums, _, nm = reloc_call(gb, sb, sc, [0, 1, 2], old_pose, rel, thr=thr, rounds=rounds, options=opt)
        syncs.append(lvb_ctx.sync_count() - n0)
        counts.append(lvb_ctx.launch_count() - l0)
        kept.append(nm[0])
        stops.append([x.num_iterations for x in sums])
    assert syncs == [2, 1, 1, 1]
    assert counts[0] == counts[1] + 6                     # the first call's bounding boxes of the six map_append clouds
    assert len(set(counts[1:])) == 1 and counts[1] == _expected_launches(4, (len(g["scan"]), len(s["scan"])), rounds)
    assert kept[0] != kept[2]
    assert min(stops[0]) > 0 and stops[3] == [0, 0]


def test_errors_change_no_state(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    (gb, sb), _ = _three_keyframes(lvb_ctx, sc)
    args = (sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"])
    # key 8: a ground plane too wide for the voxel grid at any ring, found on the device after SegmentGround; stored with its box
    rng = np.random.default_rng(3)
    wide = np.zeros((4000, 4), np.float32)
    wide[:, :2] = rng.uniform(-5e4, 5e4, (4000, 2))
    new_call(gb, sb, sc, [], 8, args[0], args[1], _to_robot(wide, args[1]), s["scan"])
    new_call(gb, sb, sc, [0, 1, 2], 3, *args)          # the map frames every failed call must leave in place
    old_pose, rel = _candidate(sc, 1)
    reloc_call(gb, sb, sc, [0, 1], old_pose, rel)       # a relocation slot of the size the failed calls would need

    def snapshot():
        return [(fa.map_download(), fa.knn3(c, g["frame_pose"], 0.9 * cell * cell)) for fa, c, cell in
                ((gb, g["scan"], g["cell_size"]), (sb, s["scan"], s["cell_size"]))]

    def same(a, b):
        for (ma, (ia, da)), (mb, (ib, db)) in zip(a, b):
            assert np.array_equal(ma.view(np.uint32), mb.view(np.uint32)) and np.array_equal(ia, ib)
            assert np.array_equal(da.view(np.uint32), db.view(np.uint32))

    snap = snapshot()
    n0 = lvb_ctx.launch_count()
    capped = backend.default_options(lvb_ctx.api, max_num_iterations=4, linear_solver_type=backend.DENSE_QR, max_solver_time_in_seconds=1.0)
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        reloc_call(gb, sb, sc, [0, 1], old_pose, rel, options=capped)
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        reloc_call(gb, sb, sc, [0, 42], old_pose, rel)                           # not resident
    for bad_rounds in (0, 17):
        with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
            reloc_call(gb, sb, sc, [0, 1], old_pose, rel, rounds=bad_rounds)
    api = lvb_ctx.api
    prm = _capi.MapOptimizeParams()
    api.default_options(C.byref(prm.options))
    prm.options.max_num_iterations = 4
    for m in range(2):
        prm.weight[m], prm.huber_a[m], prm.dist_thr[m] = (g, s)[m]["weight"], (g, s)[m]["huber_a"], (g, s)[m]["thr"]
    k = (C.c_longlong * 3)(0, 1, 2)
    cs = np.array([g["cell_size"], s["cell_size"]], np.float32)
    outs = [np.zeros(7), np.zeros(7), np.zeros(2)]
    cg, cs_ = np.ascontiguousarray(g["scan"], np.float32), np.ascontiguousarray(s["scan"], np.float32)

    def raw(n_keys, prior_weight):
        prm.prior_weight = prior_weight
        return api.icp_map_relocate(gb.h, sb.h, k, n_keys, cs.ctypes.data_as(_capi.c_float_p), GT, backend._dp(np.array(args[0])),
                                    backend._dp(old_pose), backend._dp(rel), cg.ctypes.data_as(C.c_void_p), len(cg),
                                    cs_.ctypes.data_as(C.c_void_p), len(cs_), 16, C.byref(prm), 4, backend._dp(outs[0]),
                                    backend._dp(outs[1]), None, backend._dp(outs[2]), None)
    assert raw(0, -1.0) == -1                      # n_keys = 0: the reference dereferences an empty map there
    assert raw(4, -1.0) == -1
    assert raw(3, 0.0) == -1 and raw(3, 5.0) == -1  # the relocation never has a prior
    assert lvb_ctx.launch_count() == n0
    with pytest.raises(RuntimeError, match=r"failed \(-5\)"):
        reloc_call(gb, sb, sc, [0, 8], old_pose, rel)                           # found on the device
    same(snapshot(), snap)
    assert raw(3, -1.0) == 0                        # and the next call runs
    same(snapshot(), snap)


def test_sharded_context_is_unsupported():
    """world_size > 1 reports LVB_ERR_UNSUPPORTED and launches nothing (2 ranks; skipped on a single-GPU box)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29523", os.path.join(ROOT, "tests", "map_relocate_multigpu_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert "MAP RELOCATE MULTIGPU OK" in p.stdout


def _cloud(f, c):
    np.array([len(c)], np.int32).tofile(f)
    np.ascontiguousarray(np.asarray(c, np.float32)[:, :4]).tofile(f)


@pytest.mark.parametrize("place", sorted(PLACES))
def test_shim_relocate_keyframe_equals_the_per_call_sequence(lvb_ctx, scene, tmp_path, place):
    """include/lvio_b200/association.h: RelocateKeyframe against the reference's ScanToMapWith*(relocate = true) + ceres::Solve
    rounds on host map clouds (tests/cpp/relocate_shim.cpp): the same relative_o_c and the same integer score."""
    sc = scene
    g, s = sc["g"], sc["s"]
    keys, old = PLACES[place]
    old_pose, rel = _candidate(sc, old)
    (ga, sa), _ = _three_keyframes(lvb_ctx, sc)
    ga.map_build(keys, g["cell_size"], GT)          # the old map frame's clouds for the per-call sequence: merged, SegmentGround
    sa.map_build(keys, s["cell_size"])
    with open(tmp_path / "in.bin", "wb") as f:
        np.array([len(sc["kfs"])], np.int32).tofile(f)
        for pose, cg, cs in sc["kfs"]:
            np.asarray(pose, np.float64).tofile(f)
            _cloud(f, cg)
            _cloud(f, cs)
        np.array([len(keys)], np.int32).tofile(f)
        np.array(keys, np.int64).tofile(f)
        for x in (sc["kfs"][keys[0]][0], old_pose, rel, [GT]):
            np.asarray(x, np.float64).tofile(f)
        _cloud(f, g["scan"])
        _cloud(f, s["scan"])
        _cloud(f, ga.map_download())
        _cloud(f, sa.map_download())
    exe = str(tmp_path / "relocate_shim")
    lib_dir = os.path.join(ROOT, "lvio_fusion_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++14", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "relocate_shim.cpp"), "-L" + lib_dir, "-llvio_b200", "-Wl,-rpath," + lib_dir])
    p = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    out = np.fromfile(tmp_path / "out.bin").reshape(2, 8)
    assert np.max(np.abs(out[0, :7] - out[1, :7])) < 1e-9
    assert out[0, 7] == out[1, 7]


def test_python_argument_checks(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    (gb, sb), _ = _three_keyframes(lvb_ctx, sc)
    old_pose, rel = _candidate(sc, 1)
    with pytest.raises(ValueError):
        backend.relocate(gb, None, [0, 1], (g["cell_size"], s["cell_size"]), GT, sc["kfs"][0][0], old_pose, rel, g["scan"], s["scan"],
                         (g["weight"], s["weight"]), (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]))
    wide = np.zeros((len(s["scan"]), 8), np.float32)
    wide[:, :4] = s["scan"]
    with pytest.raises(ValueError):
        reloc_call(gb, sb, sc, [0, 1], old_pose, rel, cs=wide)
    opt = backend.default_options(lvb_ctx.api, max_num_iterations=4, linear_solver_type=backend.DENSE_QR)
    _, _, sums, _, _ = reloc_call(gb, sb, sc, [0, 1], old_pose, rel, options=opt, gradient_tolerance=1e30)
    assert [x.num_iterations for x in sums] == [0, 0] and opt.gradient_tolerance == 1e-10
