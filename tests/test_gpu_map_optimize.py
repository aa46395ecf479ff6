"""Mapping::Optimize for one keyframe in one device call (lvb_icp_map_optimize_keyframe, mapping.cpp:147-185): both scan-to-map
solves, the pose hand-off between them and ToWorld, against the step-by-step path through the existing entry points (map_build x2,
scan_to_map mode 0, the pose through synth's host conversions, scan_to_map mode 1 from the updated pose, map_append x2) and against
the CPU oracle."""
import os
import subprocess
import sys

import numpy as np
import pytest

from lvio_fusion_b200 import backend, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

INT_FIELDS = ("num_iterations", "num_successful_steps", "termination_type", "num_residual_blocks", "num_residual_blocks_reduced")


def _perturbed(pose, rng, t_sigma, r_sigma):
    out = pose.copy()
    out[4:] += rng.normal(0, t_sigma, 3)
    out[:4] = synth.quat_mul(synth.quat_from_rotvec(rng.normal(0, r_sigma, 3)[None]), pose[:4][None])[0]
    return out


def _to_robot(world, pose):
    out = np.zeros((len(world), 4), dtype=np.float32)
    out[:, :3] = synth.se3_inv_apply(np.broadcast_to(pose, (len(world), 7)), world[:, :3].astype(np.float64)).astype(np.float32)
    return out


def make_scene(n_ground, n_surf, n_map=60000, seed=31):
    """A ground scene and a surf scene of make_icp_problem (same robot, map frame and initial pose), their maps split into three
    keyframes: (pose, robot-frame ground cloud, robot-frame surf cloud)."""
    g = synth.make_icp_problem(n_ground, n_map, seed=seed, kind="ground")
    s = synth.make_icp_problem(n_surf, n_map, seed=seed, kind="surf")
    rng = np.random.default_rng(seed)
    kfs = []
    for ig, is_ in zip(np.array_split(np.arange(n_map), 3), np.array_split(np.arange(n_map), 3)):
        pose = _perturbed(g["map_pose"], rng, 0.5, 0.02)
        kfs.append((pose, _to_robot(g["map"][ig], pose), _to_robot(s["map"][is_], pose)))
    return dict(g=g, s=s, kfs=kfs, pw=g["n_features_left"] * synth.W_VISUAL, rng=rng)


@pytest.fixture(scope="module")
def scene():
    return make_scene(6000, 5000)


def _handles(ctx, sc):
    """One (ground, surf) pair holding the scene's three keyframes under keys 0, 1, 2."""
    ga, sa = backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)
    for k, (pose, cg, cs) in enumerate(sc["kfs"]):
        ga.map_append(k, cg, pose)
        sa.map_append(k, cs, pose)
    return ga, sa


def _build(ga, sa, sc, keys):
    if ga is not None:
        ga.map_build(keys, sc["g"]["cell_size"])
    if sa is not None:
        sa.map_build(keys, sc["s"]["cell_size"])


def step_by_step(ga, sa, sc, key, map_pose, pose, ground_scan, surf_scan, **kw):
    """mapping.cpp:147-185 through the per-registration entry points, the pose composed on the host."""
    g, s = sc["g"], sc["s"]
    e = synth.relative_rpyxyz(map_pose, pose)
    sums = [None, None]
    if ga is not None:
        e, sums[0] = ga.scan_to_map(0, ground_scan, pose, map_pose, e, g["weight"], sc["pw"], g["huber_a"], g["thr"], **kw)
        pose = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
    if sa is not None:
        e, sums[1] = sa.scan_to_map(1, surf_scan, pose, map_pose, e, s["weight"], sc["pw"], s["huber_a"], s["thr"], **kw)
        pose = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
    for fa in (ga, sa):
        if fa is not None:
            fa.map_evict(key)
            fa.map_append(key, None, pose)
    return pose, e, sums


def one_call(gb, sb, sc, key, map_pose, pose, ground_scan, surf_scan, **kw):
    g, s = sc["g"], sc["s"]
    return backend.optimize_keyframe(gb, sb, key, map_pose, pose, ground_scan, surf_scan, (g["weight"], s["weight"]), sc["pw"],
                                     (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]), **kw)


def _same_summary(a, b):
    for f in INT_FIELDS:
        assert getattr(a, f) == getattr(b, f), f
    for f in ("initial_cost", "final_cost"):
        assert abs(getattr(a, f) - getattr(b, f)) <= 1e-12 * max(1e-30, abs(getattr(b, f))), f


def _same_result(step, call):
    (ps, es, ss), (pc, ec, sc_) = step, call
    assert np.max(np.abs(pc - ps)) < 1e-11
    assert np.max(np.abs(ec - es)) < 1e-11
    for a, b in zip(sc_, ss):
        if b is not None:
            _same_summary(a, b)


def _stored(fa, key, cell):
    fa.map_build([key], cell)
    return fa.map_download()


def test_one_keyframe_equals_step_by_step(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    ga, sa = _handles(lvb_ctx, sc)
    gb, sb = _handles(lvb_ctx, sc)
    map_pose = sc["kfs"][2][0]
    _build(ga, sa, sc, [0, 1, 2])
    step = step_by_step(ga, sa, sc, 3, map_pose, g["frame_pose"], g["scan"], s["scan"])
    _build(gb, sb, sc, [0, 1, 2])
    call = one_call(gb, sb, sc, 3, map_pose, g["frame_pose"], g["scan"], s["scan"])
    _same_result(step, call)
    assert call[2][0].num_residual_blocks > 1000 and call[2][1].num_residual_blocks > 1000
    assert call[2][0].num_iterations > 0 and call[2][1].num_iterations > 0
    # ToWorld: the clouds stored under the key are map_append of the same clouds with the returned pose, bit for bit
    ref_g, ref_s = backend.FeatureAssociation(lvb_ctx), backend.FeatureAssociation(lvb_ctx)
    ref_g.map_append(3, g["scan"], call[0])
    ref_s.map_append(3, s["scan"], call[0])
    for fb, fr, cell in ((gb, ref_g, g["cell_size"]), (sb, ref_s, s["cell_size"])):
        assert np.array_equal(_stored(fb, 3, cell).view(np.uint32), _stored(fr, 3, cell).view(np.uint32))
    # the scan of the call stays on the device for lvb_icp_map_append(NULL)
    sb.map_append(50, None, call[0])
    assert np.array_equal(_stored(sb, 50, s["cell_size"]).view(np.uint32), _stored(ref_s, 3, s["cell_size"]).view(np.uint32))


def _sliding_inputs(sc, n):
    rng = np.random.default_rng(77)
    return [_perturbed(sc["g"]["frame_pose"], rng, 0.05, 0.002) for _ in range(n)]


def test_sliding_run_of_six_keyframes(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    ga, sa = _handles(lvb_ctx, sc)
    gb, sb = _handles(lvb_ctx, sc)
    poses = {k: kf[0] for k, kf in enumerate(sc["kfs"])}
    for j, guess in enumerate(_sliding_inputs(sc, 6)):
        key = 3 + j
        keys = [key - 3, key - 2, key - 1]
        map_pose = poses[key - 1]
        _build(ga, sa, sc, keys)
        step = step_by_step(ga, sa, sc, key, map_pose, guess, g["scan"], s["scan"])
        _build(gb, sb, sc, keys)
        call = one_call(gb, sb, sc, key, map_pose, guess, g["scan"], s["scan"])
        _same_result(step, call)
        poses[key] = call[0]
        for fa in (ga, sa, gb, sb):
            fa.map_evict(key - 3)


def test_sliding_run_against_the_oracle(lvb_ctx, orc_ctx, scene):
    """The same sequence through orc_icp_scan_to_map with the map frames merged and the poses composed on the host."""
    sc = scene
    g, s = sc["g"], sc["s"]
    gb, sb = _handles(lvb_ctx, sc)
    og, os_ = backend.FeatureAssociation(orc_ctx), backend.FeatureAssociation(orc_ctx)
    world = {k: (og.transform_cloud(cg, p), os_.transform_cloud(cs, p)) for k, (p, cg, cs) in enumerate(sc["kfs"])}
    poses = {k: kf[0] for k, kf in enumerate(sc["kfs"])}
    for j, guess in enumerate(_sliding_inputs(sc, 3)):
        key = 3 + j
        keys = [key - 3, key - 2, key - 1]
        map_pose = poses[key - 1]
        og.set_map(np.concatenate([world[k][0] for k in keys]), g["cell_size"])
        os_.set_map(np.concatenate([world[k][1] for k in keys]), s["cell_size"])
        e = synth.relative_rpyxyz(map_pose, guess)
        e, _ = og.scan_to_map(0, g["scan"], guess, map_pose, e, g["weight"], sc["pw"], g["huber_a"], g["thr"])
        p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
        e, _ = os_.scan_to_map(1, s["scan"], p, map_pose, e, s["weight"], sc["pw"], s["huber_a"], s["thr"])
        p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
        world[key] = (og.transform_cloud(g["scan"], p), os_.transform_cloud(s["scan"], p))
        _build(gb, sb, sc, keys)
        pc, ec, _ = one_call(gb, sb, sc, key, map_pose, guess, g["scan"], s["scan"])
        assert np.max(np.abs(pc - p)) < 1e-7 and np.max(np.abs(ec - e)) < 1e-7
        poses[key] = pc


@pytest.mark.parametrize("skip", ["ground", "surf"])
def test_null_handle_skips_its_registration(lvb_ctx, scene, skip):
    sc = scene
    g, s = sc["g"], sc["s"]
    ga, sa = _handles(lvb_ctx, sc)
    gb, sb = _handles(lvb_ctx, sc)
    if skip == "ground":
        ga = gb = None
    else:
        sa = sb = None
    map_pose = sc["kfs"][2][0]
    _build(ga, sa, sc, [0, 1, 2])
    step = step_by_step(ga, sa, sc, 3, map_pose, g["frame_pose"], g["scan"], s["scan"])
    _build(gb, sb, sc, [0, 1, 2])
    call = one_call(gb, sb, sc, 3, map_pose, g["frame_pose"], None if skip == "ground" else g["scan"], None if skip == "surf" else s["scan"])
    _same_result(step, call)
    skipped = call[2][0 if skip == "ground" else 1]
    assert skipped.termination_type == -1 and skipped.num_iterations == 0 and skipped.num_residual_blocks == 0
    ran = call[2][1 if skip == "ground" else 0]
    assert ran.num_iterations > 0 and ran.num_residual_blocks > 1000
    if skip == "ground":      # the surf registration starts from the unchanged rpyxyz and the incoming pose
        e0 = synth.relative_rpyxyz(map_pose, g["frame_pose"])
        assert np.max(np.abs(call[1][[1, 2, 5]] - e0[[1, 2, 5]])) < 1e-12


def test_resident_key_is_replaced(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    gb, sb = _handles(lvb_ctx, sc)
    _build(gb, sb, sc, [0, 1, 2])
    p1 = one_call(gb, sb, sc, 1, sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"])[0]      # key 1 is resident
    assert gb.map_build([1], g["cell_size"]) == len(g["scan"]) and sb.map_build([1], s["cell_size"]) == len(s["scan"])
    ref = backend.FeatureAssociation(lvb_ctx)
    ref.map_append(1, s["scan"], p1)
    assert np.array_equal(_stored(sb, 1, s["cell_size"]).view(np.uint32), _stored(ref, 1, s["cell_size"]).view(np.uint32))
    with pytest.raises(RuntimeError):
        sb.map_append(1, s["scan"], p1)          # map_append keeps refusing a resident key


def test_errors_change_no_state(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    gb, sb = _handles(lvb_ctx, sc)
    _build(gb, sb, sc, [0, 1, 2])
    n0 = lvb_ctx.launch_count()
    capped = backend.default_options(lvb_ctx.api, max_num_iterations=4, linear_solver_type=backend.DENSE_QR, max_solver_time_in_seconds=1.0)
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        one_call(gb, sb, sc, 3, sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"], options=capped)
    fresh = backend.FeatureAssociation(lvb_ctx)
    with pytest.raises(RuntimeError, match=r"failed \(-3\)"):
        one_call(gb, fresh, sc, 3, sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"])
    assert lvb_ctx.launch_count() == n0
    for fa in (gb, sb):
        with pytest.raises(RuntimeError):
            fa.map_build([3], 1.0)                # nothing was stored
    # the maps built before are still there: the same call without the cap runs
    _, _, sums = one_call(gb, sb, sc, 3, sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"])
    assert sums[0].num_iterations > 0 and sums[1].num_iterations > 0


def _expected_launches(iters, sizes):
    n = 1
    for k in sizes:
        n += (5 if k >= 4096 else 0) + (1 if k > 0 else 0) + 4 * (iters + 1) + 1 + (1 if k > 0 else 0)
    return n


@pytest.mark.parametrize("n_ground,n_surf", [(6000, 5000), (3000, 2000), (6000, 2000)])
@pytest.mark.parametrize("iters", [1, 4])
def test_launch_count_is_fixed(lvb_ctx, n_ground, n_surf, iters):
    sc = make_scene(n_ground, n_surf, n_map=30000, seed=5)
    g, s = sc["g"], sc["s"]
    gb, sb = _handles(lvb_ctx, sc)
    counts, stops = [], []
    for gtol in (1e-10, 1e30):     # the second solver stops before its first step
        _build(gb, sb, sc, [0, 1, 2])
        opt = backend.default_options(lvb_ctx.api, max_num_iterations=iters, linear_solver_type=backend.DENSE_QR, gradient_tolerance=gtol)
        n0 = lvb_ctx.launch_count()
        _, _, sums = one_call(gb, sb, sc, 3, sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"], options=opt)
        counts.append(lvb_ctx.launch_count() - n0)
        stops.append([x.num_iterations for x in sums])
    assert counts[0] == counts[1] == _expected_launches(iters, (n_ground, n_surf))
    assert min(stops[0]) > 0 and stops[1] == [0, 0]


def _shim_frames(sc):
    """Mapping::Optimize's keyframes for the shim loop: the scene's three keyframes (each registered against the ones before it; the
    first has no map frame), then two registrations of the scans."""
    g, s = sc["g"], sc["s"]
    return list(sc["kfs"]) + [(guess, g["scan"], s["scan"]) for guess in _sliding_inputs(sc, 2)]


def test_shim_mapping_loop_equals_c_abi(lvb_ctx, scene, tmp_path):
    """include/lvio_b200/association.h: BuildMapFrame + OptimizeKeyframe over Mapping::Optimize's loop, the first keyframe
    included.  Its BuildMapFrame has no keys, so nothing is registered, and ToWorld still stores its clouds (mapping.cpp:185):
    without them no later map frame could be built.  Every pose must match the same sequence through the C ABI."""
    sc = scene
    frames = _shim_frames(sc)
    exe = str(tmp_path / "map_optimize_shim")
    lib_dir = os.path.join(ROOT, "lvio_fusion_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++14", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "map_optimize_shim.cpp"), "-L" + lib_dir, "-llvio_b200", "-Wl,-rpath," + lib_dir])
    with open(tmp_path / "in.bin", "wb") as f:
        np.array([len(frames)], np.int32).tofile(f)
        np.array([synth.W_VISUAL], np.float64).tofile(f)
        np.array([sc["g"]["n_features_left"]], np.int32).tofile(f)
        for pose, cg, cs in frames:
            np.asarray(pose, np.float64).tofile(f)
            for c in (cg, cs):
                np.array([len(c)], np.int32).tofile(f)
                np.ascontiguousarray(c[:, :4], np.float32).tofile(f)
    p = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    out = np.fromfile(tmp_path / "out.bin").reshape(len(frames), 9)
    ga, sa = backend.FeatureAssociation(lvb_ctx), backend.FeatureAssociation(lvb_ctx)
    poses = {}
    for k, (pose, cg, cs) in enumerate(frames):
        keys = [j for j in range(k - 3, k) if j >= 0]
        if keys:
            _build(ga, sa, sc, keys)
            pk, _, sums = one_call(ga, sa, sc, k, poses[keys[-1]], pose, cg, cs)
            terms = [x.termination_type for x in sums]
        else:                       # the first keyframe: ToWorld only
            ga.map_append(k, cg, pose)
            sa.map_append(k, cs, pose)
            pk, terms = np.asarray(pose), [-1, -1]
        if k >= 3:
            ga.map_evict(k - 3)
            sa.map_evict(k - 3)
        poses[k] = pk
        assert np.max(np.abs(out[k, :7] - pk)) < 1e-11, k
        assert list(out[k, 7:]) == terms, k
    assert list(out[0, 7:]) == [-1, -1] and (out[1:, 7:] >= 0).all()


def test_sharded_context_is_unsupported():
    """world_size > 1 reports LVB_ERR_UNSUPPORTED and stores nothing (2 ranks; skipped on a single-GPU box)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29519", os.path.join(ROOT, "tests", "map_optimize_multigpu_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert "MAP OPTIMIZE MULTIGPU OK" in p.stdout


def test_python_argument_checks(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    gb, sb = _handles(lvb_ctx, sc)
    wide = np.zeros((len(s["scan"]), 8), np.float32)
    wide[:, :4] = s["scan"]
    with pytest.raises(ValueError):             # one record stride for both clouds
        one_call(gb, sb, sc, 3, sc["kfs"][2][0], g["frame_pose"], g["scan"], wide)
    with pytest.raises(ValueError):
        one_call(None, None, sc, 3, sc["kfs"][2][0], g["frame_pose"], None, None)
    # keyword options apply on top of an explicit options structure, which is left as it was
    _build(gb, sb, sc, [0, 1, 2])
    opt = backend.default_options(lvb_ctx.api, max_num_iterations=4, linear_solver_type=backend.DENSE_QR)
    _, _, sums = one_call(gb, sb, sc, 3, sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"], options=opt, gradient_tolerance=1e30)
    assert [x.num_iterations for x in sums] == [0, 0] and opt.gradient_tolerance == 1e-10
