"""Mapping::Optimize(active_kfs) for a chain of keyframes in one device call (lvb_icp_map_optimize_keyframes, mapping.cpp:139-191):
the incoming poses chained through the earlier keyframes' transforms, map frames that merge clouds stored earlier in the call, both
registrations and ToWorld, with one host synchronisation.  Checked against the per-keyframe loop (lvb_icp_map_build_optimize_keyframe
per keyframe, the incoming poses composed by lvio_fusion_b200.se3 on the host), against the CPU oracle and through the C++ shim.

The linearisation adds its block sums atomically, so two runs of the same registration agree to the last bits only up to the order of
those sums: poses are held to 1e-11 as in the other keyframe tests.  Everything that does not depend on that order -- the transforms
against the host restatement, the stored clouds, the map frames, the 3-NN against them, the sizes -- is compared bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from lvio_fusion_b200 import _capi, backend, se3, synth
from test_gpu_map_optimize import _same_result, make_scene
from test_gpu_map_build_keyframe import GT, _frames, _pair, _same_handles, new_call

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0.0])


@pytest.fixture(scope="module")
def scene():
    return make_scene(6000, 5000)


def chain(gb, sb, sc, kfs, thr=GT, **kw):
    """kfs: (key, map_keys, map_pose, incoming pose, ground cloud, surf cloud) in time order."""
    g, s = sc["g"], sc["s"]
    return backend.build_and_optimize_keyframes(gb, sb, kfs, (g["cell_size"], s["cell_size"]), thr, (g["weight"], s["weight"]), sc["pw"],
                                                (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]), **kw)


def loop(ga, sa, sc, kfs, thr=GT, scenes=None, **kw):
    """The per-keyframe form of Mapping::Optimize: one lvb_icp_map_build_optimize_keyframe per keyframe, ForwardUpdate on the host.
    scenes: one scene per keyframe (its weights and prior weight), else sc for all.  Returns (pose, transform, rpyxyz, summaries,
    map points) per keyframe, as the chained call does."""
    out, Ts, poses = [], [], {}
    for i, (key, map_keys, map_pose, pose_in, cg, cs) in enumerate(kfs):
        incoming = se3.forward_update(Ts, pose_in)
        if map_keys and map_keys[-1] in poses:
            map_pose = poses[map_keys[-1]]
        p, e, sums, nm = new_call(ga, sa, scenes[i] if scenes else sc, list(map_keys), key, map_pose, incoming, cg, cs, thr=thr, **kw)
        T = se3.transform(p, incoming)
        Ts.append(T)
        poses[key] = p
        out.append((p, T, e, sums, nm))
    return out


def _check_transforms(kfs, call):
    """The device's transforms and incoming poses are the host restatement's, bit for bit, given the device's optimised poses."""
    Ts = []
    for (key, _, _, pose_in, _, _), (p, T, _, _, _) in zip(kfs, call):
        want = se3.transform(p, se3.forward_update(Ts, pose_in))
        assert np.array_equal(T.view(np.uint64), want.view(np.uint64)), key
        Ts.append(T)


def _same_chain(step, call):
    assert len(step) == len(call)
    for k, (a, b) in enumerate(zip(step, call)):
        _same_result((a[0], a[2], a[3]), (b[0], b[2], b[3]))
        assert np.max(np.abs(a[1] - b[1])) < 1e-11, k
        assert list(a[4]) == list(b[4]), k


def _stored(fa, key, cell):
    fa.map_build([key], cell)
    return fa.map_download()


def _both(fn, fa, fb):
    """fn on both handles: equal results, or both fail (no map frame yet, an empty stored cloud)."""
    out = []
    for f in (fa, fb):
        try:
            out.append(fn(f))
        except RuntimeError:
            out.append(None)
    assert (out[0] is None) == (out[1] is None)
    return out


def _same_state(sc, ha, hb, keys, probe):
    """Map frames, the 3-NN of a probe scan against them and map_append(NULL), then every stored cloud: bit for bit."""
    (ga, sa), (gb, sb) = ha, hb
    g, s = sc["g"], sc["s"]
    for fa, fb, scan, cell in ((ga, gb, probe[1], g["cell_size"]), (sa, sb, probe[2], s["cell_size"])):
        if _both(lambda f: f.map_download(), fa, fb)[0] is not None:
            _same_handles(fa, fb, scan, probe[0], cell)
    for fa, fb, cell in ((ga, gb, g["cell_size"]), (sa, sb, s["cell_size"])):
        fa.map_append(999, None, probe[0])
        fb.map_append(999, None, probe[0])
        for key in list(keys) + [999]:
            a, b = _both(lambda f: _stored(f, key, cell), fa, fb)
            assert a is None or np.array_equal(a.view(np.uint32), b.view(np.uint32)), key
        fa.map_evict(999)
        fb.map_evict(999)


def _window(frames, first, n):
    """Keyframes first .. first+n-1 of `frames`, each with the (up to) three keyframes before it as map keys."""
    return [(k, [j for j in range(k - 3, k) if j >= 0], IDENTITY, frames[k][0], frames[k][1], frames[k][2]) for k in range(first, first + n)]


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6])
def test_chain_from_the_first_keyframe_equals_the_loop(lvb_ctx, scene, n):
    """n_keys 0, 1, 2, 3, 3, 3: every map frame after the first merges clouds the call itself stored."""
    sc = scene
    frames = _frames(sc, 3)
    kfs = _window(frames, 0, n)
    ha, hb = _pair(lvb_ctx), _pair(lvb_ctx)
    step = loop(*ha, sc, kfs)
    n0 = lvb_ctx.sync_count()
    call = chain(*hb, sc, kfs)
    assert lvb_ctx.sync_count() - n0 == 1
    _same_chain(step, call)
    _check_transforms(kfs, call)
    if n > 1:
        assert all(x.num_iterations > 0 for x in call[-1][3]) and min(call[-1][4]) > 0
    _same_state(sc, ha, hb, range(n), frames[n - 1])


@pytest.mark.parametrize("n", [1, 3])
def test_chain_from_mid_map_equals_the_loop(lvb_ctx, scene, n):
    """Keyframes 3 .. 3+n-1 after three keyframes stored by earlier calls: map keys resident before the call and keys of the call."""
    sc = scene
    frames = _frames(sc, 3)
    ha, hb = _pair(lvb_ctx), _pair(lvb_ctx)
    poses = {k: r[0] for k, r in enumerate(loop(*ha, sc, _window(frames, 0, 3)))}
    loop(*hb, sc, _window(frames, 0, 3))
    kfs = [(k, mk, poses.get(mk[-1], IDENTITY), p, cg, cs) for k, mk, _, p, cg, cs in _window(frames, 3, n)]
    step = loop(*ha, sc, kfs)
    n0 = lvb_ctx.sync_count()
    call = chain(*hb, sc, kfs)
    assert lvb_ctx.sync_count() - n0 == 1
    _same_chain(step, call)
    _check_transforms(kfs, call)
    _same_state(sc, ha, hb, range(3 + n), frames[2 + n])


def test_each_keyframe_registers_with_its_own_weights(lvb_ctx, scene):
    """ScanToMapWith* take the lidar weights and the prior weight (features_left.size() * weights.visual) from each frame: keyframes
    with different ones give the loop's poses, and not those of one set of weights for the whole chain."""
    sc = scene
    g, s = sc["g"], sc["s"]
    frames = _frames(sc, 3)
    kfs = _window(frames, 0, 6)
    scenes = [sc]
    for k in range(1, 6):
        gk, sk = dict(g, weight=g["weight"] * (1.0 + 0.3 * k)), dict(s, weight=s["weight"] * (1.0 + 0.2 * (k % 3)))
        scenes.append(dict(sc, g=gk, s=sk, pw=sc["pw"] * (0.2 + 0.4 * k)))
    ha, hb = _pair(lvb_ctx), _pair(lvb_ctx)
    step = loop(*ha, sc, kfs, scenes=scenes)
    call = backend.build_and_optimize_keyframes(*hb, kfs, (g["cell_size"], s["cell_size"]), GT,
                                                [(x["g"]["weight"], x["s"]["weight"]) for x in scenes], [x["pw"] for x in scenes],
                                                (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]))
    _same_chain(step, call)
    _check_transforms(kfs, call)
    _same_state(sc, ha, hb, range(6), frames[5])
    shared = chain(*_pair(lvb_ctx), sc, kfs)                   # one set of weights for every keyframe registers elsewhere
    assert max(np.max(np.abs(a[0] - b[0])) for a, b in zip(call, shared)) > 1e-9


def test_one_keyframe_is_the_single_keyframe_call(lvb_ctx, scene):
    """n_kf = 1: lvb_icp_map_build_optimize_keyframe's result, stored clouds, launches and synchronisations."""
    sc = scene
    frames = _frames(sc, 1)
    ha, hb = _pair(lvb_ctx), _pair(lvb_ctx)
    for h in (ha, hb):
        loop(*h, sc, _window(frames, 0, 3))
    kfs = [(3, [0, 1, 2], frames[2][0], frames[3][0], frames[3][1], frames[3][2])]
    l0, n0 = lvb_ctx.launch_count(), lvb_ctx.sync_count()
    one = new_call(*ha, sc, [0, 1, 2], 3, frames[2][0], frames[3][0], frames[3][1], frames[3][2])
    l1, n1 = lvb_ctx.launch_count(), lvb_ctx.sync_count()
    call = chain(*hb, sc, kfs)
    assert lvb_ctx.launch_count() - l1 == l1 - l0 and lvb_ctx.sync_count() - n1 == n1 - n0 == 1
    _same_result(one[:3], (call[0][0], call[0][2], call[0][3]))
    assert list(one[3]) == list(call[0][4])
    _check_transforms(kfs, call)
    _same_state(sc, ha, hb, [0, 1, 2, 3], frames[3])


def test_launches_depend_on_sizes_only(lvb_ctx):
    """Two scenes of the same sizes, different data, different SegmentGround thresholds and solvers that stop at different
    iterations: the same launch count for a chain of 4, one synchronisation each."""
    counts, kept, stops = [], [], []
    for seed, thr, gtol in ((5, 0.02, 1e-10), (8, 0.3, 1e30)):
        sc = make_scene(6000, 3000, n_map=30000, seed=seed)
        frames = _frames(sc, 1)
        gb, sb = _pair(lvb_ctx)
        l0, n0 = lvb_ctx.launch_count(), lvb_ctx.sync_count()
        call = chain(gb, sb, sc, _window(frames, 0, 4), thr=thr, gradient_tolerance=gtol)
        assert lvb_ctx.sync_count() - n0 == 1
        counts.append(lvb_ctx.launch_count() - l0)
        kept.append([c[4][0] for c in call])
        stops.append([x.num_iterations for c in call[1:] for x in c[3]])
    assert counts[0] == counts[1]
    assert kept[0] != kept[1]
    assert min(stops[0]) > 0 and max(stops[1]) == 0


@pytest.mark.parametrize("side", ["ground", "surf"])
def test_skipped_sides_mid_chain_equal_the_loop(lvb_ctx, scene, side):
    """ground: keyframes 1 and 2 store one ground point, so the ground map frames of keyframes 2 and 3 keep no point after
    SegmentGround and the handle keeps keyframe 1's; surf: keyframe 1 stores no surf point, so keyframe 2 has no surf map frame."""
    sc = scene
    frames = _frames(sc, 1)
    kfs = []
    for k in range(4):
        pose, cg, cs = frames[k]
        if side == "ground" and k in (1, 2):
            cg = cg[:1]
        if side == "surf" and k == 1:
            cs = np.zeros((0, 4), np.float32)
        kfs.append((k, [k - 1] if k else [], IDENTITY, pose, cg, cs))
    ha, hb = _pair(lvb_ctx), _pair(lvb_ctx)
    step = loop(*ha, sc, kfs)
    call = chain(*hb, sc, kfs)
    _same_chain(step, call)
    _check_transforms(kfs, call)
    m = 0 if side == "ground" else 1
    assert call[2][4][m] == 0 and call[2][3][m].termination_type == -1 and call[2][4][1 - m] > 0
    if side == "ground":
        assert call[1][4][0] > 0 and call[3][4][0] == 0
    _same_state(sc, ha, hb, range(4), frames[3])


def test_cloud_outside_its_estimate_equals_the_loop(lvb_ctx, scene):
    """Keyframe 4 lies 2 km from keyframe 3 and is not registered, so keyframe 3's transform moves it by metres from the pose the caller
    gave: the map frame of keyframe 5 (a resident cloud at that pose and keyframe 4's) is larger than the host sized it for.  The grid
    kernel takes a coarser ring and the result is the loop's, which sizes from exact boxes.  Without the pose prior, keyframe 3's
    registration takes out most of its guess's 1 degree yaw error, which moves a keyframe 2 km away by tens of metres."""
    sc = dict(scene, pw=-1.0)
    g, s = sc["g"], sc["s"]
    far = g["frame_pose"].copy()
    far[4] += 2000.0
    ha, hb = _pair(lvb_ctx), _pair(lvb_ctx)
    for ga, sa in (ha, hb):
        for k, (pose, cg, cs) in enumerate(sc["kfs"]):
            ga.map_append(k, cg, pose)
            sa.map_append(k, cs, pose)
        ga.map_append(10, g["scan"], far)
        sa.map_append(10, s["scan"], far)
    kfs = [(3, [0, 1, 2], sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"]),
           (4, [], IDENTITY, far, g["scan"], s["scan"]),
           (5, [10, 4], IDENTITY, far, g["scan"], s["scan"])]
    step = loop(*ha, sc, kfs)
    call = chain(*hb, sc, kfs)
    _same_chain(step, call)
    _check_transforms(kfs, call)
    assert min(call[2][4]) > 0 and all(x.termination_type >= 0 for x in call[2][3])       # keyframe 5 registered on both sides
    # keyframe 4's cloud left the box the host estimated for it (robot-frame box at the caller's pose, widened by 1 m), and keyframe
    # 5's surf map frame -- the handle's map frame afterwards -- was hashed at a coarser ring than the loop's exactly sized one
    moved = np.max(np.abs(call[1][0][4:] - far[4:]))
    assert moved > 1.5, moved
    assert _grid(ha[1])[0] == 4 and _grid(hb[1])[0] < 4, (_grid(ha[1]), _grid(hb[1]))
    _same_state(sc, ha, hb, [3, 4, 5, 10], (call[2][0], g["scan"], s["scan"]))


def test_grid_that_fits_no_ring_commits_nothing(lvb_ctx, scene):
    """As above with keyframe 7 100 km away: keyframe 6's transform moves it by hundreds of metres, so keyframe 8's surf map frame does
    not fit the capacity sized for it even at ring 1.  Found on the device: LVB_ERR_UNSUPPORTED after the synchronisation, and no cloud,
    map frame or map_append(NULL) scan changes."""
    sc = dict(scene, pw=-1.0)
    g, s = sc["g"], sc["s"]
    far = g["frame_pose"].copy()
    far[4] += 1.0e5
    gb, sb = _pair(lvb_ctx)
    for k, (pose, cg, cs) in enumerate(sc["kfs"]):
        gb.map_append(k, cg, pose)
        sb.map_append(k, cs, pose)
    gb.map_append(10, g["scan"], far)
    sb.map_append(10, s["scan"], far)
    done = chain(gb, sb, sc, [(3, [0, 1, 2], sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"])])
    snap = [fa.map_download() for fa in (gb, sb)]
    grids = [_grid(fa) for fa in (gb, sb)]
    with pytest.raises(RuntimeError, match=r"failed \(-5\).*map frame"):
        chain(gb, sb, sc, [(6, [0, 1, 2], sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"]),
                           (7, [], IDENTITY, far, g["scan"], s["scan"]),
                           (8, [10, 7], IDENTITY, far, g["scan"], s["scan"])])
    for fa, before, grid in zip((gb, sb), snap, grids):
        assert np.array_equal(fa.map_download().view(np.uint32), before.view(np.uint32)) and _grid(fa) == grid
    ref = _pair(lvb_ctx)
    for fa, fr, cell, cloud in ((gb, ref[0], g["cell_size"], g["scan"]), (sb, ref[1], s["cell_size"], s["scan"])):
        fa.map_append(77, None, done[0][0])                      # still keyframe 3's scan
        fr.map_append(77, cloud, done[0][0])
        assert np.array_equal(_stored(fa, 77, cell).view(np.uint32), _stored(fr, 77, cell).view(np.uint32))
        for key in (6, 7, 8):
            with pytest.raises(RuntimeError):
                fa.map_build([key], 1.0)                          # nothing was stored


def _grid(fa):
    out = np.zeros(4, np.int32)
    fa.api.check(fa.api.debug_icp_map_grid(fa.h, out.ctypes.data_as(_capi.c_int_p)), "debug_icp_map_grid")
    return [int(x) for x in out]


def _raw_records(kfs):
    recs = (_capi.MapKeyframe * len(kfs))()
    keep = []
    for r, (key, mk, mp, p, cg, cs) in zip(recs, kfs):
        r.key, r.n_map_keys = key, len(mk)
        for i, x in enumerate(mk):
            r.map_keys[i] = x
        cg, cs = np.ascontiguousarray(cg, np.float32), np.ascontiguousarray(cs, np.float32)
        keep += [cg, cs]
        r.n_ground, r.n_surf = len(cg), len(cs)
        r.ground_pts, r.surf_pts = cg.ctypes.data_as(C.c_void_p), cs.ctypes.data_as(C.c_void_p)
        for i in range(7):
            r.map_pose[i], r.pose[i] = float(mp[i]), float(p[i])
    return recs, keep


def test_errors_change_no_state(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    frames = _frames(sc, 1)
    gb, sb = _pair(lvb_ctx)
    chain(gb, sb, sc, _window(frames, 0, 4))
    snap = [fa.map_download() for fa in (gb, sb)]
    api = lvb_ctx.api
    prm = _capi.MapOptimizeParams()
    api.default_options(C.byref(prm.options))
    prm.options.max_num_iterations = 4
    prm.options.linear_solver_type = backend.DENSE_QR
    for m, x in enumerate((g, s)):
        prm.weight[m], prm.huber_a[m], prm.dist_thr[m] = x["weight"], x["huber_a"], x["thr"]
    prm.prior_weight = sc["pw"]
    cs = np.array([g["cell_size"], s["cell_size"]], np.float32)
    f = frames[3]

    def raw(kfs, p=prm):
        recs, keep = _raw_records(kfs)
        return api.icp_map_optimize_keyframes(gb.h, sb.h, recs, len(kfs), cs.ctypes.data_as(_capi.c_float_p), GT, 16, C.byref(p))

    l0, n0 = lvb_ctx.launch_count(), lvb_ctx.sync_count()
    assert raw([(5, [42], IDENTITY, f[0], f[1], f[2])]) == -1                                        # unknown
    assert raw([(5, [3, 6], IDENTITY, f[0], f[1], f[2]), (6, [5], IDENTITY, f[0], f[1], f[2])]) == -1   # future
    assert raw([(5, [3], IDENTITY, f[0], f[1], f[2]), (5, [3], IDENTITY, f[0], f[1], f[2])]) == -1      # listed twice
    assert raw([(5, [3, 5], IDENTITY, f[0], f[1], f[2])]) == -1                                      # its own map key
    capped = _capi.MapOptimizeParams.from_buffer_copy(prm)
    capped.options.max_solver_time_in_seconds = 1.0
    assert raw([(5, [3], IDENTITY, f[0], f[1], f[2])], capped) == -1                                 # time limit
    bad_cells = cs.copy()
    bad_cells[0] = 0.0
    recs, keep = _raw_records([(5, [3], IDENTITY, f[0], f[1], f[2])])
    assert api.icp_map_optimize_keyframes(gb.h, sb.h, recs, 1, bad_cells.ctypes.data_as(_capi.c_float_p), GT, 16, C.byref(prm)) == -1  # cell size
    wide = _capi.MapOptimizeParams.from_buffer_copy(prm)
    wide.dist_thr[1] = 2.0 * float(cs[1]) ** 2
    assert raw([(5, [3], IDENTITY, f[0], f[1], f[2])], wide) == -1                                   # gate beyond the cell size
    other = backend.Context(api)
    so = backend.FeatureAssociation(other)
    assert api.icp_map_optimize_keyframes(gb.h, so.h, recs, 1, cs.ctypes.data_as(_capi.c_float_p), GT, 16, C.byref(prm)) == -1  # two contexts
    so.close()
    other.close()
    assert raw([]) == 0
    assert lvb_ctx.launch_count() == l0 and lvb_ctx.sync_count() == n0
    # found on the device after the synchronisation: keyframe 6's surf map frame merges keyframe 5's cloud, which holds an infinite point
    bad = f[2].copy()
    bad[5, 0] = np.inf
    with pytest.raises(RuntimeError, match=r"failed \(-1\).*finite"):
        chain(gb, sb, sc, [(5, [3], IDENTITY, f[0], f[1], bad), (6, [3, 5], IDENTITY, f[0], f[1], f[2])])
    for fa, before in zip((gb, sb), snap):
        assert np.array_equal(fa.map_download().view(np.uint32), before.view(np.uint32))
        for key in (5, 6):
            with pytest.raises(RuntimeError):
                fa.map_build([key], 1.0)                                  # nothing was stored
    # map_append(NULL) still refers to the last successful call's last scan
    ref = _pair(lvb_ctx)
    loop(*ref, sc, _window(frames, 0, 4))
    for fa, fr, cell, cloud in ((gb, ref[0], g["cell_size"], f[1]), (sb, ref[1], s["cell_size"], f[2])):
        fa.map_append(77, None, f[0])
        fr.map_append(77, cloud, f[0])
        assert np.array_equal(_stored(fa, 77, cell).view(np.uint32), _stored(fr, 77, cell).view(np.uint32))
    out = chain(gb, sb, sc, [(5, [3], IDENTITY, f[0], f[1], f[2])])       # and the next call runs
    assert all(x.num_iterations > 0 for x in out[0][3])


def test_chain_against_the_oracle(lvb_ctx, orc_ctx, scene):
    """The same chain through the oracle: CPU merge of the world clouds, SegmentGround, orc_icp_scan_to_map, ForwardUpdate on the host."""
    sc = scene
    g, s = sc["g"], sc["s"]
    frames = _frames(sc, 3)
    kfs = _window(frames, 0, 6)
    call = chain(*_pair(lvb_ctx), sc, kfs)
    og, os_ = _pair(orc_ctx)
    lidar = backend.LidarFeatures(orc_ctx)
    world, poses, Ts = {}, {}, []
    for (key, keys, _, pose_in, cg, cs), got in zip(kfs, call):
        p = se3.forward_update(Ts, pose_in)
        incoming = p.copy()
        if keys:
            map_pose = poses[keys[-1]]
            og.set_map(lidar.segment_ground(np.concatenate([world[j][0] for j in keys]), GT), g["cell_size"])
            os_.set_map(np.concatenate([world[j][1] for j in keys]), s["cell_size"])
            e = synth.relative_rpyxyz(map_pose, p)
            e, _ = og.scan_to_map(0, cg, p, map_pose, e, g["weight"], sc["pw"], g["huber_a"], g["thr"])
            p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
            e, _ = os_.scan_to_map(1, cs, p, map_pose, e, s["weight"], sc["pw"], s["huber_a"], s["thr"])
            p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
        world[key] = (og.transform_cloud(cg, p), os_.transform_cloud(cs, p))
        Ts.append(se3.transform(p, incoming))
        poses[key] = p
        assert np.max(np.abs(got[0] - p)) < 1e-7, key


def test_shim_chain_equals_per_keyframe_loop(lvb_ctx, scene, tmp_path):
    """include/lvio_b200/association.h: a Mapping::Optimize-shaped pass through OptimizeKeyframes against the per-keyframe
    OptimizeKeyframe + host ForwardUpdate loop of the same harness: the same poses and the same stored clouds."""
    sc = scene
    frames = _frames(sc, 3)
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
    exe = str(tmp_path / "shim")
    subprocess.check_call(["g++", "-O2", "-std=c++14", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "map_optimize_keyframes_shim.cpp"), "-L" + lib_dir, "-llvio_b200",
                           "-Wl,-rpath," + lib_dir])
    p = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr + p.stdout
    assert "SAME CLOUDS" in p.stdout, p.stdout
    out = np.fromfile(tmp_path / "out.bin").reshape(2, len(frames), 7)
    assert np.max(np.abs(out[0] - out[1])) < 1e-11


def test_sharded_context_is_unsupported():
    """world_size > 1 reports LVB_ERR_UNSUPPORTED and stores nothing (2 ranks; skipped on a single-GPU box)."""
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29525", os.path.join(ROOT, "tests", "map_optimize_keyframes_multigpu_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert "MAP OPTIMIZE KEYFRAMES MULTIGPU OK" in p.stdout
