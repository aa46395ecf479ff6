"""Mapping::ToWorld(start) on the device-resident keyframe clouds (lvb_icp_map_to_world, mapping.cpp:206-229): after a GNSS or loop
correction the world clouds of any number of keyframes are re-made from their robot-frame records, kept on the device since they were
stored, in one kernel with one host synchronisation.  Checked against map_evict + map_append of the host robot clouds on a second pair
of handles with the same history (clouds stored by every entry point that stores one), against the CPU oracle's MergeScan, and for
leaving everything it does not list alone."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from lvio_fusion_b200 import backend, synth
from test_gpu_map_build_keyframe import GT, _pair, _same_handles, _three_keyframes, new_call
from test_gpu_map_optimize import _perturbed, _same_result, _same_summary, _stored, make_scene, one_call
from test_gpu_map_relocate import _candidate, reloc_call

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def scene():
    return make_scene(6000, 5000)


def _strided(cloud, stride):
    """The cloud's records at `stride` bytes: 12 (x y z), 16 (x y z intensity) or 32 (pcl::PointXYZI with its padding)."""
    out = np.zeros((len(cloud), stride // 4), np.float32)
    k = min(4, stride // 4)
    out[:, :k] = cloud[:, :k]
    if stride == 32:
        out[:, 4:] = np.arange(4, dtype=np.float32) + 7.0          # padding the store must not carry over
    return out


def _history(ctx, sc):
    """Two handle pairs with the same history, clouds stored by every path: map_append at strides 16 (keys 0-2), 12 (key 10) and
    32 (key 11), map_append(NULL) of a knn3 scan (key 12), optimize_keyframe (key 3) and build_and_optimize_keyframe (key 4).
    Returns the pairs, the robot-frame clouds and the poses they were stored with on the first pair (key -> (ground, surf), key ->
    pose; the keyframe calls' poses of the two pairs may differ in the last bits: their reductions add in any order)."""
    g, s = sc["g"], sc["s"]
    pairs = _three_keyframes(ctx, sc)
    robot = {k: (cg, cs) for k, (_, cg, cs) in enumerate(sc["kfs"])}
    pose = {k: p for k, (p, _, _) in enumerate(sc["kfs"])}
    rng = np.random.default_rng(17)
    for key, stride, src in ((10, 12, 0), (11, 32, 1)):
        pose[key] = _perturbed(sc["kfs"][src][0], rng, 0.3, 0.01)
        robot[key] = (_strided(sc["kfs"][src][1], stride), _strided(sc["kfs"][src][2], stride))
    pose[12] = _perturbed(g["frame_pose"], rng, 0.05, 0.002)
    robot[12] = (g["scan"], s["scan"])
    guess3, guess4 = _perturbed(g["frame_pose"], rng, 0.05, 0.002), _perturbed(g["frame_pose"], rng, 0.05, 0.002)
    for j, (ga, sa) in enumerate(pairs):
        for key in (10, 11):
            ga.map_append(key, robot[key][0], pose[key])
            sa.map_append(key, robot[key][1], pose[key])
        for fa, cell, c in ((ga, g["cell_size"], g["scan"]), (sa, s["cell_size"], s["scan"])):
            fa.map_build([0, 1, 2], cell)
            fa.knn3(c, g["frame_pose"], 0.9 * cell * cell)            # leaves its scan on the device
            fa.map_append(12, None, pose[12])
        p3, _, _ = one_call(ga, sa, sc, 3, sc["kfs"][2][0], guess3, g["scan"], s["scan"])
        p4, _, _, _ = new_call(ga, sa, sc, [1, 2, 3], 4, p3, guess4, g["scan"], s["scan"])
        if j == 0:
            pose[3], pose[4] = p3, p4
    robot[3] = robot[4] = (g["scan"], s["scan"])
    return pairs, robot, pose


KEYS = [0, 1, 2, 3, 4, 10, 11, 12]


def _moved(pose, keys, seed=23):
    rng = np.random.default_rng(seed)
    return {k: _perturbed(pose[k], rng, 0.2, 0.01) for k in keys}


def _evict_append(fa, fs, robot, moved):
    for k, p in moved.items():
        fa.map_evict(k)
        fa.map_append(k, robot[k][0], p)
        fs.map_evict(k)
        fs.map_append(k, robot[k][1], p)


def _to_world(fa, fs, moved):
    keys = list(moved)
    backend.map_to_world(fa, fs, keys, np.array([moved[k] for k in keys]))


def _same_clouds(a, b, sc, keys):
    for fa, fb, cell in ((a[0], b[0], sc["g"]["cell_size"]), (a[1], b[1], sc["s"]["cell_size"])):
        for k in keys:
            assert np.array_equal(_stored(fa, k, cell).view(np.uint32), _stored(fb, k, cell).view(np.uint32)), k


def test_equals_evict_and_append(lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    ((ga, sa), (gb, sb)), robot, pose = _history(lvb_ctx, sc)
    moved = _moved(pose, KEYS)
    _to_world(ga, sa, dict(reversed(list(moved.items()))))             # any order
    _evict_append(gb, sb, robot, moved)
    _same_clouds((ga, sa), (gb, sb), sc, KEYS)
    # merged three-key map frames, with and without the ground RANSAC, and 3-NN against them
    for keys in ([0, 3, 11], [12, 4, 10], [1, 2, 4]):
        for thr in (GT, -1.0):
            ga.map_build(keys, g["cell_size"], thr)
            gb.map_build(keys, g["cell_size"], thr)
            _same_handles(ga, gb, g["scan"], moved[keys[-1]], g["cell_size"])
        sa.map_build(keys, s["cell_size"])
        sb.map_build(keys, s["cell_size"])
        _same_handles(sa, sb, s["scan"], moved[keys[-1]], s["cell_size"])


def test_against_the_oracle(lvb_ctx, orc_ctx, scene):
    """The re-anchored clouds are the oracle's MergeScan of the robot-frame clouds at the new poses, bit for bit."""
    sc = scene
    ((ga, sa), _), robot, pose = _history(lvb_ctx, sc)
    og, os_ = _pair(orc_ctx)
    moved = _moved(pose, KEYS, seed=29)
    _to_world(ga, sa, moved)
    for m, (fa, o, cell) in enumerate(((ga, og, sc["g"]["cell_size"]), (sa, os_, sc["s"]["cell_size"]))):
        for k in KEYS:
            want = o.transform_cloud(robot[k][m], moved[k])[:, :3]
            got = _stored(fa, k, cell)[:, :3]
            assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(want).view(np.uint32)), (m, k)


def test_downstream_calls_agree(lvb_ctx, scene):
    """After re-anchoring, the next keyframe call and a relocation of an old candidate give what they give after evict + append; a
    relocation between the correction and the next keyframe call changes nothing for that call."""
    sc = scene
    g, s = sc["g"], sc["s"]
    (pa, pb), robot, pose = _history(lvb_ctx, sc)
    moved = _moved(pose, KEYS, seed=31)
    _to_world(*pa, moved)
    _evict_append(*pb, robot, moved)
    old_pose = moved[1]
    rel = synth.se3_mul(synth.se3_inv(old_pose), _perturbed(g["frame_pose"], np.random.default_rng(11), 0.05, 0.002))
    outs = []
    for fa, fs in (pa, pb):
        r = backend.relocate(fa, fs, [0, 1, 2], (g["cell_size"], s["cell_size"]), GT, moved[0], old_pose, rel, g["scan"], s["scan"],
                             (g["weight"], s["weight"]), (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]))
        guess = _perturbed(g["frame_pose"], np.random.default_rng(3), 0.05, 0.002)
        k = new_call(fa, fs, sc, [3, 4, 10], 5, moved[10], guess, g["scan"], s["scan"])
        outs.append((r, k))
    (ra, ka), (rb, kb) = outs
    assert np.max(np.abs(ra[0] - rb[0])) < 1e-11 and np.max(np.abs(ra[1] - rb[1])) < 1e-11
    for m in range(2):
        _same_summary(ra[2][m], rb[2][m])
        assert ra[3][m] == rb[3][m] and ra[4][m] == rb[4][m]
    assert min(ra[4]) > 0 and all(x.num_iterations > 0 for x in ra[2])
    _same_result(kb[:3], ka[:3])
    assert ka[3] == kb[3] and min(ka[3]) > 0
    _same_handles(pa[0], pb[0], g["scan"], ka[0], g["cell_size"])
    _same_handles(pa[1], pb[1], s["scan"], ka[0], s["cell_size"])


def test_no_drift(lvb_ctx, scene):
    """Re-anchoring at A then B equals re-anchoring once at B; re-anchoring at the stored poses changes no bit."""
    sc = scene
    (pa, pb), _, pose = _history(lvb_ctx, sc)
    first, second = _moved(pose, KEYS, seed=41), _moved(pose, KEYS, seed=43)
    for _ in range(3):
        _to_world(*pa, first)
        _to_world(*pa, second)
    _to_world(*pb, second)
    _same_clouds(pa, pb, sc, KEYS)
    (pa, _), _, pose = _history(lvb_ctx, sc)
    cells = (sc["g"]["cell_size"], sc["s"]["cell_size"])
    before = [[_stored(fa, k, cell) for k in KEYS] for fa, cell in zip(pa, cells)]
    _to_world(*pa, {k: pose[k] for k in KEYS})
    for fa, cell, b in zip(pa, cells, before):
        for k, cloud in zip(KEYS, b):
            assert np.array_equal(_stored(fa, k, cell).view(np.uint32), cloud.view(np.uint32)), k


def _counted(ctx, fn):
    n0, l0 = ctx.sync_count(), ctx.launch_count()
    fn()
    return ctx.launch_count() - l0, ctx.sync_count() - n0


def test_counts(lvb_ctx, scene):
    """One launch and one synchronisation whatever the number of keys; none for no key.  The boxes the call records spare the next
    keyframe call the synchronisation it would spend on clouds stored by map_append."""
    sc = scene
    g, s = sc["g"], sc["s"]
    fa, fs = _pair(lvb_ctx)
    rng = np.random.default_rng(5)
    poses = {}
    for k in range(300):
        poses[k] = _perturbed(g["map_pose"], rng, 1.0, 0.05)
        fa.map_append(k, rng.normal(0, 5, (200 + k, 4)).astype(np.float32), poses[k])
        fs.map_append(k, rng.normal(0, 5, (100 + k, 4)).astype(np.float32), poses[k])
    for n in (1, 10, 300):
        keys = list(range(300 - n, 300))
        assert _counted(lvb_ctx, lambda: backend.map_to_world(fa, fs, keys, np.array([poses[k] for k in keys]))) == (1, 1), n
    assert _counted(lvb_ctx, lambda: backend.map_to_world(fa, fs, [], np.zeros((0, 7)))) == (0, 0)
    assert _counted(lvb_ctx, lambda: backend.map_to_world(fa, None, [3, 4], np.array([poses[3], poses[4]]))) == (1, 1)
    # keyframe calls on clouds stored by map_append: 2 synchronisations without the re-anchoring (test_gpu_map_build_keyframe), 1 after
    (gb, sb), (gc, sc_) = _three_keyframes(lvb_ctx, sc)
    backend.map_to_world(gb, sb, [0, 1, 2], np.array([sc["kfs"][k][0] for k in range(3)]))
    args = ([0, 1, 2], 3, sc["kfs"][2][0], g["frame_pose"], g["scan"], s["scan"])
    assert _counted(lvb_ctx, lambda: new_call(gb, sb, sc, *args))[1] == 1
    assert _counted(lvb_ctx, lambda: new_call(gc, sc_, sc, *args))[1] == 2


def test_nothing_else_moves(lvb_ctx, scene):
    """The handles' current map frames (knn3 against them), the map_append(NULL) scan and the clouds not listed are as they were."""
    sc = scene
    g, s = sc["g"], sc["s"]
    (pa, pb), _, pose = _history(lvb_ctx, sc)
    listed = [0, 3, 10, 12]
    frames = [fa.map_download() for fa in pa]           # the keyframe call's map frames (reading them changes nothing)
    _to_world(*pa, _moved(pose, listed, seed=47))
    p = _perturbed(pose[4], np.random.default_rng(2), 0.1, 0.01)
    for fa, fb in zip(pa, pb):
        fa.map_append(50, None, p)           # the keyframe call's scan, still the one map_append(NULL) stores
        fb.map_append(50, None, p)
    for fa, fb, c, cell, mf in ((pa[0], pb[0], g["scan"], g["cell_size"], frames[0]), (pa[1], pb[1], s["scan"], s["cell_size"], frames[1])):
        assert np.array_equal(fa.map_download().view(np.uint32), mf.view(np.uint32))
        _same_handles(fa, fb, c, pose[4], cell)
        fa.map_append(51, c, p)
        assert np.array_equal(_stored(fa, 50, cell).view(np.uint32), _stored(fa, 51, cell).view(np.uint32))
    _same_clouds(pa, pb, sc, [1, 2, 11])
    # a relocation between the correction and the next keyframe call leaves that call as it is without the relocation
    (pa, pb), _, pose = _history(lvb_ctx, sc)
    moved = _moved(pose, listed, seed=53)
    _to_world(*pa, moved)
    _to_world(*pb, moved)
    old_pose, rel = _candidate(sc, 1)
    reloc_call(*pa, sc, [0, 1, 2], old_pose, rel)
    guess = _perturbed(g["frame_pose"], np.random.default_rng(4), 0.05, 0.002)
    ka, kb = [new_call(fa, fs, sc, [2, 3, 4], 5, pose[4], guess, g["scan"], s["scan"]) for fa, fs in (pa, pb)]
    _same_result(kb[:3], ka[:3])
    assert ka[3] == kb[3]


def test_errors_change_no_state(lvb_ctx, scene):
    sc = scene
    (pa, pb), _, pose = _history(lvb_ctx, sc)
    api = lvb_ctx.api
    pa[0].map_append(60, sc["kfs"][0][1], pose[0])          # resident on the ground handle only
    pb[0].map_append(60, sc["kfs"][0][1], pose[0])
    other = backend.Context(api)
    foreign = backend.FeatureAssociation(other)
    poses = np.array([_perturbed(pose[k], np.random.default_rng(k), 0.2, 0.01) for k in range(3)])

    def raw(g, s, keys, n=None, p=poses):
        k = None if keys is None else (C.c_longlong * max(1, len(keys)))(*keys)
        return api.icp_map_to_world(g, s, k, len(keys) if n is None else n, None if p is None else backend._dp(np.ascontiguousarray(p)))
    ga, sa = pa[0].h, pa[1].h
    l0, n0 = lvb_ctx.launch_count(), lvb_ctx.sync_count()
    assert raw(ga, sa, [0, 1, 42]) == -1                     # not resident
    assert raw(ga, sa, [0, 60, 1]) == -1                     # not resident on the surf handle
    assert raw(ga, sa, [0, 1, 0]) == -1                      # listed twice
    assert raw(ga, sa, None, n=3) == -1
    assert raw(ga, sa, [0, 1, 2], p=None) == -1
    assert raw(ga, sa, [0, 1, 2], n=-1) == -1
    assert raw(None, None, [0, 1, 2]) == -1
    assert raw(ga, ga, [0, 1, 2]) == -1
    assert raw(ga, foreign.h, [0, 1, 2]) == -1               # another context
    assert raw(ga, sa, [], n=0, p=None) == 0                 # nothing to do
    assert (lvb_ctx.launch_count(), lvb_ctx.sync_count()) == (l0, n0)
    _same_clouds(pa, pb, sc, KEYS)
    assert np.array_equal(_stored(pa[0], 60, sc["g"]["cell_size"]).view(np.uint32), _stored(pb[0], 60, sc["g"]["cell_size"]).view(np.uint32))
    # the Python argument checks
    for bad in ((None, None, [0], poses[:1]), (pa[0], pa[0], [0], poses[:1]), (pa[0], pa[1], [0, 1], poses[:1]),
                (pa[0], pa[1], [0, 0], poses[:2]), (pa[0], pa[1], [0], np.zeros((1, 6)))):
        with pytest.raises(ValueError):
            backend.map_to_world(*bad)
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        backend.map_to_world(pa[0], pa[1], [0, 42], poses[:2])
    foreign.close()
    other.close()


def test_beyond_65535_blocks(lvb_ctx):
    """One call over more than 16 M points per side, past 65 535 blocks of the kernel's grid: equal to evict + append."""
    rng = np.random.default_rng(9)
    n = 17_000_000
    cloud = np.empty((n, 4), np.float32)
    cloud[:, :3] = rng.uniform(-100.0, 100.0, (n, 3)).astype(np.float32)
    cloud[:, 3] = rng.uniform(0, 255, n).astype(np.float32)
    ident = np.array([0, 0, 0, 1, 0, 0, 0.0])
    pa, pb = _pair(lvb_ctx), _pair(lvb_ctx)
    for fa, fs in (pa, pb):
        for k in (0, 1):
            fa.map_append(k, cloud, ident)
            fs.map_append(k, cloud, ident)
    moved = _moved({0: ident, 1: ident}, [0, 1], seed=53)
    assert _counted(lvb_ctx, lambda: _to_world(*pa, moved)) == (1, 1)
    _evict_append(*pb, {0: (cloud, cloud), 1: (cloud, cloud)}, moved)
    for fa, fb in zip(pa, pb):
        for k in (0, 1):
            assert np.array_equal(_stored(fa, k, 5.0).view(np.uint32), _stored(fb, k, 5.0).view(np.uint32)), k


def _cloud(f, c):
    np.array([len(c)], np.int32).tofile(f)
    np.ascontiguousarray(np.asarray(c, np.float32)[:, :4]).tofile(f)


def test_shim_to_world_keyframes_equals_append_keyframe(lvb_ctx, scene, tmp_path):
    """include/lvio_b200/association.h: ToWorldKeyframes against AppendKeyframe of every lidar keyframe (tests/cpp/map_to_world_shim.cpp):
    keyframes, a correction from some keyframe on, the re-anchoring over a range with a never-stored lidar keyframe and a frame
    without lidar, further keyframes and a relocation give the same poses and the same integer score."""
    sc = scene
    g, s = sc["g"], sc["s"]
    rng = np.random.default_rng(61)
    guesses = [_perturbed(g["frame_pose"], rng, 0.05, 0.002) for _ in range(6)]
    frames = [(p, 1, cg, cs) for p, cg, cs in sc["kfs"]]
    frames.append((guesses[0], 0, np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32)))     # frame 3: no lidar
    frames += [(q, 1, g["scan"], s["scan"]) for q in guesses[1:]]                                 # frames 4 .. 8
    n_first, start = 5, 1                     # frames 0 .. 4 registered, the correction moves frames 1 .. 5 (5 not stored yet)
    correction = synth.se3_mul(np.array([0, 0, 0, 1, 0.04, -0.03, 0.02]), np.r_[synth.quat_from_rotvec(np.array([[0, 0, 0.004]]))[0], 0, 0, 0])
    keys, old = [0, 1, 2], 1
    with open(tmp_path / "in.bin", "wb") as f:
        np.array([len(frames)], np.int32).tofile(f)
        np.array([synth.W_VISUAL], np.float64).tofile(f)
        np.array([g["n_features_left"]], np.int32).tofile(f)
        for pose, has_lidar, cg, cs in frames:
            np.asarray(pose, np.float64).tofile(f)
            np.array([has_lidar], np.int32).tofile(f)
            _cloud(f, cg)
            _cloud(f, cs)
        np.array([n_first, start], np.int32).tofile(f)
        np.asarray(correction, np.float64).tofile(f)
        np.array([len(keys)], np.int32).tofile(f)
        np.array(keys, np.int64).tofile(f)
        np.array([old], np.int32).tofile(f)
        np.asarray(_perturbed(g["frame_pose"], rng, 0.05, 0.002), np.float64).tofile(f)
        np.array([GT], np.float64).tofile(f)
    exe = str(tmp_path / "map_to_world_shim")
    lib_dir = os.path.join(ROOT, "lvio_fusion_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++14", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "map_to_world_shim.cpp"), "-L" + lib_dir, "-llvio_b200", "-Wl,-rpath," + lib_dir])
    outs = []
    for mode in (0, 1):
        p = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / ("out%d.bin" % mode)), str(mode)], capture_output=True, text=True)
        assert p.returncode == 0, p.stderr
        outs.append(np.fromfile(tmp_path / ("out%d.bin" % mode)))
    K = len(frames)
    a, b = outs
    assert np.max(np.abs(a[:7 * K] - b[:7 * K])) < 1e-11
    assert a[7 * K] == b[7 * K] and a[7 * K] > 0                                  # the integer score
    assert np.max(np.abs(a[7 * K + 1:7 * K + 8] - b[7 * K + 1:7 * K + 8])) < 1e-11  # relative_o_c
    assert a[-1] == 2 * 4 and b[-1] == 1 + 2     # AppendKeyframe: 2 per lidar keyframe; ToWorldKeyframes: 1, + 2 for the new one
    poses = a[:7 * K].reshape(K, 7)
    assert np.max(np.abs(poses[6:] - np.array([q for q, _, _, _ in frames[6:]]))) > 0    # the later keyframes were registered
