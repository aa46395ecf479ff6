"""Resident keyframe clouds shared across threads (lvb_icp_share): a handle pair on another thread's context reads and extracts into
the store of the mapping thread's pair, without a lock around the calls.

Every concurrent case starts its threads behind a barrier and asserts what every interleaving must give: the result of one of the
serial orders of the calls.  The linearisation adds its block sums atomically, so two runs of one registration agree to the last bits
only up to the order of those sums: poses are held to 1e-11 and costs to 1e-12, as in the other keyframe tests; clouds, counts and
termination types exactly."""
import ctypes as C
import threading

import numpy as np
import pytest

from lvio_fusion_b200 import backend, synth
from test_gpu_map_build_keyframe import _frames
from test_gpu_map_extract_keyframe import _capacity, _chain as _extract_chain
from test_gpu_map_optimize import _same_summary, make_scene
from test_gpu_map_optimize_keyframes import _window, chain
from test_gpu_map_relocate import PLACES, _candidate, reloc_call

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scene():
    return make_scene(6000, 5000)


def _pair(ctx):
    return backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)


def _share(pair, ctx):
    return pair[0].share(ctx), pair[1].share(ctx)


def _appended(ctx, sc, poses=None):
    """A pair holding the scene's three keyframes under keys 0, 1, 2 (map_append: the same clouds on every pair, bit for bit)."""
    ga, sa = _pair(ctx)
    for k, (pose, cg, cs) in enumerate(sc["kfs"]):
        ga.map_append(k, cg, pose if poses is None else poses[k])
        sa.map_append(k, cs, pose if poses is None else poses[k])
    return ga, sa


def _same_reloc(a, b):
    (ra, pa, sa, sca, nma), (rb, pb, sb, scb, nmb) = a, b
    assert np.max(np.abs(pa - pb)) < 1e-11 and np.max(np.abs(ra - rb)) < 1e-11
    assert list(nma) == list(nmb)
    for m in range(2):
        _same_summary(sa[m], sb[m])
        assert sa[m].termination_type == sb[m].termination_type
        assert (np.isnan(sca[m]) and np.isnan(scb[m])) or abs(sca[m] - scb[m]) < 1e-9


def _cloud(fa, key, cell, ctx):
    """the world cloud stored under `key`, read through a handle shared on ctx (the handle's own map frame stays as it is)"""
    r = fa.share(ctx)
    r.map_build([key], cell)
    out = r.map_download()
    r.close()
    return out


def _run(*fns):
    """the functions on their own threads, started together behind a barrier; their results, or the exceptions they raised"""
    bar = threading.Barrier(len(fns))
    out = [None] * len(fns)

    def body(i, fn):
        bar.wait()
        try:
            out[i] = fn()
        except Exception as e:          # noqa: BLE001 -- the caller checks what each thread may raise
            out[i] = e.with_traceback(None)          # no reference cycle through this frame
    ts = [threading.Thread(target=body, args=(i, fn)) for i, fn in enumerate(fns)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out


def _ok(x):
    if isinstance(x, Exception):
        raise x
    return x


@pytest.mark.parametrize("place", sorted(PLACES))
def test_relocation_on_a_shared_pair(lvb, lvb_ctx, scene, place):
    sc = scene
    g, s = sc["g"], sc["s"]
    keys, old = PLACES[place]
    run = _window(_frames(sc, 0), 0, 3)
    owner, same = _pair(lvb_ctx), _pair(lvb_ctx)          # `same`: the same history without any relocation
    chain(*owner, sc, run)
    chain(*same, sc, run)
    old_pose, rel = _candidate(sc, old)
    want = reloc_call(*owner, sc, keys, old_pose, rel)
    ctx2 = backend.Context(lvb)
    shared = _share(owner, ctx2)
    got = _run(lambda: reloc_call(*shared, sc, keys, old_pose, rel))[0]
    _same_reloc(_ok(got), want)
    assert min(want[4]) > 0
    # the owner's map_append(NULL) scan (still the last keyframe's), map frames, 3-NN and stored clouds are those of `same`
    pose = np.array([0, 0, 0, 1, 0.5, 0, 0.0])
    for fa, fs, c, cell in ((owner[0], same[0], g["scan"], g["cell_size"]), (owner[1], same[1], s["scan"], s["cell_size"])):
        fa.map_append(99, None, pose)
        fs.map_append(99, None, pose)
        assert np.array_equal(fa.map_download().view(np.uint32), fs.map_download().view(np.uint32))
        ia, da = fa.knn3(c, g["frame_pose"], 0.9 * cell * cell)
        ib, db = fs.knn3(c, g["frame_pose"], 0.9 * cell * cell)
        assert np.array_equal(ia, ib) and np.array_equal(da.view(np.uint32), db.view(np.uint32))
        for k in (0, 1, 2, 99):
            assert np.array_equal(_cloud(fa, k, cell, ctx2).view(np.uint32), _cloud(fs, k, cell, ctx2).view(np.uint32)), k


def test_extraction_on_a_shared_pair_is_consumed_by_key_on_the_owner(lvb, lvb_ctx):
    sc = make_scene(200, 200)
    poses = [np.array([0, 0, np.sin(0.01 * k), np.cos(0.01 * k), 0.4 * k, 0.05 * k, 0.0]) for k in range(2)]
    scans = [synth.make_lidar_scan(seed=51 + k) for k in range(2)]
    kfs = [(5, [], poses[0], None, None), (6, [5], poses[1], None, None)]
    ref = _pair(lvb_ctx)
    lf = backend.LidarFeatures(lvb_ctx)
    want = [lf.extract_into(*ref, 5 + k, scans[k]) for k in range(2)]
    want_chain = _extract_chain(*ref, sc, kfs)
    owner = _pair(lvb_ctx)
    ctx2 = backend.Context(lvb)
    shared = _share(owner, ctx2)
    lf2 = backend.LidarFeatures(ctx2)
    got = _run(lambda: [lf2.extract_into(*shared, 5 + k, scans[k]) for k in range(2)])[0]
    for a, b in zip(_ok(got), want):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert _capacity(owner[0], 5)[2] == len(want[0][0]) and _capacity(shared[1], 6)[2] == len(want[1][1])
    got_chain = _extract_chain(*owner, sc, kfs)
    for a, b in zip(got_chain, want_chain):
        assert np.max(np.abs(a[0] - b[0])) < 1e-11 and list(a[4]) == list(b[4])
    for fa, fr, cell in ((owner[0], ref[0], sc["g"]["cell_size"]), (owner[1], ref[1], sc["s"]["cell_size"])):
        for key in (5, 6):
            assert np.array_equal(_cloud(fa, key, cell, ctx2).view(np.uint32), _cloud(fr, key, cell, ctx2).view(np.uint32)), key
            assert _capacity(fa, key)[2] == -1


def test_relocation_loop_concurrent_with_a_keyframe_chain(lvb, lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    frames = _frames(sc, 6)
    kfs = [(k, mk, sc["kfs"][2][0], p, cg, cs) for k, mk, _, p, cg, cs in _window(frames, 3, 6)]
    cands = [(PLACES[p][0],) + _candidate(sc, PLACES[p][1], seed=20 + i) for i, p in enumerate(sorted(PLACES) * 3)][:8]
    owner, ref = _appended(lvb_ctx, sc), _appended(lvb_ctx, sc)
    want_r = [reloc_call(*owner, sc, keys, op, rel) for keys, op, rel in cands]
    want_c = chain(*ref, sc, kfs)
    ctx2 = backend.Context(lvb)
    shared = _share(owner, ctx2)
    got_c, got_r = _run(lambda: chain(*owner, sc, kfs), lambda: [reloc_call(*shared, sc, keys, op, rel) for keys, op, rel in cands])
    for a, b in zip(_ok(got_r), want_r):
        _same_reloc(a, b)
    for k, (a, b) in enumerate(zip(_ok(got_c), want_c)):
        assert np.max(np.abs(a[0] - b[0])) < 1e-11 and np.max(np.abs(a[1] - b[1])) < 1e-11, k
        assert list(a[4]) == list(b[4]), k
        for m in range(2):
            _same_summary(a[3][m], b[3][m])
    for fa, fr, cell in ((owner[0], ref[0], g["cell_size"]), (owner[1], ref[1], s["cell_size"])):
        for key in range(9):
            assert np.array_equal(_cloud(fa, key, cell, ctx2).view(np.uint32), _cloud(fr, key, cell, ctx2).view(np.uint32)), key


def test_re_anchoring_during_a_relocation(lvb, lvb_ctx, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    keys, old = PLACES["middle"]
    old_pose, rel = _candidate(sc, old)
    moved = [p.copy() for p, _, _ in sc["kfs"]]
    for p in moved:
        p[4] += 0.3
    owner, after = _appended(lvb_ctx, sc), _appended(lvb_ctx, sc, moved)
    want = (reloc_call(*owner, sc, keys, old_pose, rel), reloc_call(*after, sc, keys, old_pose, rel))
    ctx2 = backend.Context(lvb)
    shared = _share(owner, ctx2)
    tw, got = _run(lambda: backend.map_to_world(*owner, [0, 1, 2], moved), lambda: reloc_call(*shared, sc, keys, old_pose, rel))
    _ok(tw)
    got = _ok(got)
    matches = []
    for w in want:
        try:
            _same_reloc(got, w)
            matches.append(True)
        except AssertionError:
            matches.append(False)
    assert any(matches), "the relocation is neither the one before the correction nor the one after it"
    for fa, fr, cell, m in ((owner[0], after[0], g["cell_size"], 1), (owner[1], after[1], s["cell_size"], 2)):
        for k in range(3):
            assert np.array_equal(_cloud(fa, k, cell, ctx2).view(np.uint32), _cloud(fr, k, cell, ctx2).view(np.uint32)), k
            n = len(sc["kfs"][k][m])
            assert _capacity(fa, k) == (n, n, -1)


def test_eviction_during_a_relocation(lvb, lvb_ctx, scene):
    sc = scene
    keys, old = PLACES["middle"]
    old_pose, rel = _candidate(sc, old)
    owner = _appended(lvb_ctx, sc)
    want = reloc_call(*owner, sc, keys, old_pose, rel)
    ctx2 = backend.Context(lvb)
    shared = _share(owner, ctx2)
    ev, got = _run(lambda: (owner[0].map_evict(1), owner[1].map_evict(1)), lambda: reloc_call(*shared, sc, keys, old_pose, rel))
    _ok(ev)
    if isinstance(got, RuntimeError):
        assert "failed (-1)" in str(got) and "key 1 is not resident" in str(got), got
    else:
        _same_reloc(_ok(got), want)
    assert _capacity(shared[0], 1) == (-1, -1, -1)


def test_lifetime_and_errors(lvb, lvb_ctx, scene):
    sc = scene
    keys, old = PLACES["end"]
    old_pose, rel = _candidate(sc, old)
    ctx1, ctx2, ctx3 = backend.Context(lvb), backend.Context(lvb), backend.Context(lvb)
    owner = _appended(ctx1, sc)
    want = reloc_call(*owner, sc, keys, old_pose, rel)
    shared = _share(owner, ctx2)
    for fa in owner:
        fa.close()
    ctx1.close()
    _same_reloc(reloc_call(*shared, sc, keys, old_pose, rel), want)
    # a share of a share is on the same store
    again = _share(shared, ctx3)
    again[0].map_append(7, sc["kfs"][0][1], sc["kfs"][0][0])
    assert _capacity(shared[0], 7)[0] == len(sc["kfs"][0][1])
    shared[0].map_evict(7)
    assert _capacity(again[0], 7) == (-1, -1, -1)
    _same_reloc(reloc_call(*again, sc, keys, old_pose, rel), want)
    # NULL arguments fail before anything is created
    h = C.c_void_p()
    assert lvb.icp_share(None, shared[0].h, C.byref(h)) == -1 and not h.value
    assert lvb.icp_share(ctx2.h, None, C.byref(h)) == -1 and not h.value
    assert lvb.icp_share(ctx2.h, shared[0].h, None) == -1


def _costs(ctx, pair, sc, kfs, cand, moved):
    out = []
    for fn in (lambda: chain(*pair, sc, kfs), lambda: backend.map_to_world(*pair, [0, 1, 2], moved),
               lambda: reloc_call(*pair, sc, cand[0], cand[1], cand[2])):
        s0, l0 = ctx.sync_count(), ctx.launch_count()
        fn()
        out.append((ctx.sync_count() - s0, ctx.launch_count() - l0))
    return out


def test_no_added_cost(lvb, lvb_ctx, scene):
    """a chain, a re-anchoring and a relocation on an unshared store: one synchronisation each (the chain records the boxes the
    relocation needs), one kernel for the re-anchoring; on a store another handle shares, the owner's calls cost the same"""
    sc = scene
    frames = _frames(sc, 2)
    kfs = [(k, mk, sc["kfs"][2][0], p, cg, cs) for k, mk, _, p, cg, cs in _window(frames, 3, 2)]
    moved = [p.copy() for p, _, _ in sc["kfs"]]
    for p in moved:
        p[5] += 0.2
    cand = (PLACES["middle"][0],) + _candidate(sc, PLACES["middle"][1])
    alone = _appended(lvb_ctx, sc)
    reloc_call(*alone, sc, *cand)                  # the boxes of the appended clouds are computed here, not in the counted calls
    base = _costs(lvb_ctx, alone, sc, kfs, cand, moved)
    assert [x[0] for x in base] == [1, 1, 1] and base[1][1] == 1, base
    owner = _appended(lvb_ctx, sc)
    reloc_call(*owner, sc, *cand)
    ctx2 = backend.Context(lvb)
    shared = _share(owner, ctx2)
    assert _costs(lvb_ctx, owner, sc, kfs, cand, moved) == base
    assert shared[0].h
