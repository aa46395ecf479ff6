"""Context stream priorities (lvb_ctx_create_with_priority): the priority both of a context's streams actually get, and that a priority
changes only when work is dispatched -- the same results, launches and synchronisations as a default-priority context.

The linearisations add their block sums atomically, so two runs of one solve agree to the last bits only up to the order of those
sums: the window solve is held to the tolerances of two launch paths of one device solve (test_gpu_lm_schedule), the keyframe calls
and relocations to those of the other keyframe tests (poses 1e-11, costs 1e-12); iterations, termination types, clouds, feature
counts and extracted features exactly."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from lvio_fusion_b200 import backend, synth
from test_gpu_lm_schedule import _assert_same_path, _solve
from test_gpu_map_build_keyframe import _frames
from test_gpu_map_extract_keyframe import _counted
from test_gpu_map_optimize import _same_summary, make_scene
from test_gpu_map_optimize_keyframes import _window, chain
from test_gpu_map_relocate import PLACES, _candidate, reloc_call
from test_gpu_map_share import _appended, _cloud, _ok, _pair, _run, _same_reloc, _share
from test_gpu_map_share_shim import _cloud as _cloud_out, _frames_out

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def scene():
    return make_scene(6000, 5000)


@pytest.fixture(scope="module")
def prange(lvb):
    return backend.priority_range(lvb, 0)


def _stream_priorities(lvb, ctx):
    p = (ctypes.c_int * 2)()
    lvb.check(lvb.debug_ctx_stream_priorities(ctx.h, p), "debug_ctx_stream_priorities")
    return p[0], p[1]


def test_priority_range(prange):
    least, greatest = prange
    assert greatest <= least
    assert greatest <= 0 <= least


def test_effective_priority(lvb, prange):
    import torch
    least, greatest = prange
    top = backend.Context(lvb, priority=greatest)
    assert _stream_priorities(lvb, top) == (greatest, greatest) and top.priority == greatest
    for asked, clamped in ((greatest - 100, greatest), (least + 100, least)):
        c = backend.Context(lvb, priority=asked)
        assert _stream_priorities(lvb, c) == (clamped, clamped) and c.priority == clamped, asked
    plain = backend.Context(lvb)
    assert _stream_priorities(lvb, plain) == (0, 0) and plain.priority == 0
    # a caller's stream: the context's side stream takes its priority
    with torch.cuda.device(0):
        s = torch.cuda.Stream(priority=-1)
    assert s.priority < 0
    on_torch = backend.Context(lvb, stream=s.cuda_stream)
    assert _stream_priorities(lvb, on_torch) == (s.priority, s.priority) and on_torch.priority == s.priority
    with pytest.raises(ValueError):
        backend.Context(lvb, stream=s.cuda_stream, priority=greatest)


def _contexts(lvb, prange):
    return backend.Context(lvb), backend.Context(lvb, priority=prange[1])


def test_window_solve_is_the_same_at_the_greatest_priority(lvb, prange):
    """Two solves of one configs[1] window on each context: the second replays the pass graph."""
    d = synth.make_ba_problem(10, 4000, with_imu=True, seed=synth.SEED)
    out = []
    for ctx in _contexts(lvb, prange):
        p = backend.Problem.from_dict(ctx, d)
        out.append([_counted(ctx, lambda: _solve(p, d, max_num_iterations=10)) for _ in range(2)])
    (a1, a2), (b1, b2) = out
    for (x, cx), (y, cy), what in ((a1, b1, "first"), (a2, b2, "second")):
        _assert_same_path(y, x, what=what)
        assert cx == cy, (what, cx, cy)


def test_keyframe_chain_relocation_and_extraction_are_the_same(lvb, prange, scene):
    sc = scene
    frames = _frames(sc, 3)
    kfs = [(k, mk, sc["kfs"][2][0], p, cg, cs) for k, mk, _, p, cg, cs in _window(frames, 3, 3)]
    keys, old = PLACES["middle"]
    old_pose, rel = _candidate(sc, old)
    sweep = synth.make_lidar_scan(seed=71)
    out = []
    for ctx in _contexts(lvb, prange):
        pair = _appended(ctx, sc)
        lf = backend.LidarFeatures(ctx)
        out.append((_counted(ctx, lambda: chain(*pair, sc, kfs)),
                    _counted(ctx, lambda: reloc_call(*pair, sc, keys, old_pose, rel)),
                    _counted(ctx, lambda: lf.extract_into(*pair, 500, sweep))))
    ((ca, nca), (ra, nra), (ea, nea)), ((cb, ncb), (rb, nrb), (eb, neb)) = out
    assert nca == ncb and nra == nrb and nea == neb, (nca, ncb, nra, nrb, nea, neb)
    for k, (a, b) in enumerate(zip(cb, ca)):
        assert np.max(np.abs(a[0] - b[0])) < 1e-11 and np.max(np.abs(a[1] - b[1])) < 1e-11, k
        assert list(a[4]) == list(b[4]), k
        for m in range(2):
            _same_summary(a[3][m], b[3][m])
    _same_reloc(rb, ra)
    assert len(ea[0]) > 0 and np.array_equal(ea[0].view(np.uint32), eb[0].view(np.uint32))
    assert np.array_equal(ea[1].view(np.uint32), eb[1].view(np.uint32))


def test_three_priorities_over_one_store_give_the_serial_results(lvb, prange, scene):
    """The keyframe chain on the owner's context at the greatest priority, a relocation loop on a shared pair at the default, and
    extractions on a third context one step lower than the chain's, all at once: each gives what it gives alone."""
    least, greatest = prange
    sc = scene
    g, s = sc["g"], sc["s"]
    frames = _frames(sc, 6)
    kfs = [(k, mk, sc["kfs"][2][0], p, cg, cs) for k, mk, _, p, cg, cs in _window(frames, 3, 6)]
    cands = [(PLACES[p][0],) + _candidate(sc, PLACES[p][1], seed=20 + i) for i, p in enumerate(sorted(PLACES) * 3)][:8]
    sweeps = [synth.make_lidar_scan(seed=81 + e) for e in range(3)]
    ref_ctx = backend.Context(lvb)
    lf_ref = backend.LidarFeatures(ref_ctx)
    want_e = [lf_ref.extract_into(*_pair(ref_ctx), 1000 + e, sw) for e, sw in enumerate(sweeps)]
    owner_ref, ref = _appended(ref_ctx, sc), _appended(ref_ctx, sc)
    want_r = [reloc_call(*owner_ref, sc, k, op, rel) for k, op, rel in cands]
    want_c = chain(*ref, sc, kfs)

    hi, mid, lo = backend.Context(lvb, priority=greatest), backend.Context(lvb, priority=min(greatest + 1, least)), backend.Context(lvb)
    owner = _appended(hi, sc)
    reloc_pair, lidar_pair = _share(owner, lo), _share(owner, mid)
    lf = backend.LidarFeatures(mid)
    got_c, got_r, got_e = _run(lambda: chain(*owner, sc, kfs),
                               lambda: [reloc_call(*reloc_pair, sc, k, op, rel) for k, op, rel in cands],
                               lambda: [lf.extract_into(*lidar_pair, 1000 + e, sw) for e, sw in enumerate(sweeps)])
    for a, b in zip(_ok(got_r), want_r):
        _same_reloc(a, b)
    for k, (a, b) in enumerate(zip(_ok(got_c), want_c)):
        assert np.max(np.abs(a[0] - b[0])) < 1e-11 and np.max(np.abs(a[1] - b[1])) < 1e-11, k
        assert list(a[4]) == list(b[4]), k
        for m in range(2):
            _same_summary(a[3][m], b[3][m])
    for a, b in zip(_ok(got_e), want_e):
        assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
    for fa, fr, cell in ((owner[0], ref[0], g["cell_size"]), (owner[1], ref[1], s["cell_size"])):
        for key in range(9):
            assert np.array_equal(_cloud(fa, key, cell, lo).view(np.uint32), _cloud(fr, key, cell, lo).view(np.uint32)), key


M, RELOCS, EXTRACTS = 4, 8, 4


def test_shim_threads_at_their_priorities_equal_the_locked_program(tmp_path, scene):
    sc = scene
    g, s = sc["g"], sc["s"]
    frames = _frames(sc, M)
    old_pose, rel = _candidate(sc, PLACES["middle"][1])
    with open(tmp_path / "in.bin", "wb") as f:
        _frames_out(f, frames[:3])
        _frames_out(f, frames[3:3 + M])
        np.asarray(old_pose, np.float64).tofile(f)
        np.asarray(rel, np.float64).tofile(f)
        _cloud_out(f, g["scan"])
        _cloud_out(f, s["scan"])
        _cloud_out(f, synth.make_lidar_scan(seed=61))
    exe = str(tmp_path / "ctx_priority_shim")
    lib_dir = os.path.join(ROOT, "lvio_fusion_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++14", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "ctx_priority_shim.cpp"), "-L" + lib_dir, "-llvio_b200", "-Wl,-rpath," + lib_dir])
    out = {}
    for mode in ("priority", "locked"):
        p = subprocess.run([exe, mode, str(tmp_path / "in.bin"), str(tmp_path / (mode + ".bin"))], capture_output=True, text=True)
        assert p.returncode == 0, p.stderr
        d = np.fromfile(tmp_path / (mode + ".bin"))
        out[mode] = (d[:7 * M].reshape(M, 7), d[7 * M:7 * M + 8 * RELOCS].reshape(RELOCS, 8), d[7 * M + 8 * RELOCS:].reshape(EXTRACTS, 2))
    (pp, rp, cp), (pl, rl, cl) = out["priority"], out["locked"]
    assert np.all(rl[:, 7] > 0) and cl.min() > 0
    assert np.max(np.abs(pp - pl)) < 1e-11
    assert np.max(np.abs(rp[:, :7] - rl[:, :7])) < 1e-11 and np.array_equal(rp[:, 7], rl[:, 7])
    assert np.array_equal(cp, cl)
