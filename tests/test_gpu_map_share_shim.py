"""The shim's mapping, relocator and lidar threads on one FeatureAssociation without a lock (tests/cpp/map_share_shim.cpp): the
Relocator and the lidar callback run on handles of their own, shared from the mapping thread's, and every result equals that of the
same program run under one lock (in whichever order the threads take it) and to that of the Relocator's and the lidar thread's calls
after the mapping pass -- poses to 1e-11 (the linearisation adds its block sums atomically), integer scores and feature counts
exactly."""
import os
import subprocess

import numpy as np
import pytest

from lvio_fusion_b200 import synth
from test_gpu_map_build_keyframe import _frames
from test_gpu_map_optimize import make_scene
from test_gpu_map_relocate import PLACES, _candidate

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M, RELOCS, EXTRACTS = 4, 8, 4


def _cloud(f, c):
    np.array([len(c)], np.int32).tofile(f)
    np.ascontiguousarray(c, np.float32).reshape(-1, 4).tofile(f)


def _frames_out(f, frames):
    np.array([len(frames)], np.int32).tofile(f)
    for pose, cg, cs in frames:
        np.asarray(pose, np.float64).tofile(f)
        _cloud(f, cg)
        _cloud(f, cs)


def test_threads_without_a_lock_equal_the_locked_program(tmp_path):
    sc = make_scene(6000, 5000)
    g, s = sc["g"], sc["s"]
    frames = _frames(sc, M)
    old_pose, rel = _candidate(sc, PLACES["middle"][1])
    with open(tmp_path / "in.bin", "wb") as f:
        _frames_out(f, frames[:3])
        _frames_out(f, frames[3:3 + M])
        np.asarray(old_pose, np.float64).tofile(f)
        np.asarray(rel, np.float64).tofile(f)
        _cloud(f, g["scan"])
        _cloud(f, s["scan"])
        _cloud(f, synth.make_lidar_scan(seed=61))
    exe = str(tmp_path / "map_share_shim")
    lib_dir = os.path.join(ROOT, "lvio_fusion_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++14", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "map_share_shim.cpp"), "-L" + lib_dir, "-llvio_b200", "-Wl,-rpath," + lib_dir])
    out = {}
    for mode in ("free", "locked", "after"):
        p = subprocess.run([exe, mode, str(tmp_path / "in.bin"), str(tmp_path / (mode + ".bin"))], capture_output=True, text=True)
        assert p.returncode == 0, p.stderr
        d = np.fromfile(tmp_path / (mode + ".bin"))
        out[mode] = (d[:7 * M].reshape(M, 7), d[7 * M:7 * M + 8 * RELOCS].reshape(RELOCS, 8), d[7 * M + 8 * RELOCS:].reshape(EXTRACTS, 2))
    pl, rl, cl = out["locked"]
    assert np.all(rl[:, 7] > 0) and cl.min() > 0
    for mode in ("free", "after"):
        pf, rf, cf = out[mode]
        assert np.max(np.abs(pf - pl)) < 1e-11, mode
        assert np.max(np.abs(rf[:, :7] - rl[:, :7])) < 1e-11 and np.array_equal(rf[:, 7], rl[:, 7]), mode
        assert np.array_equal(cf, cl), mode
