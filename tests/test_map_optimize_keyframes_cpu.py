"""CPU-side checks of lvb_icp_map_optimize_keyframes: the symbol is exported, the Python driver's argument checks raise before any
library call, and the host restatement of its SE3 arithmetic (lvio_fusion_b200/se3.py) agrees with the C++ shim's
(include/lvio_b200/se3.h), which replays PoseGraph::ForwardUpdate with the transforms the call returns."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from lvio_fusion_b200 import _capi, backend, se3, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbol_is_exported():
    assert "lvb_icp_map_optimize_keyframes" in _capi.EXPORTED_SYMBOLS
    assert hasattr(ctypes.CDLL(_capi.LIB_PATH), "lvb_icp_map_optimize_keyframes")


class _NoDevice:
    """An api table whose every library call fails the test: the checks must raise first."""
    def __getattr__(self, name):
        raise AssertionError("library call %s before the argument checks" % name)


class _Handle:
    def __init__(self):
        self.api, self.h = _NoDevice(), None


def _kf(key, map_keys, pose=None, n=10, width=4):
    pts = np.zeros((n, width), np.float32)
    return (key, map_keys, np.array([0, 0, 0, 1, 0, 0, 0.0]), np.array([0, 0, 0, 1, 0, 0, 0.0]) if pose is None else pose, pts, pts)


@pytest.mark.parametrize("case", ["one_handle", "same_handle", "four_keys", "twice", "own_key", "pose_size", "strides", "weights",
                                  "prior_weights"])
def test_argument_checks_raise_before_any_library_call(case):
    g, s = _Handle(), _Handle()
    kfs = [_kf(1, []), _kf(2, [1])]
    if case == "one_handle":
        s = None
    elif case == "same_handle":
        s = g
    elif case == "four_keys":
        kfs[1] = _kf(2, [-3, -2, -1, 1])
    elif case == "twice":
        kfs[1] = _kf(1, [])
    elif case == "own_key":
        kfs[1] = _kf(2, [1, 2])
    elif case == "pose_size":
        kfs[1] = _kf(2, [1], pose=np.zeros(6))
    elif case == "strides":
        kfs[1] = _kf(2, [1], width=8)
    weight, prior = (1, 1), 1.0
    if case == "weights":
        weight = [(1, 1)] * 3                        # one pair per keyframe: 2 keyframes
    elif case == "prior_weights":
        prior = [1.0, 2.0, 3.0]
    with pytest.raises(ValueError):
        backend.build_and_optimize_keyframes(g, s, kfs, (1.0, 1.0), 0.05, weight, prior, (0, 0.1), (1, 1), options=_capi.SolveOptions())


_DRIVER = r"""
#include <cstdio>
#include "lvio_b200/se3.h"
int main() {
    double a[7], b[7], c[7], d[7];
    while (std::fread(a, 8, 7, stdin) == 7 && std::fread(b, 8, 7, stdin) == 7) {
        lvb::se3::mul(a, b, c); lvb::se3::inv(a, d);
        std::fwrite(c, 8, 7, stdout); std::fwrite(d, 8, 7, stdout);
    }
    return 0;
}
"""


def test_host_restatement_matches_the_shim(tmp_path):
    src, exe = tmp_path / "se3.cpp", str(tmp_path / "se3")
    src.write_text(_DRIVER)
    subprocess.check_call(["g++", "-O2", "-std=c++14", "-I" + os.path.join(ROOT, "include"), "-o", exe, str(src)])
    rng = np.random.default_rng(11)
    poses = []
    for _ in range(400):
        q = synth.quat_from_rotvec(rng.normal(0, 1.0, 3)[None])[0] * rng.uniform(0.999, 1.001)     # not quite unit, as poses drift
        poses.append(np.concatenate([q, rng.normal(0, 100.0, 3)]))
    pairs = np.array([np.concatenate([poses[i], poses[(i * 7 + 3) % len(poses)]]) for i in range(len(poses))])
    out = np.frombuffer(subprocess.run([exe], input=pairs.tobytes(), capture_output=True, check=True).stdout, np.float64).reshape(-1, 2, 7)
    for (ab, (c, d)) in zip(pairs, out):
        a, b = ab[:7], ab[7:]
        scale = max(1.0, np.max(np.abs(a[4:])), np.max(np.abs(b[4:])))
        assert np.max(np.abs(se3.mul(a, b) - c)) <= 1e-15 * scale
        assert np.max(np.abs(se3.inv(a) - d)) <= 1e-15 * scale
    # the chain: forward_update composes in order, and the transform undoes the incoming pose
    Ts = [se3.transform(poses[i + 1], poses[i]) for i in range(3)]
    p = se3.forward_update(Ts, poses[0])
    want = poses[0]
    for T in Ts:
        want = se3.mul(T, want)
    assert np.array_equal(p, want)
    a, b = (np.concatenate([x[:4] / np.linalg.norm(x[:4]), x[4:]]) for x in (poses[4], poses[5]))       # unit quaternions
    assert np.max(np.abs(se3.mul(se3.transform(b, a), a) - b)) < 1e-12
