"""CPU-side checks of lvb_icp_map_extract_keyframe and of registering by key: the symbol is exported; without a device no context,
hence no handle, can be made (LVB_ERR_CUDA: there is no CPU fallback to extract into), and the call stops at its argument checks when
given no handles; the Python drivers' argument checks raise before any library call."""
import ctypes

import numpy as np
import pytest

from lvio_fusion_b200 import _capi, backend
from test_capi_cpu import _has_gpu


def test_symbol_is_exported():
    assert "lvb_icp_map_extract_keyframe" in _capi.EXPORTED_SYMBOLS
    assert hasattr(ctypes.CDLL(_capi.LIB_PATH), "lvb_icp_map_extract_keyframe")


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a machine without a GPU")
def test_no_device():
    lvb = _capi.load()
    h = ctypes.c_void_p()
    assert lvb.ctx_create(0, None, ctypes.byref(h)) == -2           # LVB_ERR_CUDA: no context, hence no handle to extract into
    cfg = _capi.LidarConfig()
    lvb.lidar_default_config(ctypes.byref(cfg))
    n = np.zeros(2, np.int32)
    ip = _capi.c_int32_p
    # without handles the call stops at its argument checks
    assert lvb.icp_map_extract_keyframe(None, None, ctypes.byref(cfg), 1, None, 0, 16, n[:1].ctypes.data_as(ip), n[1:].ctypes.data_as(ip),
                                        None, None) == -1


class _NoDevice:
    """An api table whose every library call fails the test: the checks must raise first."""
    def __getattr__(self, name):
        raise AssertionError("library call %s before the argument checks" % name)


class _Ctx:
    def __init__(self):
        self.api, self.h = _NoDevice(), None


class _Handle:
    def __init__(self, ctx):
        self.ctx, self.api, self.h = ctx, ctx.api, None


def _pipe(ctx):
    lf = backend.LidarFeatures.__new__(backend.LidarFeatures)
    lf.ctx, lf.cfg = ctx, _capi.LidarConfig()
    return lf


@pytest.mark.parametrize("case", ["no_surf", "same_handle", "other_context"])
def test_extract_into_checks(case):
    ctx = _Ctx()
    g, s = _Handle(ctx), _Handle(ctx)
    if case == "no_surf":
        s = None
    elif case == "same_handle":
        s = g
    elif case == "other_context":
        s = _Handle(_Ctx())
    with pytest.raises(ValueError):
        _pipe(ctx).extract_into(g, s, 1, np.zeros((10, 4), np.float32))


@pytest.mark.parametrize("side", [0, 1])
def test_by_key_is_both_sides_or_neither(side):
    ctx = _Ctx()
    g, s = _Handle(ctx), _Handle(ctx)
    pose = np.array([0, 0, 0, 1, 0, 0, 0.0])
    cloud = np.zeros((10, 4), np.float32)
    clouds = [None, None]
    clouds[side] = cloud
    with pytest.raises(ValueError):
        backend.build_and_optimize_keyframe(g, s, [], (1, 1), 0.05, 1, pose, pose, clouds[0], clouds[1], (1, 1), 1.0, (0, 0.1), (1, 1))
    with pytest.raises(ValueError):
        backend.build_and_optimize_keyframes(g, s, [(1, [], pose, pose, clouds[0], clouds[1])], (1, 1), 0.05, (1, 1), 1.0, (0, 0.1), (1, 1))
