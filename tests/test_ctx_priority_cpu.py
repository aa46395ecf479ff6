"""CPU-side checks of the context priority entry points: the symbols are exported and bound; without a device they fail as
lvb_ctx_create does (LVB_ERR_CUDA, "no CPU fallback") and leave `out` NULL; the Python driver raises; a C++14 program that sets its
thread's priority through the shim compiles and reports the failure."""
import ctypes
import os
import subprocess

import pytest

from lvio_fusion_b200 import _capi, backend
from test_capi_cpu import _has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["lvb_ctx_create_with_priority", "lvb_ctx_priority", "lvb_device_priority_range", "lvb_debug_ctx_stream_priorities"]
no_device = pytest.mark.skipif(_has_gpu(), reason="only meaningful on a machine without a GPU")


def test_symbols_are_exported():
    lib = ctypes.CDLL(_capi.LIB_PATH)
    for s in NEW:
        assert s in _capi.EXPORTED_SYMBOLS and hasattr(lib, s), s


@no_device
def test_no_device():
    lvb = _capi.load()
    out = ctypes.c_void_p()
    assert lvb.ctx_create_with_priority(0, -1, ctypes.byref(out)) == -2 and not out.value        # LVB_ERR_CUDA
    assert b"no CPU fallback" in lvb.last_error()
    least, greatest = ctypes.c_int(7), ctypes.c_int(7)
    assert lvb.device_priority_range(0, ctypes.byref(least), ctypes.byref(greatest)) == -2
    assert b"no CPU fallback" in lvb.last_error()
    assert least.value == 7 and greatest.value == 7
    # argument checks come first
    assert lvb.ctx_create_with_priority(0, 0, None) == -1
    assert lvb.device_priority_range(0, None, ctypes.byref(greatest)) == -1
    p = (ctypes.c_int * 2)()
    assert lvb.ctx_priority(None, p) == -1 and lvb.debug_ctx_stream_priorities(None, p) == -1


@no_device
def test_driver_raises_without_a_device():
    lvb = _capi.load()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        backend.Context(lvb, priority=-1)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        backend.priority_range(lvb, 0)


def test_stream_and_priority_together_are_refused():
    with pytest.raises(ValueError, match="not both"):
        backend.Context(_capi.load(), stream=1, priority=0)


SHIM = r'''
#include <cstdio>
#include "lvio_b200/ceres_shim.h"
int main() {
    int least = 0, greatest = 0;
    if (lvb_device_priority_range(0, &least, &greatest) != LVB_OK) std::fprintf(stderr, "range: %s\n", lvb_last_error());
    lvb::Runtime& rt = lvb::Runtime::get();
    if (!rt.set_thread_priority(greatest)) return 4;                 // no context yet: accepted
    if (!rt.ensure()) { std::fprintf(stderr, "no device: %s\n", rt.error.c_str()); return 3; }
    return 0;
}
'''


@no_device
def test_shim_priority_compiles_as_cpp14_and_reports_failure(tmp_path):
    src, exe = tmp_path / "prio.cpp", tmp_path / "prio"
    src.write_text(SHIM)
    lib_dir = os.path.join(ROOT, "lvio_fusion_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++14", "-Wall", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src),
                           "-L" + lib_dir, "-llvio_b200", "-Wl,-rpath," + lib_dir])
    p = subprocess.run([str(exe)], capture_output=True, text=True)
    assert p.returncode == 3 and "no CPU fallback" in p.stderr, (p.returncode, p.stderr)
