"""CPU-side checks of lvb_icp_share: the symbol is exported and bound; without a device no context, hence no handle to share, can be
made (LVB_ERR_CUDA: there is no CPU fallback), and the call stops at its argument checks; the shim headers with the per-thread shared
handles compile as C++14."""
import ctypes
import os
import subprocess

import pytest

from lvio_fusion_b200 import _capi
from test_capi_cpu import _has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbol_is_exported():
    assert "lvb_icp_share" in _capi.EXPORTED_SYMBOLS
    assert hasattr(ctypes.CDLL(_capi.LIB_PATH), "lvb_icp_share")


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a machine without a GPU")
def test_no_device():
    lvb = _capi.load()
    ctx = ctypes.c_void_p()
    assert lvb.ctx_create(0, None, ctypes.byref(ctx)) == -2          # LVB_ERR_CUDA: no context, hence no handle to share
    out = ctypes.c_void_p()
    assert lvb.icp_share(None, None, ctypes.byref(out)) == -1 and not out.value
    assert lvb.icp_share(None, None, None) == -1


def test_shim_headers_compile_as_cpp14(tmp_path):
    src = tmp_path / "assoc.cpp"
    src.write_text('#include "lvio_b200/association.h"\n'
                   'struct P { float x, y, z, intensity; };\n'
                   'int main() { lvio_fusion::FeatureAssociation a; (void)a; return 0; }\n')
    p = subprocess.run(["g++", "-std=c++14", "-fsyntax-only", "-Wall", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
