"""The single-CTA reduced-system solver alone: random SPD (banded) systems against numpy, with the SM-clock phase split
(warp 0's diagonal-block factorisations / the all-warp panel + head block / warp 0's wait, backward pass).
With an argument DIR, also writes each shape's solution to DIR/x_<n>_<band>.npy, to compare two builds bit for bit."""
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lvio_fusion_b200 import _capi, backend
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from test_gpu_band_solver import _band_spd, _pack

lvb = _capi.load(); ctx = backend.Context(lvb)
out_dir = sys.argv[1] if len(sys.argv) > 1 else None
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
worst = 0.0
for n, tb in ((150, 149), (300, 299), (300, 91), (47, 46), (95, 20), (129, 128), (160, 64), (33, 32), (32, 31), (20, 19), (1, 0), (64, 5), (736, 100),
              (150, 40), (300, 59), (300, 60)):
    rng = np.random.default_rng(n * 7 + tb)
    s = _band_spd(n, tb, rng); b = rng.normal(size=n)
    want = np.linalg.solve(s, b)
    band = max(31, tb + 31)
    packed = np.ascontiguousarray(_pack(s, band)); x = np.zeros(n); lv = C.c_int(-1)
    out = (C.c_longlong * 8)()
    lvb.check(lvb.debug_cholesky_clocks(out, 1), "clocks")
    lvb.check(lvb.debug_band_solve(ctx.h, n, band, packed.ctypes.data_as(_capi.c_double_p), b.ctypes.data_as(_capi.c_double_p), x.ctypes.data_as(_capi.c_double_p), 0, C.byref(lv)), "solve")
    lvb.check(lvb.debug_cholesky_clocks(out, 1), "clocks")
    err = np.max(np.abs(x - want)) / np.max(np.abs(want)); res = np.max(np.abs(s @ x - b)) / np.max(np.abs(b))
    worst = max(worst, err)
    if out_dir:
        np.save(os.path.join(out_dir, "x_%d_%d.npy" % (n, tb)), x)
    print("n=%4d band=%4d %s err %.1e resid %.1e   load %6d  factorisation %6d panel+head %6d wait %6d   backward %6d  total %6d cycles %s"
          % (n, tb, "resident" if out[7] else "global  ", err, res, out[6], out[0], out[1], out[2], out[3], out[4], "" if err < 1e-8 else "  <-- WRONG"))
print("worst", worst)
