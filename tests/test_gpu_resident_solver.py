"""The two storages of the single-CTA reduced-system solve: the envelope resident in shared memory (chosen whenever it fits) and S in
global memory.  Each shape checks which kernel ran, through the call counters of lvb_debug_cholesky_clocks, and solves against numpy
at the tolerances of test_gpu_band_solver.py."""
import ctypes as C

import numpy as np
import pytest

from lvio_fusion_b200 import _capi
from test_gpu_band_solver import _band_spd, _pack

pytestmark = pytest.mark.gpu


def _solve(lvb_ctx, s, b, band):
    """Single-CTA solve (no tree); returns (rc, x, resident) where resident says which storage the kernel used."""
    api = lvb_ctx.api
    n = len(b)
    packed = np.ascontiguousarray(_pack(s, band)); x = np.zeros(n); lv = C.c_int(-1)
    clocks = (C.c_longlong * 8)()
    api.check(api.debug_cholesky_clocks(clocks, 1), "clocks")
    rc = api.debug_band_solve(lvb_ctx.h, n, band, packed.ctypes.data_as(_capi.c_double_p), b.ctypes.data_as(_capi.c_double_p),
                              x.ctypes.data_as(_capi.c_double_p), 0, C.byref(lv))
    api.check(api.debug_cholesky_clocks(clocks, 1), "clocks")
    assert lv.value == 0 and clocks[5] == 1, (lv.value, clocks[5])
    assert clocks[7] in (0, 1)
    return rc, x, bool(clocks[7])


# (n, true half bandwidth, resident): the single-CTA sizes of test_gpu_band_solver.py split by the shared-memory rule, and the two
# shapes at its edge (300 unknowns: a true band of 59 is the widest envelope that fits, 60 the narrowest that does not)
@pytest.mark.parametrize("n,true_band,resident", [(150, 149, True), (160, 64, True), (33, 32, True), (300, 299, False), (300, 91, False), (736, 100, False),
                                                  (300, 59, True), (300, 60, False)])
def test_storage_choice_and_solution(lvb_ctx, n, true_band, resident):
    rng = np.random.default_rng(n * 7 + true_band)
    s = _band_spd(n, true_band, rng)
    b = rng.normal(size=n)
    want = np.linalg.solve(s, b)
    rc, x, used = _solve(lvb_ctx, s, b, max(31, true_band + 31))
    lvb_ctx.api.check(rc, "debug_band_solve")
    assert used == resident
    err = np.max(np.abs(x - want)) / np.max(np.abs(want))
    resid = np.max(np.abs(s @ x - b)) / np.max(np.abs(b))
    assert err < 1e-9 and resid < 1e-10, (err, resid)


@pytest.mark.parametrize("n,pivot,resident", [(150, 101, True), (300, 201, False)])
def test_non_positive_pivot_is_reported_by_both_storages(lvb_ctx, n, pivot, resident):
    rng = np.random.default_rng(3)
    s = _band_spd(n, n - 1, rng)
    s[pivot, pivot] = -5.0
    rc, _, used = _solve(lvb_ctx, s, np.ones(n), n - 1 + 31)
    assert used == resident
    assert rc != 0 and b"pivot" in lvb_ctx.api.last_error()
