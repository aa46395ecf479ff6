"""plan_reduced_solver's choice of the resident single-CTA solve (the whole envelope of S in shared memory) on the CPU: the windows
take it, the banded and loop-closure problems keep the separator tree / wide solver, and the band shapes of
test_gpu_resident_solver.py fall on the side of the shared-memory limit that test expects.  The planner header is compiled with g++
into tests/cpp/test_ba_plan_resident.cpp; no CUDA is involved."""
import os
import subprocess

import pytest

import shim_util
from lvio_fusion_b200 import synth
from test_ba_plan import _problem

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("plan") / "test_ba_plan_resident")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", out, os.path.join(ROOT, "tests", "cpp", "test_ba_plan_resident.cpp")])
    return out


def _plan(exe, tmp_path, d):
    src = tmp_path / "problem.bin"
    shim_util.dump_ba(src, d, 0)
    p = subprocess.run([exe, "problem", str(src)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    head, rmax = p.stdout.splitlines()
    n, resident, smem, limit, levels, wide = map(int, head.split())
    return dict(n=n, resident=bool(resident), smem=smem, limit=limit, levels=levels, wide=bool(wide), rmax=[int(r) for r in rmax.split()])


def _resident_smem(rmax, n):
    """The layout of chol_resident_columns: (Dt, invd) x 2, partial sums, rhs, block columns of 34-double rows."""
    cols = sum((rmax[kb // 32] - kb + 1) * 34 for kb in range(0, n, 32))
    return (2 * (32 * 34 + 32) + 256 + ((n + 1) & ~1) + cols) * 8


@pytest.mark.parametrize("name", ["window_10", "window_20", "window_priors", "fullba"])
def test_windows_solve_resident(exe, tmp_path, name):
    d = synth.make_ba_problem(20, 8000, with_imu=True, seed=synth.SEED) if name == "window_20" else _problem(name)
    p = _plan(exe, tmp_path, d)
    n, rmax = p["n"], p["rmax"]
    assert p["resident"] and p["levels"] == 0 and not p["wide"]
    assert p["smem"] == _resident_smem(rmax, n) <= p["limit"]
    # the envelope rows the layout relies on: non-decreasing per step, never above the step's own last column
    assert len(rmax) == (n + 31) // 32
    assert rmax == sorted(rmax) and all(rmax[s] >= min(n, 32 * s + 32) - 1 for s in range(len(rmax)))


@pytest.mark.parametrize("name", ["banded_imu", "banded_visual", "loop_closure"])
def test_banded_and_loop_closure_keep_their_solver(exe, tmp_path, name):
    p = _plan(exe, tmp_path, _problem(name))
    assert not p["resident"]
    if name == "loop_closure":
        assert p["wide"] and p["levels"] == 0
    else:
        assert p["levels"] > 0 and not p["wide"]


def _band(exe, n, band, no_tree):
    r, smem, limit = map(int, subprocess.run([exe, "band", str(n), str(band), str(int(no_tree))], capture_output=True, text=True, check=True).stdout.split())
    return bool(r), smem, limit


# (n, true half bandwidth, resident) with band = true + 31: the single-CTA sizes of test_gpu_band_solver.py and the two shapes at
# the edge of the shared-memory limit (300 unknowns: a true band of 59 is the widest that fits, 60 the narrowest that does not)
SHAPES = [(1, 0, True), (20, 19, True), (32, 31, True), (33, 32, True), (47, 46, True), (64, 5, True), (95, 20, True), (129, 128, True),
          (150, 149, True), (160, 64, True), (300, 299, False), (300, 91, False), (736, 100, False), (300, 59, True), (300, 60, False)]


@pytest.mark.parametrize("n,true_band,resident", SHAPES)
def test_single_cta_storage_choice(exe, n, true_band, resident):
    r, smem, limit = _band(exe, n, max(31, true_band + 31), True)
    assert r == resident and (smem <= limit) == resident


def test_resident_boundary_is_tight(exe):
    _, fits, limit = _band(exe, 300, 59 + 31, True)
    _, over, _ = _band(exe, 300, 60 + 31, True)
    assert fits <= limit < over


def test_tree_takes_precedence(exe):
    # a banded system the separator tree splits is not solved by one CTA even when its envelope would fit
    assert not _band(exe, 700, 45 + 31, False)[0]
