"""The bundle-adjustment structure planner (lvio_fusion_b200/csrc/ba_plan.h) on the CPU: the ordering, CSR, Schur grouping, envelope
and solver decisions behind the GPU parity suite, checked as invariants on the problems that suite solves.  The planner header is
compiled with g++ into tests/cpp/test_ba_plan.cpp; no CUDA is involved."""
import functools
import os
import subprocess

import numpy as np
import pytest

import shim_util
from lvio_fusion_b200 import synth
from lvio_fusion_b200.backend import IMU, POSE_GRAPH, POSE_ONLY, POSE_PRIOR, TWO_CAMERA, TWO_FRAME

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_TRACK = 16
SCALARS = {"dimc", "n_pose_free", "n_vec3_free", "n_rho_free", "n_schur_warps", "schur_cols_max", "band", "true_band", "dense", "srow", "soff", "nS",
           "solvable", "tc_ok", "tree_levels", "wide", "chol_smem", "max_cta_smem"}


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("plan") / "test_ba_plan")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-o", out, os.path.join(ROOT, "tests", "cpp", "test_ba_plan.cpp")])
    return out


def _with_factor(d, kind, consts, idx):
    d = dict(d)
    d["factors"] = dict(d["factors"])
    d["factors"][kind] = (consts, idx)
    return d


# the problems of test_gpu_ba.py (constant values do not shape the plan: zero records stand in for the priors' measurements)
@functools.lru_cache(maxsize=None)
def _problem(name):
    if name.startswith("window_priors"):
        d = synth.make_ba_problem(5, 2000, with_imu=True, seed=synth.SEED)
        d = _with_factor(d, POSE_GRAPH, np.zeros((1, 8)), np.array([[0, 1]], dtype=np.int32))
        d = _with_factor(d, POSE_PRIOR, np.zeros((1, 9)), np.array([[2]], dtype=np.int32))
        if name.endswith("const"):
            rc = np.zeros(len(d["rho"]), dtype=np.uint8); rc[::7] = 1
            vc = np.zeros(len(d["vec3"]), dtype=np.uint8); vc[1] = 1
            d["pose_const"], d["vec3_const"], d["rho_const"] = np.array([1, 0, 0, 0, 0], dtype=np.uint8), vc, rc
        return d
    if name == "window_10":
        return synth.make_ba_problem(10, 4000, with_imu=True, seed=7)
    if name == "fullba":
        return synth.make_fullba_problem(6, 600, seed=23)
    if name == "banded_imu":
        return synth.make_ba_problem(80, 3000, with_imu=True, seed=11)
    if name == "banded_visual":
        d = synth.make_ba_problem(150, 3000, with_imu=False, seed=11)
        return _with_factor(d, POSE_PRIOR, np.zeros((1, 9)), np.zeros((1, 1), dtype=np.int32))
    if name == "loop_closure":
        d = synth.make_ba_problem(80, 3000, with_imu=True, seed=13)
        return _with_factor(d, POSE_GRAPH, np.zeros((1, 8)), np.array([[0, 79]], dtype=np.int32))
    raise KeyError(name)


def _run(exe, tmp_path, d):
    src, out = tmp_path / "problem.bin", tmp_path / "plan.bin"
    shim_util.dump_ba(src, d, 0)
    if any(k in d for k in ("pose_const", "vec3_const", "rho_const")):
        with open(src, "ab") as f:
            for key, n in (("pose_const", len(d["poses"])), ("vec3_const", len(d["vec3"])), ("rho_const", len(d["rho"]))):
                np.asarray(d.get(key, np.zeros(n)), dtype=np.uint8).tofile(f)
    p = subprocess.run([exe, "problem", str(src), str(out)], capture_output=True, text=True)
    return p, out


def _plan(exe, tmp_path, d):
    p, out = _run(exe, tmp_path, d)
    assert p.returncode == 0, p.stdout + p.stderr
    phases = [l[len("phase "):] for l in p.stdout.splitlines() if l.startswith("phase ")]
    assert phases == ["validate", "block order", "factor sort + pad", "landmark CSR", "schur groups", "envelope"]
    raw, plan, pos = out.read_bytes(), {}, 0
    while pos < len(raw):
        n = int(np.frombuffer(raw, np.int32, 1, pos)[0]); pos += 4
        name = raw[pos:pos + n].decode(); pos += n
        cnt = int(np.frombuffer(raw, np.int64, 1, pos)[0]); pos += 8
        plan[name] = np.frombuffer(raw, np.int64, cnt, pos).copy(); pos += 8 * cnt
    return {k: int(v[0]) if k in SCALARS else v for k, v in plan.items()}


def _idx(d, kind, width):
    f = d["factors"].get(kind)
    return np.zeros((0, width), dtype=np.int64) if f is None else np.asarray(f[1], dtype=np.int64).reshape(-1, width)


def _const(d, key, n):
    return np.asarray(d.get(key, np.zeros(n)), dtype=bool)


def _check_unknowns(d, p):
    pc, vc = _const(d, "pose_const", len(d["poses"])), _const(d, "vec3_const", len(d["vec3"]))
    rc = _const(d, "rho_const", len(d["rho"]))
    npf, nvf = int((~pc).sum()), int((~vc).sum())
    assert p["dimc"] == 6 * npf + 3 * nvf and p["n_rho_free"] == int((~rc).sum())
    assert np.all(p["pose_off"][pc] == -1) and np.all(p["vec3_off"][vc] == -1)
    assert np.all(p["rho_slot"][rc] == -1) and np.array_equal(p["rho_slot"][~rc], np.arange(int((~rc).sum())))
    canon = p["canon"]
    assert np.array_equal(np.sort(canon), np.arange(p["dimc"]))
    # poses first (in pose order), then the vec3 blocks
    for slot, i in enumerate(np.nonzero(~pc)[0]):
        assert np.array_equal(canon[p["pose_off"][i] + np.arange(6)], 6 * slot + np.arange(6))
    for slot, i in enumerate(np.nonzero(~vc)[0]):
        assert np.array_equal(canon[p["vec3_off"][i] + np.arange(3)], 6 * npf + 3 * slot + np.arange(3))
    # keyframe by keyframe: free poses in pose order
    assert np.all(np.diff(p["pose_off"][~pc]) > 0)


def _check_factor_order(d, p):
    n_poses = len(d["poses"])
    tf, po = _idx(d, TWO_FRAME, 3), _idx(d, POSE_ONLY, 1)
    keys = {TWO_FRAME: tf[:, 1] * n_poses + tf[:, 2], POSE_ONLY: po[:, 0]}
    for k in range(6):
        ordk = p["order%d" % k]
        n = len(d["factors"][k][1]) if k in d["factors"] else 0
        assert len(ordk) == p["nd"][k]
        real = ordk[ordk >= 0]
        assert np.array_equal(np.sort(real), np.arange(n))                    # every caller block exactly once
        if k not in keys or not p["solvable"]:
            assert np.array_equal(ordk, np.arange(n))
            continue
        src = np.where(ordk >= 0, ordk, -1 - ordk)                           # padding: an encoded copy of a block of the same key
        kk = keys[k][src]
        assert np.all(np.diff(kk) >= 0)                                      # sorted by key ...
        rk = keys[k][real]
        assert np.all((np.diff(rk) > 0) | (np.diff(real) > 0))               # ... stably
        starts = np.concatenate([[0], np.nonzero(np.diff(kk))[0] + 1])
        if p["dense"]:
            assert len(ordk) % 32 == 0 and np.all(starts % 32 == 0)          # every key run padded to a multiple of 32
            run_real = np.add.reduceat((ordk >= 0).astype(np.int64), starts)
            assert np.all(np.diff(np.concatenate([starts, [len(ordk)]])) - run_real < 32)
        else:
            assert np.all(ordk >= 0)


def _pose_sets(d, p):
    """The sorted set of free pose offsets of every free landmark (its TwoFrame observations)."""
    rc = _const(d, "rho_const", len(d["rho"]))
    tf = _idx(d, TWO_FRAME, 3)
    sets = {l: set() for l in np.nonzero(~rc)[0]}
    for l, a, b in tf:
        if l in sets:
            for q in (a, b):
                if p["pose_off"][q] >= 0:
                    sets[l].add(int(p["pose_off"][q]))
    return {l: sorted(s) for l, s in sets.items()}


def _check_csr(d, p):
    nr = len(d["rho"])
    tf, tc = _idx(d, TWO_FRAME, 3), _idx(d, TWO_CAMERA, 1)
    o0 = p["order0"]
    pos = np.nonzero(o0 >= 0)[0]
    want = sorted(zip(tf[o0[pos], 0].tolist(), pos.tolist())) + sorted(zip(tc[:, 0].tolist(), (-np.arange(len(tc)) - 1).tolist()))
    ls = p["lm_start"]
    assert len(ls) == nr + 1 and ls[0] == 0 and ls[-1] == len(tf) + len(tc)
    got = list(zip(np.repeat(np.arange(nr), np.diff(ls)).tolist(), p["lm_fac"][:ls[-1]].tolist()))
    assert sorted(got) == sorted(want)                                       # every observation exactly once, under its landmark


def _check_schur_groups(d, p):
    sets = _pose_sets(d, p)
    nw = p["n_schur_warps"]
    sw_lm = p["sw_lm"][:32 * nw].reshape(nw, 32) if nw else np.zeros((0, 32), dtype=np.int64)
    members = sw_lm[sw_lm >= 0]
    assert np.array_equal(np.sort(members), np.array(sorted(sets), dtype=np.int64))      # every free landmark in exactly one warp
    grp = np.repeat(p["sw_group"][:nw], 32).reshape(nw, 32)[sw_lm >= 0]
    group_of = dict(zip(members.tolist(), grp.tolist()))
    goff = p["grp_off"].reshape(-1, MAX_TRACK)
    assert p["schur_cols_max"] == (max(6 * len(s) + 1 for s in sets.values()) if sets else 0)
    for l, s in sets.items():
        g = group_of[l]
        assert p["grp_ns"][g] == len(s)
        assert goff[g, :len(s)].tolist() == s and np.all(goff[g, len(s):] == -1)
    tf = _idx(d, TWO_FRAME, 3)
    o0, n_tf = p["order0"], p["nd"][0]
    slots = p["tf_slot"].reshape(2, -1)[:, :n_tf]
    for i in range(n_tf):
        l = tf[o0[i], 0] if o0[i] >= 0 else -1
        for side in (0, 1):
            if l < 0 or l not in sets or p["pose_off"][tf[o0[i], 1 + side]] < 0:
                assert slots[side, i] == -1
            else:
                assert goff[group_of[l], slots[side, i]] == p["pose_off"][tf[o0[i], 1 + side]]


def _check_envelope(d, p):
    """Every coupling the assembly can create lies inside the envelope (and inside the band of banded storage)."""
    width = np.zeros(p["dimc"], dtype=np.int64)
    width[p["pose_off"][p["pose_off"] >= 0]] = 6
    width[p["vec3_off"][p["vec3_off"] >= 0]] = 3
    pairs = []
    for s in _pose_sets(d, p).values():
        pairs += [(a, b) for i, a in enumerate(s) for b in s[:i]]
    po = p["pose_off"]
    for kind in (TWO_FRAME, POSE_GRAPH):
        ix = _idx(d, kind, 3 if kind == TWO_FRAME else 2)
        cols = ix[:, 1:3] if kind == TWO_FRAME else ix
        pairs += list(zip(po[cols[:, 0]].tolist(), po[cols[:, 1]].tolist()))
    for row in _idx(d, IMU, 8):
        offs = [-1 if v < 0 else int(po[v] if b in (0, 4) else p["vec3_off"][v]) for b, v in enumerate(row)]
        pairs += [(offs[a], offs[b]) for a in range(8) for b in range(a)]
    pairs = np.array([(max(a, b), min(a, b)) for a, b in pairs if a >= 0 and b >= 0 and a != b], dtype=np.int64).reshape(-1, 2)
    assert len(pairs) > 0
    hi, lo = pairs[:, 0], pairs[:, 1]
    rmax, cmin = p["chol_rmax"], p["chol_cmin"]
    last_row = hi + width[hi] - 1
    for k in range(6):
        c = np.minimum(lo + k, lo + width[lo] - 1)
        assert np.all(rmax[c // 32] >= last_row)
        r = np.minimum(hi + k, last_row)
        assert np.all(cmin[r // 32] <= lo)
        if not p["dense"]:
            assert np.all(r - lo <= p["band"])


PROBLEMS = ["window_priors", "window_priors_const", "window_10", "fullba", "banded_imu", "banded_visual", "loop_closure"]


@pytest.mark.parametrize("name", PROBLEMS)
def test_plan_invariants(exe, tmp_path, name):
    d = _problem(name)
    p = _plan(exe, tmp_path, d)
    assert p["solvable"]
    _check_unknowns(d, p)
    _check_factor_order(d, p)
    _check_csr(d, p)
    _check_schur_groups(d, p)
    _check_envelope(d, p)
    if name.startswith(("window", "fullba")):
        # window-sized: dense storage, the single-CTA envelope kernel, tensor-core maps over the free poses
        assert p["dense"] and p["srow"] == p["dimc"] and p["soff"] == 0
        assert p["tree_levels"] == 0 and not p["wide"] and p["chol_smem"] <= p["max_cta_smem"]
        assert p["tc_ok"] and np.array_equal(np.sort(p["tc_off"][:6 * p["n_pose_free"]]), np.sort(p["pose_off"][p["pose_off"] >= 0][:, None] + np.arange(6), axis=None))
    else:
        assert not p["dense"] and p["dimc"] > 736 and p["srow"] == p["soff"] == p["band"] and not p["tc_ok"]
        assert p["band"] >= min(p["true_band"] + 31, p["dimc"] - 1)          # room for 32-column steps from any first unknown
    if name == "loop_closure":
        # the loop's coupling makes the envelope as wide as the system: no tree, no shared-memory panel
        assert p["true_band"] >= p["dimc"] - 15 and p["tree_levels"] == 0 and p["wide"] and p["chol_smem"] > p["max_cta_smem"]


def _band(exe, n, band, no_tree):
    levels, wide, smem, limit = map(int, subprocess.run([exe, "band", str(n), str(band), str(int(no_tree))], capture_output=True, text=True, check=True).stdout.split())
    return levels, bool(wide), smem, limit


# the shapes of test_gpu_band_solver.py (band = true half bandwidth + 31), with its expected tree / no-tree answer
@pytest.mark.parametrize("n,true_band,expect_tree", [(150, 40, False), (700, 45, True), (1200, 59, True), (2500, 33, True), (4000, 75, True), (9000, 50, True),
                                                     (900, 23, True), (1500, 10, True), (600, 31, True), (2000, 5, True)])
def test_reduced_solver_tree_choice(exe, n, true_band, expect_tree):
    levels, wide, smem, limit = _band(exe, n, true_band + 31, False)
    assert (levels > 0) == expect_tree and not wide and smem <= limit
    assert _band(exe, n, true_band + 31, True)[:2] == (0, False)


@pytest.mark.parametrize("n,true_band", [(1500, 1200), (2100, 2099), (1000, 930)])
def test_wide_envelopes_plan_the_multi_grid_solver(exe, n, true_band):
    for no_tree in (False, True):
        levels, wide, smem, limit = _band(exe, n, true_band + 31, no_tree)
        assert levels == 0 and wide and smem > limit


def test_out_of_range_index_is_rejected(exe, tmp_path):
    d = synth.make_ba_problem(3, 20, with_imu=False, seed=1)
    d["factors"][TWO_FRAME][1][0, 1] = 99
    p, _ = _run(exe, tmp_path, d)
    assert p.returncode == 3 and p.stdout.strip() == "error -1 factor kind 0 block 0: index 99 out of range [0,3)"


def test_landmark_seen_from_too_many_keyframes_is_unsupported(exe, tmp_path):
    d = synth.make_ba_problem(20, 200, with_imu=False, seed=5)
    c, ix = d["factors"][TWO_FRAME]
    extra = np.array([[0, 0, k] for k in range(1, 20)], dtype=np.int32)        # landmark 0 seen from all 20 keyframes
    d = _with_factor(d, TWO_FRAME, np.concatenate([c, np.repeat(c[:1], len(extra), 0)]), np.concatenate([ix, extra]))
    p, _ = _run(exe, tmp_path, d)
    assert p.returncode == 3 and p.stdout.strip() == "error -5 landmark 0 is observed from more than %d keyframes" % MAX_TRACK
