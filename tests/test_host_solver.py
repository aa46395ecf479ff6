"""The small host-side LM behind the ceres-shaped shim for the reference's off-path solves (SURVEY 8(f).4): AutoDiff
functors, quaternion parameterisation, constant / variable / bounded blocks.  CPU only; the pose-graph case is compared with
the oracle's LM (same published Ceres trust-region semantics) on the equivalent factor set."""
import os
import subprocess

import numpy as np
import pytest

from lvio_fusion_b200 import backend, synth
from lvio_fusion_b200.backend import POSE_GRAPH, POSE_PRIOR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    lib_dir = os.path.join(ROOT, "lvio_fusion_b200", "csrc")
    out = str(tmp_path_factory.mktemp("host") / "test_host_solver")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-o", out, os.path.join(ROOT, "tests", "cpp", "test_host_solver.cpp"),
                           "-L" + lib_dir, "-llvio_b200", "-Wl,-rpath," + lib_dir])
    return out


def test_autodiff_and_rotation_templates(exe):
    out = subprocess.run([exe, "autodiff"], capture_output=True, text=True, check=True).stdout.split()
    assert float(out[1]) < 1e-7                        # AutoDiffCostFunction vs central differences
    assert float(out[3]) < 1e-14 and float(out[4]) < 1e-14
    assert abs(float(out[6]) - np.linalg.norm([0.3, -1.2, 2.0])) < 1e-12     # rotation preserves length
    # NumericDiffCostFunction: forward quotient (step ~1e-6 |x|, >= 1.5e-8) and central quotient against AutoDiff, same residuals
    assert float(out[8]) < 1e-4 and float(out[9]) < 1e-6 and float(out[10]) == 0.0


def test_navsat_shaped_two_stage_and_bounded_solve(exe):
    lines = subprocess.run([exe, "navsat", "5"], capture_output=True, text=True, check=True).stdout.splitlines()
    s1, s2, b = (l.split() for l in lines)
    assert s1[0] == "stage1" and float(s1[4]) == 0.0 and s1[-1] == "0"          # x stayed constant in stage 1
    assert float(s1[8]) < float(s1[6])                                           # cost decreased
    assert abs(float(s2[2]) - 0.7) < 1e-4 and abs(float(s2[4]) - 12.5) < 5e-3 and abs(float(s2[6]) + 4.25) < 5e-3
    assert abs(float(b[2]) - 13.5) < 1e-12                                       # clamped at the lower bound x_true + 1


@pytest.mark.parametrize("huber", [0, 1])
def test_pose_graph_matches_oracle_lm(exe, orc, orc_ctx, tmp_path, huber):
    rng = np.random.default_rng(17)
    n = 7
    truth = synth.Trajectory(n).poses()
    meas = truth.copy()
    meas[:, 4:] += rng.normal(0, 0.02, (n, 3)); meas[:, :4] += rng.normal(0, 0.002, (n, 4)); meas[:, :4] /= np.linalg.norm(meas[:, :4], axis=1, keepdims=True)
    init = truth.copy()
    init[:, 4:] += rng.normal(0, 0.3, (n, 3)); init[:, :4] += rng.normal(0, 0.02, (n, 4)); init[:, :4] /= np.linalg.norm(init[:, :4], axis=1, keepdims=True)
    gps = truth[:, 4:] + rng.normal(0, 0.05, (n, 3))
    gps[3] += [3.0, -2.0, 0.5]                                                   # one outlier for the Huber case
    w_edge, v_edge, w_gps = 10.0, 2.0, 3.0
    with open(tmp_path / "in.bin", "wb") as f:
        np.array([n, huber, 40], dtype=np.int32).tofile(f)
        init.astype(np.float64).tofile(f); meas.astype(np.float64).tofile(f); gps.astype(np.float64).tofile(f)
        np.array([w_edge, v_edge, w_gps], dtype=np.float64).tofile(f)
    p = subprocess.run([exe, "posegraph", str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert p.returncode == 0 and "host LM" in p.stderr
    res = np.fromfile(tmp_path / "out.bin", dtype=np.float64)
    head, poses = res[:4], res[4:].reshape(n, 7)
    # the same problem for the oracle: PoseGraphError edges + PoseError priors with v = 0 about identity-rotation origins
    e = np.zeros((n - 1, 8))
    inv, rel, six = np.zeros(7), np.zeros(7), np.zeros(6)
    for i in range(n - 1):
        orc.se3_inverse(backend._dp(meas[i].copy()), backend._dp(inv)); orc.se3_compose(backend._dp(inv), backend._dp(meas[i + 1].copy()), backend._dp(rel))
        orc.se3_to_rpyxyz(backend._dp(rel), backend._dp(six))
        e[i, :6] = six; e[i, 6] = w_edge; e[i, 7] = v_edge
    prior = np.zeros((n, 9)); prior[:, 3] = 1.0; prior[:, 4:7] = gps; prior[:, 7] = w_gps; prior[:, 8] = 0.0
    d = {"cameras": synth.kitti_cameras(), "poses": init.copy(), "vec3": np.zeros((0, 3)), "rho": np.zeros(0),
         "factors": {POSE_GRAPH: (e, np.stack([np.arange(n - 1), np.arange(1, n)], 1).astype(np.int32)), POSE_PRIOR: (prior, np.arange(n, dtype=np.int32)[:, None])},
         "loss": {POSE_PRIOR: 0.5} if huber else {}}
    po = backend.Problem.from_dict(orc_ctx, d)
    so = po.solve(max_num_iterations=40)
    assert abs(head[0] - so.initial_cost) < 1e-9 * so.initial_cost
    assert abs(head[1] - so.final_cost) < 1e-9 * so.final_cost
    assert int(head[3]) == so.termination_type
    assert np.max(np.abs(poses - po.poses())) < 1e-8
    # and exactly the same after a fixed small number of iterations
    with open(tmp_path / "in.bin", "r+b") as f:
        f.seek(8); np.array([6], dtype=np.int32).tofile(f)
    subprocess.run([exe, "posegraph", str(tmp_path / "in.bin"), str(tmp_path / "out6.bin")], capture_output=True, check=True)
    res6 = np.fromfile(tmp_path / "out6.bin", dtype=np.float64)
    po6 = backend.Problem.from_dict(orc_ctx, d)
    so6 = po6.solve(max_num_iterations=6)
    assert abs(res6[1] - so6.final_cost) < 1e-10 * so6.final_cost
    assert np.max(np.abs(res6[4:].reshape(n, 7) - po6.poses())) < 1e-9
    assert head[1] < 0.05 * head[0]


def test_shim_pose_factors_reproduce_the_reference_functors(exe, tmp_path):
    """PoseGraphError / PoseError as the shim evaluates them on the host (factors.h + ceres_autodiff.h) against the fixture
    produced by the reference's own pose_error.hpp (tests/golden/ref_factors.npz)."""
    ref = np.load(os.path.join(ROOT, "tests", "golden", "ref_factors.npz"))
    n = len(ref["pg"])
    with open(tmp_path / "cases.bin", "wb") as f:
        np.array([n], dtype=np.int32).tofile(f)
        ref["pg"].astype(np.float64).tofile(f); ref["pe"].astype(np.float64).tofile(f)
    subprocess.run([exe, "refcases", str(tmp_path / "cases.bin"), str(tmp_path / "out.bin")], check=True)
    o = np.fromfile(tmp_path / "out.bin", dtype=np.float64)
    pg = o[:n * 90].reshape(n, 90); pe = o[n * 90:].reshape(n, 48)
    assert np.max(np.abs(pg[:, :6] - ref["pg_r"])) < 1e-12 * max(1.0, np.abs(ref["pg_r"]).max())
    assert np.max(np.abs(pg[:, 6:].reshape(n, 6, 14) - ref["pg_J"])) < 1e-11 * max(1.0, np.abs(ref["pg_J"]).max())
    assert np.max(np.abs(pe[:, :6] - ref["pe_r"])) < 1e-12 * max(1.0, np.abs(ref["pe_r"]).max())
    assert np.max(np.abs(pe[:, 6:].reshape(n, 6, 7) - ref["pe_J"])) < 1e-11 * max(1.0, np.abs(ref["pe_J"]).max())


def test_reference_navsat_functors_drop_onto_the_shim():
    """The reference's navsat_error.hpp / base.hpp, compiled where they lie, against the PRODUCT shim (<ceres/ceres.h> resolves
    to include/lvio_b200 through tests/cpp/compat_product): NavsatInitError::Create + the two-stage solve of navsat.cpp:104-129.
    The binary is oracle/_ref/ref_navsat_functors, made by `make -C oracle ref` with the other reference drop-ins."""
    out = os.path.join(ROOT, "oracle", "_ref", "ref_navsat_functors")
    if not os.path.exists(out):
        pytest.skip("oracle/_ref/ref_navsat_functors is built only where the reference sources are present")
    p = subprocess.run([out], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "host LM" in p.stdout
