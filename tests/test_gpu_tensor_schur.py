"""schur_mode = 1: the landmark marginalisation S -= W^T D W on the tensor cores (wgmma, bf16 x3 split operands, FP32
accumulation in registers over 256-landmark slices, FP64 across slices), checked against the FP64 CUDA-core path that
carries the parity claims.  Stated tolerance: 2e-5 of max|S| on the reduced system (2^-23 per product plus FP32
accumulation), 1e-5 relative on the converged cost, 1e-5 on poses -- the gradient side (rhs) stays FP64, so the
fixed point of the LM iteration is unchanged and only the step direction is perturbed."""
import numpy as np
import pytest

from lvio_fusion_b200 import backend, synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n_kf,n_lm", [(10, 1000), (20, 3000)])
def test_reduced_system_close_to_fp64(lvb_ctx, n_kf, n_lm):
    d = synth.make_ba_problem(n_kf, n_lm, with_imu=True, seed=41)
    p = backend.Problem.from_dict(lvb_ctx, d)
    S0, b0, c0 = p.reduced_system(1e4)
    p.set_schur_mode(1)
    S1, b1, c1 = p.reduced_system(1e4)
    assert c0 == pytest.approx(c1, rel=1e-12)
    assert np.max(np.abs(b1 - b0)) < 1e-9 * np.abs(b0).max()          # the right-hand side stays FP64
    err = np.max(np.abs(S1 - S0)) / np.abs(S0).max()
    assert 0 < err < 2e-5, err                                         # > 0: the tensor path really ran


def test_solve_converges_to_the_same_point(lvb_ctx):
    d = synth.make_ba_problem(10, 2000, with_imu=True, seed=42)
    p0, p1 = backend.Problem.from_dict(lvb_ctx, d), backend.Problem.from_dict(lvb_ctx, d)
    s0 = p0.solve(max_num_iterations=50)
    s1 = p1.solve(max_num_iterations=50, schur_mode=1)
    assert s1.termination_type == 0
    assert abs(s1.final_cost - s0.final_cost) < 1e-5 * s0.final_cost
    assert np.max(np.abs(p1.poses() - p0.poses())) < 1e-5


def test_falls_back_when_too_many_poses(lvb_ctx):
    d = synth.make_ba_problem(24, 600, with_imu=False, seed=43)      # 144 pose dimensions > 128
    d["factors"] = dict(d["factors"])
    d["factors"][5] = (np.concatenate([d["poses"][0], [100.0, 0.0]])[None], np.zeros((1, 1), dtype=np.int32))
    p = backend.Problem.from_dict(lvb_ctx, d)
    S0, _, _ = p.reduced_system(1e4)
    p.set_schur_mode(1)
    S1, _, _ = p.reduced_system(1e4)
    assert np.max(np.abs(S1 - S0)) < 1e-9 * np.abs(S0).max()           # silently stayed on the FP64 path
