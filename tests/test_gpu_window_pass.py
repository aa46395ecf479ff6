"""The single-GPU window pass in six kernels (ba.cu, launch_linearize_and_reduce / launch_step):

    ba_linearize_all_kernel<0> | ba_schur_kernel | ba_cholesky_kernel | ba_update_kernel | ba_linearize_all_kernel<1>
    | ba_post_wide_kernel

S and rhs reach the Schur kernel as zeros and are assembled there (lower(Hpp), damping, -gc) by adds that commute with the
elimination's atomics; its last CTA runs the LM pre-check.  The cost kernel clears S and rhs for the next pass and its last CTA
decides the step; a grid-wide kernel copies an accepted candidate and clears the accumulators.  Both last-CTA counters must come back to zero after every launch, including passes that return on `done`.
Banded and sharded problems keep their own sequences."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from lvio_fusion_b200 import backend, synth
from test_gpu_lm_schedule import _assert_same_path, _assert_same_solve, _params, _scenario, _start

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WINDOW_PASS = ["ba_linearize_all_kernel<0>", "ba_schur_kernel", "ba_cholesky_kernel", "ba_update_kernel", "ba_linearize_all_kernel<1>",
               "ba_post_wide_kernel"]


def _window():
    return synth.make_ba_problem(10, 4000, with_imu=True, seed=synth.SEED)       # bench.py's configs[1] window


def _timed_kernels(lvb, run):
    """Kernel names of run() in launch order (per-kernel timing: direct launches), without the once-per-solve clear."""
    lvb.check(lvb.debug_timing(1), "debug_timing")
    buf = ctypes.create_string_buffer(1 << 22)
    try:
        run()
    finally:
        lvb.check(lvb.debug_timing_report(buf, len(buf)), "debug_timing_report")
    names = [ln.rsplit(" ", 1)[0].strip("()") for ln in buf.value.decode().splitlines()]
    return [n for n in names if n not in ("begin", "ba_zero_kernel")]


def _rel(a, b):
    return np.max(np.abs(a - b)) / np.abs(b).max()


def test_window_pass_is_six_kernels(lvb, lvb_ctx):
    d = _window()
    p = backend.Problem.from_dict(lvb_ctx, d)
    names = _timed_kernels(lvb, lambda: p.solve(max_num_iterations=4))
    assert len(names) >= len(WINDOW_PASS) and len(names) % len(WINDOW_PASS) == 0, names
    assert names == WINDOW_PASS * (len(names) // len(WINDOW_PASS)), names


def test_banded_problem_keeps_its_sequence(lvb, lvb_ctx):
    d = synth.make_ba_problem(80, 3000, with_imu=True, seed=11)       # camera system above the dense cap: banded storage
    p = backend.Problem.from_dict(lvb_ctx, d)
    assert p.dims()[0] > 736
    names = _timed_kernels(lvb, lambda: p.solve(max_num_iterations=2))
    passes = names.count("ba_update_kernel")
    assert passes >= 1
    for k in ("ba_linearize_kernel<0>", "ba_linearize_other_kernel<0>", "ba_build_S_kernel<1>", "ba_schur_kernel",
              "ba_linearize_kernel<1>", "ba_linearize_other_kernel<1>", "ba_post_kernel"):
        assert names.count(k) == passes, (k, names)


TWO_RANK_SCRIPT = textwrap.dedent("""
    import ctypes, os, sys
    sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
    import torch, torch.distributed as dist
    from lvio_fusion_b200 import _capi, backend, synth
    import test_gpu_window_pass as t
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    lvb = _capi.load()
    ctx = backend.Context(lvb, device=rank)
    uid = ctypes.create_string_buffer(128)
    if rank == 0:
        lvb.check(lvb.comm_unique_id(uid), "comm_unique_id")
    box = [uid.raw]
    dist.broadcast_object_list(box, src=0)
    ctx.comm_init(rank, world, box[0])
    d = synth.shard_ba_problem(synth.make_ba_problem(8, 1500, with_imu=True, seed=31), rank, world)
    p = backend.Problem.from_dict(ctx, d)
    names = t._timed_kernels(lvb, lambda: p.solve(max_num_iterations=3))
    passes = names.count("ba_update_kernel")
    assert passes >= 1, names
    for k in ("ba_build_S_kernel<0>", "ba_schur_kernel", "ba_post_kernel"):
        assert names.count(k) == passes, (k, names)
    assert "ba_build_S_kernel<1>" not in names, names
    dist.barrier()
    print("SEQUENCE OK", rank)
    dist.destroy_process_group()
""")


def test_two_rank_problem_keeps_its_sequence(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "two_rank_sequence.py"
    script.write_text(TWO_RANK_SCRIPT.format(root=ROOT, tests=os.path.join(ROOT, "tests")))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("SEQUENCE OK") == 2


@pytest.mark.parametrize("schur_mode", [0, 1])
def test_reduced_system_matches_oracle(lvb_ctx, orc_ctx, schur_mode):
    """lvb_ba_reduced_system runs the first half of the pass: S assembled in the Schur kernel from a zeroed S, damping included.
    schur_mode = 1 assembles in the packing pass and subtracts U^T U on the tensor cores afterwards (S then within the 2e-5 of
    max|S| test_gpu_tensor_schur.py states; the rhs stays FP64)."""
    d = _window()
    pg, po = backend.Problem.from_dict(lvb_ctx, d), backend.Problem.from_dict(orc_ctx, d)
    pg.set_schur_mode(schur_mode)
    for radius in (1e4, 1.0):                         # twice on one problem: the second call starts from the first one's S
        Sg, bg, cg = pg.reduced_system(radius)
        So, bo, co = po.reduced_system(radius)
        assert abs(cg - co) < 1e-10 * co
        assert _rel(bg, bo) < 1e-9
        assert _rel(Sg, So) < (1e-9 if schur_mode == 0 else 2e-5), (radius, _rel(Sg, So))


def _solve(p, d, **opts):
    p.update_params(*_start(d))
    return p.solve(**opts), _params(p)


def test_counters_reset_across_solves_and_graph_retargeting(lvb):
    """Back-to-back solves on one problem (its own pass graph from the second on), a second problem that re-targets the context's
    cached graph, then solves that end in their first pass (max_num_iterations = 0: every kernel after the Schur kernel returns
    on `done`) and after one iteration.  A counter left non-zero would lose its last CTA: no pre-check, no decision."""
    a = _window()
    b = synth.make_ba_problem(10, 4000, with_imu=True, seed=synth.SEED + 5)
    runs = [(a, dict(max_num_iterations=10))] * 3 + [(b, dict(max_num_iterations=10))] + \
           [(a, dict(max_num_iterations=0)), (a, dict(max_num_iterations=1)), (a, dict(max_num_iterations=10))]
    ctx = backend.Context(lvb)
    pa, pb = backend.Problem.from_dict(ctx, a), backend.Problem.from_dict(ctx, b)
    for i, (d, opts) in enumerate(runs):
        got = _solve(pa if d is a else pb, d, **opts)
        fresh = _solve(backend.Problem.from_dict(backend.Context(lvb), d), d, **opts)
        assert got[0].num_iterations == opts["max_num_iterations"] or got[0].termination_type != 1, (i, got[0].num_iterations)
        _assert_same_path(got, fresh, what="run %d" % i)


@pytest.mark.parametrize("name", ["reject_run", "invalid"])
def test_rejected_and_invalid_steps_match_oracle(lvb, lvb_ctx, orc_ctx, name):
    """Rejected and invalid steps keep Hpp and rebuild S with the new damping; the window runs the six-kernel pass."""
    d, opts = _scenario(name)
    pg, po = backend.Problem.from_dict(lvb_ctx, d), backend.Problem.from_dict(orc_ctx, d)
    names = _timed_kernels(lvb, lambda: pg.solve(max_num_iterations=1, **opts))
    assert names == WINDOW_PASS * (len(names) // len(WINDOW_PASS)), names
    sg, xg = _solve(pg, d, max_num_iterations=25, **opts)
    so, xo = _solve(po, d, max_num_iterations=25, **opts)
    assert sg.num_iterations > sg.num_successful_steps           # some steps were rejected or invalid
    _assert_same_solve(sg, xg, so, xo, what=name)
