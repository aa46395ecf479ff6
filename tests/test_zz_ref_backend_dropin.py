"""Drop-in proof for SURVEY 8(a1/a2/a9): the REFERENCE's own src/backend.cpp + src/tools.cpp (and frame / landmark / map /
manager / preintegration), compiled where they lie, drive the product's header-only host side (include/lvio_b200/*.h).

tests/cpp/ref_backend_dropin.cpp plays the frontend (fills the reference's Map through the reference's own classes) and then
calls Backend::BuildProblem, adapt::Solve, imu::RecoverBias, imu::FullBA and compute_reprojection_error.  Three builds of it
live in oracle/_ref/ (made by `make -C oracle ref` where /root/reference is mounted; the binaries travel to the GPU box):

  ref_backend_truth   recording ceres + the reference's own factor headers: the cost the reference's functors assign
  ref_backend_orc     product shim, C ABI served by the CPU oracle (lvb_* renamed to orc_*)
  ref_backend_lvb     product shim bound to liblvio_b200.so: the CUDA path
  ref_mapping_*       the same for src/mapping.cpp (tests/cpp/ref_mapping_dropin.cpp), see the mapping test below

(The file sorts last on purpose: it is the only GPU test that runs prebuilt reference-derived binaries.)"""
import os
import re
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
HAVE_REFERENCE = os.path.isdir("/root/reference/src/lvio_fusion/include")


def _binary(name):
    if HAVE_REFERENCE:
        subprocess.check_call(["make", "-s", "-j4", "-C", os.path.join(ROOT, "oracle"), "ref"])
    path = os.path.join(REF_DIR, name)
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/%s is built only where the reference tree is mounted" % name)
    return path


def _run(name, mode, dump=None):
    args = [_binary(name), str(mode)] + ([dump] if dump else [])
    out = subprocess.run(args, check=True, capture_output=True, text=True, timeout=300).stdout
    rec = {}
    for line in out.splitlines():
        tag, rest = line.split(" ", 1)
        if tag in ("solve", "fullba") and "msg" in rest:
            rest, rec["msg"] = rest.split(" msg ", 1)
        toks = rest.split()
        if tag in ("mode", "blocks"):                   # "mode 0 keyframes 10 ...": the tag is the first key
            toks = [tag] + toks
        if tag in ("before", "after", "solve", "reference", "types", "kinds", "mode", "blocks"):
            for k, v in zip(toks[0::2], toks[1::2]):
                rec[tag + "." + k] = float(v)
        elif tag == "fullba" and toks[0] == "bias":
            rec["fullba.bias"] = np.array([float(v) for v in toks[1:7]])
        elif tag == "init" and toks[0] == "tilt_before":
            rec["init.tilt_before"] = float(toks[1])
        elif tag == "init" and toks[0] == "ok":
            rec["init.ok"], rec["init.initialized"], rec["init.tilt_after"] = int(toks[1]), int(toks[3]), float(toks[5])
            rec["init.bias"] = np.array([float(v) for v in toks[7:13]])
    rec["stdout"] = out
    return rec


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


@pytest.mark.parametrize("mode", [0, 1])
def test_reference_backend_builds_the_same_problem_on_the_shim(mode):
    """Backend::BuildProblem (src/backend.cpp:96-183) run against the product's ceres::Problem / factors.h and against the
    reference's own factors: same block census, and the cost the solver starts from (through the C ABI, oracle-served) is the
    cost the reference's functors assign to that problem -- reprojection, IMU and weak-constraint blocks, Huber(1) included."""
    t, o = _run("ref_backend_truth", mode), _run("ref_backend_orc", mode)
    for k in ("types.visual", "types.weak", "types.imu", "types.other", "types.frames", "types.global_end", "mode.reproj_n", "mode.landmarks"):
        assert t[k] == o[k], k
    assert o["kinds.two_frame"] + o["kinds.pose_only"] == o["types.visual"] + o["types.weak"] > 500      # backend.cpp:114,128,138
    assert o["kinds.two_camera"] + o["kinds.pose_graph"] + o["kinds.pose_prior"] == o["types.other"]       # :124,171,176
    assert o["kinds.imu"] == o["types.imu"] == (7 if mode == 0 else 0)
    assert o["kinds.pose_only"] > 100 and o["types.weak"] > 50                                               # landmarks born before the window; Far()
    if mode == 1:
        assert o["kinds.pose_graph"] == 2 and o["kinds.pose_prior"] == 0                                     # the two starved keyframes (:164-177)
    assert t["reference.initial_cost"] > 1e5
    assert _rel(o["solve.initial_cost"], t["reference.initial_cost"]) < 1e-12
    # compute_reprojection_error (backend.cpp:185-190): the host form of PoseOnlyReprojectionError in factors.h vs the reference's functor
    assert _rel(o["mode.reproj_sum"], t["mode.reproj_sum"]) < 1e-13
    # and adapt::Solve does its job on it (parameters are written back into Frame::pose / Landmark::inv_depth in place)
    assert o["solve.term"] == 0 and o["solve.final_cost"] < 0.25 * o["solve.initial_cost"]
    assert o["after.rel_t"] < 0.6 * o["before.rel_t"] and o["after.rel_r"] < 0.2 * o["before.rel_r"]
    assert o["after.reproj_sum"] < 0.25 * o["mode.reproj_sum"]


def test_reference_fullba_runs_on_the_shim():
    """imu::FullBA (src/tools.cpp:92-171) with the priors of Initializer::Initialize: ImuInitError blocks sharing one ba / bg
    block, every keyframe free.  The absolute pose is a gauge (no anchor in that problem), the relative motion is not."""
    o = _run("ref_backend_orc", 2)
    assert o["after.rel_t"] < 0.05 * o["before.rel_t"] and o["after.rel_r"] < 0.05 * o["before.rel_r"]
    assert np.max(np.abs(o["fullba.bias"])) < 1e-3            # the zero-mean bias prior of ImuInitError (Ba_j = Bg_j = 0) dominates


def test_reference_initializer_runs_on_the_shim():
    """SURVEY 8(f).1, "the unmodified Backend + Initializer run on the new solver": Initializer::Initialize(frames, 1e4, 1e2)
    (src/initializer.cpp:32-55, compiled in place) on a tilted, not yet gravity-aligned visual map with unknown biases --
    EstimateVelAndRwg, imu::InertialOptimization (the reference's loop over ImuInitGError::Create; factors.h builds it as a
    NumericDiffCostFunction around the caller's Preintegration::Evaluate(..., Rg), solved by the host LM with the quaternion
    parameterisation on Rwg), Map::ApplyGravityRotation, imu::FullBA (device path, oracle-served here)."""
    o = _run("ref_backend_orc", 3)
    assert o["init.ok"] == 1 and o["init.initialized"] == 1
    assert o["init.tilt_before"] > 0.15 and o["init.tilt_after"] < 0.12 * o["init.tilt_before"]        # 0.188 rad -> 0.014 rad
    assert o["after.rel_t"] < 0.12 * o["before.rel_t"] and o["after.rel_r"] < 0.05 * o["before.rel_r"]
    assert np.max(np.abs(o["init.bias"])) < 0.1


def test_reference_environment_single_frame_solve_runs_on_the_shim():
    """Environment::Optimize (src/environment.cpp:18-113, compiled in place; the weight-adaptation module's use of the hot path): one
    keyframe re-solved against fixed landmarks -- PoseOnlyReprojectionError for each of its features plus one ImuError whose other
    seven parameter blocks are SetParameterBlockConstant -- through the shim (constant flags on pose / vec3 blocks, DENSE_QR)."""
    out = _run("ref_backend_orc", 4)["stdout"].splitlines()[-1].split()
    rec = dict(zip(out[1::2], out[2::2]))
    assert int(rec["features"]) > 100 and int(rec["frame_untouched"]) == 1            # it works on a copy of the frame (:24-25)
    assert float(rec["reproj_after"]) < 0.9 * float(rec["reproj_before"]) and 1e-3 < float(rec["moved_t"]) < 0.5


def test_product_build_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    o = _run("ref_backend_lvb", 0)
    assert o["solve.term"] == 2 and "no CPU fallback" in o["msg"]
    assert o["after.rel_t"] == o["before.rel_t"]


def _run_mapping(name, dump):
    out = subprocess.run([_binary(name), dump], check=True, capture_output=True, text=True, timeout=300).stdout
    rec = {"stdout": out}
    for line in out.splitlines():
        t = line.split()
        if t[0] in ("before", "after"):
            rec[(t[0], int(t[2]))] = (float(t[4]), float(t[6]))
        elif t[0] == "map":
            rec["clouds"], rec["forward_updates"] = int(t[2]), int(t[4])
        elif t[0] == "relocate":
            rec["score"], rec["relocate_err"] = int(t[2]), (float(t[4]), float(t[6]))
    return rec, np.fromfile(dump)           # three optimised poses, the relocated relative pose, the score


def test_reference_mapping_optimize_runs_on_the_shim(tmp_path):
    """Mapping::Optimize (src/mapping.cpp:139-194, compiled in place): BuildMapFrame over the last three lidar keyframes,
    ScanToMapWithGround / ScanToMapWithSegmented, adapt::Solve(DENSE_QR, 4 iterations), rpyxyz2se3, ToWorld -- three
    keyframes in turn, each registered against a map that already holds its predecessor.

    ref_mapping_orc     the two ScanToMap members forward to lvio_b200/association.h (one fused cost per call, C ABI served
                        by the oracle); this is the INTEGRATION.md section 3 substitution
    ref_mapping_hostlm  nothing substituted: the reference's own kd-tree loop and one LidarPlaneError AutoDiff block per accepted
                        point plus the PoseErrorRPZ / YXY prior, solved by the shim's host LM
    Same poses from both: the fused association + closed-form Jacobians + LM of the device API do what the reference's block-
    per-point formulation does."""
    o, po = _run_mapping("ref_mapping_orc", str(tmp_path / "o.bin"))
    h, ph = _run_mapping("ref_mapping_hostlm", str(tmp_path / "h.bin"))
    assert o["clouds"] == 6 and o["forward_updates"] == 3                        # ToWorld for every optimised keyframe, PoseGraph::ForwardUpdate each time
    for k in (3, 4, 5):
        assert o[("after", k)][0] < 0.15 * o[("before", k)][0] and o[("after", k)][1] < 0.05 * o[("before", k)][1]
        assert o[("after", k)][0] < 0.025 and o[("after", k)][1] < 5e-4
    assert np.max(np.abs(po - ph)) < 1e-9
    # Mapping::Relocate (:246-300): relocate = true (no prior), four rounds of both solves, scored from the Summary fields -- the
    # one place the reference reads them (num_residual_blocks_reduced, final_cost): same score, same relative pose from both builds
    assert o["score"] == h["score"] >= 40 and po[-1] == ph[-1] == o["score"]
    assert o["relocate_err"][0] < 0.01 and o["relocate_err"][1] < 1e-3                     # from an 18 cm / 20 mrad initial guess


def test_reference_pose_graph_runs_on_the_host_lm():
    """SURVEY 8(f).4: PoseGraph::BuildProblem / Optimize (src/pose_graph.cpp:163-224, compiled in place, the reference's own
    PoseGraphError / RError AutoDiff functors) on a drifted lap whose loop start was relocated between the two calls, as
    Relocator::CorrectLoop does: two constant end poses, five free section poses with the quaternion parameterisation, solved by
    the shim's host LM; ForwardUpdate then moves the keyframes of each section.  Translation drift 1.06 m -> 0.39 m rms (what
    is left is the piecewise-rigid correction inside a section), constants untouched."""
    out = subprocess.run([_binary("ref_posegraph")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout
    t = out.stdout.split()
    rec = dict(zip(t[0::2], t[1::2]))
    assert int(rec["sections"]) == 5 and int(rec["blocks"]) == 7 and int(rec["residuals"]) == 11
    assert float(rec["rmse_after"]) < 0.5 * float(rec["rmse_before"]) and float(rec["moved_const"]) == 0.0


def test_reference_relocator_submap_rotation_runs_on_the_host_lm():
    """SURVEY 8(f).4: Relocator::UpdateNewSubmap (src/relocator.cpp:247-282, compiled in place): one bare quaternion block under
    EigenQuaternionParameterization, a RelocateRError per keyframe of the new submap, DENSE_QR.  The harness re-evaluates the
    objective with the reference's functor: the solved rotation beats the identity, the planted rotation and 2 000 perturbed
    candidates (to Ceres' function tolerance), and every other keyframe moves by the same rigid transform."""
    out = subprocess.run([_binary("ref_relocator")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout


def test_reference_navsat_runs_on_the_host_lm():
    """SURVEY 8(f).4: src/navsat.cpp compiled in place with its own AutoDiff functors.  Navsat::AddPoint interpolates the fixes
    onto the keyframes and fires Navsat::Initialize after the first 10 m (two-stage solve: yaw with x, y constant, then all three);
    Navsat::Optimize(section) then removes a heading error picked up in a bend: OptimizeBC (scalar blocks, some constant, z
    bounded, HuberLoss(0.1), a one-parameter roll pre-solve), OptimizeAB (PoseGraphError + TError, quaternion parameterisation),
    the per-keyframe x corrections.  All on include/lvio_b200/host_solver.h."""
    out = subprocess.run([_binary("ref_navsat")], capture_output=True, text=True, timeout=120, check=True).stdout.splitlines()
    a, b = out[0].split(), out[1].split()
    assert int(a[2]) == 1 and int(a[10]) >= 60                                           # initialised; nearly every keyframe got a fix
    assert abs(float(a[4]) - 0.3) < 5e-3 and abs(float(a[6]) - 5.0) < 0.05 and abs(float(a[8]) + 3.0) < 0.1      # yaw, x, y of the extrinsic from 10 m of driving
    rec = dict(zip(b[1::2], map(float, b[2::2])))
    assert rec["rms_after"] < 0.3 * rec["rms_before"] and rec["yaw_after"] < 0.1 * rec["yaw_before"] and rec["ab_rms"] < 0.15


@pytest.mark.gpu
def test_reference_mapping_optimize_drives_the_cuda_path(tmp_path):
    o, po = _run_mapping("ref_mapping_orc", str(tmp_path / "o.bin"))
    g, pg = _run_mapping("ref_mapping_lvb", str(tmp_path / "g.bin"))
    assert g["clouds"] == 6 and g["forward_updates"] == 3, g["stdout"]
    # three registrations in sequence, each map holding the previous result through a float32 transform: allow the cascade
    assert np.max(np.abs(pg[:-1] - po[:-1])) < 1e-5, g["stdout"]
    assert abs(g["score"] - o["score"]) <= 1, g["stdout"]                                  # an integer cast of a sum of two scores


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4])
def test_reference_backend_drives_the_cuda_path(mode, tmp_path):
    """The same binaries on the GPU: the reference's Backend::BuildProblem / adapt::Solve / imu::FullBA through the shim on
    liblvio_b200.so, against the oracle-served run of the identical problem."""
    fo, fg = str(tmp_path / "orc.bin"), str(tmp_path / "lvb.bin")
    o, g = _run("ref_backend_orc", mode, fo), _run("ref_backend_lvb", mode, fg)
    so, sg = np.fromfile(fo), np.fromfile(fg)
    assert so.shape == sg.shape and len(so) > 100
    if mode == 4:
        a, b = g["stdout"].splitlines()[-1].split(), o["stdout"].splitlines()[-1].split()
        ga, oa = dict(zip(a[1::2], map(float, a[2::2]))), dict(zip(b[1::2], map(float, b[2::2])))
        assert abs(ga["reproj_after"] - oa["reproj_after"]) < 1e-6 * oa["reproj_after"] and abs(ga["moved_t"] - oa["moved_t"]) < 1e-7
    elif mode < 2:
        assert g["solve.term"] == 0, g["stdout"]
        assert _rel(g["solve.initial_cost"], o["solve.initial_cost"]) < 1e-9
        assert _rel(g["solve.final_cost"], o["solve.final_cost"]) < 1e-5
        assert np.max(np.abs(so - sg)) < 1e-4
    else:
        # gauge-free problem: compare what is observable
        # same bounds as the CPU twins above: FullBA alone reaches 2 %, the whole Initializer chain 7 % of the initial translation error
        assert g["after.rel_t"] < (0.05 if mode == 2 else 0.12) * g["before.rel_t"] and g["after.rel_r"] < 0.05 * g["before.rel_r"]
        # (the indefinite-prior whitening makes these problems stiff -- entries ~1e9 -- and they have a gauge: the two LM runs are
        # compared on what they achieve, not digit by digit)
        assert abs(g["after.rel_t"] - o["after.rel_t"]) < 0.05 * o["after.rel_t"] + 1e-5 and abs(g["after.rel_r"] - o["after.rel_r"]) < 0.05 * o["after.rel_r"] + 1e-6
        if mode == 2:
            assert np.max(np.abs(g["fullba.bias"] - o["fullba.bias"])) < 5e-5
        else:
            assert g["init.ok"] == 1 and abs(g["init.tilt_after"] - o["init.tilt_after"]) < 1e-3 and np.max(np.abs(g["init.bias"] - o["init.bias"])) < 2e-3


@pytest.mark.gpu
def test_shim_solves_from_two_threads_on_the_device(tmp_path):
    """tests/test_capi_cpu.py::test_shim_solves_from_several_threads_at_once on the GPU: two host threads, each with its own
    per-thread context and stream (graph capture is thread-local), solve the same window at once; both must equal the single-threaded
    result.  Bounded by a timeout so that a wedged run cannot hold the box."""
    import shim_util
    from lvio_fusion_b200 import synth
    exe = shim_util.build_shim_binary()
    d = synth.make_ba_problem(4, 150, with_imu=True, seed=9)
    shim_util.dump_ba(tmp_path / "in.bin", d, 6)
    subprocess.run([exe, "ba", str(tmp_path / "in.bin"), str(tmp_path / "single.bin")], check=True, timeout=90)
    subprocess.run([exe, "ba_threads", str(tmp_path / "in.bin"), str(tmp_path / "multi.bin"), "2"], check=True, timeout=90)
    single = np.fromfile(tmp_path / "single.bin")
    for k in range(2):
        multi = np.fromfile(str(tmp_path / "multi.bin") + ".%d" % k)
        assert multi.shape == single.shape and np.max(np.abs(multi[:-4] - single[:-4])) < 1e-9
