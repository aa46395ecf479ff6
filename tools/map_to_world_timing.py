"""Wall time of Mapping::ToWorld(start) after a correction (mapping.cpp:222-229): the world clouds of N resident keyframes, ground and
surf, re-made at new poses, two ways, alternated:

  loop  per keyframe and side lvb_icp_map_evict + lvb_icp_map_append of the robot-frame cloud from the host (what the shim's
        AppendKeyframe does): a pageable upload, an allocation, a kernel and a host synchronisation each
  call  lvb_icp_map_to_world over all N keyframes on both handles: one table upload, one kernel, one synchronisation

at N = 10, 100, 1000 keyframes and 3 000 (the reference's voxel-filtered size) and 40 000 points per keyframe and side.  Also the
kernel alone (CUDA events around it, lvb_debug_timing) and its achieved bandwidth from the algorithmic bytes: 32 B per point (the
robot record read, the world record written) plus the table (48 B per entry and side, its 4-byte block prefix, the 24-byte box written
back).  Both variants' clouds are compared bit for bit at the end.  Prints one JSON line per size (min / median / max ms per
re-anchoring of all N keyframes, launches and synchronisations, the GPU's name, power limit and max SM clock); --out also writes them.

    python tools/map_to_world_timing.py [--reps 20] [--warmup 3] [--keyframes 10,100,1000] [--points 3000,40000] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lvio_fusion_b200 import backend, synth  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def kernel_us(api, fn, n):
    """CUDA-event time of icp_map_to_world_kernel over n calls of fn (per-kernel timing on), median in microseconds."""
    api.debug_timing(1)
    for _ in range(n):
        fn()
    buf = C.create_string_buffer(1 << 20)
    api.debug_timing_report(buf, len(buf))
    t = [float(m.group(1)) for m in re.finditer(r"icp_map_to_world_kernel ([0-9.]+)", buf.value.decode())]
    return float(np.median(t)) if t else float("nan")


def one_size(ctx, n_kf, n_pts, reps, warmup):
    rng = np.random.default_rng(n_kf * 7 + n_pts)
    base = synth.make_icp_problem(1000, 3 * n_pts, seed=synth.SEED, kind="surf")["map_pose"]
    robot = [rng.normal(0, 10, (n_pts, 4)).astype(np.float32) for _ in range(2)]        # ground, surf (shared by every keyframe)
    poses = np.array([synth.se3_mul(base, np.r_[0, 0, 0, 1, 2.0 * k, 0, 0]) for k in range(n_kf)])
    keys = list(range(n_kf))

    def handles():
        fg, fs = backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)
        for k in keys:
            fg.map_append(k, robot[0], poses[k])
            fs.map_append(k, robot[1], poses[k])
        return fg, fs

    hl, hc = handles(), handles()
    state = {"i": 0}

    def moved():          # a new correction every repetition: both variants get the same one
        c = np.r_[synth.quat_from_rotvec(np.array([[0, 0, 1e-3 * (state["i"] % 7)]]))[0], 0.01 * (state["i"] % 5), 0, 0]
        return np.array([synth.se3_mul(c, p) for p in poses])

    def loop(p):
        for k in keys:
            for fa, cl in zip(hl, robot):
                fa.map_evict(k)
                fa.map_append(k, cl, p[k])

    def call(p):
        backend.map_to_world(hc[0], hc[1], keys, p)

    variants = {"loop": loop, "call": call}
    launches, syncs = {}, {}
    for name, fn in variants.items():
        for _ in range(warmup):
            fn(moved())
        p = moved()
        ctx.synchronize()
        n0, s0 = ctx.launch_count(), ctx.sync_count()
        fn(p)
        launches[name] = ctx.launch_count() - n0
        syncs[name] = ctx.sync_count() - s0
    times = {k: [] for k in variants}
    order = list(variants)
    for r in range(reps):
        state["i"] = r
        p = moved()
        for name in order[r % 2:] + order[:r % 2]:          # alternate who goes first
            ctx.synchronize()
            t0 = time.perf_counter()
            variants[name](p)
            times[name].append((time.perf_counter() - t0) * 1e3)
    # the clouds of the last repetition: identical
    same = True
    for fl, fc in zip(hl, hc):
        for k in sorted({0, n_kf // 2, n_kf - 1}):
            fl.map_build([k], 1.0)
            fc.map_build([k], 1.0)
            same = same and np.array_equal(fl.map_download().view(np.uint32), fc.map_download().view(np.uint32))
    p = moved()
    k_us = kernel_us(ctx.api, lambda: call(p), max(5, reps))
    pts = 2 * n_kf * n_pts
    nbytes = 32 * pts + (2 * n_kf) * (48 + 4 + 24)
    res = {"workload": "Mapping::ToWorld(start): %d keyframes x 2 sides x %d points re-anchored" % (n_kf, n_pts),
           "gpu": gpu_info(), "reps": reps, "warmup": warmup, "launches": launches, "syncs": syncs, "clouds_identical": bool(same),
           "kernel_us_median": k_us, "kernel_bytes": nbytes, "kernel_GBps": nbytes / (k_us * 1e3) if k_us == k_us else None}
    for k, v in times.items():
        res[k] = {"min_ms": float(np.min(v)), "median_ms": float(np.median(v)), "max_ms": float(np.max(v))}
    for fa in hl + hc:
        fa.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--keyframes", default="10,100,1000")
    ap.add_argument("--points", default="3000,40000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = backend.Context()
    lines = []
    for n_pts in [int(x) for x in a.points.split(",")]:
        for n_kf in [int(x) for x in a.keyframes.split(",")]:
            line = json.dumps(one_size(ctx, n_kf, n_pts, a.reps, a.warmup))
            print(line, flush=True)
            lines.append(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
