"""Per-keyframe wall time of Mapping::Optimize (mapping.cpp:114-185) on the device-resident map, three ways, alternated:

  step  the existing entry points: lvb_icp_map_build x2, lvb_icp_scan_to_map (ground), the pose composed on the host,
        lvb_icp_scan_to_map (surf) from that pose, lvb_icp_map_append(NULL) x2 -- a host synchronisation after every LM pass
  call  lvb_icp_map_build x2, then lvb_icp_map_optimize_keyframe -- one synchronisation at the end
  one   lvb_icp_map_build_optimize_keyframe: the two builds and the registrations in one call, one synchronisation
  build lvb_icp_map_build x2 alone (the part step and call share)

Clouds are configs[2]-shaped: a 120 k-point scan against a 1 M-point map frame merged from three resident keyframes, for the surf and
for the ground registration; the keyframe appended by each iteration is evicted again so that every iteration sees the same map.
The reference's own load is a few thousand voxel-filtered points per feature cloud: --scan 3000 --map 9000.
Prints one JSON line (min / median ms per keyframe, launches and host synchronisations per keyframe, the GPU's name and power
limit); --out also writes it there.

    python tools/mapping_keyframe_timing.py [--reps 20] [--warmup 3] [--scan 120000] [--map 1000000] [--out FILE]
"""
import argparse
import json
import os
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--scan", type=int, default=120000)
    ap.add_argument("--map", type=int, default=1000000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    ctx = backend.Context()
    g = synth.make_icp_problem(a.scan, a.map, seed=synth.SEED, kind="ground")
    s = synth.make_icp_problem(a.scan, a.map, seed=synth.SEED, kind="surf")
    pw = g["n_features_left"] * synth.W_VISUAL
    ident = np.array([0, 0, 0, 1, 0, 0, 0.0])
    map_pose, guess = g["map_pose"], g["frame_pose"]

    def handles():
        fg, fs = backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)
        for k, (ig, is_) in enumerate(zip(np.array_split(np.arange(a.map), 3), np.array_split(np.arange(a.map), 3))):
            fg.map_append(k, np.ascontiguousarray(g["map"][ig]), ident)
            fs.map_append(k, np.ascontiguousarray(s["map"][is_]), ident)
        return fg, fs

    def build(fg, fs):
        fg.map_build([0, 1, 2], g["cell_size"])
        fs.map_build([0, 1, 2], s["cell_size"])

    def evict(fg, fs):
        fg.map_evict(3)
        fs.map_evict(3)

    hs, hc, ho, hb = handles(), handles(), handles(), handles()

    def step():
        fg, fs = hs
        build(fg, fs)
        e = synth.relative_rpyxyz(map_pose, guess)
        e, _ = fg.scan_to_map(0, g["scan"], guess, map_pose, e, g["weight"], pw, g["huber_a"], g["thr"])
        p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
        e, _ = fs.scan_to_map(1, s["scan"], p, map_pose, e, s["weight"], pw, s["huber_a"], s["thr"])
        p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
        fg.map_append(3, None, p)
        fs.map_append(3, None, p)
        evict(fg, fs)
        return p

    def call():
        fg, fs = hc
        build(fg, fs)
        p, _, _ = backend.optimize_keyframe(fg, fs, 3, map_pose, guess, g["scan"], s["scan"], (g["weight"], s["weight"]), pw,
                                            (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]))
        evict(fg, fs)
        return p

    def one():
        fg, fs = ho
        p, _, _, _ = backend.build_and_optimize_keyframe(fg, fs, [0, 1, 2], (g["cell_size"], s["cell_size"]), -1.0, 3, map_pose, guess,
                                                         g["scan"], s["scan"], (g["weight"], s["weight"]), pw, (g["huber_a"], s["huber_a"]),
                                                         (g["thr"], s["thr"]))
        evict(fg, fs)
        return p

    def build_only():
        build(*hb)
        ctx.synchronize()

    variants = {"step": step, "call": call, "one": one, "build": build_only}
    launches, syncs = {}, {}
    for name, fn in variants.items():
        for _ in range(a.warmup):
            fn()
        n0, s0 = ctx.launch_count(), ctx.sync_count()
        fn()
        launches[name] = ctx.launch_count() - n0
        syncs[name] = ctx.sync_count() - s0
    ps, pc, po = step(), call(), one()
    pose_diff = float(np.max(np.abs(ps - pc)))
    pose_diff_one = float(np.max(np.abs(ps - po)))
    times = {k: [] for k in variants}
    order = list(variants)
    for r in range(a.reps):
        for name in order[r % len(order):] + order[:r % len(order)]:          # rotate who goes first
            ctx.synchronize()
            t0 = time.perf_counter()
            variants[name]()
            times[name].append((time.perf_counter() - t0) * 1e3)
    res = {"workload": "Mapping::Optimize per keyframe: %d-point ground + %d-point surf scans vs %d-point map frames (3 resident keyframes), "
                       "map builds included" % (a.scan, a.scan, a.map),
           "gpu": gpu_info(), "reps": a.reps, "launches_per_keyframe": launches, "syncs_per_keyframe": syncs,
           "max_pose_difference_step_vs_call": pose_diff, "max_pose_difference_step_vs_one": pose_diff_one}
    for k, v in times.items():
        res[k] = {"min_ms": float(np.min(v)), "median_ms": float(np.median(v)), "max_ms": float(np.max(v))}
    res["step_minus_call_median_ms"] = res["step"]["median_ms"] - res["call"]["median_ms"]
    res["call_minus_one_median_ms"] = res["call"]["median_ms"] - res["one"]["median_ms"]
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
