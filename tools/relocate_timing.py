"""Wall time of Mapping::Relocate for one loop-closure candidate (mapping.cpp:78-112, 251-300), three ways, alternated:

  percall  the per-call path of the shim's ScanToMapWith* members: the old map frame's merged clouds handed over from the host,
           lvb_icp_set_map + lvb_icp_scan_to_map for each of the 8 registrations (4 rounds x ground, surf), the poses composed on
           the host -- 8 map uploads and voxel-hash builds, a host synchronisation after every LM pass
  step     the resident clouds, step by step: lvb_icp_map_build x2, then the 8 lvb_icp_scan_to_map calls
  call     lvb_icp_map_relocate: the two builds into the relocation slots and the 4 rounds in one call, one synchronisation

The old map frame is merged from three resident keyframes (no SegmentGround, so that the three variants register against the same
clouds).  Default clouds are configs[2]-shaped: a 120 k-point scan against a 1 M-point map frame, for the surf and for the ground
registration; the reference's own load is a few thousand voxel-filtered points per feature cloud: --scan 3000 --map 9000.
Prints one JSON line (min / median ms per candidate, launches and host synchronisations per candidate, the largest difference of
relative_o_c between the variants, the GPU's name and power limit); --out also writes it there.

    python tools/relocate_timing.py [--reps 20] [--warmup 3] [--scan 120000] [--map 1000000] [--out FILE]
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

ROUNDS = 4


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
    ident = np.array([0, 0, 0, 1, 0, 0, 0.0])
    map_pose = g["map_pose"]                  # the earliest old keyframe's pose
    old_pose = g["map_pose"]
    rel = synth.se3_mul(synth.se3_inv(old_pose), g["frame_pose"])
    cells = (g["cell_size"], s["cell_size"])
    keys = [0, 1, 2]

    def handles():
        fg, fs = backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)
        for k, (ig, is_) in enumerate(zip(np.array_split(np.arange(a.map), 3), np.array_split(np.arange(a.map), 3))):
            fg.map_append(k, np.ascontiguousarray(g["map"][ig]), ident)
            fs.map_append(k, np.ascontiguousarray(s["map"][is_]), ident)
        return fg, fs

    hp, hs, hc = handles(), handles(), handles()
    # the merged old map frame as the host would hand it over (pcl::PointXYZI-sized records, as the reference's clouds)
    host = []
    for fa, cell in zip(hp, cells):
        fa.map_build(keys, cell)
        m = np.zeros((len(fa.map_download()), 8), np.float32)
        m[:, :4] = fa.map_download()
        host.append(m)

    def rounds(fg, fs, per_call):
        p = synth.se3_mul(old_pose, rel)
        for _ in range(ROUNDS):
            e = synth.relative_rpyxyz(map_pose, p)
            if per_call:
                fg.set_map(host[0], cells[0])
            e, _ = fg.scan_to_map(0, g["scan"], p, map_pose, e, g["weight"], -1.0, g["huber_a"], g["thr"])
            p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
            if per_call:
                fs.set_map(host[1], cells[1])
            e, _ = fs.scan_to_map(1, s["scan"], p, map_pose, e, s["weight"], -1.0, s["huber_a"], s["thr"])
            p = synth.se3_mul(map_pose, synth.rpyxyz2se3(e))
        return synth.se3_mul(synth.se3_inv(old_pose), p)

    def percall():
        return rounds(*hp, True)

    def step():
        fg, fs = hs
        fg.map_build(keys, cells[0])
        fs.map_build(keys, cells[1])
        return rounds(fg, fs, False)

    def call():
        r, _, _, _, _ = backend.relocate(hc[0], hc[1], keys, cells, -1.0, map_pose, old_pose, rel, g["scan"], s["scan"],
                                         (g["weight"], s["weight"]), (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]), rounds=ROUNDS)
        return r

    variants = {"percall": percall, "step": step, "call": call}
    launches, syncs = {}, {}
    for name, fn in variants.items():
        for _ in range(a.warmup):
            fn()
        n0, s0 = ctx.launch_count(), ctx.sync_count()
        fn()
        launches[name] = ctx.launch_count() - n0
        syncs[name] = ctx.sync_count() - s0
    rp, rs, rc = percall(), step(), call()
    times = {k: [] for k in variants}
    order = list(variants)
    for r in range(a.reps):
        for name in order[r % len(order):] + order[:r % len(order)]:          # rotate who goes first
            ctx.synchronize()
            t0 = time.perf_counter()
            variants[name]()
            times[name].append((time.perf_counter() - t0) * 1e3)
    res = {"workload": "Mapping::Relocate per candidate (%d rounds): %d-point ground + %d-point surf scans vs %d-point old map frames "
                       "(3 resident keyframes), map builds included" % (ROUNDS, a.scan, a.scan, a.map),
           "gpu": gpu_info(), "reps": a.reps, "launches_per_candidate": launches, "syncs_per_candidate": syncs,
           "max_relative_o_c_difference_percall_vs_call": float(np.max(np.abs(rp - rc))),
           "max_relative_o_c_difference_step_vs_call": float(np.max(np.abs(rs - rc)))}
    for k, v in times.items():
        res[k] = {"min_ms": float(np.min(v)), "median_ms": float(np.median(v)), "max_ms": float(np.max(v))}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
