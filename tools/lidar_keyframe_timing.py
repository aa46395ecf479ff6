"""Wall time of a lidar keyframe's way from the raw scan into the resident map, two ways, alternated in one run:

  extract   lvb_lidar_extract_features alone (one host synchronisation), at a kitti-sized scan (64 x 1800) and a 16-ring scan
  host      extraction to the host (lvb_lidar_extract_features) + lvb_icp_map_optimize_keyframes fed with those host clouds
  by_key    lvb_icp_map_extract_keyframe (pending features, no host copies) + the same call registering them by key

for a pass of 1 and of 5 keyframes (one scan each, extracted and registered per pass; every keyframe merges up to three before it).
The pass's keyframes are evicted after each repetition.  Prints one JSON line (min / median ms per case, host synchronisations and
launches per case, the GPU's name, power limit and maximum SM clock); --out also writes it there.

    python tools/lidar_keyframe_timing.py [--reps 20] [--warmup 3] [--out FILE]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from lvio_fusion_b200 import backend, synth  # noqa: E402
from test_gpu_map_optimize import make_scene  # noqa: E402

GT = 0.05


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
    ap.add_argument("--out")
    a = ap.parse_args()
    ctx = backend.Context()
    sc = make_scene(200, 200)
    g, s = sc["g"], sc["s"]
    lf = backend.LidarFeatures(ctx)
    lf16 = backend.LidarFeatures(ctx, num_scans=16, ang_res_y=2.0, ang_bottom=15.1, ground_rows=7, max_range=50.0)
    scan64 = synth.make_lidar_scan(seed=81)
    scan16 = synth.make_lidar_scan(seed=82, num_scans=16, ang_res_y=2.0, ang_bottom=15.1)
    scans = [synth.make_lidar_scan(seed=90 + k) for k in range(5)]
    poses = [np.array([0, 0, np.sin(0.01 * k), np.cos(0.01 * k), 0.4 * k, 0.05 * k, 0.0]) for k in range(5)]
    ga, sa = backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)

    def chain(kfs):
        backend.build_and_optimize_keyframes(ga, sa, kfs, (g["cell_size"], s["cell_size"]), GT, (g["weight"], s["weight"]), sc["pw"],
                                             (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]))

    def keyframes(n, clouds):
        return [(k, list(range(max(0, k - 3), k)), poses[k], poses[k], clouds[k][0], clouds[k][1]) for k in range(n)]

    def host(n):
        chain(keyframes(n, [lf.extract(scans[k]) for k in range(n)]))

    def by_key(n):
        for k in range(n):
            lf.extract_into(ga, sa, k, scans[k], copies=False)
        chain(keyframes(n, [(None, None)] * n))

    cases = {
        "extract_64x1800": lambda: lf.extract(scan64),
        "extract_16x1800": lambda: lf16.extract(scan16),
        "host_1": lambda: host(1), "by_key_1": lambda: by_key(1),
        "host_5": lambda: host(5), "by_key_5": lambda: by_key(5),
    }
    times = {k: [] for k in cases}
    counts = {}
    for rep in range(a.warmup + a.reps):
        for name, fn in cases.items():
            ctx.synchronize()
            s0, l0 = ctx.sync_count(), ctx.launch_count()
            t0 = time.perf_counter()
            fn()
            dt = time.perf_counter() - t0
            counts[name] = (ctx.sync_count() - s0, ctx.launch_count() - l0)
            ga.map_evict(-1); sa.map_evict(-1)
            if rep >= a.warmup:
                times[name].append(dt * 1e3)
    res = {"gpu": gpu_info(), "reps": a.reps,
           "cases": {k: {"min_ms": round(min(v), 4), "median_ms": round(float(np.median(v)), 4), "syncs": counts[k][0], "launches": counts[k][1]}
                     for k, v in times.items()}}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
