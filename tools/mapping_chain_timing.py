"""Wall time of Mapping::Optimize(active_kfs) for a backend pass that left N = 1 .. 5 lidar keyframes behind, two ways, alternated:

  loop   the per-keyframe form: lvb_icp_map_build_optimize_keyframe per keyframe, PoseGraph::ForwardUpdate of the later keyframes'
         incoming poses on the host (lvio_fusion_b200.se3) between the calls -- one host synchronisation per keyframe
  chain  lvb_icp_map_optimize_keyframes: all N keyframes in one call, one synchronisation

Every keyframe of the pass merges the three keyframes before it: three resident keyframes (the map split in three) at the start, then
the clouds the pass itself stores.  The pass's keyframes are evicted after each repetition so that every repetition starts from the
same map.  Two sizes: the reference's own load, a few thousand voxel-filtered points per feature cloud (--small 3000,9000: scan, map),
and configs[2] (--large 120000,1000000).  Prints one JSON line (per size and N: min / median / max ms per pass, launches and host
synchronisations per pass, the largest pose difference between the two ways, the GPU's name, power limit and maximum SM clock); --out also
writes it there.

    python tools/mapping_chain_timing.py [--reps 20] [--warmup 3] [--small 3000,9000] [--large 120000,1000000] [--out FILE]
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

from lvio_fusion_b200 import backend, se3, synth  # noqa: E402

GT = 0.05           # SegmentGround distance threshold of the ground map frames


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def measure(ctx, n_scan, n_map, reps, warmup):
    g = synth.make_icp_problem(n_scan, n_map, seed=synth.SEED, kind="ground")
    s = synth.make_icp_problem(n_scan, n_map, seed=synth.SEED, kind="surf")
    pw = g["n_features_left"] * synth.W_VISUAL
    ident = np.array([0, 0, 0, 1, 0, 0, 0.0])
    rng = np.random.default_rng(3)
    guesses = []
    for _ in range(5):                          # the incoming poses of the pass: the scene's guess, a few centimetres apart
        p = g["frame_pose"].copy()
        p[4:] += rng.normal(0, 0.03, 3)
        guesses.append(p)
    args = ((g["cell_size"], s["cell_size"]), GT)
    prm = ((g["weight"], s["weight"]), pw, (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]))

    def handles():
        fg, fs = backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)
        for k, (ig, is_) in enumerate(zip(np.array_split(np.arange(n_map), 3), np.array_split(np.arange(n_map), 3))):
            fg.map_append(k, np.ascontiguousarray(g["map"][ig]), ident)
            fs.map_append(k, np.ascontiguousarray(s["map"][is_]), ident)
        return fg, fs

    def evict(h, n):
        for fa in h:
            for k in range(3, 3 + n):
                fa.map_evict(k)

    hl, hc = handles(), handles()

    def loop(n):
        Ts, poses = [], {2: g["map_pose"]}
        for k in range(3, 3 + n):
            incoming = se3.forward_update(Ts, guesses[k - 3])
            p, _, _, _ = backend.build_and_optimize_keyframe(*hl, [k - 3, k - 2, k - 1], *args, k, poses[k - 1], incoming, g["scan"], s["scan"], *prm)
            Ts.append(se3.transform(p, incoming))
            poses[k] = p
        evict(hl, n)
        return [poses[k] for k in range(3, 3 + n)]

    def chain(n):
        kfs = [(k, [k - 3, k - 2, k - 1], g["map_pose"], guesses[k - 3], g["scan"], s["scan"]) for k in range(3, 3 + n)]
        out = backend.build_and_optimize_keyframes(*hc, kfs, *args, *prm)
        evict(hc, n)
        return [r[0] for r in out]

    res = {}
    for n in range(1, 6):
        variants = {"loop": lambda: loop(n), "chain": lambda: chain(n)}
        launches, syncs = {}, {}
        for name, fn in variants.items():
            for _ in range(warmup):
                fn()
            l0, s0 = ctx.launch_count(), ctx.sync_count()
            fn()
            launches[name], syncs[name] = ctx.launch_count() - l0, ctx.sync_count() - s0
        diff = float(max(np.max(np.abs(a - b)) for a, b in zip(loop(n), chain(n))))
        times = {k: [] for k in variants}
        order = list(variants)
        for r in range(reps):
            for name in order[r % 2:] + order[:r % 2]:          # alternate who goes first
                ctx.synchronize()
                t0 = time.perf_counter()
                variants[name]()
                times[name].append((time.perf_counter() - t0) * 1e3)
        row = {"launches": launches, "syncs": syncs, "max_pose_difference": diff}
        for k, v in times.items():
            row[k] = {"min_ms": float(np.min(v)), "median_ms": float(np.median(v)), "max_ms": float(np.max(v))}
        row["loop_minus_chain_median_ms"] = row["loop"]["median_ms"] - row["chain"]["median_ms"]
        res["N=%d" % n] = row
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--small", default="3000,9000")
    ap.add_argument("--large", default="120000,1000000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = backend.Context()
    out = {"workload": "Mapping::Optimize(active_kfs) for N lidar keyframes, each against the three before it (ground and surf map "
                       "frames, SegmentGround on the ground side); times per pass, the evictions of its keyframes included in both ways",
           "gpu": gpu_info(), "reps": a.reps}
    for label, spec in (("small", a.small), ("large", a.large)):
        n_scan, n_map = (int(x) for x in spec.split(","))
        out[label] = {"scan": n_scan, "map": n_map, **measure(ctx, n_scan, n_map, a.reps, a.warmup)}
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
