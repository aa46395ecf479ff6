"""The mapping, relocator and lidar threads on one resident keyframe store, two ways, alternated:

  shared  each thread on its own context and its own handle pair over one store (lvb_icp_share), no lock: the backend thread runs
          the keyframe chain on the owner pair, the relocator thread lvb_icp_map_relocate on a shared pair, the lidar thread
          lvb_icp_map_extract_keyframe on another shared pair
  locked  the same work on one pair and one context under one lock -- the integration before the store could be shared, where
          FeatureAssociation::Process and Mapping::Relocate took the mapping thread's lock

Per repetition: the backend thread runs --passes five-keyframe lvb_icp_map_optimize_keyframes passes (Mapping::Optimize of a backend
pass; the five keys are re-stored every pass, their map frames slide over three resident keyframes and the call's own clouds), the
relocator thread --relocs relocations against the three resident keyframes, and the lidar thread extracts a 64-ring scan every 2 ms
until the backend thread is done.  Reported per mode (medians over the repetitions): the wall time until all three threads are done,
the backend pass's median and p90 latency, the extraction latency (request to return, a lock wait included) while passes run, and the
relocation's median.  No SegmentGround in the map frames (ground_threshold < 0), so that the synthetic ground clouds register as the
surf ones do.

Default clouds are configs[2]-shaped: 120 k-point scans against three 333 k-point resident keyframes; the reference's own load is a
few thousand voxel-filtered points per feature cloud: --scan 3000 --map 9000.  Prints one JSON line with the GPU's name and power
limit; --out also writes it there.

    python tools/map_share_timing.py [--reps 5] [--passes 6] [--relocs 12] [--scan 120000] [--map 1000000] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lvio_fusion_b200 import _capi, backend, synth  # noqa: E402

IDENT = np.array([0, 0, 0, 1, 0, 0, 0.0])
CHAIN_KEYS = [100, 101, 102, 103, 104]
EXTRACT_KEY = 1000


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--passes", type=int, default=6)
    ap.add_argument("--relocs", type=int, default=12)
    ap.add_argument("--scan", type=int, default=120000)
    ap.add_argument("--map", type=int, default=1000000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    g = synth.make_icp_problem(a.scan, a.map, seed=synth.SEED, kind="ground")
    s = synth.make_icp_problem(a.scan, a.map, seed=synth.SEED, kind="surf")
    cells = (g["cell_size"], s["cell_size"])
    weight, huber, thr = (g["weight"], s["weight"]), (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"])
    prior = g["n_features_left"] * synth.W_VISUAL
    rng = np.random.default_rng(7)
    poses = []
    for _ in CHAIN_KEYS:
        p = g["frame_pose"].copy()
        p[4:] += rng.normal(0, 0.03, 3)
        poses.append(p)
    # keyframe k's map frame: the three keys before it, resident (0, 1, 2) or stored earlier in the pass
    order = [0, 1, 2] + CHAIN_KEYS
    kfs = [(key, order[i:i + 3], g["map_pose"], poses[i], g["scan"], s["scan"]) for i, key in enumerate(CHAIN_KEYS)]
    rel = synth.se3_mul(synth.se3_inv(g["map_pose"]), g["frame_pose"])
    sweep = synth.make_lidar_scan(seed=synth.SEED)

    def resident(ctx):
        fg, fs = backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)
        for k, (ig, is_) in enumerate(zip(np.array_split(np.arange(a.map), 3), np.array_split(np.arange(a.map), 3))):
            fg.map_append(k, np.ascontiguousarray(g["map"][ig]), IDENT)
            fs.map_append(k, np.ascontiguousarray(s["map"][is_]), IDENT)
        return fg, fs

    def chain(pair):
        return backend.build_and_optimize_keyframes(pair[0], pair[1], kfs, cells, -1.0, weight, prior, huber, thr)

    def relocate(pair):
        return backend.relocate(pair[0], pair[1], [0, 1, 2], cells, -1.0, g["map_pose"], g["map_pose"], rel, g["scan"], s["scan"], weight, huber, thr)

    # mode -> the three threads' (pair, context-bound LidarFeatures) and the lock around every call (None: no lock)
    lib = _capi.load()
    owner_ctx = backend.Context(lib)
    owner = resident(owner_ctx)
    ctx_r, ctx_l = backend.Context(lib), backend.Context(lib)
    shared_r = (owner[0].share(ctx_r), owner[1].share(ctx_r))
    shared_l = (owner[0].share(ctx_l), owner[1].share(ctx_l))
    lone_ctx = backend.Context(lib)
    lone = resident(lone_ctx)
    modes = {
        "shared": dict(backend=owner, reloc=shared_r, lidar=shared_l, lf=backend.LidarFeatures(ctx_l), lock=None),
        "locked": dict(backend=lone, reloc=lone, lidar=lone, lf=backend.LidarFeatures(lone_ctx), lock=threading.Lock()),
    }
    # the passes' results do not depend on the mode: the first pass of each is compared
    ref = {m: chain(v["backend"]) for m, v in modes.items()}
    diff = max(float(np.max(np.abs(x[0] - y[0]))) for x, y in zip(ref["shared"], ref["locked"]))

    def run(v):
        lock = v["lock"]

        def call(fn, *args):
            t0 = time.perf_counter()
            if lock is None:
                fn(*args)
            else:
                with lock:
                    fn(*args)
            return time.perf_counter() - t0

        done = threading.Event()
        out = {"pass": [], "reloc": [], "extract": []}
        bar = threading.Barrier(3)

        def backend_thread():
            bar.wait()
            for _ in range(a.passes):
                out["pass"].append(call(chain, v["backend"]))
            done.set()

        def reloc_thread():
            bar.wait()
            for _ in range(a.relocs):
                out["reloc"].append(call(relocate, v["reloc"]))

        def lidar_thread():
            bar.wait()
            while not done.is_set():
                out["extract"].append(call(v["lf"].extract_into, v["lidar"][0], v["lidar"][1], EXTRACT_KEY, sweep, False))
                time.sleep(0.002)

        ts = [threading.Thread(target=f) for f in (backend_thread, reloc_thread, lidar_thread)]
        t0 = time.perf_counter()
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        out["wall"] = time.perf_counter() - t0
        return out

    for v in modes.values():           # warm-up: every call shape on every context
        run(v)
    res = {m: [] for m in modes}
    for _ in range(a.reps):
        for m, v in modes.items():
            res[m].append(run(v))

    def ms(x, q=50):
        return round(1e3 * float(np.percentile(x, q)), 3)

    line = {"tool": "map_share_timing", "gpu": gpu_info(), "scan": a.scan, "map": a.map, "passes": a.passes, "relocs": a.relocs,
            "reps": a.reps, "max_pose_diff_between_modes": diff}
    for m, rs in res.items():
        line[m] = {
            "wall_ms": ms([r["wall"] for r in rs]),
            "pass_median_ms": ms(np.concatenate([r["pass"] for r in rs])),
            "pass_p90_ms": ms(np.concatenate([r["pass"] for r in rs]), 90),
            "extract_median_ms": ms(np.concatenate([r["extract"] for r in rs])),
            "extract_p90_ms": ms(np.concatenate([r["extract"] for r in rs]), 90),
            "reloc_median_ms": ms(np.concatenate([r["reloc"] for r in rs])),
            "extractions": int(sum(len(r["extract"]) for r in rs)),
        }
    s_ = json.dumps(line)
    print(s_)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write(s_ + "\n")


if __name__ == "__main__":
    main()
