"""The backend, relocator and lidar threads on one resident keyframe store, with and without stream priorities, modes alternated:

  solo      the backend thread alone, default priority
  shared    the three threads on their own contexts over one store (lvb_icp_share), no lock, every context at the default priority
  priority  the same, with the backend thread's context at the device's greatest priority, the lidar thread's one step lower and the
            relocator's at the default (lvb_ctx_create_with_priority) -- the priorities INTEGRATION.md gives the reference's threads

The backend thread's pass follows Backend::Optimize: a configs[1] window solve (10 keyframes, 4000 landmarks, stereo + IMU; 10 LM
iterations from the same start every pass, tolerances off) and then Mapping::Optimize of five keyframes in one
lvb_icp_map_optimize_keyframes call (the five keys re-stored every pass; their map frames slide over three resident keyframes and the
call's own clouds).  The relocator thread runs --relocs lvb_icp_map_relocate calls against the three resident keyframes, the lidar
thread extracts a 64-ring scan every 2 ms until the backend thread is done.  No SegmentGround in the map frames (ground_threshold < 0),
so that the synthetic ground clouds register as the surf ones do.

Reported per mode, over all repetitions: the backend pass's median and p90 and the window solve's median share of a pass, the
relocation's median, the latency (request to return) of the extractions that start while a pass is in flight, median and p90, and the
median wall time until all three threads are done.  The first pass's results of each mode are compared with the solo one's.

Default clouds are configs[2]-shaped: 120 k-point scans against three 333 k-point resident keyframes; the reference's own load is a
few thousand voxel-filtered points per feature cloud: --scan 3000 --map 9000.  Prints one JSON line with the GPU's name and power
limit; --out also appends it there.

    python tools/map_priority_timing.py [--reps 5] [--passes 6] [--relocs 12] [--scan 120000] [--map 1000000] [--out FILE]
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
WINDOW_ITERS = 10


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
    window = synth.make_ba_problem(10, 4000, with_imu=True, seed=synth.SEED)          # configs[1]
    start = (window["poses"], window["vec3"] if len(window["vec3"]) else None, window["rho"])

    lib = _capi.load()
    least, greatest = backend.priority_range(lib, 0)
    opts = backend.default_options(lib, max_num_iterations=WINDOW_ITERS, function_tolerance=0.0, gradient_tolerance=0.0,
                                   parameter_tolerance=0.0)

    def resident(ctx):
        fg, fs = backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)
        for k, idx in enumerate(np.array_split(np.arange(a.map), 3)):
            fg.map_append(k, np.ascontiguousarray(g["map"][idx]), IDENT)
            fs.map_append(k, np.ascontiguousarray(s["map"][idx]), IDENT)
        return fg, fs

    def threads(prio_backend, prio_lidar, prio_reloc):
        """the three threads' contexts at these priorities (None: lvb_ctx_create), the store owned by the backend thread's pair"""
        def ctx(p):
            return backend.Context(lib) if p is None else backend.Context(lib, priority=p)
        cb, cr, cl = ctx(prio_backend), ctx(prio_reloc), ctx(prio_lidar)
        owner = resident(cb)
        return dict(backend=owner, problem=backend.Problem.from_dict(cb, window), reloc=(owner[0].share(cr), owner[1].share(cr)),
                    lidar=(owner[0].share(cl), owner[1].share(cl)), lf=backend.LidarFeatures(cl), contexts=(cb, cr, cl))

    shared = threads(None, None, None)
    prio = threads(greatest, min(greatest + 1, least), None)
    modes = {"solo": dict(shared, solo=True), "shared": dict(shared, solo=False), "priority": dict(prio, solo=False)}

    def backend_pass(v):
        """Backend::Optimize: the window solve, then Mapping::Optimize of the pass's keyframes; (window s, pass s, results)"""
        t0 = time.perf_counter()
        v["problem"].update_params(*start)
        v["problem"].solve(opts)
        t1 = time.perf_counter()
        out = backend.build_and_optimize_keyframes(v["backend"][0], v["backend"][1], kfs, cells, -1.0, weight, prior, huber, thr)
        return t1 - t0, time.perf_counter() - t0, (v["problem"].poses(), out)

    def relocate(pair):
        return backend.relocate(pair[0], pair[1], [0, 1, 2], cells, -1.0, g["map_pose"], g["map_pose"], rel, g["scan"], s["scan"], weight, huber, thr)

    # the passes' results do not depend on the mode
    first = {m: backend_pass(v)[2] for m, v in modes.items()}
    diff = 0.0
    for m in ("shared", "priority"):
        diff = max(diff, float(np.max(np.abs(first[m][0] - first["solo"][0]))))
        diff = max(diff, max(float(np.max(np.abs(x[0] - y[0]))) for x, y in zip(first[m][1], first["solo"][1])))

    def run(v):
        done = threading.Event()
        out = {"window": [], "pass": [], "pass_span": [], "reloc": [], "extract": []}
        n = 1 if v["solo"] else 3
        bar = threading.Barrier(n)

        def backend_thread():
            bar.wait()
            for _ in range(a.passes):
                t = time.perf_counter()
                w, p, _ = backend_pass(v)
                out["window"].append(w)
                out["pass"].append(p)
                out["pass_span"].append((t, t + p))
            done.set()

        def reloc_thread():
            bar.wait()
            for _ in range(a.relocs):
                t0 = time.perf_counter()
                relocate(v["reloc"])
                out["reloc"].append(time.perf_counter() - t0)

        def lidar_thread():
            bar.wait()
            while not done.is_set():
                t0 = time.perf_counter()
                v["lf"].extract_into(v["lidar"][0], v["lidar"][1], EXTRACT_KEY, sweep, False)
                out["extract"].append((t0, time.perf_counter() - t0))
                time.sleep(0.002)

        fns = [backend_thread] if v["solo"] else [backend_thread, reloc_thread, lidar_thread]
        ts = [threading.Thread(target=f) for f in fns]
        t0 = time.perf_counter()
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        out["wall"] = time.perf_counter() - t0
        # extractions that started while a pass was in flight
        out["extract_in_pass"] = [d for t, d in out["extract"] if any(b <= t < e for b, e in out["pass_span"])]
        return out

    for v in modes.values():           # warm-up: every call shape on every context
        run(v)
    res = {m: [] for m in modes}
    for _ in range(a.reps):
        for m, v in modes.items():
            res[m].append(run(v))

    def ms(x, q=50):
        return round(1e3 * float(np.percentile(x, q)), 3) if len(x) else None

    line = {"tool": "map_priority_timing", "gpu": gpu_info(), "scan": a.scan, "map": a.map, "passes": a.passes, "relocs": a.relocs,
            "reps": a.reps, "window": "configs[1], %d LM iterations" % WINDOW_ITERS, "priority_range": [least, greatest],
            "priorities": {"backend": greatest, "lidar": min(greatest + 1, least), "relocator": 0},
            "max_result_diff_between_modes": diff}
    for m, rs in res.items():
        passes = np.concatenate([r["pass"] for r in rs])
        share = np.concatenate([np.array(r["window"]) / np.array(r["pass"]) for r in rs])
        line[m] = {"wall_ms": ms([r["wall"] for r in rs]), "pass_median_ms": ms(passes), "pass_p90_ms": ms(passes, 90),
                   "window_share_of_pass": round(float(np.median(share)), 3)}
        if m != "solo":
            ext = np.concatenate([r["extract_in_pass"] for r in rs])
            line[m].update({"reloc_median_ms": ms(np.concatenate([r["reloc"] for r in rs])),
                            "extract_in_pass_median_ms": ms(ext), "extract_in_pass_p90_ms": ms(ext, 90), "extractions_in_pass": int(len(ext))})
    s_ = json.dumps(line)
    print(s_)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write(s_ + "\n")


if __name__ == "__main__":
    main()
