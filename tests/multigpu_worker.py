"""torchrun worker: solve one window sharded by landmark over WORLD_SIZE GPUs (one NCCL all-reduce of the reduced
system per LM iteration) and compare with the single-process CPU oracle.  Also a sharded scan-to-map.
Launched by tests/test_gpu_multi.py."""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch
import torch.distributed as dist

from lvio_fusion_b200 import _capi, backend, synth


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lvb = _capi.load()
    ctx = backend.Context(lvb, device=local)
    uid = ctypes.create_string_buffer(128)
    if rank == 0:
        lvb.check(lvb.comm_unique_id(uid), "comm_unique_id")
    box = [uid.raw]
    dist.broadcast_object_list(box, src=0)
    ctx.comm_init(rank, world, box[0])

    d = synth.make_ba_problem(8, 1500, with_imu=True, seed=31)
    p = backend.Problem.from_dict(ctx, synth.shard_ba_problem(d, rank, world))
    s = p.solve(max_num_iterations=25)
    P, V = p.poses(), p.vec3()
    rho = torch.from_numpy(np.where(np.arange(len(d["rho"])) % world == rank, p.inv_depths(), 0.0)).cuda()
    dist.all_reduce(rho)                                   # every rank owns the depths l % world == rank
    # a map-scale problem: banded storage, the envelope is the min over ranks of the local envelopes
    db = synth.make_ba_problem(60, 2500, with_imu=True, seed=33)
    pb = backend.Problem.from_dict(ctx, synth.shard_ba_problem(db, rank, world))
    sb = pb.solve(max_num_iterations=10)
    Pb = pb.poses()
    sc = synth.make_icp_problem(4000, 50000, seed=32, kind="ground")
    fa = backend.FeatureAssociation(ctx)
    fa.set_map(sc["map"], sc["cell_size"])
    e0 = synth.relative_rpyxyz(sc["map_pose"], sc["frame_pose"])
    lo, hi = rank * len(sc["scan"]) // world, (rank + 1) * len(sc["scan"]) // world
    e, si = fa.scan_to_map(sc["mode"], sc["scan"][lo:hi], sc["frame_pose"], sc["map_pose"], e0, sc["weight"], -1.0, sc["huber_a"], sc["thr"])
    # wall-clock cap on a sharded solve (Backend::Optimize always sets one, backend.cpp:208): the stop decision is collective,
    # so a tiny budget must end the solve early on every rank together instead of leaving a peer inside a collective
    pc = backend.Problem.from_dict(ctx, synth.shard_ba_problem(d, rank, world))
    scap = pc.solve(max_num_iterations=40, function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0, max_solver_time_in_seconds=2e-3)
    caps = torch.tensor([scap.num_iterations], device="cuda")
    gathered = [torch.zeros_like(caps) for _ in range(world)]
    dist.all_gather(gathered, caps)
    cap_iters = [int(g.item()) for g in gathered]
    ok = True
    if rank == 0:
        from oracle import binding
        orc = binding.load()
        octx = backend.Context(orc)
        po = backend.Problem.from_dict(octx, d)
        so = po.solve(max_num_iterations=25, num_threads=4)
        fo = backend.FeatureAssociation(octx)
        fo.set_map(sc["map"], sc["cell_size"])
        eo, sio = fo.scan_to_map(sc["mode"], sc["scan"], sc["frame_pose"], sc["map_pose"], e0, sc["weight"], -1.0, sc["huber_a"], sc["thr"])
        pbo = backend.Problem.from_dict(octx, db)
        sbo = pbo.solve(max_num_iterations=10, num_threads=4)
        checks = {
            "banded_cost": abs(sb.final_cost - sbo.final_cost) < 1e-6 * sbo.final_cost,
            "banded_iterations": sb.num_iterations == sbo.num_iterations,
            "banded_poses": np.max(np.abs(Pb - pbo.poses())) < 1e-5,
            "final_cost": abs(s.final_cost - so.final_cost) < 1e-6 * so.final_cost,
            "iterations": s.num_iterations == so.num_iterations,
            "poses": np.max(np.abs(P - po.poses())) < 1e-6,
            "vec3": np.max(np.abs(V - po.vec3())) < 1e-5,
            "rho": np.max(np.abs(rho.cpu().numpy() - po.inv_depths())) < 1e-6,
            "icp_blocks": si.num_residual_blocks == sio.num_residual_blocks,
            "icp_pose": np.max(np.abs(e - eo)) < 1e-7,
            "capped_same_iterations_everywhere": len(set(cap_iters)) == 1 and 1 <= cap_iters[0] < 40,
        }
        ok = all(checks.values())
        print("MULTIGPU", "OK" if ok else "FAIL", checks, "cost", s.final_cost, so.final_cost)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
