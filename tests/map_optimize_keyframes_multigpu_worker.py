"""torchrun worker: lvb_icp_map_optimize_keyframes on a context with world_size > 1 reports LVB_ERR_UNSUPPORTED (sharded
registration stays with lvb_icp_scan_to_map), launches nothing and stores nothing.  Launched by tests/test_gpu_map_optimize_keyframes.py."""
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

    g = synth.make_icp_problem(3000, 30000, seed=5, kind="ground")
    s = synth.make_icp_problem(3000, 30000, seed=5, kind="surf")
    ident = np.array([0, 0, 0, 1, 0, 0, 0.0])
    fg, fs = backend.FeatureAssociation(ctx), backend.FeatureAssociation(ctx)
    fg.map_append(0, g["map"], ident)
    fs.map_append(0, s["map"], ident)
    n0 = ctx.launch_count()
    kfs = [(1, [0], g["map_pose"], g["frame_pose"], g["scan"], s["scan"]), (2, [1], ident, g["frame_pose"], g["scan"], s["scan"])]
    try:
        backend.build_and_optimize_keyframes(fg, fs, kfs, (g["cell_size"], s["cell_size"]), -1.0, (g["weight"], s["weight"]), -1.0,
                                             (g["huber_a"], s["huber_a"]), (g["thr"], s["thr"]))
        raise SystemExit("rank %d: no error on a sharded context" % rank)
    except RuntimeError as e:
        assert "(-5)" in str(e), str(e)
    assert ctx.launch_count() == n0
    for fa in (fg, fs):
        for key in (1, 2):
            try:
                fa.map_build([key], 1.0)
                raise SystemExit("rank %d: the failed call stored key %d" % (rank, key))
            except RuntimeError:
                pass
    dist.barrier()
    if rank == 0:
        print("MAP OPTIMIZE KEYFRAMES MULTIGPU OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
