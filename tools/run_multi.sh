#!/bin/bash
N=${1:-2}
timeout 300 python -m pytest tests/test_gpu_multi.py tests/test_gpu_map_optimize.py::test_sharded_context_is_unsupported -q -x 2>&1 | tail -4
timeout 200 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29531 bench.py --gpus $N --steps 40 --warmup 10 --skip-roofline --skip-icp --skip-global 2>&1 | grep -o '"value": [0-9.]*, "unit": "rows/s", "n_gpus": [0-9]*, "steps": [0-9]*, "warmup": 10, "ms_per_step": [0-9.]*' 
LVB_NO_P2P=1 timeout 200 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29532 bench.py --gpus $N --steps 40 --warmup 10 --skip-roofline --skip-icp --skip-global 2>&1 | grep -o '"value": [0-9.]*, "unit": "rows/s", "n_gpus": [0-9]*, "steps": [0-9]*, "warmup": 10, "ms_per_step": [0-9.]*'
