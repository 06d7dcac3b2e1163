"""torchrun check of the sharded CUDA path (NCCL, one GPU per rank): `ShardedB200Ranker` over WORLD_SIZE GPUs == fp64 oracle on
every row, with and without threshold sharing over NVLink peer memory, host inputs (`rank`) and device inputs
(`rank_device`), item sharding and -- with 3 or 4 ranks -- subject sharding and the item x subject grid.  The cases are the
table of tests/sharded_cases.py, which also runs on one GPU (tests/test_gpu_sharded_processes.py).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port <free port> \\
        scripts/dist_gpu_check.py [--out DIR]
"""
import os
import sys
import tempfile

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tests.sharded_cases import main  # noqa: E402

if __name__ == "__main__":
    args = sys.argv[1:]
    if "--out" not in args:  # (every rank of the node must name the same directory)
        args += ["--out", os.path.join(tempfile.gettempdir(), f"dist_gpu_check_{os.environ.get('MASTER_PORT', '0')}")]
    main(["--backend", "nccl", "--provider", "engine", "--check", *args])
