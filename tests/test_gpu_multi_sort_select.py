"""Each rank's share of a real multi-GPU Sort and ReduceToIndex against the one-device simulation (tg_sort_select) and the
oracle: launches tests/multi_gpu_sort_worker.py with one process per GPU (torch.distributed.run), in both exchange modes (stores
into mapped peer windows, TG_EXCHANGE=nccl) and both sort pipelines.  Skipped where the machine has too few GPUs."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CASES = [(w, x, pl) for w in (2, 3, 4, 8) for x in ("p2p", "nccl") for pl in ("classify", "merge") if x == "p2p" or w <= 3]


@pytest.mark.parametrize("world,exchange,pipeline", CASES)
def test_rank_shares_match_the_simulation(world, exchange, pipeline):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs, the machine has %d" % (world, torch.cuda.device_count()))
    port = 29800 + CASES.index((world, exchange, pipeline))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(HERE, "multi_gpu_sort_worker.py")]
    env = dict(os.environ, TG_SORT_PIPELINE=pipeline)
    if exchange == "nccl":
        env["TG_EXCHANGE"] = "nccl"
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    assert res.returncode == 0 and "SORT_SELECT_MULTI_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-5000:]
