"""Worker of test_gpu_hll.py::test_hll_on_n_gpus: one process per GPU (torchrun), runs tg_hyperloglog on shards placed as the
layouts of tests/golden/reference_outputs_hll.npz at p = world place them (uneven and empty shards included) and checks that every
rank gets the reference's registers; then a shard of a real 2^30-item buffer on rank 0: TG_ERR_TOO_LARGE on every rank.
Exit code 0 and MULTI_GPU_HLL_OK = parity."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import hll_ref as H  # noqa: E402
from thrill_b200 import api  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "reference_outputs_hll.npz")
TG_ERR_TOO_LARGE = -4


def run(tg, shard, ib, p):
    d = tg.to_device(shard)
    out = np.full(1 << p, 0xEE, np.uint8)
    st = tg.L.tg_hyperloglog(tg.h, ib, p, d, len(shard) // (ib // 8), out.ctypes.data)
    assert st == 0, (st, tg.L.tg_last_error(tg.h))
    tg.free(d)
    return out


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    tg = ctx.tg
    g = H.Golden(GOLDEN)
    checked = 0
    for i, name in enumerate(g.names):
        if g.mode(i) == "hash":
            continue
        words, ib = np.ascontiguousarray(g.words(i)), g.item_bytes(i)
        for _, _, counts in g.layouts(i):
            if len(counts) != world:
                continue
            shard = H.shards_of(words, ib, counts)[rank]
            for p in g.precisions:
                regs = run(tg, shard, ib, p)
                assert np.array_equal(H.digest(regs), g.digest(i, p)), (name, p, rank)
                stored = g.regs(i, p)
                assert stored is None or np.array_equal(regs, stored), (name, p, rank)
                checked += 1
    assert checked >= 60

    # one worker holds a real buffer of 2^30 items: every rank returns TG_ERR_TOO_LARGE, and the ctx keeps working
    n = (1 << 30) if rank == 0 else 16
    big = torch.empty(n, dtype=torch.int64, device="cuda:%d" % tg.device)
    out = np.zeros(1 << 10, np.uint8)
    st = tg.L.tg_hyperloglog(tg.h, 8, 10, big.data_ptr(), n, out.ctypes.data)
    assert st == TG_ERR_TOO_LARGE, st
    del big
    torch.cuda.empty_cache()
    x = np.arange(1000 * world, dtype=np.uint64)
    regs = run(tg, x[1000 * rank:1000 * (rank + 1)], 8, 10)
    assert np.array_equal(regs, H.registers(x, 8, 10))

    tg.barrier()
    if rank == 0:
        print("MULTI_GPU_HLL_OK world=%d cases=%d" % (world, checked), flush=True)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
