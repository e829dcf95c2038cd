"""Worker of test_gpu_sample.py::test_sample_on_n_gpus: one process per GPU (torchrun).  Every rank runs tg_sample /
tg_bernoulli_sample on its shard with a seed of its own (rank 0's wins) and checks its output against its slice of the model
(sample_ref.py) for rank 0's seed; shardings include empty workers and all items on one worker.  Exit code 0 and
MULTI_GPU_SAMPLE_OK = parity."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch.distributed as dist  # noqa: E402

import sample_ref as S  # noqa: E402
from thrill_b200 import api  # noqa: E402


def run(tg, items, sizes, rank, bern, param, seed):
    ib = items.shape[1] * 4
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    mine = np.ascontiguousarray(items[off[rank]:off[rank + 1]])
    d = tg.to_device(mine) if len(mine) else None
    out, n = C.c_void_p(), C.c_size_t()
    fn = tg.L.tg_bernoulli_sample if bern else tg.L.tg_sample
    tg.ck(fn(tg.h, ib, d, len(mine), param, seed + 1000 * rank, C.byref(out), C.byref(n)))
    got = tg.download(out.value, n.value * ib).view(np.uint32).reshape(n.value, ib // 4) if n.value else mine[:0]
    if d is not None:
        tg.free(d)
    mask = S.bernoulli_mask(seed, len(items), param) if bern else S.sample_mask(seed, len(items), param)
    want = S.split(items, mask, sizes)[rank]
    assert np.array_equal(got, want), (bern, param, sizes, rank)


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    tg = ctx.tg
    checked = 0
    for ib, N in ((8, 1_000_000), (24, 50_001), (100, 4097)):
        g = np.arange(N, dtype=np.uint64)
        items = np.zeros((N, ib // 4), np.uint32)
        items[:, 0] = (g & np.uint64(0xFFFFFFFF)).astype(np.uint32)
        items[:, 1:] = 7
        even = [N * (r + 1) // world - N * r // world for r in range(world)]
        holes = list(even)
        holes[0] += holes[-1]
        holes[-1] = 0
        one = [0] * world
        one[world - 1] = N
        for sizes in (even, holes, one):
            for s in (0, 1, 10, N - 1, N, N + 5):
                run(tg, items, sizes, rank, False, s, 77)
                checked += 1
            for q in (0.0, 1e-6, 0.3, 1.0):
                run(tg, items, sizes, rank, True, q, 78)
                checked += 1
    tg.barrier()
    if rank == 0:
        print("MULTI_GPU_SAMPLE_OK world=%d cases=%d" % (world, checked), flush=True)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
