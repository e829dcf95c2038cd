"""Worker of test_gpu_merge.py::test_merge_on_n_gpus: one process per GPU (torchrun), runs tg_merge over globally sorted
inputs sharded across the workers and checks every worker's exact share and the concatenation against merge_ref.  Exit
code 0 and MULTI_GPU_MERGE_OK = parity."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch.distributed as dist  # noqa: E402

import merge_ref as M  # noqa: E402
import sort_ref as R  # noqa: E402
from sort_ref import BE, LE, Desc  # noqa: E402
from thrill_b200 import api  # noqa: E402

U64 = Desc(8, 0, 8, LE)
PAIR = Desc(16, 0, 8, LE)


def gather(arr, world):
    parts = [None] * world
    dist.all_gather_object(parts, np.ascontiguousarray(arr))
    return parts


def merge_shards(tg, d, ptrs, sizes):
    k = len(ptrs)
    out, n = C.c_void_p(), C.c_size_t()
    tg.ck(tg.L.tg_merge(tg.h, C.byref(d.capi()), (C.c_void_p * k)(*ptrs), (C.c_size_t * k)(*sizes), k, C.byref(out), C.byref(n)))
    if not n.value:
        return np.zeros((0, d.item_bytes), np.uint8)
    return tg.download(out.value, n.value * d.item_bytes).reshape(-1, d.item_bytes)


def check(name, d, runs, out, rank, world, k):
    """runs: every worker's shards (runs[w * k + j]); out: this worker's result"""
    parts = gather(out, world)
    if rank == 0:
        n = sum(len(r) for r in runs)
        t = M.targets(world, n)
        sizes = [len(x) for x in parts]
        assert sizes == [int(t[w + 1] - t[w]) for w in range(world)], (name, sizes)
        assert np.array_equal(np.concatenate(parts), M.merged(runs, world, k, d)), name
        print("merge %s: %d items over %d workers ok" % (name, n, world), flush=True)


def case(tg, name, d, inputs, rank, world, shape, seed):
    """inputs: the k global (sorted) inputs, the same on every worker; sharded by `shape` with a shared seed"""
    k = len(inputs)
    runs = M.make_runs(inputs, world, np.random.RandomState(seed), shape)
    mine = [R.rows(runs[rank * k + j], d.item_bytes) for j in range(k)]
    ptrs = [tg.to_device(x) for x in mine]
    out = merge_shards(tg, d, ptrs, [len(x) for x in mine])
    for p_ in ptrs:
        tg.free(p_)
    check(name, d, runs, out, rank, world, k)


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    tg = ctx.tg
    rng = np.random.RandomState(11)          # the same stream on every worker

    def sorted_input(d, n, dist):
        return R.sort(R.make_items(d, n, dist, int(rng.randint(1 << 30))), d)

    # shards of very different sizes, empty shards, one worker holding everything
    for shape in ("random", "gaps", "one"):
        case(tg, "u64_k2_" + shape, U64, [sorted_input(U64, 200000, "uniform"), sorted_input(U64, 150001, "uniform")],
             rank, world, shape, 1)
        case(tg, "pair_k4_few_" + shape, PAIR, [sorted_input(PAIR, int(rng.randint(0, 90000)), "few") for _ in range(4)],
             rank, world, shape, 2)
    # all keys equal (the order is input-major, each input in position order)
    case(tg, "pair_k2_equal", PAIR, [sorted_input(PAIR, 70000, "equal"), sorted_input(PAIR, 50000, "equal")], rank, world, "random", 3)
    case(tg, "be16_k3", Desc(16, 0, 16, BE), [sorted_input(Desc(16, 0, 16, BE), 40000, "few") for _ in range(3)],
         rank, world, "random", 4)
    case(tg, "u64_desc_k2", Desc(8, 0, 8, LE, 1), [sorted_input(Desc(8, 0, 8, LE, 1), 60000, "few") for _ in range(2)],
         rank, world, "random", 5)
    # fewer items than workers, and nothing at all
    case(tg, "tiny", U64, [np.array([[7, 0, 0, 0, 0, 0, 0, 0]], np.uint8), np.zeros((0, 8), np.uint8)], rank, world, "random", 6)
    case(tg, "empty", U64, [np.zeros((0, 8), np.uint8)] * 2, rank, world, "random", 7)

    # an un-detached tg_sort result (it may lie in this worker's exchange window) as input 0
    local = np.random.RandomState(100 + rank).randint(0, 1 << 40, size=50000 + 20000 * rank).astype(np.uint64)
    d_in = tg.to_device(local)
    sout, sn = C.c_void_p(), C.c_size_t()
    tg.ck(tg.L.tg_sort(tg.h, C.byref(U64.capi()), d_in, len(local), 3, C.byref(sout), C.byref(sn)))
    other = M.make_runs([sorted_input(U64, 123457, "uniform")], world, np.random.RandomState(8), "random")
    mine1 = R.rows(other[rank], 8)
    d1 = tg.to_device(mine1)
    sorted_share = tg.download(sout.value, sn.value * 8).reshape(-1, 8)
    out = merge_shards(tg, U64, [sout.value, d1], [sn.value, len(mine1)])
    shares = gather(sorted_share, world)
    runs = []
    for w in range(world):
        runs += [shares[w], R.rows(other[w], 8)]
    check("sort_result_input", U64, runs, out, rank, world, 2)
    tg.free(d_in)
    tg.free(d1)

    tg.barrier()
    if rank == 0:
        print("MULTI_GPU_MERGE_OK world=%d" % world, flush=True)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
