"""Worker of test_gpu_reduce_records.py::test_reduce_records_on_n_gpus: one process per GPU (torchrun), runs
tg_reduce_by_key_records over records sharded across the workers (the operator's p > 1 path: pre phase, partition, count matrix,
exchange into the owners' windows, post phase) and checks every worker's exact result against reduce_records_ref; a worker of 2^30
items gives TG_ERR_TOO_LARGE on every rank.  Exit code 0 and MULTI_GPU_REDUCE_RECORDS_OK = parity."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch.distributed as dist  # noqa: E402

import join_records_ref as J  # noqa: E402
import reduce_records_ref as RR  # noqa: E402
from thrill_b200 import api, capi  # noqa: E402

TG_ERR_TOO_LARGE = -4


def split(arr, world):
    bounds = [api._local_range(len(arr), world, r) for r in range(world)]
    return [arr[lo:hi] for lo, hi in bounds]


def reduce_shard(tg, rec, key, runs, n=None):
    s = rec.shape[1]
    dp = tg.to_device(rec)
    out, m = C.c_void_p(), C.c_size_t()
    d = capi.reduce_records_desc(s, key[0], key[1], runs)
    st = tg.L.tg_reduce_by_key_records(tg.h, C.byref(d), dp, len(rec) if n is None else n, C.byref(out), C.byref(m))
    res = None
    if st == 0:
        res = tg.download(out.value, m.value * s).reshape(-1, s) if m.value else np.zeros((0, s), np.uint8)
    tg.free(dp)
    return st, res


def case(tg, name, rec, key, runs, rank, world):
    shards = split(rec, world)
    st, out = reduce_shard(tg, shards[rank], key, runs)
    assert st == 0, (name, st, tg.L.tg_last_error(tg.h))
    want = RR.reduce(shards, key, runs)[rank]
    assert np.array_equal(out, want), (name, rank, len(out), len(want))
    one = RR.reduce_local(rec, key, runs)                   # exact folds: the one-worker result, placed by the owner
    assert np.array_equal(out, one[J.owner(J.keys_of(one, *key), world) == rank]), (name, rank)
    if rank == 0:
        print("reduce_records %s ok on %d workers" % (name, world), flush=True)


def records(n, s, key, keys, runs, seed):
    rec = RR.make(n, s, key, keys, seed)
    for j, (off, cnt, op) in enumerate(runs):
        RR.set_fields(rec, off, cnt, RR.values(op, n, cnt, seed * 13 + j))
    return rec


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    tg = ctx.tg
    rng = np.random.default_rng(1)           # the same global records on every worker
    km = [(8, 3, 0), (32, 1, 1)]
    case(tg, "kmeans", records(400000, 40, (0, 8), rng.integers(0, 1024, 400000, dtype=np.uint64), km, 1), (0, 8), km, rank, world)
    li = [(8, 1, 1), (16, 3, 0), (40, 1, 2), (48, 1, 5)]
    case(tg, "line_items", records(100000, 176, (0, 1), rng.integers(0, 4, 100000, dtype=np.uint64), li, 2), (0, 1), li, rank, world)
    mk = [(0, 2, 3), (20, 2, 4)]
    case(tg, "zipf_unaligned_key", records(200000, 36, (16, 3), J.zipf_keys(200000, 50000, 1.0, 3), mk, 3), (16, 3), mk, rank, world)
    case(tg, "distinct", records(100000, 16, (0, 8), rng.permutation(100000).astype(np.uint64), [(8, 1, 0)], 4), (0, 8), [(8, 1, 0)],
         rank, world)
    case(tg, "one_key", records(50000, 24, (0, 8), np.full(50000, 9, np.uint64), [(8, 2, 1)], 5), (0, 8), [(8, 2, 1)], rank, world)
    case(tg, "key_only", records(30000, 4, (0, 4), rng.integers(0, 700, 30000, dtype=np.uint64), [], 6), (0, 4), [], rank, world)
    case(tg, "tiny", records(1, 12, (0, 4), np.ones(1, np.uint64), [(4, 1, 1)], 7), (0, 4), [(4, 1, 1)], rank, world)

    # 2^30 items on the last worker (nothing is read): TG_ERR_TOO_LARGE on every rank, and the ctx works afterwards
    small = records(1000, 40, (0, 8), rng.integers(0, 50, 1000, dtype=np.uint64), km, 8)
    st, _ = reduce_shard(tg, split(small, world)[rank], (0, 8), km, n=(1 << 30) if rank == world - 1 else None)
    assert st == TG_ERR_TOO_LARGE, (rank, st)
    case(tg, "after_too_large", small, (0, 8), km, rank, world)

    tg.barrier()
    if rank == 0:
        print("MULTI_GPU_REDUCE_RECORDS_OK world=%d" % world, flush=True)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
