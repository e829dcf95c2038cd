"""Worker of test_gpu_join_records.py::test_join_records_on_n_gpus: one process per GPU (torchrun), runs tg_inner_join_records
over record sides sharded across the workers and checks every worker's exact result against join_records_ref, and a 16-byte
pair join through the record path against the pair join's rows.  Exit code 0 and MULTI_GPU_JOIN_RECORDS_OK = parity."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch.distributed as dist  # noqa: E402

import join_records_ref as J  # noqa: E402
from thrill_b200 import api, capi  # noqa: E402

TG_ERR_TOO_LARGE = -4


def split(arr, world):
    bounds = [api._local_range(len(arr), world, r) for r in range(world)]
    return [arr[lo:hi] for lo, hi in bounds]


def join_shards(tg, lk, rk, l, r):
    lb, rb = l.shape[1], r.shape[1]
    dl, dr = tg.to_device(l), tg.to_device(r)
    out, n = C.c_void_p(), C.c_size_t()
    d = capi.JoinRecordsDesc(lb, rb, lk[0], lk[1], rk[0], rk[1])
    st = tg.L.tg_inner_join_records(tg.h, C.byref(d), dl, len(l), dr, len(r), C.byref(out), C.byref(n))
    res = None
    if st == 0:
        res = tg.download(out.value, n.value * (lb + rb)).reshape(-1, lb + rb) if n.value else np.zeros((0, lb + rb), np.uint8)
    tg.free(dl)
    tg.free(dr)
    return st, res


def case(tg, name, left, right, lk, rk, rank, world):
    lefts, rights = split(left, world), split(right, world)
    st, out = join_shards(tg, lk, rk, lefts[rank], rights[rank])
    assert st == 0, (name, st, tg.L.tg_last_error(tg.h))
    want = J.join(lefts, rights, lk, rk)[rank]
    assert np.array_equal(out, want), (name, rank, len(out), len(want))
    if rank == 0:
        print("join_records %s ok on %d workers" % (name, world), flush=True)


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    tg = ctx.tg
    rng = np.random.default_rng(1)           # the same global sides on every worker
    def side(n, s, key, keys, seed):
        return J.set_keys(J.make_records(n, s, seed), key[0], key[1], keys)
    case(tg, "uniform", side(200000, 24, (3, 5), rng.integers(0, 50000, 200000, dtype=np.uint64), 1),
         side(150001, 12, (5, 2), rng.integers(0, 50000, 150001, dtype=np.uint64), 2), (3, 5), (5, 2), rank, world)
    case(tg, "tpch_shaped", side(60000, 176, (0, 8), rng.integers(0, 15000, 60000, dtype=np.uint64), 3),
         side(15000, 152, (0, 8), rng.permutation(15000).astype(np.uint64), 4), (0, 8), (0, 8), rank, world)
    case(tg, "zipf", side(60000, 16, (8, 8), J.zipf_keys(60000, 3000, 1.0, 5), 5),
         side(50000, 4, (0, 4), J.zipf_keys(50000, 3000, 1.0, 6), 6), (8, 8), (0, 4), rank, world)
    case(tg, "one_key", side(3000, 8, (0, 8), np.full(3000, 7, np.uint64), 7),
         side(2000, 8, (0, 8), np.full(2000, 7, np.uint64), 8), (0, 8), (0, 8), rank, world)
    case(tg, "empty_right", side(5000, 1024, (1016, 8), rng.integers(0, 10, 5000, dtype=np.uint64), 9),
         side(0, 100, (0, 1), np.zeros(0, np.uint64), 10), (1016, 8), (0, 1), rank, world)
    case(tg, "tiny", side(1, 4, (0, 4), np.ones(1, np.uint64), 11), side(1, 4, (0, 4), np.ones(1, np.uint64), 12),
         (0, 4), (0, 4), rank, world)

    # an output over the limit on the worker that owns the hot key: TG_ERR_TOO_LARGE on every rank
    a, b = side(40000, 8, (0, 8), np.full(40000, 5, np.uint64), 13), side(30000, 8, (0, 8), np.full(30000, 5, np.uint64), 14)
    st, _ = join_shards(tg, (0, 8), (0, 8), split(a, world)[rank], split(b, world)[rank])
    assert st == TG_ERR_TOO_LARGE, st

    # an un-detached ReducePair result (it may lie in this worker's exchange window) joined with itself as records
    local = np.zeros(40000 + 10000 * rank, api.KV)
    local["key"] = np.random.default_rng(100 + rank).integers(0, 5000, len(local), dtype=np.uint64)
    local["val"] = np.arange(len(local), dtype=np.uint64)
    d_in = tg.to_device(local)
    rout, rn = C.c_void_p(), C.c_size_t()
    tg.ck(tg.L.tg_reduce_by_key(tg.h, C.byref(capi.KVDesc(16, capi.OP_SUM_U64)), d_in, len(local), C.byref(rout), C.byref(rn)))
    reduced = tg.download(rout.value, rn.value * 16).reshape(-1, 16) if rn.value else np.zeros((0, 16), np.uint8)
    out, n = C.c_void_p(), C.c_size_t()
    d = capi.JoinRecordsDesc(16, 16, 0, 8, 0, 8)
    tg.ck(tg.L.tg_inner_join_records(tg.h, C.byref(d), rout.value, rn.value, rout.value, rn.value, C.byref(out), C.byref(n)))
    got = tg.download(out.value, n.value * 32).reshape(-1, 32) if n.value else np.zeros((0, 32), np.uint8)
    shards = [None] * world
    dist.all_gather_object(shards, reduced)
    want = J.join(shards, shards, (0, 8), (0, 8))[rank]
    assert np.array_equal(got, want), ("reduce_result_self_join", rank)
    tg.free(d_in)

    tg.barrier()
    if rank == 0:
        print("MULTI_GPU_JOIN_RECORDS_OK world=%d" % world, flush=True)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
