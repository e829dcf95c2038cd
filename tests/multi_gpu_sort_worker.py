"""Worker of tests/test_gpu_multi_sort_select.py: one process per GPU (torchrun).  Pins what each rank of a real multi-GPU run
receives to the one-device simulation of the same workers:

- Sort: rank 0 gathers every rank's shard and runs tg_sort_select with the operator's seed; each rank's tg_sort result must be
  the stable sort of the items the simulation sent to that rank (this also checks the speculative top bit of the received
  items' local sort, which is derived from the rank's two splitters);
- ReduceToIndex with result sizes below the world size and not a multiple of it: each rank's dense array is its slice of
  oracle_lib.reduce_to_index.

Exit code 0 and SORT_SELECT_MULTI_OK on rank 0's stdout = every rank matched."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch.distributed as dist  # noqa: E402

import oracle_lib as O  # noqa: E402
import sample_sort_ref as S  # noqa: E402
import sort_ref as R  # noqa: E402
from sort_ref import BE, LE, Desc  # noqa: E402
from thrill_b200 import api, capi  # noqa: E402

DESCS = [Desc(8, 0, 8, LE), Desc(8, 0, 8, LE, 1), Desc(8, 0, 5, LE), Desc(8, 4, 4, BE), Desc(16, 0, 8, LE),
         Desc(16, 9, 6, LE), Desc(16, 0, 16, BE), Desc(16, 0, 10, BE, 1)]


def gather(arr, world):
    parts = [None] * world
    dist.all_gather_object(parts, np.ascontiguousarray(arr))
    return parts


def device_sort(tg, d, rows, seed):
    """tg_sort of this rank's shard (collective): its share of the result"""
    ib = d.item_bytes
    din = tg.to_device(rows)
    out, n = C.c_void_p(), C.c_size_t()
    tg.ck(tg.L.tg_sort(tg.h, C.byref(d.capi()), din, len(rows), seed, C.byref(out), C.byref(n)))
    res = tg.download(out.value, n.value * ib).reshape(-1, ib) if n.value else np.zeros((0, ib), np.uint8)
    tg.free(din)
    return res


def simulated_shares(tg, d, shards, p, seed):
    """what tg_sort_select sends to each rank, stably sorted: the received items arrive grouped by source in rank order"""
    ib = d.item_bytes
    din = [tg.to_device(s) if len(s) else None for s in shards]
    dout = [tg.alloc(max(len(s) * ib, 16)) for s in shards]
    spl = np.zeros((p - 1, ib + 8), np.uint8)
    counts = np.zeros(p * p, np.uint64)
    tg.ck(tg.L.tg_sort_select(tg.h, C.byref(d.capi()), (C.c_void_p * p)(*din), (C.c_size_t * p)(*[len(s) for s in shards]), p,
                              seed, spl.ctypes.data, (C.c_void_p * p)(*dout), counts.ctypes.data_as(C.POINTER(C.c_uint64)), None))
    counts = counts.reshape(p, p).astype(np.int64)
    grouped = [tg.download(o, len(s) * ib).reshape(-1, ib) if len(s) else np.zeros((0, ib), np.uint8) for o, s in zip(dout, shards)]
    for q in din + dout:
        if q:
            tg.free(q)
    w_spl, w_counts, w_grouped, _ = S.select(shards, d, p, seed)
    assert np.array_equal(spl, w_spl) and np.array_equal(counts, w_counts.astype(np.int64)), d.name
    shares = []
    for r in range(p):
        recv = [grouped[src][counts[src, :r].sum():counts[src, :r + 1].sum()] for src in range(p)]
        shares.append(R.sort(np.concatenate(recv), d))
    return shares


def main():
    ctx = api.Context.from_env(rng_seed=5)
    tg = ctx.tg
    rank, world = ctx.my_rank(), ctx.num_workers()
    checked = 0

    # ---- Sort: each rank's share is the simulation's ----
    for di, d in enumerate(DESCS):
        for dist_name, n in (("uniform", 30000), ("few", 20000), ("onetop", 25000), ("equal", 5000)):
            seed = 1000 * di + len(dist_name)
            local = S.make_items(d, n + 131 * rank, dist_name, 77 * rank + di)
            shards = gather(local, world)
            parts = gather(device_sort(tg, d, local, seed), world)
            if rank == 0:
                shares = simulated_shares(tg, d, shards, world, seed)
                for r in range(world):
                    assert np.array_equal(parts[r], shares[r]), "sort %s %s: rank %d's share" % (d.name, dist_name, r)
            checked += 1

    # ---- ReduceToIndex: result sizes below / not a multiple of the world size ----
    kvd = capi.KVDesc(16, capi.OP_SUM_U64)
    neutral = np.array([7, 9], dtype=np.uint64)
    for size in sorted({max(world - 1, 1), world + 1, 3 * world + 1, 1000 * world + 7}):
        kv = np.zeros(3000 + 17 * rank, dtype=O.KV)
        rs = np.random.RandomState(size + rank)
        kv["key"] = rs.randint(0, size, size=len(kv))
        kv["val"] = rs.randint(0, 1 << 40, size=len(kv))
        allkv = np.concatenate(gather(kv, world))
        din = tg.to_device(kv)
        out, n, begin = C.c_void_p(), C.c_size_t(), C.c_uint64()
        tg.ck(tg.L.tg_reduce_to_index(tg.h, C.byref(kvd), din, len(kv), size, neutral.ctypes.data, C.byref(out), C.byref(n),
                                      C.byref(begin)))
        res = tg.download(out.value, n.value * 16).view(O.KV) if n.value else np.zeros(0, O.KV)
        tg.free(din)
        want = O.reduce_to_index(allkv, size, O.OP_SUM_U64, neutral=(7, 9))
        b0, b1 = S.begin_of_part(rank, size, world), S.begin_of_part(rank + 1, size, world)
        assert begin.value == b0 and n.value == b1 - b0, (size, rank, begin.value, n.value)
        assert np.array_equal(res, want[b0:b1]), "reduce_to_index size %d: rank %d's slice" % (size, rank)
        checked += 1

    flags = gather(np.array([checked]), world)
    dist.barrier()
    if rank == 0:
        print("SORT_SELECT_MULTI_OK world=%d exchange=%s pipeline=%s checks=%s" % (
            world, os.environ.get("TG_EXCHANGE", "p2p"), os.environ.get("TG_SORT_PIPELINE", "classify"),
            [int(f[0]) for f in flags]))
    ctx.close()


if __name__ == "__main__":
    main()
