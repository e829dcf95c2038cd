"""Worker of test_gpu_group.py::test_group_on_n_gpus: one process per GPU (torchrun), runs tg_group_by_key / tg_group_to_index
over inputs sharded across the workers and checks every worker's exact result against group_ref, and its rows of the group
functions against the reference's worker at this p in tests/golden/reference_outputs_group.npz.  Exit code 0 and
MULTI_GPU_GROUP_OK = parity."""
import ctypes as C
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch.distributed as dist  # noqa: E402

import group_ref as G  # noqa: E402
from thrill_b200 import api  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "reference_outputs_group.npz")
TG_ERR_ARG = -3


def run(tg, shard, size):
    d = tg.to_device(shard)
    out, n, b, e = C.c_void_p(), C.c_size_t(), C.c_uint64(), C.c_uint64()
    if size is None:
        st = tg.L.tg_group_by_key(tg.h, d, len(shard), C.byref(out), C.byref(n))
    else:
        st = tg.L.tg_group_to_index(tg.h, d, len(shard), size, C.byref(out), C.byref(n), C.byref(b), C.byref(e))
    res = None
    if st == 0:
        res = tg.download(out.value, n.value * 16).view(G.KV) if n.value else np.zeros(0, G.KV)
    tg.free(d)
    return st, res, b.value, e.value


def expected(inp, size, world):
    shards = G.split_shards(inp, world)
    own = (lambda k: G.owner_mod(k, world)) if size is None else (lambda k: G.owner_range(k, size, world))
    return [G.grouped(x) for x in G.exchange(shards, own)]


def case(tg, name, inp, size, rank, world):
    st, res, b, e = run(tg, G.split_shards(inp, world)[rank], size)
    assert st == 0, (name, st, tg.L.tg_last_error(tg.h))
    assert np.array_equal(res.view(np.uint64), expected(inp, size, world)[rank].view(np.uint64)), (name, rank)
    if size is not None:
        assert (b, e) == (G.range_begin(rank, size, world), G.range_begin(rank + 1, size, world)), (name, rank, b, e)
    return res


def gather(arr, world):
    parts = [None] * world
    dist.all_gather_object(parts, np.ascontiguousarray(arr))
    return parts


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    tg = ctx.tg
    case(tg, "uniform", G.make_input(200001, 1 << 40, 1), None, rank, world)
    case(tg, "uniform_index", G.make_input(200001, 50000, 1), 50000, rank, world)
    case(tg, "index_size_3", G.make_input(1000, 3, 2), 3, rank, world)
    case(tg, "one_key", G.make_input(30000, 1, 3), None, rank, world)
    case(tg, "empty", G.make_input(0, 1, 4), None, rank, world)
    case(tg, "empty_index", G.make_input(0, 1, 4), 5, rank, world)

    # the reference's outputs: this worker's rows are the reference's worker `rank` at p = world
    g = np.load(GOLDEN)
    for k in sorted(g.files):
        if k.endswith("/in") or k.endswith("_counts") or not k.endswith("_p%d" % world):
            continue
        name, rest = k.split("/")
        cname = rest.rsplit("_p", 1)[0]
        size = None if cname.startswith("key_") else int(cname[6:])
        res = case(tg, name, g[name + "/in"].view(G.KV), size, rank, world)
        rows = G.group_rows(res, cname[4:], rank) if size is None else G.index_rows(res, size, world, rank)
        parts = gather(rows, world)
        assert [len(x) for x in parts] == g[k + "_counts"].tolist(), k
        allrows = np.concatenate(parts)
        ref = g[k]
        if ref.dtype == np.uint8:
            assert hashlib.sha256(np.ascontiguousarray(allrows).tobytes()).digest() == ref.tobytes(), k
        else:
            assert np.array_equal(allrows, ref.reshape(-1, 7)), k

    # an index >= size on one worker's shard only: TG_ERR_ARG on every rank
    shard = G.pairs([1, 2, 3], [0, 0, 0]) if rank != 0 else G.pairs([1, 99], [0, 0])
    st, _, _, _ = run(tg, shard, 10)
    assert st == TG_ERR_ARG, st
    st, _, _, _ = run(tg, G.pairs([1, 2], [0, 0]), 10)
    assert st == 0

    # an un-detached ReducePair result (it may lie in this worker's exchange window) as the input
    from thrill_b200 import capi
    local = G.make_input(40000 + 1000 * rank, 5000, 100 + rank)
    d_in = tg.to_device(local)
    rout, rn = C.c_void_p(), C.c_size_t()
    tg.ck(tg.L.tg_reduce_by_key(tg.h, C.byref(capi.KVDesc(16, capi.OP_SUM_U64)), d_in, len(local), C.byref(rout), C.byref(rn)))
    reduced = tg.download(rout.value, rn.value * 16).view(G.KV) if rn.value else np.zeros(0, G.KV)
    out, n = C.c_void_p(), C.c_size_t()
    tg.ck(tg.L.tg_group_by_key(tg.h, rout.value, rn.value, C.byref(out), C.byref(n)))
    res = tg.download(out.value, n.value * 16).view(G.KV) if n.value else np.zeros(0, G.KV)
    shards = gather(reduced, world)
    want = G.grouped(G.exchange(shards, lambda k: G.owner_mod(k, world))[rank])
    assert np.array_equal(res.view(np.uint64), want.view(np.uint64)), ("reduce_result", rank)
    tg.free(d_in)

    tg.barrier()
    if rank == 0:
        print("MULTI_GPU_GROUP_OK world=%d" % world, flush=True)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
