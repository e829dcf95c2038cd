"""Worker of test_gpu_join.py::test_join_on_n_gpus: one process per GPU (torchrun), runs tg_inner_join over sides sharded
across the workers and checks every worker's exact result against join_ref, and the concatenation's multiset against the
reference's outputs in tests/golden/reference_outputs_join.npz where that file is present.  Exit code 0 and
MULTI_GPU_JOIN_OK = parity."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch.distributed as dist  # noqa: E402

import join_ref as J  # noqa: E402
from thrill_b200 import api, capi  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "reference_outputs_join.npz")
TG_ERR_TOO_LARGE = -4


def gather(arr, world):
    parts = [None] * world
    dist.all_gather_object(parts, np.ascontiguousarray(arr))
    return parts


def join_shards(tg, fn, dl, nl, dr, nr):
    out, n = C.c_void_p(), C.c_size_t()
    st = tg.L.tg_inner_join(tg.h, C.byref(capi.JoinDesc(16, fn)), dl, nl, dr, nr, C.byref(out), C.byref(n))
    if st != 0:
        return st, None
    dt = J.out_dtype(fn)
    return 0, (tg.download(out.value, n.value * dt.itemsize).view(dt) if n.value else np.zeros(0, dt))


def case(tg, name, left, right, fn, rank, world):
    """left, right: the global sides (the same on every worker), split evenly into shards"""
    lefts, rights = J.split_shards(left, world), J.split_shards(right, world)
    dl, dr = tg.to_device(lefts[rank]), tg.to_device(rights[rank])
    st, out = join_shards(tg, fn, dl, len(lefts[rank]), dr, len(rights[rank]))
    tg.free(dl)
    tg.free(dr)
    assert st == 0, (name, st, tg.L.tg_last_error(tg.h))
    want = J.join(lefts, rights, fn)[rank]
    assert np.array_equal(out.view(np.uint64), want.view(np.uint64)), (name, rank, len(out), len(want))
    parts = gather(out, world)
    if rank == 0:
        print("join %s: %d outputs over %d workers ok" % (name, sum(len(x) for x in parts), world), flush=True)
    return parts


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    tg = ctx.tg
    for fn in (J.KEY_VALUES, J.VALUES):
        case(tg, "uniform_%d" % fn, J.make_side(200000, 50000, 1), J.make_side(150001, 50000, 2), fn, rank, world)
        case(tg, "zipf_%d" % fn, J.make_side(60000, 3000, 3, zipf=1.0), J.make_side(50000, 3000, 4, zipf=1.0), fn, rank, world)
        case(tg, "one_key_%d" % fn, J.make_side(3000, 1, 5), J.make_side(2000, 1, 6), fn, rank, world)
        case(tg, "empty_right_%d" % fn, J.make_side(5000, 10, 7), J.make_side(0, 10, 8), fn, rank, world)
        case(tg, "tiny_%d" % fn, J.make_side(1, 1, 9), J.make_side(1, 1, 10), fn, rank, world)

    # the reference's outputs: the concatenation of the workers' results has the stored multiset
    if os.path.exists(GOLDEN):
        g = np.load(GOLDEN)
        for name in sorted({k.split("/")[0] for k in g.files}):
            parts = case(tg, "golden_" + name, g[name + "/left"].view(J.KV), g[name + "/right"].view(J.KV), J.KEY_VALUES,
                         rank, world)
            ref_keys = [k for k in g.files if k.startswith(name + "/out_p") and g[k].dtype != np.uint8]
            if rank == 0 and ref_keys:
                rows = np.concatenate(parts).view(np.uint64).reshape(-1, 3)
                rows = rows[np.lexsort(rows.T[::-1])]
                for k in ref_keys:
                    assert np.array_equal(rows, g[k].reshape(-1, 3)), k

    # an output over the limit on the worker that owns the hot key: TG_ERR_TOO_LARGE on every rank
    a, b = np.zeros(40000, J.KV), np.zeros(30000, J.KV)
    a["key"], b["key"] = 5, 5
    la, lb = J.split_shards(a, world)[rank], J.split_shards(b, world)[rank]
    dl, dr = tg.to_device(la), tg.to_device(lb)
    st, _ = join_shards(tg, J.VALUES, dl, len(la), dr, len(lb))
    assert st == TG_ERR_TOO_LARGE, st
    tg.free(dl)
    tg.free(dr)

    # an un-detached ReducePair result (it may lie in this worker's exchange window) as both sides: a self-join
    local = J.make_side(40000 + 10000 * rank, 5000, 100 + rank)
    d_in = tg.to_device(local)
    rout, rn = C.c_void_p(), C.c_size_t()
    tg.ck(tg.L.tg_reduce_by_key(tg.h, C.byref(capi.KVDesc(16, capi.OP_SUM_U64)), d_in, len(local), C.byref(rout), C.byref(rn)))
    reduced = tg.download(rout.value, rn.value * 16).view(J.KV) if rn.value else np.zeros(0, J.KV)
    st, out = join_shards(tg, J.KEY_VALUES, rout.value, rn.value, rout.value, rn.value)
    assert st == 0, tg.L.tg_last_error(tg.h)
    shards = gather(reduced, world)
    want = J.join(shards, shards, J.KEY_VALUES)[rank]
    assert np.array_equal(out.view(np.uint64), want.view(np.uint64)), ("reduce_result_self_join", rank)
    tg.free(d_in)

    tg.barrier()
    if rank == 0:
        print("MULTI_GPU_JOIN_OK world=%d" % world, flush=True)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
