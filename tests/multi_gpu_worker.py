"""Worker of tests/test_gpu_multi.py: one process per GPU (torchrun), runs the collective operators through the
C ABI and checks them against the oracle / golden outputs of the unmodified reference.  Exit code 0 = parity."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch.distributed as dist  # noqa: E402

import oracle_lib as O  # noqa: E402
import reduce_ref as RR  # noqa: E402
import sort_ref as R  # noqa: E402
from golden_util import golden, golden_r2, sha  # noqa: E402
from gpu_util import make_blocks  # noqa: E402
from thrill_b200 import api, capi  # noqa: E402


def gather(arr, world):
    parts = [None] * world
    dist.all_gather_object(parts, np.ascontiguousarray(arr))
    return parts


def sort_records_file(tg, local, d):
    """tg_sort_file of this worker's records (collective) and the fetch of its share of the result"""
    blocks, nb, raw = make_blocks(capi, local, 1 << 16)
    n_out = C.c_size_t()
    tg.ck(tg.L.tg_sort_file(tg.h, C.byref(d.capi()), blocks, nb, 9, C.byref(n_out)))
    out = np.empty((n_out.value, d.item_bytes), dtype=np.uint8)
    ob, onb, _ = make_blocks(capi, out, 1 << 16)
    tg.ck(tg.L.tg_fetch_output(tg.h, ob, onb))
    return out


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    g = golden()

    # ---- Sort: the golden 1e6 uniform case (reference output is independent of the worker count) ----
    n = 1000000
    dia = api.Generate(ctx, n, lambda idx: O.gen_sort_uniform(int(idx[0]) if len(idx) else 0, len(idx)))
    out = dia.Sort()
    parts = gather(out.items, world)
    if rank == 0:
        cat = np.concatenate(parts)
        assert sha(cat) == str(g["sort_uniform_1000000_w4_sha256"]), "sort uniform: differs from the reference"
        sizes = [len(p) for p in parts]
        assert max(sizes) <= 1.25 * n / world + 1000, sizes           # eps = 0.1 balance (api/sort.hpp:298)

    # ---- Sort: Zipf keys (massive duplicates -> splitter tie-break by global index) ----
    cdf = O.zipf_cdf(1024)
    dia = api.Generate(ctx, 50000, lambda idx: O.gen_sort_zipf(int(idx[0]) if len(idx) else 0, len(idx), cdf))
    parts = gather(dia.Sort().items, world)
    if rank == 0:
        cat = np.concatenate(parts)
        assert sha(cat) == str(g["sort_zipf_u1024_50000_w5_sha256"]), "sort zipf: differs from the reference"
        assert max(len(p) for p in parts) <= 2.0 * 50000 / world + 2000      # ties are split across workers

    # ---- Sort: all-equal keys, tiny and empty inputs, everything on one worker ----
    for name, local in (("all_equal", np.ones(10000 // world, dtype=np.uint64)),
                        ("one_item", np.zeros(1 if rank == 0 else 0, dtype=np.uint64)),
                        ("empty", np.zeros(0, dtype=np.uint64)),
                        ("one_worker_has_all", O.gen_sort_uniform(0, 30000) if rank == world - 1 else np.zeros(0, np.uint64))):
        inp = gather(local, world)
        parts = gather(api.DIA(ctx, local).Sort().items, world)
        if rank == 0:
            assert np.array_equal(np.concatenate(parts), np.sort(np.concatenate(inp))), name
            if name == "all_equal" and world > 1:
                assert max(len(p) for p in parts) <= 10000 // world * 2, [len(p) for p in parts]

    # ---- Sort of pairs by key: stable (SortStable contract: equal keys keep global input order) ----
    nloc = 40000
    kv = np.zeros(nloc, dtype=api.KV)
    kv["key"] = np.random.RandomState(rank).randint(0, 100, size=nloc)
    kv["val"] = rank * nloc + np.arange(nloc)                               # global input index
    parts = gather(api.DIA(ctx, kv).SortStable().items, world)
    if rank == 0:
        cat = np.concatenate(parts)
        assert np.all(np.diff(cat["key"].astype(np.int64)) >= 0)
        same = cat["key"][1:] == cat["key"][:-1]
        assert np.all(cat["val"][1:][same] > cat["val"][:-1][same]), "SortStable order violated"

    # ---- Sort of pairs with std::greater (KV + Greater): descending, equal keys in global input order ----
    kv = np.zeros(nloc + 17 * rank, dtype=api.KV)
    kv["key"] = np.random.RandomState(100 + rank).randint(0, 300, size=len(kv)).astype(np.uint64) << np.uint64(40)
    kv["val"] = np.random.RandomState(200 + rank).randint(0, 2**62, size=len(kv))
    inp = gather(kv, world)
    parts = gather(api.DIA(ctx, kv).Sort(api.Greater).items, world)
    if rank == 0:
        cat = np.concatenate(inp)
        want = R.sort(cat, R.Desc(16, 0, 8, R.LE, 1)).view(api.KV).ravel()
        assert np.array_equal(np.concatenate(parts), want), "KV Sort(Greater) differs from the stable descending sort"

    # ---- 4- and 20-byte records: per-worker shares that are not multiples of 16 bytes, so the exchange windows of the
    # record scatter start at unaligned offsets (its word-by-word head and tail run) ----
    for d, nrec in ((R.Desc(4, 1, 3, R.BE), 30001), (R.Desc(20, 5, 12, R.BE), 20003)):
        local = R.make_items(d, nrec + 13 * rank, "few", 300 + rank)
        inp = gather(local, world)
        parts = gather(sort_records_file(ctx.tg, local, d), world)
        if rank == 0:
            assert np.array_equal(np.concatenate(parts), R.sort(np.concatenate(inp), d)), "records " + d.name

    # ---- TeraSort records (100 B, 10-byte key) vs the reference ----
    dia = api.Generate(ctx, 20000, lambda idx: O.gen_records(int(idx[0]) if len(idx) else 0, len(idx)), dtype=None)
    parts = gather(dia.Sort().items, world)
    if rank == 0:
        cat = np.concatenate(parts)
        assert np.array_equal(cat[:8], g["terasort_20000_w3_head"])
        assert sha(cat) == str(g["terasort_20000_w3_sha256"]), "terasort: differs from the reference"

    # ---- round-2 fixtures: TeraSort 1e6 records and 5e6 Zipf(1, 2^20) keys, byte-identical to the reference ----
    g2 = golden_r2()
    dia = api.Generate(ctx, 1000000, lambda idx: O.gen_records(int(idx[0]) if len(idx) else 0, len(idx)), dtype=None)
    parts = gather(dia.Sort().items, world)
    if rank == 0:
        cat = np.concatenate(parts)
        assert np.array_equal(cat[:4], g2["terasort_1000000_head"]) and np.array_equal(cat[-4:], g2["terasort_1000000_tail"])
        assert sha(cat) == str(g2["terasort_1000000_sha256"]), "terasort 1e6: differs from the reference"
        assert max(len(q) for q in parts) <= 1.25 * 1000000 / world + 1000
    cdf = O.zipf_cdf(1 << 20)
    dia = api.Generate(ctx, 5000000, lambda idx: O.gen_sort_zipf(int(idx[0]) if len(idx) else 0, len(idx), cdf))
    parts = gather(dia.Sort().items, world)
    if rank == 0:
        assert sha(np.concatenate(parts)) == str(g2["sort_zipf_u2^20_5000000_sha256"]), "sort zipf 5e6: differs from the reference"
        assert max(len(q) for q in parts) <= 1.3 * 5000000 / world + 1000, [len(q) for q in parts]

    # ---- ReducePair: Zipf f64 sums vs the reference (tolerance) and exact mode (bit-exact), ownership ----
    cdf = O.zipf_cdf(4096)
    for exact, key, tol in ((0, "reduce_f64_zipf_u4096_200000_w3", 1e-9), (1, "reduce_f64_exact_zipf_u4096_200000_w4", 0.0)):
        dia = api.Generate(ctx, 200000, lambda idx: O.gen_reduce_zipf(int(idx[0]) if len(idx) else 0, len(idx), cdf, exact=exact), dtype=None)
        red = api.DIA(ctx, dia.items.view(api.KV)).ReducePair(api.PlusDouble).items
        # every key sits on worker Hash128to64(0,key) % p, as in the reference
        assert np.all(O.hash_partition_ids(red["key"], world) == rank), "key on the wrong worker"
        parts = gather(red, world)
        if rank == 0:
            cat = np.sort(np.concatenate(parts), order="key")
            ref = g[key]
            assert np.array_equal(cat["key"], ref["key"])
            a, b = cat["val"].view(np.float64), ref["val"].view(np.float64)
            if tol:
                assert np.all(np.abs(a - b) <= tol * np.maximum(1.0, np.abs(b)))
            else:
                assert np.array_equal(cat["val"], ref["val"])

    # ---- device-resident collective at scale: 2e7 keys per GPU, properties ----
    tg = ctx.tg
    n = 20000000
    d = tg.alloc(n * 8)
    tg.ck(tg.L.tg_gen_sort_uniform(tg.h, d, rank * n, n, 42))
    before = tg.checksum(d, n, 8)
    op, on = C.c_void_p(), C.c_size_t()
    tg.ck(tg.L.tg_sort(tg.h, C.byref(capi.u64_desc()), d, n, 3, C.byref(op), C.byref(on)))
    assert tg.is_sorted(capi.u64_desc(), op.value, on.value)
    after = tg.checksum(op.value, on.value, 8)
    first_last = tg.download(op.value, 8, np.uint64)[0], tg.download(op.value + (on.value - 1) * 8, 8, np.uint64)[0]
    allv = gather(np.array([before[0], before[1], after[0], after[1], on.value, first_last[0], first_last[1]], dtype=np.uint64), world)
    if rank == 0:
        m = np.stack(allv)
        assert int(m[:, 4].sum()) == n * world
        assert np.uint64(np.sum(m[:, 0], dtype=np.uint64)) == np.uint64(np.sum(m[:, 2], dtype=np.uint64))      # multiset sum
        assert np.bitwise_xor.reduce(m[:, 1]) == np.bitwise_xor.reduce(m[:, 3])                                 # multiset xor
        assert all(m[r, 6] <= m[r + 1, 5] for r in range(world - 1))                                            # ranges ordered
    tg.free(d)

    # ---- ReduceByKey above the threshold of the partitioned aggregation (pre phase, exchange, post phase): exact sums ----
    nr, U = 3000000, 1 << 20
    cdf = O.zipf_cdf(U)
    d_cdf = tg.to_device(cdf)
    d = tg.alloc(nr * 16)
    tg.ck(tg.L.tg_gen_reduce_zipf(tg.h, d, rank * nr, nr, 42, d_cdf, U, 1))
    rp, rc = C.c_void_p(), C.c_size_t()
    tg.ck(tg.L.tg_reduce_by_key(tg.h, C.byref(capi.KVDesc(16, capi.OP_SUM_F64)), d, nr, C.byref(rp), C.byref(rc)))
    red = tg.download(rp.value, rc.value * 16, O.KV)
    assert np.all(O.hash_partition_ids(red["key"], world) == rank), "key on the wrong worker"
    parts = gather(red, world)
    if rank == 0:
        cat = np.sort(np.concatenate(parts), order="key")
        ref = O.reduce_simple(O.gen_reduce_zipf(0, nr * world, cdf, exact=1), O.OP_SUM_F64)
        assert np.array_equal(cat, ref), "large ReduceByKey differs from the oracle"
    tg.free(d); tg.free(d_cdf)

    # ---- special values of one key split across the workers: the pre phase's partial aggregates of a key must fold into
    # the contract's result in the post phase (reduce_ref.check), below and above the partitioned aggregation's threshold ----
    inf, m0 = np.float64(np.inf).view(np.uint64), np.uint64(0x8000000000000000)
    split = [(1, [m0] * 3),                                                      # -0.0 on every worker
             (2, [m0] if rank == 0 else []),                                     # a lone -0.0 on one worker
             (3, [np.uint64(RR.NAN_PAYLOADS[1])] if rank == 0 else list(np.array([rank, -rank], np.float64).view(np.uint64))),
             (4, [np.uint64(RR.NAN_PAYLOADS[rank % len(RR.NAN_PAYLOADS)])]),     # NaN everywhere, payloads differ
             (5, [inf] if rank == 0 else [inf ^ np.uint64(1 << 63)] if rank == world - 1 else [])]     # +inf and -inf
    sk = np.concatenate([np.full(len(v), k, np.uint64) for k, v in split])
    sv = np.array([x for _, v in split for x in v], dtype=np.uint64)
    for nloc in (5000, 300000):
        keys = np.random.default_rng(700 + rank).integers(1000, 1 << 40, size=nloc).astype(np.uint64)
        for op, mix in (("sum_f64", "f64_special"), ("min_f64", "f64_special"), ("max_f64", "f64_special"), ("first", "u64"),
                        ("sum_u64", "u64")):
            kv = np.zeros(nloc + len(sk), dtype=O.KV)
            kv["key"] = np.r_[keys, sk]
            kv["val"] = np.r_[RR.gen_values(mix, keys, 900 + rank), sv]
            d = tg.to_device(kv)
            rp, rc = C.c_void_p(), C.c_size_t()
            tg.ck(tg.L.tg_reduce_by_key(tg.h, C.byref(capi.KVDesc(16, RR.OPS.index(op))), d, len(kv), C.byref(rp), C.byref(rc)))
            red = tg.download(rp.value, rc.value * 16, O.KV)
            tg.free(d)
            assert np.all(O.hash_partition_ids(red["key"], world) == rank), "key on the wrong worker"
            ins, outs = gather(kv, world), gather(red, world)
            if rank == 0:
                RR.check(np.concatenate(ins), np.concatenate(outs), op)

    # ---- ReduceToIndex (PageRank step): the concatenation over the workers is the dense array of the reference ----
    cdf = O.zipf_cdf(1000)
    dia = api.Generate(ctx, 20000, lambda idx: O.gen_reduce_zipf(int(idx[0]) if len(idx) else 0, len(idx), cdf, exact=1), dtype=None)
    kv = dia.items.view(api.KV).copy()
    kv["key"] %= 1000
    red = api.DIA(ctx, kv).ReduceToIndex(api.KeyIsFirst, api.PlusDouble, 1000)
    assert red.index_begin == (rank * 1000 + world - 1) // world
    parts = gather(red.items, world)
    if rank == 0:
        assert np.array_equal(np.concatenate(parts), g["reduce_to_index_zipf_u1000_20000_exact1_w3"]), "ReduceToIndex differs from the reference"

    # ---- the item limit: one worker holds 2^30 records (a real buffer), the others a few; every rank gets TG_ERR_TOO_LARGE
    # and nobody is left waiting in a collective.  Then the ctx still reduces. ----
    big = rank == world - 1
    n_local = (1 << 30) if big else 1000
    d = tg.alloc(n_local * 16)
    tg.upload(d, np.zeros(2 * min(n_local, 1000), dtype=np.uint64))
    kvd = capi.KVDesc(16, capi.OP_SUM_U64)
    rp, rc, rb = C.c_void_p(), C.c_size_t(), C.c_uint64()
    neutral = np.zeros(2, dtype=np.uint64)
    for name, call in (("reduce_by_key", lambda: tg.L.tg_reduce_by_key(tg.h, C.byref(kvd), d, n_local, C.byref(rp), C.byref(rc))),
                       ("reduce_to_index", lambda: tg.L.tg_reduce_to_index(tg.h, C.byref(kvd), d, n_local, 1 << 20, neutral.ctypes.data,
                                                                           C.byref(rp), C.byref(rc), C.byref(rb)))):
        st = call()
        assert st == -4, "%s: rank %d (n_local %d) returned %d, expected TG_ERR_TOO_LARGE on every rank" % (name, rank, n_local, st)
    tg.free(d)
    kv = np.zeros(1000, dtype=O.KV)
    kv["key"] = np.arange(1000) % 7
    kv["val"] = 1
    d = tg.to_device(kv)
    tg.ck(tg.L.tg_reduce_by_key(tg.h, C.byref(kvd), d, len(kv), C.byref(rp), C.byref(rc)))
    red = tg.download(rp.value, rc.value * 16, O.KV)
    tg.free(d)
    outs = gather(red, world)
    if rank == 0:
        cat = np.concatenate(outs)
        assert np.array_equal(np.sort(cat["key"]), np.arange(7)) and int(cat["val"].sum()) == 1000 * world
    dist.barrier()
    ctx.close()
    if rank == 0:
        print("MULTI_GPU_PARITY_OK world=%d" % world)


if __name__ == "__main__":
    main()
