"""ReduceByKey on records (tg_reduce_by_key_records, its _file form and the Python mirror) on one H100, bit for bit against the
numpy model in reduce_records_ref.py: item sizes 4..1024, keys of 1..8 bytes at aligned and unaligned offsets, every op on
several runs, random payload bytes, special values under the reduce_ref contract, the tile edges of every tile size, double sums
within the stated bound and reproducible, File forms and chaining, the argument errors and the limit, agreement with the pair
reduce, and simulated workers (the operator's p > 1 path step for step).  pytest -m gpu."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import reduce_ref
import reduce_records_ref as RR
import join_records_ref as J
from gpu_util import make_blocks

pytestmark = pytest.mark.gpu
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4
U = 2.0 ** -53
SUM_F64, SUM_U64, MIN_U64, MAX_U64, MIN_F64, MAX_F64 = range(6)


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(0)
    yield c
    c.close()


def desc(s, key, runs):
    return _capi().reduce_records_desc(s, key[0], key[1], runs)


def reduce_raw(ctx, dp, n, s, key, runs):
    """tg_reduce_by_key_records on a device pointer: (status, output pointer, output count)"""
    out, m = C.c_void_p(), C.c_size_t()
    st = ctx.L.tg_reduce_by_key_records(ctx.h, C.byref(desc(s, key, runs)), dp, n, C.byref(out), C.byref(m))
    return st, out.value, m.value


def reduce_dev(ctx, rec, key, runs, s=None):
    """tg_reduce_by_key_records of a host record array on one worker: (status, result rows)"""
    s = rec.shape[1] if s is None else s
    dp = ctx.to_device(rec)
    st, o, m = reduce_raw(ctx, dp, len(rec), s, key, runs)
    res = None
    if st == 0:
        res = ctx.download(o, m * s).reshape(-1, s) if m else np.zeros((0, s), np.uint8)
    ctx.free(dp)
    return st, res


def check(ctx, rec, key, runs):
    st, res = reduce_dev(ctx, rec, key, runs)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    ref = RR.reduce_local(rec, key, runs)
    assert res.shape == ref.shape
    assert np.array_equal(res, ref)
    return res


def records(n, s, key, keys, runs, seed, exact=True):
    rec = RR.make(n, s, key, keys, seed)
    for j, (off, cnt, op) in enumerate(runs):
        RR.set_fields(rec, off, cnt, RR.values(op, n, cnt, seed * 13 + j, exact=exact))
    return rec


def tile_items(runs):
    """the tile size T of the segmented reduce for these runs"""
    f = sum(c for _, c, _ in runs)
    return 2048 if f == 0 else min(2048, 1 << int(math.floor(math.log2(4096 // f))))


# ---- shapes: item sizes, keys, runs ----------------------------------------------------------------------------------------
# (item bytes, key (offset, bytes), runs)
SHAPES = [
    (4, (0, 4), []),                                             # key-only items
    (4, (1, 2), []),
    (12, (0, 4), [(4, 1, SUM_U64)]),                             # a field at an offset that is not a multiple of 8
    (16, (0, 8), [(8, 1, SUM_F64)]),                             # the pair shape
    (40, (0, 8), [(8, 3, SUM_F64), (32, 1, SUM_U64)]),           # k-means, D = 3
    (40, (0, 8), [(32, 1, SUM_U64)]),                            # its count-only second reduce
    (36, (32, 3), [(0, 2, MIN_F64), (16, 2, MAX_F64)]),
    (56, (13, 5), [(0, 1, MIN_U64), (20, 2, MAX_U64), (40, 2, SUM_F64)]),
    (176, (3, 1), [(8, 2, SUM_U64), (24, 3, SUM_F64), (56, 1, MIN_U64), (64, 4, MAX_F64)]),   # line items
    (100, (99, 1), [(0, 12, SUM_F64)]),
    (328, (0, 8), [(8, 8, SUM_U64), (80, 8, SUM_F64), (152, 8, MIN_F64), (224, 8, MAX_U64), (296, 2, MIN_U64),
                   (312, 1, MAX_F64), (320, 1, SUM_U64), (72, 1, SUM_F64)]),                    # 8 runs, 37 fields
    (1024, (1016, 8), [(0, 127, SUM_U64)]),                      # the most fields: T = 32
    (1024, (0, 1), [(4, 64, SUM_F64), (520, 62, MAX_U64)]),
    (516, (512, 4), [(0, 16, MIN_F64), (256, 16, SUM_U64)]),
]


@pytest.mark.parametrize("s,key,runs", SHAPES, ids=["%d_k%d_%d_f%d" % (s, k[0], k[1], sum(c for _, c, _ in r)) for s, k, r in SHAPES])
def test_shapes(ctx, s, key, runs):
    rng = np.random.default_rng(s + key[0])
    for n, distinct in [(1, 1), (777, 40), (20000, 3000), (60000, 17)]:
        keys = rng.integers(0, min(distinct, 1 << (8 * key[1])), size=n, dtype=np.uint64)
        check(ctx, records(n, s, key, keys, runs, seed=n + s), key, runs)


@pytest.mark.parametrize("kb", range(1, 9))
@pytest.mark.parametrize("off", [0, 1, 3, 5])
def test_key_widths_and_offsets(ctx, kb, off):
    s = 32
    runs = [(16, 2, SUM_U64)]
    key = (off, kb)
    keys = np.random.default_rng(kb * 10 + off).integers(0, 1 << min(8 * kb, 20), size=30000, dtype=np.uint64)
    if kb == 8:
        keys |= np.uint64(0xF0F0F0F000000000)                   # keys beyond 32 bits
    check(ctx, records(30000, s, key, keys, runs, seed=kb), key, runs)


@pytest.mark.parametrize("op", range(6))
def test_every_op_on_several_runs(ctx, op):
    s, key = 72, (64, 8)
    runs = [(0, 2, op), (16, 1, op), (28, 4, op)]
    keys = np.random.default_rng(op).integers(0, 2000, size=100000, dtype=np.uint64)
    check(ctx, records(100000, s, key, keys, runs, seed=op), key, runs)


@pytest.mark.parametrize("op", [SUM_F64, MIN_F64, MAX_F64])
def test_special_values(ctx, op):
    """±0, NaN payloads, ±inf, subnormals and huge values: the reduce_ref contract per field"""
    s, key = 48, (0, 8)
    runs = [(8, 2, op), (32, 2, op)]
    n = 50000
    keys = np.random.default_rng(7 + op).integers(0, 3000, size=n, dtype=np.uint64)
    rec = RR.make(n, s, key, keys, seed=9)
    for j, (off, cnt, _) in enumerate(runs):
        RR.set_fields(rec, off, cnt, np.stack([reduce_ref.gen_values("f64_special", keys, 100 * op + 10 * j + c) for c in range(cnt)], 1))
    st, res = reduce_dev(ctx, rec, key, runs)
    assert st == 0
    RR.check(rec, res, key, runs)
    if op != SUM_F64:                                            # min / max: the model's pick exactly
        assert np.array_equal(res, RR.reduce_local(rec, key, runs))


# ---- tile edges ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("runs", [[], [(8, 1, SUM_U64)], [(8, 2, SUM_U64)], [(8, 4, MAX_U64)], [(8, 9, SUM_F64)], [(8, 100, SUM_U64)]],
                         ids=lambda r: "f%d" % sum(c for _, c, _ in r))
@pytest.mark.parametrize("kind", ["on_edges", "one_key", "alternating", "distinct", "runs_of_tile_minus_one", "zipf"])
def test_tile_edges(ctx, runs, kind):
    s = 8 + 8 * sum(c for _, c, _ in runs)
    key = (0, 8)
    T = tile_items(runs)
    n = 7 * T + 5 if kind != "zipf" else 40 * T + 3
    i = np.arange(n, dtype=np.uint64)
    if kind == "on_edges":
        keys = i // np.uint64(T)                                 # every group ends exactly on a tile edge
    elif kind == "one_key":
        keys = np.full(n, 42, np.uint64)                         # one key spanning every tile
    elif kind == "alternating":
        keys = i % np.uint64(2)
    elif kind == "distinct":
        keys = np.random.default_rng(1).permutation(n).astype(np.uint64)
    elif kind == "runs_of_tile_minus_one":
        keys = i // np.uint64(max(T - 1, 1))
    else:
        keys = J.zipf_keys(n, 1000, 1.2, 5)
    check(ctx, records(n, s, key, keys, runs, seed=n), key, runs)


@pytest.mark.parametrize("n", [0, 1, 2, 31, 32, 33, 1023, 1024, 1025, 2047, 2048, 2049, 4097, 100003, 3000017])
def test_sizes(ctx, n):
    s, key = 40, (0, 8)
    runs = [(8, 3, SUM_F64), (32, 1, SUM_U64)]
    keys = np.random.default_rng(n).integers(0, max(1, n // 3), size=n, dtype=np.uint64)
    check(ctx, records(n, s, key, keys, runs, seed=n), key, runs)


def test_group_spanning_many_tiles_with_neighbours(ctx):
    """a 2e6-item key between small groups: cut groups of one piece and of thousands of pieces in one call"""
    s, key = 24, (0, 8)
    runs = [(8, 1, SUM_U64), (16, 1, MAX_U64)]
    keys = np.concatenate([np.arange(5000, dtype=np.uint64), np.full(2000000, 5000, np.uint64), 5001 + np.arange(7000, dtype=np.uint64) // 3])
    keys = keys[np.random.default_rng(2).permutation(len(keys))]
    check(ctx, records(len(keys), s, key, keys, runs, seed=3), key, runs)


# ---- double sums ----------------------------------------------------------------------------------------------------------------
def _chain_bound(n, runs):
    """D of one local reduce of n records (include/thrill_gpu.h)"""
    T = tile_items(runs)
    t = (n + T - 1) // T
    return 32 + (t + 255) // 256


@pytest.mark.parametrize("n,distinct", [(200000, 10), (1000000, 1), (1000000, 1000)])
def test_double_sums_within_the_bound_and_reproducible(ctx, n, distinct):
    s, key = 40, (0, 8)
    runs = [(8, 3, SUM_F64)]
    rng = np.random.default_rng(n + distinct)
    keys = rng.integers(0, distinct, size=n, dtype=np.uint64)
    rec = RR.make(n, s, key, keys, seed=4)
    vals = np.ldexp(rng.random((n, 3)) - 0.3, rng.integers(-30, 31, size=(n, 3)))
    RR.set_fields(rec, 8, 3, vals.view(np.uint64))
    st, res = reduce_dev(ctx, rec, key, runs)
    assert st == 0
    st2, res2 = reduce_dev(ctx, rec, key, runs)
    assert st2 == 0 and np.array_equal(res, res2)              # the same bytes on a second call
    D = _chain_bound(n, runs)
    gamma = D * U / (1 - D * U)
    order = np.argsort(keys, kind="stable")
    ks = keys[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    ends = np.r_[starts[1:], n]
    got = RR.fields(res, 8, 3).view(np.float64)
    for g, (a, b) in enumerate(zip(starts, ends)):
        xs = vals[order[a:b]]
        for j in range(3):
            exact = math.fsum(xs[:, j])
            tol = gamma * math.fsum(np.abs(xs[:, j])) + U * abs(exact)
            assert abs(got[g, j] - exact) <= tol, (g, j, got[g, j], exact, tol)


# ---- File forms, chaining, inputs left intact --------------------------------------------------------------------------------
def _fetch(ctx, n, s):
    capi = _capi()
    out = np.empty(n * s, np.uint8)
    blocks, nb, _ = make_blocks(capi, out, 1 << 16)
    ctx.ck(ctx.L.tg_fetch_output(ctx.h, blocks, nb))
    return out.reshape(n, s)


def test_file_host_and_device(ctx):
    capi = _capi()
    s, key = 40, (0, 8)
    runs = [(8, 3, SUM_F64), (32, 1, SUM_U64)]
    keys = np.random.default_rng(8).integers(0, 900, size=50000, dtype=np.uint64)
    rec = records(50000, s, key, keys, runs, seed=8)
    ref = RR.reduce_local(rec, key, runs)
    d = desc(s, key, runs)
    n = C.c_size_t()
    # host Blocks that cut items
    blocks, nb, raw = make_blocks(capi, rec, 1000 + 37)
    inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
    ctx.ck(ctx.L.tg_reduce_by_key_records_file(ctx.h, C.byref(d), C.byref(inp), C.byref(n)))
    assert np.array_equal(_fetch(ctx, n.value, s), ref)
    # a device File, read in place and left intact; no PCIe traffic
    dp = ctx.to_device(rec)
    before = ctx.checksum(dp, len(rec), s)
    f = capi.DevFile(dp, len(rec), s, 0)
    inp = capi.MergeInput(C.pointer(f), None, 0)
    h0, d0 = C.c_uint64(), C.c_uint64()
    ctx.L.tg_transfer_bytes(ctx.h, C.byref(h0), C.byref(d0))
    ctx.ck(ctx.L.tg_reduce_by_key_records_file(ctx.h, C.byref(d), C.byref(inp), C.byref(n)))
    h1, d1 = C.c_uint64(), C.c_uint64()
    ctx.L.tg_transfer_bytes(ctx.h, C.byref(h1), C.byref(d1))
    assert (h1.value, d1.value) == (h0.value, d0.value)
    out = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(out)))
    assert out.item_bytes == s and out.items == len(ref)
    assert np.array_equal(ctx.download(out.dptr, out.items * s).reshape(-1, s), ref)
    assert ctx.checksum(dp, len(rec), s) == before
    # the detached result reduced again (its count field only): the same rows
    inp2 = capi.MergeInput(C.pointer(out), None, 0)
    ctx.ck(ctx.L.tg_reduce_by_key_records_file(ctx.h, C.byref(desc(s, key, [(32, 1, SUM_U64)])), C.byref(inp2), C.byref(n)))
    assert np.array_equal(_fetch(ctx, n.value, s), ref)
    ctx.L.tg_dev_file_free(ctx.h, C.byref(out))
    ctx.free(dp)


def test_undetached_results_as_inputs(ctx):
    """the un-detached result of an earlier reduce on records (in this operator's output slot) and of a records join"""
    s, key = 24, (0, 8)
    runs = [(8, 1, SUM_U64), (16, 1, MIN_U64)]
    keys = np.random.default_rng(12).integers(0, 5000, size=40000, dtype=np.uint64)
    rec = records(40000, s, key, keys, runs, seed=12)
    dp = ctx.to_device(rec)
    st, o, m = reduce_raw(ctx, dp, len(rec), s, key, runs)
    assert st == 0
    first = RR.reduce_local(rec, key, runs)
    # reduce the un-detached result by a coarser key (its low 1 byte)
    k2 = (0, 1)
    st, o2, m2 = reduce_raw(ctx, o, m, s, k2, runs)
    assert st == 0
    assert np.array_equal(ctx.download(o2, m2 * s).reshape(-1, s), RR.reduce_local(first, k2, runs))
    # a records join's result (left 24 + right 16 bytes) reduced on the left key, summing the right record's second word
    right = J.set_keys(J.make_records(3000, 16, 5), 0, 8, np.random.default_rng(13).integers(0, 5000, 3000, dtype=np.uint64))
    dr = ctx.to_device(right)
    jd = _capi().JoinRecordsDesc(24, 16, 0, 8, 0, 8)
    jo, jn = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_inner_join_records(ctx.h, C.byref(jd), dp, len(rec), dr, len(right), C.byref(jo), C.byref(jn)))
    joined = J.join_local(rec, right, (0, 8), (0, 8))
    jr = [(8, 1, SUM_U64), (32, 1, SUM_U64)]
    st, o3, m3 = reduce_raw(ctx, jo.value, jn.value, 40, (0, 8), jr)
    assert st == 0
    assert np.array_equal(ctx.download(o3, m3 * 40).reshape(-1, 40), RR.reduce_local(joined, (0, 8), jr))
    ctx.free(dp)
    ctx.free(dr)


def test_python_mirror():
    from thrill_b200 import api, capi
    c = api.Context(rank=0, nranks=1, device=0, rng_seed=3)
    try:
        s, key = 40, (0, 8)
        runs = [(8, 3, SUM_F64), (32, 1, SUM_U64)]
        keys = np.random.default_rng(21).integers(0, 500, size=30000, dtype=np.uint64)
        rec = records(30000, s, key, keys, runs, seed=21)
        cc3 = np.dtype([("cluster_id", "<u8"), ("p", "<f8", (3,)), ("count", "<u8")])
        out = api.DIA(c, rec.view(cc3).reshape(-1)).ReduceByKey(
            api.KeyField(0, 8), api.FieldReduce([(8, 3, api.PlusDouble), (32, 1, api.PlusU64)]))
        assert out.items.dtype == cc3
        assert np.array_equal(out.items.view(np.uint8).reshape(-1, s), RR.reduce_local(rec, key, runs))
        pv = rec[:, :16].copy()
        out = api.DIA(c, pv.view(np.dtype((np.void, 16))).reshape(-1)).ReduceByKey(api.KeyIsFirst, api.FieldReduce([(8, 1, api.MaxDouble)]))
        assert np.array_equal(out.items.view(np.uint8).reshape(-1, 16), RR.reduce_local(pv, (0, 8), [(8, 1, MAX_F64)]))
        with pytest.raises(capi.ThrillGpuError):
            api.FieldReduce([(8, 1, api.First)])
        with pytest.raises(capi.ThrillGpuError):                 # a run over the key
            api.DIA(c, rec.view(cc3).reshape(-1)).ReduceByKey(api.KeyField(0, 8), api.FieldReduce([(0, 1, api.PlusU64)]))
        # the pair ReduceByKey is unchanged
        kv = rec[:, :16].copy().view(api.KV).reshape(-1)
        a = api.DIA(c, kv).ReduceByKey(api.KeyIsFirst, api.PlusU64).items
        assert len(a) == len(np.unique(kv["key"]))
    finally:
        c.close()


# ---- agreement with the pair reduce -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", range(6))
def test_pairs_agree_with_the_pair_reduce(ctx, op):
    capi = _capi()
    n = 300000
    rng = np.random.default_rng(40 + op)
    keys = rng.integers(0, 20000, size=n, dtype=np.uint64)
    rec = RR.make(n, 16, (0, 8), keys, 40)
    RR.set_fields(rec, 8, 1, RR.values(op, n, 1, 40 + op, exact=True))
    st, res = reduce_dev(ctx, rec, (0, 8), [(8, 1, op)])
    assert st == 0
    dp = ctx.to_device(rec)
    out, m = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_reduce_by_key(ctx.h, C.byref(capi.KVDesc(16, op)), dp, n, C.byref(out), C.byref(m)))
    pair = ctx.download(out.value, m.value * 16).reshape(-1, 16)
    pair = pair[np.argsort(pair[:, :8].copy().view("<u8").reshape(-1), kind="stable")]
    ctx.free(dp)
    if op in (MIN_F64, MAX_F64):                                 # equal zeros: each path keeps one of them
        assert np.array_equal(res[:, :8], pair[:, :8])
        assert np.array_equal(res[:, 8:].copy().view(np.float64), pair[:, 8:].copy().view(np.float64))
    else:
        assert np.array_equal(res, pair)


# ---- errors and the limits ----------------------------------------------------------------------------------------------------
def test_argument_errors(ctx):
    capi = _capi()
    a = records(3, 40, (0, 8), np.arange(3, dtype=np.uint64), [], 1)
    ok = [(8, 3, SUM_F64)]
    bad = [
        (0, (0, 1), []), (22, (0, 8), []), (1028, (0, 8), []), (40, (0, 0), []), (40, (0, 9), []), (40, (36, 8), []),
        (40, (0, 8), [(8, 0, SUM_F64)]),                         # a count of 0
        (40, (0, 8), [(8, 1, 6)]), (40, (0, 8), [(8, 1, 99)]),   # an op outside the six (TG_OP_FIRST included)
        (40, (0, 8), [(10, 1, SUM_U64)]),                        # an offset that is not a multiple of 4
        (40, (0, 8), [(8, 5, SUM_U64)]), (40, (0, 8), [(36, 1, SUM_U64)]), (40, (0, 8), [(1 << 31, 1, SUM_U64)]),
        (40, (0, 8), [(8, 1 << 30, SUM_U64)]),                   # runs outside the item
        (40, (0, 8), [(4, 1, SUM_U64)]), (40, (12, 2), [(8, 2, SUM_U64)]), (40, (39, 1), [(32, 1, SUM_U64)]),    # over the key
        (40, (0, 8), [(8, 2, SUM_U64), (16, 1, MIN_U64)]), (40, (0, 8), [(24, 2, SUM_U64), (8, 3, MIN_U64)]),    # overlapping runs
    ]
    for s, key, runs in bad:
        assert reduce_dev(ctx, a, key, runs, s=s)[0] == TG_ERR_ARG, (s, key, runs)
    d = capi.reduce_records_desc(40, 0, 8, ok)
    d.nruns = 9                                                  # more than 8 runs
    out, m = C.c_void_p(), C.c_size_t()
    dp = ctx.to_device(a)
    assert ctx.L.tg_reduce_by_key_records(ctx.h, C.byref(d), dp, 3, C.byref(out), C.byref(m)) == TG_ERR_ARG
    d = desc(40, (0, 8), ok)
    assert ctx.L.tg_reduce_by_key_records(ctx.h, C.byref(d), None, 3, C.byref(out), C.byref(m)) == TG_ERR_ARG
    assert ctx.L.tg_reduce_by_key_records(ctx.h, C.byref(d), dp + 2, 1, C.byref(out), C.byref(m)) == TG_ERR_ARG   # misaligned
    n = C.c_size_t()
    f = capi.DevFile(dp, 3, 16, 0)                               # a device File of another item size
    inp = capi.MergeInput(C.pointer(f), None, 0)
    assert ctx.L.tg_reduce_by_key_records_file(ctx.h, C.byref(d), C.byref(inp), C.byref(n)) == TG_ERR_ARG
    blocks, nb, raw = make_blocks(capi, np.zeros(60, np.uint8), 60)     # 60 bytes: not whole 40-byte items
    inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
    assert ctx.L.tg_reduce_by_key_records_file(ctx.h, C.byref(d), C.byref(inp), C.byref(n)) == TG_ERR_ARG
    ctx.free(dp)
    check(ctx, a, (0, 8), ok)                                    # the ctx still works


def test_input_over_the_limit_is_too_large(ctx):
    """refused before anything is read or allocated"""
    dp = ctx.to_device(np.zeros(64, np.uint8))
    assert reduce_raw(ctx, dp, 1 << 30, 40, (0, 8), [(8, 3, SUM_F64)])[0] == TG_ERR_TOO_LARGE
    assert reduce_raw(ctx, dp, (1 << 30) - 1 + (1 << 40), 4, (0, 4), [])[0] == TG_ERR_TOO_LARGE
    ctx.free(dp)
    # a host File of 2^30 items (one Block that claims 4 GiB over a small buffer): refused before it is uploaded
    capi = _capi()
    small = np.zeros(64, np.uint8)
    blocks = (capi.Block * 1)()
    blocks[0].data, blocks[0].bytes = small.ctypes.data, 4 << 30
    inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), 1)
    n = C.c_size_t()
    d = desc(4, (0, 4), [])
    assert ctx.L.tg_reduce_by_key_records_file(ctx.h, C.byref(d), C.byref(inp), C.byref(n)) == TG_ERR_TOO_LARGE
    check(ctx, np.arange(40, dtype=np.uint32).view(np.uint8).reshape(-1, 4), (0, 4), [])     # the ctx still works


# ---- simulated workers ---------------------------------------------------------------------------------------------------------
def _select(ctx, mode, shards, key, p):
    """tg_exchange_records_select: the windows' contents"""
    s = shards[0].shape[1]
    dsh = [ctx.to_device(x) if len(x) else None for x in shards]
    counts = (C.c_uint64 * (p * p))()
    sh_arr = (C.c_void_p * p)(*dsh)
    n_arr = (C.c_size_t * p)(*[len(x) for x in shards])
    ctx.ck(ctx.L.tg_exchange_records_select(ctx.h, 0, s, key[0], key[1], sh_arr, n_arr, p, None, None, counts))
    recv = [sum(counts[src * p + d] for src in range(p)) for d in range(p)]
    wins = [ctx.alloc(max(16, r * s)) for r in recv]
    win = (C.c_void_p * p)(*wins)
    wb = (C.c_size_t * p)(*[r * s for r in recv])
    ctx.ck(ctx.L.tg_exchange_records_select(ctx.h, mode, s, key[0], key[1], sh_arr, n_arr, p, win, wb, counts))
    out = [ctx.download(w, r * s).reshape(-1, s) for w, r in zip(wins, recv)]
    for x in dsh + wins:
        if x:
            ctx.free(x)
    return out


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("p", [1, 2, 3, 4, 7, 16])
def test_simulated_workers(ctx, mode, p):
    """the operator's p > 1 path step for step: the reduce of each shard, the records' exchange of its results, the reduce of
    each window; against the model, and with exact folds the one-worker result placed by Hash128to64(0, key) % p"""
    s, key = 56, (13, 5)
    runs = [(0, 1, MIN_U64), (20, 2, MAX_U64), (40, 2, SUM_F64)]
    rng = np.random.default_rng(p * 2 + mode)
    ns = [int(x) for x in rng.integers(0, 30000, p)]
    if p > 2:
        ns[1] = 0                                                # an empty shard
    allrec = records(sum(ns), s, key, J.zipf_keys(sum(ns), 3000, 1.1, p), runs, seed=p)
    shards = np.split(allrec, np.cumsum(ns)[:-1])
    pre = []
    for sh in shards:
        st, r = reduce_dev(ctx, sh, key, runs)
        assert st == 0 and np.array_equal(r, RR.reduce_local(sh, key, runs))
        pre.append(r)
    wins = _select(ctx, mode, pre, key, p)
    ref = RR.reduce(shards, key, runs)
    one = RR.reduce_local(allrec, key, runs)
    own = J.owner(J.keys_of(one, *key), p)
    for d in range(p):
        st, r = reduce_dev(ctx, wins[d], key, runs)
        assert st == 0 and np.array_equal(r, ref[d]), d
        assert np.array_equal(r, one[own == d]), d


# ---- inside Thrill, and several GPUs --------------------------------------------------------------------------------------------
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HOST_BIN = os.path.join(ROOT, "oracle", "_ref", "host", "gpu_reduce_records_test")
HOST_PASS = 7


def _host_run(workers, n):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([HOST_BIN, str(n)], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in res.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert len(lines) == HOST_PASS and all(l.startswith("PASS") for l in lines), lines


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_reduce_records_test not built "
                    "(make -C tests/host -f gpu_reduce_records_test.mk)")
def test_reduce_records_inside_thrill_single_worker():
    _host_run(1, 99999)


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_reduce_records_test not built")
def test_reduce_records_inside_thrill_two_workers_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _host_run(2, 200000)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_reduce_records_on_n_gpus(world, exchange):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    env = dict(os.environ)
    if exchange == "nccl":
        env["TG_EXCHANGE"] = "nccl"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29941 + world), os.path.join(HERE, "multi_gpu_reduce_records_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert res.returncode == 0 and "MULTI_GPU_REDUCE_RECORDS_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]
