"""InnerJoin on records (tg_inner_join_records, its _file form, tg_exchange_records_select and the Python mirror) on one H100,
bit for bit against the numpy model in join_records_ref.py: item sizes 4..1024 on either side, keys of 1..8 bytes at aligned and
unaligned offsets, random payload bytes, the count and emit tile edges, key distributions, the pair join's rows, File forms and
chaining, the argument errors and the limits, simulated workers, a TPC-H-shaped case and the multi-GPU worker.  pytest -m gpu."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import join_ref as JP
import join_records_ref as J
from gpu_util import make_blocks

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4
GB = float(1 << 30)


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(0)
    yield c
    c.close()


def desc(lb, lk, rb, rk):
    return _capi().JoinRecordsDesc(lb, rb, lk[0], lk[1], rk[0], rk[1])


def join_dev(ctx, left, right, lk, rk, lb=None, rb=None):
    """tg_inner_join_records of two host record arrays on one worker: (status, result rows)"""
    lb = left.shape[1] if lb is None else lb
    rb = right.shape[1] if rb is None else rb
    dl, dr = ctx.to_device(left), ctx.to_device(right)
    out, n = C.c_void_p(), C.c_size_t()
    st = ctx.L.tg_inner_join_records(ctx.h, C.byref(desc(lb, lk, rb, rk)), dl, len(left), dr, len(right), C.byref(out), C.byref(n))
    res = None
    if st == 0:
        s = lb + rb
        res = ctx.download(out.value, n.value * s).reshape(-1, s) if n.value else np.zeros((0, s), np.uint8)
    ctx.free(dl)
    ctx.free(dr)
    return st, res


def check(ctx, left, right, lk, rk):
    st, res = join_dev(ctx, left, right, lk, rk)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    ref = J.join_local(left, right, lk, rk)
    assert res.shape == ref.shape
    assert np.array_equal(res, ref)
    return len(ref)


def side(n, s, key, keys, seed):
    return J.set_keys(J.make_records(n, s, seed), key[0], key[1], keys)


# ---- shapes: item sizes, key widths and offsets -------------------------------------------------------------------------
# (left bytes, left key (offset, bytes), right bytes, right key)
SHAPES = [
    (4, (0, 4), 4, (0, 4)),            # the key is the whole item
    (4, (1, 2), 8, (6, 2)),            # unaligned 2-byte keys, the right one ends at the item's last byte
    (8, (0, 8), 16, (0, 8)),
    (12, (5, 2), 24, (3, 5)),
    (16, (8, 8), 12, (4, 8)),          # key ending at the last byte on both sides
    (24, (3, 5), 100, (95, 5)),
    (100, (0, 1), 152, (151, 1)),      # 1-byte keys, one at the very end
    (152, (0, 8), 176, (0, 8)),        # TPC-H-shaped: orders / line items, the key at offset 0
    (176, (17, 4), 4, (0, 4)),
    (1024, (1019, 5), 24, (7, 5)),
    (1024, (0, 8), 1024, (1016, 8)),
]


@pytest.mark.parametrize("lb,lk,rb,rk", SHAPES)
def test_shapes(ctx, lb, lk, rb, rk):
    rng = np.random.default_rng(lb * 7 + rb)
    u = min(1 << (8 * min(lk[1], rk[1])), 3000)
    nl, nr = (20000, 15000) if max(lb, rb) < 1024 else (3000, 2500)
    check(ctx, side(nl, lb, lk, rng.integers(0, u, nl, dtype=np.uint64), 1), side(nr, rb, rk, rng.integers(0, u, nr, dtype=np.uint64), 2), lk, rk)


@pytest.mark.parametrize("kb", [1, 2, 4, 5, 8])
@pytest.mark.parametrize("off", [0, 1, 2, 3, 4])
def test_key_widths_and_offsets(ctx, kb, off):
    # keys spread over their whole width (so high bytes matter) with many collisions; the bytes around the key are random
    rng = np.random.default_rng(kb * 10 + off)
    base = rng.integers(0, 500, 4000, dtype=np.uint64)
    top = np.uint64((1 << (8 * kb)) - 1)
    spread = (base * np.uint64(0x9E3779B97F4A7C15)) & top if kb < 8 else base * np.uint64(0x9E3779B97F4A7C15)
    s = ((off + kb + 3) // 4) * 4 + 4
    l = side(4000, s, (off, kb), spread, 3)
    r = side(3000, s + 8, (off, kb), spread[rng.integers(0, 4000, 3000)], 4)
    assert check(ctx, l, r, (off, kb), (off, kb)) > 0


@pytest.mark.parametrize("n", [0, 1, 1023, 1024, 1025, 2047, 2048, 2049])
def test_sizes_and_tile_edges(ctx, n):
    # the count kernel's tiles hold 2048 merged (left, right) items, the emit kernel's 1024 (left items, outputs)
    lk, rk = (3, 5), (0, 8)
    rng = np.random.default_rng(n)
    for nl, nr, kl, kr in [
        (n, n, rng.integers(0, n // 3 + 1, n, dtype=np.uint64), rng.integers(0, n // 3 + 1, n, dtype=np.uint64)),
        (n, 3, np.full(n, 9, np.uint64), np.full(3, 9, np.uint64)),
        (3, n, np.full(3, 9, np.uint64), np.full(n, 9, np.uint64)),
        (n, n // 2 + 1, np.arange(n, dtype=np.uint64), np.arange(n // 2 + 1, dtype=np.uint64) * np.uint64(2)),
        (n, 0, np.arange(n, dtype=np.uint64), np.zeros(0, np.uint64)),
        (0, n, np.zeros(0, np.uint64), np.arange(n, dtype=np.uint64)),
    ]:
        check(ctx, side(nl, 24, lk, kl, 5), side(nr, 12, rk, kr, 6), lk, rk)


@pytest.mark.parametrize("kind", ["foreign_key", "many_to_many", "hot_key", "zipf", "disjoint"])
def test_key_distributions_1e5(ctx, kind):
    lk, rk = (0, 8), (4, 8)
    rng = np.random.default_rng(11)
    n = 100_000
    if kind == "foreign_key":
        kr = rng.permutation(n // 4).astype(np.uint64)
        kl = rng.integers(0, n // 4, n, dtype=np.uint64)
    elif kind == "many_to_many":
        kl, kr = rng.integers(0, 20000, n, dtype=np.uint64), rng.integers(0, 20000, n, dtype=np.uint64)
    elif kind == "hot_key":
        kl = np.where(rng.random(n) < 0.01, 7, rng.integers(0, 1 << 40, n)).astype(np.uint64)
        kr = np.where(rng.random(n) < 0.01, 7, rng.integers(0, 1 << 40, n)).astype(np.uint64)
    elif kind == "zipf":
        kl, kr = J.zipf_keys(n, 50000, 1.0, 1), J.zipf_keys(n // 2, 50000, 1.0, 2)
    else:
        kl, kr = np.arange(0, 2 * n, 2, dtype=np.uint64), np.arange(1, 2 * n, 2, dtype=np.uint64)
    check(ctx, side(n, 40, lk, kl, 7), side(len(kr), 20, rk, kr, 8), lk, rk)


def test_payload_bit_copies(ctx):
    # NaN payloads, -0.0 and infinities in the payload come through as bits
    vals = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 1.5, -2.25], np.float64).view(np.uint64).copy()
    vals[0] |= np.uint64(0x1234)
    l = side(7, 16, (0, 8), np.arange(7, dtype=np.uint64) % np.uint64(3), 9)
    l[:, 8:16] = vals.view(np.uint8).reshape(7, 8)
    check(ctx, l, l.copy(), (0, 8), (0, 8))


def test_pairs_through_the_record_path_match_the_pair_join(ctx):
    """16-byte pairs joined as records give the rows of JoinKeyValues, re-laid out as (l, r) = (key, v1, key, v2)"""
    left, right = JP.make_side(30000, 4000, 1), JP.make_side(25000, 4000, 2)
    st, rows = join_dev(ctx, left.view(np.uint8).reshape(-1, 16), right.view(np.uint8).reshape(-1, 16), (0, 8), (0, 8))
    assert st == 0
    ref = JP.join_local(left, right, JP.KEY_VALUES)
    got = rows.view(np.uint64).reshape(-1, 4)
    assert len(got) == len(ref)
    assert np.array_equal(got[:, 0], ref["key"]) and np.array_equal(got[:, 2], ref["key"])
    assert np.array_equal(got[:, 1], ref["v1"]) and np.array_equal(got[:, 3], ref["v2"])


# ---- File forms, chaining, inputs left intact ---------------------------------------------------------------------------
def _dev_file(ctx, arr):
    capi = _capi()
    d = ctx.to_device(arr)
    return capi.DevFile(d, len(arr), arr.shape[1], 0), d


def _host_input(arr, block_bytes):
    capi = _capi()
    blocks, nb, raw = make_blocks(capi, arr, block_bytes)
    return capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb), (blocks, raw)


def _fetch(ctx, n, s):
    capi = _capi()
    out = np.empty(n * s, np.uint8)
    blocks, nb, _ = make_blocks(capi, out, 1 << 16)
    ctx.ck(ctx.L.tg_fetch_output(ctx.h, blocks, nb))
    return out.reshape(n, s)


def test_file_host_device_and_mixed(ctx):
    capi = _capi()
    lk, rk = (5, 2), (3, 5)
    rng = np.random.default_rng(3)
    left = side(30000, 12, lk, rng.integers(0, 5000, 30000, dtype=np.uint64), 21)
    right = side(20000, 24, rk, rng.integers(0, 5000, 20000, dtype=np.uint64), 22)
    ref = J.join_local(left, right, lk, rk)
    d = desc(12, lk, 24, rk)
    for mode in ("host", "device", "left_device", "right_device"):
        keep, sides, devs = [], [], []
        for j, arr in enumerate((left, right)):
            if mode == "device" or (mode == "left_device" and j == 0) or (mode == "right_device" and j == 1):
                f, dp = _dev_file(ctx, arr)
                devs.append((dp, arr))
                sides.append(capi.MergeInput(C.pointer(f), None, 0))
                keep.append(f)
            else:
                inp, k = _host_input(arr, 1000 + 37 * j)      # Blocks that cut items
                sides.append(inp)
                keep.append(k)
        h2d0, d2h0 = C.c_uint64(), C.c_uint64()
        ctx.L.tg_transfer_bytes(ctx.h, C.byref(h2d0), C.byref(d2h0))
        n = C.c_size_t()
        ctx.ck(ctx.L.tg_inner_join_records_file(ctx.h, C.byref(d), C.byref(sides[0]), C.byref(sides[1]), C.byref(n)))
        h2d1, d2h1 = C.c_uint64(), C.c_uint64()
        ctx.L.tg_transfer_bytes(ctx.h, C.byref(h2d1), C.byref(d2h1))
        assert d2h1.value == d2h0.value            # no device File goes to the host
        if mode == "device":
            assert h2d1.value == h2d0.value
        assert np.array_equal(_fetch(ctx, n.value, 36), ref), mode
        for dp, arr in devs:                       # device Files are left intact
            assert np.array_equal(ctx.download(dp, arr.size).reshape(arr.shape), arr)
            ctx.free(dp)


def test_self_join_on_one_device_file_then_sample(ctx):
    """a self-join of one device File, its detached result fed to Sample (outputs of at most 256 bytes), inputs unchanged"""
    capi = _capi()
    lk = (2, 4)
    a = side(5000, 20, lk, np.random.default_rng(5).integers(0, 800, 5000, dtype=np.uint64), 23)
    f, dp = _dev_file(ctx, a)
    before = ctx.checksum(dp, len(a), 20)
    inp = capi.MergeInput(C.pointer(f), None, 0)
    n = C.c_size_t()
    ctx.ck(ctx.L.tg_inner_join_records_file(ctx.h, C.byref(desc(20, lk, 20, lk)), C.byref(inp), C.byref(inp), C.byref(n)))
    out = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(out)))
    assert out.item_bytes == 40 and out.items == n.value
    ref = J.join_local(a, a, lk, lk)
    assert np.array_equal(ctx.download(out.dptr, n.value * 40).reshape(-1, 40), ref)
    assert ctx.checksum(dp, len(a), 20) == before
    # Sample(all) of the joined records keeps every row, in order
    sin = capi.MergeInput(C.pointer(out), None, 0)
    ns = C.c_size_t()
    ctx.ck(ctx.L.tg_sample_file(ctx.h, 40, C.byref(sin), n.value + 5, 1, C.byref(ns)))
    assert ns.value == n.value
    assert np.array_equal(_fetch(ctx, ns.value, 40), ref)
    ctx.L.tg_dev_file_free(ctx.h, C.byref(out))
    ctx.free(dp)


def test_device_inputs_left_unchanged(ctx):
    lk, rk = (0, 8), (1, 5)
    l = side(9000, 176, lk, np.arange(9000, dtype=np.uint64) % np.uint64(700), 31)
    r = side(7000, 152, rk, np.arange(7000, dtype=np.uint64) % np.uint64(900), 32)
    dl, dr = ctx.to_device(l), ctx.to_device(r)
    cl, cr = ctx.checksum(dl, len(l), 176), ctx.checksum(dr, len(r), 152)
    out, n = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_inner_join_records(ctx.h, C.byref(desc(176, lk, 152, rk)), dl, len(l), dr, len(r), C.byref(out), C.byref(n)))
    assert np.array_equal(ctx.download(out.value, n.value * 328).reshape(-1, 328), J.join_local(l, r, lk, rk))
    assert (ctx.checksum(dl, len(l), 176), ctx.checksum(dr, len(r), 152)) == (cl, cr)
    ctx.free(dl)
    ctx.free(dr)


def test_undetached_results_as_inputs(ctx):
    """the un-detached result of a join (in the output slot) or of GroupByKey (in the slot of the join's tuples) as an input,
    on either side and on both (a self-join): copied out of the way before the join writes those slots"""
    capi = _capi()
    lk, rk = (3, 5), (0, 8)
    rng = np.random.default_rng(17)
    l = side(6000, 24, lk, rng.integers(0, 700, 6000, dtype=np.uint64), 61)
    r = side(5000, 16, rk, rng.integers(0, 700, 5000, dtype=np.uint64), 62)
    dl, dr = ctx.to_device(l), ctx.to_device(r)
    first = J.join_local(l, r, lk, rk)
    other = side(3000, 8, (0, 4), rng.integers(0, 700, 3000, dtype=np.uint64), 63)
    do = ctx.to_device(other)
    jk = (3, 5)                                             # the left record's key inside a joined row

    def join_raw(pl, nl, lb, lkey, pr, nr, rb, rkey):
        out, n = C.c_void_p(), C.c_size_t()
        ctx.ck(ctx.L.tg_inner_join_records(ctx.h, C.byref(desc(lb, lkey, rb, rkey)), pl, nl, pr, nr, C.byref(out), C.byref(n)))
        return out.value, n.value

    for case in ("left", "right", "both"):
        o, m = join_raw(dl, len(l), 24, lk, dr, len(r), 16, rk)       # the result stays in the ctx's output slot
        assert m == len(first)
        if case == "left":
            o2, m2 = join_raw(o, m, 40, jk, do, len(other), 8, (0, 4))
            ref = J.join_local(first, other, jk, (0, 4))
        elif case == "right":
            o2, m2 = join_raw(do, len(other), 8, (0, 4), o, m, 40, jk)
            ref = J.join_local(other, first, (0, 4), jk)
        else:
            o2, m2 = join_raw(o, m, 40, jk, o, m, 40, jk)
            ref = J.join_local(first, first, jk, jk)
        s = ref.shape[1]
        assert np.array_equal(ctx.download(o2, m2 * s).reshape(-1, s), ref), case
    # GroupByKey's result (16-byte pairs sorted by key, in the join's tuple slot) joined with itself on .first
    kv = JP.make_side(20000, 3000, 64)
    dkv = ctx.to_device(kv)
    g, ng = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_group_by_key(ctx.h, dkv, len(kv), C.byref(g), C.byref(ng)))
    grouped = ctx.download(g.value, ng.value * 16).reshape(-1, 16)
    o2, m2 = join_raw(g.value, ng.value, 16, (0, 8), g.value, ng.value, 16, (0, 8))
    assert np.array_equal(ctx.download(o2, m2 * 32).reshape(-1, 32), J.join_local(grouped, grouped, (0, 8), (0, 8)))
    for d in (dl, dr, do, dkv):
        ctx.free(d)


def test_python_mirror():
    from thrill_b200 import api, capi
    c = api.Context(rank=0, nranks=1, device=0, rng_seed=3)
    try:
        lk, rk = (3, 5), (0, 8)
        rng = np.random.default_rng(9)
        l = side(7000, 24, lk, rng.integers(0, 900, 7000, dtype=np.uint64), 41)
        r = side(9000, 16, rk, rng.integers(0, 900, 9000, dtype=np.uint64), 42)
        lv = l.view(np.dtype((np.void, 24))).reshape(-1)
        rv = r.view(np.dtype([("key", "<u8"), ("val", "<u8")])).reshape(-1)       # structured pair items
        out = api.InnerJoin(api.DIA(c, lv), api.DIA(c, rv), api.KeyField(*lk), api.KeyIsFirst, api.JoinPair)
        assert out.items.dtype == np.dtype((np.void, 40))
        assert np.array_equal(out.items.view(np.uint8).reshape(-1, 40), J.join_local(l, r, lk, rk))
        with pytest.raises(capi.ThrillGpuError):
            api.InnerJoin(api.DIA(c, lv), api.DIA(c, rv), api.KeyField(0, 9), api.KeyIsFirst, api.JoinPair)
        l4 = l[:, :4].copy().view(np.dtype((np.void, 4))).reshape(-1)
        with pytest.raises(capi.ThrillGpuError):            # an 8-byte key on 4-byte items
            api.InnerJoin(api.DIA(c, l4), api.DIA(c, rv), api.KeyField(0, 8), api.KeyIsFirst, api.JoinPair)
        with pytest.raises(capi.ThrillGpuError):
            api.InnerJoin(api.DIA(c, lv), api.DIA(c, rv), api.Less, api.KeyIsFirst, api.JoinPair)
        with pytest.raises(capi.ThrillGpuError):
            api.InnerJoin(api.DIA(c, np.arange(10, dtype=np.uint64)), api.DIA(c, rv), api.KeyField(0, 8), api.KeyIsFirst, api.JoinPair)
        # the existing pair calls are unchanged
        a, b = JP.make_side(700, 90, 1), JP.make_side(900, 90, 2)
        out = api.InnerJoin(api.DIA(c, a.view(api.KV)), api.DIA(c, b.view(api.KV)), api.KeyIsFirst, api.KeyIsFirst, api.JoinValues)
        assert np.array_equal(out.items.view(np.uint64), JP.join_local(a, b, JP.VALUES).view(np.uint64))
    finally:
        c.close()


# ---- errors and the limits ----------------------------------------------------------------------------------------------
def test_argument_errors(ctx):
    capi = _capi()
    a = side(3, 24, (0, 8), np.arange(3, dtype=np.uint64), 1)
    ok = (0, 8)
    for lb, lk, rb, rk in [(0, (0, 1), 24, ok), (22, ok, 24, ok), (24, ok, 1028, ok), (24, (0, 0), 24, ok), (24, ok, 24, (0, 9)),
                           (24, (17, 8), 24, ok), (24, ok, 24, (23, 2)), (24, (1 << 31, 4), 24, ok),
                           # keys longer than the item, and offsets past it
                           (4, (0, 8), 24, ok), (4, (0, 5), 24, ok), (4, (100, 5), 24, ok), (24, ok, 4, (2, 4)), (24, ok, 8, (1 << 31, 8))]:
        assert join_dev(ctx, a, a, lk, rk, lb=lb, rb=rb)[0] == TG_ERR_ARG, (lb, lk, rb, rk)
    out, n = C.c_void_p(), C.c_size_t()
    d24 = desc(24, ok, 24, ok)
    assert ctx.L.tg_inner_join_records(ctx.h, C.byref(d24), None, 3, None, 0, C.byref(out), C.byref(n)) == TG_ERR_ARG
    dp = ctx.to_device(a)
    assert ctx.L.tg_inner_join_records(ctx.h, C.byref(d24), dp + 2, 1, dp, 1, C.byref(out), C.byref(n)) == TG_ERR_ARG
    f = capi.DevFile(dp, 3, 16, 0)                          # a device File of another item size
    inp = capi.MergeInput(C.pointer(f), None, 0)
    assert ctx.L.tg_inner_join_records_file(ctx.h, C.byref(d24), C.byref(inp), C.byref(inp), C.byref(n)) == TG_ERR_ARG
    odd, keep = _host_input(np.zeros(40, np.uint8), 40)     # 40 bytes: not whole 24-byte items
    assert ctx.L.tg_inner_join_records_file(ctx.h, C.byref(d24), C.byref(odd), C.byref(odd), C.byref(n)) == TG_ERR_ARG
    ctx.free(dp)
    check(ctx, a, a, ok, ok)                                # the ctx still works
    # the pair join still takes 16-byte items only
    assert ctx.L.tg_inner_join(ctx.h, C.byref(capi.JoinDesc(24, 0)), None, 0, None, 0, C.byref(out), C.byref(n)) == TG_ERR_ARG


def test_output_over_the_limit_is_too_large(ctx):
    # 40 000 x 30 000 records on one key: 1.2e9 outputs > 2^30 - 1, refused before the output is allocated
    l, r = side(40000, 8, (0, 4), np.full(40000, 5, np.uint64), 1), side(30000, 4, (0, 4), np.full(30000, 5, np.uint64), 2)
    assert J.too_large([l], [r], (0, 4), (0, 4))
    assert join_dev(ctx, l, r, (0, 4), (0, 4))[0] == TG_ERR_TOO_LARGE
    check(ctx, l[:300], r[:200], (0, 4), (0, 4))


def test_input_over_the_limit_is_too_large(ctx):
    out, n = C.c_void_p(), C.c_size_t()
    dp = ctx.to_device(np.zeros(64, np.uint8))
    st = ctx.L.tg_inner_join_records(ctx.h, C.byref(desc(8, (0, 8), 8, (0, 8))), dp, 1 << 30, dp, 1, C.byref(out), C.byref(n))
    assert st == TG_ERR_TOO_LARGE
    ctx.free(dp)


# ---- simulated workers -----------------------------------------------------------------------------------------------------
def _select(ctx, mode, shards, key, p, guard=64):
    """tg_exchange_records_select into windows carved from one buffer with guard bytes around each: (counts, windows)"""
    s = shards[0].shape[1]
    n = [len(x) for x in shards]
    dsh = [ctx.to_device(x) if len(x) else None for x in shards]
    counts = (C.c_uint64 * (p * p))()
    sh_arr = (C.c_void_p * p)(*dsh)
    n_arr = (C.c_size_t * p)(*n)
    ctx.ck(ctx.L.tg_exchange_records_select(ctx.h, 0, s, key[0], key[1], sh_arr, n_arr, p, None, None, counts))
    recv = [sum(counts[src * p + d] for src in range(p)) for d in range(p)]
    sizes = [r * s for r in recv]
    offs, tot = [], guard
    for b in sizes:
        offs.append(tot)
        tot += ((b + 15) // 16) * 16 + guard
    fill = np.full(tot, 0xA5, np.uint8)
    base = ctx.to_device(fill)
    win = (C.c_void_p * p)(*[base + o for o in offs])
    wb = (C.c_size_t * p)(*sizes)
    ctx.ck(ctx.L.tg_exchange_records_select(ctx.h, mode, s, key[0], key[1], sh_arr, n_arr, p, win, wb, counts))
    raw = ctx.download(base, tot)
    for o, b in zip(offs, sizes):                           # guard bytes and the padding after each window untouched
        assert np.all(raw[o - guard:o] == 0xA5) and np.all(raw[o + b:o + ((b + 15) // 16) * 16 + guard] == 0xA5)
    windows = [raw[o:o + b].reshape(-1, s) for o, b in zip(offs, sizes)]
    for x in dsh:
        if x:
            ctx.free(x)
    ctx.free(base)
    return np.array(counts[:], np.uint64), windows


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("p", [1, 2, 3, 4, 7, 16])
def test_simulated_workers(ctx, mode, p):
    lk, rk = (5, 2), (3, 5)
    rng = np.random.default_rng(p * 2 + mode)
    nls = [int(x) for x in rng.integers(0, 3000, p)]
    nrs = [int(x) for x in rng.integers(0, 2000, p)]
    if p > 2:
        nls[1] = 0                                          # an empty shard
    lefts, rights, first_l, first_r = [], [], 0, 0
    for w in range(p):
        l = J.set_keys(J.make_records(nls[w], 12, 51, first_l), lk[0], lk[1], rng.integers(0, 700, nls[w], dtype=np.uint64))
        r = J.set_keys(J.make_records(nrs[w], 24, 52, first_r), rk[0], rk[1], rng.integers(0, 700, nrs[w], dtype=np.uint64))
        lefts.append(l); rights.append(r)
        first_l += nls[w]; first_r += nrs[w]
    cl, wl = _select(ctx, mode, lefts, lk, p)
    cr, wr = _select(ctx, mode, rights, rk, p)
    assert np.array_equal(cl, J.exchange_counts(lefts, lk, p)) and np.array_equal(cr, J.exchange_counts(rights, rk, p))
    el, er = J.exchange(lefts, lk, p), J.exchange(rights, rk, p)
    for d in range(p):
        assert np.array_equal(wl[d], el[d]) and np.array_equal(wr[d], er[d]), d
    # each worker's join on its windows is the model's per-worker result
    ref = J.join(lefts, rights, lk, rk)
    for d in range(p):
        st, res = join_dev(ctx, wl[d], wr[d], lk, rk, lb=12, rb=24)
        assert st == 0 and np.array_equal(res, ref[d]), d


@pytest.mark.parametrize("mode", [0, 1])
def test_simulated_workers_against_the_goldens(ctx, mode):
    """the stock api::InnerJoin's outputs at 1-4 workers: the p simulated exchanges of each side, a join per window, the
    concatenation's multiset equal to the stored one, and every worker's result equal to the model's"""
    g = np.load(os.path.join(HERE, "golden", "reference_outputs_join_records.npz"))
    for name, left, right, lk, rk, outs in J.golden_cases(g):
        for p, stored in outs.items():
            lefts = [left[(r * len(left)) // p:((r + 1) * len(left)) // p] for r in range(p)]
            rights = [right[(r * len(right)) // p:((r + 1) * len(right)) // p] for r in range(p)]
            _, wl = _select(ctx, mode, lefts, lk, p)
            _, wr = _select(ctx, mode, rights, rk, p)
            ref = J.join(lefts, rights, lk, rk)
            parts = []
            for d in range(p):
                st, res = join_dev(ctx, wl[d], wr[d], lk, rk, lb=left.shape[1], rb=right.shape[1])
                assert st == 0 and np.array_equal(res, ref[d]), (name, p, d)
                parts.append(res)
            assert J.matches_golden(np.concatenate(parts), stored), (name, p)


def test_simulated_workers_errors(ctx):
    counts = (C.c_uint64 * 4)()
    one = (C.c_size_t * 2)(1, 1)
    dp = ctx.to_device(np.zeros(64, np.uint8))
    sh = (C.c_void_p * 2)(dp, dp)
    assert ctx.L.tg_exchange_records_select(ctx.h, 2, 8, 0, 8, sh, one, 2, None, None, counts) == TG_ERR_ARG
    assert ctx.L.tg_exchange_records_select(ctx.h, 0, 8, 0, 9, sh, one, 2, None, None, counts) == TG_ERR_ARG
    assert ctx.L.tg_exchange_records_select(ctx.h, 0, 4, 0, 8, sh, one, 2, None, None, counts) == TG_ERR_ARG
    assert ctx.L.tg_exchange_records_select(ctx.h, 0, 4, 100, 5, sh, one, 2, None, None, counts) == TG_ERR_ARG
    assert ctx.L.tg_exchange_records_select(ctx.h, 0, 8, 0, 8, sh, one, 17, None, None, counts) == TG_ERR_ARG
    big = (C.c_size_t * 2)(1 << 30, 1)
    assert ctx.L.tg_exchange_records_select(ctx.h, 0, 8, 0, 8, sh, big, 2, None, None, counts) == TG_ERR_TOO_LARGE
    win = (C.c_void_p * 2)(dp, dp)
    small = (C.c_size_t * 2)(0, 0)
    keys = np.array([1, 1], np.uint64)
    ctx.upload(dp, np.concatenate([keys, keys]))
    assert ctx.L.tg_exchange_records_select(ctx.h, 0, 8, 0, 8, sh, one, 2, win, small, counts) == TG_ERR_ARG
    ctx.free(dp)


# ---- a TPC-H-shaped join ----------------------------------------------------------------------------------------------------
def _need(nbytes, what):
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < nbytes + 2 * (1 << 30):
        pytest.skip("%s needs %.1f GB of device memory (+2 GB), %.1f GB are free" % (what, nbytes / GB, free / GB))


def test_tpch_shaped_foreign_key_join(ctx):
    """6e7 x 176-byte line items (key: orderkey at offset 0) against 1.5e7 x 152-byte orders with distinct keys: 6e7 x 328-byte
    outputs, by the order-independent checksum of the whole output against the model built on the device, plus sampled rows"""
    import torch
    nl, nr, lb, rb = 60_000_000, 15_000_000, 176, 152
    _need(nl * lb + nr * rb + 2 * nl * (lb + rb) + 32 * (nl + nr) * 2, "the TPC-H-shaped join")
    try:
        _tpch_case(ctx, torch, nl, nr, lb, rb)
    finally:
        # the tensors are gone; hand their memory back to the driver for the tests that follow in this process
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _tpch_case(ctx, torch, nl, nr, lb, rb):
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(5)
    left = torch.randint(-(1 << 31), 1 << 31, (nl, lb // 4), dtype=torch.int32, device=dev, generator=g)
    right = torch.randint(-(1 << 31), 1 << 31, (nr, rb // 4), dtype=torch.int32, device=dev, generator=g)
    rkey = torch.randperm(nr, device=dev, generator=g)
    lkey = torch.randint(0, nr, (nl,), device=dev, generator=g)
    left.view(torch.int64)[:, 0] = lkey
    right.view(torch.int64)[:, 0] = rkey
    torch.cuda.synchronize()
    out, m = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_inner_join_records(ctx.h, C.byref(desc(lb, (0, 8), rb, (0, 8))), left.data_ptr(), nl, right.data_ptr(), nr,
                                       C.byref(out), C.byref(m)))
    assert m.value == nl
    got = ctx.checksum(out.value, nl, lb + rb)
    # the model: left records in (key, position) order, each followed by the one right record with its key
    inv = torch.empty(nr, dtype=torch.int64, device=dev)
    inv[rkey] = torch.arange(nr, device=dev)
    order = torch.sort(lkey, stable=True).indices
    ref = torch.empty((nl, (lb + rb) // 4), dtype=torch.int32, device=dev)
    step = 5_000_000
    for a in range(0, nl, step):
        o = order[a:a + step]
        ref[a:a + step, :lb // 4] = left[o]
        ref[a:a + step, lb // 4:] = right[inv[lkey[o]]]
    del order
    torch.cuda.synchronize()
    assert ctx.checksum(ref.data_ptr(), nl, lb + rb) == got
    rng = np.random.default_rng(1)
    for j in np.concatenate([[0, 1, nl - 1], rng.integers(0, nl, 200)]):
        row = ctx.download(out.value + int(j) * (lb + rb), lb + rb)
        assert np.array_equal(row, ref[int(j)].cpu().numpy().view(np.uint8)), j


# ---- inside a real Thrill job (GpuJoinNode with tg_join_records_desc against the stock api::InnerJoin) -----------------------
HOST_BIN = os.path.join(ROOT, "oracle", "_ref", "host", "gpu_join_records_test")
HOST_PASS = 9


def _host_run(workers, n):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([HOST_BIN, str(n)], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in res.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert len(lines) == HOST_PASS and all(l.startswith("PASS") for l in lines), lines


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_join_records_test not built "
                    "(make -C tests/host -f gpu_join_records_test.mk)")
def test_join_records_inside_thrill_single_worker():
    _host_run(1, 9999)


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_join_records_test not built")
def test_join_records_inside_thrill_two_workers_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _host_run(2, 100000)


# ---- several GPUs ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_join_records_on_n_gpus(world, exchange):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    env = dict(os.environ)
    if exchange == "nccl":
        env["TG_EXCHANGE"] = "nccl"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29881 + world), os.path.join(HERE, "multi_gpu_join_records_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert res.returncode == 0 and "MULTI_GPU_JOIN_RECORDS_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]
