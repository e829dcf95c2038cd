"""Sort, ReduceByKey and ReduceToIndex at the top of the per-call size range (up to 2^30 - 1 items, more than 4 GiB of
items), on one H100, checked in O(n) against the inputs of tests/large_ref.py; and the 2^30 item limit of every entry
point.  pytest -m "gpu and large" (pytest -m "gpu and not large" leaves them out).

Each case names the device memory it needs (inputs, scratch, the operator's workspaces) and skips if less than that plus
2 GB is free.  Each group of cases (a class) has one ctx, closed at the end of the group, so that one group's workspaces
are released before the next.  Every case asserts the path it took as well as its result: launch counts of
tg_profile_get, tg_prefix_sort_fallbacks and tg_hot_records (see test_gpu_sort_descriptors.py and reduce_ref.path).
"""
import ctypes as C
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest

import large_ref as L
import reduce_ref as RR
from sort_ref import Desc, LE

# `large` selects these cases by name (-m "gpu and not large" leaves them out).  It is used only in this module and is not
# registered with the suite's markers, so its unknown-marker warning is silenced here, where the mark is made.
with warnings.catch_warnings():
    warnings.simplefilter("ignore", pytest.PytestUnknownMarkWarning)
    pytestmark = [pytest.mark.gpu, pytest.mark.large]

HERE = os.path.dirname(os.path.abspath(__file__))
GB = 1 << 30
LIMIT = 1 << 30
TG_ERR_TOO_LARGE = -4


def _capi():
    from thrill_b200 import capi
    return capi


def need(nbytes, what):
    """skip unless nbytes + 2 GB of device memory are free"""
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < nbytes + 2 * GB:
        pytest.skip("%s needs %.1f GB of device memory (+2 GB), %.1f GB are free" % (what, nbytes / GB, free / GB))


def report(what):
    """the device memory in use while a case holds its buffers (printed: pytest -s shows it)"""
    import torch
    free, total = torch.cuda.mem_get_info(0)
    print("[large] %s: %.1f GB of device memory in use" % (what, (total - free) / GB))


@pytest.fixture(scope="class")
def ctx():
    c = _capi().Ctx(device=0)
    c.profile_enable(True)
    yield c
    c.close()


class Buffers(object):
    """device buffers of a case, freed at the end"""

    def __init__(self, ctx):
        self.ctx, self.ptrs = ctx, []

    def alloc(self, nbytes):
        p = self.ctx.alloc(max(nbytes, 16))
        self.ptrs.append(p)
        return p

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for p in self.ptrs:
            self.ctx.free(p)


# ---- the path of a sort -------------------------------------------------------------------------------------------------

def prefix_digits(n):
    """tg_radix_sort.cu prefix_digits_for: K with 2^(8K) >= 16 n"""
    bits = 4
    while bits < 64 and (1 << bits) < n * 16:
        bits += 1
    return (bits + 7) // 8


def counts(ctx):
    capi = _capi()
    c = {name: ctx.profile_get(cls)[1] for name, cls in (("hist", capi.K_RADIX_HIST), ("part", capi.K_PARTITION),
                                                         ("fixup", capi.K_FIXUP), ("seg", capi.K_SEGCOUNT),
                                                         ("merge", capi.K_MERGE))}
    c["fallback"] = int(ctx.L.tg_prefix_sort_fallbacks(ctx.h))
    return c


def delta(before, after):
    return {k: after[k] - before[k] for k in after}


def expected_counts(path, n, active=8):
    """launch counts of one sort of n well-spread u64 keys (module docstring of test_gpu_sort_descriptors.py):
    prefix        the prefix sort (speculative or histogram-first): K partition passes, one segmented count (K - 1
                  positions inside the buckets of the top digit), one finishing pass
    general       the speculative attempt declined (its top digit has fewer than 32 values), then the general path's
                  prefix section with its own segmented count: 2K passes, two finishing passes
    general_flat  as general, but the top digit of the general path has fewer than 32 values too: its K passes are global
    spec_miss     the speculative attempt, then `active` LSD passes"""
    K = prefix_digits(n)
    return {"prefix": dict(hist=1, part=K, fixup=1, seg=1, fallback=0),
            "general": dict(hist=2, part=2 * K, fixup=2, seg=2, fallback=0),
            "general_flat": dict(hist=2, part=2 * K, fixup=2, seg=1, fallback=0),
            "spec_miss": dict(hist=2, part=K + active, fixup=1, seg=1, fallback=0)}[path]


def assert_path(path, d, n, active=8):
    want = expected_counts(path, n, active)
    got = {k: d[k] for k in want}
    assert got == want, "expected the %s path (K=%d): launch counts %r, expected %r" % (path, prefix_digits(n), got, want)


def reset_sort_state(ctx):
    """what a ctx learns from its sorts (the assumed top key bit, the penalties after a miss) back to a fresh ctx's:
    ten sorts of 2^16 well-spread u64 keys"""
    n = 1 << 16
    keys = L.mix(np.arange(n, dtype=np.uint64))
    with Buffers(ctx) as b:
        d, t = b.alloc(n * 8), b.alloc(n * 8)
        desc = _capi().u64_desc()
        for _ in range(10):
            ctx.upload(d, keys)
            ctx.ck(ctx.L.tg_radix_sort_local(ctx.h, C.byref(desc), d, t, n))
        assert np.array_equal(ctx.download(d, n * 8, np.uint64), np.sort(keys))


# ---- Sort: u64 keys and 16-byte items --------------------------------------------------------------------------------

def run_local_sort(ctx, case, path, active=8, reset=True, what=""):
    """tg_radix_sort_local of case's items: the O(n) check, then the path"""
    n, ib = case.n, case.item_bytes
    need(int(2.3 * n * ib), "sorting %d %d-byte items%s" % (n, ib, what))
    if reset:
        reset_sort_state(ctx)
    with Buffers(ctx) as b:
        d, t = b.alloc(n * ib), b.alloc(n * ib)
        L.stream_to_device_parallel(ctx, d, n, ib, case.items)
        before = counts(ctx)
        ctx.ck(ctx.L.tg_radix_sort_local(ctx.h, C.byref(case.desc().capi()), d, t, n))
        ctx.sync()
        d_counts = delta(before, counts(ctx))
        report("sort of %d %d-byte items%s" % (n, ib, what))
        L.check_on_device(ctx, d, n, ib, case.checker())
    assert_path(path, d_counts, n, active)


SPREAD_SIZES = [1 << 20, (1 << 20) + 1, 1 << 28, (1 << 28) + 1, LIMIT - 1]


class TestSortU64(object):
    @pytest.mark.parametrize("n", SPREAD_SIZES)
    def test_spread(self, ctx, n):
        """distinct well-spread keys: K prefix passes and one finishing pass (K = 3, 4, 4, 5, 5), the speculative path"""
        run_local_sort(ctx, L.SortCase(n), "prefix")

    def test_general_prefix_then_learned_top_bit(self, ctx):
        """K = 5 through the general path's prefix section: keys whose top byte is constant make the speculative attempt
        decline (its top digit has one value); the general path sorts the 7 varying bytes with 4 segmented positions.  The
        ctx learns the top bit 56, and a second sort of such keys takes the speculative path."""
        case = L.SortCase((1 << 28) + 1, bits=56, top=0x5A)
        run_local_sort(ctx, case, "general", what=" (top byte constant)")
        run_local_sort(ctx, case, "prefix", reset=False, what=" (top byte constant, learned top bit)")

    def test_histogram_first(self, ctx):
        """K = 5 through the histogram-first prefix path: TG_SORT_OPTIMISTIC=0, read once per process, so in a subprocess"""
        n = (1 << 28) + 1
        need(int(2.3 * n * 8) + GB, "the histogram-first sort of %d keys in a subprocess" % n)
        env = dict(os.environ, TG_SORT_OPTIMISTIC="0")
        code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_large as T; T.histogram_first_main(%d)"
                % (os.path.dirname(HERE), HERE, n))
        res = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
        assert res.returncode == 0 and "HISTOGRAM_FIRST_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]

    def test_limit_hot_bucket(self, ctx):
        """2^30 - 1 keys whose most significant byte is the same for all but one: one bucket of the top digit holds
        2^30 - 2 items, the most the 30-bit look-back field carries.  The speculative attempt declines, the general path's
        top digit has 2 values: K global passes."""
        n = LIMIT - 1
        run_local_sort(ctx, L.SortCase(n, bits=56, top=0x21, odd=n - 1), "general_flat", what=" (one item outside the top bucket)")

    def test_limit_narrow_keys(self, ctx):
        """2^30 - 1 keys below 2^24, 64 items per key: the general path's LSD passes over 3 bytes with long equal runs"""
        run_local_sort(ctx, L.SortCase(LIMIT - 1, m=64, bits=24), "spec_miss", active=3, what=" (keys < 2^24)")

    def test_limit_descending(self, ctx):
        run_local_sort(ctx, L.SortCase(LIMIT - 1, descending=True), "prefix", what=" (descending)")


def histogram_first_main(n):
    """test_histogram_first, in a process with TG_SORT_OPTIMISTIC=0"""
    ctx = _capi().Ctx(device=0)
    ctx.profile_enable(True)
    try:
        run_local_sort(ctx, L.SortCase(n), "prefix", what=" (histogram first)")
    finally:
        ctx.close()
    print("HISTOGRAM_FIRST_OK")


class TestSortItem16(object):
    @pytest.mark.parametrize("m", [1, 3])
    def test_radix_sort_local(self, ctx, m):
        """2^28 + 1 16-byte items (4 GiB + 16 bytes, K = 5), value = input position, m items per key: stable across 4 GiB"""
        run_local_sort(ctx, L.SortCase((1 << 28) + 1, item_bytes=16, m=m), "prefix", what=" (m=%d)" % m)

    @pytest.mark.parametrize("m", [1, 3])
    def test_sort_operator(self, ctx, m):
        """the same through tg_sort with one rank"""
        case = L.SortCase((1 << 28) + 1, item_bytes=16, m=m)
        n = case.n
        need(int(2.3 * n * 16), "tg_sort of %d 16-byte items" % n)
        reset_sort_state(ctx)
        with Buffers(ctx) as b:
            d = b.alloc(n * 16)
            L.stream_to_device_parallel(ctx, d, n, 16, case.items)
            before = counts(ctx)
            op, on = C.c_void_p(), C.c_size_t()
            ctx.ck(ctx.L.tg_sort(ctx.h, C.byref(case.desc().capi()), d, n, 7, C.byref(op), C.byref(on)))
            ctx.sync()
            d_counts = delta(before, counts(ctx))
            report("tg_sort of %d 16-byte items (m=%d)" % (n, m))
            assert on.value == n
            L.check_on_device(ctx, op.value, n, 16, case.checker())
        assert_path("prefix", d_counts, n)


# ---- Sort: records -------------------------------------------------------------------------------------------------------

class TestRecords(object):
    @pytest.mark.parametrize("n", [50_000_000, 125_000_000])
    @pytest.mark.parametrize("key_offset", [0, 90])
    def test_records(self, ctx, n, key_offset):
        """100-byte records with a 10-byte big-endian key at the front (TeraSort) or at the end, 2 records per key, more
        than 4 GiB: every byte of every output record checked, and one gather of the records"""
        case = L.RecordCase(n, m=2, key_offset=key_offset)
        need(int(2.6 * n * 100), "sorting %d records" % n)
        with Buffers(ctx) as b:
            d = b.alloc(n * 100)
            L.stream_to_device_parallel(ctx, d, n, 100, case.items, chunk=1 << 22)
            before = counts(ctx)
            op, on = C.c_void_p(), C.c_size_t()
            ctx.ck(ctx.L.tg_sort(ctx.h, C.byref(case.desc().capi()), d, n, 3, C.byref(op), C.byref(on)))
            ctx.sync()
            d_counts = delta(before, counts(ctx))
            report("tg_sort of %d records (key at %d)" % (n, key_offset))
            assert on.value == n
            L.check_on_device(ctx, op.value, n, 100, case.checker(), chunk=1 << 22)
        assert d_counts["merge"] == 1 and d_counts["fallback"] == 0, d_counts


# ---- ReduceByKey ---------------------------------------------------------------------------------------------------------

REDUCE_OPS = [0, 1, 2, 3, 6]       # SUM_F64 (exact integer values), SUM_U64, MIN_U64, MAX_U64, FIRST


class TestReduce(object):
    @pytest.mark.parametrize("dist", ["distinct", "groups", "skewed"])
    @pytest.mark.parametrize("n", [(1 << 27) + 1, 1 << 28])
    def test_reduce(self, ctx, n, dist):
        """tg_reduce_by_key (one rank) and tg_hash_aggregate, every op with a closed form, at sizes where the average hash
        segment is longer than an aggregation unit: all-distinct keys go through the cut-segment / HBM-merge path"""
        case = L.ReduceCase(n, dist)
        need(int(n * 16 * 6.5), "reducing %d records" % n)
        capi = _capi()
        with Buffers(ctx) as b:
            d_in, d_out = b.alloc(n * 16), b.alloc((n + 2) * 16)
            loaded = None
            for op in REDUCE_OPS:
                kind = "f64" if op == 0 else "u64"
                if loaded != kind:
                    L.stream_to_device_parallel(ctx, d_in, n, 16, lambda a, b_: case.items(a, b_, op))
                    loaded = kind
                desc = capi.KVDesc(16, op)
                for entry in ("reduce_by_key", "hash_aggregate"):
                    before = RR.counters(ctx)
                    if entry == "reduce_by_key":
                        op_ptr, on = C.c_void_p(), C.c_size_t()
                        ctx.ck(ctx.L.tg_reduce_by_key(ctx.h, C.byref(desc), d_in, n, C.byref(op_ptr), C.byref(on)))
                        out, m = op_ptr.value, on.value
                    else:
                        dist_n = C.c_uint64()
                        ctx.ck(ctx.L.tg_hash_aggregate(ctx.h, C.byref(desc), d_in, n, d_out, C.byref(dist_n)))
                        out, m = d_out, dist_n.value
                    ctx.sync()
                    table, hot = RR.path(before, RR.counters(ctx))
                    if op == 0 and entry == "reduce_by_key":
                        report("%s of %d records (%s)" % (entry, n, dist))
                    assert m == case.num_groups, (entry, op, m, case.num_groups)
                    L.check_on_device(ctx, out, m, 16, case.checker(op))
                    if dist == "distinct":
                        assert table == "merge" and hot == 0, (entry, op, table, hot)
                    elif dist == "skewed" and op != 6:     # (FIRST folds nothing early: no hot records)
                        assert hot >= n // 4, (entry, op, table, hot)
                    elif op == 6:
                        assert hot == 0, (entry, op, table, hot)


# ---- ReduceToIndex -------------------------------------------------------------------------------------------------------

class TestReduceToIndex(object):
    @pytest.mark.parametrize("size", [LIMIT + 1, (1 << 31) - 1])
    def test_dense_larger_than_item_limit(self, ctx, size):
        """a dense result of more than 2^30 items from 2^22 records over 2^20 indices, 0 and size - 1 among them; every
        slot checked, neutral or folded"""
        case = L.IndexCase(size, 1 << 20, 4)
        need((size + 2) * 16 + case.n * 16 * 8, "a dense result of %d slots" % size)
        capi = _capi()
        neutral = np.array(case.neutral, dtype=np.uint64)
        with Buffers(ctx) as b:
            d_in = b.alloc(case.n * 16)
            L.stream_to_device(ctx, d_in, case.n, 16, case.items)
            op_ptr, on, begin = C.c_void_p(), C.c_size_t(), C.c_uint64()
            ctx.ck(ctx.L.tg_reduce_to_index(ctx.h, C.byref(capi.KVDesc(16, capi.OP_SUM_U64)), d_in, case.n, size,
                                            neutral.ctypes.data, C.byref(op_ptr), C.byref(on), C.byref(begin)))
            report("reduce_to_index with %d slots" % size)
            assert on.value == size and begin.value == 0
            L.stream_from_device(ctx, op_ptr.value, size, 16, lambda a, x: case.check_slots(a, x, capi.OP_SUM_U64))

    def test_index_range_too_large(self, ctx):
        capi = _capi()
        with Buffers(ctx) as b:
            d_in = b.alloc(16 * 4)
            ctx.upload(d_in, np.array([[0, 1], [5, 2]], dtype=np.uint64))
            neutral = np.zeros(2, dtype=np.uint64)
            op_ptr, on, begin = C.c_void_p(), C.c_size_t(), C.c_uint64()
            st = ctx.L.tg_reduce_to_index(ctx.h, C.byref(capi.KVDesc(16, capi.OP_SUM_U64)), d_in, 2, 1 << 31,
                                          neutral.ctypes.data, C.byref(op_ptr), C.byref(on), C.byref(begin))
            assert st == TG_ERR_TOO_LARGE


# ---- the limit itself ----------------------------------------------------------------------------------------------------

ENTRY_POINTS = ["radix_sort_local", "sort", "classify_scatter", "hash_partition", "hash_aggregate", "reduce_by_key",
                "reduce_to_index"]


@pytest.fixture(scope="class")
def full_buffers(ctx):
    """two buffers of 2^30 16-byte items: a missing check would compute on valid memory"""
    need(2 * LIMIT * 16, "the limit cases (two buffers of 2^30 16-byte items)")
    a, b = ctx.alloc(LIMIT * 16), ctx.alloc(LIMIT * 16)
    yield a, b
    ctx.free(a)
    ctx.free(b)


class TestLimit(object):
    @pytest.mark.parametrize("entry", ENTRY_POINTS)
    def test_too_large(self, ctx, full_buffers, entry):
        """n = 2^30 is TG_ERR_TOO_LARGE at every entry point, and the ctx still sorts afterwards"""
        capi = _capi()
        A, B = full_buffers
        n = LIMIT
        u64 = capi.u64_desc()
        kv = capi.KVDesc(16, capi.OP_SUM_U64)
        op_ptr, on = C.c_void_p(), C.c_size_t()
        counts_out = (C.c_uint64 * 2)()
        if entry == "radix_sort_local":
            st = ctx.L.tg_radix_sort_local(ctx.h, C.byref(u64), A, B, n)
        elif entry == "sort":
            st = ctx.L.tg_sort(ctx.h, C.byref(capi.kv_key_desc()), A, n, 1, C.byref(op_ptr), C.byref(on))
        elif entry == "classify_scatter":
            spl = np.array([1 << 63, 0], dtype=np.uint64)             # one splitter: (item, global index)
            st = ctx.L.tg_classify_scatter(ctx.h, C.byref(u64), A, n, 0, spl.ctypes.data, 2, B, counts_out)
        elif entry == "hash_partition":
            st = ctx.L.tg_hash_partition(ctx.h, C.byref(kv), A, n, 2, B, counts_out)
        elif entry == "hash_aggregate":
            distinct = C.c_uint64()
            st = ctx.L.tg_hash_aggregate(ctx.h, C.byref(kv), A, n, B, C.byref(distinct))
        elif entry == "reduce_by_key":
            st = ctx.L.tg_reduce_by_key(ctx.h, C.byref(kv), A, n, C.byref(op_ptr), C.byref(on))
        else:
            neutral = np.zeros(2, dtype=np.uint64)
            begin = C.c_uint64()
            st = ctx.L.tg_reduce_to_index(ctx.h, C.byref(kv), A, n, 1 << 20, neutral.ctypes.data, C.byref(op_ptr),
                                          C.byref(on), C.byref(begin))
        ctx.sync()
        assert st == TG_ERR_TOO_LARGE, "%s with n = 2^30 returned %d (%s)" % (entry, st, ctx.L.tg_last_error(ctx.h).decode())
        reset_sort_state(ctx)                                       # (ends with a checked small sort)
