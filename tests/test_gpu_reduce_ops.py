"""The reduce operators across every reduce function and aggregation path on one H100, checked by the contract of
tests/reduce_ref.py (per key; exact where the operation is).  pytest -m gpu.

Every case also asserts which path of run_partitioned_aggregate it took (reduce_ref.path, from the launch counts of one
call with profiling on and tg_hot_records): the HBM table alone below 2^18 records, else the shared-memory units, with
the HBM merge of partial aggregates where a segment was cut or a unit flushed mid-way, and with or without hot-key folding.
The rare paths are forced at small n with keys whose hash has chosen bit fields (reduce_ref.keys_with_hash):
bits 24..39 pick the segment, 40..51 the home slot of the shared-memory table, 52..63 the hot table's, the top bits the
HBM table's.
"""
import ctypes as C
import os
import re
import subprocess
import sys
import zlib

import numpy as np
import pytest

import oracle_lib as O
import reduce_ref as RR
from gpu_util import make_blocks

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
TG_ERR_ARG = -3
PART_MIN = 1 << 18                          # below: the HBM table alone
SIZES = [0, 1, 2, 31, 33, 2047, 2049, PART_MIN - 1, PART_MIN, PART_MIN + 1, 700001, 3000000]
DISTS = ["uniform", "zipf", "small", "zero", "one"]
OP_MIXES = [(op, mix) for op in RR.OPS for mix in RR.VALUE_MIXES[op]]
FORCED_OPS = [("sum_f64", "f64_exact"), ("min_f64", "f64_special"), ("sum_u64", "u64"), ("first", "u64")]


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(device=0)
    yield c
    c.close()


_ZIPF = {}


def make_keys(n, dist, seed):
    rng = np.random.default_rng(seed)
    if dist == "uniform":
        return rng.integers(1, RR.M64, size=n, dtype=np.uint64, endpoint=True)
    if dist == "zipf":
        if "cdf" not in _ZIPF:
            _ZIPF["cdf"] = O.zipf_cdf(1 << 20)
        return O.gen_reduce_zipf(0, n, _ZIPF["cdf"], seed=seed)["key"].copy()
    if dist == "small":
        return rng.integers(1, 100, size=n).astype(np.uint64)
    if dist == "zero":                      # the key 0 (side slot) on a fifth of the records
        k = rng.integers(1, 10000, size=n).astype(np.uint64)
        k[rng.random(n) < 0.2] = 0
        return k
    if dist == "one":
        return np.full(n, 0x5DEECE66D, dtype=np.uint64)
    raise ValueError(dist)


def make_kv(keys, mix, seed):
    kv = np.zeros(len(keys), dtype=O.KV)
    kv["key"] = keys
    kv["val"] = RR.gen_values(mix, kv["key"], seed)
    return kv


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def _code(op):
    return RR.OPS.index(op)


# ---- one call, its result and its path ----------------------------------------------------------------------------------

def hash_aggregate(ctx, kv, op):
    n = len(kv)
    d_in = ctx.to_device(kv)
    d_out = ctx.alloc(n * 16 + 64)
    nd = C.c_uint64()
    try:
        ctx.ck(ctx.L.tg_hash_aggregate(ctx.h, C.byref(_capi().KVDesc(16, _code(op))), d_in, n, d_out, C.byref(nd)))
        return ctx.download(d_out, nd.value * 16, O.KV)
    finally:
        ctx.free(d_in)
        ctx.free(d_out)


def reduce_by_key(ctx, kv, op):
    d_in = ctx.to_device(kv)
    rp, rc = C.c_void_p(), C.c_size_t()
    try:
        ctx.ck(ctx.L.tg_reduce_by_key(ctx.h, C.byref(_capi().KVDesc(16, _code(op))), d_in, len(kv), C.byref(rp), C.byref(rc)))
        return ctx.download(rp.value, rc.value * 16, O.KV)
    finally:
        ctx.free(d_in)


def reduce_file(ctx, kv, op, in_block=4093, out_block=1021):
    """tg_reduce_file over host Blocks that are not multiples of 16 bytes, fetched into such Blocks"""
    capi = _capi()
    blocks, nb, raw = make_blocks(capi, kv, in_block)
    n_out = C.c_size_t()
    ctx.ck(ctx.L.tg_reduce_file(ctx.h, C.byref(capi.KVDesc(16, _code(op))), blocks, nb, C.byref(n_out)))
    out = np.zeros(n_out.value, dtype=O.KV)
    ob, onb, _ = make_blocks(capi, out, out_block)
    ctx.ck(ctx.L.tg_fetch_output(ctx.h, ob, onb))
    return out


def reduce_dev(ctx, kv, op):
    capi = _capi()
    d_in = ctx.to_device(kv)
    try:
        f = capi.DevFile(d_in, len(kv), 16, 0)
        n_out = C.c_size_t()
        ctx.ck(ctx.L.tg_reduce_dev(ctx.h, C.byref(capi.KVDesc(16, _code(op))), C.byref(f), C.byref(n_out)))
        out = np.zeros(n_out.value, dtype=O.KV)
        ob, onb, _ = make_blocks(capi, out, 1 << 20)
        ctx.ck(ctx.L.tg_fetch_output(ctx.h, ob, onb))
        return out
    finally:
        ctx.free(d_in)


def run(ctx, fn, kv, op):
    """(result, path) of one call on a ctx whose profile has just been reset"""
    ctx.profile_enable(True)
    before = RR.counters(ctx)
    out = fn(ctx, kv, op)
    p = RR.path(before, RR.counters(ctx))
    ctx.profile_enable(False)
    return out, p


def check(kv, out, op, mix, where):
    try:
        RR.check(kv, out, op, exact=(mix == "f64_exact"))
    except AssertionError as e:
        raise AssertionError("%s: %s" % (where, e)) from None


def assert_table(p, n, op):
    if n < PART_MIN:
        assert p == ("hbm", 0), p           # the HBM table alone: no counting read, nothing folded
    else:
        assert p[0] in ("units", "merge"), p
    if op == "first":
        assert p[1] == 0, p                 # FIRST folds nothing early


# ---- the operator matrix ------------------------------------------------------------------------------------------------

# (the largest size on two distributions and one value mix per op: the host-side check dominates the time there)
MATRIX = [(op, mix, dist, n) for op, mix in OP_MIXES for dist in DISTS for n in SIZES
          if n < 3000000 or (dist in ("uniform", "zipf") and mix == RR.VALUE_MIXES[op][-1])]


@pytest.mark.parametrize("op,mix,dist,n", MATRIX, ids=["%s-%s-%s-n%d" % c for c in MATRIX])
def test_matrix(ctx, op, mix, dist, n):
    """tg_hash_aggregate and tg_reduce_by_key on the same input"""
    seed = _seed(op, mix, dist, n)
    kv = make_kv(make_keys(n, dist, seed), mix, seed + 1)
    for name, fn in (("tg_hash_aggregate", hash_aggregate), ("tg_reduce_by_key", reduce_by_key)):
        out, p = run(ctx, fn, kv, op)
        check(kv, out, op, mix, name)
        assert_table(p, n, op)
        if dist == "one" and n >= PART_MIN:
            # one key: folded whole by the counting read (no unit left), or for FIRST one segment cut into 64K pieces
            assert p == (("merge", 0) if op == "first" else ("units", n)), p


FILE_CASES = [(op, mix, dist, n) for op, mix in OP_MIXES for dist, n in (("zero", 2049), ("zipf", 700001))]


@pytest.mark.parametrize("op,mix,dist,n", FILE_CASES, ids=["%s-%s-%s-n%d" % c for c in FILE_CASES])
def test_file_and_dev_entry_points(ctx, op, mix, dist, n):
    """tg_reduce_file (records straddle the Blocks on upload and on fetch) and tg_reduce_dev"""
    seed = _seed("file", op, mix, dist, n)
    kv = make_kv(make_keys(n, dist, seed), mix, seed + 1)
    for name, fn in (("tg_reduce_file", reduce_file), ("tg_reduce_dev", reduce_dev)):
        out, p = run(ctx, fn, kv, op)
        check(kv, out, op, mix, name)
        assert_table(p, n, op)


# ---- forced paths -------------------------------------------------------------------------------------------------------

def _filler(n, seed):
    """distinct uniform keys, none of them hot"""
    return np.random.default_rng(seed).integers(1, RR.M64, size=n, dtype=np.uint64, endpoint=True)


def _mix_in(parts, seed):
    keys = np.concatenate(parts)
    return np.random.default_rng(seed).permutation(keys)


def forced_keys(case):
    """(keys, expected table, expected hot records: an int, or "some" = 0 < hot < the hot keys' records, None = any)"""
    if case == "mid_unit_flush":
        # one segment of 6000 distinct keys x 3 records: the unit's table passes 7/8 full and is flushed as partials
        k = RR.keys_with_hash(6000, {(24, 16): 0x3C5A}, seed=1)
        return _mix_in([np.repeat(k, 3), _filler(250000, 2)], 3), "merge", 0
    if case == "cut_segment":
        # one segment of 150000 records (5 of each of 30000 keys): longer than 64K, cut into pieces
        k = RR.keys_with_hash(30000, {(24, 16): 0x0101}, seed=4)
        return _mix_in([np.repeat(k, 5), _filler(200000, 5)], 6), "merge", None
    if case == "super_hot_over_64":
        # 100 keys with 0.5 % of the records each: all hot, more than the 64 warp-private accumulators
        k = RR.keys_with_hash(100, {}, seed=7)
        return _mix_in([np.repeat(k, 2000), _filler(200000, 8)], 9), "units", 200000
    if case == "hot_candidates_over_1024":
        # 2000 keys seen ~16 times each in the sample: the threshold rises until at most 1024 are hot
        k = RR.keys_with_hash(2000, {}, seed=10)
        return _mix_in([np.repeat(k, 100), _filler(200000, 11)], 12), None, "some"
    if case == "hot_find_chain_wrap":
        # 300 hot keys on hot-table home slot 4095: one chain of 300 that wraps to slot 0
        k = RR.keys_with_hash(300, {(52, 12): 4095}, seed=13)
        return _mix_in([np.repeat(k, 1000), _filler(100000, 14)], 15), "units", 300000
    if case == "all_hot_no_zero":
        # every record hot (n_rest == 0): 200 keys x 2000
        k = RR.keys_with_hash(200, {}, seed=16)
        return _mix_in([np.repeat(k, 2000)], 17), "units", 400000
    if case == "smem_chain_wrap":
        # one segment, 1500 keys x 2 whose shared-memory home slot is 4095: a probe chain that wraps to slot 0
        k = RR.keys_with_hash(1500, {(24, 16): 0x7777, (40, 12): 4095}, seed=18)
        return _mix_in([np.repeat(k, 2), _filler(260000, 19)], 20), "units", 0
    if case == "crowded_rows":
        # one segment, 1000 keys x 3 on one tag slot of the in-warp leader election (home & 1023) but 4 home slots: every
        # warp row holds lanes with different keys in the same tag slot
        k = RR.keys_with_hash(1000, {(24, 16): 0x2468, (40, 10): 0x155}, seed=21)
        return _mix_in([np.repeat(k, 3), _filler(260000, 22)], 23), "units", 0
    if case == "hbm_wrap":
        # the HBM table alone: 40 keys on slot cap-1 (top 16 hash bits set) wrap to slot 0, among 3000 others
        k = RR.keys_with_hash(40, {(48, 16): 0xFFFF}, seed=24)
        return _mix_in([np.repeat(k, 5), _filler(3000, 25)], 26), "hbm", 0
    raise ValueError(case)


FORCED = ["mid_unit_flush", "cut_segment", "super_hot_over_64", "hot_candidates_over_1024", "hot_find_chain_wrap",
          "all_hot_no_zero", "smem_chain_wrap", "crowded_rows", "hbm_wrap"]
FORCED_CASES = [(case, op, mix) for case in FORCED for op, mix in FORCED_OPS]


@pytest.mark.parametrize("case,op,mix", FORCED_CASES, ids=["%s-%s-%s" % c for c in FORCED_CASES])
def test_forced_path(ctx, case, op, mix):
    keys, table, hot = forced_keys(case)
    kv = make_kv(keys, mix, _seed(case, op))
    out, p = run(ctx, hash_aggregate, kv, op)
    check(kv, out, op, mix, case)
    if op == "first":
        hot = 0                             # FIRST folds nothing early: hot keys go through the units
        if table == "units" and case in ("super_hot_over_64", "hot_find_chain_wrap", "all_hot_no_zero"):
            table = None                    # ... where their 2000- and 1000-record segments may fill units past 7/8
    if table is not None:
        assert p[0] == table, p
    if hot == "some":
        assert 0 < p[1] < 200000, p
    elif hot is not None:
        assert p[1] == hot, p


@pytest.mark.parametrize("op", ["min_f64", "max_f64"])
def test_super_hot_nan_keys_seen_by_one_warp(ctx, op):
    """Two super-hot keys whose only values are NaNs other than the identity's (the x86 default NaN 0xFFF8..., and a
    signalling NaN), each key on one fixed thread of hot_hist_kernel: every record at a position that is 0 (or 256) mod 512
    (chunks start at multiples of 512 records) is read by warp 0 (or 8), never by the last warp.  The warp-private
    accumulators of the other warps stay at the identity; folding them must keep the input's NaN."""
    n = PART_MIN                                            # the sample reads every 4th record: all 512 of each key
    kv = np.zeros(n, dtype=O.KV)
    kv["key"] = _filler(n, 40)
    kv["val"] = RR.gen_values("f64_wide", kv["key"], 41)
    pos = np.arange(n)
    for k, at, nan in ((0x1234567, 0, 0xFFF8000000000000), (0x7654321, 256, 0x7FF0000000000001)):
        kv["key"][pos % 512 == at] = k
        kv["val"][pos % 512 == at] = nan
    out, p = run(ctx, hash_aggregate, kv, op)
    check(kv, out, op, "f64_wide", "super-hot NaN keys")
    assert p == ("units", 1024), p


# ---- ReduceToIndex ------------------------------------------------------------------------------------------------------

def reduce_to_index(ctx, kv, size, op, neutral, entry="dev_ptr"):
    capi = _capi()
    neu = np.zeros(1, dtype=O.KV)
    neu["key"], neu["val"] = neutral
    desc = capi.KVDesc(16, _code(op))
    on, ob = C.c_size_t(), C.c_uint64()
    if entry == "file":
        blocks, nb, raw = make_blocks(capi, kv, 4093)
        ctx.ck(ctx.L.tg_reduce_to_index_file(ctx.h, C.byref(desc), blocks, nb, size, neu.ctypes.data, C.byref(on), C.byref(ob)))
    else:
        d_in = ctx.to_device(kv)
        try:
            if entry == "dev":
                f = capi.DevFile(d_in, len(kv), 16, 0)
                ctx.ck(ctx.L.tg_reduce_to_index_dev(ctx.h, C.byref(desc), C.byref(f), size, neu.ctypes.data, C.byref(on), C.byref(ob)))
            else:
                op_ = C.c_void_p()
                ctx.ck(ctx.L.tg_reduce_to_index(ctx.h, C.byref(desc), d_in, len(kv), size, neu.ctypes.data, C.byref(op_),
                                                C.byref(on), C.byref(ob)))
                assert ob.value == 0
                return ctx.download(op_.value, on.value * 16, O.KV)
        finally:
            ctx.free(d_in)
    assert ob.value == 0
    out = np.zeros(on.value, dtype=O.KV)
    o, onb, _ = make_blocks(capi, out, 1021)
    ctx.ck(ctx.L.tg_fetch_output(ctx.h, o, onb))
    return out


def index_kv(n, size, mix, seed):
    """indices below size; 0 and size-1 on a tenth of the records each"""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, size, size=n).astype(np.uint64)
    r = rng.random(n)
    k[r < 0.1] = 0
    k[(r >= 0.1) & (r < 0.2)] = size - 1
    return make_kv(k, mix, seed + 1)


TO_INDEX = [(op, mix, n, size) for op, mix in OP_MIXES for n, size in
            ((5000, 1), (5000, 2), (5000, "exact"), (5000, 1 << 22), (0, 7), (400000, 300001))]


@pytest.mark.parametrize("op,mix,n,size", TO_INDEX, ids=["%s-%s-n%d-size%s" % c for c in TO_INDEX])
def test_reduce_to_index(ctx, op, mix, n, size):
    seed = _seed("idx", op, mix, n, size)
    if size == "exact":
        kv = index_kv(n, 3001, mix, seed)
        size = int(kv["key"].max()) + 1
    else:
        kv = index_kv(n, size, mix, seed)
    neutral = (0xABCDEF, 0x8000000000000000)
    ctx.profile_enable(True)
    before = RR.counters(ctx)
    out = reduce_to_index(ctx, kv, size, op, neutral)
    p = RR.path(before, RR.counters(ctx))
    ctx.profile_enable(False)
    RR.to_index_check(kv, out, size, op, neutral=neutral, exact=(mix == "f64_exact"))
    assert_table(p, n, op)


@pytest.mark.parametrize("entry", ["file", "dev"])
def test_reduce_to_index_entry_points(ctx, entry):
    for op, mix in (("min_f64", "f64_special"), ("sum_u64", "u64")):
        kv = index_kv(300000, 100003, mix, 77)
        out = reduce_to_index(ctx, kv, 100003, op, (1, 2), entry=entry)
        RR.to_index_check(kv, out, 100003, op, neutral=(1, 2))


@pytest.mark.parametrize("n", [1000, 300000])
def test_reduce_to_index_rejects_index_2_64_minus_1(ctx, n):
    """an index at 2^64-1 is not below result_size: TG_ERR_ARG from the HBM table's path and from the partitioned one"""
    capi = _capi()
    kv = index_kv(n, 5000, "u64", n)
    kv["key"][n // 2] = np.uint64(RR.M64)
    d_in = ctx.to_device(kv)
    neu = np.zeros(1, dtype=O.KV)
    op_, on, ob = C.c_void_p(), C.c_size_t(), C.c_uint64()
    st = ctx.L.tg_reduce_to_index(ctx.h, C.byref(capi.KVDesc(16, capi.OP_SUM_U64)), d_in, n, 5000, neu.ctypes.data,
                                  C.byref(op_), C.byref(on), C.byref(ob))
    ctx.free(d_in)
    assert st == TG_ERR_ARG


# ---- the paths behind environment switches (read once per process) -------------------------------------------------------

def _group_log2_without_regrouping(n_rest):
    """run_partitioned_aggregate's segments per unit (log2) before the skew-based regrouping that TG_REDUCE_GROUP=0 turns off"""
    g = 0
    while g < 16 and (max(n_rest, 1) << (g + 1)) // (1 << 16) <= 1024:
        g += 1
    return g


def reduced_matrix():
    """a few ops x distributions x sizes on one ctx, run in a subprocess by test_env_switches: results, and the paths the
    switch set in the environment forces (TG_REDUCE_HBM_TABLE: the HBM table alone at every n; TG_REDUCE_NO_HOT: nothing
    folded by the counting read)"""
    from thrill_b200 import capi
    hbm_only, no_hot = "TG_REDUCE_HBM_TABLE" in os.environ, "TG_REDUCE_NO_HOT" in os.environ
    ctx = capi.Ctx(device=0)

    def one(kv, op, mix, where):
        out, p = run(ctx, hash_aggregate, kv, op)
        check(kv, out, op, mix, where)
        if hbm_only:
            assert p == ("hbm", 0), (where, p)
        elif len(kv) >= PART_MIN:
            assert p[0] in ("units", "merge"), (where, p)
        if no_hot:
            assert p[1] == 0, (where, p)

    try:
        for op, mix in FORCED_OPS + [("max_f64", "f64_special"), ("min_u64", "u64")]:
            for dist in ("zipf", "zero", "small"):
                for n in (2049, PART_MIN + 1, 700001):
                    seed = _seed(op, dist, n)
                    one(make_kv(make_keys(n, dist, seed), mix, seed + 1), op, mix, "%s %s %s n=%d" % (op, mix, dist, n))
            for case in ("mid_unit_flush", "hot_find_chain_wrap"):
                keys, _, _ = forced_keys(case)
                one(make_kv(keys, mix, 5), op, mix, case)
        # skewed and large enough for the regrouping to act (2^(group_log2) < 64 before it)
        kv = make_kv(make_keys(3000000, "zipf", 31), "f64_exact", 32)
        one(kv, "sum_f64", "f64_exact", "zipf n=3000000")
    finally:
        ctx.close()
    print("REDUCED_MATRIX_OK")


@pytest.mark.parametrize("var,value", [("TG_REDUCE_HBM_TABLE", "1"), ("TG_REDUCE_NO_HOT", "1"), ("TG_REDUCE_UNSTABLE", "0"),
                                       ("TG_REDUCE_GROUP", "0"), (None, None)])
def test_env_switches(var, value):
    """TG_REDUCE_HBM_TABLE and TG_REDUCE_NO_HOT act on presence and are checked on the paths (reduced_matrix);
    TG_REDUCE_GROUP=0 on the unit grouping that TG_DEBUG_REDUCE reports for every partitioned call.  TG_REDUCE_UNSTABLE=0
    only swaps the ranking of the two hash passes, which leaves no trace outside the library: its results are checked.
    Without a switch, the regrouping must act on the large Zipf case (so that TG_REDUCE_GROUP=0 is seen to turn it off)."""
    env = dict(os.environ)
    if var:
        env[var] = value
    env["TG_DEBUG_REDUCE"] = "1"
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_reduce_ops as t; t.reduced_matrix()" % (
        HERE, os.path.dirname(HERE))
    res = subprocess.run([sys.executable, "-c", code], env=env, cwd=os.path.dirname(HERE), capture_output=True, text=True,
                         timeout=900)
    assert res.returncode == 0 and "REDUCED_MATRIX_OK" in res.stdout, res.stdout[-2000:] + res.stderr[-3000:]
    lines = re.findall(r"\[tg_reduce\] n=(\d+) hot records=(\d+) group_log2=(\d+)", res.stderr)
    if var == "TG_REDUCE_HBM_TABLE":
        assert not lines, lines[:3]                                    # no call took the partitioned path
    else:
        assert len(lines) >= 30, res.stderr[-2000:]
    if var == "TG_REDUCE_GROUP":
        for n, hot, g in lines:
            assert int(g) == _group_log2_without_regrouping(int(n) - int(hot)), (n, hot, g)
    if var is None:
        assert any(int(g) > _group_log2_without_regrouping(int(n) - int(hot)) for n, hot, g in lines), lines
