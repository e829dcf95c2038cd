"""PrefixSum / ExPrefixSum / ZipWithIndex on one H100: tg_prefix_sum, tg_zip_with_index, their _file and _select forms,
tg_scan_local_total and the Python mirror against the numpy restatement in scan_ref.py and against the reference's outputs in
tests/golden/reference_outputs_scan.npz, including p = 2, 3, 4, 8 and 16 workers simulated on one GPU through the kernel-level
entries.  Integer results are compared bit for bit; double sums (bracketed by tiles, not left to right) within
1e-9 * max(1, the prefix over |x|), with NaN, inf and the sign of zero exact.  Tile edges, device Files, argument errors, the size
limit, full-size cases, the multi-GPU worker and the in-Thrill test binary where the machine has what they need.  pytest -m gpu."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import scan_ref as S
from gpu_util import make_blocks

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "reference_outputs_scan.npz")
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4
TILE = {8: 4096, 16: 2048}                 # items per tile of the scan kernels
INT_OPS = [S.OP_SUM_U64, S.OP_MIN_U64, S.OP_MAX_U64]
NEG0 = 0x8000000000000000


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(0)
    yield c
    c.close()


def _desc(op, pair):
    return _capi().ScanDesc(16 if pair else 8, op)


def _init_buf(initial, pair):
    return np.array(initial if pair else [initial[1]], np.uint64)


def _download(ctx, dptr, n, pair):
    if not n:
        return np.zeros(0, S.KV if pair else np.uint64)
    return ctx.download(dptr, n * (16 if pair else 8)).view(S.KV if pair else np.uint64)


def scan_dev(ctx, items, op, pair=False, initial=(0, 0), inclusive=True):
    """tg_prefix_sum of a host array on one worker: (status, outputs)"""
    d = ctx.to_device(items)
    out, n = C.c_void_p(), C.c_size_t()
    ini = _init_buf(initial, pair)
    st = ctx.L.tg_prefix_sum(ctx.h, C.byref(_desc(op, pair)), d, len(items), ini.ctypes.data, int(inclusive), C.byref(out), C.byref(n))
    res = _download(ctx, out.value, n.value, pair) if st == 0 else None
    if st == 0:        # the input is read, never modified
        assert n.value == len(items)
        assert np.array_equal(_download(ctx, d, len(items), pair).view(np.uint64), np.ascontiguousarray(items).view(np.uint64))
    ctx.free(d)
    return st, res


def zip_dev(ctx, items, index_first):
    d = ctx.to_device(items)
    out, n = C.c_void_p(), C.c_size_t()
    st = ctx.L.tg_zip_with_index(ctx.h, d, len(items), int(index_first), C.byref(out), C.byref(n))
    res = _download(ctx, out.value, n.value, True) if st == 0 else None
    ctx.free(d)
    return st, res


def words(a):
    return np.ascontiguousarray(a).view(np.uint64).reshape(-1)


def values(a, pair):
    return words(a).reshape(-1, 2)[:, 1] if pair else words(a)


def assert_f64_close(got, ref, scale):
    """got, ref: double bits; NaN, inf and the sign of a zero exact, the rest within 1e-9 * max(1, scale)"""
    g, r = np.asarray(got, np.uint64).view(np.float64), np.asarray(ref, np.uint64).view(np.float64)
    assert np.array_equal(np.isnan(g), np.isnan(r))
    inf = np.isinf(r)
    assert np.array_equal(g[inf], r[inf]) and not np.isinf(g[~inf]).any()
    both0 = (g == 0) & (r == 0)
    assert np.array_equal(np.signbit(g[both0]), np.signbit(r[both0]))
    fin = np.isfinite(r)
    tol = 1e-9 * np.maximum(1.0, np.asarray(scale, np.float64)[fin])
    assert (np.abs(g[fin] - r[fin]) <= tol).all(), float(np.max(np.abs(g[fin] - r[fin]) - tol))


def check(ctx, items, op, pair=False, initial=(0, 0), inclusive=True):
    st, res = scan_dev(ctx, items, op, pair, initial, inclusive)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    ref = S.prefix_sum([items], op, pair, initial, inclusive)[0]
    if pair:
        assert np.array_equal(res["key"], ref["key"])
    if op == S.OP_SUM_F64:
        scale = S.f64_abs_prefix([items], pair, float(np.array([initial[1]], np.uint64).view(np.float64)[0]))[0]
        assert_f64_close(values(res, pair), values(ref, pair), scale)
    else:
        assert np.array_equal(words(res), words(ref))
    return res


def gen_u64(n, seed, bits=64):
    rng = np.random.RandomState(seed)
    x = rng.randint(0, 1 << 62, size=n, dtype=np.uint64) * np.uint64(4) + rng.randint(0, 4, size=n, dtype=np.uint64)
    return x >> np.uint64(64 - bits) if bits < 64 else x


def gen_f64(n, seed):
    rng = np.random.RandomState(seed)
    return S.f64_words(rng.standard_normal(n) * 10.0 ** rng.randint(-8, 9, n))


def make_items(n, seed, op, pair):
    v = gen_f64(n, seed) if op == S.OP_SUM_F64 else gen_u64(n, seed)
    return S.pairs(S.splitmix64(np.arange(n, dtype=np.uint64) + np.uint64(seed)), v) if pair else v


# ---- one worker: every op, item size and form ------------------------------------------------------------------------------
@pytest.mark.parametrize("inclusive", [True, False])
@pytest.mark.parametrize("pair", [False, True])
@pytest.mark.parametrize("op", INT_OPS)
def test_integer_ops_exact(ctx, op, pair, inclusive):
    for n, seed in [(1, 1), (777, 2), (100000, 3), (1 << 20, 4)]:
        items = make_items(n, seed, op, pair)
        check(ctx, items, op, pair, (3, 12345), inclusive)
        check(ctx, items, op, pair, (0, (1 << 64) - 1 - seed), inclusive)      # wraps (sum), absorbs (min)


@pytest.mark.parametrize("inclusive", [True, False])
@pytest.mark.parametrize("pair", [False, True])
def test_f64_integer_valued_is_exact(ctx, pair, inclusive):
    """integer-valued doubles whose every partial sum is below 2^53: every bracketing gives the stock bits"""
    rng = np.random.RandomState(7)
    n = 1 << 20
    v = S.f64_words(rng.randint(-(1 << 30), 1 << 30, n).astype(np.float64))
    items = S.pairs(np.arange(n), v) if pair else v
    st, res = scan_dev(ctx, items, S.OP_SUM_F64, pair, (9, int(S.f64_words([-17.0])[0])), inclusive)
    ref = S.prefix_sum([items], S.OP_SUM_F64, pair, (9, int(S.f64_words([-17.0])[0])), inclusive)[0]
    assert st == 0 and np.array_equal(words(res), words(ref))


@pytest.mark.parametrize("inclusive", [True, False])
@pytest.mark.parametrize("pair", [False, True])
def test_f64_general_and_reproducible(ctx, pair, inclusive):
    items = make_items(300000, 21, S.OP_SUM_F64, pair)
    a = check(ctx, items, S.OP_SUM_F64, pair, (0, int(S.f64_words([0.75])[0])), inclusive)
    _, b = scan_dev(ctx, items, S.OP_SUM_F64, pair, (0, int(S.f64_words([0.75])[0])), inclusive)
    assert np.array_equal(words(a), words(b))              # the same bracketing on every run


def test_f64_zero_signs_and_specials(ctx):
    negz = S.f64_words(np.full(10000, -0.0))
    res = check(ctx, negz, S.OP_SUM_F64, False, (0, NEG0))
    assert (res == NEG0).all()                              # -0.0 only where every summand is -0.0
    assert (check(ctx, negz, S.OP_SUM_F64, False, (0, 0)) == 0).all()
    assert (check(ctx, negz, S.OP_SUM_F64, False, (0, NEG0), inclusive=False) == NEG0).all()
    x = np.random.RandomState(4).standard_normal(50000)
    x[1000], x[30000], x[40000] = np.inf, -np.inf, np.nan
    check(ctx, S.f64_words(x), S.OP_SUM_F64)
    y = np.random.RandomState(5).standard_normal(50000)
    y[20000] = -np.inf
    check(ctx, S.f64_words(y), S.OP_SUM_F64, inclusive=False)


# ---- tile edges -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", [False, True])
def test_tile_edges(ctx, pair):
    t = TILE[16 if pair else 8]
    for n in [0, 1, 2, 3, t - 1, t, t + 1, 2 * t, 5 * t + 3, 37 * t + t // 2 + 1]:
        for op in INT_OPS + [S.OP_SUM_F64]:
            items = make_items(n, n + op, op, pair)
            for inclusive in (True, False):
                check(ctx, items, op, pair, (11, 5), inclusive)
    for n in [0, 1, 2, 1023, 1024, 1025, 3 * 1024 + 5]:
        x = gen_u64(n, n)
        for first in (True, False):
            st, res = zip_dev(ctx, x, first)
            assert st == 0 and np.array_equal(res, S.zip_with_index([x], first)[0])


def test_local_total(ctx):
    capi = _capi()
    for op in INT_OPS + [S.OP_SUM_F64]:
        for pair in (False, True):
            for n in (0, 1, 5000, 100001):
                items = make_items(n, n + 1, op, pair)
                d = ctx.to_device(items)
                tot = np.zeros(2 if pair else 1, np.uint64)
                ctx.ck(ctx.L.tg_scan_local_total(ctx.h, C.byref(capi.ScanDesc(16 if pair else 8, op)), d, n, tot.ctypes.data))
                ctx.free(d)
                ref = S.totals_of([items], op, pair)[0]
                if op == S.OP_SUM_F64:
                    scale = S.f64_abs_prefix([items], pair)[0]
                    assert_f64_close(tot[-1:], [ref[1] if pair else ref], scale[-1:] if n else [0.0])
                    if pair:
                        assert int(tot[0]) == ref[0]
                else:
                    assert tot.tolist() == (list(ref) if pair else [ref])


# ---- several workers simulated on one GPU ------------------------------------------------------------------------------------
def simulate(ctx, case_op, pair, shards, initial, inclusive, zip_first=None):
    """worker r of p = len(shards) through tg_prefix_sum_select / tg_zip_with_index_select"""
    capi = _capi()
    p = len(shards)
    outs = []
    if zip_first is not None:
        sizes = np.array([len(s) for s in shards], np.uint64)
        for r, s in enumerate(shards):
            d = ctx.to_device(s)
            out, n = C.c_void_p(), C.c_size_t()
            ctx.ck(ctx.L.tg_zip_with_index_select(ctx.h, d, len(s), r, p, sizes.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                  int(zip_first), C.byref(out), C.byref(n)))
            outs.append(_download(ctx, out.value, n.value, True))
            ctx.free(d)
        return outs
    desc = capi.ScanDesc(16 if pair else 8, case_op)
    devs = [ctx.to_device(s) for s in shards]
    totals = np.zeros((p, 2 if pair else 1), np.uint64)
    for r, s in enumerate(shards):
        ctx.ck(ctx.L.tg_scan_local_total(ctx.h, C.byref(desc), devs[r], len(s), totals[r].ctypes.data))
    ini = _init_buf(initial, pair)
    for r, s in enumerate(shards):
        out, n = C.c_void_p(), C.c_size_t()
        ctx.ck(ctx.L.tg_prefix_sum_select(ctx.h, C.byref(desc), devs[r], len(s), r, p, totals.ctypes.data, ini.ctypes.data,
                                          int(inclusive), C.byref(out), C.byref(n)))
        assert n.value == len(s)
        outs.append(_download(ctx, out.value, n.value, pair))
    for d in devs:
        ctx.free(d)
    return outs


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/reference_outputs_scan.npz is not present")
    return np.load(GOLDEN)


def check_rows(case, p, outs, ref_rows):
    rows = S.as_rows(outs)
    if case.op != S.OP_SUM_F64:
        assert S.rows_equal(rows, ref_rows), (case.name, p)
        return
    assert np.array_equal(rows[:, :2], ref_rows[:, :2]), (case.name, p)
    init = float(np.array([case.initial[1]], np.uint64).view(np.float64)[0])
    scale = np.concatenate(S.f64_abs_prefix(case.shards(p), case.pair, init))
    assert_f64_close(rows[:, 2], ref_rows[:, 2], scale)


@pytest.mark.parametrize("p", [1, 2, 3, 4, 8])
def test_simulated_workers_equal_the_reference(ctx, p):
    g = _golden()
    for name in S.case_names(g):
        case = S.Case(g, name)
        shards = case.shards(p)
        if case.op is None:
            outs = simulate(ctx, None, True, shards, None, None, zip_first=case.mode == "zip_first")
        else:
            outs = simulate(ctx, case.op, case.pair, shards, case.initial, case.inclusive)
        check_rows(case, p, outs, case.rows(p))
        if p == 1:          # the operator itself at p = 1
            if case.op is None:
                st, res = zip_dev(ctx, case.items, case.mode == "zip_first")
            else:
                st, res = scan_dev(ctx, case.items, case.op, case.pair, case.initial, case.inclusive)
            assert st == 0
            check_rows(case, 1, [res], case.rows(1))


@pytest.mark.parametrize("op", INT_OPS + [S.OP_SUM_F64])
def test_sixteen_simulated_workers(ctx, op):
    """p = 16 with empty workers and tile-crossing shards, against the model"""
    for pair in (False, True):
        n = 16 * 3000 + 7
        items = make_items(n, 16 + op, op, pair)
        counts = [0, 5000, 1, 0, 4096, 4097, 2047, 0, 9000, 3, 2048, 6000, 0, 7000, 1] + [0]
        counts[-1] = n - sum(counts)
        shards = S.shards_of(items, counts)
        for inclusive in (True, False):
            outs = simulate(ctx, op, pair, shards, (42, 9), inclusive)
            ref = S.prefix_sum(shards, op, pair, (42, 9), inclusive)
            for o, r in zip(outs, ref):
                if pair:
                    assert np.array_equal(o["key"], r["key"])
                if op != S.OP_SUM_F64:
                    assert np.array_equal(words(o), words(r))
            if op == S.OP_SUM_F64:
                scale = np.concatenate(S.f64_abs_prefix(shards, pair, float(np.array([9], np.uint64).view(np.float64)[0])))
                assert_f64_close(np.concatenate([values(o, pair) for o in outs]),
                                 np.concatenate([values(r, pair) for r in ref]), scale)
    x = gen_u64(50000, 3)
    shards = S.shards_of(x, [3000 * (r % 3) for r in range(15)] + [50000 - sum(3000 * (r % 3) for r in range(15))])
    for first in (True, False):
        outs = simulate(ctx, None, True, shards, None, None, zip_first=first)
        assert all(np.array_equal(o, r) for o, r in zip(outs, S.zip_with_index(shards, first)))


# ---- the _file forms, device Files, the Python mirror ---------------------------------------------------------------------------
@pytest.mark.parametrize("pair", [False, True])
def test_file_host_device_and_detached(ctx, pair):
    capi = _capi()
    op = S.OP_MAX_U64 if pair else S.OP_SUM_U64
    items = make_items(60001, 5, op, pair)
    ib = 16 if pair else 8
    ref = S.prefix_sum([items], op, pair, (1, 2), False)[0]
    ini = _init_buf((1, 2), pair)
    desc = capi.ScanDesc(ib, op)
    n = C.c_size_t()
    # a host File with Blocks that cut items
    blocks, nb, keep = make_blocks(capi, items, 1000)
    inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
    ctx.ck(ctx.L.tg_prefix_sum_file(ctx.h, C.byref(desc), C.byref(inp), ini.ctypes.data, 0, C.byref(n)))
    out = np.empty(n.value * ib, np.uint8)
    ob, onb, _ = make_blocks(capi, out, 1 << 16)
    ctx.ck(ctx.L.tg_fetch_output(ctx.h, ob, onb))
    assert np.array_equal(out.view(np.uint64), words(ref))
    # a device File: read in place, left intact, nothing crosses PCIe; the result detached as a device File
    d = ctx.to_device(items)
    f = capi.DevFile(d, len(items), ib, 0)
    h0, d0 = C.c_uint64(), C.c_uint64()
    ctx.L.tg_transfer_bytes(ctx.h, C.byref(h0), C.byref(d0))
    ctx.ck(ctx.L.tg_prefix_sum_file(ctx.h, C.byref(desc), C.byref(capi.MergeInput(C.pointer(f), None, 0)), ini.ctypes.data, 0,
                                    C.byref(n)))
    det = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(det)))
    h1, d1 = C.c_uint64(), C.c_uint64()
    ctx.L.tg_transfer_bytes(ctx.h, C.byref(h1), C.byref(d1))
    assert (h1.value, d1.value) == (h0.value, d0.value)
    assert det.item_bytes == ib and det.items == n.value == len(items)
    # the detached result is an input of its own
    ctx.ck(ctx.L.tg_prefix_sum_file(ctx.h, C.byref(desc), C.byref(capi.MergeInput(C.pointer(det), None, 0)), None, 1,
                                    C.byref(n)))
    det2 = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(det2)))
    again = _download(ctx, det2.dptr, n.value, pair)
    assert np.array_equal(words(again), words(S.prefix_sum([ref], op, pair, (0, 0), True)[0]))
    ctx.L.tg_dev_file_free(ctx.h, C.byref(det2))
    assert np.array_equal(_download(ctx, det.dptr, len(items), pair).view(np.uint64), words(ref))
    assert np.array_equal(_download(ctx, d, len(items), pair).view(np.uint64), words(items))
    ctx.L.tg_dev_file_free(ctx.h, C.byref(det))
    # ZipWithIndex from a device File of 8-byte items, and from a host File
    x = gen_u64(30001, 9)
    dx = ctx.to_device(x)
    fx = capi.DevFile(dx, len(x), 8, 0)
    ctx.ck(ctx.L.tg_zip_with_index_file(ctx.h, C.byref(capi.MergeInput(C.pointer(fx), None, 0)), 0, C.byref(n)))
    zd = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(zd)))
    assert zd.item_bytes == 16 and zd.items == len(x)
    assert np.array_equal(_download(ctx, zd.dptr, len(x), True), S.zip_with_index([x], False)[0])
    ctx.L.tg_dev_file_free(ctx.h, C.byref(zd))
    xb, xnb, _ = make_blocks(capi, x, 999)
    ctx.ck(ctx.L.tg_zip_with_index_file(ctx.h, C.byref(capi.MergeInput(None, C.cast(xb, C.POINTER(capi.Block)), xnb)), 1,
                                        C.byref(n)))
    zo = np.empty(n.value * 16, np.uint8)
    zb, znb, _ = make_blocks(capi, zo, 1 << 15)
    ctx.ck(ctx.L.tg_fetch_output(ctx.h, zb, znb))
    assert np.array_equal(zo.view(S.KV), S.zip_with_index([x], True)[0])
    assert np.array_equal(_download(ctx, dx, len(x), False), x)
    ctx.free(dx)
    ctx.free(d)


def test_python_scan_operators():
    from thrill_b200 import api, capi
    c = api.Context(rank=0, nranks=1, device=0, rng_seed=3)
    try:
        x = gen_u64(20000, 8)
        out = api.DIA(c, x).PrefixSum().items
        assert np.array_equal(out, S.prefix_sum([x], "sum_u64")[0])
        out = api.DIA(c, x).ExPrefixSum(api.MaxU64, 7).items
        assert np.array_equal(out, S.prefix_sum([x], "max_u64", initial=(0, 7), inclusive=False)[0])
        f = np.arange(1000, dtype=np.float64)
        out = api.DIA(c, f).PrefixSum(api.PlusDouble).items
        assert out.dtype == np.float64 and np.array_equal(out, np.cumsum(f))
        kv = S.pairs(np.arange(5000), gen_u64(5000, 2) % np.uint64(100))
        out = api.DIA(c, kv.view(api.KV)).PrefixSum(api.ScanSecond(api.MaxU64)).items
        assert np.array_equal(words(out), words(S.prefix_sum([kv], "max_u64", pair=True)[0]))
        out = api.DIA(c, kv.view(api.KV)).ExPrefixSum(api.ScanSecond(api.MaxU64), (5, 6)).items
        assert np.array_equal(words(out), words(S.prefix_sum([kv], "max_u64", True, (5, 6), False)[0]))
        z = api.DIA(c, x).ZipWithIndex(api.IndexFirst).items
        assert np.array_equal(z.view(np.uint64), words(S.zip_with_index([x], True)[0]))
        z = api.DIA(c, f).ZipWithIndex(api.IndexSecond).items
        assert np.array_equal(z.view(np.uint64), words(S.zip_with_index([f.view(np.uint64)], False)[0]))
        with pytest.raises(capi.ThrillGpuError):
            api.DIA(c, f).PrefixSum(api.MinDouble)
        with pytest.raises(capi.ThrillGpuError):
            api.DIA(c, kv.view(api.KV)).PrefixSum(api.MaxU64)             # pairs need ScanSecond
        with pytest.raises(capi.ThrillGpuError):
            api.DIA(c, kv.view(api.KV)).ZipWithIndex(api.IndexFirst)      # 16-byte items
    finally:
        c.close()


# ---- errors and the size limit -----------------------------------------------------------------------------------------------
def test_argument_errors(ctx):
    capi = _capi()
    d = ctx.to_device(np.arange(4, dtype=np.uint64))
    out, n = C.c_void_p(), C.c_size_t()
    for ib, op in [(8, 4), (8, 5), (8, 6), (16, 4), (16, 5), (16, 6), (4, 1), (24, 1), (0, 1), (8, 7)]:
        st = ctx.L.tg_prefix_sum(ctx.h, C.byref(capi.ScanDesc(ib, op)), d, 2, None, 1, C.byref(out), C.byref(n))
        assert st == TG_ERR_ARG, (ib, op)
        tot = np.zeros(2, np.uint64)
        assert ctx.L.tg_scan_local_total(ctx.h, C.byref(capi.ScanDesc(ib, op)), d, 2, tot.ctypes.data) == TG_ERR_ARG
    desc = capi.ScanDesc(8, S.OP_SUM_U64)
    assert ctx.L.tg_prefix_sum(ctx.h, None, d, 2, None, 1, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert ctx.L.tg_prefix_sum(ctx.h, C.byref(desc), None, 2, None, 1, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert ctx.L.tg_zip_with_index(ctx.h, None, 2, 1, C.byref(out), C.byref(n)) == TG_ERR_ARG
    totals = np.zeros(4, np.uint64)
    sizes = np.zeros(17, np.uint64)
    assert ctx.L.tg_prefix_sum_select(ctx.h, C.byref(desc), d, 2, 2, 2, totals.ctypes.data, None, 1, C.byref(out),
                                      C.byref(n)) == TG_ERR_ARG          # rank >= p
    assert ctx.L.tg_prefix_sum_select(ctx.h, C.byref(desc), d, 2, 0, 17, totals.ctypes.data, None, 1, C.byref(out),
                                      C.byref(n)) == TG_ERR_ARG          # p > 16
    assert ctx.L.tg_zip_with_index_select(ctx.h, d, 2, 0, 0, sizes.ctypes.data_as(C.POINTER(C.c_uint64)), 1, C.byref(out),
                                          C.byref(n)) == TG_ERR_ARG
    f16 = capi.DevFile(d, 2, 16, 0)                          # a device File of 16-byte items into ZipWithIndex
    assert ctx.L.tg_zip_with_index_file(ctx.h, C.byref(capi.MergeInput(C.pointer(f16), None, 0)), 1, C.byref(n)) == TG_ERR_ARG
    raw = np.zeros(20, np.uint8)                            # 20 bytes: not whole items
    ob, onb, _ = make_blocks(capi, raw, 20)
    assert ctx.L.tg_prefix_sum_file(ctx.h, C.byref(desc), C.byref(capi.MergeInput(None, C.cast(ob, C.POINTER(capi.Block)), onb)),
                                    None, 1, C.byref(n)) == TG_ERR_ARG
    ctx.free(d)
    check(ctx, np.arange(10, dtype=np.uint64), S.OP_SUM_U64)     # the ctx still works


def test_input_over_the_limit_is_too_large(ctx):
    capi = _capi()
    d = ctx.to_device(np.arange(2, dtype=np.uint64))
    out, n = C.c_void_p(), C.c_size_t()
    # 2^30 items are refused before anything is read (the buffer holds two)
    for ib in (8, 16):
        desc = capi.ScanDesc(ib, S.OP_SUM_U64)
        assert ctx.L.tg_prefix_sum(ctx.h, C.byref(desc), d, 1 << 30, None, 1, C.byref(out), C.byref(n)) == TG_ERR_TOO_LARGE
        tot = np.zeros(2, np.uint64)
        assert ctx.L.tg_scan_local_total(ctx.h, C.byref(desc), d, 1 << 30, tot.ctypes.data) == TG_ERR_TOO_LARGE
    assert ctx.L.tg_zip_with_index(ctx.h, d, 1 << 30, 1, C.byref(out), C.byref(n)) == TG_ERR_TOO_LARGE
    ctx.free(d)
    check(ctx, np.arange(10, dtype=np.uint64), S.OP_SUM_U64)


# ---- full size ----------------------------------------------------------------------------------------------------------------
class _Dev(object):
    """a zero-copy torch view of n x w int64 words at a device pointer"""

    def __init__(self, ptr, n, w):
        self.__cuda_array_interface__ = {"shape": (n, w), "typestr": "<i8", "data": (ptr, False), "version": 3}


@pytest.mark.parametrize("what", ["sum_u64", "pair_max_excl", "zip_first"])
def test_1e8(ctx, what):
    """1e8 items of each item size, checked exactly against the model on the host"""
    import torch
    n = 100_000_000
    free, _ = torch.cuda.mem_get_info(0)
    if free < n * 16 * 3 + (2 << 30):
        pytest.skip("needs %.1f GB of device memory" % (n * 48 / 1e9 + 2))
    rng = np.random.RandomState(1)
    if what == "sum_u64":
        items = rng.randint(0, 1 << 62, size=n, dtype=np.uint64) * np.uint64(3)
        st, res = scan_dev(ctx, items, S.OP_SUM_U64, False, (0, 99), True)
        assert st == 0
        ref = np.cumsum(items, dtype=np.uint64) + np.uint64(99)
        assert np.array_equal(res, ref)
    elif what == "pair_max_excl":
        items = S.pairs(np.arange(n, dtype=np.uint64), np.where(rng.randint(0, 8, n) == 0, np.arange(n, dtype=np.uint64), 0))
        st, res = scan_dev(ctx, items, S.OP_MAX_U64, True, (7, 0), False)
        assert st == 0
        inc = np.maximum.accumulate(items["val"])
        assert res["val"][0] == 0 and np.array_equal(res["val"][1:], inc[:-1])
        assert res["key"][0] == 7 and np.array_equal(res["key"][1:], items["key"][:-1])
    else:
        items = rng.randint(0, 1 << 62, size=n, dtype=np.uint64)
        st, res = zip_dev(ctx, items, True)
        assert st == 0
        assert np.array_equal(res["key"], np.arange(n, dtype=np.uint64)) and np.array_equal(res["val"], items)
    del res, items


# ---- several GPUs --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
def test_scan_on_n_gpus(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29911 + world), os.path.join(HERE, "multi_gpu_scan_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0 and "MULTI_GPU_SCAN_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


# ---- inside a real Thrill job (the GPU nodes against the stock operators) -----------------------------------------------------
HOST_BIN = os.path.join(ROOT, "oracle", "_ref", "host", "gpu_scan_test")
HOST_PASS = 9


def _host_run(workers, n):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([HOST_BIN, str(n)], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in res.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert len(lines) == HOST_PASS and all(l.startswith("PASS") for l in lines), lines


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_scan_test not built (make -C tests/host -f gpu_scan_test.mk)")
def test_scan_inside_thrill_single_worker():
    _host_run(1, 9999)


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_scan_test not built")
def test_scan_inside_thrill_two_workers_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _host_run(2, 200000)
