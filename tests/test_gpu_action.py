"""Sum / Min / Max / AllReduce on one H100: tg_all_reduce, its _file and _select forms and the Python mirror against the numpy
restatement in action_ref.py and against the reference's results in tests/golden/reference_outputs_action.npz, including p = 2,
3, 4, 8 and 16 workers simulated on one GPU through tg_all_reduce_select.  Integer results and Min / Max on doubles are compared
bit for bit (NaN bits included); double sums against the exact sum within the rounding bound of the header (gamma_D A + u |exact|),
with NaN, inf and the sign of zero exact, and run twice to show they are bitwise reproducible.  Tile edges, device Files, argument
errors, the size limit, a full-size case, the multi-GPU worker and the in-Thrill test binary where the machine has what they
need.  pytest -m gpu."""
import ctypes as C
import math
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

import action_ref as A
import scan_exact as X
import scan_ref as S
from gpu_util import make_blocks

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "reference_outputs_action.npz")
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4
TILE = {8: 4096, 16: 2048}                 # items per tile of the tile reduce
OPS = list(range(6))
NEG0, QNAN = 0x8000000000000000, 0x7FF8000000000000


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(0)
    yield c
    c.close()


def _ib(pair):
    return 16 if pair else 8


def _init_buf(initial, pair):
    if initial is None:
        return None
    return np.array(initial if pair else [initial[1]], np.uint64)


def _result(out, pair):
    return (int(out[0]), int(out[1])) if pair else (0, int(out[0]))


def reduce_dev(ctx, items, op, pair=False, initial=None):
    """tg_all_reduce of a host array on one worker: (status, (first, value))"""
    d = ctx.to_device(items)
    out = np.zeros(2, np.uint64)
    ini = _init_buf(initial, pair)
    st = ctx.L.tg_all_reduce(ctx.h, C.byref(_capi().ScanDesc(_ib(pair), op)), d, len(items),
                             None if ini is None else ini.ctypes.data, out.ctypes.data)
    if st == 0:        # the input is read, never modified
        assert np.array_equal(ctx.download(d, max(len(items) * _ib(pair), 0)).view(np.uint64) if len(items) else
                              np.zeros(0, np.uint64), np.ascontiguousarray(items).view(np.uint64).reshape(-1))
    ctx.free(d)
    return st, _result(out, pair)


def select(ctx, shards, op, pair=False, initial=None):
    """worker 0..p-1 of p = len(shards) through tg_all_reduce_select"""
    devs = [ctx.to_device(s) for s in shards]
    ptrs = (C.c_void_p * len(shards))(*devs)
    ns = (C.c_size_t * len(shards))(*[len(s) for s in shards])
    out = np.zeros(2, np.uint64)
    ini = _init_buf(initial, pair)
    ctx.ck(ctx.L.tg_all_reduce_select(ctx.h, C.byref(_capi().ScanDesc(_ib(pair), op)), ptrs, ns, len(shards),
                                      None if ini is None else ini.ctypes.data, out.ctypes.data))
    for d in devs:
        ctx.free(d)
    return _result(out, pair)


def depth(shards, pair):
    """D = k + 31 + ceil(T / 512) + p of include/thrill_gpu.h"""
    ib = _ib(pair)
    t = max(X.ntiles(len(s), ib) for s in shards)
    return (16 if ib == 8 else 8) + 31 + -(-t // 512) + len(shards)


def check_sum_f64(got, shards, pair, initial):
    """a double sum: specials and the sign of zero as the stock fold, finite values within gamma_D A + u |exact|"""
    stock = A.all_reduce(shards, A.OP_SUM_F64, pair, initial)
    g, st = A._f(got[1]), A._f(stock[1])
    assert got[0] == stock[0]
    if math.isnan(st) or math.isinf(st):
        assert (math.isnan(g) and math.isnan(st)) or g == st, (g, st)
        return
    if g == 0 and st == 0:
        assert math.copysign(1, g) == math.copysign(1, st), (g, st)
    # the summands: every worker's items; an empty worker contributes T() = +0.0 or the initial value; worker 0 folds the initial
    terms = []
    for r, s in enumerate(shards):
        v = S.split_values(s, pair)[1]
        if initial is not None and (r == 0 or len(v) == 0):
            terms.append(A._f(initial[1]))
        terms.extend(np.asarray(v, np.uint64).view(np.float64).tolist())
    exact = sum(X.to_fixed(x) for x in terms)
    a = sum(abs(X.to_fixed(x)) for x in terms)
    gm = X.gamma(depth(shards, pair))
    assert (1 + gm) * X.to_double(a) < X.DBL_MAX
    assert math.isfinite(g)
    diff = abs(exact - X.to_fixed(g))
    u = Fraction(X.U)
    assert diff <= (Fraction(gm) * a + u * abs(exact)) * (1 + 16 * u), (g, X.to_double(exact), diff / X.SCALE)


def check(got, shards, op, pair=False, initial=None):
    if op == A.OP_SUM_F64:
        check_sum_f64(got, shards, pair, initial)
    else:
        assert got == A.all_reduce(shards, op, pair, initial), (got, A.all_reduce(shards, op, pair, initial))


def gen_vals(n, seed, op):
    rng = np.random.RandomState(seed)
    if op in A.F64_OPS:
        return S.f64_words(rng.standard_normal(n) * 10.0 ** rng.randint(-8, 9, n))
    return rng.randint(0, 1 << 62, size=n, dtype=np.uint64) * np.uint64(4) + rng.randint(0, 4, size=n, dtype=np.uint64)


def make_items(n, seed, op, pair):
    v = gen_vals(n, seed, op)
    return S.pairs(S.splitmix64(np.arange(n, dtype=np.uint64) + np.uint64(seed)), v) if pair else v


def one(ctx, items, op, pair=False, initial=None):
    st, got = reduce_dev(ctx, items, op, pair, initial)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    check(got, [items], op, pair, initial)
    return got


# ---- one worker: every op and item size -------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", [False, True])
@pytest.mark.parametrize("op", OPS)
def test_every_op(ctx, op, pair):
    init_value = int(S.f64_words([0.75])[0]) if op in A.F64_OPS else (1 << 64) - 5
    for n, seed in [(0, 1), (1, 2), (777, 3), (100000, 4), (1 << 20, 5)]:
        items = make_items(n, seed, op, pair)
        one(ctx, items, op, pair)
        one(ctx, items, op, pair, (3, init_value))
    if op == A.OP_SUM_F64:        # bitwise reproducible
        items = make_items(300001, 9, op, pair)
        assert reduce_dev(ctx, items, op, pair)[1] == reduce_dev(ctx, items, op, pair)[1]


@pytest.mark.parametrize("pair", [False, True])
def test_f64_min_max_specials(ctx, pair):
    """NaN first sticks (its bits), later NaNs are skipped, the earlier of +-0 wins, infinities; at structural positions"""
    t = TILE[_ib(pair)]
    rng = np.random.RandomState(3)
    pay = 0x7FF8000000012345
    for n in (5, t - 1, t + 1, 3 * t + 17):
        base = rng.uniform(1.0, 2.0, n)
        for op, sign in ((A.OP_MIN_F64, 1.0), (A.OP_MAX_F64, -1.0)):
            x = S.f64_words(sign * base)

            def run(words, initial=None):
                items = S.pairs(np.arange(n), words) if pair else words
                return one(ctx, items, op, pair, initial)
            w = x.copy(); w[0] = pay
            assert run(w)[1] == pay
            for pos in {1, 16, 17, 511, 512, n // 2, n - 1} & set(range(1, n)):
                w = x.copy(); w[pos] = pay
                run(w)
                w = x.copy(); w[pos] = 0; w[n - 1 - (pos % 3)] = NEG0
                run(w)
                w = x.copy(); w[pos] = NEG0; w[(pos * 7) % n] = 0
                run(w)
            w = x.copy(); w[n // 2] = S.f64_words([-sign * np.inf])[0]
            run(w)
            run(x, (1, pay))
            run(x, (1, NEG0))
            w = x.copy(); w[:] = QNAN
            run(w)
            run(w, (2, int(S.f64_words([5.0])[0])))


def test_f64_sum_zero_signs_and_specials(ctx):
    negz = S.f64_words(np.full(10000, -0.0))
    assert one(ctx, negz, A.OP_SUM_F64)[1] == NEG0
    assert one(ctx, negz, A.OP_SUM_F64, initial=(0, 0))[1] == 0
    x = np.random.RandomState(4).standard_normal(50000)
    x[1000], x[30000] = np.inf, -np.inf
    one(ctx, S.f64_words(x), A.OP_SUM_F64)
    x[30000] = 1.0
    assert one(ctx, S.f64_words(x), A.OP_SUM_F64)[1] == int(S.f64_words([np.inf])[0])
    x[2000] = np.nan
    one(ctx, S.f64_words(x), A.OP_SUM_F64)


# ---- tile edges -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", [False, True])
def test_tile_edges(ctx, pair):
    t = TILE[_ib(pair)]
    for n in [2, 3, t - 1, t, t + 1, 2 * t, 5 * t + 3, 37 * t + t // 2 + 1, 600 * t + 5]:
        for op in OPS:
            items = make_items(n, n + op, op, pair)
            one(ctx, items, op, pair)
            one(ctx, items, op, pair, (11, 5))


# ---- several workers simulated on one GPU ------------------------------------------------------------------------------------
def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/reference_outputs_action.npz is not present")
    return A.Golden(GOLDEN)


def equal_stock(op, got, want):
    if op == A.OP_SUM_F64 and got[0] == want[0] and math.isnan(A._f(got[1])) and math.isnan(A._f(want[1])):
        return True            # a sum's NaN payload is left open
    return got == want


@pytest.mark.parametrize("p", [1, 2, 3, 4, 8])
def test_simulated_workers_equal_the_reference(ctx, p):
    g = _golden()
    for name in A.case_names(g):
        case = A.Case(g, name)
        shards = case.shards(p)
        got = select(ctx, shards, case.op, case.pair, case.initial)
        want = case.result(p)
        if case.op == A.OP_SUM_F64:
            assert (got[0], np.isnan(A._f(got[1]))) == (want[0], np.isnan(A._f(want[1]))), (name, p)
            check_sum_f64(got, shards, case.pair, case.initial)
            if not math.isnan(A._f(want[1])) and A._f(want[1]) in (0.0, np.inf, -np.inf):
                assert got == want, (name, p)
        else:
            assert got == want, (name, p, got, want)
        if p == 1:          # the operator itself at p = 1
            st, res = reduce_dev(ctx, case.items, case.op, case.pair, case.initial)
            assert st == 0 and res == got, name


@pytest.mark.parametrize("op", OPS)
def test_sixteen_simulated_workers(ctx, op):
    """p = 16 with empty workers (first and last among them) and tile-crossing shards, against the model"""
    for pair in (False, True):
        n = 16 * 3000 + 7
        items = make_items(n, 16 + op, op, pair)
        counts = [0, 5000, 1, 0, 4096, 4097, 2047, 0, 9000, 3, 2048, 6000, 0, 7000, 1] + [0]
        counts[-2] += n - sum(counts)
        shards = S.shards_of(items, counts)
        for initial in (None, (42, 9)):
            check(select(ctx, shards, op, pair, initial), shards, op, pair, initial)
        if op == A.OP_SUM_F64:
            assert select(ctx, shards, op, pair) == select(ctx, shards, op, pair)


# ---- the _file form, device Files, the Python mirror ---------------------------------------------------------------------------
@pytest.mark.parametrize("pair", [False, True])
def test_file_host_and_device(ctx, pair):
    capi = _capi()
    ib = _ib(pair)
    for op in OPS:
        items = make_items(60001, 5 + op, op, pair)
        ini = _init_buf((1, 2), pair)
        desc = capi.ScanDesc(ib, op)
        out = np.zeros(2, np.uint64)
        # a host File with Blocks that cut items
        blocks, nb, keep = make_blocks(capi, items, 1000)
        inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
        ctx.ck(ctx.L.tg_all_reduce_file(ctx.h, C.byref(desc), C.byref(inp), ini.ctypes.data, out.ctypes.data))
        host = _result(out, pair)
        check(host, [items], op, pair, (1, 2))
        # a device File: read in place, left intact, only the result crosses PCIe (not through the File codec)
        d = ctx.to_device(items)
        f = capi.DevFile(d, len(items), ib, 0)
        h0, d0 = C.c_uint64(), C.c_uint64()
        ctx.L.tg_transfer_bytes(ctx.h, C.byref(h0), C.byref(d0))
        out[:] = 0
        ctx.ck(ctx.L.tg_all_reduce_file(ctx.h, C.byref(desc), C.byref(capi.MergeInput(C.pointer(f), None, 0)), ini.ctypes.data,
                                        out.ctypes.data))
        h1, d1 = C.c_uint64(), C.c_uint64()
        ctx.L.tg_transfer_bytes(ctx.h, C.byref(h1), C.byref(d1))
        assert (h1.value, d1.value) == (h0.value, d0.value)
        assert _result(out, pair) == host
        assert np.array_equal(ctx.download(d, len(items) * ib).view(np.uint64), np.ascontiguousarray(items).view(np.uint64).reshape(-1))
        ctx.free(d)


def test_python_actions():
    from thrill_b200 import api, capi
    c = api.Context(rank=0, nranks=1, device=0, rng_seed=3)
    try:
        x = gen_vals(20000, 8, A.OP_SUM_U64)
        assert int(api.DIA(c, x).Sum()) == A.all_reduce([x], A.OP_SUM_U64)[1]
        assert int(api.DIA(c, x).Min()) == int(x.min())
        assert int(api.DIA(c, x).Max(7)) == int(x.max())
        assert int(api.DIA(c, x[:0]).Min(7)) == 7
        f = np.arange(1000, dtype=np.float64) - 500.0
        assert api.DIA(c, f).Sum() == -500.0
        assert api.DIA(c, f).Sum(api.PlusDouble, 0.5) == -499.5
        assert api.DIA(c, f).Min() == -500.0 and api.DIA(c, f).Max() == 499.0
        g = f.copy(); g[0] = np.nan
        assert np.isnan(api.DIA(c, g).Max())
        kv = S.pairs(np.arange(5000), gen_vals(5000, 2, A.OP_SUM_U64) % np.uint64(100))
        assert api.DIA(c, kv.view(api.KV)).AllReduce(api.ScanSecond(api.MaxU64)) == A.all_reduce([kv], A.OP_MAX_U64, True)
        assert api.DIA(c, kv.view(api.KV)).AllReduce(api.ScanSecond(api.PlusU64), (5, 6)) == \
            A.all_reduce([kv], A.OP_SUM_U64, True, (5, 6))
        with pytest.raises(capi.ThrillGpuError):
            api.DIA(c, f).AllReduce(api.MinU64)                          # a uint64_t function on doubles
        with pytest.raises(capi.ThrillGpuError):
            api.DIA(c, kv.view(api.KV)).AllReduce(api.MaxU64)            # pairs need ScanSecond
        with pytest.raises(capi.ThrillGpuError):
            api.DIA(c, x).AllReduce(api.First)
    finally:
        c.close()


# ---- errors and the size limit -----------------------------------------------------------------------------------------------
def test_argument_errors(ctx):
    capi = _capi()
    d = ctx.to_device(np.arange(4, dtype=np.uint64))
    out = np.zeros(2, np.uint64)
    for ib, op in [(8, 6), (16, 6), (8, 7), (4, 1), (24, 1), (0, 1), (12, 4)]:
        st = ctx.L.tg_all_reduce(ctx.h, C.byref(capi.ScanDesc(ib, op)), d, 2, None, out.ctypes.data)
        assert st == TG_ERR_ARG, (ib, op)
    desc = capi.ScanDesc(8, A.OP_SUM_U64)
    assert ctx.L.tg_all_reduce(ctx.h, None, d, 2, None, out.ctypes.data) == TG_ERR_ARG
    assert ctx.L.tg_all_reduce(ctx.h, C.byref(desc), None, 2, None, out.ctypes.data) == TG_ERR_ARG
    assert ctx.L.tg_all_reduce(ctx.h, C.byref(desc), d, 2, None, None) == TG_ERR_ARG
    assert ctx.L.tg_all_reduce_file(ctx.h, C.byref(desc), None, None, out.ctypes.data) == TG_ERR_ARG
    ptrs = (C.c_void_p * 17)(*([d] * 17))
    ns = (C.c_size_t * 17)(*([2] * 17))
    assert ctx.L.tg_all_reduce_select(ctx.h, C.byref(desc), ptrs, ns, 0, None, out.ctypes.data) == TG_ERR_ARG
    assert ctx.L.tg_all_reduce_select(ctx.h, C.byref(desc), ptrs, ns, 17, None, out.ctypes.data) == TG_ERR_ARG
    ptrs[1] = None
    assert ctx.L.tg_all_reduce_select(ctx.h, C.byref(desc), ptrs, ns, 2, None, out.ctypes.data) == TG_ERR_ARG
    f16 = capi.DevFile(d, 2, 16, 0)                          # a device File of 16-byte items into an 8-byte action
    assert ctx.L.tg_all_reduce_file(ctx.h, C.byref(desc), C.byref(capi.MergeInput(C.pointer(f16), None, 0)), None,
                                    out.ctypes.data) == TG_ERR_ARG
    raw = np.zeros(20, np.uint8)                            # 20 bytes: not whole items
    ob, onb, _ = make_blocks(capi, raw, 20)
    assert ctx.L.tg_all_reduce_file(ctx.h, C.byref(desc), C.byref(capi.MergeInput(None, C.cast(ob, C.POINTER(capi.Block)), onb)),
                                    None, out.ctypes.data) == TG_ERR_ARG
    ctx.free(d)
    one(ctx, np.arange(10, dtype=np.uint64), A.OP_SUM_U64)     # the ctx still works


def test_input_over_the_limit_is_too_large(ctx):
    capi = _capi()
    d = ctx.to_device(np.arange(2, dtype=np.uint64))
    out = np.zeros(2, np.uint64)
    # 2^30 items are refused before anything is read (the buffer holds two)
    for ib in (8, 16):
        desc = capi.ScanDesc(ib, A.OP_SUM_U64)
        assert ctx.L.tg_all_reduce(ctx.h, C.byref(desc), d, 1 << 30, None, out.ctypes.data) == TG_ERR_TOO_LARGE
        ptrs = (C.c_void_p * 3)(d, d, d)
        ns = (C.c_size_t * 3)(1, 1 << 30, 1)
        assert ctx.L.tg_all_reduce_select(ctx.h, C.byref(desc), ptrs, ns, 3, None, out.ctypes.data) == TG_ERR_TOO_LARGE
    ctx.free(d)
    one(ctx, np.arange(10, dtype=np.uint64), A.OP_SUM_U64)


# ---- full size ----------------------------------------------------------------------------------------------------------------
def test_full_size(ctx):
    """2^30 - 1 uint64_t items from the device generator (the largest a worker may hold), checked with torch on the device"""
    import torch
    n = (1 << 30) - 1
    free, _ = torch.cuda.mem_get_info(0)
    if free < n * 8 * 4 + (2 << 30):
        pytest.skip("needs %.1f GB of device memory" % (n * 32 / 1e9 + 2))
    buf = torch.empty(n + 1, dtype=torch.int64, device="cuda:0")
    ctx.ck(ctx.L.tg_gen_sort_uniform(ctx.h, buf.data_ptr(), 0, n, 12345))
    ctx.sync()
    t = buf[:n]
    flip = t ^ torch.iinfo(torch.int64).min                  # uint64_t order as int64 order
    want = {A.OP_SUM_U64: int(t.sum().item()) & A.M64,
            A.OP_MIN_U64: (int(flip.min().item()) ^ -(1 << 63)) & A.M64,
            A.OP_MAX_U64: (int(flip.max().item()) ^ -(1 << 63)) & A.M64}
    out = np.zeros(1, np.uint64)
    for op, w in want.items():
        ctx.ck(ctx.L.tg_all_reduce(ctx.h, C.byref(_capi().ScanDesc(8, op)), buf.data_ptr(), n, None, out.ctypes.data))
        assert int(out[0]) == w, op
    # doubles: the same mantissas with the exponent of [2, 4): Max / Min exact, Sum within the bound (no overflow, no NaN)
    del flip
    dv = (t & ((1 << 52) - 1)) | (1 << 62)
    mx, mn = dv.view(torch.float64).max(), dv.view(torch.float64).min()
    for op, w in ((A.OP_MAX_F64, mx), (A.OP_MIN_F64, mn)):
        ctx.ck(ctx.L.tg_all_reduce(ctx.h, C.byref(_capi().ScanDesc(8, op)), dv.data_ptr(), n, None, out.ctypes.data))
        assert A._f(int(out[0])) == float(w.item()), op
    ctx.ck(ctx.L.tg_all_reduce(ctx.h, C.byref(_capi().ScanDesc(8, A.OP_SUM_F64)), dv.data_ptr(), n, None, out.ctypes.data))
    # every value is 2 + m * 2^-51 (m < 2^52 the mantissa): the exact sum in units of 2^-51, the mantissas summed in two 26-bit
    # halves so that no int64 partial sum overflows
    m = t & ((1 << 52) - 1)
    exact = (int((m >> 26).sum().item()) << 26) + int((m & ((1 << 26) - 1)).sum().item()) + n * (1 << 52)
    del m
    a = exact
    gm = X.gamma(16 + 31 + -(-X.ntiles(n, 8) // 512) + 1)
    got = A._f(int(out[0]))
    assert abs(int(got * 2.0 ** 51) - exact) <= gm * a + X.U * exact, (got, exact / 2.0 ** 51)      # (got * 2^51 is an integer)
    del dv, t, buf
    torch.cuda.empty_cache()


# ---- several GPUs --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
def test_action_on_n_gpus(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29931 + world), os.path.join(HERE, "multi_gpu_action_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0 and "MULTI_GPU_ACTION_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


# ---- inside a real Thrill job (the GPU nodes against the stock actions) ------------------------------------------------------
HOST_BIN = os.path.join(ROOT, "oracle", "_ref", "host", "gpu_action_test")
HOST_PASS = 6


def _host_run(workers, n):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([HOST_BIN, str(n)], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in res.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert len(lines) == HOST_PASS and all(l.startswith("PASS") for l in lines), lines


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_action_test not built (make -C tests/host -f gpu_action_test.mk)")
def test_action_inside_thrill_single_worker():
    _host_run(1, 9999)


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_action_test not built")
def test_action_inside_thrill_two_workers_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _host_run(2, 200000)
