"""Window on one H100: tg_window, its _file and _select forms and the Python mirror against the stock-fold model of window_ref.py
and the reference's outputs in tests/golden/reference_outputs_window.npz (p = 1, 2, 3, 4, 8 through tg_window_select, and up to
16 simulated workers).  Integer results and Min / Max on doubles are compared bit for bit (NaN bits included); double sums bit
for bit against the emulation of the kernel's bracketing (window_ref.emulate_sum), whose error bound test_window_ref.py checks,
and across shardings.  Every op x item size x form, k from 2 to 4096 with windows and blocks astride the CTA tiles, device Files
in and out, argument errors, the size limits, a 1e8-item case, the multi-GPU worker and the in-Thrill test binary where the
machine has what they need.  pytest -m gpu."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import scan_ref as S
import window_ref as W
from gpu_util import make_blocks

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "reference_outputs_window.npz")
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4
QNAN, NAN_PAYLOAD = 0x7FF8000000000000, 0x7FF8000000012345
KS = [2, 3, 31, 32, 33, 64, 4095, 4096]


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


def host_items(words, pair):
    """(n, 2) words -> the items as they lie in memory"""
    return np.ascontiguousarray(words if pair else words[:, 1])


def rows(raw, pair):
    raw = np.asarray(raw, np.uint64)
    if pair:
        return raw.reshape(-1, 2)
    return np.stack([np.zeros(len(raw), np.uint64), raw], axis=1)


def _download(ctx, dptr, n, pair):
    if not n:
        return np.zeros((0, 2), np.uint64)
    return rows(ctx.download(dptr, n * _ib(pair)).view(np.uint64), pair)


def run_one(ctx, words, op, pair, k, form):
    """tg_window on one worker: the output rows; the input is left intact"""
    items = host_items(words, pair)
    d = ctx.to_device(items) if len(items) else None
    out, n = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_window(ctx.h, C.byref(_capi().ScanDesc(_ib(pair), op)), d, len(items), k, form, C.byref(out), C.byref(n)))
    got = _download(ctx, out.value, n.value, pair)
    if d is not None:
        assert np.array_equal(ctx.download(d, items.nbytes).view(np.uint64), items.view(np.uint64).reshape(-1))
        ctx.free(d)
    return got


def run_select(ctx, words, sizes, op, pair, k, form):
    """workers 0..p-1 through tg_window_select: (concatenated rows, per-worker output counts)"""
    items = host_items(words, pair)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    devs = [ctx.to_device(items[off[r]:off[r + 1]]) if sizes[r] else None for r in range(len(sizes))]
    ptrs = (C.c_void_p * len(sizes))(*devs)
    ns = (C.c_size_t * len(sizes))(*sizes)
    desc = _capi().ScanDesc(_ib(pair), op)
    parts, cnt = [], []
    for r in range(len(sizes)):
        out, n = C.c_void_p(), C.c_size_t()
        ctx.ck(ctx.L.tg_window_select(ctx.h, C.byref(desc), ptrs, ns, len(sizes), r, k, form, C.byref(out), C.byref(n)))
        parts.append(_download(ctx, out.value, n.value, pair))
        cnt.append(n.value)
    for d in devs:
        if d is not None:
            ctx.free(d)
    return np.concatenate(parts), cnt


def check(got, words, op, k, form):
    """the model (integers, Min / Max) or the emulated bracketing (double sums), bit for bit"""
    want = W.outputs(words, op, k, form)
    if op == W.OP_SUM_F64:
        want[:, 1] = W.emulate_sum(words[:, 1], k, form)
    assert W.same(got, want, op), (op, k, form, len(words))


def gen_words(n, seed, op, pair):
    rng = np.random.RandomState(seed)
    if op in W.F64_OPS:
        x = rng.standard_normal(n) * 10.0 ** rng.randint(-20, 20, n)
        v = S.f64_words(x)
        if op != W.OP_SUM_F64:
            v[::37] = NAN_PAYLOAD                      # window firsts and items inside windows
            v[5::41] = QNAN
            v[7::13] = 0                               # +0.0 / -0.0 ties
            v[8::13] = 0x8000000000000000
            v[11::53] = S.f64_words(np.array([np.inf]))[0]
    else:
        v = S.splitmix64(np.arange(n, dtype=np.uint64) + np.uint64(seed))
        v[::3] = rng.randint(0, 50, len(v[::3])).astype(np.uint64)     # ties
    first = S.splitmix64(np.arange(n, dtype=np.uint64) + np.uint64(1000 + seed)) if pair else np.zeros(n, np.uint64)
    return np.stack([first, v], axis=1)


def _sizes(n, p, rng, k):
    """a sharding with small workers (fewer than k - 1 items) and empty ones"""
    if p == 1:
        return [n]
    if p >= 3:                                      # random first, p - 2 small workers, the rest on the last
        small = max(1, (k - 1) // 3)
        a = int(rng.randint(0, max(1, n - small * (p - 2))))
        if a + small * (p - 2) <= n:
            return [a] + [small] * (p - 2) + [n - a - small * (p - 2)]
    cuts = np.sort(rng.randint(0, n + 1, p - 1))
    return list(np.diff(np.concatenate([[0], cuts, [n]])).astype(int))


# ---- every op x item size x form x k -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("form", [W.FULL, W.PARTIAL, W.DISJOINT])
@pytest.mark.parametrize("pair", [False, True])
@pytest.mark.parametrize("op", list(range(6)))
def test_every_op(ctx, op, pair, form, k):
    """one worker, and three simulated ones with small shards; N astride the CTA tiles (4096 items of own blocks for k <= 2048)"""
    n = 3 * 4096 + 2 * k + 17 if k < 4000 else 3 * k + 123
    words = gen_words(n, k + 7 * op, op, pair)
    check(run_one(ctx, words, op, pair, k, form), words, op, k, form)
    rng = np.random.RandomState(op * 100 + k)
    for p in (3, 5):
        sizes = _sizes(n, p, rng, k)
        got, cnt = run_select(ctx, words, sizes, op, pair, k, form)
        assert cnt == W.counts(form, k, sizes)
        check(got, words, op, k, form)


@pytest.mark.parametrize("op", [W.OP_MIN_F64, W.OP_MAX_F64])
def test_nan_first_inside_and_zero_ties(ctx, op):
    """a NaN first item is the output (its bits); a NaN inside is skipped; of +0.0 / -0.0 the earlier wins"""
    v = S.f64_words(np.array([1.0, 2.0, 0.0, -0.0, 3.0, -0.0, 0.0, 4.0, 5.0, 6.0]))
    v[0] = NAN_PAYLOAD
    v[4] = QNAN
    words = np.stack([np.zeros(len(v), np.uint64), v], axis=1)
    for k in (2, 3, 5):
        for form in (W.FULL, W.PARTIAL, W.DISJOINT):
            got = run_one(ctx, words, op, False, k, form)
            assert W.same(got, W.outputs(words, op, k, form), op)
    got = run_one(ctx, words, op, False, 3, W.FULL)
    assert int(got[0, 1]) == NAN_PAYLOAD                       # [NaN, 2, +0]
    assert int(got[2, 1]) == 0                                  # [+0, -0, NaN]: the earlier zero, the NaN skipped


# ---- the reference's fixtures at every simulated worker count -------------------------------------------------------------------
FIX = W.load_fixtures(GOLDEN)


@pytest.mark.parametrize("c", FIX, ids=[c["name"] for c in FIX])
def test_fixtures(ctx, c):
    for p in W.WORKERS:
        got, cnt = run_select(ctx, c["items"], c["shards"][p], c["op"], c["pair"], c["k"], c["form"])
        assert cnt == c["counts"][p], p
        if c["op"] == W.OP_SUM_F64:
            # the stock left fold within the bound (test_window_ref.py), the kernel's bracketing bit for bit
            check(got, c["items"], c["op"], c["k"], c["form"])
            assert W.bound_violations(got[:, 1], c["items"][:, 1], c["k"], c["form"]) == []
            assert np.array_equal(got[:, 0], c["out"][:, 0])
        else:
            assert W.same(got, c["out"], c["op"]), p


@pytest.mark.parametrize("form", [W.FULL, W.PARTIAL, W.DISJOINT])
def test_shardings_give_identical_bytes(ctx, form):
    """one input, p = 1 .. 16 and several shardings: byte-identical concatenated outputs, double sums included"""
    for op in (W.OP_SUM_F64, W.OP_MAX_U64):
        for k in (5, 64, 4096):
            n = 3 * k + 4099
            words = gen_words(n, k, op, True)
            ref = run_one(ctx, words, op, True, k, form)
            rng = np.random.RandomState(k + form)
            for p in (1, 2, 4, 7, 16):
                got, _ = run_select(ctx, words, _sizes(n, p, rng, k), op, True, k, form)
                assert np.array_equal(got, ref), (op, k, p)


# ---- Files, device Files, the Python mirror --------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", [False, True])
def test_file_host_and_device(ctx, pair):
    capi = _capi()
    ib = _ib(pair)
    op, k, form = W.OP_SUM_F64, 33, W.PARTIAL
    words = gen_words(50001, 3, op, pair)
    items = host_items(words, pair)
    want = run_one(ctx, words, op, pair, k, form)
    desc = capi.ScanDesc(ib, op)
    n = C.c_size_t()
    blocks, nb, keep = make_blocks(capi, items, 1000)
    inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
    ctx.ck(ctx.L.tg_window_file(ctx.h, C.byref(desc), C.byref(inp), k, form, C.byref(n)))
    assert n.value == len(want)
    out = np.zeros(n.value * ib, np.uint8)
    ob, onb, _ = make_blocks(capi, out, 4096)
    ctx.ck(ctx.L.tg_fetch_output(ctx.h, C.cast(ob, C.POINTER(capi.Block)), onb))
    assert np.array_equal(rows(out.view(np.uint64), pair), want)
    # a device File in: read in place and left intact, nothing crosses PCIe; the result detached as a device File
    d = ctx.to_device(items)
    f = capi.DevFile(d, len(items), ib, 0)
    h0, d0 = C.c_uint64(), C.c_uint64()
    ctx.L.tg_transfer_bytes(ctx.h, C.byref(h0), C.byref(d0))
    ctx.ck(ctx.L.tg_window_file(ctx.h, C.byref(desc), C.byref(capi.MergeInput(C.pointer(f), None, 0)), k, form, C.byref(n)))
    det = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(det)))
    h1, d1 = C.c_uint64(), C.c_uint64()
    ctx.L.tg_transfer_bytes(ctx.h, C.byref(h1), C.byref(d1))
    assert (h1.value, d1.value) == (h0.value, d0.value)
    assert det.item_bytes == ib and det.items == len(want)
    # the detached result is an input of its own (a Window of a Window)
    ctx.ck(ctx.L.tg_window_file(ctx.h, C.byref(desc), C.byref(capi.MergeInput(C.pointer(det), None, 0)), 2, W.DISJOINT,
                                C.byref(n)))
    det2 = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(det2)))
    assert W.same(_download(ctx, det2.dptr, n.value, pair), run_one(ctx, want, op, pair, 2, W.DISJOINT), op)
    ctx.L.tg_dev_file_free(ctx.h, C.byref(det2))
    assert np.array_equal(_download(ctx, det.dptr, len(want), pair), want)
    assert np.array_equal(ctx.download(d, items.nbytes).view(np.uint64), items.view(np.uint64).reshape(-1))
    ctx.L.tg_dev_file_free(ctx.h, C.byref(det))
    ctx.free(d)


def test_python_mirror():
    from thrill_b200 import api
    c = api.Context(rank=0, nranks=1, device=0, rng_seed=3)
    try:
        u = gen_words(20000, 1, W.OP_MAX_U64, False)
        r = api.DIA(c, u[:, 1].copy()).Window(64, api.MaxU64).items
        assert np.array_equal(rows(r, False), W.outputs(u, W.OP_MAX_U64, 64, W.FULL))
        f = gen_words(20000, 2, W.OP_MIN_F64, False)
        r = api.DIA(c, f[:, 1].view(np.float64).copy()).Window(5, api.MinDouble, partial=True).items
        assert W.same(rows(r.view(np.uint64), False), W.outputs(f, W.OP_MIN_F64, 5, W.PARTIAL), W.OP_MIN_F64)
        kv = gen_words(20000, 3, W.OP_SUM_F64, True)
        r = api.DIA(c, kv.copy().view(api.KV).reshape(-1)).Window(7, api.ScanSecond(api.PlusDouble), disjoint=True).items
        want = W.outputs(kv, W.OP_SUM_F64, 7, W.DISJOINT)
        want[:, 1] = W.emulate_sum(kv[:, 1], 7, W.DISJOINT)
        assert W.same(r.view(np.uint64).reshape(-1, 2), want, W.OP_SUM_F64)
        with pytest.raises(Exception):
            api.DIA(c, u[:, 1].copy()).Window(1, api.PlusU64)
        with pytest.raises(Exception):
            api.DIA(c, u[:, 1].copy()).Window(4, api.PlusDouble)
    finally:
        c.close()


# ---- errors and the size limits ------------------------------------------------------------------------------------------------
def test_argument_errors(ctx):
    capi = _capi()
    d = ctx.to_device(np.arange(8, dtype=np.uint64))
    out, n = C.c_void_p(), C.c_size_t()
    desc = capi.ScanDesc(8, W.OP_SUM_U64)
    for k in (0, 1, 4097, 1 << 31):
        assert ctx.L.tg_window(ctx.h, C.byref(desc), d, 8, k, W.FULL, C.byref(out), C.byref(n)) == TG_ERR_ARG, k
    for ib, op in [(8, 6), (16, 6), (8, 7), (4, 1), (24, 1), (0, 1), (12, 4)]:
        assert ctx.L.tg_window(ctx.h, C.byref(capi.ScanDesc(ib, op)), d, 2, 2, W.FULL, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert ctx.L.tg_window(ctx.h, C.byref(desc), d, 8, 2, 3, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert ctx.L.tg_window(ctx.h, None, d, 8, 2, W.FULL, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert ctx.L.tg_window(ctx.h, C.byref(desc), None, 8, 2, W.FULL, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert ctx.L.tg_window_file(ctx.h, C.byref(desc), None, 2, W.FULL, C.byref(n)) == TG_ERR_ARG
    ptrs = (C.c_void_p * 17)(*([d] * 17))
    ns = (C.c_size_t * 17)(*([2] * 17))
    for p, r in ((0, 0), (17, 0), (2, 2)):
        assert ctx.L.tg_window_select(ctx.h, C.byref(desc), ptrs, ns, p, r, 2, W.FULL, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert ctx.L.tg_window_select(ctx.h, C.byref(desc), ptrs, ns, 2, 0, 4097, W.FULL, C.byref(out), C.byref(n)) == TG_ERR_ARG
    ptrs[1] = None
    assert ctx.L.tg_window_select(ctx.h, C.byref(desc), ptrs, ns, 2, 0, 2, W.FULL, C.byref(out), C.byref(n)) == TG_ERR_ARG
    f16 = capi.DevFile(d, 2, 16, 0)
    assert ctx.L.tg_window_file(ctx.h, C.byref(desc), C.byref(capi.MergeInput(C.pointer(f16), None, 0)), 2, W.FULL,
                                C.byref(n)) == TG_ERR_ARG
    ctx.free(d)
    words = gen_words(100, 1, W.OP_SUM_U64, False)
    check(run_one(ctx, words, W.OP_SUM_U64, False, 3, W.FULL), words, W.OP_SUM_U64, 3, W.FULL)     # the ctx still works


def test_size_limits(ctx):
    """2^30 items on a worker, or 2^30 outputs on the last one (n + k - 1 for a partial Window), are refused before any read"""
    capi = _capi()
    d = ctx.to_device(np.arange(8192, dtype=np.uint64))
    out, n = C.c_void_p(), C.c_size_t()
    for ib in (8, 16):
        desc = capi.ScanDesc(ib, W.OP_SUM_U64)
        assert ctx.L.tg_window(ctx.h, C.byref(desc), d, 1 << 30, 2, W.FULL, C.byref(out), C.byref(n)) == TG_ERR_TOO_LARGE
        ptrs = (C.c_void_p * 3)(d, d, d)
        for r in range(3):
            ns = (C.c_size_t * 3)(1, 1 << 30, 1)
            assert ctx.L.tg_window_select(ctx.h, C.byref(desc), ptrs, ns, 3, r, 2, W.FULL, C.byref(out),
                                          C.byref(n)) == TG_ERR_TOO_LARGE
            # the last worker holds 2^30 - 1 items after 4095 others: a partial Window would give it 2^30 + 4094 outputs
            ns = (C.c_size_t * 3)(4095, 0, (1 << 30) - 1)
            assert ctx.L.tg_window_select(ctx.h, C.byref(desc), ptrs, ns, 3, r, 4096, W.PARTIAL, C.byref(out),
                                          C.byref(n)) == TG_ERR_TOO_LARGE
    ctx.free(d)
    words = gen_words(100, 1, W.OP_SUM_U64, False)
    check(run_one(ctx, words, W.OP_SUM_U64, False, 3, W.FULL), words, W.OP_SUM_U64, 3, W.FULL)


# ---- scale ---------------------------------------------------------------------------------------------------------------------
def test_1e8_items(ctx):
    """1e8 uint64_t: the sliding sums (k = 64) against the model by a full comparison (prefix sums mod 2^64), the maxima
    (k = 4096) at sampled positions, and the disjoint sums by checksum"""
    n = 100_000_000
    x = S.splitmix64(np.arange(n, dtype=np.uint64))
    d = ctx.to_device(x)
    desc = lambda op: C.byref(_capi().ScanDesc(8, op))      # noqa: E731
    out, m = C.c_void_p(), C.c_size_t()
    cs = np.concatenate([[np.uint64(0)], np.cumsum(x, dtype=np.uint64)])
    ctx.ck(ctx.L.tg_window(ctx.h, desc(W.OP_SUM_U64), d, n, 64, W.FULL, C.byref(out), C.byref(m)))
    assert m.value == n - 63
    got = ctx.download(out.value, m.value * 8).view(np.uint64)
    assert np.array_equal(got, cs[64:] - cs[:-64])
    del got
    ctx.ck(ctx.L.tg_window(ctx.h, desc(W.OP_SUM_U64), d, n, 4096, W.DISJOINT, C.byref(out), C.byref(m)))
    got = ctx.download(out.value, m.value * 8).view(np.uint64)
    ends = np.append(np.arange(4096, n + 1, 4096), n)
    starts = np.append(np.arange(0, n - 4095, 4096), n - n % 4096)
    assert m.value == len(ends) and np.array_equal(got, cs[ends] - cs[starts])
    ctx.ck(ctx.L.tg_window(ctx.h, desc(W.OP_MAX_U64), d, n, 4096, W.PARTIAL, C.byref(out), C.byref(m)))
    assert m.value == n
    got = ctx.download(out.value, m.value * 8).view(np.uint64)
    rng = np.random.RandomState(1)
    for i in np.concatenate([rng.randint(0, n - 4095, 2000), [0, n - 4096], np.arange(n - 4095, n)]):
        want = x[i:i + 4096].max()
        assert got[i] == want, i
    ctx.free(d)


# ---- several GPUs --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
def test_window_on_n_gpus(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29961 + world), os.path.join(HERE, "multi_gpu_window_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0 and "MULTI_GPU_WINDOW_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


# ---- inside a real Thrill job (GpuWindowNode against the stock Window) ---------------------------------------------------------
HOST_BIN = os.path.join(ROOT, "oracle", "_ref", "host", "gpu_window_test")


def _host_run(workers, n):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([HOST_BIN, str(n)], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in res.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert lines and all(l.startswith("PASS") for l in lines), lines


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_window_test not built (make -C tests/host -f gpu_window_test.mk)")
def test_window_inside_thrill_single_worker():
    _host_run(1, 9999)


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_window_test not built")
def test_window_inside_thrill_two_workers_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _host_run(2, 200000)
