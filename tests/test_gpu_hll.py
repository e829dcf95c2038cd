"""HyperLogLog on one H100: tg_hyperloglog, its _file and _select forms and the Python mirror against the numpy model in hll_ref.py
(SipHash-2-4 and the dense register rule) and against the reference's registers in tests/golden/reference_outputs_hll.npz, bit for
bit: the registers are a max over the items, so one run against the model is the whole check.  Every precision 4..18 and both item
sizes, tile edges, an odd number of 8-byte items, 1e7 items, p = 1..16 workers simulated on one GPU, host and device Files,
argument errors, the size limit, the multi-GPU worker and the in-Thrill test binary where the machine has what they need.
A hash whose low 64 - p bits are all zero (the w == 0 branch of the register rule) cannot be found by searching items: the odds
are 2^(p - 64) per item.  The model is pinned on such hashes against the reference's insert_hash (test_hll_ref.py); the kernel
computes min(clz(h << p), 64 - p) + 1, which has no branch to miss.  pytest -m gpu."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import hll_ref as H
from gpu_util import make_blocks

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "reference_outputs_hll.npz")
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4
TILE = {8: 4096, 16: 2048}                 # items per 32 KB tile of the update kernel
PRECISIONS = list(range(4, 19))


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def golden():
    return H.Golden(GOLDEN)


def items_of(n, ib, seed):
    """n all-distinct items as words: consecutive integers from a seed-dependent start (SipHash does the mixing)"""
    return np.uint64(seed << 40) + np.arange(n * (ib // 8), dtype=np.uint64)


def hll_dev(ctx, words, ib, p):
    """tg_hyperloglog of a host array on one worker: (status, registers); the input is read, never modified"""
    n = len(words) // (ib // 8)
    d = ctx.to_device(words)
    out = np.full(1 << p, 0xEE, np.uint8)
    st = ctx.L.tg_hyperloglog(ctx.h, ib, p, d, n, out.ctypes.data)
    if st == 0 and n:
        assert np.array_equal(ctx.download(d, n * ib).view(np.uint64), words)
    ctx.free(d)
    return st, out


def select(ctx, shards, ib, p):
    devs = [ctx.to_device(s) for s in shards]
    ptrs = (C.c_void_p * len(shards))(*devs)
    ns = (C.c_size_t * len(shards))(*[len(s) // (ib // 8) for s in shards])
    out = np.full(1 << p, 0xEE, np.uint8)
    ctx.ck(ctx.L.tg_hyperloglog_select(ctx.h, ib, p, ptrs, ns, len(shards), out.ctypes.data))
    for d in devs:
        ctx.free(d)
    return out


def one(ctx, words, ib, p, hashes=None):
    st, regs = hll_dev(ctx, words, ib, p)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    want = H.registers_from_hashes(hashes, p) if hashes is not None else H.registers(words, ib, p)
    assert np.array_equal(regs, want), (ib, p, len(words), np.flatnonzero(regs != want)[:5])
    return regs


# ---- one worker: every precision and item size ---------------------------------------------------------------------------------
@pytest.mark.parametrize("ib", [8, 16])
@pytest.mark.parametrize("p", PRECISIONS)
def test_every_precision(ctx, p, ib):
    t = TILE[ib]
    for n in (0, 1, 2, 3, t - 1, t, t + 1, 5 * t + 3, 100001):
        regs = one(ctx, items_of(n, ib, n + 1), ib, p)
        if n == 0:
            assert not regs.any()
        if n == 1:
            assert np.count_nonzero(regs) == 1
    # heavy duplicates: 50 distinct items, and one item 20000 times (exactly one non-zero register)
    pool = items_of(50, ib, 3).reshape(50, ib // 8)
    one(ctx, pool[np.random.RandomState(p).randint(0, 50, 30000)].reshape(-1), ib, p)
    assert np.count_nonzero(one(ctx, np.tile(items_of(1, ib, 9), 20000), ib, p)) == 1


@pytest.mark.parametrize("ib", [8, 16])
def test_ten_million_items(ctx, ib):
    """many tiles per CTA, every register raised many times; one SipHash pass of the model serves every precision"""
    words = items_of(10 ** 7, ib, 77)
    hashes = H.siphash24(words, ib)
    for p in (4, 11, 16, 17, 18):
        one(ctx, words, ib, p, hashes)


def test_doubles_are_hashed_as_bits(ctx):
    d = np.array([0.0, -0.0, 1.5, np.nan, np.inf, -1.5, 1e-310] * 300, np.float64)
    one(ctx, d.view(np.uint64), 8, 10)


# ---- the reference's registers ---------------------------------------------------------------------------------------------------
def test_registers_equal_the_reference(ctx, golden):
    checked = 0
    for i, name in enumerate(golden.names):
        if golden.mode(i) == "hash":
            continue
        words, ib = golden.words(i), golden.item_bytes(i)
        for p in golden.precisions:
            st, regs = hll_dev(ctx, np.ascontiguousarray(words), ib, p)
            assert st == 0, ctx.L.tg_last_error(ctx.h)
            assert np.array_equal(H.digest(regs), golden.digest(i, p)), (name, p)
            stored = golden.regs(i, p)
            if stored is not None:
                assert np.array_equal(regs, stored), (name, p)
            if name.endswith("all_equal"):
                assert np.count_nonzero(regs) == 1
            checked += 1
    assert checked >= 70


# ---- several workers simulated on one GPU ------------------------------------------------------------------------------------
def test_simulated_workers_equal_one_worker(ctx, golden):
    """the fixture's shard layouts (1, 2, 3, 4 and 8 workers, empty shards among them): the registers of the concatenation"""
    for i, name in enumerate(golden.names):
        if golden.mode(i) == "hash":
            continue
        words, ib = np.ascontiguousarray(golden.words(i)), golden.item_bytes(i)
        for p in (4, 12, 17, 18):
            whole = None
            for _, _, counts in golden.layouts(i):
                got = select(ctx, H.shards_of(words, ib, counts), ib, p)
                whole = got if whole is None else whole          # (the first layout is one worker)
                assert np.array_equal(got, whole), (name, p, counts)
            if p in golden.precisions:
                assert np.array_equal(H.digest(whole), golden.digest(i, p)), (name, p)


@pytest.mark.parametrize("ib", [8, 16])
def test_one_to_sixteen_workers(ctx, ib):
    n = 16 * 3000 + 7
    words = items_of(n, ib, 16)
    for p in (5, 14, 18):
        want = H.registers(words, ib, p)
        for workers in range(1, 17):
            counts = [n // workers] * workers
            counts[-1] += n - sum(counts)
            assert np.array_equal(select(ctx, H.shards_of(words, ib, counts), ib, p), want), (p, workers)
        # empty workers first, last and in between, tile-crossing shards
        counts = [0, 5000, 1, 0, 4096, 4097, 2047, 0, 9000, 3, 2048, 6000, 0, 7000, 1] + [0]
        counts[-2] += n - sum(counts)
        assert np.array_equal(select(ctx, H.shards_of(words, ib, counts), ib, p), want), p


# ---- the _file form, device Files, the Python mirror ---------------------------------------------------------------------------
@pytest.mark.parametrize("ib", [8, 16])
def test_file_host_and_device(ctx, ib):
    capi = _capi()
    words = items_of(60001, ib, 5)
    for p in (4, 13, 18):
        want = H.registers(words, ib, p)
        out = np.zeros(1 << p, np.uint8)
        # a host File with Blocks that cut items
        blocks, nb, keep = make_blocks(capi, words, 1000)
        inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
        ctx.ck(ctx.L.tg_hyperloglog_file(ctx.h, ib, p, C.byref(inp), out.ctypes.data))
        assert np.array_equal(out, want)
        # a device File: read in place, left intact; nothing but the registers crosses PCIe (not through the File codec)
        d = ctx.to_device(words)
        f = capi.DevFile(d, len(words) // (ib // 8), ib, 0)
        h0, d0 = C.c_uint64(), C.c_uint64()
        ctx.L.tg_transfer_bytes(ctx.h, C.byref(h0), C.byref(d0))
        out[:] = 0
        ctx.ck(ctx.L.tg_hyperloglog_file(ctx.h, ib, p, C.byref(capi.MergeInput(C.pointer(f), None, 0)), out.ctypes.data))
        h1, d1 = C.c_uint64(), C.c_uint64()
        ctx.L.tg_transfer_bytes(ctx.h, C.byref(h1), C.byref(d1))
        assert h1.value == h0.value and d1.value - d0.value <= (1 << p)
        assert np.array_equal(out, want)
        assert np.array_equal(ctx.download(d, len(words) * 8).view(np.uint64), words)
        ctx.free(d)
    # an empty host File
    out = np.full(16, 7, np.uint8)
    ctx.ck(ctx.L.tg_hyperloglog_file(ctx.h, ib, 4, C.byref(capi.MergeInput(None, None, 0)), out.ctypes.data))
    assert not out.any()


def test_python_mirror():
    from thrill_b200 import api, capi
    c = api.Context(rank=0, nranks=1, device=0, rng_seed=3)
    try:
        x = items_of(20000, 8, 8)
        assert np.array_equal(api.DIA(c, x).HyperLogLog(12), H.registers(x, 8, 12))
        f = np.arange(1000, dtype=np.float64) / 8.0
        assert np.array_equal(api.DIA(c, f).HyperLogLog(6), H.registers(f.view(np.uint64), 8, 6))
        kv = items_of(5000, 16, 2)
        assert np.array_equal(api.DIA(c, kv.view(api.KV)).HyperLogLog(18), H.registers(kv, 16, 18))
        assert not api.DIA(c, x[:0]).HyperLogLog(4).any()
        for bad in (3, 19):
            with pytest.raises(capi.ThrillGpuError):
                api.DIA(c, x).HyperLogLog(bad)
        with pytest.raises(capi.ThrillGpuError):
            api.DIA(c, x.astype(np.uint32)).HyperLogLog(8)
    finally:
        c.close()


# ---- errors and the size limit -----------------------------------------------------------------------------------------------
def test_argument_errors(ctx):
    capi = _capi()
    d = ctx.to_device(np.arange(4, dtype=np.uint64))
    out = np.zeros(1 << 18, np.uint8)
    for ib, p in [(8, 3), (8, 19), (16, 0), (8, 64), (4, 8), (24, 8), (0, 8), (12, 8)]:
        assert ctx.L.tg_hyperloglog(ctx.h, ib, p, d, 2, out.ctypes.data) == TG_ERR_ARG, (ib, p)
    assert ctx.L.tg_hyperloglog(ctx.h, 8, 8, None, 2, out.ctypes.data) == TG_ERR_ARG
    assert ctx.L.tg_hyperloglog(ctx.h, 8, 8, d, 2, None) == TG_ERR_ARG
    assert ctx.L.tg_hyperloglog_file(ctx.h, 8, 8, None, out.ctypes.data) == TG_ERR_ARG
    ptrs = (C.c_void_p * 17)(*([d] * 17))
    ns = (C.c_size_t * 17)(*([2] * 17))
    assert ctx.L.tg_hyperloglog_select(ctx.h, 8, 8, ptrs, ns, 0, out.ctypes.data) == TG_ERR_ARG
    assert ctx.L.tg_hyperloglog_select(ctx.h, 8, 8, ptrs, ns, 17, out.ctypes.data) == TG_ERR_ARG
    assert ctx.L.tg_hyperloglog_select(ctx.h, 8, 2, ptrs, ns, 2, out.ctypes.data) == TG_ERR_ARG
    ptrs[1] = None
    assert ctx.L.tg_hyperloglog_select(ctx.h, 8, 8, ptrs, ns, 2, out.ctypes.data) == TG_ERR_ARG
    f16 = capi.DevFile(d, 2, 16, 0)                          # a device File of 16-byte items hashed as 8-byte items
    assert ctx.L.tg_hyperloglog_file(ctx.h, 8, 8, C.byref(capi.MergeInput(C.pointer(f16), None, 0)), out.ctypes.data) == TG_ERR_ARG
    raw = np.zeros(20, np.uint8)                            # 20 bytes: not whole items
    ob, onb, _ = make_blocks(capi, raw, 20)
    assert ctx.L.tg_hyperloglog_file(ctx.h, 8, 8, C.byref(capi.MergeInput(None, C.cast(ob, C.POINTER(capi.Block)), onb)),
                                     out.ctypes.data) == TG_ERR_ARG
    ctx.free(d)
    one(ctx, np.arange(10, dtype=np.uint64), 8, 8)            # the ctx still works


def test_input_over_the_limit_is_too_large(ctx):
    d = ctx.to_device(np.arange(2, dtype=np.uint64))
    out = np.zeros(256, np.uint8)
    # 2^30 items are refused before anything is read (the buffer holds two)
    for ib in (8, 16):
        assert ctx.L.tg_hyperloglog(ctx.h, ib, 8, d, 1 << 30, out.ctypes.data) == TG_ERR_TOO_LARGE
        ptrs = (C.c_void_p * 3)(d, d, d)
        ns = (C.c_size_t * 3)(1, 1 << 30, 1)
        assert ctx.L.tg_hyperloglog_select(ctx.h, ib, 8, ptrs, ns, 3, out.ctypes.data) == TG_ERR_TOO_LARGE
    ctx.free(d)
    one(ctx, np.arange(10, dtype=np.uint64), 8, 8)


def test_kernel_is_timed_under_its_profile_class(ctx):
    capi = _capi()
    before = ctx.profile_get(capi.K_HLL)[1]
    ctx.profile_enable(True)
    try:
        one(ctx, items_of(50000, 8, 1), 8, 12)
        ms, launches = ctx.profile_get(capi.K_HLL)
        assert launches == before + 1 and ms > 0
    finally:
        ctx.profile_enable(False)


# ---- several GPUs --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
def test_hll_on_n_gpus(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29951 + world), os.path.join(HERE, "multi_gpu_hll_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0 and "MULTI_GPU_HLL_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


# ---- inside a real Thrill job (the GPU node against the stock node) ----------------------------------------------------------
HOST_BIN = os.path.join(ROOT, "oracle", "_ref", "host", "gpu_hll_test")
HOST_PASS = 15


def _host_run(workers, n):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([HOST_BIN, str(n)], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in res.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert len(lines) == HOST_PASS and all(l.startswith("PASS") for l in lines), lines
    return lines


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_hll_test not built (make -C tests/host -f gpu_hll_test.mk)")
def test_hll_inside_thrill_single_worker():
    small = _host_run(1, 9999)             # the stock node is still sparse at the larger precisions
    large = _host_run(1, 400000)           # ... and dense at every precision
    assert any("ends sparse" in l for l in small) and any("ends dense" in l for l in small)
    assert sum("ends dense" in l for l in large) > sum("ends dense" in l for l in small)


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_hll_test not built")
def test_hll_inside_thrill_two_workers_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _host_run(2, 9999)
    _host_run(2, 400000)
