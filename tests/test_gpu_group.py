"""GroupByKey / GroupToIndex on one H100: tg_group_by_key, tg_group_to_index, their _file forms and the Python mirror against
the numpy restatement in group_ref.py (bit-exact: sorted by key, stable within a key) and against the reference's outputs in
tests/golden/reference_outputs_group.npz (p = 2, 3, 4 and 8 workers simulated on one GPU through the real exchange are in
test_gpu_exchange.py); device Files, argument errors and the size limit, a full-size case, the multi-GPU worker and the
in-Thrill test binary where the machine has what they need.  pytest -m gpu."""
import ctypes as C
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import group_ref as G
from gpu_util import make_blocks

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "reference_outputs_group.npz")
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


def _download(ctx, dptr, n):
    return ctx.download(dptr, n * 16).view(G.KV) if n else np.zeros(0, G.KV)


def group_dev(ctx, arr, size=None):
    """tg_group_by_key (size None) or tg_group_to_index of a host KV array on one worker: (status, result, begin, end)"""
    d = ctx.to_device(arr)
    out, n, b, e = C.c_void_p(), C.c_size_t(), C.c_uint64(), C.c_uint64()
    if size is None:
        st = ctx.L.tg_group_by_key(ctx.h, d, len(arr), C.byref(out), C.byref(n))
    else:
        st = ctx.L.tg_group_to_index(ctx.h, d, len(arr), size, C.byref(out), C.byref(n), C.byref(b), C.byref(e))
    res = _download(ctx, out.value, n.value) if st == 0 else None
    if st == 0:       # the input is read, never modified
        assert np.array_equal(_download(ctx, d, len(arr)), arr)
    ctx.free(d)
    return st, res, b.value, e.value


def check(ctx, arr, size=None):
    st, res, b, e = group_dev(ctx, arr, size)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    assert np.array_equal(res.view(np.uint64), G.grouped(arr).view(np.uint64))
    if size is not None:
        assert (b, e) == (0, size)
    return res


# ---- exact results, one worker --------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,universe", [(1, 1), (7, 3), (1000, 10), (50000, 1 << 40), (100000, 1000), (300000, 1 << 26),
                                        (1 << 20, 7)])
def test_group_random(ctx, n, universe):
    arr = G.make_input(n, universe, n + 3)
    check(ctx, arr)
    check(ctx, arr, universe)


@pytest.mark.parametrize("n", [8191, 8192, 8193, 16383, 16384, 16385, 3 * 8192 + 1])
def test_group_tile_edges(ctx, n):
    # the partition pass's tiles hold 8192 pairs (16384 items in two rounds); runs of equal keys straddle them
    rng = np.random.RandomState(n)
    check(ctx, G.pairs(rng.randint(0, n // 5 + 1, n), np.arange(n)))
    check(ctx, G.pairs(np.arange(n) // 700, rng.randint(0, 1 << 62, n)), n // 700 + 1)
    check(ctx, G.pairs(np.full(n, 9), np.arange(n)))


def test_group_edge_keys(ctx):
    st, res, _, _ = group_dev(ctx, np.zeros(0, G.KV))
    assert st == 0 and len(res) == 0
    st, res, b, e = group_dev(ctx, np.zeros(0, G.KV), 10)
    assert st == 0 and len(res) == 0 and (b, e) == (0, 10)
    check(ctx, G.pairs([0, 0, 5, (1 << 64) - 1, 1 << 63, 0], np.arange(6)))
    check(ctx, G.pairs(np.zeros(3000), np.arange(3000)), 1)


def test_heavy_duplicates_take_the_lsd_fallback():
    """2000 random 64-bit keys, 150 items each: the prefix sort gives up and sorts by plain LSD passes, stably"""
    c = _capi().Ctx(0)
    try:
        rng = np.random.RandomState(12)
        pool = rng.randint(0, 2**63 - 1, size=2000, dtype=np.int64).astype(np.uint64)
        keys = np.repeat(pool, 150)
        rng.shuffle(keys)
        arr = G.pairs(keys, np.arange(len(keys)))
        before = c.L.tg_prefix_sort_fallbacks(c.h)
        check(c, arr)
        assert c.L.tg_prefix_sort_fallbacks(c.h) == before + 1
    finally:
        c.close()


# ---- the reference's outputs -------------------------------------------------------------------------------------------
def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/reference_outputs_group.npz is not present")
    return np.load(GOLDEN)


def _cases(g, p):
    out = []
    for k in g.files:
        if k.endswith("/in") or k.endswith("_counts"):
            continue
        name, rest = k.split("/")
        case, q = rest.rsplit("_p", 1)
        if int(q) == p:
            out.append((name, case))
    return sorted(out)


def _same(rows, ref):
    if ref.dtype == np.uint8:
        return hashlib.sha256(np.ascontiguousarray(rows, np.uint64).tobytes()).digest() == ref.tobytes()
    return np.array_equal(rows, ref.reshape(-1, 7))


def _rows(grouped, case, p, d):
    """the host loop over worker d's grouped items"""
    if case.startswith("key_"):
        return G.group_rows(grouped, case[4:], d)
    return G.index_rows(grouped, int(case[6:]), p, d)


def test_fixture_shapes_one_worker(ctx):
    g = _golden()
    for name, case in _cases(g, 1):
        inp = g[name + "/in"].view(G.KV)
        size = None if case.startswith("key_") else int(case[6:])
        st, res, _, _ = group_dev(ctx, inp, size)
        assert st == 0, (name, case, ctx.L.tg_last_error(ctx.h))
        rows = _rows(res, case, 1, 0)
        assert [len(rows)] == g["%s/%s_p1_counts" % (name, case)].tolist()
        assert _same(rows, g["%s/%s_p1" % (name, case)]), (name, case)


# ---- the _file form, device Files, the Python mirror --------------------------------------------------------------------
def _run_file(ctx, inp, size):
    n, b, e = C.c_size_t(), C.c_uint64(), C.c_uint64()
    if size is None:
        ctx.ck(ctx.L.tg_group_by_key_file(ctx.h, C.byref(inp), C.byref(n)))
    else:
        ctx.ck(ctx.L.tg_group_to_index_file(ctx.h, C.byref(inp), size, C.byref(n), C.byref(b), C.byref(e)))
        assert (b.value, e.value) == (0, size)
    return n.value


@pytest.mark.parametrize("size", [None, 5000])
def test_group_file_host_device_and_detached(ctx, size):
    capi = _capi()
    arr = G.make_input(60000, 5000, 41)
    ref = G.grouped(arr)
    # a host File with Blocks that cut items
    blocks, nb, keep = make_blocks(capi, arr, 1000)
    inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
    n = _run_file(ctx, inp, size)
    out = np.empty(n * 16, np.uint8)
    ob, onb, _ = make_blocks(capi, out, 1 << 16)
    ctx.ck(ctx.L.tg_fetch_output(ctx.h, ob, onb))
    assert np.array_equal(out.view(G.KV).view(np.uint64), ref.view(np.uint64))
    # a device File: read in place, left intact, nothing crosses PCIe; the result detached as a device File
    d = ctx.to_device(arr)
    f = capi.DevFile(d, len(arr), 16, 0)
    h0, d0 = C.c_uint64(), C.c_uint64()
    ctx.L.tg_transfer_bytes(ctx.h, C.byref(h0), C.byref(d0))
    n = _run_file(ctx, capi.MergeInput(C.pointer(f), None, 0), size)
    det = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(det)))
    h1, d1 = C.c_uint64(), C.c_uint64()
    ctx.L.tg_transfer_bytes(ctx.h, C.byref(h1), C.byref(d1))
    assert (h1.value, d1.value) == (h0.value, d0.value)
    assert det.item_bytes == 16 and det.items == n == len(arr)
    # the detached result is an input of its own: group it again (already grouped: unchanged)
    n2 = _run_file(ctx, capi.MergeInput(C.pointer(det), None, 0), size)
    assert n2 == n
    assert np.array_equal(_download(ctx, det.dptr, n), ref)
    assert np.array_equal(_download(ctx, d, len(arr)), arr)
    ctx.L.tg_dev_file_free(ctx.h, C.byref(det))
    ctx.free(d)


def test_python_group_operators():
    from thrill_b200 import api, capi
    c = api.Context(rank=0, nranks=1, device=0, rng_seed=3)
    try:
        arr = G.make_input(20000, 700, 51)
        ref = G.group_rows(G.grouped(arr), G.STATS, 0)
        dt = np.dtype([("key", "<u8"), ("count", "<u8"), ("sum", "<u8")])

        def stats(it, key):
            cnt, s = 0, 0
            while it.HasNext():
                k, v = it.Next()
                assert k == key
                cnt, s = cnt + 1, (s + v) % (1 << 64)
            return key, cnt, s

        out = api.DIA(c, arr.view(api.KV)).GroupByKey(api.KeyIsFirst, stats, dt).items
        assert out["key"].tolist() == ref[:, 1].tolist() and out["count"].tolist() == ref[:, 2].tolist()
        assert out["sum"].tolist() == ref[:, 3].tolist()

        def partial(it, key):
            r = 0
            while r < 3 and it.HasNext():
                it.Next()
                r += 1
            return key, r, 0

        out = api.DIA(c, arr.view(api.KV)).GroupByKey(api.KeyIsFirst, partial, dt).items
        pref = G.group_rows(G.grouped(arr), G.PARTIAL, 0)
        assert out["key"].tolist() == pref[:, 1].tolist() and out["count"].tolist() == pref[:, 2].tolist()

        res = api.DIA(c, arr.view(api.KV)).GroupToIndex(api.KeyIsFirst, stats, 1000, (0, 0, 0), dt)
        assert res.index_begin == 0 and len(res.items) == 1000
        full = G.index_rows(G.grouped(arr), 1000, 1, 0)
        present = full[:, 1] != np.uint64(G.U64_MAX)
        assert res.items["count"].tolist() == np.where(present, full[:, 2], 0).tolist()
        with pytest.raises(capi.ThrillGpuError):
            api.DIA(c, arr.view(api.KV)).GroupToIndex(api.KeyIsFirst, stats, 699, (0, 0, 0), dt)
        with pytest.raises(capi.ThrillGpuError):
            api.DIA(c, arr.view(api.KV)).GroupByKey(api.Less, stats, dt)
        with pytest.raises(capi.ThrillGpuError):
            api.DIA(c, np.arange(10, dtype=np.uint64)).GroupByKey(api.KeyIsFirst, stats, dt)
    finally:
        c.close()


# ---- errors and the size limit -----------------------------------------------------------------------------------------
def _mod_exchange(ctx, d, n, p):
    """tg_exchange_select by key % p, counts only: shard 0 holds n items at d, the other shards are empty"""
    q = max(p, 1)
    counts = (C.c_uint64 * (q * q))()
    return ctx.L.tg_exchange_select(ctx.h, _capi().ROUTE_MOD, 1, None, 0, 0, (C.c_void_p * q)(d, *([None] * (q - 1))),
                                    (C.c_size_t * q)(n, *([0] * (q - 1))), p, None, None, counts)


def test_argument_errors(ctx):
    capi = _capi()
    out, n, b, e = C.c_void_p(), C.c_size_t(), C.c_uint64(), C.c_uint64()
    assert ctx.L.tg_group_by_key(ctx.h, None, 3, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert ctx.L.tg_group_by_key(ctx.h, None, 0, None, C.byref(n)) == TG_ERR_ARG
    assert ctx.L.tg_group_to_index(ctx.h, None, 0, 10, C.byref(out), C.byref(n), None, C.byref(e)) == TG_ERR_ARG
    arr = G.pairs([1, 2, 3], [4, 5, 6])
    d = ctx.to_device(arr)
    f8 = capi.DevFile(d, 6, 8, 0)                           # a device File of 8-byte items
    inp = capi.MergeInput(C.pointer(f8), None, 0)
    assert ctx.L.tg_group_by_key_file(ctx.h, C.byref(inp), C.byref(n)) == TG_ERR_ARG
    raw40 = np.zeros(40, np.uint8)                          # 40 bytes: not whole pairs
    ob, onb, _ = make_blocks(capi, raw40, 40)
    oin = capi.MergeInput(None, C.cast(ob, C.POINTER(capi.Block)), onb)
    assert ctx.L.tg_group_to_index_file(ctx.h, C.byref(oin), 10, C.byref(n), C.byref(b), C.byref(e)) == TG_ERR_ARG
    # GroupByKey's exchange (the key % p route) takes 2..16 workers
    for p in (0, 1, 17):
        assert _mod_exchange(ctx, d, 3, p) == TG_ERR_ARG, p
    ctx.free(d)
    check(ctx, arr)                                          # the ctx still works


def test_index_at_or_above_size_is_an_error(ctx):
    arr = G.pairs([0, 5, 9, 3], [1, 2, 3, 4])
    assert group_dev(ctx, arr, 9)[0] == TG_ERR_ARG
    assert group_dev(ctx, arr, 0)[0] == TG_ERR_ARG
    assert group_dev(ctx, arr, 10)[0] == 0
    assert group_dev(ctx, G.pairs([(1 << 64) - 1], [0]), (1 << 64) - 1)[0] == TG_ERR_ARG
    check(ctx, arr, 10)


def test_input_over_the_limit_is_too_large(ctx):
    out, n, b, e = C.c_void_p(), C.c_size_t(), C.c_uint64(), C.c_uint64()
    d = ctx.to_device(G.pairs([1], [1]))
    # 2^30 items are refused before anything is allocated or read (the buffer holds one)
    assert ctx.L.tg_group_by_key(ctx.h, d, 1 << 30, C.byref(out), C.byref(n)) == TG_ERR_TOO_LARGE
    assert ctx.L.tg_group_to_index(ctx.h, d, 1 << 30, 10, C.byref(out), C.byref(n), C.byref(b), C.byref(e)) == TG_ERR_TOO_LARGE
    # ... and by the exchange (a worker's shard of 2^30 items: its count step reads nothing)
    assert _mod_exchange(ctx, d, 1 << 30, 4) == TG_ERR_TOO_LARGE
    ctx.free(d)


# ---- full size ----------------------------------------------------------------------------------------------------------
class _Dev(object):
    """a zero-copy torch view of n x 2 int64 words at a device pointer"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n, 2), "typestr": "<i8", "data": (ptr, False), "version": 3}


@pytest.mark.parametrize("size", [None, (1 << 26) + 1])
def test_group_1e8(ctx, size):
    """1e8 pairs with keys uniform over 2^26 (1 + splitmix % 2^26) and value = global index: the multiset is unchanged, keys are
    non-decreasing and values increase wherever adjacent keys are equal (stability), checked on the device"""
    import torch
    n, u = 100_000_000, 1 << 26
    free, _ = torch.cuda.mem_get_info(0)
    if free < n * 16 * 4 + 2 * (1 << 30):
        pytest.skip("needs %.1f GB of device memory" % (n * 64 / GB + 2))
    t = torch.empty((n, 2), dtype=torch.int64, device="cuda:0")
    ctx.ck(ctx.L.tg_gen_reduce_uniform(ctx.h, t.data_ptr(), 0, n, 17, u, 1))
    ctx.sync()
    t[:, 1] = torch.arange(n, dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    before = ctx.checksum(t.data_ptr(), n, 16)
    out, m, b, e = C.c_void_p(), C.c_size_t(), C.c_uint64(), C.c_uint64()
    if size is None:
        ctx.ck(ctx.L.tg_group_by_key(ctx.h, t.data_ptr(), n, C.byref(out), C.byref(m)))
    else:
        ctx.ck(ctx.L.tg_group_to_index(ctx.h, t.data_ptr(), n, size, C.byref(out), C.byref(m), C.byref(b), C.byref(e)))
    assert m.value == n
    assert ctx.checksum(out.value, n, 16) == before
    ctx.sync()
    r = torch.as_tensor(_Dev(out.value, n), device="cuda:0")
    k, v = r[:, 0], r[:, 1]
    assert bool((k[1:] >= k[:-1]).all())
    eq = k[1:] == k[:-1]
    assert bool((v[1:][eq] > v[:-1][eq]).all())
    assert int(k[0]) >= 1 and int(k[-1]) <= u
    del r, k, v, eq, t
    torch.cuda.empty_cache()


# ---- several GPUs -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_group_on_n_gpus(world, exchange):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    env = dict(os.environ)
    if exchange == "nccl":
        env["TG_EXCHANGE"] = "nccl"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29881 + world), os.path.join(HERE, "multi_gpu_group_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert res.returncode == 0 and "MULTI_GPU_GROUP_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


# ---- inside a real Thrill job (the GpuGroupNode against the stock operators) -------------------------------------------
HOST_BIN = os.path.join(ROOT, "oracle", "_ref", "host", "gpu_group_test")
HOST_PASS = 8


def _host_run(workers, n):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([HOST_BIN, str(n)], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in res.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert len(lines) == HOST_PASS and all(l.startswith("PASS") for l in lines), lines


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_group_test not built (make -C tests/host -f gpu_group_test.mk)")
def test_group_inside_thrill_single_worker():
    _host_run(1, 9999)


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_group_test not built")
def test_group_inside_thrill_two_workers_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _host_run(2, 200000)
