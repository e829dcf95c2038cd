"""InnerJoin (api::InnerJoin) on one H100: tg_inner_join, tg_inner_join_file and the Python mirror against the numpy
restatement in join_ref.py (exact, including the order); device Files, the GPU chain without PCIe traffic, the argument
errors and the size limit, large cases, and the multi-GPU worker where the machine has several GPUs.  pytest -m gpu."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import join_ref as J
from gpu_util import make_blocks

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4
FNS = [J.KEY_VALUES, J.VALUES]
GB = float(1 << 30)


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(0)
    yield c
    c.close()


def join_dev(ctx, left, right, fn, item_bytes=16):
    """tg_inner_join of two host KV arrays on one worker: (status, result)"""
    capi = _capi()
    dl, dr = ctx.to_device(left), ctx.to_device(right)
    out, n = C.c_void_p(), C.c_size_t()
    desc = capi.JoinDesc(item_bytes, fn)
    st = ctx.L.tg_inner_join(ctx.h, C.byref(desc), dl, len(left), dr, len(right), C.byref(out), C.byref(n))
    res = None
    if st == 0:
        dt = J.out_dtype(fn)
        res = ctx.download(out.value, n.value * dt.itemsize).view(dt) if n.value else np.zeros(0, dt)
    ctx.free(dl)
    ctx.free(dr)
    return st, res


def check(ctx, left, right, fn):
    st, res = join_dev(ctx, left, right, fn)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    ref = J.join_local(left, right, fn)
    assert len(res) == len(ref)
    assert np.array_equal(res.view(np.uint64), ref.view(np.uint64))


def pairs(keys, vals=None):
    out = np.empty(len(keys), J.KV)
    out["key"] = np.asarray(keys, np.uint64)
    out["val"] = np.arange(len(keys), dtype=np.uint64) * np.uint64(7) + np.uint64(3) if vals is None else vals
    return out


# ---- exact results, one worker ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("nl,nr,universe", [(1, 1, 1), (5, 7, 3), (1000, 1000, 500), (6000, 3000, 2000),
                                             (20000, 50000, 1 << 40), (40000, 40000, 40000), (3000, 100000, 64)])
def test_join_random(ctx, fn, nl, nr, universe):
    check(ctx, J.make_side(nl, universe, nl + 1), J.make_side(nr, universe, nr + 2), fn)


@pytest.mark.parametrize("fn", FNS)
def test_join_reference_shapes(ctx, fn):
    # tests/api/join_test.cpp: identity keys, every item on one key, and 100 x 333 on small keys
    n = 9999
    check(ctx, pairs(np.arange(n)), pairs(np.arange(n)), fn)
    check(ctx, pairs(np.full(333, 1)), pairs(np.full(333, 1)), fn)
    check(ctx, pairs(np.arange(100) % 10), pairs(np.arange(333) % 7), fn)


@pytest.mark.parametrize("fn", FNS)
def test_join_edge_cases(ctx, fn):
    empty = np.zeros(0, J.KV)
    for l, r in [(empty, empty), (pairs([1, 2, 3]), empty), (empty, pairs([1, 2]))]:
        st, res = join_dev(ctx, l, r, fn)
        assert st == 0 and len(res) == 0
    # no matches
    st, res = join_dev(ctx, pairs(np.arange(0, 20000, 2)), pairs(np.arange(1, 20000, 2)), fn)
    assert st == 0 and len(res) == 0
    # key 0 is an ordinary key, as is the largest key
    check(ctx, pairs([0, 0, 5, (1 << 64) - 1]), pairs([0, 7, 0, (1 << 64) - 1, 0]), fn)
    check(ctx, pairs(np.zeros(3000)), pairs(np.zeros(500)), fn)
    # every item on one key
    check(ctx, pairs(np.full(2500, 42)), pairs(np.full(1700, 42)), fn)


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("n", [1023, 1024, 1025, 2047, 2048, 2049, 4095, 4097])
def test_join_tile_edges(ctx, fn, n):
    # the count kernel's tiles hold 2048 merged (left, right) items, the emit kernel's 1024 (left items, outputs); runs of
    # equal keys straddle both
    rng = np.random.RandomState(n)
    check(ctx, pairs(np.sort(rng.randint(0, n // 3 + 1, n))), pairs(rng.randint(0, n // 3 + 1, n // 2 + 1)), fn)
    check(ctx, pairs(np.arange(n) // 700), pairs(np.arange(n) // 300), fn)
    check(ctx, pairs(np.full(n, 9)), pairs(np.full(3, 9)), fn)
    check(ctx, pairs(np.full(3, 9)), pairs(np.full(n, 9)), fn)
    check(ctx, pairs(np.arange(n)), pairs(np.arange(n) // 2), fn)


def test_join_values_are_bit_copies(ctx):
    # V2 holding doubles: NaN payloads, -0.0 and infinities come through as bits
    vals = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 1.5, -2.25], np.float64).view(np.uint64).copy()
    vals[0] |= np.uint64(0x1234)
    right = pairs(np.arange(7) % 3, vals)
    left = pairs(np.arange(5) % 3)
    for fn in FNS:
        check(ctx, left, right, fn)


# ---- the _file form, device Files, the Python mirror -----------------------------------------------------------------
def _dev_file(ctx, arr):
    capi = _capi()
    d = ctx.to_device(arr)
    return capi.DevFile(d, len(arr), 16, 0), d


def _host_input(arr, block_bytes):
    capi = _capi()
    blocks, nb, raw = make_blocks(capi, arr, block_bytes)
    return capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb), (blocks, raw)


@pytest.mark.parametrize("fn", FNS)
def test_join_file_host_device_and_mixed(ctx, fn):
    capi = _capi()
    left, right = J.make_side(30000, 5000, 11), J.make_side(20000, 5000, 12)
    ref = J.join_local(left, right, fn)
    dt = J.out_dtype(fn)
    for mode in ("host", "device", "left_device", "right_device"):
        keep = []
        sides = []
        devs = []
        for j, arr in enumerate((left, right)):
            if mode == "device" or (mode == "left_device" and j == 0) or (mode == "right_device" and j == 1):
                f, d = _dev_file(ctx, arr)
                devs.append((f, d, arr))
                sides.append(capi.MergeInput(C.pointer(f), None, 0))
                keep.append(f)
            else:
                inp, k = _host_input(arr, 1000 + 37 * j)      # Blocks that cut items
                sides.append(inp)
                keep.append(k)
        h2d0, d2h0 = C.c_uint64(), C.c_uint64()
        ctx.L.tg_transfer_bytes(ctx.h, C.byref(h2d0), C.byref(d2h0))
        n = C.c_size_t()
        ctx.ck(ctx.L.tg_inner_join_file(ctx.h, C.byref(capi.JoinDesc(16, fn)), C.byref(sides[0]), C.byref(sides[1]), C.byref(n)))
        h2d1, d2h1 = C.c_uint64(), C.c_uint64()
        ctx.L.tg_transfer_bytes(ctx.h, C.byref(h2d1), C.byref(d2h1))
        assert d2h1.value == d2h0.value            # no device File goes to the host
        if mode == "device":
            assert h2d1.value == h2d0.value
        out = np.empty(n.value * dt.itemsize, np.uint8)
        blocks, nb, _ = make_blocks(capi, out, 1 << 16)
        ctx.ck(ctx.L.tg_fetch_output(ctx.h, blocks, nb))
        assert np.array_equal(out.view(dt).view(np.uint64), ref.view(np.uint64)), mode
        for f, d, arr in devs:                     # device Files are left intact
            assert np.array_equal(ctx.download(d, len(arr) * 16).view(J.KV), arr)
            ctx.free(d)


def test_self_join_on_one_device_file(ctx):
    capi = _capi()
    a = J.make_side(5000, 800, 5)
    f, d = _dev_file(ctx, a)
    inp = capi.MergeInput(C.pointer(f), None, 0)
    n = C.c_size_t()
    ctx.ck(ctx.L.tg_inner_join_file(ctx.h, C.byref(capi.JoinDesc(16, J.KEY_VALUES)), C.byref(inp), C.byref(inp), C.byref(n)))
    out = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(out)))
    assert out.item_bytes == 24 and out.items == n.value
    res = ctx.download(out.dptr, n.value * 24).view(J.KEY_V1_V2)
    assert np.array_equal(res.view(np.uint64), J.join_local(a, a, J.KEY_VALUES).view(np.uint64))
    assert np.array_equal(ctx.download(d, len(a) * 16).view(J.KV), a)
    ctx.L.tg_dev_file_free(ctx.h, C.byref(out))
    ctx.free(d)


def test_reduce_join_reduce_chain_moves_nothing_over_pcie(ctx):
    """ReducePair -> InnerJoin(JoinValues) -> ReducePair, each result handed on as a device File"""
    capi = _capi()
    a, b = J.make_side(40000, 3000, 21), J.make_side(30000, 3000, 22)
    a["val"] = np.arange(len(a), dtype=np.uint64) % np.uint64(1000)
    b["val"] = np.arange(len(b), dtype=np.uint64) % np.uint64(977)
    files = []
    for arr in (a, b):
        blocks, nb, _ = make_blocks(capi, arr, 1 << 20)
        n = C.c_size_t()
        ctx.ck(ctx.L.tg_reduce_file(ctx.h, C.byref(capi.KVDesc(16, capi.OP_SUM_U64)), blocks, nb, C.byref(n)))
        f = capi.DevFile()
        ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(f)))
        files.append(f)
    h2d0, d2h0 = C.c_uint64(), C.c_uint64()
    ctx.L.tg_transfer_bytes(ctx.h, C.byref(h2d0), C.byref(d2h0))
    sides = [capi.MergeInput(C.pointer(f), None, 0) for f in files]
    n = C.c_size_t()
    ctx.ck(ctx.L.tg_inner_join_file(ctx.h, C.byref(capi.JoinDesc(16, J.VALUES)), C.byref(sides[0]), C.byref(sides[1]), C.byref(n)))
    j = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(j)))
    assert j.item_bytes == 16
    n2 = C.c_size_t()
    ctx.ck(ctx.L.tg_reduce_dev(ctx.h, C.byref(capi.KVDesc(16, capi.OP_SUM_U64)), C.byref(j), C.byref(n2)))
    h2d1, d2h1 = C.c_uint64(), C.c_uint64()
    ctx.L.tg_transfer_bytes(ctx.h, C.byref(h2d1), C.byref(d2h1))
    assert (h2d1.value, d2h1.value) == (h2d0.value, d2h0.value)
    out = np.empty(n2.value * 16, np.uint8)
    blocks, nb, _ = make_blocks(capi, out, 1 << 20)
    ctx.ck(ctx.L.tg_fetch_output(ctx.h, blocks, nb))
    res = np.sort(out.view(J.KV), order="key")
    # the model: both reductions, the join on the sums, the sum of v2 per v1
    def reduce(x):
        k, inv = np.unique(x["key"], return_inverse=True)
        s = np.zeros(len(k), np.uint64)
        np.add.at(s, inv, x["val"])
        return pairs(k, s)
    ra, rb = reduce(a), reduce(b)
    jv = J.join_local(ra, rb, J.VALUES)
    ref = reduce(pairs(jv["v1"], jv["v2"]))
    assert np.array_equal(res.view(np.uint64), ref.view(np.uint64))
    for f in files + [j]:
        ctx.L.tg_dev_file_free(ctx.h, C.byref(f))


def test_python_inner_join():
    from thrill_b200 import api, capi
    c = api.Context(rank=0, nranks=1, device=0, rng_seed=3)
    try:
        left, right = J.make_side(7000, 900, 31), J.make_side(9000, 900, 32)
        for fn, jf in ((J.KEY_VALUES, api.JoinKeyValues), (J.VALUES, api.JoinValues)):
            out = api.InnerJoin(api.DIA(c, left.view(api.KV)), api.DIA(c, right.view(api.KV)), api.KeyIsFirst, api.KeyIsFirst, jf)
            assert out.items.dtype == (api.KEY_V1_V2 if fn == J.KEY_VALUES else api.V1_V2)
            assert np.array_equal(out.items.view(np.uint64), J.join_local(left, right, fn).view(np.uint64))
        a, b = api.DIA(c, left.view(api.KV)), api.DIA(c, right.view(api.KV))
        with pytest.raises(capi.ThrillGpuError):
            api.InnerJoin(a, b, api.KeyIsFirst, api.KeyIsFirst, api.PlusDouble)
        with pytest.raises(capi.ThrillGpuError):
            api.InnerJoin(a, b, api.Less, api.KeyIsFirst, api.JoinValues)
        with pytest.raises(capi.ThrillGpuError):
            api.InnerJoin(api.DIA(c, np.arange(10, dtype=np.uint64)), b, api.KeyIsFirst, api.KeyIsFirst, api.JoinValues)
    finally:
        c.close()


# ---- errors and the size limit -----------------------------------------------------------------------------------------
def test_argument_errors(ctx):
    capi = _capi()
    a = pairs([1, 2, 3])
    assert join_dev(ctx, a, a, J.VALUES, item_bytes=8)[0] == TG_ERR_ARG
    assert join_dev(ctx, a, a, J.VALUES, item_bytes=24)[0] == TG_ERR_ARG
    assert join_dev(ctx, a, a, 2)[0] == TG_ERR_ARG
    out, n = C.c_void_p(), C.c_size_t()
    assert ctx.L.tg_inner_join(ctx.h, C.byref(capi.JoinDesc(16, 0)), None, 3, None, 0, C.byref(out), C.byref(n)) == TG_ERR_ARG
    d = ctx.to_device(a)
    f8 = capi.DevFile(d, 6, 8, 0)                          # a device File of 8-byte items
    inp = capi.MergeInput(C.pointer(f8), None, 0)
    assert ctx.L.tg_inner_join_file(ctx.h, C.byref(capi.JoinDesc(16, 0)), C.byref(inp), C.byref(inp), C.byref(n)) == TG_ERR_ARG
    odd, keep = _host_input(np.zeros(40, np.uint8), 40)     # 40 bytes: not whole pairs
    assert ctx.L.tg_inner_join_file(ctx.h, C.byref(capi.JoinDesc(16, 0)), C.byref(odd), C.byref(odd), C.byref(n)) == TG_ERR_ARG
    ctx.free(d)
    check(ctx, a, a, J.KEY_VALUES)                          # the ctx still works


def test_output_over_the_limit_is_too_large(ctx):
    # 40 000 x 30 000 items on one key: 1.2e9 outputs > 2^30 - 1, a documented limit
    left, right = pairs(np.full(40000, 5)), pairs(np.full(30000, 5))
    assert J.output_counts(left, right) > J.LIMIT
    st, _ = join_dev(ctx, left, right, J.VALUES)
    assert st == TG_ERR_TOO_LARGE
    check(ctx, left[:300], right[:200], J.VALUES)


# ---- large cases ---------------------------------------------------------------------------------------------------------
def _need(nbytes, what):
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < nbytes + 2 * (1 << 30):
        pytest.skip("%s needs %.1f GB of device memory (+2 GB), %.1f GB are free" % (what, nbytes / GB, free / GB))


def test_foreign_key_join_1e8(ctx):
    """1e8 left pairs with keys uniform over 2^26 against the 2^26 distinct right keys: 1e8 outputs, by checksum"""
    n, u = 100_000_000, 1 << 26
    _need(n * 16 * 12, "the foreign-key join")
    rng = np.random.default_rng(7)
    left = np.empty(n, J.KV)
    left["key"] = rng.integers(0, u, n, dtype=np.uint64)
    left["val"] = np.arange(n, dtype=np.uint64)
    right = np.empty(u, J.KV)
    right["key"] = rng.permutation(u).astype(np.uint64)
    right["val"] = rng.integers(0, 1 << 63, u, dtype=np.uint64)
    capi = _capi()
    dl, dr = ctx.to_device(left), ctx.to_device(right)
    out, m = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_inner_join(ctx.h, C.byref(capi.JoinDesc(16, J.KEY_VALUES)), dl, n, dr, u, C.byref(out), C.byref(m)))
    assert m.value == n
    got = ctx.checksum(out.value, m.value, 24)
    # the model: every left item matches the one right item with its key; right is a permutation, so its index is known
    inv = np.empty(u, np.int64)
    inv[right["key"].astype(np.int64)] = np.arange(u)
    order = np.argsort(left["key"], kind="stable")
    ref = np.empty(n, J.KEY_V1_V2)
    ref["key"] = left["key"][order]
    ref["v1"] = left["val"][order]
    ref["v2"] = right["val"][inv[ref["key"].astype(np.int64)]]
    del order
    # exact order: a sample of positions, then the multiset by checksum
    pos = np.unique(np.concatenate([np.arange(1000), np.arange(n - 1000, n), rng.integers(0, n, 2000)]))
    for p_ in pos[::97]:
        row = ctx.download(out.value + int(p_) * 24, 24).view(J.KEY_V1_V2)
        assert row.view(np.uint64).tolist() == ref[p_:p_ + 1].view(np.uint64).tolist()
    dref = ctx.to_device(ref)
    assert ctx.checksum(dref, n, 24) == got
    for d in (dl, dr, dref):
        ctx.free(d)


def test_hot_key_near_the_output_limit(ctx):
    """32 768 x 32 767 items on one key: 1 073 709 056 outputs (2^30 - 32 768), by count, checksum of slices and positions"""
    nl, nr = 32768, 32767
    m_ref = nl * nr
    _need(m_ref * 16 + (1 << 30), "the hot-key join")
    capi = _capi()
    left, right = pairs(np.full(nl, 77)), pairs(np.full(nr, 77))
    left["val"] = np.arange(nl, dtype=np.uint64)
    right["val"] = np.arange(nr, dtype=np.uint64) << np.uint64(32)
    dl, dr = ctx.to_device(left), ctx.to_device(right)
    out, m = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_inner_join(ctx.h, C.byref(capi.JoinDesc(16, J.VALUES)), dl, nl, dr, nr, C.byref(out), C.byref(m)))
    assert m.value == m_ref
    # output j = (j // nr, (j % nr) << 32)
    rng = np.random.default_rng(1)
    starts = np.concatenate([[0, m_ref - 4096, nr - 100, 1024 * 1000 - 7], rng.integers(0, m_ref - 4096, 40)])
    for s in starts:
        s = int(s)
        got = ctx.download(out.value + s * 16, 4096 * 16).view(np.uint64).reshape(-1, 2)
        j = np.arange(s, s + 4096, dtype=np.uint64)
        assert np.array_equal(got[:, 0], j // np.uint64(nr))
        assert np.array_equal(got[:, 1], (j % np.uint64(nr)) << np.uint64(32))
    # whole slices by checksum: the nr outputs of sampled left items against the model's rows built on the host
    ref = np.empty((nr, 2), np.uint64)
    ref[:, 1] = right["val"]
    dref = ctx.alloc(nr * 16)
    for i in _sample_left(nl):
        ref[:, 0] = i
        ctx.upload(dref, ref)
        assert ctx.checksum(out.value + int(i) * nr * 16, nr, 16) == ctx.checksum(dref, nr, 16)
    for d in (dl, dr, dref):
        ctx.free(d)


def _sample_left(nl):
    return sorted(set([0, 1, nl // 2, nl - 2, nl - 1] + [int(x) for x in np.random.default_rng(3).integers(0, nl, 20)]))


def test_input_over_the_limit_is_too_large(ctx):
    capi = _capi()
    out, n = C.c_void_p(), C.c_size_t()
    d = ctx.to_device(pairs([1]))
    st = ctx.L.tg_inner_join(ctx.h, C.byref(capi.JoinDesc(16, 0)), d, 1 << 30, d, 1, C.byref(out), C.byref(n))
    assert st == TG_ERR_TOO_LARGE
    ctx.free(d)


# ---- several GPUs -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_join_on_n_gpus(world, exchange):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    env = dict(os.environ)
    if exchange == "nccl":
        env["TG_EXCHANGE"] = "nccl"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29861 + world), os.path.join(HERE, "multi_gpu_join_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert res.returncode == 0 and "MULTI_GPU_JOIN_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


# ---- inside a real Thrill job (the GpuJoinNode against the stock api::InnerJoin) ---------------------------------------
HOST_BIN = os.path.join(ROOT, "oracle", "_ref", "host", "gpu_join_test")
HOST_PASS = 7


def _host_run(workers, n):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([HOST_BIN, str(n)], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in res.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert len(lines) == HOST_PASS and all(l.startswith("PASS") for l in lines), lines


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_join_test not built (make -C tests/host -f gpu_join_test.mk)")
def test_join_inside_thrill_single_worker():
    _host_run(1, 9999)


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_join_test not built")
def test_join_inside_thrill_two_workers_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _host_run(2, 200000)
