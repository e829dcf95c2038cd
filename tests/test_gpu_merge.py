"""Merge (DIA::Merge / api::Merge) on one H100: tg_merge, tg_merge_file, tg_merge_select and the Python mirror against the
stable sort of the input-major concatenation (merge_ref.py); the multi-GPU worker and the in-Thrill host binary where the
machine has what they need.  pytest -m gpu."""
import ctypes as C
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest

import merge_ref as M
import sort_ref as R
from gpu_util import make_blocks
from sort_ref import BE, LE, Desc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4

U64 = Desc(8, 0, 8, LE)
PAIR = Desc(16, 0, 8, LE)                      # pair<uint64_t, 8-byte value> by .first
DESCS = [U64, Desc(8, 0, 8, LE, 1), Desc(8, 0, 5, LE), Desc(8, 3, 5, LE), Desc(8, 7, 1, LE), Desc(8, 0, 8, BE),
         PAIR, Desc(16, 8, 8, LE, 1), Desc(16, 0, 10, BE), Desc(16, 0, 16, BE), Desc(16, 3, 10, BE, 1), Desc(16, 4, 12, BE)]


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(0)
    yield c
    c.close()


def sorted_inputs(d, sizes, dist, seed):
    """one sorted (n, item_bytes) uint8 input per size; the bytes outside the key are random (they show the tie order)"""
    return [R.sort(R.make_items(d, n, dist, seed + 17 * j), d) for j, n in enumerate(sizes)]


def merge(ctx, d, inputs, desc=None):
    """tg_merge of host arrays on one worker: (status, result rows)"""
    k = len(inputs)
    ptrs = [ctx.to_device(R.rows(a, d.item_bytes)) for a in inputs]
    P = (C.c_void_p * k)(*ptrs)
    N = (C.c_size_t * k)(*[len(R.rows(a, d.item_bytes)) for a in inputs])
    out, n = C.c_void_p(), C.c_size_t()
    st = ctx.L.tg_merge(ctx.h, C.byref(desc or d.capi()), P, N, k, C.byref(out), C.byref(n))
    res = None
    if st == 0:
        res = ctx.download(out.value, n.value * d.item_bytes).reshape(-1, d.item_bytes) if n.value else \
            np.zeros((0, d.item_bytes), np.uint8)
    for p_ in ptrs:
        ctx.free(p_)
    return st, res


def check_merge(ctx, d, inputs):
    st, res = merge(ctx, d, inputs)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    assert np.array_equal(res, M.merged(inputs, 1, len(inputs), d))


# ---- tg_merge, one worker -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [2, 3, 4, 5, 16])
@pytest.mark.parametrize("d", DESCS, ids=lambda d: d.name)
def test_merge_descriptors(ctx, d, k):
    rng = np.random.RandomState(k * 31 + d.item_bytes + d.key_bytes)
    for dist in ("uniform", "few"):
        check_merge(ctx, d, sorted_inputs(d, rng.randint(0, 6000, size=k), dist, 5 + k))


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


@pytest.mark.parametrize("shape", ["two_balanced", "four_balanced", "two_imbalanced", "different_size"])
def test_merge_reference_shapes(ctx, shape):
    """the four cases of the reference's tests/api/merge_node_test.cpp"""
    n = 5000
    i = np.arange(n, dtype=np.uint64)
    if shape == "two_balanced":
        inputs, expected = [i * 2, i * 2 + 1], np.arange(2 * n)
    elif shape == "four_balanced":
        inputs, expected = [i * 4 + j for j in range(4)], np.arange(4 * n)
    elif shape == "two_imbalanced":
        inputs, expected = [i, i + 10000], np.concatenate([i, i + 10000])
    else:
        inputs, expected = [i, np.arange(2 * n, dtype=np.uint64) + 2500], np.sort(np.concatenate([i, np.arange(2 * n) + 2500]))
    st, res = merge(ctx, U64, inputs)
    assert st == 0 and np.array_equal(res.view(np.uint64).reshape(-1), _u64(expected))


def _pairs(keys, tag):
    """pair<u64, u64> rows: value = (input tag << 32) | position"""
    out = np.zeros(len(keys), dtype=[("k", "<u8"), ("v", "<u8")])
    out["k"] = keys
    out["v"] = (np.uint64(tag) << np.uint64(32)) | np.arange(len(keys), dtype=np.uint64)
    return R.rows(out, 16)


@pytest.mark.parametrize("k", [2, 3, 16])
def test_merge_special_shapes(ctx, k):
    # all keys equal: input-major, each input in position order
    check_merge(ctx, PAIR, [_pairs(np.full(300 + 7 * j, 42, np.uint64), j) for j in range(k)])
    # an empty input, and all inputs empty
    ins = [_pairs(np.sort(np.random.RandomState(j).randint(0, 100, size=0 if j == 1 else 500)).astype(np.uint64), j)
           for j in range(k)]
    check_merge(ctx, PAIR, ins)
    check_merge(ctx, PAIR, [_pairs(np.zeros(0, np.uint64), j) for j in range(k)])
    check_merge(ctx, U64, [np.zeros(0, np.uint64)] * k)
    # one item
    check_merge(ctx, U64, [_u64([5])] + [np.zeros(0, np.uint64)] * (k - 1))
    # lengths at the merge tile size +- 1 (4096 items of 8 bytes, 2048 of 16)
    rng = np.random.RandomState(k)
    for tile, d in ((4096, U64), (2048, PAIR)):
        for n in (tile - 1, tile, tile + 1, 2 * tile + 1):
            check_merge(ctx, d, sorted_inputs(d, [n + j % 2 for j in range(k)], "few", int(rng.randint(1000))))


def test_unsorted_inputs_give_a_permutation(ctx):
    """unsorted input: the result is unspecified, but every search stays in bounds and the items are all there"""
    rng = np.random.RandomState(9)
    for k in (2, 3, 5):
        for d in (U64, PAIR, Desc(16, 0, 16, BE)):
            ins = [R.make_items(d, int(rng.randint(0, 20000)), "uniform", 40 + j) for j in range(k)]
            st, res = merge(ctx, d, ins)
            assert st == 0
            cat = np.concatenate(ins)
            whole = Desc(d.item_bytes, 0, d.item_bytes, BE) if d.item_bytes <= 16 else d      # every byte a key byte
            assert np.array_equal(R.sort(res, whole), R.sort(cat, whole))


def test_argument_errors(ctx):
    capi = _capi()
    a = np.arange(10, dtype=np.uint64)
    assert merge(ctx, U64, [a])[0] == TG_ERR_ARG                              # k = 1
    assert merge(ctx, U64, [a] * 17)[0] == TG_ERR_ARG                         # k = 17
    rec = Desc(100, 0, 10, BE)
    assert merge(ctx, rec, [np.zeros((4, 100), np.uint8)] * 2)[0] == TG_ERR_ARG
    d = U64.capi()
    p = ctx.to_device(a)
    P = (C.c_void_p * 2)(p, p)
    N = (C.c_size_t * 2)(10, 10)
    out, n = C.c_void_p(), C.c_size_t()
    L = ctx.L
    assert L.tg_merge(ctx.h, C.byref(d), None, N, 2, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert L.tg_merge(ctx.h, C.byref(d), P, None, 2, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert L.tg_merge(ctx.h, C.byref(d), P, N, 2, None, C.byref(n)) == TG_ERR_ARG
    assert L.tg_merge(ctx.h, None, P, N, 2, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert L.tg_merge(ctx.h, C.byref(d), (C.c_void_p * 2)(p, None), N, 2, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert L.tg_merge_file(ctx.h, C.byref(d), None, 2, C.byref(n)) == TG_ERR_ARG
    wrong = capi.DevFile(p, 5, 16, 0)                                          # a 16-byte File for an 8-byte descriptor
    ins = (capi.MergeInput * 2)()
    ins[0].dev = C.pointer(wrong)
    ins[1].dev = C.pointer(wrong)
    assert L.tg_merge_file(ctx.h, C.byref(d), ins, 2, C.byref(n)) == TG_ERR_ARG
    bounds = np.zeros(64, np.uint64)
    assert L.tg_merge_select(ctx.h, C.byref(d), P, N, 1, 1, bounds.ctypes.data_as(C.POINTER(C.c_uint64))) == TG_ERR_ARG
    assert L.tg_merge_select(ctx.h, C.byref(d), P, N, 17, 2, bounds.ctypes.data_as(C.POINTER(C.c_uint64))) == TG_ERR_ARG
    ctx.free(p)


# ---- the selection for p simulated workers ----------------------------------------------------------------------------
def select(ctx, d, runs, p, k):
    ptrs = [ctx.to_device(R.rows(r, d.item_bytes)) for r in runs]
    P = (C.c_void_p * len(runs))(*ptrs)
    N = (C.c_size_t * len(runs))(*[len(R.rows(r, d.item_bytes)) for r in runs])
    out = np.zeros(p * k * (p + 1), np.uint64)
    st = ctx.L.tg_merge_select(ctx.h, C.byref(d.capi()), P, N, p, k, out.ctypes.data_as(C.POINTER(C.c_uint64)))
    for q in ptrs:
        ctx.free(q)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    return out


@pytest.mark.parametrize("p", [2, 3, 8, 16])
@pytest.mark.parametrize("d", [U64, Desc(8, 0, 8, LE, 1), Desc(8, 2, 3, LE), PAIR, Desc(16, 0, 16, BE), Desc(16, 3, 10, BE, 1)],
                         ids=lambda d: d.name)
def test_select_matches_restatement(ctx, d, p):
    rng = np.random.RandomState(p * 7 + d.key_bytes)
    for k in (2, 3, 4):
        for dist, shape in (("uniform", "random"), ("few", "random"), ("equal", "random"), ("few", "one"), ("uniform", "gaps")):
            inputs = sorted_inputs(d, rng.randint(0, 2500, size=k), dist, int(rng.randint(10000)))
            runs = M.make_runs(inputs, p, rng, shape)
            assert np.array_equal(select(ctx, d, runs, p, k), M.bounds(runs, p, k, d)), (k, dist, shape)
    # N < p
    runs = M.make_runs(sorted_inputs(d, [1, 0], "uniform", 3), p, rng)
    assert np.array_equal(select(ctx, d, runs, p, 2), M.bounds(runs, p, 2, d))


# ---- the drop-in entry point --------------------------------------------------------------------------------------------
def _transfer(ctx):
    h, d = C.c_uint64(), C.c_uint64()
    ctx.ck(ctx.L.tg_transfer_bytes(ctx.h, C.byref(h), C.byref(d)))
    return h.value, d.value


def _fetch(ctx, n, ib):
    capi = _capi()
    out = np.zeros((n, ib), np.uint8)
    ob, nob, _ = make_blocks(capi, out, 1 << 16)
    ctx.ck(ctx.L.tg_fetch_output(ctx.h, ob, nob))
    return out


def _dev_file(ctx, d, rows):
    """a device File holding `rows` (sorted): a stable tg_sort_file of sorted rows, detached"""
    capi = _capi()
    blocks, nb, _ = make_blocks(capi, rows, 1 << 16)
    n = C.c_size_t()
    ctx.ck(ctx.L.tg_sort_file(ctx.h, C.byref(d.capi()), blocks, nb, 1, C.byref(n)))
    f = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(f)))
    return f


def merge_file(ctx, d, specs):
    """specs: per input either ("host", rows) or ("dev", DevFile); returns the result size"""
    capi = _capi()
    ins = (capi.MergeInput * len(specs))()
    keep = []
    for j, (kind, x) in enumerate(specs):
        if kind == "dev":
            ins[j].dev = C.pointer(x)
        else:
            blocks, nb, raw = make_blocks(capi, x, 1 << 15)
            keep.append((blocks, raw))
            ins[j].blocks = C.cast(blocks, C.POINTER(capi.Block))
            ins[j].nblocks = nb
    n = C.c_size_t()
    ctx.ck(ctx.L.tg_merge_file(ctx.h, C.byref(d.capi()), ins, len(specs), C.byref(n)))
    return n.value


@pytest.mark.parametrize("d", [U64, PAIR, Desc(16, 0, 10, BE)], ids=lambda d: d.name)
def test_merge_file_host_device_and_mixed(ctx, d):
    capi = _capi()
    ins = sorted_inputs(d, [70000, 50001, 33333], "few", 77)
    expected = M.merged(ins, 1, 3, d)
    # host Files only, fetched
    n = merge_file(ctx, d, [("host", x) for x in ins])
    assert np.array_equal(_fetch(ctx, n, d.item_bytes), expected)
    # device Files only, and a mix; the handles stay intact and can be used again, their contents unchanged
    files = [_dev_file(ctx, d, x) for x in ins]
    sums = [ctx.checksum(f.dptr, f.items, f.item_bytes) for f in files]
    for specs in ([("dev", f) for f in files], [("dev", files[0]), ("host", ins[1]), ("dev", files[2])],
                  [("host", ins[0]), ("dev", files[1]), ("host", ins[2])]):
        n = merge_file(ctx, d, specs)
        assert np.array_equal(_fetch(ctx, n, d.item_bytes), expected)
    # the same device File as two inputs (Merge(a, a)), result detached as a device File
    n = merge_file(ctx, d, [("dev", files[0]), ("dev", files[0])])
    g = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(g)))
    assert g.items == n == 2 * len(ins[0])
    out = np.zeros((n, d.item_bytes), np.uint8)
    ob, nob, _ = make_blocks(capi, out, 1 << 20)
    ctx.ck(ctx.L.tg_dev_file_fetch(ctx.h, C.byref(g), ob, nob))
    assert np.array_equal(out, M.merged([ins[0], ins[0]], 1, 2, d))
    for f, s in zip(files, sums):
        assert f.dptr and ctx.checksum(f.dptr, f.items, f.item_bytes) == s
        ctx.ck(ctx.L.tg_dev_file_free(ctx.h, C.byref(f)))
    ctx.ck(ctx.L.tg_dev_file_free(ctx.h, C.byref(g)))


def test_sort_then_merge_moves_nothing_over_pcie(ctx):
    capi = _capi()
    rng = np.random.RandomState(4)
    a = rng.randint(0, 1 << 40, size=400000).astype(np.uint64)
    b = rng.randint(0, 1 << 40, size=300001).astype(np.uint64)
    fa, fb = _dev_file(ctx, U64, a), _dev_file(ctx, U64, b)        # tg_sort_file + detach: sorted device Files
    h0, d0 = _transfer(ctx)
    n = merge_file(ctx, U64, [("dev", fa), ("dev", fb)])
    g = capi.DevFile()
    ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(g)))
    assert _transfer(ctx) == (h0, d0)                                 # nothing crossed PCIe between the operators
    assert n == g.items == len(a) + len(b)
    assert ctx.is_sorted(U64.capi(), g.dptr, g.items)
    out = np.zeros(n, np.uint64)
    ob, nob, _ = make_blocks(capi, out, 1 << 20)
    ctx.ck(ctx.L.tg_dev_file_fetch(ctx.h, C.byref(g), ob, nob))
    assert np.array_equal(out, np.sort(np.concatenate([a, b])))
    for f in (fa, fb, g):
        ctx.ck(ctx.L.tg_dev_file_free(ctx.h, C.byref(f)))


# ---- the Python mirror ------------------------------------------------------------------------------------------------
def test_python_merge():
    from thrill_b200 import api, capi
    ctx = api.Context(rank=0, nranks=1, device=0, rng_seed=1)
    try:
        rng = np.random.RandomState(2)
        a = api.DIA(ctx, np.sort(rng.randint(0, 1000, size=30000).astype(np.uint64)))
        b = api.DIA(ctx, np.sort(rng.randint(0, 1000, size=20000).astype(np.uint64)))
        c = api.DIA(ctx, np.sort(rng.randint(0, 1000, size=100).astype(np.uint64)))
        assert np.array_equal(a.Merge(b).items, np.sort(np.concatenate([a.items, b.items])))
        assert np.array_equal(api.Merge(api.Less, a, b, c).items, np.sort(np.concatenate([a.items, b.items, c.items])))
        g1, g2 = api.DIA(ctx, a.items[::-1].copy()), api.DIA(ctx, b.items[::-1].copy())
        assert np.array_equal(g1.Merge(g2, api.Greater).items, np.sort(np.concatenate([a.items, b.items]))[::-1])
        kv1 = np.zeros(5000, dtype=api.KV); kv1["key"] = np.sort(rng.randint(0, 50, size=5000)); kv1["val"] = np.arange(5000)
        kv2 = np.zeros(4000, dtype=api.KV); kv2["key"] = np.sort(rng.randint(0, 50, size=4000)); kv2["val"] = 10000 + np.arange(4000)
        m = api.DIA(ctx, kv1).Merge(api.DIA(ctx, kv2)).items
        cat = np.concatenate([kv1, kv2])
        assert np.array_equal(m, cat[np.argsort(cat["key"], kind="stable")])
        # rejections
        with pytest.raises(capi.ThrillGpuError):
            a.Merge(b, object())
        with pytest.raises(capi.ThrillGpuError):
            a.Merge(api.DIA(ctx, kv1))
        with pytest.raises(capi.ThrillGpuError):
            api.Merge(None, a)
        recs = api.DIA(ctx, np.zeros((10, 100), np.uint8))
        with pytest.raises(capi.ThrillGpuError):
            recs.Merge(recs)
    finally:
        ctx.close()


# ---- several GPUs -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_merge_on_n_gpus(world, exchange):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29660 + world + (20 if exchange == "nccl" else 0)),
           os.path.join(HERE, "multi_gpu_merge_worker.py")]
    env = dict(os.environ)
    if exchange == "nccl":
        env["TG_EXCHANGE"] = "nccl"
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    assert res.returncode == 0 and "MULTI_GPU_MERGE_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-5000:]


HOST_BIN = os.path.join(ROOT, "oracle", "_ref", "host", "gpu_merge_test")
HOST_PASS = 8


def _host_run(workers, n):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([HOST_BIN, str(n)], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in res.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert len(lines) == HOST_PASS and all(l.startswith("PASS") for l in lines), lines


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_merge_test not built (make -C tests/host -f gpu_merge_test.mk)")
def test_merge_inside_thrill_single_worker():
    _host_run(1, 1000000)


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_merge_test not built")
def test_merge_inside_thrill_two_workers_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _host_run(2, 1500000)


# ---- the top of the size range (-m "gpu and not large" leaves these out) ------------------------------------------------
# `large` is registered nowhere else; its unknown-marker warning is silenced where the mark is made (as in test_gpu_large.py)
with warnings.catch_warnings():
    warnings.simplefilter("ignore", pytest.PytestUnknownMarkWarning)
    large = pytest.mark.large

GB = 1 << 30


def _need(nbytes, what):
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < nbytes + 2 * GB:
        pytest.skip("%s needs %.1f GB of device memory (+2 GB), %.1f GB are free" % (what, nbytes / GB, free / GB))


def _upload_chunks(ctx, dptr, n, gen, item_bytes, chunk=1 << 25):
    for i0 in range(0, n, chunk):
        x = np.ascontiguousarray(gen(i0, min(n, i0 + chunk)))
        ctx.ck(ctx.L.tg_upload(ctx.h, dptr + i0 * item_bytes, x.ctypes.data, x.nbytes))
        ctx.sync()


def _combine(sums):
    s, x = 0, 0
    for a, b in sums:
        s, x = (s + a) % (1 << 64), x ^ b
    return s, x


@large
class TestLarge(object):
    def test_u64_two_inputs_at_the_item_limit(self, ctx):
        """input j item i = 2 i + j, N = 2^30 - 1: the result is 0..N-1"""
        n = (1 << 30) - 1
        _need(3 * n * 8, "merge of 2^30 - 1 u64")
        sizes = [(n + 1) // 2, n // 2]
        ptrs = [ctx.alloc(s * 8) for s in sizes]
        for j, (p_, s) in enumerate(zip(ptrs, sizes)):
            _upload_chunks(ctx, p_, s, lambda a, b, j=j: np.arange(a, b, dtype=np.uint64) * np.uint64(2) + np.uint64(j), 8)
        before = _combine([ctx.checksum(p_, s, 8) for p_, s in zip(ptrs, sizes)])
        out, cnt = C.c_void_p(), C.c_size_t()
        ctx.ck(ctx.L.tg_merge(ctx.h, C.byref(U64.capi()), (C.c_void_p * 2)(*ptrs), (C.c_size_t * 2)(*sizes), 2,
                              C.byref(out), C.byref(cnt)))
        assert cnt.value == n
        assert ctx.is_sorted(U64.capi(), out.value, n)
        assert ctx.checksum(out.value, n, 8) == before
        for i in (0, 1, 4095, 4096, n // 2, n - 2, n - 1):
            assert int(ctx.download(out.value + 8 * i, 8, np.uint64)[0]) == i
        for p_ in ptrs:
            ctx.free(p_)

    def test_pairs_with_duplicate_keys_keep_input_and_position_order(self, ctx):
        """2 x 2^27 pairs, key = i // 3 in input 0 and i // 5 in input 1, value = (input << 40) | i: every run of equal keys
        must list input 0's items before input 1's, each in position order"""
        n = 1 << 27
        _need(6 * n * 16, "merge of 2^28 pairs")
        div = [3, 5]

        def gen(j):
            def g(a, b):
                i = np.arange(a, b, dtype=np.uint64)
                out = np.empty((b - a, 2), np.uint64)
                out[:, 0] = i // np.uint64(div[j])
                out[:, 1] = (np.uint64(j) << np.uint64(40)) | i
                return out
            return g
        ptrs = [ctx.alloc(n * 16) for _ in range(2)]
        for j in range(2):
            _upload_chunks(ctx, ptrs[j], n, gen(j), 16)
        before = _combine([ctx.checksum(p_, n, 16) for p_ in ptrs])
        out, cnt = C.c_void_p(), C.c_size_t()
        ctx.ck(ctx.L.tg_merge(ctx.h, C.byref(PAIR.capi()), (C.c_void_p * 2)(*ptrs), (C.c_size_t * 2)(n, n), 2,
                              C.byref(out), C.byref(cnt)))
        assert cnt.value == 2 * n and ctx.checksum(out.value, 2 * n, 16) == before
        # (key, value) strictly increasing over the whole result, in streamed chunks: with the multiset preserved this is
        # exactly the expected sequence
        prev = None
        chunk = 1 << 24
        for i0 in range(0, 2 * n, chunk):
            m = min(chunk, 2 * n - i0)
            x = ctx.download(out.value + 16 * i0, 16 * m, np.uint64).reshape(m, 2)
            if prev is not None:
                x = np.concatenate([prev, x])
            k_, v_ = x[:, 0], x[:, 1]
            ok = (k_[1:] > k_[:-1]) | ((k_[1:] == k_[:-1]) & (v_[1:] > v_[:-1]))
            assert ok.all(), i0
            prev = x[-1:]
        for p_ in ptrs:
            ctx.free(p_)

    def test_too_large_is_rejected(self, ctx):
        half = 1 << 29
        _need(2 * half * 8, "2 x 2^29 u64 buffers")
        ptrs = [ctx.alloc(half * 8) for _ in range(2)]
        out, cnt = C.c_void_p(), C.c_size_t()
        st = ctx.L.tg_merge(ctx.h, C.byref(U64.capi()), (C.c_void_p * 2)(*ptrs), (C.c_size_t * 2)(half, half), 2,
                            C.byref(out), C.byref(cnt))
        assert st == TG_ERR_TOO_LARGE
        for p_ in ptrs:
            ctx.free(p_)
