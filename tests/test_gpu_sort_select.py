"""The multi-worker Sort's device classification on one H100, bit-exact against sample_sort_ref: tg_sort_select runs the
operator's sampling, splitter selection, top-byte lookup table, SplitterDigit pass (with the global index base the selection
writes on the device) and the merge pipeline's boundaries for p simulated workers.  (ReduceToIndex's range route and the
exchange's stores are tested through tg_exchange_select in test_gpu_exchange.py.)  pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import sample_sort_ref as S
import sort_ref as R
from sort_ref import BE, LE, Desc

pytestmark = pytest.mark.gpu
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4

U64 = Desc(8, 0, 8, LE)
KV = Desc(16, 0, 8, LE)
SHAPE_DESCS = [U64, KV, Desc(16, 0, 16, BE), Desc(8, 0, 8, LE, 1)]       # records classify as Desc(16, 0, k, BE) tuples
TILE = {8: 16384, 16: 8192}                                              # items per tile of the partition pass


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(0)
    yield c
    c.close()


def _u64p(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint64))


def sort_select(ctx, d, shards, p, seed, desc=None):
    """tg_sort_select on host shards: (status, splitters, counts (p, p), grouped shards, merge bounds (p, p - 1))"""
    ib = d.item_bytes
    rows = [R.rows(s, ib) for s in shards]
    din = [ctx.to_device(r) if len(r) else None for r in rows]
    dout = [ctx.alloc(max(len(r) * ib, 16)) for r in rows]
    spl = np.zeros((p - 1, ib + 8), np.uint8)
    counts = np.zeros(p * p, np.uint64)
    bounds = np.zeros(p * (p - 1), np.uint64)
    st = ctx.L.tg_sort_select(ctx.h, C.byref(desc or d.capi()), (C.c_void_p * p)(*din), (C.c_size_t * p)(*[len(r) for r in rows]),
                              p, seed, spl.ctypes.data, (C.c_void_p * p)(*dout), _u64p(counts), _u64p(bounds))
    grouped = [ctx.download(o, len(r) * ib).reshape(-1, ib) if st == 0 and len(r) else np.zeros((0, ib), np.uint8)
               for o, r in zip(dout, rows)]
    for q in din + dout:
        if q:
            ctx.free(q)
    return st, spl, counts.reshape(p, p), grouped, bounds.reshape(p, p - 1)


def check(ctx, d, shards, p, seed):
    st, spl, counts, grouped, bounds = sort_select(ctx, d, shards, p, seed)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    w_spl, w_counts, w_grouped, w_bounds = S.select(shards, d, p, seed)
    assert np.array_equal(spl, w_spl), "splitters"
    assert np.array_equal(counts, w_counts), "counts"
    for w in range(p):
        assert np.array_equal(grouped[w], w_grouped[w]), "grouped shard %d" % w
    assert np.array_equal(bounds, w_bounds), "merge bounds"
    return w_spl


def ties_split(shards, d, spl):
    """whether items equal to some splitter's key land on both sides of it"""
    pre = S.prefix_of(shards, d)
    shi, slo, _ = S.unpack_splitters(spl, d)
    seen = {}
    for w, sh in enumerate(shards):
        hi, lo = S.canon(sh, d)
        b = S.classify(sh, d, pre[w] + np.arange(len(sh)), spl)
        for j in range(len(shi)):
            m = (hi == shi[j]) & (lo == slo[j])
            seen.setdefault(j, set()).update(set(b[m].tolist()) & {j, j + 1})
    return any(len(v) == 2 for v in seen.values())


# ---- descriptor matrix ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [3, 16])
@pytest.mark.parametrize("d", R.ITEM8 + R.ITEM16, ids=lambda d: d.name)
def test_descriptor_matrix(ctx, d, p):
    rng = np.random.RandomState(d.item_bytes * 31 + d.key_offset * 7 + d.key_bytes + 3 * p + 50 * d.descending)
    for dist in S.DISTS:
        shards = [S.make_items(d, int(n), dist, int(rng.randint(1 << 30))) for n in rng.randint(45000, 55000, size=p)]
        spl = check(ctx, d, shards, p, int(rng.randint(1 << 40)))
        if dist in ("few", "equal"):
            assert ties_split(shards, d, spl), dist


# ---- worker counts and shard shapes ---------------------------------------------------------------------------------------
def _shapes(d, p, sm_count):
    t = TILE[d.item_bytes]
    big = (2 * sm_count + 37) * t + 123               # more tiles than 2 chunks per SM: chunks of several tiles
    yield "one_worker", [30000 if w == p // 2 else 0 for w in range(p)], "few"
    yield "tiny", [(0, 1, 2)[w % 3] for w in range(p)], "uniform"
    yield "tiny_equal", [(2, 1, 0)[w % 3] for w in range(p)], "equal"
    yield "all_empty", [0] * p, "uniform"
    yield "tile_edges", [(t - 1, t, t + 1, 2 * t + 1)[w % 4] for w in range(p)], "few"
    yield "many_tiles", [big if w == 0 else 5000 for w in range(p)], "few"


@pytest.mark.parametrize("p", [2, 5, 8])
@pytest.mark.parametrize("d", SHAPE_DESCS, ids=lambda d: d.name)
def test_worker_counts_and_shard_shapes(ctx, d, p):
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.RandomState(p * 5 + d.item_bytes + d.descending)
    for name, sizes, dist in _shapes(d, p, sm):
        shards = [S.make_items(d, n, dist, int(rng.randint(1 << 30))) for n in sizes]
        try:
            check(ctx, d, shards, p, int(rng.randint(1 << 40)))
        except AssertionError as e:
            raise AssertionError("%s: %s" % (name, e))


# ---- arguments ----------------------------------------------------------------------------------------------------------------
def test_argument_errors(ctx):
    L = ctx.L
    a = np.arange(100, dtype=np.uint64)
    d = U64.capi()
    dev = ctx.to_device(a)
    out = ctx.alloc(800)
    spl = np.zeros((16, 24), np.uint8)
    counts = np.zeros(17 * 17, np.uint64)

    def call(p, desc=C.byref(d), shards=True, n=100, splitters=True, outs=True, cnt=True):
        P = (C.c_void_p * 17)(*([dev] * 17)) if shards else None
        N = (C.c_size_t * 17)(*([n] * 17))
        O_ = (C.c_void_p * 17)(*([out] * 17)) if outs else None
        return L.tg_sort_select(ctx.h, desc, P, N, p, 1, spl.ctypes.data if splitters else None, O_,
                                _u64p(counts) if cnt else None, None)

    for p in (0, 1, 17):
        assert call(p) == TG_ERR_ARG, p
    assert call(2, desc=C.byref(_capi().record_desc())) == TG_ERR_ARG
    assert call(2, desc=C.byref(_capi().KeyDesc(4, 0, 4, BE, 0, 1))) == TG_ERR_ARG
    assert call(2, desc=None) == TG_ERR_ARG
    assert call(2, shards=False) == TG_ERR_ARG
    assert call(2, splitters=False) == TG_ERR_ARG
    assert call(2, outs=False) == TG_ERR_ARG
    assert call(2, cnt=False) == TG_ERR_ARG
    P = (C.c_void_p * 2)(dev, None)
    assert L.tg_sort_select(ctx.h, C.byref(d), P, (C.c_size_t * 2)(100, 5), 2, 1, spl.ctypes.data,
                            (C.c_void_p * 2)(out, out), _u64p(counts), None) == TG_ERR_ARG           # a NULL shard of 5 items
    assert call(3, n=1 << 30) == TG_ERR_TOO_LARGE
    # ReduceToIndex's range route through the exchange (counts only): 2..16 workers, the counts, a shard pointer where there are
    # items, (size - 1) * p < 2^64, shards below 2^30 items
    rc = np.zeros(17 * 17, np.uint64)

    def rng_call(p, shard=dev, n=50, size=1000, cnt=True):
        q = max(p, 1)
        return L.tg_exchange_select(ctx.h, _capi().ROUTE_RANGE, 1, None, 0, size, (C.c_void_p * q)(shard, *([None] * (q - 1))),
                                    (C.c_size_t * q)(n, *([0] * (q - 1))), p, None, None, _u64p(rc) if cnt else None)

    for p in (0, 1, 17):
        assert rng_call(p) == TG_ERR_ARG, p
    assert rng_call(4, cnt=False) == TG_ERR_ARG
    assert rng_call(4, shard=None) == TG_ERR_ARG
    assert rng_call(4, size=(1 << 62) + 2) == TG_ERR_ARG                # k * p would overflow
    assert rng_call(4, n=1 << 30) == TG_ERR_TOO_LARGE
    assert rng_call(4) == 0 and rc[:16].tolist() == [50] + [0] * 15     # 50 items, indices 0, 2, .., 98 of 1000: worker 0
    ctx.free(dev)
    ctx.free(out)
    # the ctx still works
    rng = np.random.RandomState(3)
    check(ctx, KV, [S.make_items(KV, int(n), "few", j) for j, n in enumerate(rng.randint(0, 3000, size=4))], 4, 11)
