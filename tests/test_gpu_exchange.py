"""The collective operators' exchange on one H100: tg_exchange_select runs each simulated worker's count step and store step
(the peer-store pass, mode 1, or the local partition with the transfers as device copies, mode 0) into windows carved out of
one allocation, for every route.  Checked bit for bit against exchange_ref.py: the windows, the count matrix, the guard bytes
around and between the windows, and the shards.  Then the operators composed on the windows (the p = 1 code on each window, as
the p > 1 operators run it after their exchange) against the reference's p-worker outputs, the argument errors, and the receive
limit.  pytest -m gpu."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import exchange_ref as X
import group_ref as G
import join_ref as J
import reduce_ref as RR
import sample_sort_ref as S
import sort_ref as R

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4
TILE = {8: 16384, 16: 8192}                       # items per tile of the partition pass (128 KB)
GUARD = 128 << 10                                 # guard zone: at least one tile of bytes before, between and after the windows
PATTERN = 0xA5
RANGE_SIZE = (1 << 34) + 3
D8, D16, DREC = R.Desc(8, 0, 8, R.LE), R.Desc(16, 0, 16, R.BE), R.Desc(100, 90, 10, R.BE)
# route, item descriptor (the splitter route's key descriptor; 16-byte (key, value) items otherwise)
ROUTES = [("hash", None), ("mod", None), ("range", None), ("splitters8", D8), ("splitters16", D16), ("records", DREC)]


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _route(name):
    return X.SPLITTERS if name.startswith("splitters") or name == "records" else X.ROUTES[name]


def _ib(desc):
    return desc.item_bytes if desc is not None else 16


def _u64p(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint64))


def _align(x, a=256):
    return (x + a - 1) // a * a


def select(ctx, route, mode, shards, p, desc=None, seed=0, size=0, recv=None, windows=True, call_p=None, shard_n=None):
    """tg_exchange_select on host shards, with windows of recv[d] items each carved out of one pattern-filled allocation.
    Returns (status, counts (p, p), windows, guard_ok, shards_ok)."""
    ib = _ib(desc)
    d_sh = [ctx.to_device(s) if len(s) else None for s in shards]
    recv = recv if recv is not None else [0] * p
    wbytes = [int(r) * ib for r in recv]
    offs, o = [], GUARD
    for b in wbytes:
        offs.append(o)
        o = _align(o + b) + GUARD
    total = o
    buf = ctx.alloc(total)
    ctx.upload(buf, np.full(total, PATTERN, np.uint8))
    counts = np.zeros(p * p, np.uint64)
    P = call_p if call_p is not None else p
    kd = C.byref(desc.capi()) if desc is not None else None
    W = (C.c_void_p * p)(*[buf + off for off in offs]) if windows else None
    WB = (C.c_size_t * p)(*wbytes) if windows else None
    N = shard_n if shard_n is not None else [len(s) for s in shards]
    st = ctx.L.tg_exchange_select(ctx.h, _route(route) if isinstance(route, str) else route, mode, kd, seed, size,
                                  (C.c_void_p * p)(*d_sh), (C.c_size_t * p)(*N), P, W, WB, _u64p(counts))
    raw = ctx.download(buf, total)
    wins = [raw[off:off + b].reshape(-1, ib) for off, b in zip(offs, wbytes)]
    outside = np.ones(total, bool)
    for off, b in zip(offs, wbytes):
        outside[off:off + b] = False
    guard_ok = bool((raw[outside] == PATTERN).all())
    shards_ok = all(np.array_equal(ctx.download(d, s.nbytes).reshape(s.shape), s) for d, s in zip(d_sh, shards) if d)
    for d in d_sh + [buf]:
        if d:
            ctx.free(d)
    return st, counts.reshape(p, p), wins, guard_ok, shards_ok


def model(route, shards, p, desc=None, seed=0, size=RANGE_SIZE):
    own = X.owners(_route(route), shards, p, size=size, d=desc, seed=seed)
    return X.exchange(shards, own, p)


def check(ctx, route, mode, shards, p, desc=None, seed=0, size=RANGE_SIZE):
    wins, counts = model(route, shards, p, desc, seed, size)
    recv = counts.sum(axis=0)
    st, got_counts, got, guard_ok, shards_ok = select(ctx, route, mode, shards, p, desc, seed, size, recv)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    assert np.array_equal(got_counts, counts), "count matrix"
    for d in range(p):
        assert np.array_equal(got[d], wins[d]), "window %d" % d
    assert guard_ok, "a byte outside the windows' receive sizes was written"
    assert shards_ok, "a shard was modified"
    return counts


# ---- shard contents ----------------------------------------------------------------------------------------------------------
def _kv(keys, rng):
    """16-byte items: the keys, values with random high bits and the item's position in the low bits (order shows)"""
    n = len(keys)
    out = np.empty(n, G.KV)
    out["key"] = keys
    out["val"] = (rng.randint(0, 1 << 30, n, dtype=np.uint64) << np.uint64(32)) | np.arange(n, dtype=np.uint64)
    return R.rows(out, 16)


def _owned_pool(route, p, want, rng, k=64):
    """k keys whose owner is in `want` under the route (hash, mod or range)"""
    pool = []
    for _ in range(100):
        cand = rng.randint(0, 1 << 62, 4096, dtype=np.uint64) * np.uint64(4) + rng.randint(0, 4, 4096, dtype=np.uint64)
        if route == "range":
            cand = cand % np.uint64(RANGE_SIZE + 5)
        own = X.owners(X.ROUTES[route], [_kv(cand, rng)], p, size=RANGE_SIZE)[0]
        pool.extend(cand[np.isin(own, want)].tolist())
        if len(pool) >= k:
            return np.array(pool[:k], np.uint64)
    raise AssertionError("no keys owned by %s under %s" % (want, route))


def make_shards(route, desc, p, sizes, kind, rng):
    """one shard per size.  kind: 'random', 'one_dest' (every item to the last worker), 'some_dest' (the odd workers receive
    nothing), 'dups' (heavy duplicates)"""
    out = []
    for n in sizes:
        n = int(n)
        if desc is not None:
            dist = {"random": "uniform", "dups": "few", "one_dest": "equal", "some_dest": "few"}[kind]
            out.append(S.make_items(desc, n, dist, int(rng.randint(1 << 30))))
            continue
        if kind == "random":
            keys = rng.randint(0, 1 << 63, n, dtype=np.uint64) * np.uint64(2) + rng.randint(0, 2, n, dtype=np.uint64)
            if route == "range":
                keys %= np.uint64(RANGE_SIZE + RANGE_SIZE // 50)           # ~2% at or above the size: the last worker
        elif kind == "dups":
            pool = _owned_pool(route, p, list(range(p)), rng, 7)
            keys = pool[rng.randint(0, len(pool), n)]
        else:
            want = [p - 1] if kind == "one_dest" else list(range(0, p, 2))
            pool = _owned_pool(route, p, want, rng)
            keys = pool[rng.randint(0, len(pool), n)]
        out.append(_kv(keys, rng))
    return out


def shapes(desc, p, sm):
    """(name, sizes, kind) of the shard shapes"""
    t = TILE[_ib(desc)] if _ib(desc) in TILE else TILE[16]
    big = (2 * sm + 37) * t + 123                    # more tiles than 2 chunks per SM: chunks of several tiles, tile groups
    yield "tile_edges", [(t - 1, t, t + 1, 2 * t + 1)[w % 4] for w in range(p)], "random"
    yield "many_tiles", [big if w == 1 else 3000 for w in range(p)], "random"
    yield "empty_first_middle_last", [0 if w in (0, p // 2, p - 1) else 5000 + 77 * w for w in range(p)], "random"
    yield "one_shard", [40000 if w == p - 1 else 0 for w in range(p)], "random"
    yield "one_dest", [3000 + w for w in range(p)], "one_dest"
    yield "some_dest", [t + 5 * w for w in range(p)], "some_dest"
    yield "dups", [20000 - 100 * w for w in range(p)], "dups"
    yield "tiny", [(0, 1, 2)[w % 3] for w in range(p)], "random"


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("route,desc", ROUTES, ids=[r for r, _ in ROUTES])
def test_windows_bit_for_bit(ctx, sm_count, route, desc, mode):
    rng = np.random.RandomState(17 * mode + len(route) + _ib(desc))
    for p in (2, 3, 5, 8, 16):
        for name, sizes, kind in shapes(desc, p, sm_count):
            if name == "many_tiles" and p not in ((2,) if _ib(desc) == 100 else (2, 5, 16)):
                continue                               # (the numpy model takes seconds per shape at millions of items)
            shards = make_shards(route, desc, p, sizes, kind, rng)
            seed = int(rng.randint(1 << 40))
            try:
                counts = check(ctx, route, mode, shards, p, desc, seed)
            except AssertionError as e:
                raise AssertionError("p=%d %s: %s" % (p, name, e))
            recv = counts.sum(axis=0)
            if kind == "one_dest" and desc is None:
                assert recv[p - 1] == sum(sizes), name
            if kind == "some_dest" and desc is None:
                assert not recv[1::2].any(), name


@pytest.mark.parametrize("p", list(range(2, 17)))
def test_mod_partition(ctx, p):
    """GroupByKey's route at every worker count: a popular key, keys with the high bit set (ModDigit's two 32-bit halves)"""
    arr = G.make_input(100000, 1 << 62, p)
    arr["key"][::7] = np.uint64(p * 1000 + 3)
    arr["key"][::11] |= np.uint64(1 << 63)
    arr["key"][::13] = np.uint64((1 << 64) - 1 - p)
    arr["val"] = np.arange(len(arr))
    for mode in (1, 0):
        check(ctx, "mod", mode, [R.rows(s, 16) for s in G.split_shards(arr, p)], p)


def range_keys(rng, n, size, p):
    keys = rng.randint(0, size, size=n, dtype=np.int64).astype(np.uint64)
    edges = sorted({S.begin_of_part(r, size, p) + o for r in range(p + 1) for o in (-1, 0, 1)} | {size, (1 << 64) - 1})
    special = np.array([e for e in edges if 0 <= e < (1 << 64)], dtype=np.uint64)
    at = rng.randint(0, n, size=min(n, 3 * len(special)))
    keys[at] = special[np.arange(len(at)) % len(special)]
    return keys


@pytest.mark.parametrize("p", [2, 3, 7, 16])
def test_range_partition(ctx, p):
    """ReduceToIndex's and GroupToIndex's route: indices at and around every worker's range boundary, at and above the size"""
    rng = np.random.RandomState(p)
    for size in (1, p - 1, p, p + 1, 1000, (1 << 34) + 3):
        for n in (8191, 8192, 8193, 3 * 8192 + 1):
            items = np.zeros(n, dtype=G.KV)
            items["key"] = range_keys(rng, n, max(size, 1), p)
            items["val"] = np.arange(n, dtype=np.uint64)
            shards = [R.rows(s, 16) for s in G.split_shards(items, p)]
            for mode in (1, 0):
                try:
                    check(ctx, "range", mode, shards, p, size=size)
                except AssertionError as e:
                    raise AssertionError("size %d, n %d, mode %d: %s" % (size, n, mode, e))


# ---- the operators composed on the windows -----------------------------------------------------------------------------------
def _exchange(ctx, route, mode, shards, p, desc=None, seed=0, size=0):
    """the windows tg_exchange_select fills (their receive sizes from a counts-only call)"""
    st, counts, _, _, _ = select(ctx, route, mode, shards, p, desc, seed, size, windows=False)
    assert st == 0, ctx.L.tg_last_error(ctx.h)
    st, counts, wins, guard_ok, shards_ok = select(ctx, route, mode, shards, p, desc, seed, size, counts.sum(axis=0))
    assert st == 0 and guard_ok and shards_ok, ctx.L.tg_last_error(ctx.h)
    return wins


def _result(ctx, out, n, ib):
    return ctx.download(out.value, n.value * ib).reshape(-1, ib) if n.value else np.zeros((0, ib), np.uint8)


def _sort1(ctx, desc, rows, seed):
    """tg_sort at p = 1 (the local sort the p-worker Sort runs on what it received)"""
    d = ctx.to_device(rows)
    out, n = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_sort(ctx.h, C.byref(desc.capi()), d, len(rows), seed, C.byref(out), C.byref(n)))
    res = _result(ctx, out, n, desc.item_bytes)
    ctx.free(d)
    return res


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("p", [2, 3, 4, 8])
def test_sort_composed(ctx, p, mode):
    """the splitter route, then the p = 1 sort of each window: the windows in worker order are the global stable sort"""
    rng = np.random.RandomState(p + 10 * mode)
    for desc in (D8, R.Desc(16, 0, 8, R.LE, 1), R.Desc(8, 0, 8, R.LE, 1), D16, DREC, R.Desc(12, 1, 11, R.BE)):
        for dist in ("uniform", "few", "equal"):
            shards = [S.make_items(desc, int(n), dist, int(rng.randint(1 << 30))) for n in rng.randint(0, 30000, p)]
            seed = int(rng.randint(1 << 40))
            wins = _exchange(ctx, "splitters", mode, shards, p, desc, seed)
            got = np.concatenate([_sort1(ctx, desc, w, seed) for w in wins])
            assert np.array_equal(got, R.sort(np.concatenate(shards), desc)), (desc.name, dist)


def _reduce1(ctx, op, rows):
    d = ctx.to_device(rows)
    out, n = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_reduce_by_key(ctx.h, C.byref(_capi().KVDesc(16, op)), d, len(rows), C.byref(out), C.byref(n)))
    res = _result(ctx, out, n, 16)
    ctx.free(d)
    return res


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("p", [2, 3, 4, 8])
def test_reduce_by_key_composed(ctx, p, mode):
    """pre phase (the p = 1 reduce of each shard), the hash route, post phase (the p = 1 reduce of each window): every key on
    its owner, once, with a value the reduce contract allows"""
    capi = _capi()
    rng = np.random.RandomState(p + 20 * mode)
    for op in (capi.OP_SUM_U64, capi.OP_SUM_F64, capi.OP_MIN_F64):
        for universe in (5, 3000, 1 << 40):
            kv = [G.make_input(int(n), universe, int(rng.randint(1 << 30))) for n in rng.randint(0, 40000, p)]
            if op != capi.OP_SUM_U64:
                for s in kv:
                    s["val"] = (rng.rand(len(s)) * 1e6).astype(np.float64).view(np.uint64)
            pre = [_reduce1(ctx, op, R.rows(s, 16)) for s in kv]
            wins = _exchange(ctx, "hash", mode, pre, p)
            outs = [_reduce1(ctx, op, w).view(G.KV).reshape(-1) for w in wins]
            for d in range(p):
                assert (J.owner(outs[d]["key"], p) == d).all(), "a key away from its owner"
            RR.check(np.concatenate(kv), np.concatenate(outs), op)


def _golden(name):
    path = os.path.join(HERE, "golden", name)
    if not os.path.exists(path):
        pytest.skip("tests/golden/%s is not present" % name)
    return np.load(path)


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("p", [2, 3, 4, 8])
def test_inner_join_composed(ctx, p, mode):
    """both sides through the hash route, then tg_inner_join at p = 1 on each window pair: each worker's rows exactly as the
    model orders them, and their union the reference's output at p workers"""
    g = _golden("reference_outputs_join.npz")
    keys = [k for k in g.files if k.endswith("/out_p%d" % p)]
    if not keys:
        pytest.skip("no join fixture at p = %d" % p)
    for key in sorted(keys):
        name = key.split("/")[0]
        sides = [J.split_shards(g["%s/%s" % (name, s)].view(J.KV), p) for s in ("left", "right")]
        wl, wr = [_exchange(ctx, "hash", mode, [R.rows(s, 16) for s in side], p) for side in sides]
        outs = []
        for d in range(p):
            dl, dr = ctx.to_device(wl[d]), ctx.to_device(wr[d])
            out, n = C.c_void_p(), C.c_size_t()
            ctx.ck(ctx.L.tg_inner_join(ctx.h, C.byref(_capi().JoinDesc(16, J.KEY_VALUES)), dl, len(wl[d]), dr, len(wr[d]),
                                       C.byref(out), C.byref(n)))
            outs.append(_result(ctx, out, n, 24).view(J.KEY_V1_V2).reshape(-1))
            ctx.free(dl)
            ctx.free(dr)
        want = J.join(sides[0], sides[1], J.KEY_VALUES)
        for d in range(p):
            assert np.array_equal(outs[d].view(np.uint64), want[d].view(np.uint64)), (key, d)
        rows = np.concatenate(outs).view(np.uint64).reshape(-1, 3)
        rows = rows[np.lexsort(rows.T[::-1])]
        ref = g[key]
        if ref.dtype == np.uint8:
            assert hashlib.sha256(np.ascontiguousarray(rows).tobytes()).digest() == ref.tobytes(), key
        else:
            assert np.array_equal(rows, ref.reshape(-1, 3)), key


def group_cases(g, p):
    out = []
    for k in g.files:
        if k.endswith("/in") or k.endswith("_counts"):
            continue
        name, rest = k.split("/")
        case, q = rest.rsplit("_p", 1)
        if int(q) == p:
            out.append((name, case))
    return sorted(out)


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("p", [2, 3, 4, 8])
def test_group_composed(ctx, p, mode):
    """GroupByKey / GroupToIndex: the mod or range route, then the p = 1 group of each window: worker d's rows are the
    reference's worker d"""
    g = _golden("reference_outputs_group.npz")
    for name, case in group_cases(g, p):
        shards = [R.rows(s, 16) for s in G.split_shards(g[name + "/in"].view(G.KV), p)]
        size = 0 if case.startswith("key_") else int(case[6:])
        wins = _exchange(ctx, "mod" if case.startswith("key_") else "range", mode, shards, p, size=size)
        rows = []
        for d in range(p):
            dw = ctx.to_device(wins[d])
            out, n = C.c_void_p(), C.c_size_t()
            ctx.ck(ctx.L.tg_group_by_key(ctx.h, dw, len(wins[d]), C.byref(out), C.byref(n)))
            res = _result(ctx, out, n, 16).view(G.KV).reshape(-1)
            ctx.free(dw)
            rows.append(G.group_rows(res, case[4:], d) if case.startswith("key_") else G.index_rows(res, size, p, d))
        key = "%s/%s_p%d" % (name, case, p)
        assert [len(r) for r in rows] == g[key + "_counts"].tolist(), key
        got, ref = np.concatenate(rows), g[key]
        if ref.dtype == np.uint8:
            assert hashlib.sha256(np.ascontiguousarray(got, np.uint64).tobytes()).digest() == ref.tobytes(), key
        else:
            assert np.array_equal(got, ref.reshape(-1, 7)), key


# ---- arguments and errors ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [1, 0])
def test_errors_leave_the_windows_untouched(ctx, mode):
    rng = np.random.RandomState(5)
    p = 4
    shards = make_shards("hash", None, p, [5000, 0, 7000, 300], "random", rng)
    _, counts = model("hash", shards, p)
    recv = counts.sum(axis=0)
    # counts only
    st, got, wins, guard_ok, _ = select(ctx, "hash", mode, shards, p, recv=recv, windows=False)
    assert st == 0 and np.array_equal(got, counts) and guard_ok
    # a window one item too small, each in turn
    for d in range(p):
        small = recv.copy()
        if small[d] == 0:
            continue
        small[d] -= 1
        st, got, wins, guard_ok, shards_ok = select(ctx, "hash", mode, shards, p, recv=small)
        assert st == TG_ERR_ARG and np.array_equal(got, counts), d
        assert guard_ok and all((w == PATTERN).all() for w in wins) and shards_ok, d
    # p outside 2..16, an unknown route or mode, descriptors the splitter route rejects
    for call_p in (0, 1, 17):
        st, _, wins, guard_ok, _ = select(ctx, "hash", mode, shards, p, recv=recv, call_p=call_p)
        assert st == TG_ERR_ARG and guard_ok and all((w == PATTERN).all() for w in wins), call_p
    for route, m in ((4, mode), (X.HASH, 2)):
        st, _, wins, guard_ok, _ = select(ctx, route, m, shards, p, recv=recv)
        assert st == TG_ERR_ARG and guard_ok and all((w == PATTERN).all() for w in wins), (route, m)
    for bad in (R.Desc(100, 0, 13, R.BE), R.Desc(102, 0, 10, R.BE), R.Desc(100, 0, 10, R.BE, 1), R.Desc(16, 8, 9, R.LE),
                R.Desc(16, 0, 0, R.BE), R.Desc(8, 4, 8, R.BE)):
        rows = [np.zeros((10, bad.item_bytes), np.uint8) for _ in range(p)]
        st, _, wins, guard_ok, _ = select(ctx, "splitters", mode, rows, p, bad, recv=[10] * p)
        assert st == TG_ERR_ARG and guard_ok and all((w == PATTERN).all() for w in wins), bad
    st, _, _, _, _ = select(ctx, X.SPLITTERS, mode, shards, p, None, recv=recv)
    assert st == TG_ERR_ARG
    st, _, _, _, _ = select(ctx, "range", mode, shards, p, recv=recv, size=(1 << 62) + 2)     # (size - 1) * p >= 2^64
    assert st == TG_ERR_ARG
    # a NULL shard with items
    L = ctx.L
    cnt = np.zeros(p * p, np.uint64)
    assert L.tg_exchange_select(ctx.h, X.HASH, mode, None, 0, 0, (C.c_void_p * p)(None, None, None, None),
                                (C.c_size_t * p)(5, 0, 0, 0), p, None, None, _u64p(cnt)) == TG_ERR_ARG
    # the ctx still works
    check(ctx, "hash", mode, shards, p)


# ---- the receive limit -------------------------------------------------------------------------------------------------------
def test_receive_limit(ctx):
    """one buffer of 2^30 pairs with key 0 (all owned by worker 0 under the mod route): two shards of 2^29 are over the limit
    with nothing stored; 2^29 and 2^29 - 1 fill worker 0's window with 2^30 - 1 items in order; a shard of 2^30 is over it"""
    import torch
    n = 1 << 30
    free, _ = torch.cuda.mem_get_info(0)
    if free < 2 * n * 16 + 8 * n + (4 << 30):
        pytest.skip("needs %.0f GB of device memory" % ((2 * n * 16 + 8 * n + (4 << 30)) / 2.0 ** 30))
    a = torch.zeros((n, 2), dtype=torch.int64, device="cuda:0")
    a[:, 1] = torch.arange(n, dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    base = a.data_ptr()
    L = ctx.L
    cnt = np.zeros(4, np.uint64)
    guard = torch.full((GUARD,), PATTERN, dtype=torch.uint8, device="cuda:0")

    def call(sizes, windows, wbytes):
        return L.tg_exchange_select(ctx.h, X.MOD, 1, None, 0, 0, (C.c_void_p * 2)(base, base + (1 << 29) * 16),
                                    (C.c_size_t * 2)(*sizes), 2, windows, wbytes, _u64p(cnt))

    g = guard.data_ptr()
    W, WB = (C.c_void_p * 2)(g, g), (C.c_size_t * 2)(GUARD, GUARD)
    assert call([1 << 29, 1 << 29], W, WB) == TG_ERR_TOO_LARGE
    assert cnt.tolist() == [1 << 29, 0, 1 << 29, 0]
    assert call([1 << 30, 0], W, WB) == TG_ERR_TOO_LARGE
    torch.cuda.synchronize()
    assert bool((guard == PATTERN).all())
    del guard
    m = n - 1
    win = torch.empty((m, 2), dtype=torch.int64, device="cuda:0")
    assert call([1 << 29, (1 << 29) - 1], (C.c_void_p * 2)(win.data_ptr(), None), (C.c_size_t * 2)(m * 16, 0)) == 0, \
        L.tg_last_error(ctx.h)
    assert cnt.tolist() == [1 << 29, 0, (1 << 29) - 1, 0]
    assert ctx.checksum(win.data_ptr(), m, 16) == ctx.checksum(base, m, 16)
    torch.cuda.synchronize()
    assert bool((win[:, 1][:: 1 << 20] == torch.arange(0, m, 1 << 20, device="cuda:0")).all())
    del a, win
    torch.cuda.empty_cache()
