"""The exchange model (exchange_ref.py) against the reference's p-worker outputs stored in the join and group fixtures (the
operator downstream of the exchange run on the model's windows, worker by worker), against the placement rules of the other
models, and against tg_exchange_plan, the arithmetic every rank runs on the count matrix.  CPU only."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import exchange_ref as X
import group_ref as G
import join_ref as J
import sample_sort_ref as S
import sort_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_JOIN = os.path.join(HERE, "golden", "reference_outputs_join.npz")
GOLDEN_GROUP = os.path.join(HERE, "golden", "reference_outputs_group.npz")


def _load(path):
    if not os.path.exists(path):
        pytest.skip("%s is not present" % os.path.relpath(path, HERE))
    return np.load(path)


def _rows16(a):
    return R.rows(a, 16)


def test_windows_join_the_reference_outputs():
    """InnerJoin at p workers: each side through the hash route, then the join of window d's two sides on worker d"""
    g = _load(GOLDEN_JOIN)
    checked = 0
    for key in sorted(k for k in g.files if "/out_p" in k):
        name, p = key.split("/")[0], int(key.rsplit("_p", 1)[1])
        sides = []
        for side in ("left", "right"):
            shards = [_rows16(s) for s in J.split_shards(g["%s/%s" % (name, side)].view(J.KV), p)]
            wins, counts = X.exchange(shards, X.owners(X.HASH, shards, p), p)
            assert counts.sum() == sum(len(s) for s in shards)
            sides.append([w.view(J.KV).reshape(-1) for w in wins])
        outs = [J.join_local(sides[0][d], sides[1][d], J.KEY_VALUES) for d in range(p)]
        rows = np.concatenate(outs).view(np.uint64).reshape(-1, 3)
        rows = rows[np.lexsort(rows.T[::-1])]
        ref = g[key]
        if ref.dtype == np.uint8:
            assert hashlib.sha256(np.ascontiguousarray(rows).tobytes()).digest() == ref.tobytes(), key
        else:
            assert np.array_equal(rows, ref.reshape(-1, 3)), key
        checked += p > 1
    assert checked >= 5


def test_windows_group_the_reference_outputs():
    """GroupByKey / GroupToIndex at p workers: the mod or range route, then worker d's group loop on window d, row for row"""
    g = _load(GOLDEN_GROUP)
    checked = 0
    for k in sorted(g.files):
        if k.endswith("/in") or k.endswith("_counts"):
            continue
        name, rest = k.split("/")
        case, p = rest.rsplit("_p", 1)
        p = int(p)
        shards = [_rows16(s) for s in G.split_shards(g[name + "/in"].view(G.KV), p)]
        if case.startswith("key_"):
            wins, _ = X.exchange(shards, X.owners(X.MOD, shards, p), p)
            outs = [G.group_rows(G.grouped(w.view(G.KV).reshape(-1)), case[4:], d) for d, w in enumerate(wins)]
        else:
            size = int(case[6:])
            wins, _ = X.exchange(shards, X.owners(X.RANGE, shards, p, size=size), p)
            outs = [G.index_rows(G.grouped(w.view(G.KV).reshape(-1)), size, p, d) for d, w in enumerate(wins)]
        assert [len(o) for o in outs] == g[k + "_counts"].tolist(), k
        rows, ref = np.concatenate(outs), g[k]
        if ref.dtype == np.uint8:
            assert hashlib.sha256(np.ascontiguousarray(rows, np.uint64).tobytes()).digest() == ref.tobytes(), k
        else:
            assert np.array_equal(rows, ref.reshape(-1, 7)), k
        checked += p > 1
    assert checked >= 20


@pytest.mark.parametrize("p", [2, 3, 5, 16])
def test_windows_agree_with_the_other_models(p):
    rng = np.random.RandomState(p)
    kv = [G.make_input(int(n), 1 << 40, int(s)) for n, s in zip(rng.randint(0, 700, p), rng.randint(0, 1 << 30, p))]
    kv[p // 2] = kv[p // 2][:0]                                            # an empty shard
    shards = [_rows16(s) for s in kv]
    for route, want in ((X.HASH, J.exchange(kv, p)), (X.MOD, G.exchange(kv, lambda k: G.owner_mod(k, p))),
                        (X.RANGE, G.exchange(kv, lambda k: G.owner_range(k, 1 << 39, p)))):
        wins, counts = X.exchange(shards, X.owners(route, shards, p, size=1 << 39), p)
        for d in range(p):
            assert np.array_equal(wins[d], _rows16(want[d])), (route, d)
        assert counts.sum(axis=0).tolist() == [len(w) for w in want]
    # the splitter route: window d is bucket d of every shard's classification by tg_sort_select's model, in shard order
    d8 = R.Desc(8, 0, 8, R.LE)
    items = [S.make_items(d8, int(n), "few", int(s)) for n, s in zip(rng.randint(0, 3000, p), rng.randint(0, 1 << 30, p))]
    _, counts_ref, grouped, _ = S.select(items, d8, p, 77)
    wins, counts = X.exchange(items, X.owners(X.SPLITTERS, items, p, d=d8, seed=77), p)
    assert np.array_equal(counts, counts_ref)
    for d in range(p):
        parts = [grouped[w][int(counts_ref[w, :d].sum()):int(counts_ref[w, :d + 1].sum())] for w in range(p)]
        assert np.array_equal(wins[d], np.concatenate(parts)), d


def test_record_tuples():
    d = R.Desc(100, 90, 10, R.BE)
    rec = R.make_items(d, 5, "uniform", 3)
    t = X.tuples(rec, d)
    assert np.array_equal(t[:, :10], rec[:, 90:100]) and not t[:, 10:12].any()
    assert np.ascontiguousarray(t[:, 12:]).view("<u4").reshape(-1).tolist() == list(range(5))


@pytest.mark.parametrize("p", [1, 2, 3, 7, 16])
def test_plan_equals_tg_exchange_plan(p):
    from thrill_b200 import capi
    L = capi.lib()
    rng = np.random.RandomState(p)
    for trial in range(20):
        counts = rng.randint(0, 1 << 29, size=(p, p)).astype(np.uint32)
        counts[rng.rand(p, p) < 0.3] = 0
        if trial == 0:
            counts[:] = 0
        flat = np.ascontiguousarray(counts.reshape(-1))
        for me in range(p):
            out = [np.zeros(p, np.uint64) for _ in range(3)]
            nr, worst = C.c_uint64(), C.c_uint64()
            assert L.tg_exchange_plan(p, me, flat.ctypes.data_as(C.POINTER(C.c_uint32)),
                                      *[o.ctypes.data_as(C.POINTER(C.c_uint64)) for o in out], C.byref(nr), C.byref(worst)) == 0
            send, recv, before, n_recv, w = X.plan(counts, me)
            assert out[0].tolist() == send.tolist() and out[1].tolist() == recv.tolist() and out[2].tolist() == before.tolist()
            assert (nr.value, worst.value) == (n_recv, w)
    assert L.tg_exchange_plan(0, 0, flat.ctypes.data_as(C.POINTER(C.c_uint32)), None, None, None, None, None) == -3
    assert L.tg_exchange_plan(p, p, flat.ctypes.data_as(C.POINTER(C.c_uint32)), None, None, None, None, None) == -3


def test_size_verdict():
    a = [np.zeros((3, 16), np.uint8)] * 2
    assert not X.too_large(a, np.array([[1 << 29, 0], [(1 << 29) - 1, 0]]))
    assert X.too_large(a, np.array([[1 << 29, 0], [1 << 29, 0]]))
