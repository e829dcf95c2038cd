"""The numpy model of InnerJoin on records (join_records_ref.py) against a brute force written from the definition: key
extraction, placement, the per-worker order, the window layout of the simulated exchange, output counts and the limit verdict.
No GPU."""
import os

import numpy as np
import pytest

import join_ref as JP
import join_records_ref as J


def brute_key(row, off, nb):
    return int.from_bytes(bytes(row[off:off + nb]), "little")


def brute_join(lefts, rights, lk, rk):
    """every worker's result from the definition: all (l, r) with equal keys on the key's owner, sorted by (key, left global
    position, right global position)"""
    p = len(lefts)
    L = [(g, r) for g, r in enumerate(np.concatenate(lefts))]
    R = [(g, r) for g, r in enumerate(np.concatenate(rights))]
    out = [[] for _ in range(p)]
    for gl, l in L:
        kl = brute_key(l, *lk)
        for gr, r in R:
            if brute_key(r, *rk) == kl:
                out[int(JP.owner(np.array([kl], np.uint64), p)[0])].append((kl, gl, gr, np.concatenate([l, r])))
    res = []
    for d in range(p):
        rows = [x[3] for x in sorted(out[d], key=lambda x: x[:3])]
        s = lefts[0].shape[1] + rights[0].shape[1]
        res.append(np.array(rows, np.uint8).reshape(-1, s))
    return res


def shards_of(rec, p, seed):
    cuts = np.sort(np.random.default_rng(seed).integers(0, len(rec) + 1, p - 1))
    return np.split(rec, cuts)


@pytest.mark.parametrize("lb,lk,rb,rk", [(4, (0, 4), 4, (0, 4)), (12, (5, 2), 24, (3, 5)), (24, (3, 5), 8, (7, 1)),
                                         (16, (8, 8), 12, (4, 8)), (176, (0, 8), 152, (0, 8))])
@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_model_against_brute_force(lb, lk, rb, rk, p):
    rng = np.random.default_rng(lb + rb + p)
    l = J.set_keys(J.make_records(60, lb, 1), lk[0], lk[1], rng.integers(0, 9, 60, dtype=np.uint64))
    r = J.set_keys(J.make_records(45, rb, 2), rk[0], rk[1], rng.integers(0, 9, 45, dtype=np.uint64))
    lefts, rights = shards_of(l, p, 1), shards_of(r, p, 2)
    got, want = J.join(lefts, rights, lk, rk), brute_join(lefts, rights, lk, rk)
    for d in range(p):
        assert np.array_equal(got[d], want[d]), d
    assert sum(len(x) for x in got) == J.output_count(J.keys_of(l, *lk), J.keys_of(r, *rk))


def test_key_extraction():
    rec = J.make_records(500, 24, 7)
    for off, nb in [(0, 1), (3, 5), (16, 8), (21, 3), (7, 2)]:
        k = J.keys_of(rec, off, nb)
        assert [int(x) for x in k[:50]] == [brute_key(row, off, nb) for row in rec[:50]]
        assert np.all(k < np.uint64(1 << (8 * nb))) if nb < 8 else True
    # set_keys writes exactly the key bytes
    before = rec.copy()
    J.set_keys(rec, 3, 5, np.arange(500, dtype=np.uint64) * np.uint64(1 << 33))
    assert np.array_equal(rec[:, :3], before[:, :3]) and np.array_equal(rec[:, 8:], before[:, 8:])
    assert np.array_equal(J.keys_of(rec, 3, 5), (np.arange(500, dtype=np.uint64) * np.uint64(1 << 33)) & np.uint64((1 << 40) - 1))


def test_records_are_a_pure_function_of_the_global_index():
    a = J.make_records(100, 16, 3)
    assert np.array_equal(a[40:], J.make_records(60, 16, 3, first=40))
    assert not np.array_equal(a, J.make_records(100, 16, 4))


def test_exchange_layout_and_counts():
    rng = np.random.default_rng(5)
    p = 5
    shards = [J.set_keys(J.make_records(n, 12, 9, first=10000 * w), 5, 2, rng.integers(0, 300, n, dtype=np.uint64))
              for w, n in enumerate([30, 0, 17, 50, 1])]
    win = J.exchange(shards, (5, 2), p)
    counts = J.exchange_counts(shards, (5, 2), p).reshape(p, p)
    for d in range(p):
        # grouped by source worker in rank order, each group in input order
        exp = [sh[JP.owner(J.keys_of(sh, 5, 2), p) == d] for sh in shards]
        assert np.array_equal(win[d], np.concatenate(exp))
        assert len(win[d]) == counts[:, d].sum()
    assert counts.sum() == sum(len(x) for x in shards)


def test_pairs_match_the_pair_join_model():
    left, right = JP.make_side(3000, 400, 1), JP.make_side(2500, 400, 2)
    rows = J.join_local(left.view(np.uint8).reshape(-1, 16), right.view(np.uint8).reshape(-1, 16), (0, 8), (0, 8))
    ref = JP.join_local(left, right, JP.KEY_VALUES)
    w = rows.view(np.uint64).reshape(-1, 4)
    assert np.array_equal(w[:, 0], ref["key"]) and np.array_equal(w[:, 1], ref["v1"]) and np.array_equal(w[:, 3], ref["v2"])


def test_limits():
    one = np.zeros((1, 8), np.uint8)
    assert not J.too_large([one], [one], (0, 8), (0, 8))
    kl, kr = np.full(40000, 5, np.uint64), np.full(30000, 5, np.uint64)
    assert J.output_count(kl, kr) == 1_200_000_000 > J.LIMIT
    a = J.set_keys(np.zeros((40000, 4), np.uint8), 0, 4, kl)
    b = J.set_keys(np.zeros((30000, 4), np.uint8), 0, 4, kr)
    assert J.too_large([a], [b], (0, 4), (0, 4))
    assert J.too_large([a[:20000], a[20000:]], [b[:1], b[1:]], (0, 4), (0, 4))
    assert not J.too_large([a[:300]], [b[:200]], (0, 4), (0, 4))


def test_digest_is_order_independent():
    rows = J.make_records(1000, 40, 3)
    perm = rows[np.random.default_rng(1).permutation(1000)]
    assert J.digest(rows) == J.digest(perm)
    rows2 = rows.copy()
    rows2[5, 7] ^= 1
    assert J.digest(rows2) != J.digest(rows)
    assert np.array_equal(J.multiset(rows), J.multiset(perm))


# ---- the stock api::InnerJoin's outputs (tests/golden/reference_outputs_join_records.npz) ------------------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_outputs_join_records.npz")


def test_goldens_against_the_model():
    g = np.load(GOLDEN)
    seen = 0
    for name, left, right, lk, rk, outs in J.golden_cases(g):
        # the fixture's inputs are the ones the generator makes now
        assert tuple(int(x) for x in g[name + "/inputs"]) == J.digest(left) + J.digest(right), name
        assert sorted(outs) == [1, 2, 3, 4], name
        for p, stored in outs.items():
            lefts = [left[a:b] for a, b in (shard_range(len(left), p, r) for r in range(p))]
            rights = [right[a:b] for a, b in (shard_range(len(right), p, r) for r in range(p))]
            rows = np.concatenate(J.join(lefts, rights, lk, rk))
            assert J.matches_golden(rows, stored), (name, p)
            seen += 1
    assert seen == 44


def shard_range(n, p, r):
    return (r * n) // p, ((r + 1) * n) // p
