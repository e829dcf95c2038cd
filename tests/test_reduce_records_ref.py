"""CPU checks of the numpy model of ReduceByKey on records (reduce_records_ref.py): against a brute force per key, across worker
counts, and under the reduce_ref contract."""
import struct

import numpy as np
import pytest

import reduce_records_ref as RR
from join_records_ref import keys_of

# (item bytes, key (offset, bytes), runs)
SHAPES = [
    (40, (0, 8), [(8, 3, 0), (32, 1, 1)]),                      # k-means: {cluster_id; {double p[3]; size_t count}}
    (40, (0, 8), [(32, 1, 1)]),                                 # ... its count-only second reduce
    (176, (3, 1), [(8, 2, 1), (24, 3, 0), (56, 1, 2), (64, 4, 5)]),
    (24, (13, 5), [(4, 1, 3)]),
    (4, (0, 4), []),
    (36, (32, 3), [(0, 2, 4), (16, 2, 5)]),
]


def _brute(rec, key, runs):
    ops = {0: lambda a, b: struct.unpack("<Q", struct.pack("<d", struct.unpack("<d", struct.pack("<Q", a))[0] +
                                                              struct.unpack("<d", struct.pack("<Q", b))[0]))[0],
           1: lambda a, b: (a + b) % (1 << 64), 2: min, 3: max}
    first, acc = {}, {}
    for i, k in enumerate(keys_of(rec, *key).tolist()):
        if k not in first:
            first[k] = rec[i].copy()
            acc[k] = [RR.fields(rec[i:i + 1], off, cnt)[0].tolist() for off, cnt, _ in runs]
            continue
        for r, (off, cnt, op) in enumerate(runs):
            v = RR.fields(rec[i:i + 1], off, cnt)[0].tolist()
            acc[k][r] = [ops[op](a, b) for a, b in zip(acc[k][r], v)]
    out = []
    for k in sorted(first):
        row = first[k]
        for r, (off, cnt, _) in enumerate(runs):
            RR.set_fields(row[None, :], off, cnt, [acc[k][r]])
        out.append(row)
    return np.array(out, np.uint8).reshape(len(out), rec.shape[1])


@pytest.mark.parametrize("shape", range(len(SHAPES)))
def test_model_matches_brute_force(shape):
    s, key, runs = SHAPES[shape]
    runs = [r for r in runs if r[2] in (0, 1, 2, 3)]
    n = 700
    rng = np.random.default_rng(shape)
    keys = rng.integers(0, min(50, 1 << (8 * key[1])), size=n, dtype=np.uint64)
    rec = RR.make(n, s, key, keys, seed=shape)
    for j, (off, cnt, op) in enumerate(runs):
        RR.set_fields(rec, off, cnt, RR.values(op, n, cnt, seed=shape * 10 + j))
    assert np.array_equal(RR.reduce_local(rec, key, runs), _brute(rec, key, runs))


@pytest.mark.parametrize("shape", range(len(SHAPES)))
@pytest.mark.parametrize("p", [1, 2, 3, 5, 16])
def test_workers_give_the_global_result(shape, p):
    """with exact folds, p workers hold, between them, the one-worker result: each key on its owner, in ascending key order"""
    s, key, runs = SHAPES[shape]
    n = 1500
    rng = np.random.default_rng(100 + shape)
    keys = rng.integers(0, min(300, 1 << (8 * key[1])), size=n, dtype=np.uint64)
    rec = RR.make(n, s, key, keys, seed=shape + 7)
    for j, (off, cnt, op) in enumerate(runs):
        RR.set_fields(rec, off, cnt, RR.values(op, n, cnt, seed=shape * 10 + j))
    cuts = np.sort(rng.integers(0, n + 1, size=p - 1))
    shards = np.split(rec, cuts)
    outs = RR.reduce(shards, key, runs)
    one = RR.reduce_local(rec, key, runs)
    own = RR.owner(keys_of(one, *key), p)
    for d in range(p):
        assert np.array_equal(outs[d], one[own == d])
        RR.check(rec[RR.owner(keys_of(rec, *key), p) == d], outs[d], key, runs)


def test_minmax_f64_picks_the_earliest_and_skips_nans():
    key = (0, 8)
    runs = [(8, 1, 4), (16, 1, 5)]
    nan1, canon = 0x7FF0000000000001, 0x7FF8000000000000
    neg0, pos0 = 0x8000000000000000, 0
    rows = [  # key, min field, max field
        (1, canon, canon), (1, nan1, nan1), (1, canon, canon),       # every value a NaN: the first non-canonical one
        (2, pos0, neg0), (2, neg0, pos0), (2, nan1, nan1),           # equal zeros: the earliest
        (3, canon, canon),                                           # only the canonical NaN
    ]
    rec = np.zeros((len(rows), 24), np.uint8)
    RR.set_fields(rec, 0, 3, [list(r) for r in rows])
    out = RR.reduce_local(rec, key, runs)
    got = RR.fields(out, 8, 2).tolist()
    assert got == [[nan1, nan1], [pos0, neg0], [canon, canon]]
    RR.check(rec, out, key, runs)
