"""Plain restatement of GroupByKey's and GroupToIndex's results (test helper, numpy only).

The input is a DIA of pair<uint64_t, 8-byte value> (the KV dtype), given as one shard per worker; its global order is the
concatenation of the shards.  Each item goes to the owner of its key:
    GroupByKey    worker key % p (std::hash<uint64_t> is the identity)
    GroupToIndex  worker k * p // size, for k < size (worker r answers for [ceil(r * size / p), ceil((r + 1) * size / p)))
A worker's grouped items are its received items stably sorted by the key (so equal keys keep their global order).  The host
loop then calls the group function once per group (GroupByKey), or once per index of the worker's range with the neutral
element where an index has no items (GroupToIndex).  A worker holds at most 2^30 - 1 items before and after the exchange.

The group functions of the fixtures (tests/golden/make_golden_group.py) give rows of 7 uint64 words:
    stats    (rank, key, count, sum of values, xor of splitmix64(value), min value, max value)
    partial  (rank, key, items read, 0, 0, 0, 0): reads at most 3 items, so a group of c items gives ceil(c / 3) rows
GroupToIndex's neutral element is (rank, ~0, 0, 0, 0, 0, 0).
"""
import numpy as np

KV = np.dtype([("key", "<u8"), ("val", "<u8")])
LIMIT = (1 << 30) - 1
U64_MAX = (1 << 64) - 1
STATS, PARTIAL = "stats", "partial"


def splitmix64(x):
    with np.errstate(over="ignore"):
        z = np.asarray(x, np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def owner_mod(keys, p):
    """GroupByKey's owner of each key"""
    return (np.asarray(keys, np.uint64) % np.uint64(p)).astype(np.int64)


def owner_range(keys, size, p):
    """GroupToIndex's owner of each index; an index >= size is parked on the last worker"""
    k = np.asarray(keys, np.uint64)
    ok = k < np.uint64(size)
    with np.errstate(over="ignore", divide="ignore"):
        d = np.where(ok, (k * np.uint64(p)) // np.uint64(max(size, 1)), np.uint64(p - 1))
    return d.astype(np.int64)


def range_begin(r, size, p):
    return (r * size + p - 1) // p


def exchange(shards, owner):
    """each worker's received items: the items it owns, in global order.  owner(keys) -> worker of each key"""
    p = len(shards)
    allv = np.concatenate(shards) if len(shards) else np.zeros(0, KV)
    own = owner(allv["key"]) if len(allv) else np.zeros(0, np.int64)
    return [allv[own == d] for d in range(p)]


def grouped(items):
    """one worker's device result: its items stably sorted by the key"""
    return items[np.argsort(items["key"], kind="stable")]


def group_rows(items, fn, rank):
    """the group function over one worker's grouped items, GroupByKey's loop: rows of 7 uint64"""
    if not len(items):
        return np.zeros((0, 7), np.uint64)
    keys, first, counts = np.unique(items["key"], return_index=True, return_counts=True)
    if fn == PARTIAL:
        reps = (counts + 2) // 3
        rows = np.zeros((int(reps.sum()), 7), np.uint64)
        rows[:, 1] = np.repeat(keys, reps)
        read = np.full(len(rows), 3, np.uint64)
        last = np.cumsum(reps) - 1
        read[last] = (counts - 3 * (reps - 1)).astype(np.uint64)
        rows[:, 2] = read
    else:
        v = items["val"]
        rows = np.zeros((len(keys), 7), np.uint64)
        rows[:, 1] = keys
        rows[:, 2] = counts.astype(np.uint64)
        with np.errstate(over="ignore"):
            rows[:, 3] = np.add.reduceat(v, first)
        rows[:, 4] = np.bitwise_xor.reduceat(splitmix64(v), first)
        rows[:, 5] = np.minimum.reduceat(v, first)
        rows[:, 6] = np.maximum.reduceat(v, first)
    rows[:, 0] = rank
    return rows


def index_rows(items, size, p, rank):
    """GroupToIndex's loop over one worker's grouped items with the stats function: one row per index of its range"""
    b, e = range_begin(rank, size, p), range_begin(rank + 1, size, p)
    rows = np.zeros((e - b, 7), np.uint64)
    rows[:, 0] = rank
    rows[:, 1] = U64_MAX
    g = group_rows(items, STATS, rank)
    if len(g):
        assert int(g[-1, 1]) < e and int(g[0, 1]) >= b, "an index outside the worker's range"
        rows[g[:, 1].astype(np.int64) - b] = g
    return rows


def group_by_key(shards, fn):
    """the p = len(shards) workers' rows"""
    p = len(shards)
    ex = exchange(shards, lambda k: owner_mod(k, p))
    return [group_rows(grouped(ex[d]), fn, d) for d in range(p)]


def group_to_index(shards, size):
    p = len(shards)
    ex = exchange(shards, lambda k: owner_range(k, size, p))
    return [index_rows(grouped(ex[d]), size, p, d) for d in range(p)]


def split_shards(a, p):
    """an input split into p contiguous shards (Generate's even split)"""
    b = [(r * len(a) + p - 1) // p for r in range(p + 1)]
    return [a[b[r]:b[r + 1]] for r in range(p)]


def pairs(keys, vals):
    out = np.empty(len(keys), KV)
    out["key"], out["val"] = np.asarray(keys, np.uint64), np.asarray(vals, np.uint64)
    return out


def make_input(n, universe, seed):
    """n pairs with keys uniform over [0, universe) and random values"""
    rng = np.random.RandomState(seed)
    keys = rng.randint(0, universe, size=n, dtype=np.uint64) if universe else np.zeros(n, np.uint64)
    return pairs(keys, rng.randint(0, 1 << 62, size=n, dtype=np.uint64) * np.uint64(3) + np.uint64(1))
