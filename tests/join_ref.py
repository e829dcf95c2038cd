"""Plain restatement of InnerJoin's result (test helper, numpy only).

Both sides are DIAs of pair<uint64_t, 8-byte value> (the KV dtype), given as one shard per worker; a side's global order is
the concatenation of its shards.  Worker Hash128to64(0, key) % p owns a key and receives the items of both sides with that
key in global order.  Its result holds one item per matching (l, r), ordered by (key, left global position, right global
position):
    KEY_VALUES: (key, l.second, r.second)     VALUES: (l.second, r.second)
A worker's side (before or after the exchange) and a worker's output are limited to 2^30 - 1 items.
"""
import numpy as np

KV = np.dtype([("key", "<u8"), ("val", "<u8")])
KEY_V1_V2 = np.dtype([("key", "<u8"), ("v1", "<u8"), ("v2", "<u8")])
V1_V2 = np.dtype([("v1", "<u8"), ("v2", "<u8")])
KEY_VALUES, VALUES = 0, 1
LIMIT = (1 << 30) - 1


def hash128to64(upper, lower):
    """common/hash.hpp:64-73 on uint64 arrays (wrapping arithmetic)"""
    k = np.uint64(0x9DDFEA08EB382D69)
    with np.errstate(over="ignore"):
        a = (np.asarray(lower, np.uint64) ^ np.asarray(upper, np.uint64)) * k
        a ^= a >> np.uint64(47)
        b = (np.asarray(upper, np.uint64) ^ a) * k
        b ^= b >> np.uint64(47)
        b *= k
    return b


def owner(keys, p):
    """the worker that owns each key: Hash128to64(0, key) % p"""
    return (hash128to64(np.zeros(len(keys), np.uint64), np.asarray(keys, np.uint64)) % np.uint64(p)).astype(np.int64)


def out_dtype(fn):
    return KEY_V1_V2 if fn == KEY_VALUES else V1_V2


def join_local(left, right, fn):
    """one worker's result from its items of both sides, each in global order"""
    L = left[np.argsort(left["key"], kind="stable")]
    R = right[np.argsort(right["key"], kind="stable")]
    lo = np.searchsorted(R["key"], L["key"], "left").astype(np.int64)
    cnt = np.searchsorted(R["key"], L["key"], "right").astype(np.int64) - lo
    m = int(cnt.sum())
    li = np.repeat(np.arange(len(L), dtype=np.int64), cnt)
    off = np.cumsum(cnt) - cnt
    ri = lo[li] + (np.arange(m, dtype=np.int64) - off[li])
    out = np.empty(m, out_dtype(fn))
    if fn == KEY_VALUES:
        out["key"], out["v1"], out["v2"] = L["key"][li], L["val"][li], R["val"][ri]
    else:
        out["v1"], out["v2"] = L["val"][li], R["val"][ri]
    return out


def exchange(shards, p):
    """each worker's received items: the items it owns, in global order"""
    allv = np.concatenate(shards) if len(shards) else np.zeros(0, KV)
    own = owner(allv["key"], p)
    return [allv[own == d] for d in range(p)]


def output_counts(left, right):
    """the number of matching pairs of two item arrays"""
    kl, cl = np.unique(left["key"], return_counts=True)
    kr, cr = np.unique(right["key"], return_counts=True)
    _, il, ir = np.intersect1d(kl, kr, assume_unique=True, return_indices=True)
    return int((cl[il].astype(np.int64) * cr[ir].astype(np.int64)).sum())


def too_large(lefts, rights):
    """the size verdict on p = len(lefts) workers: a worker's side over the limit before or after the exchange, or a worker's
    output over the limit"""
    p = len(lefts)
    if any(len(x) > LIMIT for x in lefts) or any(len(x) > LIMIT for x in rights):
        return True
    el, er = exchange(lefts, p), exchange(rights, p)
    if any(len(x) > LIMIT for x in el) or any(len(x) > LIMIT for x in er):
        return True
    return any(output_counts(el[d], er[d]) > LIMIT for d in range(p))


def join(lefts, rights, fn):
    """the p = len(lefts) workers' results"""
    p = len(lefts)
    el, er = exchange(lefts, p), exchange(rights, p)
    return [join_local(el[d], er[d], fn) for d in range(p)]


def brute_force(lefts, rights, fn, p):
    """the same by the definition: every (l, r) pair in global order, placed by owner, ordered by (key, l pos, r pos)"""
    L = np.concatenate(lefts) if len(lefts) else np.zeros(0, KV)
    R = np.concatenate(rights) if len(rights) else np.zeros(0, KV)
    rows = [[] for _ in range(p)]
    for i in range(len(L)):
        for j in range(len(R)):
            if L["key"][i] == R["key"][j]:
                d = int(owner(np.array([L["key"][i]], np.uint64), p)[0])
                rows[d].append((int(L["key"][i]), i, j))
    outs = []
    for d in range(p):
        rows[d].sort()
        out = np.empty(len(rows[d]), out_dtype(fn))
        for t, (k, i, j) in enumerate(rows[d]):
            if fn == KEY_VALUES:
                out[t] = (k, L["val"][i], R["val"][j])
            else:
                out[t] = (L["val"][i], R["val"][j])
        outs.append(out)
    return outs


def make_side(n, universe, seed, zipf=None):
    """n pairs with keys uniform over [0, universe) (or Zipf with exponent `zipf` over 1..universe) and random values"""
    rng = np.random.RandomState(seed)
    out = np.empty(n, KV)
    if zipf is None:
        out["key"] = rng.randint(0, universe, size=n, dtype=np.uint64) if universe else 0
    else:
        w = 1.0 / np.arange(1, universe + 1) ** zipf
        out["key"] = rng.choice(universe, size=n, p=w / w.sum()).astype(np.uint64) + np.uint64(1)
    out["val"] = rng.randint(0, 1 << 62, size=n, dtype=np.uint64) * np.uint64(3) + np.uint64(1)
    return out


def split_shards(a, p):
    """a side split into p contiguous shards (Generate's even split)"""
    b = [(r * len(a) + p - 1) // p for r in range(p + 1)]
    return [a[b[r]:b[r + 1]] for r in range(p)]
