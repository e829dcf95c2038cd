"""Plain restatement of InnerJoin on records (test helper, numpy only).

Each side is a DIA of fixed-size records, held here as a 2-D uint8 array (one row per record, `s` bytes), given as one shard per
worker; a side's global order is the concatenation of its shards.  The key of a record is the unsigned little-endian integer of
`key_bytes` (1..8) bytes at byte offset `key_offset`, zero-extended to uint64.  Worker Hash128to64(0, key) % p owns a key and
receives the records of both sides with that key, grouped by source worker in rank order, each group in the sender's order (so:
in global order).  Its result holds one record per matching (l, r), the left record's bytes then the right record's, ordered by
(key, left global position, right global position).  A worker's side (before or after the exchange) and a worker's output are
limited to 2^30 - 1 items.
"""
import numpy as np

from join_ref import LIMIT, owner  # noqa: F401  (the placement and the limit are the pair join's)


def splitmix64(x):
    """SplitMix64's output for state x (wrapping uint64 arithmetic)"""
    with np.errstate(over="ignore"):
        z = np.asarray(x, np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def make_records(n, s, seed, first=0):
    """n records of s bytes (s % 4 == 0): word w of global record g is the low 32 bits of splitmix64(((g * 131 + w) << 20) ^ seed)"""
    w = s // 4
    g = np.arange(first, first + n, dtype=np.uint64)[:, None]
    idx = g * np.uint64(131) + np.arange(w, dtype=np.uint64)[None, :]
    with np.errstate(over="ignore"):
        words = splitmix64((idx << np.uint64(20)) ^ np.uint64(seed)).astype(np.uint32)
    return np.ascontiguousarray(words).view(np.uint8).reshape(n, s)


def set_keys(rec, key_offset, key_bytes, keys):
    """write keys (uint64, < 2^(8 key_bytes)) into the key field of every record, little-endian"""
    kb = np.asarray(keys, np.uint64).astype("<u8").view(np.uint8).reshape(-1, 8)
    rec[:, key_offset:key_offset + key_bytes] = kb[:, :key_bytes]
    return rec


UNIFORM, ZIPF, ONE_KEY = 0, 1, 2


def side_from_params(side):
    """the records of one side of a fixture (tests/golden/make_golden_join_records.py): side = (item bytes, key offset, key bytes,
    n, seed, draw, universe, skew x 100), keys uniform over the universe, Zipf over it, or one key"""
    s, off, nb, n, seed, draw, universe, skew = (int(x) for x in side)
    if draw == UNIFORM:
        keys = np.random.default_rng(seed).integers(0, universe, n, dtype=np.uint64)
    elif draw == ZIPF:
        keys = zipf_keys(n, universe, skew / 100.0, seed)
    else:
        keys = np.full(n, 0xABCDE, np.uint64)
    return set_keys(make_records(n, s, seed), off, nb, keys)


def keys_of(rec, key_offset, key_bytes):
    """the key of every record, zero-extended to uint64"""
    b = np.zeros((len(rec), 8), np.uint8)
    b[:, :key_bytes] = rec[:, key_offset:key_offset + key_bytes]
    return b.view("<u8").reshape(-1).astype(np.uint64)


def zipf_keys(n, universe, skew, seed):
    """n keys from 0..universe-1, P(k) proportional to 1 / (k + 1)^skew"""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, universe + 1, dtype=np.float64) ** skew
    cdf = np.cumsum(w)
    return np.minimum(np.searchsorted(cdf, rng.random(n) * cdf[-1]), universe - 1).astype(np.uint64)


def join_indices(kl, kr):
    """(li, ri): for every matching pair in the result order, the left and right record index"""
    ol = np.argsort(kl, kind="stable")
    orr = np.argsort(kr, kind="stable")
    KL, KR = kl[ol], kr[orr]
    lo = np.searchsorted(KR, KL, "left").astype(np.int64)
    cnt = np.searchsorted(KR, KL, "right").astype(np.int64) - lo
    m = int(cnt.sum())
    li = np.repeat(np.arange(len(KL), dtype=np.int64), cnt)
    off = np.cumsum(cnt) - cnt
    ri = lo[li] + (np.arange(m, dtype=np.int64) - off[li])
    return ol[li], orr[ri]


def join_local(left, right, lk, rk):
    """one worker's result (m x (sl + sr) uint8) from its records of both sides, each in global order; lk, rk = (offset, bytes)"""
    li, ri = join_indices(keys_of(left, *lk), keys_of(right, *rk))
    return np.concatenate([left[li], right[ri]], axis=1) if len(li) else np.zeros((0, left.shape[1] + right.shape[1]), np.uint8)


def exchange(shards, key, p):
    """each worker's received records (the window contents of the simulated exchange): the records it owns, grouped by source
    worker in rank order, each group in input order"""
    allv = np.concatenate(shards) if len(shards) else np.zeros((0, 4), np.uint8)
    own = owner(keys_of(allv, *key), p)
    return [allv[own == d] for d in range(p)]


def exchange_counts(shards, key, p):
    """out_counts[src * p + dst] of the simulated exchange"""
    out = np.zeros(p * p, np.uint64)
    for w, sh in enumerate(shards):
        own = owner(keys_of(sh, *key), p)
        out[w * p:(w + 1) * p] = np.bincount(own, minlength=p)
    return out


def join(lefts, rights, lk, rk):
    """every worker's result for p = len(lefts) workers"""
    p = len(lefts)
    el, er = exchange(lefts, lk, p), exchange(rights, rk, p)
    return [join_local(el[d], er[d], lk, rk) for d in range(p)]


def output_count(kl, kr):
    """the number of matching pairs of two key arrays"""
    ul, cl = np.unique(kl, return_counts=True)
    ur, cr = np.unique(kr, return_counts=True)
    _, il, ir = np.intersect1d(ul, ur, assume_unique=True, return_indices=True)
    return int((cl[il].astype(np.int64) * cr[ir].astype(np.int64)).sum())


def too_large(lefts, rights, lk, rk):
    """the size verdict on p = len(lefts) workers: a side over the limit before or after the exchange, or an output over it"""
    p = len(lefts)
    if any(len(x) > LIMIT for x in lefts + rights):
        return True
    el, er = exchange(lefts, lk, p), exchange(rights, rk, p)
    if any(len(x) > LIMIT for x in el + er):
        return True
    return any(output_count(keys_of(el[d], *lk), keys_of(er[d], *rk)) > LIMIT for d in range(p))


def multiset(rows):
    """rows (m x s uint8) as a canonical sorted multiset, for comparisons with the stock join's unordered results"""
    if len(rows) == 0:
        return rows
    v = np.ascontiguousarray(rows).view(np.dtype((np.void, rows.shape[1]))).reshape(-1)
    return np.sort(v).view(np.uint8).reshape(len(rows), rows.shape[1])


def digest(rows):
    """an order-independent digest of rows: (count, sum and xor of splitmix64 of each row's 64-bit fold)"""
    if len(rows) == 0:
        return (0, 0, 0)
    s = rows.shape[1]
    w = np.ascontiguousarray(rows).view("<u4").reshape(len(rows), s // 4).astype(np.uint64)
    h = np.zeros(len(rows), np.uint64)
    with np.errstate(over="ignore"):
        for j in range(w.shape[1]):
            h = splitmix64(h ^ (w[:, j] + (np.uint64(j) << np.uint64(32))))
        return (len(rows), int(h.sum(dtype=np.uint64)), int(np.bitwise_xor.reduce(h)))


def golden_cases(g):
    """the fixtures of reference_outputs_join_records.npz (loaded as g): (name, left, right, left key, right key, {p: stored output
    multiset: sorted rows, or a digest as 3 uint64})"""
    for name in sorted({k.split("/")[0] for k in g.files}):
        prm = g[name + "/params"]
        ls, rs = prm[:8], prm[8:]
        outs = {int(k.rsplit("_p", 1)[1]): g[k] for k in g.files if k.startswith(name + "/out_p")}
        yield name, side_from_params(ls), side_from_params(rs), (int(ls[1]), int(ls[2])), (int(rs[1]), int(rs[2])), outs


def matches_golden(rows, stored):
    """the rows (any order) have the stored multiset"""
    if stored.dtype == np.uint8:
        return rows.shape[0] == stored.shape[0] and np.array_equal(multiset(rows), stored.reshape(rows.shape))
    return tuple(int(x) for x in stored) == digest(rows)
