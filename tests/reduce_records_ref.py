"""Plain restatement of ReduceByKey on records (test helper, numpy only).

A DIA of fixed-size records is held here as a 2-D uint8 array (one row per record, `s` bytes), given as one shard per worker; its
global order is the concatenation of the shards.  The key of a record is the unsigned little-endian integer of `key_bytes` (1..8)
bytes at byte offset `key_offset`, zero-extended.  The reduce function is a list of field runs (offset, count, op): `count`
consecutive 8-byte little-endian fields from byte `offset`, each folded with op (a TG_OP_* code, reduce_ref.OPS).
One output record per distinct key: every run field holds the fold of the group's values, every other byte is the byte of the
group's first record in global order.  Worker Hash128to64(0, key) % p owns a key; its records come out in ascending key order.

The folds here are the left folds in input order.  Integer ops are exact, so is a double sum of integer-valued doubles, and
MIN/MAX_F64 pick the earliest value that is numerically the min/max of the group's numbers (-0.0 == +0.0), or, where every value
is a NaN, the first NaN that is not the canonical 0x7ff8000000000000 (that one if there is no other): the outcome of the
library's order-preserving combine under any bracketing.  A double sum of other values is checked against reduce_ref's contract.
"""
import numpy as np

import reduce_ref
from join_records_ref import keys_of, owner

CANON_NAN = np.uint64(0x7FF8000000000000)


def fields(rec, off, cnt):
    """the cnt 8-byte fields from byte off of every record: (n, cnt) uint64"""
    return np.ascontiguousarray(rec[:, off:off + 8 * cnt]).view("<u8").reshape(len(rec), cnt).astype(np.uint64)


def groups(rec, key):
    """(order, starts): the records' stable order by key, and the first index (in that order) of each group"""
    k = keys_of(rec, *key)
    order = np.argsort(k, kind="stable")
    ks = k[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]]) if len(ks) else np.zeros(0, np.int64)
    return order, starts


def _fold_minmax_f64(v, starts, op):
    x = v.view(np.float64)
    nan = np.isnan(x)
    gid = np.repeat(np.arange(len(starts)), np.diff(np.r_[starts, len(v)]))
    if op == 4:
        want = np.minimum.reduceat(np.where(nan, np.inf, x), starts)
    else:
        want = np.maximum.reduceat(np.where(nan, -np.inf, x), starts)
    idx = np.arange(len(v))
    big = len(v)
    hit = ~nan & (x == want[gid])
    first_num = np.minimum.reduceat(np.where(hit, idx, big), starts)
    first_nan = np.minimum.reduceat(np.where(nan & (v != CANON_NAN), idx, big), starts)
    first_any = starts
    pick = np.where(first_num < big, first_num, np.where(first_nan < big, first_nan, first_any))
    return v[pick]


def fold(v, starts, op):
    """the fold of each group's values (v: uint64 in group order, groups starting at `starts`)"""
    if len(starts) == 0:
        return np.zeros(0, np.uint64)
    if op == 0:
        with np.errstate(invalid="ignore", over="ignore"):
            return np.add.reduceat(v.view(np.float64), starts).view(np.uint64)
    if op == 1:
        return np.add.reduceat(v, starts)
    if op == 2:
        return np.minimum.reduceat(v, starts)
    if op == 3:
        return np.maximum.reduceat(v, starts)
    if op in (4, 5):
        return _fold_minmax_f64(v, starts, op)
    raise ValueError(op)


def reduce_local(rec, key, runs):
    """one worker's result from its records in global order: (m, s) uint8, ascending key"""
    order, starts = groups(rec, key)
    out = rec[order[starts]].copy()
    srt = rec[order]
    for off, cnt, op in runs:
        v = fields(srt, off, cnt)
        r = np.stack([fold(v[:, j], starts, op) for j in range(cnt)], axis=1) if len(starts) else np.zeros((0, cnt), np.uint64)
        out[:, off:off + 8 * cnt] = np.ascontiguousarray(r.astype("<u8")).view(np.uint8).reshape(len(starts), 8 * cnt)
    return out


def exchange(shards, key, p):
    """each worker's received records: the records it owns, grouped by source worker in rank order, each group in input order"""
    s = shards[0].shape[1]
    allv = np.concatenate(shards) if len(shards) else np.zeros((0, s), np.uint8)
    own = owner(keys_of(allv, *key), p)
    return [allv[own == d] for d in range(p)]


def reduce(shards, key, runs):
    """every worker's result for p = len(shards) workers: the pre phase on each shard, the exchange, the reduce of each window"""
    p = len(shards)
    pre = [reduce_local(sh, key, runs) for sh in shards]
    return [reduce_local(w, key, runs) for w in exchange(pre, key, p)]


def check(rec, out, key, runs, sorted_keys=True):
    """assert that `out` is a result of reducing the records `rec` (in global order) under the contract: the keys are the
    distinct keys (ascending if sorted_keys), every byte outside the runs is the first record's, every run field obeys
    reduce_ref.check for its op"""
    order, starts = groups(rec, key)
    want = rec[order[starts]]
    ok = keys_of(out, *key)
    if not sorted_keys:
        o = np.argsort(ok, kind="stable")
        out, ok = out[o], ok[o]
    assert np.array_equal(ok, keys_of(want, *key)), "keys differ: %d out, %d distinct in" % (len(ok), len(want))
    mask = np.ones(rec.shape[1], bool)
    for off, cnt, _ in runs:
        mask[off:off + 8 * cnt] = False
    assert np.array_equal(out[:, mask], want[:, mask]), "bytes outside the runs differ from the first record's"
    k = keys_of(rec, *key)
    for off, cnt, op in runs:
        vi, vo = fields(rec, off, cnt), fields(out, off, cnt)
        for j in range(cnt):
            inp = np.zeros(len(rec), reduce_ref.O.KV)
            inp["key"], inp["val"] = k, vi[:, j]
            o = np.zeros(len(out), reduce_ref.O.KV)
            o["key"], o["val"] = ok, vo[:, j]
            reduce_ref.check(inp, o, op)


def make(n, s, key, keys, seed):
    """n random records of s bytes with the given keys in the key field"""
    from join_records_ref import make_records, set_keys
    return set_keys(make_records(n, s, seed), key[0], key[1], keys)


def set_fields(rec, off, cnt, vals):
    """write (n, cnt) uint64 values into a run's fields"""
    rec[:, off:off + 8 * cnt] = np.ascontiguousarray(np.asarray(vals, np.uint64).astype("<u8")).view(np.uint8).reshape(len(rec), 8 * cnt)
    return rec


def values(op, n, cnt, seed, exact=True):
    """(n, cnt) values for a run with op: integer-valued doubles (exact sums) or wide doubles for the double ops, full-range
    integers for the integer ops"""
    mix = "u64" if op in (1, 2, 3) else ("f64_exact" if exact else "f64_wide")
    rng = np.random.default_rng(seed)
    dummy = rng.integers(0, 1 << 62, size=n, dtype=np.uint64)
    return np.stack([reduce_ref.gen_values(mix, dummy, seed * 31 + j) for j in range(cnt)], axis=1) if n else np.zeros((0, cnt), np.uint64)
