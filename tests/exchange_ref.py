"""Plain model of the collective operators' exchange (test helper, numpy only).

p workers each hold a shard (an (n_w, item_bytes) uint8 array).  Every item has an owner, the worker it is sent to:
    hash       Hash128to64(0, key) % p of a 16-byte (u64 key, value) item   ReduceByKey, InnerJoin   join_ref.owner
    mod        key % p                                                      GroupByKey               group_ref.owner_mod
    range      k < size ? k * p // size : p - 1                             ReduceToIndex,           group_ref.owner_range
                                                                            GroupToIndex
    splitters  the number of splitters (key, global index) below the item's  Sort                   sample_sort_ref.classify
               (key, global index), with the splitters the operator samples
               for the seed; records are classified by their key tuples
Window d is the concatenation over w = 0..p-1 of shard_w[owner == d], each part in input order (the layout CatStream delivers:
grouped by source worker in rank order, stable).  counts[src, dst] is the number of items shard src sends to dst, and the plan
of one worker is what every rank derives from that matrix.
"""
import numpy as np

import group_ref as G
import join_ref as J
import sample_sort_ref as S
import sort_ref as R

HASH, MOD, RANGE, SPLITTERS = 0, 1, 2, 3          # TG_ROUTE_*
ROUTES = {"hash": HASH, "mod": MOD, "range": RANGE, "splitters": SPLITTERS}
LIMIT = (1 << 30) - 1


def keys(rows):
    """the u64 key (the first 8 bytes) of 16-byte items"""
    return np.ascontiguousarray(rows[:, :8]).view("<u8").reshape(-1)


def tuples(rows, d):
    """the 16-byte key tuples a record is sorted and classified by: its key bytes zero padded to 12, then its u32 position"""
    n = len(rows)
    t = np.zeros((n, 16), np.uint8)
    t[:, :d.key_bytes] = rows[:, d.key_offset:d.key_offset + d.key_bytes]
    t[:, 12:] = np.arange(n, dtype="<u4").view(np.uint8).reshape(n, 4)
    return t


def tuple_desc(d):
    return R.Desc(16, 0, d.key_bytes, R.KEY_BYTES_BE)


def owners(route, shards, p, size=0, d=None, seed=0):
    """the owner of every item of every shard (a list of int64 arrays)"""
    if route == HASH:
        return [J.owner(keys(s), p) for s in shards]
    if route == MOD:
        return [G.owner_mod(keys(s), p) for s in shards]
    if route == RANGE:
        return [G.owner_range(keys(s), size, p) for s in shards]
    if d.item_bytes not in (8, 16):
        shards, d = [tuples(s, d) for s in shards], tuple_desc(d)
    spl = S.splitters(shards, d, p, seed)
    pre = S.prefix_of(shards, d)
    return [S.classify(s, d, pre[w] + np.arange(len(s)), spl) for w, s in enumerate(shards)]


def exchange(shards, own, p):
    """(windows, counts (p, p) [src, dst]) of shards with owners `own`"""
    ib = shards[0].shape[1]
    counts = np.zeros((p, p), np.uint64)
    wins = []
    for dst in range(p):
        parts = [s[o == dst] for s, o in zip(shards, own)]
        wins.append(np.concatenate(parts) if parts else np.zeros((0, ib), np.uint8))
    for src, o in enumerate(own):
        counts[src] = np.bincount(o, minlength=p)[:p]
    return wins, counts


def plan(counts, me):
    """what worker `me` derives from the count matrix: (send[d], recv[s], before[d], n_recv, worst) where before[d] = items of
    the ranks below `me` in worker d's window and worst = the largest receive size of any worker"""
    c = np.asarray(counts, np.uint64)
    return (c[me].copy(), c[:, me].copy(), c[:me].sum(axis=0).astype(np.uint64), int(c[:, me].sum()),
            int(c.sum(axis=0).max()) if len(c) else 0)


def too_large(shards, counts):
    """the size verdict of one exchange: a shard or a window of 2^30 items or more"""
    return any(len(s) > LIMIT for s in shards) or int(np.asarray(counts).sum(axis=0).max()) > LIMIT
