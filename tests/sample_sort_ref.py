"""Plain reference of the multi-worker Sort's classification and of ReduceToIndex's range partition (test helper, numpy only).

What p workers of Sort compute before their exchange (api/sort.hpp:151-175, :337-378, :434-535), restated from the rules:

- sample draws: worker w draws index splitmix64(seed_w + i) % n for i < min(n, tg_sample_size(n)), with
  seed_w = rng_seed * 0x9E3779B97F4A7C15 + w * 2^32 (mod 2^64); the same index may be drawn twice;
- canonical keys: sort_ref.key_columns (most significant byte first, complemented for descending descriptors);
- the global index of item i of shard w is the number of items in the shards before w plus i;
- sample order: LessSampleIndex, i.e. (key, global index);
- splitter i (1 <= i < p) is the sample at position floor(i * (S / p)) of all S samples in that order, in double arithmetic;
- classification: the bucket of an item is the number of splitters (key, global index) below its (key, global index), and each
  shard is grouped by bucket, stably;
- merge bounds (the TG_SORT_PIPELINE=merge form): in the stable sort of a shard, lower_bound of splitter j's key plus the number
  of the shard's items with that key and a global index <= the splitter's.

ReduceToIndex sends the item with index k to worker k < size ? k * p // size : p - 1 (Python integers), and worker r's index
range starts at CalculateBeginOfPart(r) = (r * size + p - 1) // p.
"""
import numpy as np

import oracle_lib as O
import sort_ref as R

SEED_MUL = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1


# sort_ref.DISTS plus "onetop": uniform keys whose most significant byte is the same everywhere, so that every splitter shares
# it with every item and the lookup table never decides alone
DISTS = R.DISTS + ("onetop",)


def make_items(d, n, dist, seed):
    if dist != "onetop":
        return R.make_items(d, n, dist, seed)
    r = R.make_items(d, n, "uniform", seed)
    r[:, d.key_offset + d.key_bytes - 1 if d.key_kind == R.KEY_UINT_LE else d.key_offset] = 0x5A
    return r


def worker_seed(rng_seed, w):
    return (rng_seed * SEED_MUL + w * (1 << 32)) & M64


def sample_count(n):
    return min(n, O.sample_size(n)) if n else 0


def sample_positions(n, seed_w):
    """the local positions worker w draws, in draw order"""
    ns = sample_count(n)
    if not ns:
        return np.zeros(0, dtype=np.int64)
    with np.errstate(over="ignore"):
        x = np.full(ns, seed_w, dtype=np.uint64) + np.arange(ns, dtype=np.uint64)
        return (R._splitmix64(x) % np.uint64(n)).astype(np.int64)


def canon(items, d):
    """(hi, lo) uint64 arrays whose lexicographic order is d's key order: the key columns padded to 16 bytes, big-endian"""
    k = R.key_columns(items, d)
    pad = np.zeros((len(k), 16), dtype=np.uint8)
    pad[:, :k.shape[1]] = k
    w = pad.view(">u8").astype(np.uint64)
    return w[:, 0].copy(), w[:, 1].copy()


def prefix_of(shards, d):
    sizes = [len(R.rows(s, d.item_bytes)) for s in shards]
    return np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)


def samples(shards, d, p, rng_seed):
    """every worker's sample: (items (S, item_bytes), hi, lo, global index), each worker's in draw order, workers in order"""
    pre = prefix_of(shards, d)
    its, gidx = [], []
    for w in range(p):
        r = R.rows(shards[w], d.item_bytes)
        pos = sample_positions(len(r), worker_seed(rng_seed, w))
        its.append(r[pos])
        gidx.append(pos + pre[w])
    its = np.concatenate(its) if its else np.zeros((0, d.item_bytes), np.uint8)
    g = np.concatenate(gidx).astype(np.uint64)
    hi, lo = canon(its, d)
    return its, hi, lo, g


def sample_order(hi, lo, g):
    """LessSampleIndex order (stable: identical draws keep draw order)"""
    return np.lexsort((g, lo, hi))


def splitters(shards, d, p, rng_seed, rank_shift=0):
    """(p - 1, item_bytes + 8) uint8: the splitter items and their global indices, packed as tg_select_splitters packs them.
    rank_shift moves every splitter by that many ranks (only to plant a wrong answer)."""
    its, hi, lo, g = samples(shards, d, p, rng_seed)
    S = len(g)
    out = np.zeros((p - 1, d.item_bytes + 8), dtype=np.uint8)
    if S == 0:
        return out
    order = sample_order(hi, lo, g)
    step = float(S) / float(p)
    for i in range(1, p):
        j = order[min(int(float(i) * step) + rank_shift, S - 1)]
        out[i - 1, :d.item_bytes] = its[j]
        out[i - 1, d.item_bytes:] = np.array([g[j]], dtype="<u8").view(np.uint8)
    return out


def unpack_splitters(spl, d):
    """(hi, lo, global index) of packed splitters"""
    hi, lo = canon(np.ascontiguousarray(spl[:, :d.item_bytes]), d)
    g = np.ascontiguousarray(spl[:, d.item_bytes:]).view("<u8").reshape(-1).astype(np.uint64)
    return hi, lo, g


def classify(items, d, gidx, spl):
    """bucket of each item: the number of splitters (key, global index) below (item key, gidx)"""
    hi, lo = canon(items, d)
    shi, slo, sg = unpack_splitters(spl, d)
    gidx = np.asarray(gidx, dtype=np.uint64)
    b = np.zeros(len(hi), dtype=np.int64)
    for j in range(len(shi)):
        below = (shi[j] < hi) | ((shi[j] == hi) & ((slo[j] < lo) | ((slo[j] == lo) & (sg[j] < gidx))))
        b += below
    return b


def group(items, buckets, p):
    """(items grouped by bucket, stably; counts per bucket)"""
    order = np.argsort(buckets, kind="stable")
    return items[order], np.bincount(buckets, minlength=p).astype(np.uint64)


def merge_bounds(shard, d, gbase, spl):
    """bnd[j] = lower_bound(stable sort of the shard, splitter j's key) + #items with that key and global index <= splitter j's"""
    r = R.rows(shard, d.item_bytes)
    hi, lo = canon(r, d)
    shi, slo, sg = unpack_splitters(spl, d)
    g = gbase + np.arange(len(r), dtype=np.uint64)
    out = np.zeros(len(shi), dtype=np.uint64)
    for j in range(len(shi)):
        less = (hi < shi[j]) | ((hi == shi[j]) & (lo < slo[j]))
        tie = (hi == shi[j]) & (lo == slo[j]) & (g <= sg[j])
        out[j] = int(less.sum()) + int(tie.sum())
    return out


def select(shards, d, p, rng_seed):
    """what tg_sort_select computes: (splitters, counts (p, p) [src, dst], grouped shards, merge bounds (p, p - 1))"""
    spl = splitters(shards, d, p, rng_seed)
    pre = prefix_of(shards, d)
    counts = np.zeros((p, p), dtype=np.uint64)
    grouped, bounds = [], np.zeros((p, p - 1), dtype=np.uint64)
    for w in range(p):
        r = R.rows(shards[w], d.item_bytes)
        b = classify(r, d, pre[w] + np.arange(len(r)), spl)
        gr, counts[w] = group(r, b, p)
        grouped.append(gr)
        bounds[w] = merge_bounds(r, d, np.uint64(pre[w]), spl)
    return spl, counts, grouped, bounds


def top_byte(items, d):
    """the most significant byte of the canonical key (canon_top_byte): the byte the splitter lookup table is indexed by"""
    return R.key_columns(items, d)[:, 0].astype(np.int64)


def lut(spl, d):
    """SplitterDigit's table: lo[b] = #splitters with top byte < b, hi[b] = #splitters with top byte <= b"""
    t = top_byte(np.ascontiguousarray(spl[:, :d.item_bytes]), d)
    b = np.arange(256)
    return (t[None, :] < b[:, None]).sum(axis=1), (t[None, :] <= b[:, None]).sum(axis=1)


def classify_lut(items, d, gidx, spl, table=None):
    """SplitterDigit's classification: the table's bucket range by the top byte, the binary search only where it holds a
    splitter (table: a (lo, hi) pair to use instead of lut(spl, d))"""
    lo_t, hi_t = table if table is not None else lut(spl, d)
    tb = top_byte(items, d)
    full = classify(items, d, gidx, spl)
    lo, hi = lo_t[tb], hi_t[tb]
    # the search over splitters [lo, hi) returns lo + #splitters of that range below the item
    return np.where(lo == hi, lo, np.clip(full, lo, hi))


# ---- ReduceToIndex ------------------------------------------------------------------------------------------------------
def begin_of_part(r, size, p):
    return (r * size + p - 1) // p


def range_dest(keys, size, p):
    return np.array([k * p // size if k < size else p - 1 for k in (int(x) for x in keys)], dtype=np.int64)


def range_partition(items, size, p):
    """(items grouped by destination, stably; counts) for 16-byte (u64 index, value) items"""
    r = R.rows(items, 16)
    k = np.ascontiguousarray(r[:, :8]).view("<u8").reshape(-1)
    return group(r, range_dest(k, size, p), p)
