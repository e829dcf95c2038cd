"""Plain restatement of Merge's result and split (test helper, numpy only).

p workers hold k inputs; run (w, j) = worker w's shard of input j, listed as runs[w * k + j].  Every input is sorted by the
key descriptor across the workers.  The merged sequence is the stable sort by key of the input-major concatenation
(input 0's shards of workers 0..p-1, then input 1's, ...): the order (key, input index, global position within the input).
Worker d receives the merged ranks [ceil(d * N / p), ceil((d + 1) * N / p)).
"""
import numpy as np

import sort_ref as R


def targets(p, n):
    """t_d = ceil(d * N / p) for d = 0..p, in integer arithmetic"""
    return np.array([(d * n + p - 1) // p for d in range(p + 1)], dtype=np.uint64)


def input_major(runs, p, k):
    """the run order of the concatenation: (j, w) for j in 0..k-1, w in 0..p-1, as indices into runs"""
    return [w * k + j for j in range(k) for w in range(p)]


def concat(runs, p, k, d):
    """(items as (N, item_bytes) uint8 rows in input-major order, run index of each row, local position of each row)"""
    order = input_major(runs, p, k)
    rows = [R.rows(runs[r], d.item_bytes) for r in order]
    items = np.concatenate(rows) if rows else np.zeros((0, d.item_bytes), np.uint8)
    run_of = np.concatenate([np.full(len(x), r, np.int64) for r, x in zip(order, rows)])
    pos = np.concatenate([np.arange(len(x), dtype=np.int64) for x in rows])
    return items, run_of, pos


def merged(runs, p, k, d):
    """the whole merged sequence as (N, item_bytes) uint8 rows"""
    items, _, _ = concat(runs, p, k, d)
    return items[R.sort_order(items, d)]


def key_ids(items, d):
    """an integer per item whose order is the descriptor's key order (equal keys, equal ids)"""
    k = R.key_columns(items, d)
    if len(k) == 0:
        return np.zeros(0, np.int64)
    _, inv = np.unique(k, axis=0, return_inverse=True)
    return inv.reshape(-1).astype(np.int64)


def bounds(runs, p, k, d):
    """bounds[(w * k + j) * (p + 1) + dd] = the first position of run (w, j) that goes to worker dd, dd = 0..p"""
    items, run_of, _ = concat(runs, p, k, d)
    rank = np.empty(len(items), np.int64)
    rank[R.sort_order(items, d)] = np.arange(len(items))
    t = targets(p, len(items)).astype(np.int64)
    out = np.zeros(p * k * (p + 1), np.uint64)
    for r in range(p * k):
        rr = rank[run_of == r]
        for dd in range(p + 1):
            out[r * (p + 1) + dd] = np.count_nonzero(rr < t[dd])
    return out


def counts(runs, p, k, d):
    """(targets, less, equal) as tg_merge_plan takes them: for d = 0..p, K_d = the key of the item at merged rank t_d (none for
    t_d = N: every item counts as less), less / equal = items of each run below / equal to K_d"""
    items, run_of, _ = concat(runs, p, k, d)
    n = len(items)
    t = targets(p, n)
    ids = key_ids(items, d)
    srt = ids[R.sort_order(items, d)]
    less = np.zeros(p * k * (p + 1), np.uint64)
    equal = np.zeros(p * k * (p + 1), np.uint64)
    for dd in range(p + 1):
        kd = srt[int(t[dd])] if int(t[dd]) < n else None
        for r in range(p * k):
            x = ids[run_of == r]
            if kd is None:
                less[r * (p + 1) + dd] = len(x)
            else:
                less[r * (p + 1) + dd] = np.count_nonzero(x < kd)
                equal[r * (p + 1) + dd] = np.count_nonzero(x == kd)
    return t, less, equal


def shard(sorted_items, p, rng, shape="random"):
    """split a sorted input into p consecutive shards: "random" cut points, "even", "one" (one worker holds all), "gaps"
    (every other worker empty)"""
    n = len(sorted_items)
    if shape == "even":
        cuts = [(w * n) // p for w in range(p + 1)]
    elif shape == "one":
        w0 = int(rng.randint(0, p))
        cuts = [0] * (w0 + 1) + [n] * (p - w0)
    elif shape == "gaps":
        inner = sorted(rng.randint(0, n + 1, size=p - 1).tolist()) if p > 1 else []
        cuts = [0] + inner + [n]
        for w in range(1, p, 2):
            cuts[w + 1] = cuts[w]
        for w in range(1, p + 1):
            cuts[w] = max(cuts[w], cuts[w - 1])
        cuts[p] = n
    else:
        cuts = [0] + sorted(rng.randint(0, n + 1, size=p - 1).tolist()) + [n]
    return [sorted_items[cuts[w]:cuts[w + 1]] for w in range(p)]


def make_runs(inputs, p, rng, shape="random"):
    """runs[w * k + j] from k sorted inputs"""
    k = len(inputs)
    per = [shard(x, p, rng, shape) for x in inputs]
    return [per[j][w] for w in range(p) for j in range(k)]
