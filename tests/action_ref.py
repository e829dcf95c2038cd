"""Plain restatement of the Sum, Min, Max and AllReduce actions (test helper, numpy only).

The input is a DIA given as one shard per worker.  The stock AllReduceNode (api/all_reduce.hpp:27-85):
    S_r = ((x_0 + x_1) + x_2) ...       the worker's items folded left to right from its first item, not from an identity
    worker 0 with an initial value folds every item into it: S_0 = ((initial + x_0) + x_1) ...
    a worker with no items contributes T() (0, +0.0, (0, 0)), or the initial value if there is one, on every worker (the
    node's value starts as the initial value everywhere; a worker other than 0 replaces it with its first item)
    result = ((S_0 + S_1) + S_2) ... + S_{p-1}, the same on every worker
Every fold here runs left to right one item at a time, so the model is bit-exact for doubles too.  The functions act on one
8-byte value: the item (uint64_t or double), or a pair's .second with ScanSecond<F>, which takes .first from the right-hand
operand: a + b = (b.first, F(a.second, b.second)).  Min / Max are std::min / std::max: min(a, b) = b < a ? b : a,
max(a, b) = a < b ? b : a (a NaN first operand sticks, a NaN second operand is skipped, of equal values the left one stays).
"""
import numpy as np

import scan_ref as S

OP_SUM_F64, OP_SUM_U64, OP_MIN_U64, OP_MAX_U64, OP_MIN_F64, OP_MAX_F64 = range(6)
F64_OPS = (OP_SUM_F64, OP_MIN_F64, OP_MAX_F64)
OPS = {"u64_sum": OP_SUM_U64, "u64_min": OP_MIN_U64, "u64_max": OP_MAX_U64,
       "f64_sum": OP_SUM_F64, "f64_min": OP_MIN_F64, "f64_max": OP_MAX_F64}
MODES = ["u64_sum", "u64_min", "u64_max", "f64_sum", "f64_min", "f64_max",
         "pair_u64_sum", "pair_u64_min", "pair_u64_max", "pair_f64_sum", "pair_f64_min", "pair_f64_max"]
KV = S.KV
M64 = (1 << 64) - 1


def _f(w):
    return float(np.array([w], np.uint64).view(np.float64)[0])


def _w(x):
    return int(np.array([x], np.float64).view(np.uint64)[0])


def fn(op, a, b):
    """a + b on two value words, the stock function"""
    if op == OP_SUM_U64:
        return (a + b) & M64
    if op == OP_MIN_U64:
        return b if b < a else a
    if op == OP_MAX_U64:
        return b if a < b else a
    x, y = _f(a), _f(b)
    if op == OP_SUM_F64:
        with np.errstate(over="ignore", invalid="ignore"):
            return _w(np.float64(x) + np.float64(y))
    if op == OP_MIN_F64:
        return b if y < x else a
    return b if x < y else a                    # OP_MAX_F64


def fold(op, start, words):
    """start + w_0 + w_1 + ... left to right (start is a word)"""
    v = int(start)
    if op == OP_SUM_F64:
        # np.add.accumulate folds left to right one item at a time: the same roundings as the loop, faster
        seq = np.concatenate([np.array([v], np.uint64), np.asarray(words, np.uint64)]).view(np.float64)
        with np.errstate(over="ignore", invalid="ignore"):
            return int(np.add.accumulate(seq)[-1:].view(np.uint64)[0])
    if op == OP_SUM_U64:
        return (v + int(np.sum(np.asarray(words, np.uint64), dtype=np.uint64))) & M64
    w = np.asarray(words, np.uint64)
    if op in (OP_MIN_U64, OP_MAX_U64) and len(w):
        return fn(op, v, int(w.min() if op == OP_MIN_U64 else w.max()))
    # Min / Max on doubles: the NaN words are skipped, and of the equal extremes the earliest stays (the sign of a zero)
    x = w.view(np.float64)
    ok = ~np.isnan(x)
    if not ok.any():
        return v
    m = x[ok].min() if op == OP_MIN_F64 else x[ok].max()
    return fn(op, v, int(w[np.flatnonzero(ok & (x == m))[0]]))


def worker_values(shards, op, pair=False, initial=None):
    """each worker's S_r as (first, value) words; initial = (first, value) words or None"""
    out = []
    for r, s in enumerate(shards):
        f, v = S.split_values(s, pair)
        take = initial is not None and r == 0
        if len(v) == 0:
            # the node's value starts as the initial value on EVERY worker; only worker 0 folds items into it
            out.append((int(initial[0]), int(initial[1])) if initial is not None else (0, 0))
            continue
        first = int(f[-1]) if pair else 0
        out.append((first, fold(op, initial[1], v) if take else fold(op, int(v[0]), v[1:])))
    return out


def all_reduce(shards, op, pair=False, initial=None):
    """the result every worker gets, as (first, value) words (first = 0 for 8-byte items)"""
    op = OPS.get(op, op)
    vals = worker_values(shards, op, pair, initial)
    v = vals[0][1]
    for _, s in vals[1:]:
        v = fn(op, v, s)
    return vals[-1][0] if pair else 0, v


def mode_op(mode):
    """(op, pair) of a fixture mode"""
    pair = mode.startswith("pair_")
    return OPS[mode[5:] if pair else mode], pair


# ---- the fixtures of tests/golden/make_golden_action.py ----------------------------------------------------------------------
# The file holds a few arrays (C cases, I distinct inputs, W = len(WORKERS)):
#   names (C,)          case names
#   meta (C, 5)         [mode index into MODES, with initial, init_first, init_second, input index]
#   in_start (I + 1,)   words[in_start[j]:in_start[j + 1]] is input j (uint64 words; pairs as (first, second) words)
#   words               the inputs, concatenated
#   counts (C, W, 8)    the items of each worker at p = WORKERS[k] (the first p entries)
#   results (C, W, 2)   the result every worker got at p = WORKERS[k]: (first word, second word); 8-byte items have first word 0
WORKERS = (1, 2, 3, 4, 8)


class Golden(object):
    """the fixture file loaded once (np.load decompresses an array on every access)"""

    def __init__(self, path):
        g = np.load(path)
        self.names = [str(x) for x in g["names"]]
        self.index = {n: i for i, n in enumerate(self.names)}
        self.meta, self.in_start, self.words = g["meta"], g["in_start"], g["words"]
        self.counts, self.results = g["counts"], g["results"]


class Case(object):
    """one stored case: .mode, .op, .pair, .initial ((first, value) words or None), .items, .ps"""

    def __init__(self, g, name):
        self.name, self.g = name, g
        self.i = g.index[name]
        meta = [int(x) for x in g.meta[self.i]]
        self.mode = MODES[meta[0]]
        self.op, self.pair = mode_op(self.mode)
        self.initial = (meta[2], meta[3]) if meta[1] else None
        words = g.words[g.in_start[meta[4]]:g.in_start[meta[4] + 1]]
        self.items = words.view(KV) if self.pair else words
        self.ps = list(WORKERS)

    def counts(self, p):
        return [int(c) for c in self.g.counts[self.i, WORKERS.index(p), :p]]

    def shards(self, p):
        return S.shards_of(self.items, self.counts(p))

    def result(self, p):
        """the stock result as (first, value) words"""
        r = self.g.results[self.i, WORKERS.index(p)]
        return int(r[0]), int(r[1])

    def model(self, p):
        return all_reduce(self.shards(p), self.op, self.pair, self.initial)


def case_names(g):
    return sorted(g.names)
