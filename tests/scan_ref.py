"""Plain restatement of PrefixSum, ExPrefixSum and ZipWithIndex (test helper, numpy only).

The input is a DIA given as one shard per worker; every worker keeps its items and gives one output per item, in order.
PrefixSum (the stock PrefixSumNode):
    S_w      = T() + x_0 + x_1 + ...            the local total, folded from the value-initialised item T() (0, +0.0, (0, 0))
    carry_0  = initial,  carry_r = initial + (S_0 + ... + S_{r-1}), the inner fold left to right
    inclusive  out_i = carry + x_0 + ... + x_i         exclusive  out_0 = carry, out_i = carry + x_0 + ... + x_{i-1}
Every fold here runs left to right one item at a time (np.*.accumulate), so the model is bit-exact for doubles too.
The sum functions act on one 8-byte value: the item (uint64_t or double), or a pair's .second with ScanSecond<F>, which takes
.first from the right-hand operand: a + b = (b.first, F(a.second, b.second)).
ZipWithIndex: item i of worker r becomes (base_r + i, x_i) (IndexFirst) or (x_i, base_r + i) (IndexSecond), base_r = the items of
the workers below r.
"""
import numpy as np

KV = np.dtype([("key", "<u8"), ("val", "<u8")])
LIMIT = (1 << 30) - 1
OP_SUM_F64, OP_SUM_U64, OP_MIN_U64, OP_MAX_U64 = 0, 1, 2, 3
OPS = {"sum_f64": OP_SUM_F64, "sum_u64": OP_SUM_U64, "min_u64": OP_MIN_U64, "max_u64": OP_MAX_U64}


def _as(op, words):
    """the 8-byte values as the op's numpy type (float64 for double sums)"""
    w = np.ascontiguousarray(words, np.uint64)
    return w.view(np.float64) if op == OP_SUM_F64 else w


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def fold_prefix(op, start, words):
    """[start + w_0, start + w_0 + w_1, ...] folded left to right, as uint64 words (start is one word)"""
    seq = np.concatenate([np.array([start], np.uint64), np.asarray(words, np.uint64)])
    v = _as(op, seq)
    with np.errstate(over="ignore", invalid="ignore"):
        if op == OP_SUM_F64 or op == OP_SUM_U64:
            acc = np.add.accumulate(v)
        elif op == OP_MIN_U64:
            acc = np.minimum.accumulate(v)
        else:
            acc = np.maximum.accumulate(v)
    return _bits(acc)[1:]


def combine(op, a, b):
    """a + b on two words"""
    return int(fold_prefix(op, a, [b])[0])


def local_total(op, words):
    """S = T() + w_0 + w_1 + ... (T() = 0 bits: 0, +0.0)"""
    if len(words) == 0:
        return 0
    return int(fold_prefix(op, 0, words)[-1])


def carries(op, totals, init_value):
    """carry_r of every worker from the workers' totals (the all-gather's records)"""
    out = [int(init_value)]
    inner = None
    for r in range(1, len(totals)):
        inner = int(totals[0]) if inner is None else combine(op, inner, int(totals[r - 1]))
        out.append(combine(op, int(init_value), inner))
    return out


def split_values(items, pair):
    """(first words or None, value words) of a shard: uint64 (n,) for 8-byte items, KV or (n, 2) uint64 for pairs"""
    a = np.ascontiguousarray(items)
    if not pair:
        return None, a.view(np.uint64).reshape(-1)
    w = a.view(np.uint64).reshape(-1, 2)
    return w[:, 0], w[:, 1]


def prefix_sum(shards, op, pair=False, initial=(0, 0), inclusive=True):
    """the p = len(shards) workers' outputs: uint64 (n,) for 8-byte items, KV for pairs.  initial = (first, value word)"""
    op = OPS.get(op, op)
    parts = [split_values(s, pair) for s in shards]
    totals = [local_total(op, v) for _, v in parts]
    last_first = [int(f[-1]) if f is not None and len(f) else 0 for f, _ in parts]
    cv = carries(op, totals, initial[1])
    outs = []
    for r, (f, v) in enumerate(parts):
        scan = fold_prefix(op, cv[r], v)
        if inclusive:
            vals = scan
        else:
            vals = np.concatenate([np.array([cv[r]], np.uint64), scan[:-1]]) if len(v) else scan
        if not pair:
            outs.append(vals.astype(np.uint64))
            continue
        carry_first = int(initial[0]) if r == 0 else last_first[r - 1]
        o = np.empty(len(v), KV)
        o["val"] = vals
        if inclusive:
            o["key"] = f
        elif len(v):
            o["key"] = np.concatenate([np.array([carry_first], np.uint64), f[:-1]])
        outs.append(o)
    return outs


def totals_of(shards, op, pair=False):
    """each worker's S as words: one word, or (S.first, S.value) for pairs"""
    op = OPS.get(op, op)
    out = []
    for s in shards:
        f, v = split_values(s, pair)
        t = local_total(op, v)
        out.append((int(f[-1]) if len(f) else 0, t) if pair else t)
    return out


def zip_with_index(shards, index_first=True):
    outs, base = [], 0
    for s in shards:
        x = np.ascontiguousarray(s).view(np.uint64).reshape(-1)
        idx = np.arange(base, base + len(x), dtype=np.uint64)
        o = np.empty(len(x), KV)
        o["key"], o["val"] = (idx, x) if index_first else (x, idx)
        outs.append(o)
        base += len(x)
    return outs


def shards_of(a, counts):
    """a split into consecutive shards of the given sizes"""
    b = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    assert b[-1] == len(a)
    return [a[b[r]:b[r + 1]] for r in range(len(counts))]


def even_counts(n, p):
    """Generate's even split"""
    b = [(r * n + p - 1) // p for r in range(p + 1)]
    return [b[r + 1] - b[r] for r in range(p)]


def splitmix64(x):
    with np.errstate(over="ignore"):
        z = np.asarray(x, np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def f64_words(x):
    return np.ascontiguousarray(np.asarray(x, np.float64)).view(np.uint64)


def pairs(first, second):
    out = np.empty(len(first), KV)
    out["key"], out["val"] = np.asarray(first, np.uint64), np.asarray(second, np.uint64)
    return out


# ---- the fixtures of tests/golden/make_golden_scan.py ------------------------------------------------------------------------
MODES = ["sum_u64", "min_u64", "max_u64", "sum_f64", "pair_max", "pair_sum_f64", "zip_first", "zip_second"]
MODE_OP = {"sum_u64": OP_SUM_U64, "min_u64": OP_MIN_U64, "max_u64": OP_MAX_U64, "sum_f64": OP_SUM_F64,
           "pair_max": OP_MAX_U64, "pair_sum_f64": OP_SUM_F64}


class Case(object):
    """one stored case: .mode, .op (None for ZipWithIndex), .pair, .inclusive, .initial, .items, .ps"""

    def __init__(self, g, name):
        self.name, self.g = name, g
        meta = [int(x) for x in g[name + "/meta"]]
        self.mode = MODES[meta[0]]
        self.op = MODE_OP.get(self.mode)
        self.inclusive, self.initial, self.pair = bool(meta[1]), (meta[2], meta[3]), bool(meta[4])
        words = g[name + "/in"]
        self.items = words.view(KV) if self.pair else words
        self.ps = sorted(int(k.split("/")[1][1:]) for k in g.files if k.startswith(name + "/p") and k.endswith("/rows"))

    def counts(self, p):
        return [int(c) for c in self.g["%s/p%d/counts" % (self.name, p)]]

    def shards(self, p):
        return shards_of(self.items, self.counts(p))

    def rows(self, p):
        """the stored outputs as (rank, first word, second word) rows; an 8-byte output has first word 0"""
        stored = self.g["%s/p%d/rows" % (self.name, p)]
        rows = np.zeros((len(stored), 3), np.uint64)
        rows[:, 0] = np.repeat(np.arange(p), self.counts(p))
        if stored.ndim == 2:
            rows[:, 1:] = stored
        else:
            rows[:, 2] = stored
        return rows

    def model(self, p):
        """the model's outputs of each worker"""
        if self.op is None:
            return zip_with_index(self.shards(p), self.mode == "zip_first")
        return prefix_sum(self.shards(p), self.op, self.pair, self.initial, self.inclusive)


def case_names(g):
    return sorted(k[:-3] for k in g.files if k.endswith("/in"))


def as_rows(outs):
    """per-worker outputs -> the fixture's (rank, first word, second word) rows"""
    rows = []
    for r, o in enumerate(outs):
        w = np.ascontiguousarray(o).view(np.uint64)
        x = np.zeros((len(o), 3), np.uint64)
        x[:, 0] = r
        if o.dtype == KV:
            x[:, 1:] = w.reshape(-1, 2)
        else:
            x[:, 2] = w
        rows.append(x)
    return np.concatenate(rows) if rows else np.zeros((0, 3), np.uint64)


def rows_equal(a, b, f64=False):
    """fixture rows equal bit for bit; with f64, two NaNs of the value word count as equal (the payload and sign of a NaN are
    not part of the contract: which operand's NaN an addition passes on is up to the compiler and the hardware)"""
    a, b = np.asarray(a, np.uint64), np.asarray(b, np.uint64)
    if a.shape != b.shape:
        return False
    eq = a == b
    if f64:
        eq[:, 2] |= np.isnan(a[:, 2].view(np.float64)) & np.isnan(b[:, 2].view(np.float64))
    return bool(eq.all())
