"""Plain reference of the reduce operators (tg_hash_aggregate, tg_reduce_by_key, tg_reduce_to_index), the counterpart of
sort_ref.py: a per-key check of the result contract, value generators with the IEEE specials, keys with chosen bit fields
of Hash128to64(0, key), and the aggregation path a call took, read from outside the library.

The reference's own result depends on the order in which a key's records arrive (floating-point sums, ties of ±0, NaN), and
with several workers that order is not fixed.  So `check` accepts what every arrival order of the reference can give:

    SUM_U64, MIN_U64, MAX_U64   exact (sums mod 2^64)
    SUM_F64   NaN if a value is NaN or both infinities occur, else the infinity that occurs; otherwise within the error bound
              of recursive summation in some order of the fsum of the values, -0.0 exactly when every value is -0.0, and
              bit-exact where the values make every order exact (exact=True) or the key has one record (a lone NaN only
              needs to stay a NaN)
    MIN_F64, MAX_F64   one of the key's own bit patterns; numerically the min / max of its non-NaN values, a NaN if it has
              none (the outcome of the reference when a number arrives first)
    FIRST     one of the key's own bit patterns
and every distinct input key exactly once, the key 0 included.
"""
import math

import numpy as np

import oracle_lib as O

OPS = ["sum_f64", "sum_u64", "min_u64", "max_u64", "min_f64", "max_f64", "first"]     # index = TG_OP_* code
U = 2.0 ** -53                                    # unit roundoff of binary64
M64 = (1 << 64) - 1
HASH_K = 0x9DDFEA08EB382D69
HASH_K_INV = pow(HASH_K, -1, 1 << 64)

NAN_PAYLOADS = [0x7FF8000000000000, 0x7FF0000000000001, 0xFFF8000000000000, 0x7FFFFFFFFFFFFFFF, 0xFFF0000000000123]


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


# ---- the contract ---------------------------------------------------------------------------------------------------

def _groups(inp):
    """input sorted by key: (distinct keys, group starts, group sizes, values in key order)"""
    order = np.argsort(inp["key"])
    k = inp["key"][order]
    starts = np.flatnonzero(np.r_[True, k[1:] != k[:-1]]) if len(k) else np.zeros(0, np.int64)
    sizes = np.diff(np.r_[starts, len(k)])
    return k[starts], starts, sizes, inp["val"][order]


def _fail(msg, key, gv, vals, op):
    vals = vals[:24]
    shown = ", ".join("%s(%016x)" % (repr(float(v)) if op.endswith("f64") else int(u), int(u))
                      for v, u in zip(vals.view(np.float64), vals))
    got = "%s (%016x)" % (repr(float(np.uint64(gv).view(np.float64))) if op.endswith("f64") else int(gv), int(gv))
    raise AssertionError("%s: key %d (0x%016x): got %s; values [%s]" % (msg, int(key), int(key), got, shown))


def _member(got, vals, starts, sizes):
    """mask over the keys: the output value is one of the key's own values (bit patterns)"""
    return np.logical_or.reduceat(vals == np.repeat(got, sizes), starts)


def check(inp, out, op, exact=False):
    """assert that `out` (the items tg_hash_aggregate / tg_reduce_by_key returned, any order) is a result of reducing
    `inp` with `op` (a TG_OP_* code or a name of OPS) under the contract of the module docstring"""
    op = OPS[op] if isinstance(op, int) else op
    inp = np.ascontiguousarray(inp, dtype=O.KV)
    out = np.ascontiguousarray(out, dtype=O.KV)
    out = out[np.argsort(out["key"])]
    keys, starts, sizes, vals = _groups(inp)
    ok = out["key"]
    if len(ok) != len(keys) or not np.array_equal(ok, keys):
        dup = ok[1:][ok[1:] == ok[:-1]]
        missing = np.setdiff1d(keys, ok)
        extra = np.setdiff1d(ok, keys)
        raise AssertionError("%s: %d keys out, %d distinct keys in; duplicated %s, missing %s, not in the input %s" % (
            op, len(ok), len(keys), dup[:5], missing[:5], extra[:5]))
    if len(keys) == 0:
        return
    got = out["val"]
    ends = starts + sizes

    def first_bad(bad, msg):
        if np.any(bad):
            i = int(np.flatnonzero(bad)[0])
            _fail("%s %s" % (op, msg), keys[i], got[i], vals[starts[i]:ends[i]], op)

    if op == "sum_u64":
        first_bad(got != np.add.reduceat(vals, starts), "differs from the sum mod 2^64")
    elif op == "min_u64":
        first_bad(got != np.minimum.reduceat(vals, starts), "differs from the minimum")
    elif op == "max_u64":
        first_bad(got != np.maximum.reduceat(vals, starts), "differs from the maximum")
    elif op == "first":
        first_bad(~_member(got, vals, starts, sizes), "is not one of the key's values")
    elif op in ("min_f64", "max_f64"):
        x = vals.view(np.float64)
        g = got.view(np.float64)
        first_bad(~_member(got, vals, starts, sizes), "is not one of the key's values")
        nan = np.isnan(x)
        all_nan = np.logical_and.reduceat(nan, starts)
        if op == "min_f64":            # (not np.fmin: it lets a signalling NaN through)
            want = np.minimum.reduceat(np.where(nan, np.inf, x), starts)
        else:
            want = np.maximum.reduceat(np.where(nan, -np.inf, x), starts)
        first_bad(all_nan != np.isnan(g), "NaN where a number is (or the reverse)")
        first_bad(~all_nan & (want != g), "differs numerically from the min/max of the numbers")
    elif op == "sum_f64":
        _check_sum_f64(keys, starts, sizes, vals, got, exact, first_bad)
    else:
        raise ValueError(op)


def _check_sum_f64(keys, starts, sizes, vals, got, exact, first_bad):
    x = vals.view(np.float64)
    g = got.view(np.float64)
    nan = np.logical_or.reduceat(np.isnan(x), starts)
    pinf = np.logical_or.reduceat(x == np.inf, starts)
    ninf = np.logical_or.reduceat(x == -np.inf, starts)
    want_nan = nan | (pinf & ninf)
    first_bad(want_nan != np.isnan(g), "NaN where there must be none (or the reverse)")
    first_bad(~want_nan & pinf & (g != np.inf), "is not +inf")
    first_bad(~want_nan & ninf & (g != -np.inf), "is not -inf")
    fin = ~(want_nan | pinf | ninf)
    all_neg0 = np.logical_and.reduceat(vals == np.uint64(0x8000000000000000), starts)
    first_bad(fin & all_neg0 & (got != np.uint64(0x8000000000000000)), "is not -0.0 (every value is -0.0)")
    first_bad(fin & ~all_neg0 & (got == np.uint64(0x8000000000000000)), "is -0.0 (not every value is -0.0)")
    first_bad(fin & (sizes == 1) & (got != vals[starts]), "differs from the key's one value")
    with np.errstate(invalid="ignore", over="ignore"):
        seq = np.add.reduceat(np.where(np.isfinite(x), x, 0.0), starts)     # one order of recursive summation
    if exact:
        first_bad(fin & (got != _bits(seq)), "differs from the exact sum")
        return
    # where the result is not the left-to-right sum: within the bound of recursive summation in any order, gamma_(m-1)
    # * sum|x| (the first-order (m-1) * 2^-53 * sum|x|), of the correctly rounded fsum (its own half ulp added)
    cand = np.flatnonzero(fin & (got != _bits(seq)))
    bad = np.zeros(len(keys), dtype=bool)
    for i in cand:
        xs = x[starts[i]:starts[i] + sizes[i]]
        m = len(xs)
        ref = math.fsum(xs)
        gm = (m - 1) * U / (1 - (m - 1) * U)
        tol = gm * math.fsum(np.abs(xs)) + U * abs(ref)
        bad[i] = not abs(float(g[i]) - ref) <= tol
    first_bad(bad, "is not within (m-1) 2^-53 sum|x| of the exact sum")


def to_index_check(inp, out, size, op, neutral=(0, 0), exact=False):
    """the dense ReduceToIndex result: item i is the reduction of the records with index i (key field i), or the neutral
    item, key field as given, where no record has index i"""
    inp = np.ascontiguousarray(inp, dtype=O.KV)
    assert len(out) == size, (len(out), size)
    idx = np.unique(inp["key"])
    assert len(idx) == 0 or int(idx[-1]) < size
    present = np.zeros(size, dtype=bool)
    present[idx.astype(np.int64)] = True
    neu = np.zeros(1, dtype=O.KV)
    neu["key"], neu["val"] = neutral
    absent = ~present
    bad = absent & ((out["key"] != neu["key"][0]) | (out["val"] != neu["val"][0]))
    assert not np.any(bad), "index %d has no record but holds %r" % (int(np.flatnonzero(bad)[0]), out[bad][0])
    sub = out[present]
    assert np.array_equal(sub["key"], idx), "key fields of the reduced indices differ from their indices"
    check(inp, sub, op, exact=exact)


# ---- values ---------------------------------------------------------------------------------------------------------

VALUE_MIXES = {                    # op -> the value mixes the tests run it with
    "sum_f64": ["f64_exact", "f64_wide", "f64_special"], "sum_u64": ["u64"], "min_u64": ["u64"], "max_u64": ["u64"],
    "min_f64": ["f64_exact", "f64_wide", "f64_special"], "max_f64": ["f64_exact", "f64_wide", "f64_special"],
    "first": ["u64", "f64_special"]}


def f64_specials(n):
    """the special values of the f64 mixes; DBL_MAX / (2n) keeps every sum of n of them finite in any order"""
    big = np.finfo(np.float64).max / (2 * max(n, 1))
    nan = NAN_PAYLOADS
    return np.array([0x8000000000000000, nan[0], *_bits([np.inf, 0.0]), nan[2], *_bits([-np.inf, 5e-324]), nan[1],
                     *_bits([big, -5e-324]), nan[3], *_bits([-big]), nan[4]], dtype=np.uint64)


def gen_values(mix, keys, seed):
    """values for records with these keys.  u64: full-range values (SUM_U64 wraps), 0, 2^64-1 and values near 2^63.
    f64_exact: integers of magnitude < 2^20 and -0.0 (every sum exact in any order at n < 2^33).  f64_wide: mixed signs,
    exponents from -80 to 80.  f64_special: f64_wide with ±0, ±inf, NaNs, the smallest subnormal and huge values mixed in.
    In every mix some keys carry only one special value each (a key per special, while there are keys)."""
    n = len(keys)
    rng = np.random.default_rng(seed)
    if mix == "u64":
        v = rng.integers(0, M64, size=n, dtype=np.uint64, endpoint=True)
        r = rng.random(n)
        v[r < 0.05] = 0
        v[(r >= 0.05) & (r < 0.10)] = np.uint64(M64)
        mid = (r >= 0.10) & (r < 0.15)
        v[mid] = np.uint64((1 << 63) - 3) + rng.integers(0, 7, size=int(mid.sum()), dtype=np.uint64)
        specials = np.array([0, M64, 1 << 63], dtype=np.uint64)
    elif mix == "f64_exact":
        v = _bits(rng.integers(-(1 << 20), 1 << 20, size=n).astype(np.float64))
        v[rng.random(n) < 0.05] = np.uint64(0x8000000000000000)
        specials = _bits([-0.0, 0.0, 1048575.0])
    else:
        v = _bits(np.ldexp(rng.random(n) - 0.5, rng.integers(-80, 81, size=n)))
        specials = f64_specials(n)
        if mix == "f64_special":
            s = rng.random(n) < 0.08
            v[s] = specials[rng.integers(0, len(specials), size=int(s.sum()))]
    # keys that carry one special only (twice each, while a key without one remains)
    if n:
        pick = np.unique(keys[rng.integers(0, n, size=min(n, 4 * len(specials)))])[:2 * len(specials)]
        pick = rng.permutation(pick)
        masks = [keys == k for k in pick]
        while masks and np.all(np.logical_or.reduce(masks)):
            masks.pop()
        for j, m in enumerate(masks):
            v[m] = specials[j % len(specials)]
    return v


# ---- keys -----------------------------------------------------------------------------------------------------------

def hash64(keys):
    """Hash128to64(0, key) on a uint64 array (tg_common.cuh hash128to64_dev)"""
    k = np.uint64(HASH_K)
    a = np.asarray(keys, dtype=np.uint64) * k
    a ^= a >> np.uint64(47)
    a *= k
    a ^= a >> np.uint64(47)
    return a * k


def unhash64(h):
    """the inverse of hash64: the hash is odd multiplications and xor-shifts by 47, each a bijection of 64-bit words (the
    xor-shift by 47 is its own inverse)"""
    ki = np.uint64(HASH_K_INV)
    b = np.asarray(h, dtype=np.uint64) * ki
    b ^= b >> np.uint64(47)
    b *= ki
    b ^= b >> np.uint64(47)
    return b * ki


def keys_with_hash(n, bits, seed=0):
    """n distinct non-zero keys whose Hash128to64(0, key) has the given bit fields, {(shift, width): value}; the other hash
    bits are random.  The hash 0 is the key 0's alone: a field set that leaves no other hash is refused."""
    rng = np.random.default_rng(seed)
    fixed = sum(w for _, w in bits)
    assert 64 - fixed >= int(np.ceil(np.log2(n + 2))) + 2, "too few free hash bits for %d keys" % n
    out = np.zeros(0, dtype=np.uint64)
    while len(out) < n:
        h = rng.integers(0, M64, size=2 * n, dtype=np.uint64, endpoint=True)
        for (shift, width), val in bits.items():
            mask = np.uint64(((1 << width) - 1) << shift)
            h = (h & ~mask) | (np.uint64(val << shift) & mask)
        h = h[h != 0]
        out = np.unique(np.r_[out, h])
    h = rng.permutation(out)[:n]
    return unhash64(h)


# ---- which aggregation path ran -------------------------------------------------------------------------------------

def counters(ctx):
    """launch counts of the aggregation's kernel classes since ctx.profile_enable(True), and tg_hot_records"""
    from thrill_b200 import capi
    return (ctx.profile_get(capi.K_PREAGG)[1], ctx.profile_get(capi.K_AGGREGATE)[1], int(ctx.L.tg_hot_records(ctx.h)))


def path(before, after):
    """(table, hot records) of one aggregation between two `counters` readings with profiling on.  table: "hbm" = the HBM
    table alone (no counting read), "units" = partitioned, the shared-memory units emitted everything, "merge" =
    partitioned, and partial aggregates (pieces of cut segments, mid-unit flushes) were merged in the HBM table"""
    preagg, agg, hot = (a - b for a, b in zip(after, before))
    if preagg == 0:
        assert agg <= 1, (preagg, agg)
        return "hbm", hot
    assert preagg == 1 and agg in (1, 2), (preagg, agg)
    return ("merge" if agg == 2 else "units"), hot
