"""Exact prefix sums of doubles and the rounding bound of tg_scan.cu's bracketing (test helper, numpy and Python ints).

The scan kernels bracket a double sum by tiles, warps and threads, not left to right, so their outputs differ from the stock
left fold (scan_ref.py) by rounding.  This module says by how much, and checks it:

    |got_i - exact_i| <= gamma_D * A_i + u * |exact_i|,    u = 2^-53,  gamma_D = D u / (1 - D u)

exact_i is the exact (unrounded) prefix: initial + every item folded into output i, the lower workers' items included (the
carry initial + (S_0 + ... + S_{r-1}) is exact arithmetic's initial + all of them).  A_i is the same sum over |x|.  D is the
longest chain of additions any summand goes through in the kernels (`depth`).  The u * |exact_i| term leaves room for the
final rounding of the exact value.  The bound holds whenever no partial sum overflows, which (1 + gamma_D) * A_i < DBL_MAX
guarantees (the safe range).  Special values are exact, as in the stock fold: NaN wherever the prefix has seen a NaN or both
infinities, the infinity where it has seen one, and the sign of a zero (-0.0 only where every summand is -0.0) as the model.

Every finite double is an integer multiple of 2^-1074, so a prefix sum is an integer at that scale and can be accumulated
exactly.  `exact_prefix` does it with Python ints (small cases, and the reference of the tests of this module);
`check` accumulates in 32-bit limbs held in int64 numpy columns, a chunk of items at a time, and so handles 1e8 items.

`emulate` restates tg_scan.cu's order of additions on the host in scalar Python floats (IEEE doubles), one function per
kernel, so that the bound can be tested against the kernels' own bracketing on adversarial inputs without a GPU.
"""
import itertools
import math

import numpy as np

import scan_ref as S

U = 2.0 ** -53
DBL_MAX = float(np.finfo(np.float64).max)
SCALE = 1 << 1074                      # every finite double times SCALE is an integer
TILE_BYTES = 32768                     # scan_reduce_kernel / scan_tiles_kernel: 256 threads x 128 bytes
SC_THREADS = 256
ST_THREADS, ST_PER = 512, 8            # scan_prefix_kernel: one CTA, 8 aggregates per thread and round
ROUND = ST_THREADS * ST_PER            # tile aggregates per round of scan_prefix_kernel
NEG0 = -0.0


def tile_items(ib):
    return TILE_BYTES // ib


def per_thread(ib):
    """values per thread in the tile reduce and the tile scan: 16 8-byte items, 8 pairs"""
    return 128 // ib


def ntiles(n, ib):
    return (n * ib + TILE_BYTES - 1) // TILE_BYTES


def rounds(n, ib):
    return max(1, -(-ntiles(n, ib) // ROUND))


def depth(counts, ib):
    """D: the most additions any summand goes through between the input and an output, for p = len(counts) workers of
    counts[r] items of ib bytes.  With k = per_thread(ib) (16 or 8) and R = the rounds of scan_prefix_kernel on the largest
    worker (ceil(tiles / 4096), at least 1):

      tile reduce     k - 1 (the thread's fold) + 5 (warp_reduce) + 7 (thread 0 folds the 8 warp totals)        = k + 11
      tile prefix     7 (the thread folds its 8 aggregates) + 5 (warp_scan) + 16 (the 16 warp totals, folded
                      from the identity) + R - 1 (`running`, one add per earlier round) + 2 (running + (wpre +
                      lane_excl)) + 7 (the thread's aggregates after the first)                                   = 36 + R
      local total     7 + 5 + 16 + R (`running`) + 1 (T() + running)                                            = 29 + R
      carry           S_0 passes r - 1 adds of the inner fold and initial + inner: at most p - 1
      tile scan       1 (carry + e: the tile prefix) + 2 ((tprefix + wpre) + lane_excl) + k (the thread's run)   = k + 3
      in the tile     k - 1 + 5 (warp_scan) + 7 (wpre over at most 7 warp totals) + 2 + k                       = 2k + 13

    A summand of an earlier tile of the same worker: tile reduce + tile prefix + tile scan = 2k + 50 + R.  A summand of a
    lower worker: tile reduce + local total + carry + tile scan = 2k + 42 + R + p.  The initial element: 1 + 1 + k + 2.
    Additions of the identity -0.0 and of T() = +0.0 are exact; counting them only makes D larger.
    At 2^30 - 1 items on one worker D = 146 for 8-byte items and 194 for pairs (gamma_D about 2.2e-14)."""
    k = per_thread(ib)
    r = max(rounds(n, ib) for n in counts) if counts else 1
    p = max(1, len(counts))
    tile_reduce, tile_prefix, local_total = k + 11, 36 + r, 29 + r
    carry, tile_scan, in_tile = p - 1, k + 3, 2 * k + 13
    return max(in_tile, tile_reduce + tile_prefix + tile_scan, tile_reduce + local_total + carry + tile_scan)


def gamma(d):
    return d * U / (1 - d * U)


# ---- the exact reference in Python ints --------------------------------------------------------------------------------
def to_fixed(x):
    """a finite double as the integer x * 2^1074"""
    num, den = float(x).as_integer_ratio()
    return num * (SCALE // den)


def to_double(v):
    """the integer v / 2^1074 rounded once to a double (int / int is correctly rounded); +-inf past DBL_MAX"""
    try:
        return v / SCALE
    except OverflowError:
        return math.copysign(math.inf, v)


def _flat(shards, pair, initial):
    """the items' values of all workers in global order as doubles, and the initial value as a double"""
    vals = [S.split_values(s, pair)[1] for s in shards]
    x = np.concatenate(vals).view(np.float64) if vals else np.zeros(0)
    return x, float(np.array([initial[1]], np.uint64).view(np.float64)[0])


def exact_prefix(shards, pair=False, initial=(0, 0), inclusive=True):
    """(exact_i, A_i) of every output in global order, as Python ints at scale 2^1074 (finite summands only)"""
    x, init = _flat(shards, pair, initial)
    fin = [to_fixed(v) if math.isfinite(v) else 0 for v in x.tolist()]
    i0 = to_fixed(init) if math.isfinite(init) else 0
    e = list(itertools.accumulate(fin, initial=i0))
    a = list(itertools.accumulate((abs(v) for v in fin), initial=abs(i0)))
    return (e[1:], a[1:]) if inclusive else (e[:-1], a[:-1])


# ---- the exact reference in limbs --------------------------------------------------------------------------------------
_M32 = np.uint64(0xFFFFFFFF)
_CHUNK_LIMBS = 1 << 21                 # limbs per chunk of `check` (16 MB of int64)


def _ulp_exp(x):
    """(m, q): |x| = m * 2^q with m < 2^53 an integer and q >= -1074 (m = 0 for zeros); x finite"""
    mf, e = np.frexp(np.abs(x))
    m = (mf * 9007199254740992.0).astype(np.uint64)
    q = e.astype(np.int64) - 53
    low = q < -1074                     # subnormals: the bits below 2^-1074 are zero
    m[low] >>= (-1074 - q[low]).astype(np.uint64)
    return m, np.maximum(q, -1074)


def _words(x, base, sign):
    """x * 2^-base (x finite, a multiple of 2^base) as three signed 32-bit words at limb k: (k, w0, w1, w2)"""
    m, q = _ulp_exp(x)
    sh = np.where(m == 0, 0, q - base)
    assert (sh >= 0).all()
    k = sh // 32
    o = (sh % 32).astype(np.uint64)
    p0 = (m & _M32) << o
    p1 = (m >> np.uint64(32)) << o
    w = [(p0 & _M32).astype(np.int64), ((p0 >> np.uint64(32)) + (p1 & _M32)).astype(np.int64),
         (p1 >> np.uint64(32)).astype(np.int64)]
    if sign:
        s = np.where(np.signbit(x), -1, 1)
        w = [s * v for v in w]
    return k, w


def _rows(x, base, nl, sign=True):
    """one row of nl limbs per item"""
    r = np.zeros((len(x), nl), np.int64)
    k, w = _words(x, base, sign)
    i = np.arange(len(x))
    for j in range(3):
        r[i, k + j] = w[j]
    return r


def _normalize(r, top):
    """limbs into [0, 2^32), the rest carried into top (the value: top * 2^(32 nl) + sum r_j 2^(32 j))"""
    c = np.zeros(len(r), np.int64)
    for j in range(r.shape[1]):
        v = r[:, j] + c
        r[:, j] = v & 0xFFFFFFFF
        c = v >> 32
    return top + c


def _magnitude(r, top):
    """(f, ex): |value| = f * 2^ex within 4u (f = 0 for zero).  r is normalized; r and top are overwritten"""
    neg = top < 0
    if neg.any():                       # -v = (-top - 1) 2^(32 nl) + sum (2^32 - 1 - r_j) 2^(32 j) + 1
        sub = 0xFFFFFFFF - r[neg]
        sub[:, 0] += 1
        top[neg] = _normalize(sub, -top[neg] - 1)
        r[neg] = sub
    assert (top == 0).all()
    nl = r.shape[1]
    nz = r != 0
    t = nl - 1 - np.argmax(nz[:, ::-1], axis=1)
    pad = np.concatenate([np.zeros((len(r), 3), np.int64), r], axis=1).astype(np.float64)
    i = np.arange(len(r))
    f = ((pad[i, t + 3] * 2.0 ** 96 + pad[i, t + 2] * 2.0 ** 64) + pad[i, t + 1] * 2.0 ** 32) + pad[i, t]
    f[~nz.any(axis=1)] = 0.0
    return f, (32 * (t - 3)).astype(np.int32)


class Result(object):
    """what `check` measured: the depth D, the largest |got - exact| / (u A) over the checked outputs (0 if none), and the
    number of outputs checked against the bound"""

    def __init__(self, d, ratio, checked):
        self.depth, self.ratio, self.checked = d, ratio, checked

    def __repr__(self):
        return "D=%d max |got-exact|/(u A)=%.3g over %d outputs" % (self.depth, self.ratio, self.checked)


def _values(outs, pair):
    """per-worker outputs (a list) -> their value words in global order; an array is taken as value words already"""
    if not isinstance(outs, (list, tuple)):
        return np.asarray(outs, np.uint64).reshape(-1)
    parts = [S.split_values(o, pair)[1] for o in outs]
    return np.concatenate(parts) if parts else np.zeros(0, np.uint64)


def check(got, shards, pair=False, initial=(0, 0), inclusive=True, stock=None, select=None, d=None, beyond="error"):
    """assert that the double-sum outputs `got` (per-worker outputs, or their value words in global order) of PrefixSum
    (inclusive) or ExPrefixSum over `shards` meet the contract of the module docstring; returns a Result.

    stock: the stock left fold's value words (default: scan_ref's bit-exact model), the source of the special values and
    the signs of zeros.  select: the global positions `got` holds (default: all).  d: the depth (default: depth() of the
    shards).  beyond: what to do with an output outside the safe range: "error" (the test's data must stay inside it),
    "skip" (no promise beyond reproducibility), or "check" (check it as if it were inside)."""
    x, init = _flat(shards, pair, initial)
    n = len(x)
    g = np.ascontiguousarray(_values(got, pair), np.uint64).view(np.float64)
    if stock is None:
        stock = _values(S.prefix_sum(shards, S.OP_SUM_F64, pair, initial, inclusive), pair)
    st = np.ascontiguousarray(stock, np.uint64).view(np.float64)
    sel = np.arange(n) if select is None else np.asarray(select, np.int64)
    st = st[sel] if len(st) == n and len(sel) != n else st
    assert len(g) == len(sel) == len(st), (len(g), len(sel), len(st))
    if d is None:
        d = depth([len(S.split_values(s, pair)[1]) for s in shards], 16 if pair else 8)
    gm = gamma(d)
    # the specials, exact
    sn, gn = np.isnan(st), np.isnan(g)
    _first_bad(sn != gn, "NaN where the stock has none (or the reverse)", sel, g, st)
    sinf = np.isinf(st)
    _first_bad(sinf & (g != st), "not the stock's infinity", sel, g, st)
    z = (g == 0) & (st == 0)
    _first_bad(z & (np.signbit(g) != np.signbit(st)), "a zero of the wrong sign", sel, g, st)
    num = np.isfinite(st)
    # the exact prefix, |x| prefix and |exact - got|, a chunk at a time
    xf = np.where(np.isfinite(x), x, 0.0)
    i0 = init if math.isfinite(init) else 0.0
    gf = np.where(np.isfinite(g), g, 0.0)
    allv = np.concatenate([xf, [i0], gf])
    nzv = allv[allv != 0]
    base = int(_ulp_exp(nzv)[1].min()) if len(nzv) else -1074
    top_bit = int(np.frexp(np.abs(nzv).max())[1]) if len(nzv) else 0
    nl = (top_bit - base + (n + 2).bit_length() + 4) // 32 + 4
    carry, ctop = _rows(np.array([i0]), base, nl)[0], 0
    acarry, atop = _rows(np.array([abs(i0)]), base, nl, sign=False)[0], 0
    ratio, checked = 0.0, 0
    chunk = max(1 << 12, _CHUNK_LIMBS // nl)
    pos = np.searchsorted(sel, np.arange(0, n + 2 * chunk, chunk))
    for c0 in range(0, n, chunk):
        c1 = min(n, c0 + chunk)
        s0, s1 = pos[c0 // chunk], pos[c0 // chunk + 1]
        xs = xf[c0:c1]
        e = np.cumsum(_rows(xs, base, nl), axis=0) + carry
        etop = _normalize(e, np.full(len(e), ctop, np.int64))
        a = np.cumsum(_rows(xs, base, nl, sign=False), axis=0) + acarry
        atp = _normalize(a, np.full(len(a), atop, np.int64))
        if not inclusive:               # output i is the inclusive prefix of item i - 1
            e, etop = np.concatenate([carry[None], e]), np.concatenate([[ctop], etop])
            a, atp = np.concatenate([acarry[None], a]), np.concatenate([[atop], atp])
        # the next chunk starts from the inclusive prefix of this chunk's last item
        carry, ctop, acarry, atop = e[-1].copy(), int(etop[-1]), a[-1].copy(), int(atp[-1])
        if not inclusive:
            e, etop, a, atp = e[:-1], etop[:-1], a[:-1], atp[:-1]
        loc = sel[s0:s1] - c0
        if not len(loc):
            continue
        e, etop, a, atp = e[loc], etop[loc], a[loc], atp[loc]
        diff = e - _rows(gf[s0:s1], base, nl)
        dtop = _normalize(diff, etop.copy())
        fd, ed = _magnitude(diff, dtop)
        fa, ea = _magnitude(a, atp)
        fe, ee = _magnitude(e, etop)
        with np.errstate(over="ignore", under="ignore", invalid="ignore"):
            big_a = np.ldexp(fa, ea + np.int32(base))
            safe = big_a * (1 + gm + 8 * U) < DBL_MAX
            lhs = np.ldexp(fd, ed - ea)
            tol = (gm * fa + U * np.ldexp(fe, ee - ea)) * (1 + 16 * U)
            ok = np.where(fa == 0, fd == 0, lhs <= tol)
            r = np.where(fa == 0, 0.0, lhs / (U * np.where(fa == 0, 1.0, fa)))
        m = num[s0:s1]
        if beyond == "error":
            _first_bad(m & ~safe, "outside the safe range (1 + gamma_D) A < DBL_MAX: the test's data is too large",
                       sel[s0:s1], g[s0:s1], st[s0:s1])
        elif beyond == "skip":
            m = m & safe
        _first_bad(m & ~np.isfinite(g[s0:s1]), "not finite where the stock's output is (inside the safe range)",
                   sel[s0:s1], g[s0:s1], st[s0:s1])
        _first_bad(m & ~ok, "|got - exact| > gamma_%d A + u |exact|" % d, sel[s0:s1], g[s0:s1], st[s0:s1])
        if m.any():
            ratio = max(ratio, float(r[m].max()))
            checked += int(m.sum())
    return Result(d, ratio, checked)


def _first_bad(bad, msg, sel, g, st):
    if np.any(bad):
        i = int(np.flatnonzero(bad)[0])
        raise AssertionError("%s at output %d (%d of %d): got %r, the stock fold gives %r" % (
            msg, int(sel[i]), int(bad.sum()), len(bad), float(g[i]), float(st[i])))


# ---- tg_scan.cu's order of additions, emulated -----------------------------------------------------------------------------
def _warp_reduce(v):
    """warp_reduce over 32 lanes: lane 0's result (a lane whose source is out of range keeps its own value)"""
    v = list(v)
    for d in (16, 8, 4, 2, 1):
        v = [v[l] + (v[l + d] if l + d < 32 else v[l]) for l in range(32)]
    return v[0]


def _warp_scan(v):
    """warp_scan: (inclusive, exclusive) of 32 lanes, Hillis-Steele from the left"""
    v = list(v)
    for d in (1, 2, 4, 8, 16):
        v = [v[l - d] + v[l] if l >= d else v[l] for l in range(32)]
    return v, [NEG0] + v[:31]


def emu_tile_reduce(vals, ib):
    """scan_reduce_kernel: the aggregate of one tile (vals: its values; the rest of the tile is the identity -0.0)"""
    vals = list(vals) + [NEG0] * (tile_items(ib) - len(vals))
    lanes = []
    for tid in range(SC_THREADS):
        if ib == 16:
            acc = vals[tid]
            for j in range(1, 8):
                acc = acc + vals[tid + 256 * j]
        else:
            u = tid
            acc = vals[2 * u] + vals[2 * u + 1]
            for j in range(1, 8):
                u = tid + 256 * j
                acc = (acc + vals[2 * u]) + vals[2 * u + 1]
        lanes.append(acc)
    ws = [_warp_reduce(lanes[32 * w:32 * w + 32]) for w in range(SC_THREADS // 32)]
    t = ws[0]
    for w in range(1, len(ws)):
        t = t + ws[w]
    return t


def emu_tile_prefix(agg, carry):
    """scan_prefix_kernel: (the tile prefixes seeded with carry, the local total T() + the fold of the aggregates)"""
    nt = len(agg)
    out = [None] * nt
    running = NEG0
    for base in range(0, nt, ROUND):
        v = [[agg[i] if i < nt else NEG0 for i in range(base + tid * ST_PER, base + tid * ST_PER + ST_PER)]
             for tid in range(ST_THREADS)]
        t = []
        for vv in v:
            s = vv[0]
            for k in range(1, ST_PER):
                s = s + vv[k]
            t.append(s)
        excl, wsum = [], []
        for w in range(ST_THREADS // 32):
            inc, exc = _warp_scan(t[32 * w:32 * w + 32])
            excl += exc
            wsum.append(inc[31])
        wpre, chunk = [], NEG0
        for w in range(len(wsum)):
            wpre.append(chunk)
            chunk = chunk + wsum[w]
        for tid in range(ST_THREADS):
            e = running + (wpre[tid // 32] + excl[tid])
            i0 = base + tid * ST_PER
            for k in range(ST_PER):
                if i0 + k < nt:
                    out[i0 + k] = carry + e
                e = e + v[tid][k]
        running = running + chunk
    return out, 0.0 + running


def emu_tile_scan(vals, tprefix, ib, inclusive):
    """scan_tiles_kernel: the outputs of one tile from its tile prefix"""
    n = len(vals)
    k = per_thread(ib)
    vals = list(vals) + [NEG0] * (tile_items(ib) - n)
    t = []
    for tid in range(SC_THREADS):
        s = vals[k * tid]
        for j in range(1, k):
            s = s + vals[k * tid + j]
        t.append(s)
    excl, wsum = [], []
    for w in range(SC_THREADS // 32):
        inc, exc = _warp_scan(t[32 * w:32 * w + 32])
        excl += exc
        wsum.append(inc[31])
    out = []
    for tid in range(SC_THREADS):
        wpre = NEG0
        for w in range(tid // 32):
            wpre = wpre + wsum[w]
        run = (tprefix + wpre) + excl[tid]
        for j in range(k):
            x = vals[k * tid + j]
            if inclusive:
                run = run + x
                out.append(run)
            else:
                out.append(run)
                run = run + x
    return out[:n]


def emulate(shards, pair=False, initial=(0, 0), inclusive=True):
    """the value words of every worker's outputs, in global order, as tg_scan.cu computes them"""
    ib = 16 if pair else 8
    ti = tile_items(ib)
    vals = [S.split_values(s, pair)[1].view(np.float64).tolist() for s in shards]
    init = float(np.array([initial[1]], np.uint64).view(np.float64)[0])
    tiles = [[v[i:i + ti] for i in range(0, len(v), ti)] for v in vals]
    aggs = [[emu_tile_reduce(t, ib) for t in tl] for tl in tiles]
    totals = [emu_tile_prefix(a, 0.0)[1] for a in aggs]
    out = []
    for r in range(len(shards)):
        c = init
        if r:
            inner = totals[0]
            for i in range(1, r):
                inner = inner + totals[i]
            c = init + inner
        pre, _ = emu_tile_prefix(aggs[r], c)
        for t, tp in zip(tiles[r], pre):
            out += emu_tile_scan(t, tp, ib, inclusive)
    return S.f64_words(np.array(out, np.float64))


# ---- data ------------------------------------------------------------------------------------------------------------------
KINDS = ["small", "subnormal", "subnormal_mixed", "wide", "cancel", "top"]


def edges(ib, n):
    """the structural edges of a worker of n items, as local positions: a thread's run, lane 31, warp 7, the tile, the
    next tile's first warp, and the partial last tile"""
    k, t = per_thread(ib), tile_items(ib)
    e = {k, 31 * k, 32 * k, 7 * 32 * k, t - k, t, t + 32 * k, 2 * t, n - 1, n - k}
    e |= {j * t for j in range(3, n // t + 1)}
    return sorted(x for x in e if 0 < x < n)


def gen(kind, counts, ib, seed):
    """the values (doubles) of sum(counts) items for one kind of test data:
      small            magnitudes 1e-300 .. 1e-12, random signs
      subnormal        subnormals only, so small that every partial sum stays subnormal: every sum is exact
      subnormal_mixed  subnormals mixed with normal values of 1e-300 .. 1
      wide             exponents 2^-1000 .. 2^1000 (the largest prefix over |x| stays below 2^1000 n)
      cancel           noise of magnitude 1 with (x, -x), x up to 1e20, astride every structural edge of every worker
      top              positive values whose sum over |x| ends just below the safe limit DBL_MAX / (1 + gamma_D)"""
    n = int(sum(counts))
    rng = np.random.RandomState(seed)
    sgn = np.where(rng.randint(0, 2, n) == 1, -1.0, 1.0)
    if kind == "small":
        return sgn * rng.uniform(1, 10, n) * 10.0 ** rng.randint(-300, -12, n)
    if kind == "subnormal":
        lim = (1 << 52) // (n + 2)
        return np.ldexp(rng.randint(-lim, lim + 1, n).astype(np.float64), -1074)
    if kind == "subnormal_mixed":
        x = np.ldexp(rng.randint(-(1 << 52) + 1, 1 << 52, n).astype(np.float64), -1074)
        big = rng.randint(0, 3, n) == 0
        x[big] = sgn[big] * rng.uniform(1, 10, int(big.sum())) * 10.0 ** rng.randint(-300, 0, int(big.sum()))
        return x
    if kind == "wide":
        return np.ldexp(rng.uniform(-1, 1, n), rng.randint(-1000, 1001, n))
    if kind == "cancel":
        x = rng.standard_normal(n)
        off = 0
        for c in counts:
            for e in edges(ib, c) + ([0] if c else []):
                if off + e >= 1:
                    big = sgn[off + e] * rng.uniform(1, 10) * 10.0 ** rng.randint(12, 20)
                    x[off + e - 1], x[off + e] = big, -big
            off += c
        return x
    if kind == "top":
        w = rng.uniform(0.5, 1.0, n)
        lim = DBL_MAX / (1 + gamma(depth(counts, ib)) + 8 * U)
        return w * (0.999 * lim / w.sum())
    raise ValueError(kind)


def items_of(values, pair, seed=0):
    """8-byte items (the value words) or pairs with positional keys"""
    v = S.f64_words(values)
    if not pair:
        return v
    return S.pairs(S.splitmix64(np.arange(len(v), dtype=np.uint64) + np.uint64(seed)), v)
