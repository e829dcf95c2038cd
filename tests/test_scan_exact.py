"""The exact reference and the error bound of PrefixSum's double sums (scan_exact.py), on the host: the exact prefix against
fractions.Fraction, the limb accumulation of `check` against Python ints, tg_scan.cu's bracketing (emulated in scalar
doubles) within the bound on adversarial inputs at every structural edge, and planted errors the check must reject.  CPU only."""
import math
from fractions import Fraction

import numpy as np
import pytest

import scan_exact as X
import scan_ref as S

LAYOUTS = {1: [[3 * 4096 + 517]], 2: [[4096 + 31, 2 * 4096 + 17]], 3: [[5000, 0, 6001]],
           8: [[0, 4097, 1, 0, 2049, 8192, 0, 300]], 16: [[0, 700, 0, 0, 4096, 1, 0, 2047, 0, 33, 0, 0, 5000, 0, 1, 0]]}


def _layouts(ib):
    """worker sizes at p = 1, 2, 3, 8, 16 (empty workers included), in items of ib bytes (half as many pairs)"""
    return [[c * 8 // ib for c in counts] for p in sorted(LAYOUTS) for counts in LAYOUTS[p]]


def _shards(values, counts, pair, seed=0):
    return S.shards_of(X.items_of(values, pair, seed), counts)


def _fraction_prefix(x, init, inclusive):
    acc, out = Fraction(init), []
    for v in x:
        if inclusive:
            acc += Fraction(v)
            out.append(acc)
        else:
            out.append(acc)
            acc += Fraction(v)
    return out


# ---- the exact reference ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inclusive", [True, False])
@pytest.mark.parametrize("pair", [False, True])
def test_exact_prefix_equals_fractions(pair, inclusive):
    rng = np.random.RandomState(3)
    cases = [X.gen(k, [40, 0, 57], 16 if pair else 8, s) for s, k in enumerate(X.KINDS)]
    cases.append(np.array([1e308, -1e308, 5e-324, -5e-324, 2.0 ** -1022, -0.0, 0.0, 1.0, -2.0 ** -1074 * 3]))
    cases.append(np.ldexp(rng.uniform(-1, 1, 200), rng.randint(-1074, 1000, 200)))
    for i, x in enumerate(cases):
        init = [0.0, -0.0, 1e-320, -3.5e300][i % 4]
        counts = [len(x) // 3, 0, len(x) - len(x) // 3]
        shards = _shards(x, counts, pair)
        e, a = X.exact_prefix(shards, pair, (5, int(S.f64_words([init])[0])), inclusive)
        want = _fraction_prefix(x, init, inclusive)
        assert [Fraction(v, X.SCALE) for v in e] == want
        assert [Fraction(v, X.SCALE) for v in a] == _fraction_prefix(np.abs(x), abs(init), inclusive)
        assert [X.to_double(v) for v in e] == [float(f) for f in want]         # one correct rounding


@pytest.mark.parametrize("inclusive", [True, False])
def test_check_measures_the_exact_error(inclusive):
    """`check` on the correctly rounded exact prefix, over more than one chunk of its limb accumulation: the error ratio it
    reports is the one Python ints give, and at most 1 (the u |exact| term)"""
    for kind in X.KINDS:
        counts = [70001, 0, 9000]           # more than one chunk of the limb accumulation
        x = X.gen(kind, counts, 8, 11)
        shards = _shards(x, counts, False)
        init = (0, int(S.f64_words([0.25])[0]))
        e, a = X.exact_prefix(shards, False, init, inclusive)
        got = np.array([X.to_double(v) for v in e])
        res = X.check(S.f64_words(got), shards, False, init, inclusive)
        want = max(abs(Fraction(g) - Fraction(v, X.SCALE)) / (Fraction(X.U) * Fraction(w, X.SCALE))
                   for g, v, w in zip(got.tolist(), e, a) if w)
        assert res.checked == sum(counts)
        assert math.isclose(res.ratio, float(want), rel_tol=1e-12, abs_tol=1e-300), (kind, res.ratio, float(want))
        assert res.ratio <= 1.0


# ---- the kernels' bracketing is within the bound ------------------------------------------------------------------------
@pytest.mark.parametrize("inclusive", [True, False])
@pytest.mark.parametrize("pair", [False, True])
@pytest.mark.parametrize("kind", X.KINDS)
def test_emulated_bracketing_within_the_bound(kind, pair, inclusive):
    ib = 16 if pair else 8
    worst = 0.0
    for counts in _layouts(ib):
        x = X.gen(kind, counts, ib, 100 + len(counts))
        shards = _shards(x, counts, pair)
        init = (3, int(S.f64_words([x[len(x) // 2] if kind != "top" else 0.0])[0]))
        got = X.emulate(shards, pair, init, inclusive)
        res = X.check(got, shards, pair, init, inclusive)
        assert res.checked == sum(counts)
        worst = max(worst, res.ratio / res.depth)
        if kind == "subnormal":            # every partial sum is exact: the stock's bits
            stock = X._values(S.prefix_sum(shards, S.OP_SUM_F64, pair, init, inclusive), pair)
            assert np.array_equal(got, stock)
    print("emulated %s pair=%d incl=%d: max |got-exact| / (u A D) = %.3g" % (kind, pair, inclusive, worst))


def test_emulation_is_the_stock_fold_on_exact_data():
    """integer-valued doubles below 2^53: every bracketing is exact, so the emulation gives the stock's bits"""
    rng = np.random.RandomState(5)
    for pair in (False, True):
        counts = [9000, 0, 4097]
        x = rng.randint(-(1 << 30), 1 << 30, sum(counts)).astype(np.float64)
        shards = _shards(x, counts, pair)
        for inclusive in (True, False):
            got = X.emulate(shards, pair, (1, int(S.f64_words([-7.0])[0])), inclusive)
            stock = X._values(S.prefix_sum(shards, S.OP_SUM_F64, pair, (1, int(S.f64_words([-7.0])[0])), inclusive), pair)
            assert np.array_equal(got, stock)


def test_tile_prefix_over_several_rounds_within_its_depth():
    """scan_prefix_kernel alone over 3 rounds of aggregates (R = 3) with cancellation between rounds: the tile prefixes are
    within gamma_(36 + R + 1) of the exact exclusive prefix (the aggregates as exact inputs, the carry added once)"""
    rng = np.random.RandomState(8)
    nt = 2 * X.ROUND + 777
    agg = rng.standard_normal(nt) * 10.0 ** rng.randint(-3, 4, nt)
    for b in (X.ROUND, 2 * X.ROUND, 512, 4095):
        agg[b - 1], agg[b] = 3e17, -3e17
    carry = 0.3
    pre, total = X.emu_tile_prefix(agg.tolist(), carry)
    d = 36 + X.rounds(nt * 4096, 8) + 1
    assert X.rounds(nt * 4096, 8) == 3
    res = X.check(S.f64_words(pre), [S.f64_words(agg)], False, (0, int(S.f64_words([carry])[0])), False, d=d)
    assert res.checked == nt
    tot = X.check(S.f64_words([total]), [S.f64_words(agg)], False, (0, 0), True, select=[nt - 1], d=29 + 3)
    assert tot.checked == 1


def test_empty_input():
    for pair in (False, True):
        empty = S.pairs([], []) if pair else np.zeros(0, np.uint64)
        for inclusive in (True, False):
            res = X.check([empty, empty], [empty, empty], pair, (0, int(S.f64_words([1.5])[0])), inclusive)
            assert res.checked == 0


def test_depth_terms():
    assert X.depth([100], 8) == 2 * 16 + 50 + 1 and X.depth([100], 16) == 2 * 8 + 50 + 1
    assert X.depth([(1 << 30) - 1], 8) == 146 and X.depth([(1 << 30) - 1], 16) == 194
    assert X.depth([1] * 16, 8) == 2 * 16 + 42 + 1 + 16
    assert X.rounds(4096 * 4096, 8) == 1 and X.rounds(4096 * 4096 + 1, 8) == 2 and X.rounds(2048 * 4096 + 1, 16) == 2


# ---- planted errors ------------------------------------------------------------------------------------------------------
def _planted_base():
    counts = [4096 * 3 + 100]
    x = X.gen("cancel", counts, 8, 2)
    x[::7] *= 1e-6                          # small items among large ones
    return counts, x, _shards(x, counts, False)


def _above_the_bound(shards, x, d):
    """the positions whose item is above 4x the bound at that position"""
    _, a = X.exact_prefix(shards)
    tol = np.array([X.gamma(d) * X.to_double(v) for v in a])
    return np.flatnonzero(np.abs(x) > 4 * tol)


def test_check_rejects_a_dropped_item():
    """the kernels' bracketing with one item left out: the smallest item above the bound at its position"""
    counts, x, shards = _planted_base()
    res = X.check(X.emulate(shards), shards)
    cand = _above_the_bound(shards, x, res.depth)
    i = int(cand[np.argmin(np.abs(x[cand]))])
    dropped = x.copy()
    dropped[i] = 0.0
    bad = X.emulate(_shards(dropped, counts, False))
    with pytest.raises(AssertionError, match="gamma"):
        X.check(bad, shards)


def test_check_rejects_an_output_shifted_by_one():
    counts, x, shards = _planted_base()
    inc = X.emulate(shards, inclusive=True)
    exc = X.emulate(shards, inclusive=False)
    X.check(inc, shards, inclusive=True)
    X.check(exc, shards, inclusive=False)
    with pytest.raises(AssertionError):
        X.check(exc, shards, inclusive=True)
    with pytest.raises(AssertionError):
        X.check(inc, shards, inclusive=False)
    cand = _above_the_bound(shards, x, X.depth(counts, 8))
    i = int(cand[(cand > 5000) & (cand < len(x) - 1)][0])
    sh = inc.copy()
    sh[i - 1] = inc[i]                     # output i - 1 takes the next item
    with pytest.raises(AssertionError, match="gamma"):
        X.check(sh, shards)


def test_check_rejects_zeros_for_tiny_data():
    """1e-12 data: the largest prefix is far below 1e-9, yet all-zero outputs fail (the bound has no absolute floor)"""
    rng = np.random.RandomState(4)
    x = rng.uniform(0.5, 1.0, 100000) * 1e-12 * np.where(rng.randint(0, 2, 100000) == 1, -1, 1)
    shards = [S.f64_words(x)]
    X.check(X.emulate(shards), shards)
    with pytest.raises(AssertionError, match="gamma"):
        X.check(np.zeros(len(x), np.uint64), shards)


def _overflow_example():
    x = np.zeros(4096 + 64)
    x[0], x[4096], x[4097] = -1e308, 1e308, 1e308
    return x, [S.f64_words(x)]


def test_overflow_example_leaves_the_safe_range():
    """x[0] = -1e308, x[4096] = x[4097] = 1e308: the stock fold stays finite (1e308 from position 4097), but tile 1's
    thread 0 adds 1e308 + 1e308 into its run, so every output of tile 1 from its thread 1 on (position 4112) is +inf.
    The check rejects that when told the outputs are inside the safe range, and finds them outside it (A > DBL_MAX)"""
    x, shards = _overflow_example()
    got = X.emulate(shards).view(np.float64)
    stock = X._values(S.prefix_sum(shards, S.OP_SUM_F64), False).view(np.float64)
    assert (stock[4097:] == 1e308).all() and np.isfinite(stock).all()
    assert np.isfinite(got[:4112]).all() and (got[4112:] == np.inf).all()
    with pytest.raises(AssertionError, match="not finite"):
        X.check(S.f64_words(got), shards, beyond="check")
    with pytest.raises(AssertionError, match="safe range"):
        X.check(S.f64_words(got), shards)
    res = X.check(S.f64_words(got), shards, beyond="skip")
    assert res.checked == 4096                # positions 0 .. 4095: A = 1e308
