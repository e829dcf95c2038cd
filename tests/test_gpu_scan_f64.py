"""PrefixSum / ExPrefixSum double sums on one H100 against the exact prefix sums of scan_exact.py: every output within
gamma_D * A + u |exact| of the exact value, NaN, inf and the sign of zero as the stock left fold, at p = 1 and at p = 2, 3,
8 and 16 workers simulated on one GPU (empty workers included), for 8-byte items and pairs, inclusive and exclusive.  Small,
subnormal, wide and top-of-range magnitudes, cancellation astride the structural edges, a one-hot sweep over them, the
special values, several rounds of the tile-prefix kernel (every op), 1e8 items, and the overflow the bracketing can meet
outside the safe range.  Each check prints its largest |got - exact| / (u A) next to D.  pytest -m gpu."""
import numpy as np
import pytest

import scan_exact as X
import scan_ref as S
from test_gpu_scan import INT_OPS, ctx, make_items, scan_dev, simulate, words  # noqa: F401  (ctx: the fixture)

pytestmark = pytest.mark.gpu


def layouts(ib):
    """worker sizes at p = 1, 2, 3, 8 and 16, empty workers included: about three and a half tiles in all"""
    t = X.tile_items(ib)
    return [[3 * t + t // 2 + 5], [t + 31, 2 * t + 17], [t + t // 3, 0, 2 * t + 1],
            [0, t + 1, 1, 0, t // 2 + 1, 2 * t, 0, 300], [0, 700, 0, 0, t, 1, 0, t // 2 - 1, 0, 33, 0, 0, t + 900, 0, 1, 0]]


def run(ctx, shards, pair, initial, inclusive):
    """the operator at p = 1, the simulated workers otherwise; .first of pairs checked exactly against the model"""
    if len(shards) == 1:
        st, res = scan_dev(ctx, shards[0], S.OP_SUM_F64, pair, initial, inclusive)
        assert st == 0, ctx.L.tg_last_error(ctx.h)
        outs = [res]
    else:
        outs = simulate(ctx, S.OP_SUM_F64, pair, shards, initial, inclusive)
    if pair:
        ref = S.prefix_sum(shards, S.OP_SUM_F64, pair, initial, inclusive)
        for o, r in zip(outs, ref):
            assert np.array_equal(o["key"], r["key"])
    return outs


def report(name, res):
    print("SCAN_F64_MARGIN %-48s %r" % (name, res))


def _init(v):
    return (7, int(S.f64_words([v])[0]))


# ---- magnitudes and cancellation ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("inclusive", [True, False])
@pytest.mark.parametrize("pair", [False, True])
@pytest.mark.parametrize("kind", X.KINDS)
def test_kinds_within_the_bound(ctx, kind, pair, inclusive):
    ib = 16 if pair else 8
    worst = None
    for counts in layouts(ib):
        x = X.gen(kind, counts, ib, 31 + len(counts))
        shards = S.shards_of(X.items_of(x, pair, len(counts)), counts)
        init = _init(0.0 if kind == "top" else x[1])
        outs = run(ctx, shards, pair, init, inclusive)
        res = X.check(outs, shards, pair, init, inclusive)
        assert res.checked == sum(counts)
        if kind == "subnormal":          # every partial sum of these subnormals is exact: the stock's bits
            ref = S.prefix_sum(shards, S.OP_SUM_F64, pair, init, inclusive)
            assert all(np.array_equal(words(o), words(r)) for o, r in zip(outs, ref)), counts
        worst = res if worst is None or res.ratio / res.depth > worst.ratio / worst.depth else worst
    report("%s pair=%d incl=%d" % (kind, pair, inclusive), worst)


@pytest.mark.parametrize("inclusive", [True, False])
@pytest.mark.parametrize("pair", [False, True])
def test_one_hot_sweep_over_the_structural_edges(ctx, pair, inclusive):
    """1.0 over noise of 1e-20 at every structural edge of every worker: the first and last item of a thread's run, lane 31,
    warp 7, a tile's first item, the partial last tile, a worker's first and last item"""
    ib = 16 if pair else 8
    k, t = X.per_thread(ib), X.tile_items(ib)
    rng = np.random.RandomState(17)
    worst = None
    for counts in (layouts(ib)[0], layouts(ib)[2]):
        n = sum(counts)
        noise = rng.uniform(-1e-20, 1e-20, n)
        starts = np.concatenate([[0], np.cumsum(counts)])
        where = set()
        for r, c in enumerate(counts):
            local = [0, k - 1, k, 31 * k, 32 * k - 1, 7 * 32 * k, t - 1, t, t + 1, c - t // 3, c - 1]
            where |= {int(starts[r]) + j for j in local if 0 <= j < c}
        for pos in sorted(where):
            x = noise.copy()
            x[pos] = 1.0
            shards = S.shards_of(X.items_of(x, pair), counts)
            res = X.check(run(ctx, shards, pair, _init(0.0), inclusive), shards, pair, _init(0.0), inclusive)
            worst = res if worst is None or res.ratio > worst.ratio else worst
    report("one-hot pair=%d incl=%d" % (pair, inclusive), worst)


# ---- special values --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inclusive", [True, False])
@pytest.mark.parametrize("pair", [False, True])
def test_specials(ctx, pair, inclusive):
    ib = 16 if pair else 8
    t = X.tile_items(ib)
    rng = np.random.RandomState(23)
    cases = []
    # +inf and -inf in different tiles, and in different workers: NaN from the second on
    c3 = [t + 5, 0, 2 * t + 9]
    x = rng.standard_normal(sum(c3))
    x[t // 2], x[t + 5 + t + 3] = np.inf, -np.inf
    cases += [([sum(c3)], x, 0.0), (c3, x, 0.0)]
    y = rng.standard_normal(sum(c3))
    y[3 * t // 2] = -np.inf                                   # one infinity: tile 1 at p = 1, worker 2's first tile at p = 3
    cases += [([sum(c3)], y, 0.5), (c3, y, 0.5)]
    # NaN in the partial last tile
    z = rng.standard_normal(2 * t + 100)
    z[2 * t + 50] = np.nan
    cases += [([len(z)], z, 0.0), ([t, 0, t + 100], z, 0.0)]
    # -0.0 runs across tiles and empty workers
    nz = np.full(2 * t + 3, -0.0)
    for counts in ([len(nz)], [0, t + 1, 0, t + 2, 0]):
        cases += [(counts, nz, -0.0), (counts, nz, 0.0)]
    part = nz.copy()
    part[t + 7] = 0.0                                         # one +0.0: +0.0 from there on
    cases += [([len(part)], part, -0.0), ([t, 0, t + 3], part, -0.0)]
    # initial elements of +-0.0, +-inf and NaN
    w = rng.standard_normal(t + 77)
    for init in (0.0, -0.0, np.inf, -np.inf, np.nan):
        cases += [([len(w)], w, init), ([40, 0, t + 37], w, init)]
    for counts, v, init in cases:
        shards = S.shards_of(X.items_of(v, pair), counts)
        outs = run(ctx, shards, pair, _init(init), inclusive)
        X.check(outs, shards, pair, _init(init), inclusive)
        if not np.isfinite(v).all() or np.isnan(init) or np.isinf(init) or (v == 0).all():
            got = np.concatenate([X._values([o], pair) for o in outs]).view(np.float64)
            ref = X._values(S.prefix_sum(shards, S.OP_SUM_F64, pair, _init(init), inclusive), pair).view(np.float64)
            both_nan = np.isnan(got) & np.isnan(ref)
            nonfin = ~np.isfinite(ref) | (ref == 0)
            assert np.array_equal(got.view(np.uint64)[nonfin & ~both_nan], ref.view(np.uint64)[nonfin & ~both_nan])


# ---- several rounds of the tile-prefix kernel ------------------------------------------------------------------------------
@pytest.mark.parametrize("inclusive", [True, False])
@pytest.mark.parametrize("pair", [False, True])
def test_several_prefix_rounds_every_op(ctx, pair, inclusive):
    """more than 4096 tiles (16 777 217 8-byte items, 8 388 609 pairs): scan_prefix_kernel runs two rounds"""
    ib = 16 if pair else 8
    n = X.ROUND * X.tile_items(ib) + 1 + 12345
    assert X.rounds(n, ib) == 2
    for op in INT_OPS + [S.OP_SUM_F64]:
        items = make_items(n, 41 + op, op, pair)
        init = (5, (1 << 64) - 3) if op != S.OP_SUM_F64 else _init(-2.5)
        st, res = scan_dev(ctx, items, op, pair, init, inclusive)
        assert st == 0
        if op == S.OP_SUM_F64:
            if pair:
                assert np.array_equal(res["key"], S.prefix_sum([items], op, pair, init, inclusive)[0]["key"])
            r = X.check([res], [items], pair, init, inclusive)
            assert r.checked == n and r.depth == X.depth([n], ib)
            report("rounds=2 pair=%d incl=%d" % (pair, inclusive), r)
        else:
            assert np.array_equal(words(res), words(S.prefix_sum([items], op, pair, init, inclusive)[0])), op


@pytest.mark.parametrize("pair", [False, True])
def test_1e8_doubles(ctx, pair):
    """1e8 items of each size (13 or 25 rounds of the tile-prefix kernel) against the exact prefix sums"""
    import torch
    n = 100_000_000
    free, _ = torch.cuda.mem_get_info(0)
    if free < n * 16 * 3 + (2 << 30):
        pytest.skip("needs %.1f GB of device memory" % (n * 48 / 1e9 + 2))
    items = make_items(n, 5, S.OP_SUM_F64, pair)
    inclusive = not pair
    st, res = scan_dev(ctx, items, S.OP_SUM_F64, pair, _init(1e3), inclusive)
    assert st == 0
    if pair:
        assert res["key"][0] == 7 and np.array_equal(res["key"][1:], items["key"][:-1])
    r = X.check([res], [items], pair, _init(1e3), inclusive)
    assert r.checked == n
    report("1e8 pair=%d incl=%d" % (pair, inclusive), r)


# ---- outside the safe range ----------------------------------------------------------------------------------------------
def test_overflow_outside_the_safe_range_is_reproducible(ctx):
    """x[0] = -1e308, x[4096] = x[4097] = 1e308, the rest +0.0: the stock fold gives 1e308 from position 4097 on, while a
    partial sum of the kernels' bracketing may overflow (A = 2e308 there, past the safe range).  What is promised: the
    outputs inside the safe range (positions 0 .. 4095) are within the bound, and the outputs are the same bits on every run"""
    x = np.zeros(4096 + 64)
    x[0], x[4096], x[4097] = -1e308, 1e308, 1e308
    items = S.f64_words(x)
    st, a = scan_dev(ctx, items, S.OP_SUM_F64)
    st2, b = scan_dev(ctx, items, S.OP_SUM_F64)
    assert st == st2 == 0 and np.array_equal(a, b)
    res = X.check(a, [items], beyond="skip")
    assert res.checked == 4096
    g = a.view(np.float64)
    inf = np.flatnonzero(np.isinf(g))
    print("SCAN_F64_OVERFLOW first +inf at %s (the emulation: 4112); equal to the emulation: %s" % (
        int(inf[0]) if len(inf) else None, bool(np.array_equal(a, X.emulate([items])))))
