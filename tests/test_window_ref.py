"""CPU checks of the Window model (tests/window_ref.py) against the fixtures of the unmodified reference, and of the emulated
kernel bracketing of double sums against exact sums and the bound include/thrill_gpu.h states."""
import os

import numpy as np
import pytest

import scan_ref as S
import window_ref as W

FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_outputs_window.npz")
CASES = W.load_fixtures(FIXTURES)


def test_fixture_coverage():
    """every function and item type at every k, and the sizes N < k - 1, N = k - 1, N = k, N mod k = 0 and != 0 with N > k.
    One deliberate gap (tests/golden/make_golden_window.py): at k = 4096 the partial form, and the full form at N = 2k, are
    recorded for four functions only, to keep the file small; test_gpu_window.py covers every function there against the
    model."""
    forms = {c["form"] for c in CASES}
    ks = {c["k"] for c in CASES}
    assert forms == {W.FULL, W.PARTIAL, W.DISJOINT} and ks == {2, 3, 5, 64, 4096}
    fns = {(op, pr) for op in range(6) for pr in (False, True)}
    for k in ks:
        for form in (W.FULL, W.DISJOINT) if k == 4096 else (W.FULL, W.PARTIAL, W.DISJOINT):
            assert {(c["op"], c["pair"]) for c in CASES if c["k"] == k and c["form"] == form} == fns, (k, form)
        for fn in fns:
            ns = {len(c["items"]) for c in CASES if c["k"] == k and (c["op"], c["pair"]) == fn}
            assert {k - 1, k} <= ns and any(n < k - 1 for n in ns), (k, fn)
            assert any(n % k == 0 and n > k for n in ns) and any(n % k and n > k for n in ns), (k, fn)
    # a halo spanning two or more predecessors: some worker's k - 1 items before it lie on 2+ workers
    spans = 0
    for c in CASES:
        for p, sh in c["shards"].items():
            f = np.cumsum([0] + sh)
            for r in range(1, p):
                need = f[r] - max(0, f[r] - c["k"] + 1)
                held = [q for q in range(r) if sh[q] and f[q + 1] > f[r] - need]
                spans += len(held) >= 2
    assert spans > 100
    # NaN as a window's first item and elsewhere, +-0, infinities, u64 wraparound
    f64 = [c for c in CASES if c["op"] in W.F64_OPS]
    assert any(np.isnan(c["items"][:, 1].view(np.float64)).any() for c in f64)
    assert any(np.isinf(c["items"][:, 1].view(np.float64)).any() for c in f64)


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_model_matches_fixture(c):
    """the stock-fold model equals the reference's outputs bit for bit, and its per-worker counts at every worker count"""
    got = W.outputs(c["items"], c["op"], c["k"], c["form"])
    assert got.shape == c["out"].shape
    assert W.same(got, c["out"], c["op"]), c["name"]
    for p in W.WORKERS:
        assert W.counts(c["form"], c["k"], c["shards"][p]) == c["counts"][p], (c["name"], p)


def _nasty(n, seed):
    rng = np.random.RandomState(seed)
    x = rng.standard_normal(n) * 10.0 ** rng.randint(-300, 300, n)
    m = len(x[1::7])
    x[1::7] = -x[::7][:m]                           # cancellation
    x[3::11] = 5e-324
    x[5::13] = -0.0
    return S.f64_words(x)


@pytest.mark.parametrize("k", [2, 3, 5, 16, 17, 31, 32, 33, 64, 100, 257, 1025, 4095, 4096])
@pytest.mark.parametrize("form", [W.FULL, W.PARTIAL, W.DISJOINT])
def test_emulation_bound(k, form):
    """the emulated kernel sums stay within gamma_D A + u |exact| of the exact sums, D = min(k - 1, R + J - 1)"""
    n = 2 * k + 37 if k > 1000 else 5 * k + 7
    vals = _nasty(n, k * 3 + form)
    got = W.emulate_sum(vals, k, form)
    assert W.bound_violations(got, vals, k, form) == []


def test_depth():
    assert [W.depth(k) for k in (2, 16, 17, 64, 4095, 4096)] == [1, 15, 16, 19, 127, 127]


def test_emulation_equals_stock_where_exact():
    """small integers in doubles sum exactly in any bracketing: the emulation equals the stock left fold"""
    vals = S.f64_words(np.random.RandomState(5).randint(-1000, 1000, 3000).astype(np.float64))
    items = np.stack([np.zeros(3000, np.uint64), vals], axis=1)
    for k in (2, 5, 17, 64, 300, 2048):
        for form in (W.FULL, W.PARTIAL, W.DISJOINT):
            assert np.array_equal(W.emulate_sum(vals, k, form), W.outputs(items, W.OP_SUM_F64, k, form)[:, 1])


@pytest.mark.parametrize("k", [2, 5, 33, 64, 1000, 4096])
def test_emulation_independent_of_sharding(k):
    """each worker sees only its halo and its items; the concatenated outputs are the same bits for every sharding"""
    n = 3 * k + 11
    vals = _nasty(n, k)
    rng = np.random.RandomState(k)
    for form in (W.FULL, W.PARTIAL, W.DISJOINT):
        ref = W.emulate_sum(vals, k, form)
        for p in (2, 3, 7, 16):
            cuts = np.sort(rng.randint(0, n + 1, p - 1))
            sizes = list(np.diff(np.concatenate([[0], cuts, [n]])).astype(int))
            cnt = W.counts(form, k, sizes)
            off, f, parts = 0, 0, []
            for r in range(p):
                parts.append(W.emulate_worker_sum(vals, f, sizes[r], k, form)[off:off + cnt[r]])
                off += cnt[r]
                f += sizes[r]
            got = np.concatenate(parts)
            assert np.array_equal(got, ref), (form, p, sizes)
