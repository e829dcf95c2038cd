"""The numpy model of Sample / BernoulliSample (tests/sample_ref.py): against a scalar SplitMix64 loop, uniform over fixed seeds,
unrelated samples for the Python Context's successive seeds, and against the stock operators of the reference
(tests/golden/reference_outputs_sample.npz): the deterministic cases exactly, and the distributions of the frozen stock runs (the
Sample(4) subsets, the per-worker counts, the BernoulliSample counts) alike with the model's over fixed seeds.  No GPU."""
import itertools
import math
import os
import sys

import numpy as np
import pytest
from scipy import stats

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sample_ref as S  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_outputs_sample.npz")


def test_keys_match_scalar_splitmix():
    for seed in (0, 1, 42, (1 << 64) - 1, 0x9E3779B97F4A7C15, 123456789123456789):
        g = np.array([0, 1, 2, 3, 1000, (1 << 30) - 1, (1 << 34) + 5, (1 << 64) - 2], np.uint64)
        want = [S.key_int(seed, int(x)) for x in g]
        assert S.keys(seed, g).tolist() == want
    # mix(0) = 0, and the first SplitMix64 output of state 0 is the published e220a8397b1dcdaf
    assert S.mix_int(0) == 0
    assert S.mix_int(S.GAMMA) == 0xE220A8397B1DCDAF


def test_sample_exact_count_and_order():
    for N, s in ((0, 0), (0, 5), (1, 0), (1, 1), (5, 3), (4097, 4096), (10000, 10), (10000, 9999), (10000, 20000)):
        m = S.sample_mask(7, N, s)
        assert m.sum() == min(s, N)
        if 0 < s < N:
            k = S.keys(7, np.arange(N, dtype=np.uint64))
            assert k[m].max() < k[~m].min()
    shards = [np.arange(0, 3, dtype=np.uint64), np.arange(3, 3, dtype=np.uint64), np.arange(3, 40, dtype=np.uint64)]
    outs = S.sample(shards, 10, 5)
    assert sum(len(o) for o in outs) == 10
    for sh, o in zip(shards, outs):
        assert np.all(np.diff(o.astype(np.int64)) > 0) and np.isin(o, sh).all()


def test_bernoulli_threshold_edges():
    assert S.bernoulli_threshold(0.0) == 0
    assert S.bernoulli_threshold(1.0) == 1 << 53
    assert S.bernoulli_threshold(2.0 ** -53) == 1
    assert S.bernoulli_threshold(1 - 2.0 ** -53) == (1 << 53) - 1
    assert S.bernoulli_threshold(1e-6) == math.ceil(1e-6 * 2.0 ** 53)
    for bad in (float("nan"), -1e-300, 1.0000000000000002, float("inf")):
        with pytest.raises(ValueError):
            S.bernoulli_threshold(bad)
    assert not S.bernoulli_mask(3, 1000, 0.0).any() and S.bernoulli_mask(3, 1000, 1.0).all()


def test_sample_4_of_12_uniform_over_subsets():
    seeds = np.arange(99000, dtype=np.uint64) * np.uint64(0x2545F4914F6CDD1D) + np.uint64(17)
    sub = S.subsets_sample(seeds, 12, 4)
    index = {c: i for i, c in enumerate(itertools.combinations(range(12), 4))}
    counts = np.bincount([index[tuple(r)] for r in sub.tolist()], minlength=len(index))
    assert len(index) == 495
    _, pv = stats.chisquare(counts)
    assert pv > 1e-4, pv
    # every position is kept with probability 4/12
    incl = np.bincount(sub.reshape(-1), minlength=12)
    _, pv = stats.chisquare(incl)
    assert pv > 1e-4, pv


def test_bernoulli_counts_binomial():
    N, p, M = 64, 0.3, 20000
    seeds = np.arange(M, dtype=np.uint64) * np.uint64(0x9FB21C651E98DF25) + np.uint64(3)
    k = S.keys(seeds[:, None], np.arange(N, dtype=np.uint64)[None, :])
    kept = (k >> np.uint64(11)) < np.uint64(S.bernoulli_threshold(p))
    c = kept.sum(axis=1)
    lo, hi = 9, 29                                  # bins with at least ~5 expected; the tails pooled
    obs = np.array([(c <= lo).sum()] + [(c == x).sum() for x in range(lo + 1, hi)] + [(c >= hi).sum()])
    pmf = stats.binom(N, p)
    exp = np.array([pmf.cdf(lo)] + [pmf.pmf(x) for x in range(lo + 1, hi)] + [pmf.sf(hi - 1)]) * M
    _, pv = stats.chisquare(obs, exp)
    assert pv > 1e-4, pv
    incl = kept.sum(axis=0)
    _, pv = stats.chisquare(incl)
    assert pv > 1e-4, pv


def test_consecutive_context_seeds_unrelated():
    """The Python Context derives successive seeds as rng_seed + GAMMA * counter; with the outer mix(seed) the two samples are
    unrelated: the overlap of the kept positions after any shift is at chance level (without it, seed + GAMMA draws the key
    stream shifted by one position)."""
    N, p = 1 << 14, 0.5
    for rng_seed in (0, 1, 0xDEADBEEF):
        s1, s2 = (rng_seed + S.GAMMA) % (1 << 64), (rng_seed + 2 * S.GAMMA) % (1 << 64)
        a, b = S.bernoulli_mask(s1, N, p), S.bernoulli_mask(s2, N, p)
        for d in range(-64, 65):
            x, y = (a[d:], b[:N - d]) if d >= 0 else (a[:N + d], b[-d:])
            L = len(x)
            ov = int((x & y).sum())
            z = (ov - L * p * p) / math.sqrt(L * p * p * (1 - p * p))
            assert abs(z) < 6, (rng_seed, d, z)
        # what the test guards against: keys without the outer mix would coincide after a shift of one
        g = np.arange(100, dtype=np.uint64)
        with np.errstate(over="ignore"):
            raw1 = S.mix(np.uint64(s1) + (g + np.uint64(1)) * np.uint64(S.GAMMA))
            raw2 = S.mix(np.uint64(s2) + (g + np.uint64(1)) * np.uint64(S.GAMMA))
        assert np.array_equal(raw1[1:], raw2[:-1])


# ---- against the stock operators (tests/golden/reference_outputs_sample.npz, make_golden_sample.py) ---------------------------
def load_fixture():
    return np.load(GOLDEN)


def det_cases(z):
    """(sizes, mode, param, exact, per-worker stock outputs) of every deterministic case"""
    for c in range(len(z["det_workers"])):
        W = int(z["det_workers"][c])
        sizes = z["det_sizes"][c, :W].tolist()
        flat = z["det_items"][z["det_offsets"][c]:z["det_offsets"][c + 1]]
        cnt = z["det_counts"][c, :W]
        outs = np.split(flat, np.cumsum(cnt)[:-1])
        param = z["det_param"][c]
        yield sizes, int(z["det_mode"][c]), (param if z["det_mode"][c] else int(param)), bool(z["det_exact"][c]), outs


def test_fixture_deterministic_cases():
    z = load_fixture()
    n = 0
    for sizes, mode, param, exact, stock in det_cases(z):
        shards = np.split(np.arange(sum(sizes), dtype=np.int64), np.cumsum(sizes)[:-1])
        for seed in (0, 1, (1 << 64) - 1):
            model = S.bernoulli_sample(shards, param, seed) if mode else S.sample(shards, param, seed)
            if exact:
                assert all(np.array_equal(m, s) for m, s in zip(model, stock)), (sizes, mode, param)
            else:
                # one worker with s < n: the stock items are its reservoir's, the count is s
                assert len(sizes) == 1 and len(stock[0]) == len(model[0]) == param
                assert len(np.unique(stock[0])) == param and stock[0].max() < sizes[0]
        n += 1
    assert n == 21


def hypergeom_pmf(sizes, s):
    """the multivariate hypergeometric distribution of the per-worker counts of s draws from the shards: {counts: probability}"""
    from math import comb
    N = sum(sizes)
    out = {}
    for c in itertools.product(*[range(min(n, s) + 1) for n in sizes]):
        if sum(c) == s:
            out[c] = np.prod([comb(n, k) for n, k in zip(sizes, c)]) / comb(N, s)
    return out


def test_fixture_subsets_uniform():
    """the stock subsets of Sample(4) of 12 items and the model's (fixed seeds) are both consistent with uniform"""
    z = load_fixture()
    index = {c: i for i, c in enumerate(itertools.combinations(range(12), 4))}
    stock = np.bincount([index[tuple(r)] for r in z["sub_subsets"].tolist()], minlength=495)
    assert stock.sum() == 20000
    _, pv = stats.chisquare(stock)
    assert pv > 1e-4, pv
    seeds = np.arange(20000, dtype=np.uint64) * np.uint64(0xD1B54A32D192ED03) + np.uint64(99)
    model = np.bincount([index[tuple(r)] for r in S.subsets_sample(seeds, 12, 4).tolist()], minlength=495)
    _, pv = stats.chisquare(model)
    assert pv > 1e-4, pv


def test_fixture_worker_counts():
    """per sharding, the stock per-worker counts of Sample(4) and the model's have the same distribution: each against the
    multivariate hypergeometric, and the two against each other"""
    z = load_fixture()
    seeds = np.arange(5000, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(12345)
    sub = S.subsets_sample(seeds, 12, 4)
    for k in range(len(z["sub_sizes"])):
        sizes = z["sub_sizes"][k, :z["sub_workers"][k]].tolist()
        W = len(sizes)
        stock = z["sub_counts"][z["sub_config"] == k][:, :W].astype(np.int64)
        bounds = np.cumsum(sizes)
        model = np.stack([np.searchsorted(bounds, sub, side="right") == w for w in range(W)], axis=2).sum(axis=1)
        assert np.all(stock.sum(axis=1) == 4) and np.all(model.sum(axis=1) == 4)
        for w in range(W):
            assert np.all(stock[:, w] <= sizes[w]) and np.all(model[:, w] <= sizes[w])
        pmf = hypergeom_pmf(sizes, 4)
        keys = sorted(pmf)
        if len(keys) == 1:
            continue
        obs_s = np.array([np.sum(np.all(stock == np.array(c), axis=1)) for c in keys])
        obs_m = np.array([np.sum(np.all(model == np.array(c), axis=1)) for c in keys])
        exp = np.array([pmf[c] for c in keys])
        for obs in (obs_s, obs_m):
            assert obs.sum() == 5000
            _, pv = stats.chisquare(obs, exp * 5000)
            assert pv > 1e-4, (sizes, pv)
        keep = (obs_s + obs_m) > 0
        _, pv, _, _ = stats.chi2_contingency(np.stack([obs_s[keep], obs_m[keep]]))
        assert pv > 1e-4, (sizes, pv)


def test_fixture_bernoulli():
    """the stock BernoulliSample at p = 0.05 (skip path) and 0.3 (Bernoulli path) on 64 items and the model: counts against the
    binomial, every position kept at the same rate, and the two count distributions alike"""
    z = load_fixture()
    seeds = np.arange(5000, dtype=np.uint64) * np.uint64(0xBF58476D1CE4E5B9) + np.uint64(7)
    for b, p in enumerate(z["bern_p"]):
        stock = np.unpackbits(z["bern_masks"][b], axis=1, bitorder="little").astype(bool)
        k = S.keys(seeds[:, None], np.arange(64, dtype=np.uint64)[None, :])
        model = (k >> np.uint64(11)) < np.uint64(S.bernoulli_threshold(p))
        pmf = stats.binom(64, p)
        lo, hi = int(pmf.ppf(0.005)), int(pmf.isf(0.005))
        exp = np.array([pmf.cdf(lo)] + [pmf.pmf(x) for x in range(lo + 1, hi)] + [pmf.sf(hi - 1)]) * 5000
        hists = []
        for m in (stock, model):
            c = m.sum(axis=1)
            obs = np.array([(c <= lo).sum()] + [(c == x).sum() for x in range(lo + 1, hi)] + [(c >= hi).sum()])
            hists.append(obs)
            _, pv = stats.chisquare(obs, exp)
            assert pv > 1e-4, (p, pv)
            _, pv = stats.chisquare(m.sum(axis=0))
            assert pv > 1e-4, (p, pv)
        keep = (hists[0] + hists[1]) > 0
        _, pv, _, _ = stats.chi2_contingency(np.stack([hists[0][keep], hists[1][keep]]))
        assert pv > 1e-4, (p, pv)
