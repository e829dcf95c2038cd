"""The split arithmetic of Merge (tg_merge_plan, pure host code) against the numpy restatement in merge_ref.py: the global
order (key, input, position), worker d receiving the merged ranks [ceil(d * N / p), ceil((d + 1) * N / p))."""
import ctypes as C

import numpy as np
import pytest

import merge_ref as M
from gpu_util import u64p
from sort_ref import Desc, LE
from thrill_b200 import capi

TG_ERR_ARG = -3
U64 = Desc(8, 0, 8, LE)


def plan(p, k, t, less, equal):
    out = np.zeros(p * k * (p + 1), np.uint64)
    st = capi.lib().tg_merge_plan(p, k, u64p(np.ascontiguousarray(t, np.uint64)), u64p(np.ascontiguousarray(less, np.uint64)),
                                  u64p(np.ascontiguousarray(equal, np.uint64)), u64p(out))
    return st, out


def inputs_of(kind, k, rng):
    """k sorted u64 inputs of up to ~120 items"""
    out = []
    for j in range(k):
        n = int(rng.randint(0, 120))
        if kind == "uniform":
            x = rng.randint(0, 1 << 62, size=n).astype(np.uint64)
        elif kind == "equal":
            x = np.full(n, 7, np.uint64)
        elif kind == "four":
            x = rng.choice(np.array([3, 9, 1 << 40, (1 << 64) - 1], np.uint64), size=n)
        elif kind == "empty":
            x = rng.randint(0, 50, size=n if j % 2 else 0).astype(np.uint64)
        elif kind == "tiny":             # N < p
            x = rng.randint(0, 3, size=1 if j == 0 else 0).astype(np.uint64)
        out.append(np.sort(x))
    return out


@pytest.mark.parametrize("kind,shape", [("uniform", "random"), ("uniform", "even"), ("equal", "random"), ("four", "random"),
                                        ("four", "gaps"), ("empty", "random"), ("uniform", "one"), ("four", "one"),
                                        ("tiny", "random")])
@pytest.mark.parametrize("k", [2, 3, 4, 16])
@pytest.mark.parametrize("p", [1, 2, 3, 8, 16])
def test_plan_matches_restatement(p, k, kind, shape):
    rng = np.random.RandomState(1000 * p + 10 * k + len(kind) + len(shape))
    for _ in range(3):
        runs = M.make_runs(inputs_of(kind, k, rng), p, rng, shape)
        t, less, equal = M.counts(runs, p, k, U64)
        st, out = plan(p, k, t, less, equal)
        assert st == 0
        ref = M.bounds(runs, p, k, U64)
        assert np.array_equal(out, ref)
        # every worker gets its exact share, pieces are contiguous and cover each run
        b = out.reshape(p * k, p + 1).astype(np.int64)
        assert np.all(np.diff(b, axis=1) >= 0)
        assert np.array_equal(b[:, p], [len(r) for r in runs]) and np.all(b[:, 0] == 0)
        assert np.array_equal(b.sum(axis=0), t.astype(np.int64))


def test_restatement_order_is_key_input_position():
    # input 0 = [1, 2, 2], input 1 = [2, 3] on one worker: the 2 of input 0 come before the 2 of input 1
    a = np.array([1 | (0 << 8), 2 | (1 << 8), 2 | (2 << 8)], np.uint64)
    b = np.array([2 | (3 << 8), 3 | (4 << 8)], np.uint64)
    d = Desc(8, 0, 1, LE)
    out = M.merged([a, b], 1, 2, d).view(np.uint64).reshape(-1)
    assert list(out >> np.uint64(8)) == [0, 1, 2, 3, 4]
    # two workers, k = 2, one item 5 in every run: ranks 0..3 are input 0 (w0, w1), then input 1 (w0, w1), so worker 0 gets
    # both items of input 0; runs listed (w0, j0), (w0, j1), (w1, j0), (w1, j1)
    runs = [np.array([5], np.uint64)] * 4
    assert list(M.bounds(runs, 2, 2, U64)) == [0, 1, 1, 0, 0, 1, 0, 1, 1, 0, 0, 1]


def test_inconsistent_counts_are_rejected():
    rng = np.random.RandomState(3)
    p, k = 3, 2
    runs = M.make_runs(inputs_of("four", k, rng), p, rng)
    t, less, equal = M.counts(runs, p, k, U64)
    assert plan(p, k, t, less, equal)[0] == 0
    bad_t = t.copy(); bad_t[1], bad_t[2] = bad_t[2] + 1, bad_t[1]                   # decreasing targets
    assert plan(p, k, bad_t, less, equal)[0] == TG_ERR_ARG
    big_t = t.copy(); big_t[p] += 1                                                    # a target beyond less + equal
    assert plan(p, k, big_t, less, equal)[0] == TG_ERR_ARG
    more = less.copy(); more[p + 1] += int(t[1]) + 1                                   # less above the target
    assert plan(p, k, t, more, equal)[0] == TG_ERR_ARG
    # bounds of a run that would go backwards in d
    nz = np.zeros(p * k * (p + 1), np.uint64)
    back_l = nz.copy(); back_l[1] = back_l[3] = 2                                      # run 0: 2 items below K_1 and K_3 ...
    back_l[(p + 1) + 2] = 2                                                            # ... none below K_2
    back_t = np.array([0, 2, 2, 2], np.uint64)
    assert plan(p, k, back_t, back_l, nz)[0] == TG_ERR_ARG
    for args in ((0, k), (17, k), (p, 0), (p, 17)):
        assert capi.lib().tg_merge_plan(args[0], args[1], u64p(t), u64p(less), u64p(equal),
                                        u64p(np.zeros(4096, np.uint64))) == TG_ERR_ARG
    assert capi.lib().tg_merge_plan(p, k, None, u64p(less), u64p(equal), u64p(nz)) == TG_ERR_ARG
