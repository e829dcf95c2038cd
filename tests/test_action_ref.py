"""The numpy restatement of Sum / Min / Max / AllReduce (action_ref.py) against every stored result of the unmodified reference
(tests/golden/reference_outputs_action.npz), bit for bit, doubles and NaN bits included: the model folds left to right, as the
stock node does.  CPU only."""
import os

import numpy as np
import pytest

import action_ref as A

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "reference_outputs_action.npz")


@pytest.fixture(scope="module")
def golden():
    return A.Golden(GOLDEN)


def test_fixtures_cover_the_contract(golden):
    names = A.case_names(golden)
    modes = {A.Case(golden, n).mode for n in names}
    assert modes == set(A.MODES)
    for mode in A.MODES:
        inits = {A.Case(golden, n).initial is None for n in names if A.Case(golden, n).mode == mode}
        assert inits == {True, False}, mode
    ps = {p for n in names for p in A.Case(golden, n).ps}
    assert ps == {1, 2, 3, 4, 8}
    # empty workers: first, middle, last
    counts = [A.Case(golden, n).counts(8) for n in names]
    assert any(c[0] == 0 for c in counts) and any(c[-1] == 0 for c in counts) and any(c[4] == 0 and c[3] for c in counts)


def test_model_equals_the_reference(golden):
    for name in A.case_names(golden):
        case = A.Case(golden, name)
        for p in case.ps:
            assert equal(case.op, case.model(p), case.result(p)), (name, p, case.counts(p))


def equal(op, a, b):
    """two results (first, value) equal bit for bit; for double sums two NaNs are equal (a sum's NaN payload is left open: which
    operand's NaN an addition passes on is up to the compiler and the hardware)"""
    if op == A.OP_SUM_F64 and a[0] == b[0] and np.isnan(A._f(a[1])) and np.isnan(A._f(b[1])):
        return True
    return a == b


def fold_loop(op, start, words):
    v = int(start)
    for w in np.asarray(words, np.uint64).tolist():
        v = A.fn(op, v, w)
    return v


@pytest.mark.parametrize("op", range(6))
def test_fold_shortcuts_equal_the_loop(op):
    """fold's vectorised paths fold exactly as the item-by-item loop"""
    rng = np.random.RandomState(op)
    specials = A._w(np.nan), 0x7FF8000000000777, 0, 0x8000000000000000, A._w(np.inf), A._w(-np.inf)
    for trial in range(200):
        n = rng.randint(0, 40)
        if op in A.F64_OPS:
            w = A.S.f64_words(rng.standard_normal(n) * 10.0 ** rng.randint(-3, 4, n)) if n else np.zeros(0, np.uint64)
            for i in range(n):
                if rng.randint(0, 4) == 0:
                    w[i] = specials[rng.randint(0, len(specials))]
            start = specials[rng.randint(0, len(specials))] if rng.randint(0, 2) else int(A.S.f64_words([rng.standard_normal()])[0])
        else:
            w = rng.randint(0, 1 << 62, n, dtype=np.uint64) * np.uint64(rng.randint(1, 5))
            start = int(rng.randint(0, 1 << 62, dtype=np.uint64))
        a, b = A.fold(op, start, w), fold_loop(op, start, w)
        if op == A.OP_SUM_F64 and np.isnan(A._f(a)):       # a sum's NaN payload is left open
            assert np.isnan(A._f(b)), (trial, start, w)
        else:
            assert a == b, (trial, start, w)


def test_stock_rules_on_examples():
    nan, pay = A._w(np.nan), 0x7FF8000000012345
    one, two, pz, nz = A._w(1.0), A._w(2.0), 0, 0x8000000000000000
    # a NaN first item sticks, with its bits; a later NaN is skipped
    assert A.all_reduce([np.array([pay, one, two], np.uint64)], A.OP_MIN_F64) == (0, pay)
    assert A.all_reduce([np.array([two, pay, one], np.uint64)], A.OP_MIN_F64) == (0, one)
    # the earlier of two equal zeros
    assert A.all_reduce([np.array([one, nz, pz], np.uint64)], A.OP_MIN_F64) == (0, nz)
    assert A.all_reduce([np.array([one, pz, nz], np.uint64)], A.OP_MIN_F64) == (0, pz)
    # an empty worker contributes T(): +0.0 is the Min of positive doubles, 0 of uint64_t
    assert A.all_reduce([np.array([one], np.uint64), np.zeros(0, np.uint64)], A.OP_MIN_F64) == (0, pz)
    assert A.all_reduce([np.array([5, 7], np.uint64), np.zeros(0, np.uint64)], A.OP_MIN_U64) == (0, 0)
    # ... and with an initial value every empty worker contributes it; worker 0's NaN sticks
    assert A.all_reduce([np.zeros(0, np.uint64), np.array([one], np.uint64)], A.OP_MAX_F64, initial=(0, pay)) == (0, pay)
    assert A.all_reduce([np.array([5], np.uint64), np.zeros(0, np.uint64)], A.OP_SUM_U64, initial=(0, 2)) == (0, 9)
    # a NaN S_0 sticks in the fold of the workers; a later worker's NaN is skipped
    assert A.all_reduce([np.array([nan], np.uint64), np.array([one], np.uint64)], A.OP_MAX_F64) == (0, nan)
    assert A.all_reduce([np.array([one], np.uint64), np.array([pay], np.uint64)], A.OP_MAX_F64) == (0, one)
    # -0.0 only when every summand is -0.0; an empty worker's +0.0 is a summand
    assert A.all_reduce([np.array([nz, nz], np.uint64)], A.OP_SUM_F64) == (0, nz)
    assert A.all_reduce([np.array([nz, nz], np.uint64), np.zeros(0, np.uint64)], A.OP_SUM_F64) == (0, pz)
    # pairs: .first of the last worker's last item, 0 if that worker is empty
    kv = A.S.pairs([3, 4], [10, 20])
    assert A.all_reduce([kv], A.OP_SUM_U64, pair=True) == (4, 30)
    assert A.all_reduce([kv, kv[:0]], A.OP_SUM_U64, pair=True) == (0, 30)
    assert A.all_reduce([kv[:0]], A.OP_SUM_U64, pair=True, initial=(8, 1)) == (8, 1)
