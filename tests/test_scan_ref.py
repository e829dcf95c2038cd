"""The numpy restatement of PrefixSum / ExPrefixSum / ZipWithIndex (scan_ref.py) against the reference's outputs stored in
tests/golden/reference_outputs_scan.npz: every case at every worker count, bit for bit (doubles included: the model folds left to
right as the stock node does; only a NaN's payload is left open), plus the contract's corner cases on their own.  CPU only."""
import os

import numpy as np
import pytest

import scan_ref as S

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "reference_outputs_scan.npz")


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/reference_outputs_scan.npz is not present")
    return np.load(GOLDEN)


def test_the_fixture_covers_every_mode_and_worker_count():
    g = _golden()
    cases = [S.Case(g, n) for n in S.case_names(g)]
    assert {c.mode for c in cases} == set(S.MODES)
    assert all(c.ps == [1, 2, 3, 4, 8] for c in cases)
    assert {c.inclusive for c in cases if c.op is not None} == {True, False}
    # an empty worker, and one worker holding everything
    assert any(0 in c.counts(8) and c.counts(8).count(0) == 1 for c in cases)
    assert any(c.counts(8).count(0) == 7 for c in cases)


@pytest.mark.parametrize("p", [1, 2, 3, 4, 8])
def test_model_equals_the_reference_outputs(p):
    g = _golden()
    checked = 0
    for name in S.case_names(g):
        c = S.Case(g, name)
        rows = S.as_rows(c.model(p))
        assert S.rows_equal(rows, c.rows(p), c.op == S.OP_SUM_F64), (name, p)
        checked += 1
    assert checked >= 20


def test_min_absorbs_on_workers_after_the_first():
    """T() = 0 is folded into every local total: with MinU64 every output of a worker r >= 1 is 0"""
    outs = S.prefix_sum([np.array([5, 3], np.uint64), np.array([9, 8], np.uint64)], "min_u64", initial=(0, (1 << 64) - 1))
    assert outs[0].tolist() == [5, 3] and outs[1].tolist() == [0, 0]


def test_pair_carry_first_comes_from_the_previous_worker():
    sh = [S.pairs([4, 6], [1, 2]), S.pairs([], []), S.pairs([8], [0])]
    outs = S.prefix_sum(sh, "max_u64", pair=True, initial=(99, 0), inclusive=False)
    assert outs[0]["key"].tolist() == [99, 4] and outs[2]["key"].tolist() == [0]      # the empty worker's S is T() = (0, 0)
    assert outs[2]["val"].tolist() == [2]


def test_negative_zero_needs_every_summand_negative():
    nz = S.f64_words([-0.0, -0.0])
    o = S.prefix_sum([nz, nz], "sum_f64", initial=(0, 0x8000000000000000))
    assert o[0].tolist() == [0x8000000000000000] * 2      # worker 0 starts from -0.0
    assert o[1].tolist() == [0, 0]                         # S_0 = +0.0 + -0.0 + -0.0 = +0.0
