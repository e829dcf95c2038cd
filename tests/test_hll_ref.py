"""The numpy model of the HyperLogLog action (hll_ref.py) against every stored result of the unmodified reference
(tests/golden/reference_outputs_hll.npz), bit for bit: SipHash-2-4 of 8- and 16-byte items and the dense register rule, with the
published SipHash known answers.  Also what the fixture says about the reference itself: the registers its natural path (sparse
start, operator + of the workers) ends with equal the directly inserted ones in every stored case.  CPU only."""
import os

import numpy as np
import pytest

import hll_ref as H

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "reference_outputs_hll.npz")


@pytest.fixture(scope="module")
def golden():
    return H.Golden(GOLDEN)


def test_siphash_known_answers():
    """the reference implementation's test vectors (key bytes 0..15, message bytes 0, 1, 2, ...), lengths 8 and 16"""
    m = np.array([0x0706050403020100, 0x0F0E0D0C0B0A0908], np.uint64)
    assert int(H.siphash24(m[:1], 8)[0]) == 0x93F5F5799A932462
    assert int(H.siphash24(m, 16)[0]) == 0x3F2ACC7F57C29BDB
    # vectorised: every item on its own
    many = np.concatenate([m, m[::-1], m])
    assert [int(x) for x in H.siphash24(many, 16)[[0, 2]]] == [0x3F2ACC7F57C29BDB] * 2
    assert int(H.siphash24(many, 8)[0]) == 0x93F5F5799A932462
    assert len(H.siphash24(np.zeros(0, np.uint64), 8)) == 0


def test_register_rule_on_examples():
    for p in range(4, 19):
        top = np.uint64(5) << np.uint64(64 - p)
        h = np.array([top,                                            # w == 0: the value is 64 - p + 1
                      top | np.uint64(1),                             # the lowest bit: clz = 63 - p
                      top | (np.uint64(1) << np.uint64(63 - p))],     # the bit right below the index: clz = 0
                     np.uint64)
        idx, val = H.index_value(h, p)
        assert list(idx) == [5, 5, 5] and list(val) == [65 - p, 64 - p, 1], p
    assert list(H.clz64(np.array([0, 1, 1 << 63, 1 << 31], np.uint64))) == [64, 63, 0, 32]


def test_fixture_covers_the_contract(golden):
    assert golden.precisions == [4, 8, 12, 14, 16, 18]
    modes = {golden.mode(i) for i in range(len(golden.names))}
    assert modes == {"u64", "pair", "hash"}
    sizes = {golden.n_items(i) for i in range(len(golden.names))}
    assert 0 in sizes and 1 in sizes and max(sizes) >= 200000
    workers = {len(c) for _, _, c in golden.layouts()}
    assert workers == {1, 2, 3, 4, 8}
    counts = [c for _, _, c in golden.layouts() if sum(c) > 100]
    assert any(c[0] == 0 for c in counts) and any(c[-1] == 0 for c in counts) and any(len(c) == 3 and c[1] == 0 for c in counts)
    # the stock path ends sparse in some cases and dense in others, at every precision
    d = golden.z["lay_dense"]
    assert d.min(axis=0).tolist() == [0] * 6 and d.max(axis=0).tolist() == [1] * 6


def test_model_equals_the_reference(golden):
    whole = 0
    for i, name in enumerate(golden.names):
        for p in golden.precisions:
            regs = golden.model_registers(i, p)
            stored = golden.regs(i, p)
            if stored is not None:
                whole += 1
                assert np.array_equal(regs, stored), (name, p, np.flatnonzero(regs != stored)[:5])
            assert np.array_equal(H.digest(regs), golden.digest(i, p)), (name, p)
    assert whole >= 40


def test_w_zero_hashes_are_in_the_fixture(golden):
    """hashes whose low 64 - p bits are all zero reach the reference through insert_hash (no item search finds one: the odds are
    2^(p - 64) per item), and the model gives the reference's registers for them (test_model_equals_the_reference)"""
    i = golden.names.index("hash_edges")
    h = golden.words(i)
    for p in golden.precisions:
        zero = h[(h << np.uint64(p)) == 0]
        assert len(zero) >= 6
        idx, val = H.index_value(zero, p)
        assert set(val.tolist()) == {65 - p}
        stored = golden.regs(i, p)
        assert stored is not None and all(stored[k] == 65 - p for k in idx)


def test_all_equal_items_fill_one_register(golden):
    for name in ("u64_all_equal", "pair_all_equal"):
        i = golden.names.index(name)
        for p in golden.precisions:
            assert np.count_nonzero(golden.regs(i, p)) == 1
    for name in ("u64_empty", "pair_empty"):
        i = golden.names.index(name)
        assert not any(golden.regs(i, p).any() for p in golden.precisions)


def test_natural_path_registers_equal_the_direct_ones(golden):
    """sparse start, operator + in rank order and the conversion to dense give the registers direct insertion gives, in every
    stored case: the GPU's dense registers are the stock node's registers whichever format it ends in"""
    assert golden.z["lay_equal"].all()


def test_sharding_does_not_change_the_registers(golden):
    i = golden.names.index("pair_range_3000")
    words = golden.words(i)
    for p in (4, 12, 18):
        want = golden.model_registers(i, p)
        for _, _, counts in golden.layouts(i):
            parts = [H.registers(s, 16, p) for s in H.shards_of(words, 16, counts)]
            assert np.array_equal(H.merge(parts), want)


def test_dense_estimates_are_near_the_distinct_count(golden):
    """est_a is the stock result() of the dense registers: within 3 standard errors (1.04 / sqrt(2^p)) of the distinct count"""
    for name, distinct in (("u64_range_200000", 200000), ("pair_range_150000", 150000), ("u64_range_3000", 3000)):
        i = golden.names.index(name)
        for k, p in enumerate(golden.precisions):
            assert abs(golden.z["est_a"][i, k] / distinct - 1) <= 3 * 1.04 / np.sqrt(1 << p), (name, p)
