"""The plain reduce reference of tests/reduce_ref.py on the CPU: its hash inverse against the oracle's Hash128to64, its
contract check against the oracle's straightforward aggregate, and outputs it must reject."""
import numpy as np
import pytest

import oracle_lib as O
import reduce_ref as RR


def test_hash_and_inverse_against_oracle(oracle):
    rng = np.random.default_rng(1)
    keys = np.r_[np.array([1, 2, 0xFFFFFFFFFFFFFFFF, 1 << 63], dtype=np.uint64),
                 rng.integers(0, RR.M64, size=200, dtype=np.uint64, endpoint=True)]
    h = RR.hash64(keys)
    assert [int(x) for x in h] == [O.hash128to64(0, int(k)) for k in keys]
    assert np.array_equal(RR.unhash64(h), keys)
    assert RR.hash64(np.zeros(1, np.uint64))[0] == 0


@pytest.mark.parametrize("bits", [{(24, 16): 0xBEEF}, {(40, 12): 4095}, {(52, 12): 4095}, {(48, 16): 0xFFFF},
                                  {(24, 16): 77, (40, 10): 5}])
def test_keys_with_hash_fields(oracle, bits):
    keys = RR.keys_with_hash(3000, bits, seed=len(bits))
    assert len(np.unique(keys)) == 3000 and np.all(keys != 0)
    h = RR.hash64(keys)
    for (shift, width), val in bits.items():
        assert np.all((h >> np.uint64(shift)) & np.uint64((1 << width) - 1) == np.uint64(val))
    assert int(h[0]) == O.hash128to64(0, int(keys[0]))


def _kv(keys, vals):
    kv = np.zeros(len(keys), dtype=O.KV)
    kv["key"], kv["val"] = keys, vals
    return kv


@pytest.mark.parametrize("op", RR.OPS)
@pytest.mark.parametrize("n", [1, 2, 33, 5000, 200003])
def test_check_accepts_oracle(oracle, op, n):
    """the oracle folds each key left to right from its first record: a result of the contract where no key mixes NaN with
    numbers.  The f64_wide mix has NaN (and ±inf) only on keys that carry one special value alone (gen_values), where the
    oracle returns that value's bit pattern."""
    rng = np.random.default_rng(n)
    keys = rng.integers(0, max(2, n // 5), size=n).astype(np.uint64)
    for mix in ("u64",) if op.endswith("u64") else ("f64_exact", "f64_wide", "u64"):
        if op.endswith("f64") and mix == "u64":
            continue
        kv = _kv(keys, RR.gen_values(mix, keys, n + 1))
        RR.check(kv, O.reduce_simple(kv, RR.OPS.index(op)), op, exact=(mix == "f64_exact" and op == "sum_f64"))


def test_check_rejects_wrong_outputs(oracle):
    m0, nan = np.uint64(0x8000000000000000), np.uint64(0x7FF0000000000001)
    f = lambda *x: np.array(x, dtype=np.float64).view(np.uint64)
    kv = _kv(np.array([3, 3, 5, 9, 9, 9, 0], np.uint64), np.r_[[m0, m0, m0], f(1.0, 1e-12, 2.0, 4.0)])
    good = RR.check
    good(kv, _kv([0, 3, 5, 9], np.r_[f(4.0), [m0, m0], f(3.000000000001)]), "sum_f64")
    with pytest.raises(AssertionError, match="not -0.0"):          # all -0.0 (twice, and once) summed from +0.0
        RR.check(kv, _kv([0, 3, 5, 9], np.r_[f(4.0, 0.0), [m0], f(3.000000000001)]), "sum_f64")
    with pytest.raises(AssertionError, match="not -0.0"):
        RR.check(kv, _kv([0, 3, 5, 9], np.r_[f(4.0), [m0], f(0.0, 3.000000000001)]), "sum_f64")
    with pytest.raises(AssertionError, match="within"):            # a 1e-12 record dropped
        RR.check(kv, _kv([0, 3, 5, 9], np.r_[f(4.0), [m0, m0], f(3.0)]), "sum_f64")
    kn = _kv(np.array([4, 4, 6, 8, 8], np.uint64), np.r_[[nan, nan, nan], f(-1.0, 2.0)])
    RR.check(kn, _kv([4, 6, 8], np.r_[[nan, nan], f(-1.0)]), "min_f64")
    for bad in (f(np.inf, np.inf, -1.0), f(np.nan, np.nan, -1.0)):    # +inf for NaN keys; a NaN not from the input
        with pytest.raises(AssertionError):
            RR.check(kn, _kv([4, 6, 8], bad), "min_f64")
    with pytest.raises(AssertionError, match="NaN where"):          # a NaN won over a number
        RR.check(_kv(np.array([4, 4], np.uint64), np.r_[[nan], f(1.0)]), _kv([4], [nan]), "max_f64")
    RR.check(kv, _kv([0, 3, 5, 9], np.r_[f(4.0), [m0, m0], f(2.0)]), "first")
    with pytest.raises(AssertionError, match="not one of the key's values"):
        RR.check(kv, _kv([0, 3, 5, 9], np.r_[f(4.0), [m0, m0], f(4.0)]), "first")
    with pytest.raises(AssertionError, match="missing"):
        RR.check(kv, _kv([3, 5, 9], np.r_[[m0, m0], f(2.0)]), "first")
    with pytest.raises(AssertionError, match="duplicated"):
        RR.check(kv, _kv([0, 3, 5, 9, 9], np.r_[f(4.0), [m0, m0], f(2.0, 2.0)]), "first")
    with pytest.raises(AssertionError, match="sum mod"):
        RR.check(_kv(np.array([1, 1], np.uint64), [RR.M64, 2]), _kv([1], [RR.M64]), "sum_u64")
    RR.check(_kv(np.array([1, 1], np.uint64), [RR.M64, 2]), _kv([1], [1]), "sum_u64")


def test_to_index_check(oracle):
    kv = _kv(np.array([0, 0, 3], np.uint64), [5, 6, 7])
    RR.to_index_check(kv, O.reduce_to_index(kv, 5, O.OP_SUM_U64, neutral=(9, 1)), 5, "sum_u64", neutral=(9, 1))
    out = O.reduce_to_index(kv, 5, O.OP_SUM_U64, neutral=(9, 1))
    out["val"][2] = 0
    with pytest.raises(AssertionError, match="has no record"):
        RR.to_index_check(kv, out, 5, "sum_u64", neutral=(9, 1))
