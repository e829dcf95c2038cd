"""The O(n) references of tests/large_ref.py on the CPU: the mixer is a bijection, every generator and checker agrees with
the plain references (sort_ref, reduce_ref) and the oracle at small n, and every checker rejects known-wrong outputs,
including a defect that sits exactly on a chunk boundary."""
import numpy as np
import pytest

import large_ref as L
import oracle_lib as O
import reduce_ref as RR
import sort_ref as R


@pytest.mark.parametrize("bits", [16, 24, 56, 64])
def test_mixer_round_trips(bits):
    rng = np.random.default_rng(bits)
    top = (1 << bits) - 1
    x = np.r_[np.array([0, 1, 2, top, top - 1, 1 << (bits - 1)], dtype=np.uint64),
              rng.integers(0, top, size=100000, dtype=np.uint64, endpoint=True)]
    y = L.mix(x, bits)
    assert np.all(y <= np.uint64(top))
    assert np.array_equal(L.unmix(y, bits), x)
    assert np.array_equal(L.mix(L.unmix(x, bits), bits), x)
    if bits == 16:                                  # a bijection of all 2^16 words
        assert len(np.unique(L.mix(np.arange(1 << 16, dtype=np.uint64), 16))) == 1 << 16


def _feed(chk, out, chunk):
    for a in range(0, len(out), chunk):
        chk.feed(out[a:a + chunk])
    chk.finish()


def _input(case):
    return case.items(0, case.n)


SORT_CASES = [L.SortCase(5000, 8), L.SortCase(5000, 8, descending=True), L.SortCase(4099, 8, m=5),
              L.SortCase(3001, 8, m=64, bits=24), L.SortCase(3001, 8, bits=56, top=0x40, odd=3000),
              L.SortCase(5000, 16), L.SortCase(5001, 16, m=3), L.SortCase(5001, 16, m=3, descending=True)]


@pytest.mark.parametrize("case", SORT_CASES, ids=lambda c: "i%d_n%d_m%d_b%d%s%s" % (
    c.item_bytes, c.n, c.m, c.bits, "_odd" if c.odd is not None else "", "_desc" if c.descending else ""))
@pytest.mark.parametrize("chunk", [1, 7, 1024, 1 << 20])
def test_sort_checker_accepts_reference(oracle, case, chunk):
    items = _input(case)
    d = case.desc()
    ref = R.sort(items, d)
    if not d.descending:
        assert np.array_equal(O.sort_items(items, d.oracle()).view(np.uint8).reshape(ref.shape), ref)
    _feed(case.checker(), ref.view(np.uint64).reshape(case.n, -1), chunk)
    if case.odd is not None:                        # one key outside the bucket of all the others
        tops = R.sort(items, d).view(np.uint64).reshape(-1) >> np.uint64(56)
        assert np.count_nonzero(tops != tops[0]) == 1


def _sorted(case):
    return R.sort(_input(case), case.desc()).view(np.uint64).reshape(case.n, -1).copy()


def _rejects(case, out, chunk, match):
    with pytest.raises(AssertionError, match=match):
        _feed(case.checker(), out, chunk)


@pytest.mark.parametrize("chunk", [1, 100, 4096])
def test_sort_checker_rejects(chunk):
    c16 = L.SortCase(5001, 16, m=3)
    good = _sorted(c16)
    eq = int(np.flatnonzero(good[1:, 0] == good[:-1, 0])[0])
    bad = good.copy()
    bad[[eq, eq + 1]] = bad[[eq + 1, eq]]                           # two equal-key items swapped
    _rejects(c16, bad, chunk, "input order")
    _rejects(c16, np.delete(good, 77, axis=0), chunk, "items, expected|does not belong|input order")     # one dropped
    _rejects(c16, np.insert(good, 78, good[77], axis=0), chunk, "input order")                          # one duplicated
    bad = good.copy()
    bad[10, 1] += np.uint64(3 * c16.J)                              # a value of the same group that is not in the input
    _rejects(c16, bad, chunk, "does not belong")
    bad = good.copy()
    bad[[10, 4000]] = bad[[4000, 10]]                               # out of order
    _rejects(c16, bad, chunk, "follows")
    c8 = L.SortCase(5000, 8)
    good = _sorted(c8)
    _rejects(c8, np.delete(good, 5, axis=0), chunk, "has 4999 items")
    _rejects(c8, np.insert(good, 6, good[5], axis=0), chunk, "follows")
    bad = good.copy()
    bad[9] = L.mix(np.array([5000], np.uint64))[0]                  # the key of a group that does not exist
    _rejects(c8, bad, chunk, "not the key of any group")
    cm = L.SortCase(4099, 8, m=5)
    good = _sorted(cm)
    _rejects(cm, np.delete(good, 2000, axis=0), chunk, "items with key|has 4098")
    _rejects(cm, np.insert(good, 2000, good[2000], axis=0), chunk, "items with key")


@pytest.mark.parametrize("case", [L.SortCase(4096, 16, m=2), L.SortCase(4096, 8, m=4)], ids=["i16", "i8"])
def test_sort_checker_rejects_defect_on_chunk_boundary(case):
    """chunks of 1023 items: a defect between the last item of a chunk and the first of the next"""
    good = _sorted(case)
    b = 1023
    assert good[b - 1, 0] == good[b, 0]                             # an equal-key pair straddles the boundary
    bad = good.copy()
    if case.item_bytes == 16:
        bad[[b - 1, b]] = bad[[b, b - 1]]
        _rejects(case, bad, 1023, "input order")
    else:
        _rejects(case, np.delete(good, b, axis=0), 1023, "items with key")
    bad = good.copy()
    bad[b] = good[b + case.m]                                       # the next key early: order broken at the boundary
    _rejects(case, bad, 1023, "follows|items with key|does not belong|input order")
    _feed(case.checker(), good, 1023)


REC_CASES = [L.RecordCase(3000, m=1), L.RecordCase(3001, m=2), L.RecordCase(3001, m=2, key_offset=90),
             L.RecordCase(2000, m=3, item_bytes=20, key_offset=5)]


@pytest.mark.parametrize("case", REC_CASES, ids=lambda c: "r%d_%d_m%d_n%d" % (c.item_bytes, c.key_offset, c.m, c.n))
def test_record_checker_accepts_reference(oracle, case):
    items = _input(case)
    assert np.array_equal(items[5, [b for b in range(case.item_bytes) if b in case.body_cols][:8]].view("<u8"), [5])
    ref = R.sort(items, case.desc())
    if case.key_offset == 0 and case.item_bytes == 100:
        assert np.array_equal(O.sort_items(items, O.RECORD_DESC).reshape(ref.shape), ref)
    for chunk in (1, 64, 1 << 20):
        _feed(case.checker(), ref, chunk)


@pytest.mark.parametrize("chunk", [1, 64, 1000])
def test_record_checker_rejects(chunk):
    case = L.RecordCase(3001, m=2)
    good = R.sort(_input(case), case.desc())
    bad = good.copy()
    bad[1500, 57] ^= 1                                              # one value byte of one record flipped
    _rejects(case, bad, chunk, "not those of input record")
    bad = good.copy()
    bad[999, case.key_offset + 9] ^= 1                              # one key byte, on a chunk boundary of 1000
    _rejects(case, bad, chunk, "not those of input record")
    eq = int(np.flatnonzero(np.all(good[1:, :10] == good[:-1, :10], axis=1))[0])
    bad = good.copy()
    bad[[eq, eq + 1]] = bad[[eq + 1, eq]]
    _rejects(case, bad, chunk, "out of order")
    _rejects(case, np.delete(good, 3, axis=0), chunk, "has 3000 records")
    _rejects(case, np.insert(good, 3, good[3], axis=0), chunk, "out of order")
    _rejects(case, good[::-1], chunk, "out of order")


RED_CASES = [L.ReduceCase(20000, "distinct"), L.ReduceCase(20001, "groups"), L.ReduceCase(20001, "groups", D=7),
             L.ReduceCase(20000, "skewed"), L.ReduceCase(20017, "skewed"), L.ReduceCase(10, "skewed")]
CLOSED_OPS = [O.OP_SUM_F64, O.OP_SUM_U64, O.OP_MIN_U64, O.OP_MAX_U64, O.OP_FIRST]


def _kv(w):
    kv = np.zeros(len(w), dtype=O.KV)
    kv["key"], kv["val"] = w[:, 0], w[:, 1]
    return kv


@pytest.mark.parametrize("op", CLOSED_OPS, ids=lambda op: RR.OPS[op])
@pytest.mark.parametrize("case", RED_CASES, ids=lambda c: "%s_n%d_D%d" % (c.dist, c.n, c.D))
def test_reduce_checker_accepts_reference(oracle, case, op):
    inp = _kv(case.items(0, case.n, op))
    out = O.reduce_simple(inp, op)
    RR.check(inp, out, op, exact=True)
    assert len(out) == case.num_groups
    rng = np.random.default_rng(op)
    out = out[rng.permutation(len(out))]                          # the table order of the GPU is arbitrary
    w = np.stack([out["key"], out["val"]], axis=1)
    for chunk in (1, 333, 1 << 20):
        _feed(case.checker(op), w, chunk)


def test_reduce_zero_key_and_exact_f64():
    case = L.ReduceCase(1 << 20, "skewed")
    assert L.mix(np.zeros(1, np.uint64))[0] == 0                    # group 0 has the key 0
    s, stride, cnt = case.progression(np.arange(L.HOT, dtype=np.uint64))
    sums = cnt * s + stride * (cnt * (cnt - np.uint64(1)) // np.uint64(2))
    assert np.all(sums.astype(np.float64).astype(np.uint64) == sums)
    big = L.ReduceCase((1 << 28), "skewed")
    s, stride, cnt = big.progression(np.arange(L.HOT, dtype=np.uint64))
    assert float(np.max(cnt * (s + (cnt - np.uint64(1)) * stride))) < 2.0 ** 53      # every partial sum is exact


@pytest.mark.parametrize("chunk", [1, 50, 4096])
def test_reduce_checker_rejects(oracle, chunk):
    case = L.ReduceCase(3000, "groups", D=100)
    for op in CLOSED_OPS:
        out = O.reduce_simple(_kv(case.items(0, case.n, op)), op)
        good = np.stack([out["key"], out["val"]], axis=1)
        _feed(case.checker(op), good, chunk)
        if op != O.OP_FIRST:
            bad = good.copy()
            bad[50, 1] += np.uint64(1)                              # one result off by one (on a chunk boundary of 50)
            _rejects_reduce(case, op, bad, chunk, "expected")
        else:
            bad = good.copy()
            bad[50, 1] += np.uint64(1)                              # a value of another group
            _rejects_reduce(case, op, bad, chunk, "not a value")
        _rejects_reduce(case, op, np.delete(good, 49, axis=0), chunk, "distinct keys")          # a key missing
        _rejects_reduce(case, op, np.insert(good, 50, good[49], axis=0), chunk, "distinct keys")  # a key twice
        bad = good.copy()
        bad[0, 0] = L.mix(np.array([100], np.uint64))[0]            # a key that is not in the input
        _rejects_reduce(case, op, bad, chunk, "not an input key")
    skew = L.ReduceCase(20000, "skewed")
    out = O.reduce_simple(_kv(skew.items(0, skew.n, 1)), 1)
    good = np.stack([out["key"], out["val"]], axis=1)
    bad = good.copy()
    bad[0, 0] = L.mix(np.array([L.HOT + 1], np.uint64))[0]         # a tail group whose record is a hot one
    _rejects_reduce(skew, 1, bad, chunk, "not an input key")


def _rejects_reduce(case, op, out, chunk, match):
    with pytest.raises(AssertionError, match=match):
        _feed(case.checker(op), out, chunk)


@pytest.mark.parametrize("op", [O.OP_SUM_U64, O.OP_MIN_U64, O.OP_MAX_U64])
@pytest.mark.parametrize("S,D,r", [(1000, 2, 3), (1000, 1000, 1), (100003, 777, 4)])
def test_index_case_against_oracle(oracle, S, D, r, op):
    case = L.IndexCase(S, D, r)
    inp = _kv(case.items(0, case.n))
    assert case.idx[0] == 0 and case.idx[-1] == S - 1 and len(np.unique(case.idx)) == D
    dense = O.reduce_to_index(inp, S, op, neutral=case.neutral)
    RR.to_index_check(inp, dense, S, op, neutral=case.neutral, exact=True)
    w = np.stack([dense["key"], dense["val"]], axis=1)
    for chunk in (1, 97, S):
        for a in range(0, S, chunk):
            case.check_slots(a, w[a:a + chunk], op)
    bad = w.copy()
    bad[case.idx[D // 2], 1] += np.uint64(1)
    with pytest.raises(AssertionError, match="expected"):
        case.check_slots(0, bad, op)
    empty = int(np.setdiff1d(np.arange(S), case.idx)[0]) if D < S else None
    if empty is not None:
        bad = w.copy()
        bad[empty, 1] = 0
        with pytest.raises(AssertionError, match="has no record"):
            case.check_slots(0, bad, op)
