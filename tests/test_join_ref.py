"""The numpy restatement of InnerJoin (join_ref.py) against the definition (brute force over all pairs), the oracle's hash
partition, and the reference's outputs stored in tests/golden/reference_outputs_join.npz.  CPU only."""
import os

import numpy as np
import pytest

import join_ref as J

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "reference_outputs_join.npz")


def test_owner_matches_the_oracle_hash_partition(oracle):
    keys = np.concatenate([np.arange(5000, dtype=np.uint64), np.array([0, (1 << 64) - 1, 1 << 63], np.uint64),
                           np.random.RandomState(1).randint(0, 1 << 62, 5000, dtype=np.uint64) * np.uint64(3)])
    for p in (1, 2, 3, 4, 8, 16):
        assert np.array_equal(J.owner(keys, p), oracle.hash_partition_ids(keys, p).astype(np.int64))
    for k in (0, 1, 12345, (1 << 64) - 1):
        assert int(J.hash128to64(np.zeros(1, np.uint64), np.array([k], np.uint64))[0]) == oracle.hash128to64(0, k)


@pytest.mark.parametrize("fn", [J.KEY_VALUES, J.VALUES])
@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("shape", ["uniform", "one_key", "key0", "empty_left", "empty_right", "disjoint", "zipf"])
def test_model_against_brute_force(fn, p, shape):
    rng = np.random.RandomState(p * 7 + fn)
    if shape == "uniform":
        left, right = J.make_side(60, 20, 1), J.make_side(50, 20, 2)
    elif shape == "one_key":
        left, right = J.make_side(30, 1, 3), J.make_side(25, 1, 4)
    elif shape == "key0":
        left, right = J.make_side(40, 3, 5), J.make_side(40, 3, 6)
        assert (left["key"] == 0).any() and (right["key"] == 0).any()
    elif shape == "empty_left":
        left, right = J.make_side(0, 5, 7), J.make_side(30, 5, 8)
    elif shape == "empty_right":
        left, right = J.make_side(30, 5, 9), J.make_side(0, 5, 10)
    elif shape == "disjoint":
        left, right = J.make_side(40, 100, 11), J.make_side(40, 100, 12)
        right["key"] += np.uint64(1000)
    else:
        left, right = J.make_side(70, 30, 13, zipf=1.0), J.make_side(60, 30, 14, zipf=1.0)
    rng.shuffle(left)
    lefts, rights = J.split_shards(left, p), J.split_shards(right, p)
    got = J.join(lefts, rights, fn)
    want = J.brute_force(lefts, rights, fn, p)
    for d in range(p):
        assert np.array_equal(got[d].view(np.uint64), want[d].view(np.uint64))
    assert sum(len(g) for g in got) == J.output_counts(left, right)


def test_size_verdict():
    small = J.make_side(10, 3, 1)
    assert not J.too_large([small], [small])
    # 40 000 x 30 000 on one key: over the output limit on the one worker that owns the key, whatever p is
    a, b = np.zeros(40000, J.KV), np.zeros(30000, J.KV)
    a["key"], b["key"] = 5, 5
    for p in (1, 2, 4):
        assert J.too_large(J.split_shards(a, p), J.split_shards(b, p))
    # 32 768 x 32 767 is below it
    assert not J.too_large([a[:32768]], [b[:30000]])
    assert J.output_counts(np.zeros(32768, J.KV), np.zeros(32767, J.KV)) == (1 << 30) - 32768


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/reference_outputs_join.npz is not present")
    return np.load(GOLDEN)


def test_model_multisets_equal_the_reference_outputs():
    """every stored shape: the reference's output multiset (sorted rows, or a digest of them) at 1 and at 2+ workers equals the
    model's union over the workers"""
    g = _golden()
    names = sorted({k.split("/")[0] for k in g.files})
    assert names
    for name in names:
        left, right = g[name + "/left"].view(J.KV), g[name + "/right"].view(J.KV)
        for key in [k for k in g.files if k.startswith(name + "/out_p")]:
            p = int(key.rsplit("_p", 1)[1])
            outs = J.join(J.split_shards(left, p), J.split_shards(right, p), J.KEY_VALUES)
            rows = np.concatenate(outs).view(np.uint64).reshape(-1, 3)
            rows = rows[np.lexsort(rows.T[::-1])]
            ref = g[key]
            if ref.dtype == np.uint8:          # a digest of the sorted rows (the larger shapes)
                import hashlib
                assert hashlib.sha256(np.ascontiguousarray(rows).tobytes()).digest() == ref.tobytes(), key
            else:
                assert np.array_equal(rows, ref.reshape(-1, 3)), key
