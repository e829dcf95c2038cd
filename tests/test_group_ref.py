"""The numpy restatement of GroupByKey / GroupToIndex (group_ref.py) against the reference's outputs stored in
tests/golden/reference_outputs_group.npz: every shape, case and worker count, row for row in worker order (placement, key order
and the group function's loop), plus the model's placement rules on their own.  CPU only."""
import hashlib
import os

import numpy as np
import pytest

import group_ref as G

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "reference_outputs_group.npz")


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/reference_outputs_group.npz is not present")
    return np.load(GOLDEN)


def golden_cases(g):
    """(shape, case, p) of every stored output"""
    out = []
    for k in g.files:
        if k.endswith("/in") or k.endswith("_counts"):
            continue
        name, rest = k.split("/")
        case, p = rest.rsplit("_p", 1)
        out.append((name, case, int(p)))
    return sorted(out)


def model_rows(inp, case, p):
    shards = G.split_shards(inp, p)
    if case.startswith("key_"):
        return G.group_by_key(shards, case[4:])
    return G.group_to_index(shards, int(case[6:]))


def same_rows(rows, ref):
    if ref.dtype == np.uint8:             # a digest of the rows (the larger outputs)
        return hashlib.sha256(np.ascontiguousarray(rows, np.uint64).tobytes()).digest() == ref.tobytes()
    return np.array_equal(rows, ref.reshape(-1, 7))


def test_the_fixture_covers_every_worker_count_and_case():
    g = _golden()
    cases = golden_cases(g)
    assert {p for _, _, p in cases} == {1, 2, 3, 4, 8}
    assert {c.split("_")[0] for _, c, _ in cases} == {"key", "index"}
    assert any(c == "key_partial" for _, c, _ in cases)


@pytest.mark.parametrize("p", [1, 2, 3, 4, 8])
def test_model_equals_the_reference_outputs(p):
    """every stored shape at p workers: the model's rows, concatenated in worker order, and each worker's row count"""
    g = _golden()
    checked = 0
    for name, case, q in golden_cases(g):
        if q != p:
            continue
        inp = g[name + "/in"].view(G.KV)
        outs = model_rows(inp, case, p)
        key = "%s/%s_p%d" % (name, case, p)
        assert [len(o) for o in outs] == g[key + "_counts"].tolist(), key
        assert same_rows(np.concatenate(outs), g[key]), key
        checked += 1
    assert checked >= 20


def test_placement_rules():
    keys = np.array([0, 1, 7, 8, 15, 16, (1 << 63) | 5, (1 << 64) - 1], np.uint64)
    for p in (1, 2, 3, 8):
        assert G.owner_mod(keys, p).tolist() == [int(k) % p for k in keys]
    # indices: k * p // size, the last worker for k >= size; worker r's range starts at ceil(r * size / p)
    for size, p in [(10, 3), (3, 4), (1, 8), (1003, 8), (7, 7)]:
        ks = np.arange(size + 3, dtype=np.uint64)
        own = G.owner_range(ks, size, p)
        for k in range(size):
            assert G.range_begin(own[k], size, p) <= k < G.range_begin(own[k] + 1, size, p)
        assert (own[size:] == p - 1).all()
    # the largest size the operator accepts: (size - 1) * p < 2^64
    size = ((1 << 64) - 1) // 16 + 1
    assert G.owner_range(np.array([size - 1], np.uint64), size, 16).tolist() == [15]


def test_partial_function_rows():
    items = G.grouped(G.pairs([5, 5, 5, 5, 5, 5, 5, 2], np.arange(8)))
    rows = G.group_rows(items, G.PARTIAL, 0)
    assert rows[:, 1].tolist() == [2, 5, 5, 5] and rows[:, 2].tolist() == [1, 3, 3, 1]
