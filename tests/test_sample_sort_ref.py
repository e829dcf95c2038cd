"""CPU checks of sample_sort_ref, the plain reference the multi-worker Sort's device classification is compared with: against
the oracle's restatement of FindAndSendSplitters / TreeBuilder / TransmitItems (descending descriptors through sort_ref's
complement rule), against the round-2 numpy models, and against planted wrong outputs that it must tell apart."""
import numpy as np
import pytest

import oracle_lib as O
import sample_sort_ref as S
import sort_ref as R
import test_round2_models as M
from sort_ref import LE, Desc

DESCS = R.ITEM8 + R.ITEM16


def shards_for(d, sizes, dist, seed):
    return [S.make_items(d, int(n), dist, seed + 101 * w) for w, n in enumerate(sizes)]


def oracle_select(shards, d, p, rng_seed):
    """the oracle's splitters (packed, in d's own key bytes) and buckets of every shard, from the same sample draws"""
    its, _, _, g = S.samples(shards, d, p, rng_seed)
    comp, od = R.for_oracle(its, d)
    spl = O.select_splitters(O.pack_samples(comp, g, od), p, od)
    padded, k = O.pad_splitters(spl, p, od)
    tree = O.build_tree(padded, k, od)
    pre = S.prefix_of(shards, d)
    buckets = []
    for w, sh in enumerate(shards):
        c, _ = R.for_oracle(sh, d)
        b = O.classify(c, int(pre[w]), tree, k, padded, od).astype(np.int64)
        b[b == k - 1] = p - 1                    # the writer swap of TransmitItems (api/sort.hpp:460)
        buckets.append(b)
    out = np.array(spl, copy=True)
    if d.descending:
        out[:, :d.item_bytes] = R.complement_keys(out[:, :d.item_bytes], d)
    return out, buckets


@pytest.mark.parametrize("p", [3, 8])
@pytest.mark.parametrize("d", DESCS, ids=lambda d: d.name)
def test_reference_matches_the_oracle(d, p):
    rng = np.random.RandomState(d.item_bytes * 7 + d.key_offset * 3 + d.key_bytes + p + 40 * d.descending)
    for dist in ("uniform", "few", "top", "equal", "onetop"):
        shards = shards_for(d, rng.randint(0, 3000, size=p), dist, int(rng.randint(1 << 20)))
        seed = int(rng.randint(1 << 30))
        want_spl, want_b = oracle_select(shards, d, p, seed)
        spl, counts, grouped, bounds = S.select(shards, d, p, seed)
        assert np.array_equal(spl, want_spl), dist
        pre = S.prefix_of(shards, d)
        for w, sh in enumerate(shards):
            b = S.classify(sh, d, pre[w] + np.arange(len(sh)), spl)
            assert np.array_equal(b, want_b[w]), (dist, w)
            assert np.array_equal(counts[w], np.bincount(b, minlength=p))
            assert np.array_equal(grouped[w], sh[np.argsort(b, kind="stable")])
            # the merge pipeline cuts the sorted shard where the classification cuts the unsorted one
            assert np.array_equal(bounds[w], np.cumsum(counts[w])[:-1])


@pytest.mark.parametrize("p", [2, 5, 8, 16])
def test_reference_matches_the_round2_models(p):
    """u64 keys: the splitters are the round-2 reference rule's and its rank-counting device model's, and the buckets its
    plain and top-byte-table classification"""
    d = Desc(8, 0, 8, LE)
    rng = np.random.RandomState(p)
    for dist in ("uniform", "few", "low"):
        sizes = rng.randint(0, 2000, size=p)
        shards = shards_for(d, sizes, dist, p * 13)
        seed = int(rng.randint(1 << 30))
        its, _, _, g = S.samples(shards, d, p, seed)
        keys = its.view("<u8").reshape(-1)
        if len(keys) == 0:
            continue
        pre = S.prefix_of(shards, d)
        flat = [(int(k), int(i)) for k, i in zip(keys, g)]
        spl = S.splitters(shards, d, p, seed)
        pairs = [(int(s[:8].view("<u8")[0]), int(s[8:].view("<u8")[0])) for s in spl]
        assert pairs == M.reference_splitters(flat, p)
        lists, off = [], 0
        for w in range(p):
            ns = S.sample_count(int(sizes[w]))
            lists.append(sorted((k, i - int(pre[w])) for k, i in flat[off:off + ns]))
            off += ns
        assert M.device_splitters(lists, sizes, p) == pairs
        lo_t, hi_t = S.lut(spl, d)
        assert list(lo_t) == [sum(1 for s in pairs if (s[0] >> 56) < b) for b in range(256)]
        assert list(hi_t) == [sum(1 for s in pairs if (s[0] >> 56) <= b) for b in range(256)]
        w = p - 1
        b = S.classify(shards[w], d, pre[w] + np.arange(len(shards[w])), spl)
        sk = shards[w].view("<u8").reshape(-1)
        for i in range(0, len(sk), 11):
            gi = int(pre[w]) + i
            assert b[i] == M.classify_plain(int(sk[i]), gi, pairs) == M.classify_lut(int(sk[i]), gi, pairs, lo_t, hi_t)


@pytest.mark.parametrize("d", DESCS, ids=lambda d: d.name)
def test_top_byte_table_classification_for_every_descriptor(d):
    """SplitterDigit's lookup table by the canonical key's top byte (byte key_bytes - 1 of a little-endian key, the first byte of a
    byte string, complemented when descending) never changes a bucket"""
    p = 16
    for dist in S.DISTS:
        shards = shards_for(d, [1500] * p, dist, 7)
        spl = S.splitters(shards, d, p, 3)
        pre = S.prefix_of(shards, d)
        for w in (0, p // 2, p - 1):
            g = pre[w] + np.arange(len(shards[w]))
            assert np.array_equal(S.classify_lut(shards[w], d, g, spl), S.classify(shards[w], d, g, spl)), dist


def test_sample_draws_repeat_on_tiny_shards():
    """a shard of 1 or 2 items draws n positions, which may repeat; an empty shard draws nothing"""
    for n in (1, 2, 3):
        pos = S.sample_positions(n, S.worker_seed(5, 1))
        assert len(pos) == n == min(n, O.sample_size(n)) and set(pos) <= set(range(n))
    assert len(S.sample_positions(0, 7)) == 0
    assert list(S.sample_positions(2, S.worker_seed(5, 0))) == [0, 0]


# ---- planted wrong outputs: each must differ from the reference --------------------------------------------------------
def test_rejects_splitters_off_by_one_rank():
    d = Desc(16, 0, 16, R.BE)
    for p in (3, 16):
        shards = shards_for(d, [5000] * p, "uniform", p)
        spl = S.splitters(shards, d, p, 9)
        wrong = S.splitters(shards, d, p, 9, rank_shift=1)
        assert not np.array_equal(wrong, spl)
        assert not np.array_equal(wrong, oracle_select(shards, d, p, 9)[0])
        assert np.array_equal(spl, oracle_select(shards, d, p, 9)[0])


@pytest.mark.parametrize("d", [Desc(8, 0, 8, LE), Desc(16, 0, 10, R.BE, 1)], ids=lambda d: d.name)
def test_rejects_ties_broken_by_local_index(d):
    """items equal to a splitter's key fall on both sides of it by GLOBAL index; local positions move some of them"""
    p = 5
    shards = shards_for(d, [4000] * p, "few", 1)
    spl = S.splitters(shards, d, p, 4)
    pre = S.prefix_of(shards, d)
    wrong = 0
    for w in range(p):
        local = np.arange(len(shards[w]))
        right = S.classify(shards[w], d, pre[w] + local, spl)
        assert np.array_equal(right, oracle_select(shards, d, p, 4)[1][w])
        wrong += int(np.count_nonzero(S.classify(shards[w], d, local, spl) != right))
    assert wrong > 0


@pytest.mark.parametrize("d", [Desc(8, 0, 8, LE), Desc(8, 2, 4, LE), Desc(16, 0, 16, R.BE), Desc(16, 0, 8, LE, 1)],
                         ids=lambda d: d.name)
def test_rejects_a_bucket_bound_off_by_one_in_one_top_byte_range(d):
    p = 8
    shards = shards_for(d, [6000] * p, "uniform", 2)
    spl = S.splitters(shards, d, p, 6)
    lo_t, hi_t = S.lut(spl, d)
    t = int(S.top_byte(np.ascontiguousarray(spl[:, :d.item_bytes]), d)[p // 2])      # a byte range that holds a splitter
    for bad in ((lo_t, hi_t - (np.arange(256) == t)), (lo_t + (np.arange(256) == t), hi_t)):
        differs = 0
        for w in range(p):
            g = S.prefix_of(shards, d)[w] + np.arange(len(shards[w]))
            differs += int(np.count_nonzero(S.classify_lut(shards[w], d, g, spl, table=bad) != S.classify(shards[w], d, g, spl)))
        assert differs > 0


@pytest.mark.parametrize("p", [2, 3, 7, 16])
def test_range_partition_edges(p):
    """worker r holds [CalculateBeginOfPart(r), CalculateBeginOfPart(r + 1)); an edge moved by one is caught"""
    for size in (1, p - 1, p, p + 1, 1000, (1 << 34) + 3):
        if size == 0:
            continue
        edges = [S.begin_of_part(r, size, p) for r in range(p + 1)]
        assert edges[0] == 0 and edges[p] == size
        keys = sorted({e + o for e in edges for o in (-1, 0, 1) if 0 <= e + o} | {size, (1 << 64) - 1})
        dest = S.range_dest(keys, size, p)
        for k, r in zip(keys, dest):
            if k >= size:
                assert r == p - 1
            else:
                assert edges[r] <= k < edges[r + 1]
        for r in range(1, p):
            if edges[r] < size and edges[r] > edges[r - 1]:
                wrong = [r - 1 if k == edges[r] else x for k, x in zip(keys, dest)]          # the edge one index late
                assert wrong != list(dest)
