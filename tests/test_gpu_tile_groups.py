"""GPU parity of the grouped tile lists of the segmented partition passes (tg_segmented.cuh, TILE_GROUP in tg_partition.cuh):
sorts whose top-digit buckets hold 1, G-1, G, G+1 and 2G+1 tiles, one dominant bucket, mostly empty buckets, 16-byte stable
items, the hash partition, ReducePair at whole numbers of tile groups +- 1 and ReducePair on Zipf keys (records of hot keys
are dropped from the first pass).  Bit-exact against the oracle.  Runs on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

G = 8               # TILE_GROUP
TILE8 = 16384       # items of 8 bytes per tile (PartCfg<1>::TILE)
TILE16 = 8192       # items of 16 bytes per tile (PartCfg<2>::TILE)


@pytest.fixture(scope="module")
def ctx():
    from thrill_b200 import capi
    c = capi.Ctx(device=0)
    yield c
    c.close()


def _sort_on_gpu(ctx, host, desc):
    n = host.nbytes // desc.item_bytes
    d = ctx.to_device(host)
    tmp = ctx.alloc(max(host.nbytes, 16))
    ctx.ck(ctx.L.tg_radix_sort_local(ctx.h, C.byref(desc), d, tmp, n))
    out = ctx.download(d, host.nbytes)
    ctx.free(d); ctx.free(tmp)
    return out


def _keys_with_bucket_sizes(sizes, seed):
    """u64 keys whose top byte b occurs sizes[b] times (the buckets of the pass on the most significant digit); the low 56
    bits are random, shuffled"""
    rng = np.random.RandomState(seed)
    top = np.repeat(np.arange(256, dtype=np.uint64), sizes)
    keys = (top << np.uint64(56)) | rng.randint(0, 2**56, size=len(top), dtype=np.int64).astype(np.uint64)
    rng.shuffle(keys)
    return keys


def _group_edge_sizes(tile):
    """64 buckets cycling through 1, G-1, G, G+1 and 2G+1 tiles (whole, or a few items short of whole), the others small"""
    tiles = [1, G - 1, G, G + 1, 2 * G + 1]
    sizes = np.full(256, 300, dtype=np.int64)
    for i, b in enumerate(range(0, 256, 4)):
        sizes[b] = tiles[i % len(tiles)] * tile - (i // len(tiles)) % 3
    return sizes


def test_u64_buckets_at_group_edges(ctx):
    from thrill_b200 import capi
    keys = _keys_with_bucket_sizes(_group_edge_sizes(TILE8), 1)
    out = _sort_on_gpu(ctx, keys, capi.u64_desc()).view(np.uint64)
    assert np.array_equal(out, np.sort(keys))


def test_u64_one_dominant_bucket(ctx):
    """one bucket holds ~90 % of the keys: its tiles fill whole rounds alone at the tail of the list"""
    from thrill_b200 import capi
    sizes = np.full(256, 2000, dtype=np.int64)
    sizes[77] = 40 * G * TILE8 + 3
    keys = _keys_with_bucket_sizes(sizes, 2)
    out = _sort_on_gpu(ctx, keys, capi.u64_desc()).view(np.uint64)
    assert np.array_equal(out, np.sort(keys))


def test_u64_mostly_empty_buckets(ctx):
    """40 of 256 buckets hold keys, of 1 .. 2G+1 tiles"""
    from thrill_b200 import capi
    rng = np.random.RandomState(3)
    sizes = np.zeros(256, dtype=np.int64)
    used = rng.choice(256, size=40, replace=False)
    sizes[used] = rng.randint(1, (2 * G + 1) * TILE8, size=40)
    keys = _keys_with_bucket_sizes(sizes, 3)
    out = _sort_on_gpu(ctx, keys, capi.u64_desc()).view(np.uint64)
    assert np.array_equal(out, np.sort(keys))


@pytest.mark.parametrize("groups,delta", [(1, -1), (3, 0), (3, 1)])
def test_u64_uniform_at_group_multiples(ctx, groups, delta):
    """uniform keys at whole numbers of tile groups +- 1"""
    from thrill_b200 import capi
    n = groups * G * TILE8 * 16 + delta
    keys = O.gen_sort_uniform(0, n, seed=groups)
    out = _sort_on_gpu(ctx, keys, capi.u64_desc()).view(np.uint64)
    assert np.array_equal(out, O.sort_items(keys).view(np.uint64))


def test_kv_stable_buckets_at_group_edges(ctx):
    """16-byte items, keys with the bucket sizes of the u64 case, many equal keys; the value is the input position"""
    from thrill_b200 import capi
    sizes = _group_edge_sizes(TILE16)
    rng = np.random.RandomState(4)
    top = np.repeat(np.arange(256, dtype=np.uint64), sizes)
    rng.shuffle(top)
    kv = np.zeros(len(top), dtype=O.KV)
    kv["key"] = (top << np.uint64(56)) | rng.randint(0, 3000, size=len(top)).astype(np.uint64)
    kv["val"] = np.arange(len(top))
    out = _sort_on_gpu(ctx, kv, capi.kv_key_desc()).view(O.KV)
    assert np.array_equal(out, O.sort_items(kv, O.KV_DESC).view(O.KV))


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_hash_partition_at_group_multiples(ctx, delta):
    from thrill_b200 import capi
    p = 13
    n = 5 * G * TILE16 + delta
    kv = O.gen_reduce_uniform(0, n, universe=1 << 20, exact=2)
    dest = O.hash_partition_ids(kv["key"], p).astype(np.int64)
    d_in = ctx.to_device(kv); d_out = ctx.alloc(n * 16)
    oc = np.zeros(p, dtype=np.uint64)
    ctx.ck(ctx.L.tg_hash_partition(ctx.h, C.byref(capi.KVDesc(16, capi.OP_SUM_U64)), d_in, n, p, d_out,
                                   oc.ctypes.data_as(C.POINTER(C.c_uint64))))
    out = ctx.download(d_out, n * 16, O.KV)
    ctx.free(d_in); ctx.free(d_out)
    assert np.array_equal(oc.astype(np.int64), np.bincount(dest, minlength=p))
    assert np.array_equal(out, kv[np.argsort(dest, kind="stable")])


def _reduce_pair(ctx, kv):
    from thrill_b200 import capi
    n = len(kv)
    d_in = ctx.to_device(kv)
    out_p = C.c_void_p(); out_n = C.c_size_t()
    ctx.ck(ctx.L.tg_reduce_by_key(ctx.h, C.byref(capi.KVDesc(16, capi.OP_SUM_F64)), d_in, n, C.byref(out_p), C.byref(out_n)))
    out = np.sort(ctx.download(out_p.value, out_n.value * 16, O.KV), order="key")
    ctx.free(d_in)
    return out


@pytest.mark.parametrize("groups", [1, 5])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_reduce_pair_at_group_multiples(ctx, groups, delta):
    """ReducePair (hash passes above 2^18 records) at whole numbers of 16-byte tile groups +- 1; exact-mode doubles"""
    n = groups * G * TILE16 * 8 + delta
    kv = O.gen_reduce_uniform(0, n, universe=1 << 16, exact=1)
    assert np.array_equal(_reduce_pair(ctx, kv), O.reduce_simple(kv, O.OP_SUM_F64))


def test_reduce_pair_zipf(ctx):
    """Zipf keys: the records of hot keys are dropped from the first pass, so its buckets shrink unevenly"""
    n = 8 * G * TILE16 + 1
    kv = O.gen_reduce_zipf(0, n, O.zipf_cdf(1 << 20), seed=7, exact=1)
    assert np.array_equal(_reduce_pair(ctx, kv), O.reduce_simple(kv, O.OP_SUM_F64))
