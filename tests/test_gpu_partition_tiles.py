"""GPU parity of the partition pass at its tile edges (tg_partition.cuh PartCfg): sizes just around one and two tiles,
full tiles that start at odd items inside a segment (the TMA copy is shifted by one item), a tile whose items all share
one digit (one run through both exchange rounds), 16-byte items (stable) and ReducePair at the 16-byte tile edges.
Bit-exact against the oracle.  Runs on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

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


def _kv_small_keys(n, seed):
    """16-byte items with many equal keys; the value is the input position, so stability is visible"""
    rng = np.random.RandomState(seed)
    kv = np.zeros(n, dtype=O.KV)
    kv["key"] = rng.randint(0, 5000, size=n)
    kv["val"] = np.arange(n)
    return kv


@pytest.mark.parametrize("n", [TILE8 - 1, TILE8, TILE8 + 1, 2 * TILE8 + 1])
def test_u64_at_tile_edges(ctx, n):
    from thrill_b200 import capi
    keys = O.gen_sort_uniform(0, n)
    out = _sort_on_gpu(ctx, keys, capi.u64_desc()).view(np.uint64)
    assert np.array_equal(out, O.sort_items(keys).view(np.uint64))


def test_u64_segment_tiles_at_odd_starts(ctx):
    """~256 segments of ~1.5 tiles each after the top-digit pass: every segment has one full tile, and about half of them
    start at an odd item"""
    from thrill_b200 import capi
    n = 256 * (3 * TILE8 // 2) + 7
    keys = O.gen_sort_uniform(5, n)
    out = _sort_on_gpu(ctx, keys, capi.u64_desc()).view(np.uint64)
    assert np.array_equal(out, O.sort_items(keys).view(np.uint64))


def test_u64_one_digit_fills_a_tile(ctx):
    """the first tile's keys all share their top byte (one digit run covers the whole tile, through both exchange
    rounds); the second tile's top bytes vary, so the pass on that digit is not skipped"""
    from thrill_b200 import capi
    rng = np.random.RandomState(3)
    n = 2 * TILE8
    keys = rng.randint(0, 2**56, size=n, dtype=np.int64).astype(np.uint64)
    keys[:TILE8] |= np.uint64(0x5a) << np.uint64(56)
    keys[TILE8:] |= rng.randint(0, 256, size=TILE8).astype(np.uint64) << np.uint64(56)
    out = _sort_on_gpu(ctx, keys, capi.u64_desc()).view(np.uint64)
    assert np.array_equal(out, np.sort(keys))


@pytest.mark.parametrize("n", [TILE16 - 1, TILE16, TILE16 + 1, 2 * TILE16 + 1, 256 * (3 * TILE16 // 2) + 7])
def test_kv_stable_at_tile_edges(ctx, n):
    from thrill_b200 import capi
    kv = _kv_small_keys(n, n)
    out = _sort_on_gpu(ctx, kv, capi.kv_key_desc()).view(O.KV)
    assert np.array_equal(out, O.sort_items(kv, O.KV_DESC).view(O.KV))


@pytest.mark.parametrize("n", [TILE16 - 1, TILE16, TILE16 + 1, 2 * TILE16 + 1])
def test_hash_partition_at_tile_edges(ctx, n):
    """the hash-digit partition (digit kept in shared memory for the write-out): bit-exact destinations, stable"""
    from thrill_b200 import capi
    p = 13
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


@pytest.mark.parametrize("tiles", [40, 41, 300])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_reduce_pair_at_tile_edges(ctx, tiles, delta):
    """ReducePair above the size where the hash-digit partition passes run (2^18 records), at whole tiles +- 1; exact-mode
    doubles, so the sums are bit-exact"""
    from thrill_b200 import capi
    n = tiles * TILE16 + delta
    kv = O.gen_reduce_uniform(0, n, universe=1 << 16, exact=1)
    d_in = ctx.to_device(kv)
    out_p = C.c_void_p(); out_n = C.c_size_t()
    ctx.ck(ctx.L.tg_reduce_by_key(ctx.h, C.byref(capi.KVDesc(16, capi.OP_SUM_F64)), d_in, n, C.byref(out_p), C.byref(out_n)))
    out = np.sort(ctx.download(out_p.value, out_n.value * 16, O.KV), order="key")
    ctx.free(d_in)
    assert np.array_equal(out, O.reduce_simple(kv, O.OP_SUM_F64))
