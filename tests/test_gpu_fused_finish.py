"""The prefix sort's finishing pass fused into its last prefix pass (tg_radix_sort.cu FusedFinish, finish_repair_kernel) on one
H100, bit-exact against the plain reference of tests/sort_ref.py.  pytest -m gpu.

The inputs are built from groups of items that share a key prefix (the K most significant key bytes the prefix sort orders
by), so that many groups are cut where the fused pass cannot see them whole: between two tiles' runs of one digit and
between a tile's two exchange rounds.  `cuts` models where the last prefix pass puts every item (stable passes: 16-byte
items) and proves that an input has such groups; the sort must still equal the stable reference, with no fallback.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import sort_ref as R
from sort_ref import BE, LE, Desc

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
TILE = {8: 16384, 16: 8192}                 # items per tile of the partition pass; a tile's write-out runs in two halves


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture
def ctx():
    c = _capi().Ctx(device=0)
    c.profile_enable(True)
    yield c
    c.close()


def prefix_digits(n):
    bits = 4
    while bits < 64 and (1 << bits) < n * 16:
        bits += 1
    return (bits + 7) // 8


def grouped_items(d, n, seed, gmax=5, tops=32, big=()):
    """(n, item_bytes) items whose K leading key bytes come in groups of 1..gmax equal prefixes (plus one group of each size
    in `big`); the leading key byte takes `tops` values (a few tiles per segment), the key bytes below the prefix come from
    {0, 1, 2} (equal full keys: stability), every other byte is random"""
    rng = np.random.RandomState(seed)
    K = prefix_digits(n)
    kb = d.key_bytes
    sizes = np.r_[np.array(big, np.int64), rng.randint(1, gmax + 1, n)]
    sizes = sizes[:np.searchsorted(np.cumsum(sizes), n) + 1]
    sizes[-1] -= sizes.sum() - n
    sizes = sizes[sizes > 0]
    top_pool = np.concatenate([rng.choice(128, tops // 2, replace=False), 128 + rng.choice(128, tops - tops // 2, replace=False)])
    # distinct prefixes (a group is exactly the items with its prefix): distinct draws from tops * 256^(K-1) values
    code = rng.choice(tops << (8 * (K - 1)), len(sizes), replace=False)
    pre = np.empty((len(sizes), K), np.uint8)
    pre[:, 0] = top_pool[code >> (8 * (K - 1))]
    for j in range(1, K):
        pre[:, j] = (code >> (8 * (K - 1 - j))) & 255
    cols = np.concatenate([np.repeat(pre, sizes, axis=0), rng.randint(0, 3, (n, kb - K)).astype(np.uint8)], axis=1)
    cols = cols[rng.permutation(n)]
    items = rng.randint(0, 256, (n, d.item_bytes)).astype(np.uint8)
    items[:, d.key_offset:d.key_offset + kb] = cols[:, ::-1] if d.key_kind == LE else cols
    return items


def cuts(items, d):
    """how many prefix groups the last prefix pass cuts between tiles, between exchange rounds, and both, for stable passes
    (every key byte active): segments by the leading key byte, inside them the order of the K-2 prefix bytes below the
    last pass's digit (ties in input order), tiles of TILE items, and inside a tile the order of the last pass's digit"""
    n = len(items)
    K = prefix_digits(n)
    tile, half = TILE[d.item_bytes], TILE[d.item_bytes] // 2
    k = R.key_columns(items, d).astype(np.int64)
    top, dig = k[:, 0], k[:, 1]
    low = np.zeros(n, np.int64)
    for j in range(2, K):
        low = low * 256 + k[:, j]
    order = np.lexsort((low, top))                      # the last pass's input: by segment, then by the lower prefix digits
    seg_start = np.searchsorted(top[order], top[order], side="left")
    tile_id = np.empty(n, np.int64)
    tile_id[order] = top[order] * (1 << 20) + (np.arange(n) - seg_start) // tile
    local = np.empty(n, np.int64)                       # tile-local position after the pass: stable by digit inside the tile
    o2 = np.lexsort((np.argsort(np.argsort(order, kind="stable"), kind="stable"), dig, tile_id))
    first = np.searchsorted(tile_id[o2], tile_id[o2], side="left")
    local[o2] = np.arange(n) - first
    rnd = local >= half
    pre = top * (1 << 40) + dig * (1 << 32) + low
    o = np.lexsort((rnd, tile_id, pre))                 # by group, tile, round
    gp, tl, rd = pre[o], tile_id[o], rnd[o]
    gs = np.flatnonzero(np.r_[True, gp[1:] != gp[:-1]])                 # group starts
    ts = np.flatnonzero(np.r_[True, (gp[1:] != gp[:-1]) | (tl[1:] != tl[:-1])])     # (group, tile) starts
    multi_tile = np.add.reduceat(np.r_[0, (tl[1:] != tl[:-1]) & (gp[1:] == gp[:-1])], gs) > 0
    split_pt = np.maximum.reduceat(rd, ts) != np.minimum.reduceat(rd, ts)          # a (group, tile) in both rounds
    split = np.add.reduceat(split_pt.astype(np.int64), np.searchsorted(ts, gs)) > 0
    t_cut, r_cut, both = int(multi_tile.sum()), int(split.sum()), int((multi_tile & split).sum())
    return t_cut, r_cut, both


def radix_sort(ctx, items, d):
    import ctypes as C
    n = len(items)
    dp = ctx.to_device(items)
    tmp = ctx.alloc(max(items.nbytes, 16))
    try:
        ctx.ck(ctx.L.tg_radix_sort_local(ctx.h, C.byref(d.capi()), dp, tmp, n))
        return ctx.download(dp, items.nbytes).reshape(n, d.item_bytes)
    finally:
        ctx.free(dp)
        ctx.free(tmp)


def counts(ctx):
    capi = _capi()
    return {name: ctx.profile_get(cls)[1] for name, cls in (("part", capi.K_PARTITION), ("fixup", capi.K_FIXUP))}


def check(ctx, items, d, fallbacks=0):
    fb = int(ctx.L.tg_prefix_sort_fallbacks(ctx.h))
    assert np.array_equal(radix_sort(ctx, items, d), R.sort(items, d))
    assert int(ctx.L.tg_prefix_sort_fallbacks(ctx.h)) - fb == fallbacks
    c = counts(ctx)
    assert c["fixup"] == 1, c                          # one finishing launch per attempt
    return c


# 16-byte items: every pass is stable, so `cuts` models the geometry exactly
KV = Desc(16, 8, 8, LE)


def test_model_sees_every_cut():
    """the inputs below do cut groups at tile boundaries, at the round boundary and at both (checked without a GPU too)"""
    items = grouped_items(KV, 1 << 20, 27, gmax=16)          # (the input of test_cut_groups_16byte[16])
    t, r, b = cuts(items, KV)
    assert t > 100 and r > 10 and b > 0, (t, r, b)


@pytest.mark.parametrize("gmax", [2, 5, 16])
def test_cut_groups_16byte(ctx, gmax):
    """groups cut between tiles' runs, at the round boundary and both; equal full keys with random values (stability)"""
    check(ctx, grouped_items(KV, 1 << 20, 11 + gmax, gmax=gmax), KV)


def test_cut_groups_u64(ctx):
    """plain u64 keys (the benchmark's kind of item), the same grouping, partial last tiles"""
    d = Desc(8, 0, 8, LE)
    check(ctx, grouped_items(d, (1 << 21) + 12345, 5), d)


@pytest.mark.parametrize("size,fallbacks", [(64, 0), (65, 1)])
def test_group_limit(ctx, size, fallbacks):
    """a group of 64 equal prefixes is ordered; one of 65 makes the attempt fall back (counted), the result is still right"""
    check(ctx, grouped_items(KV, 1 << 20, 31, big=(size,)), KV, fallbacks)


@pytest.mark.parametrize("d", [Desc(16, 0, 10, BE, 1), Desc(8, 0, 8, LE, 1), Desc(16, 0, 16, BE), Desc(8, 1, 6, BE)],
                         ids=lambda d: d.name)
def test_descriptors(ctx, d):
    """descending, big-endian and partial-word keys (the canonical-key form of the fused pass), partial last tiles"""
    check(ctx, grouped_items(d, (1 << 20) + 777, 41), d)


def test_switch_same_bytes():
    """TG_FUSED_FINISH=0 (the separate finishing pass) and =1 give the same bytes; each setting is read once per process"""
    outs = []
    for v in ("0", "1"):
        code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_fused_finish as t; t.dump_sorts(sys.argv[1])"
                % (HERE, os.path.dirname(HERE)))
        env = dict(os.environ, TG_FUSED_FINISH=v)
        res = subprocess.run([sys.executable, "-c", code, v], env=env, cwd=os.path.dirname(HERE), capture_output=True,
                             timeout=600)
        assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-3000:]
        outs.append(res.stdout)
    assert len(outs[0]) > 0 and outs[0] == outs[1]


def dump_sorts(tag):
    """a few sorts on one ctx, their bytes hashed to stdout (run in a subprocess by test_switch_same_bytes)"""
    import hashlib
    c = _capi().Ctx(device=0)
    try:
        for d, n, seed in ((KV, 1 << 20, 3), (Desc(8, 0, 8, LE), (1 << 21) + 5, 4), (Desc(16, 0, 10, BE, 1), 300000, 5)):
            out = radix_sort(c, grouped_items(d, n, seed), d)
            sys.stdout.write(hashlib.sha256(out.tobytes()).hexdigest() + "\n")
    finally:
        c.close()


def test_descriptor_matrix_separate_pass():
    """the descriptor matrix of test_gpu_sort_descriptors with TG_FUSED_FINISH=0"""
    env = dict(os.environ, TG_FUSED_FINISH="0")
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_sort_descriptors as t; t.reduced_matrix()" % (
        HERE, os.path.dirname(HERE))
    res = subprocess.run([sys.executable, "-c", code], env=env, cwd=os.path.dirname(HERE), capture_output=True, text=True,
                         timeout=600)
    assert res.returncode == 0 and "REDUCED_MATRIX_OK" in res.stdout, res.stdout[-2000:] + res.stderr[-3000:]
