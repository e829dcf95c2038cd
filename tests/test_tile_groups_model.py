"""numpy models of the grouped tile lists of the segmented partition passes (tg_segmented.cuh): round q holds tiles
[G*q, G*q + G) of every segment that has them, one segment's group after the other, segments ordered by tile count
(descending, ties by index).  The host builder (build_tile_list) and the device closed form (seg_tiles_prepare_kernel +
seg_tiles_fill_kernel) must give the same list; every tile appears once, after its predecessor, and a group's tiles are
consecutive.  The CUDA code itself is checked on the GPU against the oracle (test_gpu_tile_groups.py)."""
import numpy as np
import pytest

G = 8               # TILE_GROUP (tg_partition.cuh)
TILE = 16384        # items of 8 bytes per tile (the lists only see it through the tile counts)


def _layout(seg_size, tile, drop_last):
    seg_size = [0 if (drop_last and s == len(seg_size) - 1) else int(v) for s, v in enumerate(seg_size)]
    nt = np.array([(v + tile - 1) // tile for v in seg_size], dtype=np.int64)
    row0 = np.concatenate(([0], np.cumsum(nt)[:-1])).astype(np.int64)
    start = np.concatenate(([0], np.cumsum(seg_size)[:-1])).astype(np.int64)
    return seg_size, nt, row0, start


def host_tile_list(seg_size, tile, g, drop_last=False):
    """build_tile_list: rounds of groups, written out one tile at a time"""
    seg_size, nt, row0, start = _layout(seg_size, tile, drop_last)
    order = sorted(range(len(seg_size)), key=lambda s: (-nt[s], s))
    out = []
    maxt = int(nt.max()) if len(nt) else 0
    for r0 in range(0, maxt, g):
        for sg in order:
            if nt[sg] <= r0:
                break
            for r in range(r0, min(r0 + g, int(nt[sg]))):
                off = r * tile
                out.append((int(start[sg] + off), min(tile, seg_size[sg] - off), int(row0[sg] + r), (sg << 20) | r))
    return out


def device_tile_list(seg_size, tile, g, drop_last=False):
    """seg_tiles_fill_kernel: tile (s, r) of the round starting at g0 sits at A(g0) + B(s) + (r - g0)"""
    seg_size, nt, row0, start = _layout(seg_size, tile, drop_last)
    S = len(seg_size)
    sortrank = np.array([sum(1 for q in range(S) if nt[q] > nt[s] or (nt[q] == nt[s] and q < s)) for s in range(S)])
    snt = np.zeros(S, dtype=np.int64)
    snt[sortrank] = nt
    P = np.concatenate(([0], np.cumsum(snt)))
    T = int(P[S])
    out = [None] * T
    for row in range(T):
        sg = int(np.searchsorted(row0, row, side="right") - 1)              # last segment with row0 <= row (it has tiles)
        r = row - int(row0[sg])
        g0 = r - r % g
        C = int(np.sum(snt > g0))
        F = int(np.sum(snt > g0 + g - 1))
        k = int(sortrank[sg])
        before = g * k if k <= F else g * F + int(P[k] - P[F]) - g0 * (k - F)
        pos = g0 * C + (T - int(P[C])) + before + (r - g0)
        assert out[pos] is None, "two tiles at one position"
        off = r * tile
        out[pos] = (int(start[sg] + off), min(tile, seg_size[sg] - off), row, (sg << 20) | r)
    return out


def _check_list(lst, seg_size, tile, g, drop_last=False):
    seg_size, nt, row0, start = _layout(seg_size, tile, drop_last)
    assert len(lst) == int(nt.sum())
    seen = set()
    where = {}
    for pos, (st, ln, row, w) in enumerate(lst):
        sg, r = w >> 20, w & 0xFFFFF
        assert (sg, r) not in seen, "tile listed twice"
        seen.add((sg, r))
        where[(sg, r)] = pos
        assert row == row0[sg] + r and st == start[sg] + r * tile and 0 < ln <= tile
    assert len(seen) == int(nt.sum()), "a tile is missing"
    for (sg, r), pos in where.items():
        if r > 0:
            assert where[(sg, r - 1)] < pos, "tile before its predecessor"
        if r % g:
            assert where[(sg, r - 1)] == pos - 1, "group not consecutive"


def _cases():
    S = 256
    cases = []
    for seed in range(6):
        rs = np.random.RandomState(seed)
        seg = rs.randint(0, 40 * TILE, size=S)
        seg[rs.randint(0, S, size=40)] = 0                                  # empty buckets
        if seed % 2:
            seg[rs.randint(0, S)] = 700 * TILE + 5                          # one dominant bucket
        cases.append(("random%d" % seed, seg))
    # segments of 0, 1, G-1, G, G+1, 2G+1 tiles (the last one partial), repeated over the buckets
    tiles = [0, 1, G - 1, G, G + 1, 2 * G + 1]
    seg = np.array([max(tiles[s % len(tiles)] * TILE - (s % 3) * 17, 0) for s in range(S)])
    cases.append(("edges", seg))
    seg = np.zeros(S, dtype=np.int64); seg[17] = 3 * TILE; seg[255] = 1
    cases.append(("sparse", seg))
    seg = np.zeros(S, dtype=np.int64); seg[200] = 2 * G * TILE + 1
    cases.append(("one_bucket", seg))
    seg = np.full(S, 23 * TILE + 9000)                                    # the 1e8-key sort's buckets: equal tile counts
    cases.append(("even", seg))
    cases.append(("empty", np.zeros(S, dtype=np.int64)))
    return cases


@pytest.mark.parametrize("g", [1, 2, 4, G])
@pytest.mark.parametrize("drop_last", [False, True])
@pytest.mark.parametrize("name,seg", _cases(), ids=[c[0] for c in _cases()])
def test_device_closed_form_equals_the_host_list(name, seg, drop_last, g):
    seg = [int(v) for v in seg]
    host = host_tile_list(seg, TILE, g, drop_last)
    assert device_tile_list(seg, TILE, g, drop_last) == host
    _check_list(host, seg, TILE, g, drop_last)


def test_one_group_is_the_round_robin_list():
    """G = 1 is the list the passes used before groups: round r holds the r-th tile of every segment"""
    seg = [int(v) for v in np.random.RandomState(9).randint(0, 30 * TILE, size=256)]
    lst = host_tile_list(seg, TILE, 1)
    rounds = [w & 0xFFFFF for (_, _, _, w) in lst]
    assert rounds == sorted(rounds)


@pytest.mark.parametrize("nchunks", [1, 3, 255, 264])
def test_chunk_lists(nchunks):
    """a chunked pass: equal chunks of whole tiles and a shorter last one (host-built only)"""
    chunk = 24 * TILE
    seg = [chunk] * (nchunks - 1) + [chunk // 3 + 5]
    lst = host_tile_list(seg, TILE, G)
    _check_list(lst, seg, TILE, G)
    # the first round holds the first group of every chunk, G tiles each
    assert [w >> 20 for (_, _, _, w) in lst[:G * nchunks:G]] == list(range(nchunks))
