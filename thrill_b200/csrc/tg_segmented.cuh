// tg_segmented.cuh — partition passes whose chained scan spans a few tiles that run at the same time, not a whole wave.
//
// A partition pass needs, for every tile and digit, the number of items with that digit in the tiles before it.
// The chained scan ("decoupled look-back", tg_partition.cuh) gets it from the tiles themselves, which makes every tile
// wait for the tiles processed at the same time on the other SMs.  Both forms below
// know the bases of coarse SEGMENTS up front, so the scan chain of a tile only spans its own segment, and list the tiles
// in rounds of groups: round q holds the q-th group of TILE_GROUP (G) neighbouring tiles of every segment.  The G tiles of
// a group run in the same wave of CTAs and write each digit's runs next to each other in memory; the predecessor of a
// group's first tile finished a whole wave earlier, and a later member waits at most for the members before it, which
// publish their counts right after ranking.  Every tile's predecessors come earlier in the list, and every CTA takes its
// tiles in list order, so the scan always makes progress.
//   * chunked pass   — any input: cut it into contiguous chunks, one counting read gives segbase[chunk][digit]
//   * segmented pass — input already partitioned by a more significant digit: the buckets are the segments, items never
//     leave their bucket, and one counting read serves every further pass inside the buckets.
// Used by the radix sort (tg_radix_sort.cu) and by the hash aggregation (tg_reduce.cu).
#pragma once
#include <algorithm>
#include <vector>

#include "tg_partition.cuh"

namespace tgp {

// up to 4 digit functions counted in one read
template <class DigitFn>
struct DigitList {
    int n;
    DigitFn fn[4];
};

// Per-chunk histogram of fn (chunk = blockIdx.x, items [chunk*chunk_items, ...)); ORAND: also OR / AND of the item words
// (orand[2w] = OR, orand[2w+1] = AND of word w; tells which digit positions are constant over the whole input).
template <int WORDS, class DigitFn, bool ORAND>
__global__ void __launch_bounds__(512) chunk_hist_kernel(const typename ItemT<WORDS>::type* __restrict__ in, u32 n, u32 chunk_items,
                                                         const DigitFn fn_param, u32* __restrict__ chunkcount /* [grid][RADIX] */,
                                                         u64* __restrict__ orand) {
    typedef typename ItemT<WORDS>::type Item;
    DigitFn fn = fn_param;
    fn.init();
    constexpr int U = 32 / (4 * WORDS);      // 64 bytes of loads in flight per thread
    __shared__ u32 sh[RADIX];
    __shared__ __align__(16) unsigned char fscratch[DigitFn::kScratch > 0 ? DigitFn::kScratch : 16];
    if constexpr (DigitFn::kScratch > 0) fn.init_shared(fscratch, (int)threadIdx.x, (int)blockDim.x);
    for (int i = threadIdx.x; i < RADIX; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const u32 lo = blockIdx.x * chunk_items;
    const u32 hi = (n - lo < chunk_items) ? n : lo + chunk_items;
    const u32 lane = lane_id();
    u64 vor[WORDS], vand[WORDS];
#pragma unroll
    for (int w = 0; w < WORDS; ++w) { vor[w] = 0; vand[w] = ~0ull; }
    for (u32 base = lo; base < hi; base += blockDim.x * U) {
        Item v[U];
        bool valid[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            u32 i = base + u * blockDim.x + threadIdx.x;
            valid[u] = i < hi;
            if (valid[u]) v[u] = in[i];
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (ORAND && valid[u]) {
#pragma unroll
                for (int w = 0; w < WORDS; ++w) { vor[w] |= item_word(v[u], w); vand[w] &= item_word(v[u], w); }
            }
            const u32 d = valid[u] ? fn(v[u], base + u * blockDim.x + threadIdx.x) : 0u;
            if (__all_sync(0xffffffffu, valid[u])) {
                // one shared-memory atomic per warp where the whole warp agrees on the digit (constant high bytes)
                const u32 d0 = __shfl_sync(0xffffffffu, d, 0);
                if (__all_sync(0xffffffffu, d == d0)) { if (lane == 0) atomicAdd(&sh[d], 32u); }
                else atomicAdd(&sh[d], 1u);
            }
            else if (valid[u]) atomicAdd(&sh[d], 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < RADIX; i += blockDim.x) chunkcount[(size_t)blockIdx.x * RADIX + i] = sh[i];
    if (ORAND) {
#pragma unroll
        for (int w = 0; w < WORDS; ++w) {
            u32 olo = __reduce_or_sync(0xffffffffu, (u32)vor[w]), ohi = __reduce_or_sync(0xffffffffu, (u32)(vor[w] >> 32));
            u32 alo = __reduce_and_sync(0xffffffffu, (u32)vand[w]), ahi = __reduce_and_sync(0xffffffffu, (u32)(vand[w] >> 32));
            if (lane == 0) {
                atomicOr(&orand[2 * w], ((u64)ohi << 32) | olo);
                atomicAnd(&orand[2 * w + 1], ((u64)ahi << 32) | alo);
            }
        }
    }
}

// totals[d], gbase[d] (exclusive scan of the totals) and segbase[chunk][d]; one CTA of 4 * RADIX threads
static __global__ void __launch_bounds__(4 * RADIX) chunk_scan_kernel(const u32* __restrict__ chunkcount, int nchunks,
                                                                      u32* __restrict__ totals, u32* __restrict__ gbase,
                                                                      u32* __restrict__ segbase) {
    __shared__ u32 part[4][RADIX];
    __shared__ u32 warp_tot[RADIX / 32];
    const int d = threadIdx.x & (RADIX - 1), g = threadIdx.x >> 8;
    const int per = (nchunks + 3) / 4;
    const int c0 = g * per, c1 = (c0 + per < nchunks) ? c0 + per : nchunks;
    u32 sum = 0;
#pragma unroll 8
    for (int c = c0; c < c1; ++c) sum += chunkcount[(size_t)c * RADIX + d];
    part[g][d] = sum;
    __syncthreads();
    u32 tot = 0, before = 0;
    for (int q = 0; q < 4; ++q) { u32 v = part[q][d]; tot += v; if (q < g) before += v; }
    u32 incl = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        u32 t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((d & 31) >= o) incl += t;
    }
    if (g == 0 && (d & 31) == 31) warp_tot[d >> 5] = incl;
    __syncthreads();
    u32 gb = incl - tot;
    for (int w = 0; w < (d >> 5); ++w) gb += warp_tot[w];
    if (g == 0) { totals[d] = tot; gbase[d] = gb; }
    u32 run = gb + before;
#pragma unroll 8
    for (int c = c0; c < c1; ++c) {
        u32 v = chunkcount[(size_t)c * RADIX + d];
        segbase[(size_t)c * RADIX + d] = run;
        run += v;
    }
}

// Per-segment histograms of up to 4 digit functions over a segmented tile list (the histogram of a digit inside a
// segment does not change while passes permute the items inside the segment: one read serves all of them).
template <int WORDS, class DigitFn, int NPOS>
__global__ void __launch_bounds__(512) seg_count_kernel(const typename ItemT<WORDS>::type* __restrict__ in, SegList sl,
                                                        const DigitList<DigitFn> dl_param, u32* __restrict__ segcount /* [seg][NPOS][RADIX] */) {
    typedef typename ItemT<WORDS>::type Item;
    DigitList<DigitFn> dl = dl_param;
#pragma unroll
    for (int p = 0; p < NPOS; ++p) dl.fn[p].init();
    __shared__ u32 sh[NPOS * RADIX];
    constexpr int U = 4;
    const u32 num_tiles = seg_num_tiles(sl);
    for (u32 j = blockIdx.x; j < num_tiles; j += gridDim.x) {
        const uint4 t = __ldg(&sl.tiles[j]);
        for (int i = threadIdx.x; i < NPOS * RADIX; i += blockDim.x) sh[i] = 0;
        __syncthreads();
        for (u32 base = 0; base < t.y; base += blockDim.x * U) {
            Item v[U];
            bool valid[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const u32 i = base + u * blockDim.x + threadIdx.x;
                valid[u] = i < t.y;
                if (valid[u]) v[u] = in[(size_t)t.x + i];
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (!valid[u]) continue;
#pragma unroll
                for (int p = 0; p < NPOS; ++p) atomicAdd(&sh[p * RADIX + dl.fn[p](v[u], t.x + base + u * blockDim.x + threadIdx.x)], 1u);
            }
        }
        __syncthreads();
        u32* dst = segcount + (size_t)(t.w >> 20) * NPOS * RADIX;
        for (int i = threadIdx.x; i < NPOS * RADIX; i += blockDim.x)
            if (sh[i]) atomicAdd(&dst[i], sh[i]);
        __syncthreads();
    }
}

// launches seg_count_kernel for dl.n = 1..4 digit functions
template <int WORDS, class DigitFn>
int launch_seg_count(tg_ctx* ctx, const void* in, const SegList& sl, const DigitList<DigitFn>& dl, u32* segcount) {
    typedef typename ItemT<WORDS>::type Item;
    int grid = ctx->sm_count * 4;
    if ((u32)grid > sl.num_tiles) grid = (int)sl.num_tiles;
    if (grid == 0) return TG_OK;
    switch (dl.n) {
    case 1: TG_LAUNCH_T(ctx, TG_K_SEGCOUNT, (seg_count_kernel<WORDS, DigitFn, 1>), grid, 512, 0, (const Item*)in, sl, dl, segcount); break;
    case 2: TG_LAUNCH_T(ctx, TG_K_SEGCOUNT, (seg_count_kernel<WORDS, DigitFn, 2>), grid, 512, 0, (const Item*)in, sl, dl, segcount); break;
    case 3: TG_LAUNCH_T(ctx, TG_K_SEGCOUNT, (seg_count_kernel<WORDS, DigitFn, 3>), grid, 512, 0, (const Item*)in, sl, dl, segcount); break;
    case 4: TG_LAUNCH_T(ctx, TG_K_SEGCOUNT, (seg_count_kernel<WORDS, DigitFn, 4>), grid, 512, 0, (const Item*)in, sl, dl, segcount); break;
    default: return tg_set_error(ctx, TG_ERR_ARG, "segment count: %d digit functions", dl.n);
    }
    return TG_OK;
}

// segbase[pos][seg][d] = seg_start[seg] + exclusive scan over d of segcount[seg][pos][.]; grid (nseg, npos), RADIX threads
static __global__ void seg_scan_kernel(const u32* __restrict__ segcount, const u32* __restrict__ seg_start, int npos, int nseg,
                                       u32* __restrict__ segbase) {
    __shared__ u32 warp_tot[RADIX / 32];
    const int seg = blockIdx.x, pos = blockIdx.y, d = threadIdx.x;
    const u32 c = segcount[((size_t)seg * npos + pos) * RADIX + d];
    u32 incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        u32 t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((d & 31) >= o) incl += t;
    }
    if ((d & 31) == 31) warp_tot[d >> 5] = incl;
    __syncthreads();
    u32 add = seg_start[seg];
    for (int w = 0; w < (d >> 5); ++w) add += warp_tot[w];
    segbase[((size_t)pos * nseg + seg) * RADIX + d] = add + incl - c;
}

// Tile list of `nseg` segments of seg_size[] items laid out back to back, interleaving groups of G = TILE_GROUP tiles of the
// segments: round q holds tiles [G*q, G*q + G) of every segment that has them (fewer in a segment's last round), one
// segment's group after the other, segments ordered by tile count (descending, ties by index).  The list is staged in pinned
// host buffer `stage` (0/1; the list staged there before must have been consumed by its copy: callers alternate the two
// buffers between stream synchronisations) and copied to *d_tiles (workspace slot `ws_slot`).
inline int build_tile_list(tg_ctx* ctx, int nseg, const u32* seg_size, u32 tile, int stage, int ws_slot, uint4** d_tiles, u32* total_out) {
    constexpr u32 G = TILE_GROUP;
    if (nseg > 4096) return tg_set_error(ctx, TG_ERR_ARG, "tile list: at most 4096 segments");
    std::vector<u32> ntiles(nseg), row0(nseg), start(nseg), order(nseg);
    u32 total = 0, acc = 0, maxt = 0;
    for (int s = 0; s < nseg; ++s) {
        ntiles[s] = (seg_size[s] + tile - 1) / tile;
        row0[s] = total;
        start[s] = acc;
        total += ntiles[s];
        acc += seg_size[s];
        if (ntiles[s] > maxt) maxt = ntiles[s];
        order[s] = (u32)s;
    }
    if (maxt >= (1u << 20)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "tile list: segment of %u tiles", maxt);
    std::sort(order.begin(), order.end(), [&](u32 a, u32 b) { return ntiles[a] != ntiles[b] ? ntiles[a] > ntiles[b] : a < b; });
    uint4* h_tiles;
    TG_TRY(tg_pinned_list(ctx, stage, (size_t)total * sizeof(uint4) + 16, (void**)&h_tiles));
    u32 w = 0;
    for (u32 r0 = 0; r0 < maxt; r0 += G) {
        for (int o = 0; o < nseg; ++o) {
            const u32 sg = order[o];
            if (ntiles[sg] <= r0) break;              // sorted by tile count: nobody further has a tile in this round
            const u32 r1 = ntiles[sg] - r0 < G ? ntiles[sg] : r0 + G;
            for (u32 r = r0; r < r1; ++r) {
                const u32 off = r * tile;
                const u32 len = seg_size[sg] - off < tile ? seg_size[sg] - off : tile;
                h_tiles[w++] = make_uint4(start[sg] + off, len, row0[sg] + r, (sg << 20) | r);
            }
        }
    }
    TG_TRY(tg_ws_get(ctx, ws_slot, (size_t)total * sizeof(uint4) + 16, (void**)d_tiles));
    if (total) TG_CUDA(ctx, cudaMemcpyAsync(*d_tiles, h_tiles, (size_t)total * sizeof(uint4), cudaMemcpyHostToDevice, ctx->stream));
    *total_out = total;
    return TG_OK;
}

// ---- the same interleaved tile list for the RADIX buckets of a pass, built on the device (no host round trip) ----------------
// aux (RADIX * 4 + 8 words): row0[s] (first status row of segment s) | sortrank[s] (position of s when the segments are ordered
// by tile count, descending) | snt[k] (tile counts in that order) | P[k] (prefix sums of snt, RADIX + 1 entries) | total.
// Round q of the list holds tiles [g0, g0 + G) (g0 = G * q) of every segment that has them, segments in sorted order.  Tile
// (s, r) of round q sits at A(g0) + B(s) + (r - g0):
//   A(g0) = tiles of the earlier rounds = sum over segments of min(tiles, g0) = g0 * C + (total - P[C]), C = #segments with > g0 tiles;
//   B(s)  = tiles of this round of the segments sorted before s (k = sortrank[s] of them, all with > g0 tiles): the first F of
//           them (F = #segments with >= g0 + G tiles) have G each, the others snt[i] - g0:  G * min(k, F) + (P[k] - P[F]) - g0 * (k - F).
static __global__ void __launch_bounds__(RADIX) seg_tiles_prepare_kernel(const u32* __restrict__ seg_size, u32 tile, int drop_last,
                                                                         u32* __restrict__ aux, u32* __restrict__ total_out) {
    __shared__ u32 nt[RADIX], incl[RADIX], snt[RADIX];
    const int s = threadIdx.x;
    const u32 size = (drop_last && s == RADIX - 1) ? 0u : seg_size[s];
    nt[s] = (size + tile - 1) / tile;
    incl[s] = nt[s];
    __syncthreads();
    for (int o = 1; o < RADIX; o <<= 1) {
        const u32 v = s >= o ? incl[s - o] : 0u;
        __syncthreads();
        incl[s] += v;
        __syncthreads();
    }
    u32 rank = 0;
    for (int q = 0; q < RADIX; ++q) rank += (nt[q] > nt[s] || (nt[q] == nt[s] && q < s)) ? 1u : 0u;
    snt[rank] = nt[s];
    aux[s] = incl[s] - nt[s];                  // row0
    aux[RADIX + s] = rank;                     // sortrank
    __syncthreads();
    aux[2 * RADIX + s] = snt[s];
    u32 p = snt[s];
    incl[s] = p;
    __syncthreads();
    for (int o = 1; o < RADIX; o <<= 1) {
        const u32 v = s >= o ? incl[s - o] : 0u;
        __syncthreads();
        incl[s] += v;
        __syncthreads();
    }
    aux[3 * RADIX + s + 1] = incl[s];          // P[s + 1]
    if (s == 0) aux[3 * RADIX] = 0;
    if (s == RADIX - 1) { aux[4 * RADIX + 1] = incl[s]; *total_out = incl[s]; }
}

static __global__ void __launch_bounds__(256) seg_tiles_fill_kernel(const u32* __restrict__ seg_size, const u32* __restrict__ seg_start, u32 tile,
                                                                    int drop_last, const u32* __restrict__ aux, uint4* __restrict__ tiles) {
    __shared__ u32 row0[RADIX], snt[RADIX], P[RADIX + 1], srank[RADIX];
    for (int i = threadIdx.x; i < RADIX; i += blockDim.x) { row0[i] = aux[i]; srank[i] = aux[RADIX + i]; snt[i] = aux[2 * RADIX + i]; P[i] = aux[3 * RADIX + i]; }
    if (threadIdx.x == 0) P[RADIX] = aux[4 * RADIX];
    __syncthreads();
    const u32 total = P[RADIX];
    const u32 row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= total) return;
    int lo = 0, hi = RADIX;                    // last segment with row0 <= row that has tiles
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (row0[mid] <= row) lo = mid; else hi = mid; }
    const u32 sg = (u32)lo, r = row - row0[sg];
    auto count_above = [&](u32 x) -> u32 {     // number of entries of the descending snt that are > x
        int c0 = 0, c1 = RADIX;
        while (c0 < c1) { const int mid = (c0 + c1) >> 1; if (snt[mid] > x) c0 = mid + 1; else c1 = mid; }
        return (u32)c0;
    };
    const u32 g0 = r - r % TILE_GROUP;         // first tile of the round
    const u32 C = count_above(g0), F = count_above(g0 + TILE_GROUP - 1), k = srank[sg];
    const u32 before = k <= F ? TILE_GROUP * k : TILE_GROUP * F + (P[k] - P[F]) - g0 * (k - F);
    const u32 pos = g0 * C + (total - P[C]) + before + (r - g0);
    const u32 size = (drop_last && sg == RADIX - 1) ? 0u : seg_size[sg];
    const u32 off = r * tile;
    tiles[pos] = make_uint4(seg_start[sg] + off, size - off < tile ? size - off : tile, row, (sg << 20) | r);
}

// tile list of the RADIX segments whose sizes / starts are DEVICE arrays; *d_tiles (workspace `ws_slot`) holds at most
// bound = ceil(n / tile) + RADIX tiles, the exact count is at *d_total (inside the same workspace)
inline int build_seg_tiles_device(tg_ctx* ctx, const u32* d_seg_size, const u32* d_seg_start, size_t n, u32 tile, bool drop_last,
                                  int ws_slot, uint4** d_tiles, const u32** d_total, u32* bound_out) {
    const u32 bound = (u32)((n + tile - 1) / tile) + RADIX;
    unsigned char* base;
    TG_TRY(tg_ws_get(ctx, ws_slot, (size_t)bound * sizeof(uint4) + (4 * RADIX + 8) * 4 + 64, (void**)&base));
    *d_tiles = (uint4*)base;
    u32* aux = (u32*)(base + (size_t)bound * sizeof(uint4));
    u32* total = aux + 4 * RADIX + 4;
    TG_LAUNCH(ctx, seg_tiles_prepare_kernel, 1, RADIX, 0, d_seg_size, tile, drop_last ? 1 : 0, aux, total);
    TG_LAUNCH(ctx, seg_tiles_fill_kernel, (bound + 255) / 256, 256, 0, d_seg_size, d_seg_start, tile, drop_last ? 1 : 0, (const u32*)aux, *d_tiles);
    *d_total = total;
    *bound_out = bound;
    return TG_OK;
}

// chunk geometry of a chunked pass over n items: ~2 chunks per SM, whole tiles
struct ChunkGeom {
    u32 chunk_items;
    int nchunks;
};
template <int WORDS>
inline ChunkGeom chunk_geometry(const tg_ctx* ctx, size_t n) {
    const u32 tile = tile_items<WORDS>();
    const u32 tiles_total = (u32)((n + tile - 1) / tile);
    u32 want = (u32)ctx->sm_count * 2;
    if (want > tiles_total) want = tiles_total;
    if (want == 0) want = 1;
    ChunkGeom g;
    g.chunk_items = ((tiles_total + want - 1) / want) * tile;
    if (g.chunk_items == 0) g.chunk_items = tile;
    g.nchunks = (int)((n + g.chunk_items - 1) / g.chunk_items);
    return g;
}

// Stand-alone stable partition of n items into <= RADIX buckets as a chunked pass (counting read, scan, pass): the
// replacement of partition_items' chained scan.  *d_totals / *d_gbase (device, RADIX u32): bucket sizes and starts.
// Uses the workspace slots WS_SORT_HIST2 (tables), WS_SEG_TILES2 (tile list), WS_SORT_STATUS (scan status).
template <int WORDS, class DigitFn>
int partition_chunked(tg_ctx* ctx, const void* in, void* out, size_t n, const DigitFn& fn, u32** d_totals, u32** d_gbase) {
    typedef typename ItemT<WORDS>::type Item;
    const ChunkGeom g = chunk_geometry<WORDS>(ctx, n);
    const size_t cw = (size_t)(g.nchunks > 0 ? g.nchunks : 1) * RADIX;
    u32* tab;
    TG_TRY(tg_ws_get(ctx, WS_SORT_HIST2, (2 * cw + 2 * RADIX + 16) * 4, (void**)&tab));
    u32* chunkcount = tab;
    u32* chunkbase = tab + cw;
    u32* totals = chunkbase + cw;
    u32* gbase = totals + RADIX;
    if (d_totals) *d_totals = totals;
    if (d_gbase) *d_gbase = gbase;
    if (n == 0) {
        TG_CUDA(ctx, cudaMemsetAsync(totals, 0, 2 * RADIX * 4, ctx->stream));
        return TG_OK;
    }
    TG_LAUNCH_T(ctx, TG_K_RADIX_HIST, (chunk_hist_kernel<WORDS, DigitFn, false>), g.nchunks, 512, 0, (const Item*)in, (u32)n,
                g.chunk_items, fn, chunkcount, (u64*)nullptr);
    TG_LAUNCH(ctx, chunk_scan_kernel, 1, 4 * RADIX, 0, chunkcount, g.nchunks, totals, gbase, chunkbase);
    std::vector<u32> chunk_size(g.nchunks, g.chunk_items);
    chunk_size[g.nchunks - 1] = (u32)(n - (size_t)(g.nchunks - 1) * g.chunk_items);
    // (pinned staging buffer 0: every operator ends with a stream synchronisation and the uses of one staging buffer inside an
    // operator are separated by one, so the list staged there before has been copied)
    uint4* d_tiles;
    u32 total = 0;
    TG_TRY(build_tile_list(ctx, g.nchunks, chunk_size.data(), tile_items<WORDS>(), 0, WS_SEG_TILES2, &d_tiles, &total));
    u32* status;
    TG_TRY(tg_ws_get(ctx, WS_SORT_STATUS, (size_t)total * RADIX * 4, (void**)&status));
    TG_CUDA(ctx, cudaMemsetAsync(status, 0, (size_t)total * RADIX * 4, ctx->stream));
    SegList sl = { d_tiles, chunkbase, total, nullptr };
    return launch_partition_seg<WORDS, DigitFn>(ctx, in, out, (u32)n, fn, status, sl);
}

}  // namespace tgp
