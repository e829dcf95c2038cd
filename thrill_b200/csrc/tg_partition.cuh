// tg_partition.cuh — the stable multi-way (<= 256 buckets) partition pass shared by
//   * the local sort                (digit = 8 key bits)                            tg_radix_sort.cu
//   * the splitter classify/scatter (digit = destination worker by the splitters)   tg_sample_sort.cu
//   * the hash aggregation          (digit = a byte of Hash128to64(0,key), or % p)  tg_reduce.cu
//
// Persistent CTAs walk a list of tiles in static round-robin order.  A tile (128 KB) is staged into shared memory by
// the TMA unit (cp.async.bulk + mbarrier; the next tile's copy starts as soon as the current tile is in registers and lands
// while it is processed), ranked stably with warp-synchronous ballots + warp-private counters, positioned by a chained scan
// with batched decoupled look-back over the tiles of its SEGMENT (the whole input for the plain pass; see tg_segmented.cuh for
// the chunked and segmented passes whose tile lists make a tile wait at most for the few tiles of its group), reordered by
// digit through a half-tile exchange buffer in two rounds and written out so that consecutive threads write consecutive
// addresses.
// HBM traffic: read n*s + write n*s + ~1.5 % scan state.
#pragma once
#include "tg_common.cuh"

namespace tgp {

constexpr int RADIX_BITS = 8;
constexpr int RADIX = 1 << RADIX_BITS;

constexpr u32 FLAG_PARTIAL = 1u << 30;
constexpr u32 FLAG_INCL = 2u << 30;
constexpr u32 VALUE_MASK = (1u << 30) - 1;

template <int WORDS> struct ItemT;
template <> struct ItemT<1> { typedef u64 type; };
template <> struct ItemT<2> { typedef ulonglong2 type; };

__device__ __forceinline__ u64 item_word(const u64& v, int) { return v; }
__device__ __forceinline__ u64 item_word(const ulonglong2& v, int w) { return w ? v.y : v.x; }

// digit functors: u32 operator()(item, position of the item in the input) -> [0, RADIX)
struct RadixDigit {
    int word, shift;
    u32 flip;
    static constexpr bool kStoreDigit = false;      // cheap to recompute in the write-out
    static constexpr bool kHasDrop = false;         // true: digit RADIX-1 means "leave this item out of the output"
    static constexpr int kScratch = 0;              // bytes of CTA shared memory the functor wants (filled by init_shared)
    __device__ __forceinline__ void init() {}
    template <class Item>
    __device__ __forceinline__ u32 operator()(const Item& v, u32) const {
        return ((u32)(item_word(v, word) >> shift) & (RADIX - 1)) ^ flip;
    }
};

// warp-wide "which lanes hold the same 8-bit digit": 8 ballots, each fixed up for the lane's own bit.
// Written in PTX so that ptxas emits, per bit, one LOP3 with a predicate result, one VOTE and one predicated
// NOT, and 3-input LOP3s for the final AND (the C++ form compiled to ~45 instructions per call, this one to 28;
// match.any.sync is a multi-cycle instruction of the ADU pipe, where this form stays on the integer and vote pipes).
__device__ __forceinline__ u32 match_digit8(u32 d) {
    u32 peers;
    asm volatile(
        "{\n"
        ".reg .pred p0, p1, p2, p3, p4, p5, p6, p7;\n"
        ".reg .b32 m0, m1, m2, m3, m4, m5, m6, m7, t;\n"
        "and.b32 t, %1, 1;   setp.ne.u32 p0, t, 0;\n"
        "and.b32 t, %1, 2;   setp.ne.u32 p1, t, 0;\n"
        "and.b32 t, %1, 4;   setp.ne.u32 p2, t, 0;\n"
        "and.b32 t, %1, 8;   setp.ne.u32 p3, t, 0;\n"
        "and.b32 t, %1, 16;  setp.ne.u32 p4, t, 0;\n"
        "and.b32 t, %1, 32;  setp.ne.u32 p5, t, 0;\n"
        "and.b32 t, %1, 64;  setp.ne.u32 p6, t, 0;\n"
        "and.b32 t, %1, 128; setp.ne.u32 p7, t, 0;\n"
        "vote.sync.ballot.b32 m0, p0, 0xffffffff;\n"
        "vote.sync.ballot.b32 m1, p1, 0xffffffff;\n"
        "vote.sync.ballot.b32 m2, p2, 0xffffffff;\n"
        "vote.sync.ballot.b32 m3, p3, 0xffffffff;\n"
        "vote.sync.ballot.b32 m4, p4, 0xffffffff;\n"
        "vote.sync.ballot.b32 m5, p5, 0xffffffff;\n"
        "vote.sync.ballot.b32 m6, p6, 0xffffffff;\n"
        "vote.sync.ballot.b32 m7, p7, 0xffffffff;\n"
        "@!p0 not.b32 m0, m0;\n"
        "@!p1 not.b32 m1, m1;\n"
        "@!p2 not.b32 m2, m2;\n"
        "@!p3 not.b32 m3, m3;\n"
        "@!p4 not.b32 m4, m4;\n"
        "@!p5 not.b32 m5, m5;\n"
        "@!p6 not.b32 m6, m6;\n"
        "@!p7 not.b32 m7, m7;\n"
        "lop3.b32 t, m0, m1, m2, 0x80;\n"
        "lop3.b32 t, t, m3, m4, 0x80;\n"
        "lop3.b32 t, t, m5, m6, 0x80;\n"
        "and.b32 %0, t, m7;\n"
        "}\n"
        : "=r"(peers)
        : "r"(d));
    return peers;
}

// Launch configuration of the partition pass: 512 threads per CTA, each owning 32 8-byte words (32 u64 items or 16 16-byte
// items), one CTA per SM: tiles of 16384 items of 8 bytes, 8192 of 16 bytes (128 KB).  The tile size is what sets the pass's
// DRAM efficiency: a tile's write-out is one run per digit, 256 runs of TILE/256 items on average at arbitrary offsets, and
// the longer the runs the fewer partial 32-byte sectors the writes leave (DESIGN.md §5 has the measured per-tile-size times).
// A 128 KB tile cannot be double buffered, so the landing buffer is single (the next tile's copy is started as soon as the
// current tile's items are in registers) and the exchange buffer holds half a tile: the write-out runs in two rounds.
constexpr int PEER_MAX = 32;        // destinations of a partition pass that stores into peer windows (<= TG_MAX_RANKS used)
template <int WORDS, bool STORE = true, bool PEER = false, int SCRATCH = 0>
struct PartCfg {
    static constexpr int THREADS = 512;
    static constexpr int MIN_BLOCKS = 1;                     // CTAs per SM
    static constexpr int ITEM_BYTES = 8 * WORDS;
    static constexpr int ITEMS = 32 / WORDS;                 // items per thread
    static constexpr int TILE = THREADS * ITEMS;             // items per tile (< 65536: 16-bit warp counters and ranks)
    static constexpr int HALF = TILE / 2;                    // items per exchange round
    static constexpr int TILE_BYTES = TILE * ITEM_BYTES;
    static constexpr int NWARPS = THREADS / 32;
    static constexpr int BUF_BYTES = TILE_BYTES + (WORDS == 1 ? 16 : 0);      // + one 16-byte granule: tiles that start at an odd 8-byte item
    // landing buffer | exchange buffer [HALF] | warp counters [NWARPS][RADIX] | goff [RADIX] | warp_tot [16] | mbar | digit
    // bytes [HALF] (only if the digit function's result is kept, kStoreDigit) | peer pointers [PEER_MAX] | functor scratch | slack
    static constexpr int SMEM = BUF_BYTES + HALF * ITEM_BYTES + NWARPS * RADIX * (int)sizeof(unsigned short) + RADIX * 4 + 64 + 16 + (STORE ? HALF : 0) + (PEER ? PEER_MAX * 8 : 0) + SCRATCH + 128;
    static_assert(SMEM <= 227 * 1024, "partition pass: shared memory of one CTA");
};
// Tiles of one segment that the tile list of a segmented pass (tg_segmented.cuh) puts next to each other.  Neighbouring tiles
// of a segment write neighbouring runs of every digit, so a group that runs in one wave writes each digit as one run G tiles
// long instead of G isolated ones (DESIGN.md §5 has the measured per-group-size times).  A group member finds the counts of
// the members before it with the first batch of its look-back (G <= LB in partition_kernel).
constexpr u32 TILE_GROUP = 8;

// What the write-out of a pass does besides storing each item at its position: nothing (NoFinish), or, in the radix sort's
// last prefix pass, ordering the groups of equal key prefix that lie inside the exchange buffer (FusedFinish,
// tg_radix_sort.cu).  kOn selects the write-out at compile time: the passes without it compile as before.
struct NoFinish {
    static constexpr bool kOn = false;
};

// exclusive scan of npass digit histograms -> global bases; skip[p] = 1 if one bin holds everything
static __global__ void scan_hist_kernel(const u32* __restrict__ ghist, u32* __restrict__ gbase, u32* __restrict__ skip,
                                 int npass, u32 n) {
    __shared__ u32 warp_tot[RADIX / 32];
    const int d = threadIdx.x;      // RADIX threads
    for (int p = 0; p < npass; ++p) {
        u32 c = ghist[p * RADIX + d];
        u32 incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            u32 t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((d & 31) >= o) incl += t;
        }
        if ((d & 31) == 31) warp_tot[d >> 5] = incl;
        __syncthreads();
        u32 add = 0;
        for (int w = 0; w < (d >> 5); ++w) add += warp_tot[w];
        gbase[p * RADIX + d] = add + incl - c;
        u32 full = __syncthreads_or(c == n);
        if (d == 0 && skip) skip[p] = full ? 1u : 0u;
        __syncthreads();
    }
}

__device__ __forceinline__ u32 lds_u32(u32 addr) {
    u32 v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts_u32(u32 addr, u32 v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
// the warp-private digit counters are 16-bit (a tile holds < 65536 items): half the shared memory of 32-bit counters
typedef unsigned short cnt_t;
__device__ __forceinline__ u32 lds_cnt(u32 addr) {
    u32 v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts_cnt(u32 addr, u32 v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }

// stable rank of the warp's ITEMS rows inside the (warp, digit) groups.  Every lane reads its group's counter, the
// lowest lane of the group bumps it (same warp, program order: the read precedes the write).  whist_w = shared
// address of the warp's RADIX counters.  rank = position inside the group | digit << 16 (if STORE).
template <bool FULL, bool STORE, int ITEMS, class Item, class DigitFn>
__device__ __forceinline__ void rank_rows(const Item (&key)[ITEMS], u32 (&rank)[ITEMS], const DigitFn& fn, u32 whist_w,
                                          u32 pos0, u32 tile_base, u32 tile_valid, u32 lt) {
#pragma unroll
    for (int i = 0; i < ITEMS; ++i) {
        const u32 p = pos0 + i * 32;
        u32 d = fn(key[i], tile_base + p);
        if (!FULL && p >= tile_valid) d = RADIX - 1;
        const u32 a = whist_w + d * (u32)sizeof(cnt_t);
        const u32 old = lds_cnt(a);
        const u32 peers = match_digit8(d);
        const u32 below = peers & lt;
        if (below == 0) sts_cnt(a, old + __popc(peers));
        rank[i] = old + __popc(below);
        if (STORE) rank[i] |= d << 16;
        __syncwarp();
    }
}

// Ranking for passes that need not be stable (items that are nothing but their key: equal keys are indistinguishable, and the
// pass is the first one on its part of the key — the most significant digit, or the first of the digits below it): every lane
// takes its rank from a shared-memory atomic on its digit's warp-private counter (two 16-bit counters per 32-bit word).  One
// ATOMS on the ADU pipe replaces the 28-instruction ballot match and the counter read/write on the ALU pipe, the busiest one
// of this kernel.
template <bool STORE, int ITEMS, class Item, class DigitFn>
__device__ __forceinline__ void rank_rows_unstable(const Item (&key)[ITEMS], u32 (&rank)[ITEMS], const DigitFn& fn, u32 whist_w,
                                                   u32 pos0, u32 tile_base) {
#pragma unroll
    for (int i = 0; i < ITEMS; ++i) {
        const u32 d = fn(key[i], tile_base + pos0 + i * 32);
        const u32 sh = (d & 1u) << 4;
        u32 old;
        asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(whist_w + (d >> 1) * 4u), "r"(1u << sh) : "memory");
        rank[i] = (old >> sh) & 0xffffu;
        if (STORE) rank[i] |= d << 16;
    }
}

// Segmented operation: the input is a sequence of independent segments (e.g. the 256 buckets of a previous pass on
// a more significant digit); every segment is partitioned on its own, with its own bases and its own chained scan.
// The tile list interleaves groups of TILE_GROUP neighbouring tiles of the segments, so the tile the scan of a group's
// first tile depends on (the previous tile of the same segment) was processed a whole wave of CTAs earlier: the look-back
// finds its inclusive prefix with one load.  The other members of a group run at the same time as the members before
// them, which publish their counts right after ranking; one batch of the look-back reaches back past the group.
//   tiles[j] = { first item, items (<= TILE), status row, (segment << 20) | index of the tile inside its segment }
//   status rows of one segment are consecutive; segbase[segment][RADIX] = output position of the segment's digit d.
struct SegList {
    const uint4* tiles;
    const u32* segbase;
    u32 num_tiles;                  // number of tiles, or an upper bound of it if num_tiles_dev is set
    const u32* num_tiles_dev;       // device-built lists (build_seg_tiles_device): the exact count lives on the device
};
__device__ __forceinline__ u32 seg_num_tiles(const SegList& sl) { return sl.num_tiles_dev ? __ldg(sl.num_tiles_dev) : sl.num_tiles; }

// One tile: rank -> start the next tile's copy -> per-digit counts (published for the chained scan) -> scatter the first
// half of the tile's positions into the exchange buffer while the look-back loads are in flight -> resolve the look-back ->
// coalesced write-out -> scatter and write out the second half.
// PEER: the buckets are destination workers; bucket d is written to dbase[d][position], where dbase[d] points into worker
// d's exchange window (mapped peer memory: the stores travel over NVLink) biased so that `position` is the position the
// plain pass would have used in `out` — the Alltoallv of the reference's MixStream exchange happens inside the pass.
// Fin: the write-out (NoFinish, or the radix sort's fused finishing pass: see FusedFinish in tg_radix_sort.cu).
template <int WORDS, class DigitFn, bool SEG, bool PEER, bool UNSTABLE, class Fin = NoFinish>
__global__ void __launch_bounds__(PartCfg<WORDS>::THREADS, PartCfg<WORDS>::MIN_BLOCKS)
partition_kernel(const typename ItemT<WORDS>::type* __restrict__ in, typename ItemT<WORDS>::type* __restrict__ out,
                 u32 n, const DigitFn fn_param, const u32* __restrict__ gbase, u32* __restrict__ status, const SegList sl,
                 typename ItemT<WORDS>::type* const* __restrict__ dbase, const Fin fin) {
    typedef typename ItemT<WORDS>::type Item;
    typedef PartCfg<WORDS, DigitFn::kStoreDigit, PEER, DigitFn::kScratch> C;
    constexpr int THREADS = C::THREADS, ITEMS = C::ITEMS, TILE = C::TILE, HALF = C::HALF, NWARPS = C::NWARPS;
    // look-back batch (predecessors fetched concurrently); the first batch is requested before the scatter.  Inside a segment
    // the predecessor of a group's first tile usually finished a wave ago and one load finds its inclusive prefix; the other
    // members of a group, a dominant segment's tiles at the tail of the list and the plain chained scan run concurrently with
    // their predecessors
    constexpr int LB = 8;
    static_assert(TILE_GROUP <= (u32)LB, "a group member reaches past its group's first tile with one batch");
    static_assert(THREADS >= RADIX, "one thread per digit in the scan phases");
    static_assert(!Fin::kOn || (SEG && !PEER && !UNSTABLE && !DigitFn::kStoreDigit && !DigitFn::kHasDrop),
                  "the fused finishing pass is a stable segmented pass of the radix sort");

    // plain pointer arithmetic on the shared array keeps the shared address space (LDS/STS, 32-bit addresses)
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    Item* const buf = reinterpret_cast<Item*>(smem_raw);                         // landing buffer
    Item* const xbuf = reinterpret_cast<Item*>(smem_raw + C::BUF_BYTES);         // exchange buffer [HALF]
    cnt_t* const whist = reinterpret_cast<cnt_t*>(xbuf + HALF);                  // [NWARPS][RADIX]
    u32* const goff = reinterpret_cast<u32*>(whist + NWARPS * RADIX);            // [RADIX]
    u32* const warp_tot = goff + RADIX;                                          // [16]
    u64* const mbar = reinterpret_cast<u64*>(warp_tot + 16);                     // the landing buffer's (16 bytes reserved)
    unsigned char* const dig = reinterpret_cast<unsigned char*>(mbar + 2);       // [HALF], only if kStoreDigit
    Item** const dptr = reinterpret_cast<Item**>(dig + (DigitFn::kStoreDigit ? HALF : 0));      // [PEER_MAX], only if PEER
    unsigned char* const fscratch = reinterpret_cast<unsigned char*>(dptr + (PEER ? PEER_MAX : 0));  // [kScratch], the functor's

    DigitFn fn = fn_param;
    fn.init();
    if constexpr (DigitFn::kScratch > 0) fn.init_shared(fscratch, (int)threadIdx.x, THREADS);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 num_tiles = SEG ? seg_num_tiles(sl) : (n + TILE - 1) / TILE;
    const u32 lt = lanemask_lt();
    cnt_t* const whist_w = whist + warp * RADIX;
    const u32 whist_w_a = smem_u32(whist_w);
    const u32 wbase = warp * 32 * ITEMS;

    // tile j: first item, items, status row, index inside its segment, segment
    struct TileInfo { u32 start, len, row, idx, seg; };
    auto tile_info = [&](u32 j) -> TileInfo {
        TileInfo ti;
        if (SEG) {
            const uint4 d = __ldg(&sl.tiles[j]);
            ti.start = d.x; ti.len = d.y; ti.row = d.z; ti.idx = d.w & 0xfffffu; ti.seg = d.w >> 20;
        }
        else {
            ti.start = j * TILE;
            ti.len = (n - ti.start < (u32)TILE) ? n - ti.start : (u32)TILE;
            ti.row = j; ti.idx = j; ti.seg = 0;
        }
        return ti;
    };
    // A whole tile is fetched by the TMA unit (16-byte granules): a tile of 8-byte items that starts at an odd item is
    // fetched from one item earlier, one granule longer (tma_shift = 1), if that stays inside the array; anything else
    // by ordinary loads.
    auto tma_shift = [&](const TileInfo& ti) -> u32 { return WORDS == 1 ? (ti.start & 1u) : 0u; };
    auto tma_ok = [&](const TileInfo& ti) -> bool {
        if (ti.len != (u32)TILE) return false;
        return tma_shift(ti) == 0 || (size_t)ti.start + TILE + 1 <= n;
    };

    if (tid == 0) {
        mbar_init(&mbar[0], 1);
        mbar_fence_init();
    }
    if (PEER && tid < PEER_MAX) dptr[tid] = dbase[tid];
    __syncthreads();

    u32 j = blockIdx.x;
    TileInfo tnext = tile_info(j < num_tiles ? j : 0);        // descriptors of the tiles of the next two iterations
    TileInfo tnext2 = tile_info(j + gridDim.x < num_tiles ? j + gridDim.x : 0);
    if (j < num_tiles) {
        const TileInfo t0 = tnext;
        if (tid == 0 && tma_ok(t0)) {
            const u32 sh = tma_shift(t0), bytes = C::TILE_BYTES + 16 * sh;
            mbar_expect_tx(&mbar[0], bytes);
            bulk_g2s(buf, in + (t0.start - sh), bytes, &mbar[0]);
        }
    }
    u32 phase = 0;        // parity of the next completion of mbar[0]

    for (; j < num_tiles; j += gridDim.x) {
        const TileInfo ti = tnext;
        // (descriptors are fetched two tiles ahead: the one of the next tile, needed below to start its TMA copy, was
        // requested a whole tile ago)
        if (j + gridDim.x < num_tiles) tnext = tnext2;
        if (SEG ? (j + 2 * gridDim.x < num_tiles) : true) tnext2 = tile_info(j + 2 * gridDim.x);
        const u32 tile_base = ti.start;
        const bool full_tile = ti.len == (u32)TILE;
        const u32 tile_valid = ti.len;
        const bool by_tma = tma_ok(ti);
        const u32* const gb = SEG ? sl.segbase + (size_t)ti.seg * RADIX : gbase;

        // zero this warp's private digit counters
#pragma unroll
        for (int i = 0; i < RADIX / 64; ++i) reinterpret_cast<u32*>(whist_w)[i * 32 + lane] = 0;

        // ---- items to registers: warp w owns tile positions [w*32*ITEMS, (w+1)*32*ITEMS), round-striped.
        // Positions past the end of a partial tile get digit RADIX-1: the stable ranking puts them behind every
        // valid item, so they land past tile_valid and are never written.
        Item key[ITEMS];
        u32 rank[ITEMS];                 // rank inside the (warp, digit) group | digit << 16 (if kStoreDigit)
        if (by_tma) {
            mbar_wait(&mbar[0], phase);
            phase ^= 1u;
            const Item* src = buf + tma_shift(ti) + wbase + lane;
#pragma unroll
            for (int i = 0; i < ITEMS; ++i) key[i] = src[i * 32];
        }
        else if (full_tile) {
            const Item* src = in + tile_base + wbase + lane;
#pragma unroll
            for (int i = 0; i < ITEMS; ++i) key[i] = src[i * 32];
        }
        else {
#pragma unroll
            for (int i = 0; i < ITEMS; ++i) {
                u32 p = wbase + i * 32 + lane;
                if (p < tile_valid) key[i] = in[(size_t)tile_base + p];
            }
        }
        __syncwarp();

        // ---- stable rank inside the warp (partial tiles always carry the digit along: padding has none)
        if (full_tile && UNSTABLE) rank_rows_unstable<DigitFn::kStoreDigit>(key, rank, fn, whist_w_a, wbase + lane, tile_base);
        else if (full_tile) rank_rows<true, DigitFn::kStoreDigit>(key, rank, fn, whist_w_a, wbase + lane, tile_base, tile_valid, lt);
        else rank_rows<false, true>(key, rank, fn, whist_w_a, wbase + lane, tile_base, tile_valid, lt);
        __syncthreads();      // all items are in registers (buf is free), all warp counters final

        // start the CTA's next tile (TMA unit, async proxy) into the landing buffer: it has the rest of this tile's time to land
        if (tid == 0 && j + gridDim.x < num_tiles) {
            const TileInfo tn = tnext;
            if (tma_ok(tn)) {
                const u32 sh = tma_shift(tn), bytes = C::TILE_BYTES + 16 * sh;
                fence_proxy_async();
                mbar_expect_tx(&mbar[0], bytes);
                bulk_g2s(buf, in + (tn.start - sh), bytes, &mbar[0]);
            }
        }

        // ---- per-digit tile count; publish PARTIAL as early as possible; start the look-back loads
        u32 count = 0, my_start = 0;
        u32 lbv[SEG ? 1 : LB];
        const u32 my_gb = tid < RADIX ? __ldg(&gb[tid]) : 0u;      // (requested early: needed after the look-back)
        u32* const my_status = status + (size_t)ti.row * RADIX + tid;       // predecessor k: my_status - k * RADIX
        if (tid < RADIX) {
#pragma unroll
            for (int w = 0; w < NWARPS; ++w) count += whist[w * RADIX + tid];
            u32 pub = count;
            if (!full_tile && tid == RADIX - 1) pub -= (u32)TILE - tile_valid;      // padding is not data
            st_relaxed_u32(my_status, pub | (ti.idx == 0 ? FLAG_INCL : FLAG_PARTIAL));
            if (SEG) {
                // a group's first tile: the predecessor finished a wave of CTAs ago, one load nearly always finds its inclusive prefix
                lbv[0] = ti.idx > 0 ? ld_relaxed_u32(my_status - RADIX) : FLAG_INCL;
            }
            else {
#pragma unroll
                for (int k = 0; k < LB; ++k)
                    lbv[k] = ((u32)(k + 1) <= ti.idx) ? ld_relaxed_u32(my_status - (size_t)(k + 1) * RADIX) : FLAG_INCL;
            }
            u32 incl = count;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                u32 v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            if (lane == 31) warp_tot[warp] = incl;
            my_start = incl - count;             // completed below with the preceding warps' totals
        }
        __syncthreads();
        if (tid < RADIX) {
            for (int w = 0; w < warp; ++w) my_start += warp_tot[w];
            // warp counters -> tile-local write positions of each (warp, digit) group
            u32 off = my_start;
#pragma unroll
            for (int w = 0; w < NWARPS; ++w) {
                u32 c = whist[w * RADIX + tid];
                whist[w * RADIX + tid] = (cnt_t)off;
                off += c;
            }
        }
        __syncthreads();

        // ---- two exchange rounds by tile-local position q: round r moves the items with q in [r*HALF, (r+1)*HALF) through the
        // exchange buffer (any digit skew takes exactly two rounds; a digit run may straddle them)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            // ---- scatter registers -> digit-ordered exchange buffer
            if (full_tile && !DigitFn::kStoreDigit) {
#pragma unroll
                for (int i = 0; i < ITEMS; ++i) {
                    u32 d = fn(key[i], 0);
                    u32 q = lds_cnt(whist_w_a + d * (u32)sizeof(cnt_t)) + rank[i] - (u32)(r * HALF);
                    if (q < (u32)HALF) xbuf[q] = key[i];
                }
            }
            else {
#pragma unroll
                for (int i = 0; i < ITEMS; ++i) {
                    u32 d = rank[i] >> 16;
                    u32 q = lds_cnt(whist_w_a + d * (u32)sizeof(cnt_t)) + (rank[i] & 0xffffu) - (u32)(r * HALF);
                    if (q < (u32)HALF) {
                        xbuf[q] = key[i];
                        if (DigitFn::kStoreDigit) dig[q] = (unsigned char)d;
                    }
                }
            }

            // ---- decoupled look-back inside the tile's segment (threads 0..RADIX-1, one digit each, LB predecessors per
            // round trip; the first batch was requested before the first scatter)
            if (r == 0 && tid < RADIX) {
                u32 excl = 0;
                if (ti.idx > 0) {
                    u32 back = 1;              // distance of the next predecessor to consume
                    bool done = false;
                    u32 v[LB];
                    if (SEG) {
                        // fast path: the prefetched predecessor carries an inclusive prefix.  Otherwise (the other members of a group,
                        // tiles of a dominant segment that run at the same time) continue with batches of LB predecessors per round trip.
                        if (lbv[0] & FLAG_INCL) { excl = lbv[0] & VALUE_MASK; done = true; }
                        else {
                            v[0] = lbv[0];
#pragma unroll
                            for (int k = 1; k < LB; ++k)
                                v[k] = (back + k <= ti.idx) ? ld_relaxed_u32(my_status - (size_t)(back + k) * RADIX) : FLAG_INCL;
                        }
                    }
                    else {
#pragma unroll
                        for (int k = 0; k < LB; ++k) v[k] = lbv[k];
                    }
                    while (!done) {
                        bool stalled = false;
#pragma unroll
                        for (int k = 0; k < LB; ++k) {
                            if (!done && !stalled) {
                                if (v[k] & FLAG_INCL) { excl += v[k] & VALUE_MASK; done = true; }
                                else if (v[k] & FLAG_PARTIAL) { excl += v[k] & VALUE_MASK; back++; }
                                else stalled = true;
                            }
                        }
                        if (done) break;
#pragma unroll
                        for (int k = 0; k < LB; ++k)
                            v[k] = (back + k <= ti.idx) ? ld_relaxed_u32(my_status - (size_t)(back + k) * RADIX) : FLAG_INCL;
                    }
                    u32 pub = count;
                    if (!full_tile && tid == RADIX - 1) pub -= (u32)TILE - tile_valid;
                    st_relaxed_u32(my_status, (excl + pub) | FLAG_INCL);
                }
                goff[tid] = my_gb + excl - my_start;
            }
            __syncthreads();

            // ---- coalesced write-out: consecutive threads write consecutive addresses inside a digit run
            if constexpr (Fin::kOn) {
                const u32 q0r = (u32)(r * HALF);
                const u32 nr = tile_valid > q0r ? (tile_valid - q0r < (u32)HALF ? tile_valid - q0r : (u32)HALF) : 0u;
                fin.template write_out<THREADS, HALF / THREADS>(xbuf, nr, q0r, goff, fn, out, tid);
            }
            else {
                const Item* const bufp = xbuf + tid;
                const u32 q0 = (u32)(r * HALF) + tid;        // tile-local position of bufp[0]
                if (full_tile) {
#pragma unroll
                    for (int i = 0; i < HALF / THREADS; ++i) {
                        Item v = bufp[i * THREADS];
                        u32 d = DigitFn::kStoreDigit ? (u32)dig[i * THREADS + tid] : fn(v, 0);
                        if (DigitFn::kHasDrop && d == RADIX - 1) continue;
                        if (PEER) dptr[d][goff[d] + q0 + (u32)(i * THREADS)] = v;
                        else out[goff[d] + q0 + (u32)(i * THREADS)] = v;
                    }
                }
                else {
#pragma unroll
                    for (int i = 0; i < HALF / THREADS; ++i) {
                        if (q0 + (u32)(i * THREADS) < tile_valid) {
                            Item v = bufp[i * THREADS];
                            u32 d = DigitFn::kStoreDigit ? (u32)dig[i * THREADS + tid] : fn(v, 0);
                            if (DigitFn::kHasDrop && d == RADIX - 1) continue;
                            if (PEER) dptr[d][goff[d] + q0 + (u32)(i * THREADS)] = v;
                            else out[goff[d] + q0 + (u32)(i * THREADS)] = v;
                        }
                    }
                }
            }
            __syncthreads();      // the exchange buffer is free for the next round or tile
        }
    }
}

template <int WORDS>
__global__ void copy_items_kernel(const typename ItemT<WORDS>::type* __restrict__ in,
                                  typename ItemT<WORDS>::type* __restrict__ out, size_t n) {
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = in[i];
}

// items per tile (the host builds tile lists and chunk geometry with it)
template <int WORDS>
constexpr u32 tile_items() { return (u32)PartCfg<WORDS>::TILE; }
template <int WORDS>
constexpr u32 num_tiles_for(size_t n) { return (u32)((n + tile_items<WORDS>() - 1) / tile_items<WORDS>()); }

template <int WORDS, class DigitFn, bool SEG, bool PEER = false, bool UNSTABLE = false, class Fin = NoFinish>
int launch_partition_v(tg_ctx* ctx, const void* in, void* out, u32 n, const DigitFn& fn, const u32* gbase, u32* status,
                       const SegList& sl, typename ItemT<WORDS>::type* const* dbase = nullptr, const Fin& fin = Fin()) {
    typedef typename ItemT<WORDS>::type Item;
    typedef PartCfg<WORDS, DigitFn::kStoreDigit, PEER, DigitFn::kScratch> C;
    auto kern = partition_kernel<WORDS, DigitFn, SEG, PEER, UNSTABLE, Fin>;
    int ctas_per_sm = 0;
    auto it = ctx->kernel_cfg.find((const void*)kern);
    if (it != ctx->kernel_cfg.end()) ctas_per_sm = it->second;
    else {
        TG_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
        // the look-back needs every CTA of the grid resident: size the grid from the real occupancy
        TG_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, kern, C::THREADS, C::SMEM));
        if (ctas_per_sm < 1) return tg_set_error(ctx, TG_ERR_CUDA, "partition kernel does not fit on an SM");
        if (ctas_per_sm > C::MIN_BLOCKS) ctas_per_sm = C::MIN_BLOCKS;
        ctx->kernel_cfg[(const void*)kern] = ctas_per_sm;
    }
    u32 num_tiles = SEG ? sl.num_tiles : (n + C::TILE - 1) / C::TILE;
    if (num_tiles == 0) return TG_OK;
    int grid = ctx->sm_count * ctas_per_sm;
    if (grid > (int)num_tiles) grid = (int)num_tiles;
    TG_LAUNCH_T(ctx, TG_K_PARTITION, kern, grid, C::THREADS, C::SMEM, (const Item*)in, (Item*)out, n, fn, gbase, status, sl, dbase, fin);
    return TG_OK;
}

// launch one partition pass with precomputed global bases (status must be zeroed, num_tiles*RADIX words)
template <int WORDS, class DigitFn>
int launch_partition(tg_ctx* ctx, const void* in, void* out, u32 n, const DigitFn& fn, const u32* gbase, u32* status) {
    return launch_partition_v<WORDS, DigitFn, false>(ctx, in, out, n, fn, gbase, status, SegList{ nullptr, nullptr, 0, nullptr });
}

// one partition pass over independent segments (see SegList) of an array of n items; status = sl.num_tiles * RADIX zeroed words
template <int WORDS, class DigitFn>
int launch_partition_seg(tg_ctx* ctx, const void* in, void* out, u32 n, const DigitFn& fn, u32* status, const SegList& sl) {
    return launch_partition_v<WORDS, DigitFn, true>(ctx, in, out, n, fn, nullptr, status, sl);
}

// one segmented pass that need not be stable (see rank_rows_unstable)
template <int WORDS, class DigitFn>
int launch_partition_seg_unstable(tg_ctx* ctx, const void* in, void* out, u32 n, const DigitFn& fn, u32* status, const SegList& sl) {
    return launch_partition_v<WORDS, DigitFn, true, false, true>(ctx, in, out, n, fn, nullptr, status, sl);
}

// one segmented partition pass whose buckets are destination workers: bucket d goes to dbase[d] (device array of PEER_MAX
// pointers into the peers' exchange windows, see tg_exchange.cuh)
template <int WORDS, class DigitFn>
int launch_partition_peer(tg_ctx* ctx, const void* in, u32 n, const DigitFn& fn, u32* status, const SegList& sl,
                          typename ItemT<WORDS>::type* const* dbase) {
    return launch_partition_v<WORDS, DigitFn, true, true>(ctx, in, nullptr, n, fn, nullptr, status, sl, dbase);
}

}  // namespace tgp
