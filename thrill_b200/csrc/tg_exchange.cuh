// tg_exchange.cuh — the all-to-all exchange of the collective operators, fused into the partition pass.
//
// Reference path replaced: data::MixStream / CatStream writers of SortNode::TransmitItems (api/sort.hpp:434-535, :615-641)
// and of ReducePrePhaseEmitter (core/reduce_pre_phase.hpp:57-61, api/reduce_by_key.hpp:109-114): every item is appended
// to the Block stream of its destination worker, the multiplexer ships the Blocks (data/mix_stream.cpp:52-236).
//
// Here every worker owns an EXCHANGE WINDOW in its HBM that all peers of the job have mapped (CUDA IPC between the
// one-process-per-GPU workers, plain peer access between the worker threads of one Thrill process).  One exchange is
//   1. chunk histograms of the destination digit (one counting read)                                 chunk_hist_kernel
//   2. ncclAllGather of the p per-destination counts of every worker -> the p x p count matrix (the only host round trip:
//      every rank derives every rank's receive size from it, so window growth / errors are decided identically everywhere)
//   3. the stable partition pass with PEER = true: bucket d is stored straight into worker d's window at this worker's
//      offset (after the items of the lower ranks), over NVLink — classification, scatter and Alltoallv are ONE kernel
//   4. a tiny collective as the "all stores have landed" barrier.
// The received items lie grouped by source worker in rank order, each group in the sender's input order — the order
// CatStream delivers (stable).  TG_EXCHANGE=nccl (or peers that cannot map each other) selects the two-step form
// instead: local partition, then grouped ncclSend/ncclRecv into the window.
#pragma once
#include "tg_segmented.cuh"

namespace tgp {

struct XchgResult {
    void* d_recv = nullptr;                 // the received items (this worker's window)
    u64 n_recv = 0;
    u64 recv_cnt[TG_MAX_RANKS] = { 0 };     // items received from each source rank (rank order = layout order)
    u64 send_cnt[TG_MAX_RANKS] = { 0 };
};

// tg_exchange.cu
int xwin_negotiate(tg_ctx* ctx);                                    // collective, first use: decides P2P vs NCCL mode
int xwin_ensure(tg_ctx* ctx, size_t bytes_all_ranks);               // collective: every rank's window >= bytes
int xwin_barrier(tg_ctx* ctx);                                      // stream-ordered cross-rank barrier
int xchg_counts(tg_ctx* ctx, const u32* d_totals, int item_bytes, XchgResult* res, u64* need_bytes_max);
const u32* xchg_matrix(tg_ctx* ctx);                                // after xchg_counts: the p x p count matrix (host)
// the destination pointers of worker me's peer-store pass (device, PEER_MAX pointers in a workspace slot)
int xchg_upload_dest(tg_ctx* ctx, const u32* counts, int p, int me, int item_bytes, void* const* windows, void*** d_dbase_out);
// the transfers of the two-step form: segment d of worker me's destination-grouped items d_part goes to worker d's window,
// after the items of the lower ranks (ncclSend / ncclRecv into this rank's window, or simulated: device copies into windows[d])
int xchg_transfer(tg_ctx* ctx, bool simulated, const void* d_part, size_t item_bytes, const u32* counts, int p, int me,
                  void* const* windows);
// inputs that lie inside the exchange window (an un-detached result of the previous collective operator) are moved out of
// the peers' way first (into WS_AUX): the span they cover is copied once, so that inputs sharing it stay consistent
int evacuate_window_inputs(tg_ctx* ctx, const void** in, const size_t* bytes, uint32_t k);

// destination worker of a 16-byte (u64 key, value) item: Hash128to64(0, key) % p (core/reduce_functional.hpp:60-72), the
// owner of a key in ReduceByKey and InnerJoin
struct HashDigit {
    u32 p;
    static constexpr bool kStoreDigit = true;
    static constexpr bool kHasDrop = false;
    static constexpr int kScratch = 0;
    __device__ __forceinline__ void init() {}
    __device__ __forceinline__ u32 operator()(const ulonglong2& v, u32) const { return (u32)(hash128to64_dev(0, v.x) % p); }
};

// destination worker of a 16-byte (u64 key, value) item: key % p, the owner of a key in GroupByKey (hash_function(key) % p,
// api/group_by_key.hpp:149-159, with the default std::hash<uint64_t>, the identity in libstdc++, :419-428).
// Computed from the two 32-bit halves, key % p = ((hi % p) * (2^32 % p) + lo % p) % p, so that no 64-bit division subroutine
// (and its register pressure: the partition pass then spills) enters the pass; exact for p <= 2^16 (the partition takes p <= 256).
struct ModDigit {
    u32 p;
    u32 two32_mod_p;                        // 2^32 % p
    static ModDigit make(u32 p) { return ModDigit{ p, (u32)((1ull << 32) % p) }; }
    static constexpr bool kStoreDigit = true;
    static constexpr bool kHasDrop = false;
    static constexpr int kScratch = 0;
    __device__ __forceinline__ void init() {}
    __device__ __forceinline__ u32 operator()(const ulonglong2& v, u32) const {
        const u32 hi = (u32)(v.x >> 32) % p, lo = (u32)v.x % p;
        return (hi * two32_mod_p + lo) % p;
    }
};

// destination worker of index k: k * p / size (ReduceByIndex / Range::FindPartition, core/reduce_functional.hpp:112-125,
// common/math.hpp:98-100; CalculatePartition in GroupToIndex, api/group_to_index.hpp:98-105); out-of-range indices are parked
// on the last worker, which reports them
struct RangeDigit {
    u64 size;
    u32 p;
    static constexpr bool kStoreDigit = true;
    static constexpr bool kHasDrop = false;
    static constexpr int kScratch = 0;
    __device__ __forceinline__ void init() {}
    __device__ __forceinline__ u32 operator()(const ulonglong2& v, u32) const {
        return v.x < size ? (u32)(v.x * p / size) : p - 1;
    }
};

// the first index of worker r's range: Range(0, size).Partition(r, p) = ceil(r * size / p) (common/math.hpp:85-94); worker r
// answers for [range_begin(r), range_begin(r + 1)), the indices RangeDigit sends to it
inline u64 range_begin(u64 r, u64 size, u64 p) { return (u64)(((unsigned __int128)r * size + p - 1) / p); }

// What the count step of one exchange leaves for its store step: the chunk geometry of the worker's pass and, in WS_SORT_HIST2,
// its per-destination totals and per-chunk bases.
struct XchgLocal {
    size_t n = 0;                   // items that take part (0 for a worker over the limit)
    ChunkGeom g = { 0, 0 };
    u32* totals = nullptr;          // [RADIX] (device): items for each destination worker
    u32* chunkbase = nullptr;       // [nchunks][RADIX] (device): where each chunk's bucket d starts in the grouped order
};

// Count step of one exchange: destination histograms per chunk (chunk_hist_kernel) and their scan (chunk_scan_kernel).
// n >= 2^30 (over the per-call limit): the worker takes part with no items and reports 2^30 items for worker 0 in its totals,
// so that the plan of the count matrix gives TG_ERR_TOO_LARGE on every rank and none is left waiting in a collective.
template <int WORDS, class DigitFn>
int exchange_count(tg_ctx* ctx, const void* d_in, size_t n, const DigitFn& fn, XchgLocal* xl) {
    typedef typename ItemT<WORDS>::type Item;
    const bool too_large = n >= (1u << 30);
    if (too_large) n = 0;
    const ChunkGeom g = chunk_geometry<WORDS>(ctx, n);
    const size_t cw = (size_t)(g.nchunks > 0 ? g.nchunks : 1) * RADIX;
    u32* tab;
    TG_TRY(tg_ws_get(ctx, WS_SORT_HIST2, (2 * cw + 2 * RADIX + 16) * 4, (void**)&tab));
    u32* chunkcount = tab;
    u32* chunkbase = tab + cw;
    u32* totals = chunkbase + cw;
    if (n) {
        TG_LAUNCH_T(ctx, TG_K_RADIX_HIST, (chunk_hist_kernel<WORDS, DigitFn, false>), g.nchunks, 512, 0, (const Item*)d_in, (u32)n,
                    g.chunk_items, fn, chunkcount, (u64*)nullptr);
        TG_LAUNCH(ctx, chunk_scan_kernel, 1, 4 * RADIX, 0, chunkcount, g.nchunks, totals, totals + RADIX, chunkbase);
    }
    else TG_CUDA(ctx, cudaMemsetAsync(totals, 0, 2 * RADIX * 4, ctx->stream));
    if (too_large) TG_CUDA(ctx, cudaMemsetAsync((char*)totals + 3, 0x40, 1, ctx->stream));     // totals[0] = 0x40000000 = 2^30
    xl->n = n;
    xl->g = g;
    xl->totals = totals;
    xl->chunkbase = chunkbase;
    return TG_OK;
}

// Store step of one exchange for worker `me` of p, after its count step (xl): counts = the p x p count matrix (host,
// counts[src * p + dst]), windows[d] = worker d's window as this process addresses it.
//   mode 1  the peer-store pass: bucket d straight into windows[d], after the items of the lower ranks
//   mode 0  the local stable partition into WS_XCHG_SEND, then the per-(src, dst) transfers (xchg_transfer)
// The receive sizes must have been checked against the windows (the plan's `worst`) before.
template <int WORDS, class DigitFn>
int exchange_store(tg_ctx* ctx, int mode, bool simulated, const void* d_in, const XchgLocal& xl, const DigitFn& fn, const u32* counts,
                   int p, int me, void* const* windows) {
    typedef typename ItemT<WORDS>::type Item;
    const size_t s = sizeof(Item), n = xl.n;
    const ChunkGeom& g = xl.g;
    void** d_dbase = nullptr;
    void* d_part = nullptr;
    if (mode == 1) { if (n) TG_TRY(xchg_upload_dest(ctx, counts, p, me, (int)s, windows, &d_dbase)); }
    else TG_TRY(tg_ws_get(ctx, WS_XCHG_SEND, (n + 2) * s, &d_part));
    if (n) {
        std::vector<u32> chunk_size(g.nchunks, g.chunk_items);
        chunk_size[g.nchunks - 1] = (u32)(n - (size_t)(g.nchunks - 1) * g.chunk_items);
        uint4* d_tiles;
        u32 total = 0;
        TG_TRY(build_tile_list(ctx, g.nchunks, chunk_size.data(), tile_items<WORDS>(), 0, WS_SEG_TILES2, &d_tiles, &total));
        u32* status;
        TG_TRY(tg_ws_get(ctx, WS_SORT_STATUS, (size_t)total * RADIX * 4, (void**)&status));
        TG_CUDA(ctx, cudaMemsetAsync(status, 0, (size_t)total * RADIX * 4, ctx->stream));
        SegList sl = { d_tiles, xl.chunkbase, total, nullptr };
        if (mode == 1) {
            // classification + scatter + Alltoallv in one pass: stores into the peers' windows
            const int xprof = ctx->profile ? tg_prof_begin(ctx, TG_K_EXCHANGE) : -1;
            TG_TRY((launch_partition_peer<WORDS, DigitFn>(ctx, d_in, (u32)n, fn, status, sl, (Item* const*)d_dbase)));
            if (xprof >= 0) tg_prof_end(ctx, xprof);
        }
        else TG_TRY((launch_partition_seg<WORDS, DigitFn>(ctx, d_in, d_part, (u32)n, fn, status, sl)));
    }
    if (mode == 1) return TG_OK;
    const int xprof = ctx->profile ? tg_prof_begin(ctx, TG_K_EXCHANGE) : -1;
    TG_TRY(xchg_transfer(ctx, simulated, d_part, s, counts, p, me, windows));
    if (xprof >= 0) tg_prof_end(ctx, xprof);
    return TG_OK;
}

// Stable partition of n local items by fn (destination worker, < p) + Alltoallv.  Collective.
// n >= 2^30 (over the per-call limit): this rank sends nothing and reports 2^30 items for worker 0 in its counts, so that
// xchg_counts returns TG_ERR_TOO_LARGE on every rank and none is left waiting in a collective.
template <int WORDS, class DigitFn>
int exchange_scatter(tg_ctx* ctx, const void* d_in, size_t n, const DigitFn& fn, XchgResult* res) {
    typedef typename ItemT<WORDS>::type Item;
    const size_t s = sizeof(Item);
    TG_TRY(xwin_negotiate(ctx));
    // (1) destination histogram per chunk
    XchgLocal xl;
    TG_TRY((exchange_count<WORDS, DigitFn>(ctx, d_in, n, fn, &xl)));
    // (2) count matrix; every rank learns every rank's receive size
    u64 need = 0;
    TG_TRY(xchg_counts(ctx, xl.totals, (int)s, res, &need));
    TG_TRY(xwin_ensure(ctx, need));
    res->d_recv = ctx->xwin.base;
    // (3) the stores into the peers' windows (or the local partition and the send/recv into the window)
    TG_TRY((exchange_store<WORDS, DigitFn>(ctx, ctx->xwin.mode, false, d_in, xl, fn, xchg_matrix(ctx), ctx->nranks, ctx->rank,
                                           ctx->xwin.peer)));
    // (4) every peer's stores into this window are complete after the barrier
    if (ctx->xwin.mode == 1) TG_TRY(xwin_barrier(ctx));
    return TG_OK;
}

// The owner-by-key pipeline of 16-byte (u64 key, value) items (InnerJoin's sides, GroupByKey, GroupToIndex).
// n items from src into workspace `slot` (items | sort scratch), then the stable local radix sort by the key; *sorted = the
// result, in the slot.  src is read, never modified.  (tg_exchange.cu)
int sort_pairs_into(tg_ctx* ctx, int slot, const void* src, u64 n, const ulonglong2** sorted);

// one exchange by fn, then the received items (every worker's, in rank order: stable) sorted in `slot`.  Collective.
template <class DigitFn>
int exchange_sort_pairs(tg_ctx* ctx, int slot, const void* d_in, size_t n, const DigitFn& fn, const ulonglong2** sorted,
                        u64* n_recv) {
    XchgResult xr;
    TG_TRY((exchange_scatter<2, DigitFn>(ctx, d_in, n, fn, &xr)));
    *n_recv = xr.n_recv;
    return sort_pairs_into(ctx, slot, xr.d_recv, xr.n_recv, sorted);
}

}  // namespace tgp
