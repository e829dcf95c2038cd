// tg_join.cu — InnerJoin (api::InnerJoin, api/inner_join.hpp:700-830) of two DIAs of 16-byte (u64 key, 8-byte value) pairs on
// the key, on H100s.  The reference's JoinNode (:61-481) hash-exchanges both sides, sorts each side and joins by a per-item
// sort-merge on the host.  Here, per worker (DESIGN.md §6):
//   1. p > 1: each side through one exchange_scatter<2, HashDigit> (owner Hash128to64(0, key) % p, as in ReduceByKey); the left
//      side's received items are copied out of the exchange window before the right side's exchange stores into it
//   2. a stable local radix sort of each side by the key (the sort behind tg_radix_sort_local)
//   3. count: merge path over (left, right), ties to the left; for left item i, lo_i = right keys < key_i and hi_i = right keys
//      <= key_i, stored packed as (lo_i << 32 | hi_i - lo_i), and one sum per tile
//   4. scan: exclusive u64 scan of the match counts -> off_i and the worker's output size m (one host round trip; with p > 1 an
//      all-reduce of the largest m decides the size limit identically on every rank)
//   5. emit, output-stationary: merge path over (off_0..off_{nl-1}, output indices 0..m-1).  Each CTA owns a fixed-size piece of
//      that merged sequence, so no CTA writes more than JE_TILE outputs whatever the key distribution (one hot key with 2^30
//      matches, or 10^8 keys with one match each).  Output j belongs to the last left item i with off_i <= j and pairs it with
//      right item lo_i + j - off_i; the outputs go through shared memory and leave as consecutive 8-byte words.
// The result is ordered by (key, left global position, right global position): the exchange and the sort are stable.
//
// InnerJoin on records (tg_inner_join_records): DIAs of fixed-size items joined on an unsigned integer key field of 1..8 bytes.
// Each side becomes 16-byte tuples {key, position} (make_tuples_kernel, shared with Sort's record path); with p > 1 the tuples
// are partitioned by the owner and the records follow them into the owners' windows (exchange_store_records).  The tuples of a
// worker's records then go through steps 2-5 as the pairs do, except that the emit (join_emit_records_kernel) writes each output
// as the left record's words followed by the right record's, read where the records lie.
#include <algorithm>
#include <initializer_list>

#include "tg_keys.cuh"
#include "tg_exchange.cuh"
#include "tg_tile_scan.cuh"
#include "tg_records.cuh"

using namespace tgp;

int tg_radix_sort_items(tg_ctx* ctx, const tg_key_desc* desc, void* d_items, void* d_tmp, size_t n, void** result);

namespace {

typedef ulonglong2 Pair;
constexpr int JN_THREADS = 256;
constexpr u32 JC_TILE = 2048;         // count / offsets: merged (left, right) items per CTA
constexpr u32 JE_TILE = 1024;         // emit: merged (left items, outputs) per CTA
constexpr u64 JOIN_LIMIT = 1ull << 30;

__device__ __forceinline__ u32 lower_bound_u64(const u64* a, u32 lo, u32 hi, u64 k) {
    while (lo < hi) {
        const u32 mid = (lo + hi) >> 1;
        if (a[mid] < k) lo = mid + 1; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ u32 upper_bound_u64(const u64* a, u32 lo, u32 hi, u64 k) {
    while (lo < hi) {
        const u32 mid = (lo + hi) >> 1;
        if (a[mid] <= k) lo = mid + 1; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ u32 upper_bound_pairs(const Pair* a, u32 lo, u32 hi, u64 k) {
    while (lo < hi) {
        const u32 mid = (lo + hi) >> 1;
        if (a[mid].x <= k) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// split[t] = left items among the first min(t * JC_TILE, nl + nr) items of the merge of (left, right), ties to the left
__global__ void join_count_splits_kernel(const Pair* __restrict__ L, u32 nl, const Pair* __restrict__ R, u32 nr, u32 ntiles,
                                         u32* __restrict__ split, KeyView kv) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t > ntiles) return;
    const u32 total = nl + nr;
    split[t] = merge_path_search(L, nl, R, nr, t * JC_TILE < total ? t * JC_TILE : total, kv);
}

// CTA = one tile of the merge of (left, right): left items [a0, a1), right items [b0, b1).  The right items before b0 have keys
// below every left key of the tile, those from b1 on keys at or above them; so lo_i is b0 + a search among the tile's right keys,
// and so is hi_i unless the right items equal to key_i run on past the tile (then one search of the right side from b1).
__global__ void __launch_bounds__(JN_THREADS)
join_count_kernel(const Pair* __restrict__ L, u32 nl, const Pair* __restrict__ R, u32 nr, const u32* __restrict__ split,
                  u64* __restrict__ packed, u64* __restrict__ tile_sum) {
    __shared__ u64 rk[JC_TILE];
    __shared__ u64 warp_tot[JN_THREADS / 32];
    const u32 total = nl + nr;
    const u32 d0 = blockIdx.x * JC_TILE, d1 = d0 + JC_TILE < total ? d0 + JC_TILE : total;
    const u32 a0 = split[blockIdx.x], a1 = split[blockIdx.x + 1];
    const u32 b0 = d0 - a0, b1 = d1 - a1, nb = b1 - b0;
    for (u32 i = threadIdx.x; i < nb; i += JN_THREADS) rk[i] = R[b0 + i].x;
    const bool more = b1 < nr;
    const u64 knext = more ? R[b1].x : 0;
    __syncthreads();
    u64 sum = 0;
    for (u32 i = a0 + threadIdx.x; i < a1; i += JN_THREADS) {
        const u64 k = L[i].x;
        const u32 lo = lower_bound_u64(rk, 0, nb, k);
        const u32 ub = upper_bound_u64(rk, lo, nb, k);
        const u32 hi = ub == nb && more && knext == k ? upper_bound_pairs(R, b1, nr, k) : b0 + ub;
        const u32 c = hi - (b0 + lo);
        packed[i] = ((u64)(b0 + lo) << 32) | c;
        sum += c;
    }
    u64 tot;
    block_excl_scan_u64<JN_THREADS>(sum, warp_tot, &tot);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = tot;
}

// off_i = tile base + the exclusive scan of the match counts of the tile's left items
__global__ void __launch_bounds__(JN_THREADS)
join_offsets_kernel(const u32* __restrict__ split, const u64* __restrict__ packed, const u64* __restrict__ tile_base,
                    u64* __restrict__ off) {
    __shared__ u64 warp_tot[JN_THREADS / 32];
    const u32 a0 = split[blockIdx.x], a1 = split[blockIdx.x + 1];
    u64 carry = tile_base[blockIdx.x];
    for (u32 first = a0; first < a1; first += JN_THREADS) {
        const u32 i = first + threadIdx.x;
        const u64 c = i < a1 ? (packed[i] & 0xffffffffull) : 0;
        u64 tot;
        const u64 ex = block_excl_scan_u64<JN_THREADS>(c, warp_tot, &tot);
        if (i < a1) off[i] = carry + ex;
        carry += tot;
    }
}

// split[t] = left items among the first min(t * JE_TILE, nl + m) items of the merge of (off_0..off_{nl-1}, 0..m-1), left item i
// before output j iff off_i <= j
__global__ void join_emit_splits_kernel(const u64* __restrict__ off, u32 nl, u64 m, u32 ntiles, u32* __restrict__ split) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t > ntiles) return;
    const u64 total = nl + m;
    const u64 d = (u64)t * JE_TILE < total ? (u64)t * JE_TILE : total;
    u64 lo = d > m ? d - m : 0, hi = d < nl ? d : nl;
    while (lo < hi) {
        const u64 mid = (lo + hi) >> 1;
        if (off[mid] <= d - 1 - mid) lo = mid + 1; else hi = mid;
    }
    split[t] = (u32)lo;
}

// CTA = one tile of that merge: outputs [j0, j1); their left items lie in [a0 - 1, a1) (the left item placed last before an
// output owns it).  W = output words per item: 3 = (key, v1, v2), 2 = (v1, v2).
template <int W>
__global__ void __launch_bounds__(JN_THREADS)
join_emit_kernel(const Pair* __restrict__ L, const Pair* __restrict__ R, u32 nl, const u64* __restrict__ off,
                 const u64* __restrict__ packed, u64 m, const u32* __restrict__ split, u64* __restrict__ out) {
    __shared__ u64 soff[JE_TILE + 1];
    __shared__ u64 sout[JE_TILE * W];
    const u64 total = nl + m;
    const u64 d0 = (u64)blockIdx.x * JE_TILE, d1 = d0 + JE_TILE < total ? d0 + JE_TILE : total;
    const u32 a0 = split[blockIdx.x], a1 = split[blockIdx.x + 1];
    const u64 j0 = d0 - a0, j1 = d1 - a1;
    const u32 base = a0 ? a0 - 1 : 0, ns = a1 - base;
    for (u32 i = threadIdx.x; i < ns; i += JN_THREADS) soff[i] = off[base + i];
    __syncthreads();
    const u32 nj = (u32)(j1 - j0);
    for (u32 t = threadIdx.x; t < nj; t += JN_THREADS) {
        const u64 j = j0 + t;
        const u32 s = upper_bound_u64(soff, 0, ns, j) - 1;       // >= 0: off of the owner <= j
        const u32 i = base + s;
        const Pair l = L[i];
        const Pair r = R[(packed[i] >> 32) + (j - soff[s])];
        if (W == 3) { sout[3 * t] = l.x; sout[3 * t + 1] = l.y; sout[3 * t + 2] = r.y; }
        else { sout[2 * t] = l.y; sout[2 * t + 1] = r.y; }
    }
    __syncthreads();
    u64* dst = out + j0 * W;
    for (u32 w = threadIdx.x; w < nj * W; w += JN_THREADS) dst[w] = sout[w];
}

// The records' emit: the same tile of the merge as join_emit_kernel, outputs [j0, j1).  First each output's left and right record
// index (the positions in the sorted tuples' .y) into shared memory, then the tile's outputs as one contiguous run of
// lw + rw words per output: word lt -> (output, word) by a multiply-high (inv = gather_reciprocal(lw + rw); lt < JE_TILE * (lw +
// rw) with lw + rw <= 512), each word read from the left or the right record where it lies, consecutive threads storing
// consecutive words.
__global__ void __launch_bounds__(JN_THREADS)
join_emit_records_kernel(const u32* __restrict__ lrec, const u32* __restrict__ rrec, const Pair* __restrict__ L,
                         const Pair* __restrict__ R, u32 nl, const u64* __restrict__ off, const u64* __restrict__ packed, u64 m,
                         const u32* __restrict__ split, u32 lw, u32 rw, u32 inv, u32* __restrict__ out) {
    __shared__ u64 soff[JE_TILE + 1];
    __shared__ u32 sl[JE_TILE], sr[JE_TILE];
    const u64 total = nl + m;
    const u64 d0 = (u64)blockIdx.x * JE_TILE, d1 = d0 + JE_TILE < total ? d0 + JE_TILE : total;
    const u32 a0 = split[blockIdx.x], a1 = split[blockIdx.x + 1];
    const u64 j0 = d0 - a0, j1 = d1 - a1;
    const u32 base = a0 ? a0 - 1 : 0, ns = a1 - base;
    for (u32 i = threadIdx.x; i < ns; i += JN_THREADS) soff[i] = off[base + i];
    __syncthreads();
    const u32 nj = (u32)(j1 - j0);
    for (u32 t = threadIdx.x; t < nj; t += JN_THREADS) {
        const u64 j = j0 + t;
        const u32 s = upper_bound_u64(soff, 0, ns, j) - 1;       // >= 0: off of the owner <= j
        const u32 i = base + s;
        sl[t] = (u32)(L[i].y >> 32);
        sr[t] = (u32)(R[(packed[i] >> 32) + (j - soff[s])].y >> 32);
    }
    __syncthreads();
    const u32 ow = lw + rw, words = nj * ow;
    u32* dst = out + j0 * ow;
#pragma unroll 4
    for (u32 lt = threadIdx.x; lt < words; lt += JN_THREADS) {
        const u32 t = __umulhi(lt, inv), w = lt - t * ow;
        dst[lt] = w < lw ? lrec[(size_t)sl[t] * lw + w] : rrec[(size_t)sr[t] * rw + (w - lw)];
    }
}

int check_join_args(tg_ctx* ctx, const tg_join_desc* desc) {
    if (!ctx || !desc || desc->item_bytes != 16 || desc->join_fn > TG_JOIN_VALUES)
        return tg_set_error(ctx, TG_ERR_ARG, "inner_join: 16-byte (u64 key, 8-byte value) inputs and TG_JOIN_KEY_VALUES / TG_JOIN_VALUES");
    if (ctx->nranks > TG_MAX_RANKS) return tg_set_error(ctx, TG_ERR_ARG, "inner_join: at most 16 ranks");
    return TG_OK;
}

// What the count leaves for the emit: the packed (lo_i, count_i), the offsets off_i, room for the emit splits, the output size m
struct JoinCounts {
    u64 *packed, *off;
    u32* esplit;
    u64 m;
};

// steps 3-4 on the sorted sides: count, scan and the output size
int join_count(tg_ctx* ctx, const Pair* L, u64 nl, const Pair* R, u64 nr, JoinCounts* jc) {
    const int p = ctx->nranks;
    // scratch: scalars (m, largest m) | packed counts | offsets | tile sums | tile bases | count splits | emit splits
    const u32 nct = (u32)((nl + nr + JC_TILE - 1) / JC_TILE);
    const u64 net_max = (nl + JOIN_LIMIT + JE_TILE - 1) / JE_TILE;
    u64* aux;
    TG_TRY(tg_ws_get(ctx, WS_JOIN_AUX, 16 + (2 * nl + 2 * (size_t)nct + 2) * 8 + ((size_t)nct + net_max + 4) * 4 + 64, (void**)&aux));
    u64* d_m = aux;
    u64* packed = aux + 2;
    u64* off = packed + nl;
    u64* tile_sum = off + nl;
    u64* tile_base = tile_sum + nct + 1;
    u32* csplit = (u32*)(tile_base + nct + 1);
    u32* esplit = csplit + nct + 2;
    const bool work = nl && nr;
    if (work) {
        const KeyView kv = { 0, 8, TG_KEY_UINT_LE, 0 };
        TG_LAUNCH_T(ctx, TG_K_JOIN, join_count_splits_kernel, (nct + 1 + 127) / 128, 128, 0, L, (u32)nl, R, (u32)nr, nct, csplit, kv);
        TG_LAUNCH_T(ctx, TG_K_JOIN, join_count_kernel, nct, JN_THREADS, 0, L, (u32)nl, R, (u32)nr, (const u32*)csplit, packed, tile_sum);
        TG_LAUNCH_T(ctx, TG_K_JOIN, join_scan_tiles_kernel, 1, JS_THREADS, 0, (const u64*)tile_sum, nct, tile_base, d_m);
        TG_LAUNCH_T(ctx, TG_K_JOIN, join_offsets_kernel, nct, JN_THREADS, 0, (const u32*)csplit, (const u64*)packed,
                    (const u64*)tile_base, off);
    }
    else TG_CUDA(ctx, cudaMemsetAsync(d_m, 0, 8, ctx->stream));
    // the output size; with several workers the largest one decides the limit on every rank
    u64* h = (u64*)ctx->pinned + 65536;          // byte offset 512 KB of the pinned scratch
    if (p > 1) {
        TG_NCCL(ctx, ncclAllReduce(d_m, d_m + 1, 1, ncclUint64, ncclMax, ctx->comm, ctx->stream));
        TG_CUDA(ctx, cudaMemcpyAsync(h, d_m, 16, cudaMemcpyDeviceToHost, ctx->stream));
    }
    else TG_CUDA(ctx, cudaMemcpyAsync(h, d_m, 8, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    jc->m = h[0];
    const u64 m_max = p > 1 ? h[1] : h[0];
    if (m_max >= JOIN_LIMIT)
        return tg_set_error(ctx, TG_ERR_TOO_LARGE, "inner_join: a worker's output has %llu items (limit 2^30 - 1)", (unsigned long long)m_max);
    jc->packed = packed;
    jc->off = off;
    jc->esplit = esplit;
    return TG_OK;
}

int join_impl(tg_ctx* ctx, const tg_join_desc* desc, const void* d_left, size_t n_left, const void* d_right, size_t n_right,
              void** out_dptr, size_t* out_n) {
    const int p = ctx->nranks;
    const Pair *L, *R;
    u64 nl, nr;
    if (p == 1) {
        if (n_left >= JOIN_LIMIT || n_right >= JOIN_LIMIT)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "inner_join: %zu x %zu items (limit 2^30 - 1 per side)", n_left, n_right);
        nl = n_left; nr = n_right;
        TG_TRY(sort_pairs_into(ctx, WS_JOIN_L, d_left, nl, &L));
        TG_TRY(sort_pairs_into(ctx, WS_JOIN_R, d_right, nr, &R));
    }
    else {
        // (an input inside the exchange window is moved out of the peers' way first; the left side's received items are in
        // its slot before the right side's exchange starts storing into the window)
        const void* in[2] = { d_left, d_right };
        const size_t bytes[2] = { n_left < JOIN_LIMIT ? n_left * 16 : 0, n_right < JOIN_LIMIT ? n_right * 16 : 0 };
        TG_TRY(xwin_negotiate(ctx));
        TG_TRY(evacuate_window_inputs(ctx, in, bytes, 2));
        const HashDigit fn = { (u32)p };
        TG_TRY(exchange_sort_pairs(ctx, WS_JOIN_L, in[0], n_left, fn, &L, &nl));
        TG_TRY(exchange_sort_pairs(ctx, WS_JOIN_R, in[1], n_right, fn, &R, &nr));
    }
    JoinCounts jc;
    TG_TRY(join_count(ctx, L, nl, R, nr, &jc));
    const u64 m = jc.m;
    u64 *off = jc.off, *packed = jc.packed;
    u32* esplit = jc.esplit;
    const int words = desc->join_fn == TG_JOIN_KEY_VALUES ? 3 : 2;
    u64* d_out;
    TG_TRY(tg_ws_get(ctx, WS_JOIN_OUT, (m + 1) * words * 8, (void**)&d_out));
    if (m) {
        const u32 net = (u32)((nl + m + JE_TILE - 1) / JE_TILE);
        TG_LAUNCH_T(ctx, TG_K_JOIN, join_emit_splits_kernel, (net + 1 + 127) / 128, 128, 0, (const u64*)off, (u32)nl, m, net, esplit);
        if (words == 3)
            TG_LAUNCH_T(ctx, TG_K_JOIN, join_emit_kernel<3>, net, JN_THREADS, 0, L, R, (u32)nl, (const u64*)off, (const u64*)packed,
                        m, (const u32*)esplit, d_out);
        else
            TG_LAUNCH_T(ctx, TG_K_JOIN, join_emit_kernel<2>, net, JN_THREADS, 0, L, R, (u32)nl, (const u64*)off, (const u64*)packed,
                        m, (const u32*)esplit, d_out);
    }
    *out_dptr = d_out;
    *out_n = (size_t)m;
    return TG_OK;
}

// ---- records ----------------------------------------------------------------------------------------------------------------
int check_join_records_args(tg_ctx* ctx, const tg_join_records_desc* d, RecSide* side) {
    if (!ctx || !d) return tg_set_error(ctx, TG_ERR_ARG, "inner_join_records: NULL argument");
    side[0] = { d->left_bytes, d->left_key_offset, d->left_key_bytes };
    side[1] = { d->right_bytes, d->right_key_offset, d->right_key_bytes };
    TG_TRY(check_side(ctx, "inner_join_records: left", side[0]));
    TG_TRY(check_side(ctx, "inner_join_records: right", side[1]));
    if (ctx->nranks > TG_MAX_RANKS) return tg_set_error(ctx, TG_ERR_ARG, "inner_join_records: at most 16 ranks");
    return TG_OK;
}

int join_records_impl(tg_ctx* ctx, const RecSide* side, const void* d_left, size_t n_left, const void* d_right, size_t n_right,
                      void** out_dptr, size_t* out_n) {
    const int p = ctx->nranks;
    const void* rec[2] = { d_left, d_right };
    u64 n[2] = { n_left, n_right };
    const size_t bytes[2] = { n_left < JOIN_LIMIT ? n_left * side[0].bytes : 0, n_right < JOIN_LIMIT ? n_right * side[1].bytes : 0 };
    // an input in a slot the join writes before its last read of the inputs (WS_JOIN_L / WS_JOIN_R: the tuples, and the result of
    // GroupByKey; WS_JOIN_OUT: the result of a join) is copied out of the way first; the two sides of a self-join stay one copy
    const int dst[2] = { WS_JOIN_IN_L, WS_JOIN_IN_R };
    TG_TRY(move_inputs_out_of_slots(ctx, rec, bytes, 2, { WS_JOIN_L, WS_JOIN_R, WS_JOIN_OUT }, dst));
    if (p == 1) {
        if (n_left >= JOIN_LIMIT || n_right >= JOIN_LIMIT)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "inner_join_records: %zu x %zu items (limit 2^30 - 1 per side)", n_left, n_right);
    }
    else {
        // each side: tuples, their partition by the owner, the count matrix, the records into the owners' windows.  An input inside
        // the exchange window is moved out of the peers' way first; the left side's received records are copied out of the window
        // before the right side's exchange stores into it.  A side of 2^30 or more items takes part with none and reports 2^30
        // for worker 0, so that the count matrix gives TG_ERR_TOO_LARGE on every rank.
        TG_TRY(xwin_negotiate(ctx));
        TG_TRY(evacuate_window_inputs(ctx, rec, bytes, 2));
        for (int j = 0; j < 2; ++j) {
            const u32 s = side[j].bytes;
            const bool too_large = n[j] >= JOIN_LIMIT;
            const size_t nj = too_large ? 0 : n[j];
            Pair* ptup;
            u32* d_tot;
            TG_TRY(partition_record_tuples(ctx, rec[j], nj, side[j], (u32)p, &ptup, &d_tot));
            if (too_large) TG_CUDA(ctx, cudaMemsetAsync((char*)d_tot + 3, 0x40, 1, ctx->stream));     // totals[0] = 2^30
            XchgResult xr;
            u64 need = 0;
            TG_TRY(xchg_counts(ctx, d_tot, (int)s, &xr, &need));                      // (synchronises; uniform verdicts)
            TG_TRY(xwin_ensure(ctx, need));
            TG_TRY(exchange_store_records(ctx, ctx->xwin.mode, false, rec[j], s, ptup, nj, xchg_matrix(ctx), p, ctx->rank, ctx->xwin.peer));
            if (ctx->xwin.mode == 1) TG_TRY(xwin_barrier(ctx));
            n[j] = xr.n_recv;
            if (j == 1) { rec[1] = ctx->xwin.base; break; }
            void* d;
            TG_TRY(tg_ws_get(ctx, WS_JOIN_LREC, (size_t)xr.n_recv * s + 16, &d));
            if (xr.n_recv) TG_CUDA(ctx, cudaMemcpyAsync(d, ctx->xwin.base, (size_t)xr.n_recv * s, cudaMemcpyDeviceToDevice, ctx->stream));
            rec[0] = d;
        }
    }
    const Pair *L, *R;
    TG_TRY(sort_record_tuples(ctx, WS_JOIN_L, rec[0], n[0], side[0], &L));
    TG_TRY(sort_record_tuples(ctx, WS_JOIN_R, rec[1], n[1], side[1], &R));
    JoinCounts jc;
    TG_TRY(join_count(ctx, L, n[0], R, n[1], &jc));
    const u64 m = jc.m, nl = n[0];
    const u32 lw = side[0].bytes / 4, rw = side[1].bytes / 4;
    u32* d_out;
    TG_TRY(tg_ws_get(ctx, WS_JOIN_OUT, m * (lw + rw) * 4 + 16, (void**)&d_out));
    if (m) {
        const u32 net = (u32)((nl + m + JE_TILE - 1) / JE_TILE);
        TG_LAUNCH_T(ctx, TG_K_JOIN, join_emit_splits_kernel, (net + 1 + 127) / 128, 128, 0, (const u64*)jc.off, (u32)nl, m, net, jc.esplit);
        TG_LAUNCH_T(ctx, TG_K_JOIN, join_emit_records_kernel, net, JN_THREADS, 0, (const u32*)rec[0], (const u32*)rec[1], L, R, (u32)nl,
                    (const u64*)jc.off, (const u64*)jc.packed, m, (const u32*)jc.esplit, lw, rw, gather_reciprocal(lw + rw), d_out);
    }
    *out_dptr = d_out;
    *out_n = (size_t)m;
    return TG_OK;
}

}  // namespace

namespace tgp {

int check_side(tg_ctx* ctx, const char* what, const RecSide& s) {
    if (s.bytes == 0 || s.bytes % 4 || s.bytes > 1024 || s.key_bytes == 0 || s.key_bytes > 8 || (u64)s.key_off + s.key_bytes > s.bytes)
        return tg_set_error(ctx, TG_ERR_ARG, "%s: item size %u (a multiple of 4, 4..1024) with a key of %u bytes at offset %u (1..8 bytes "
                            "inside the item)", what, s.bytes, s.key_bytes, s.key_off);
    return TG_OK;
}

// the n records' tuples in workspace `slot` (tuples | sort scratch), stably sorted by the key: *sorted
int sort_record_tuples(tg_ctx* ctx, int slot, const void* rec, u64 n, const RecSide& s, const Pair** sorted) {
    Pair* buf;
    TG_TRY(tg_ws_get(ctx, slot, (2 * n + 2) * 16, (void**)&buf));
    *sorted = buf;
    if (!n) return TG_OK;
    TG_LAUNCH(ctx, make_tuples_kernel, ctx->sm_count * 8, 256, 0, (const u32*)rec, (u32)n, s.bytes / 4, s.key_off, s.key_bytes, buf);
    const tg_key_desc sd = { 16, 0, 8, TG_KEY_UINT_LE, 0, 1 };
    void* res = buf;
    TG_TRY(tg_radix_sort_items(ctx, &sd, buf, buf + n + 1, n, &res));
    *sorted = (const Pair*)res;
    return TG_OK;
}

// worker w's n records: their tuples into tup, partitioned by the owner into ptup; *d_tot = the per-destination counts (device)
int partition_record_tuples(tg_ctx* ctx, const void* rec, size_t n, const RecSide& s, u32 p, Pair** ptup, u32** d_tot) {
    Pair* tup;
    TG_TRY(tg_ws_get(ctx, WS_JOIN_L, (n + 1) * 16, (void**)&tup));
    TG_TRY(tg_ws_get(ctx, WS_JOIN_R, (n + 1) * 16, (void**)ptup));
    if (n) TG_LAUNCH(ctx, make_tuples_kernel, ctx->sm_count * 8, 256, 0, (const u32*)rec, (u32)n, s.bytes / 4, s.key_off, s.key_bytes, tup);
    const HashDigit fn = { p };
    return partition_chunked<2, HashDigit>(ctx, tup, *ptup, n, fn, d_tot, nullptr);
}

// An input that lies in one of `slots` is copied out of the way first, input j into dst_slots[j].  Inputs that are the same span
// as input 0 stay one copy.
int move_inputs_out_of_slots(tg_ctx* ctx, const void** rec, const size_t* bytes, int k, std::initializer_list<int> slots,
                             const int* dst_slots) {
    const void* orig0 = rec[0];
    for (int j = 0; j < k; ++j) {
        const char* q = (const char*)rec[j];
        bool inside = false;
        for (const int s : slots) {
            const char* b = (const char*)ctx->ws[s];
            if (bytes[j] && b && q >= b && q < b + ctx->ws_bytes[s]) inside = true;
        }
        if (!inside) continue;
        if (j > 0 && rec[j] == orig0 && bytes[j] == bytes[0]) { rec[j] = rec[0]; continue; }
        void* d;
        TG_TRY(tg_ws_get(ctx, dst_slots[j], bytes[j], &d));
        TG_CUDA(ctx, cudaMemcpyAsync(d, q, bytes[j], cudaMemcpyDeviceToDevice, ctx->stream));
        rec[j] = d;
    }
    return TG_OK;
}

}  // namespace tgp

extern "C" {

int tg_inner_join(tg_ctx* ctx, const tg_join_desc* desc, const void* d_left, size_t n_left, const void* d_right, size_t n_right,
                  void** out_dptr, size_t* out_n) {
    TG_TRY(check_join_args(ctx, desc));
    if (!out_dptr || !out_n || (!d_left && n_left) || (!d_right && n_right))
        return tg_set_error(ctx, TG_ERR_ARG, "inner_join: NULL argument");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return join_impl(ctx, desc, d_left, n_left, d_right, n_right, out_dptr, out_n);
}

int tg_inner_join_file(tg_ctx* ctx, const tg_join_desc* desc, const tg_merge_input* left, const tg_merge_input* right,
                       size_t* out_items) {
    TG_TRY(check_join_args(ctx, desc));
    if (!left || !right || !out_items) return tg_set_error(ctx, TG_ERR_ARG, "inner_join_file: NULL argument");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    // host Files go up into one staging buffer (each side at a 16-byte aligned offset), device Files are read where they are
    const tg_merge_input* side[2] = { left, right };
    size_t n[2] = { 0, 0 }, off[2] = { 0, 0 }, staged = 0;
    for (int j = 0; j < 2; ++j) {
        const tg_merge_input& in = *side[j];
        if (in.dev) {
            if (in.dev->item_bytes != 16 || (!in.dev->dptr && in.dev->items))
                return tg_set_error(ctx, TG_ERR_ARG, "inner_join_file: device File %d has item size %u, the join takes 16", j, in.dev->item_bytes);
            n[j] = in.dev->items;
            continue;
        }
        if (!in.blocks && in.nblocks) return tg_set_error(ctx, TG_ERR_ARG, "inner_join_file: input %d has no blocks", j);
        size_t bytes = 0;
        for (size_t i = 0; i < in.nblocks; ++i) bytes += in.blocks[i].bytes;
        if (bytes % 16) return tg_set_error(ctx, TG_ERR_ARG, "inner_join_file: input %d: %zu bytes is not a multiple of 16", j, bytes);
        n[j] = bytes / 16;
        off[j] = staged;
        staged += bytes;
    }
    char* d_stage = nullptr;
    if (staged) TG_TRY(tg_ws_get(ctx, WS_IN, staged + 16, (void**)&d_stage));
    const void* ptrs[2];
    for (int j = 0; j < 2; ++j) {
        if (side[j]->dev) { ptrs[j] = side[j]->dev->dptr; continue; }
        ptrs[j] = d_stage ? d_stage + off[j] : nullptr;
        if (n[j]) TG_TRY(tg_upload_blocks(ctx, d_stage + off[j], side[j]->blocks, side[j]->nblocks, nullptr));
    }
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(join_impl(ctx, desc, ptrs[0], n[0], ptrs[1], n[1], &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = desc->join_fn == TG_JOIN_KEY_VALUES ? 24 : 16;
    *out_items = n_out;
    return TG_OK;
}

int tg_inner_join_records(tg_ctx* ctx, const tg_join_records_desc* desc, const void* d_left, size_t n_left, const void* d_right,
                          size_t n_right, void** out_dptr, size_t* out_n) {
    RecSide side[2];
    TG_TRY(check_join_records_args(ctx, desc, side));
    if (!out_dptr || !out_n || (!d_left && n_left) || (!d_right && n_right))
        return tg_set_error(ctx, TG_ERR_ARG, "inner_join_records: NULL argument");
    if (((uintptr_t)d_left | (uintptr_t)d_right) & 3) return tg_set_error(ctx, TG_ERR_ARG, "inner_join_records: records must be 4-byte aligned");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return join_records_impl(ctx, side, d_left, n_left, d_right, n_right, out_dptr, out_n);
}

int tg_inner_join_records_file(tg_ctx* ctx, const tg_join_records_desc* desc, const tg_merge_input* left,
                               const tg_merge_input* right, size_t* out_items) {
    RecSide side[2];
    TG_TRY(check_join_records_args(ctx, desc, side));
    if (!left || !right || !out_items) return tg_set_error(ctx, TG_ERR_ARG, "inner_join_records_file: NULL argument");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    // host Files go up into one staging buffer (each side at a 16-byte aligned offset), device Files are read where they are
    const tg_merge_input* in[2] = { left, right };
    size_t n[2] = { 0, 0 }, off[2] = { 0, 0 }, staged = 0;
    for (int j = 0; j < 2; ++j) {
        const u32 s = side[j].bytes;
        if (in[j]->dev) {
            const tg_dev_file& f = *in[j]->dev;
            if (f.item_bytes != s || (!f.dptr && f.items) || ((uintptr_t)f.dptr & 3))
                return tg_set_error(ctx, TG_ERR_ARG, "inner_join_records_file: device File %d has item size %u, the descriptor says %u", j, f.item_bytes, s);
            n[j] = f.items;
            continue;
        }
        if (!in[j]->blocks && in[j]->nblocks) return tg_set_error(ctx, TG_ERR_ARG, "inner_join_records_file: input %d has no blocks", j);
        size_t bytes = 0;
        for (size_t i = 0; i < in[j]->nblocks; ++i) bytes += in[j]->blocks[i].bytes;
        if (bytes % s) return tg_set_error(ctx, TG_ERR_ARG, "inner_join_records_file: input %d: %zu bytes is not a multiple of %u", j, bytes, s);
        n[j] = bytes / s;
        off[j] = staged;
        staged += (bytes + 15) & ~(size_t)15;
    }
    char* d_stage = nullptr;
    if (staged) TG_TRY(tg_ws_get(ctx, WS_IN, staged + 16, (void**)&d_stage));
    const void* ptrs[2];
    for (int j = 0; j < 2; ++j) {
        if (in[j]->dev) { ptrs[j] = in[j]->dev->dptr; continue; }
        ptrs[j] = d_stage ? d_stage + off[j] : nullptr;
        if (n[j]) TG_TRY(tg_upload_blocks(ctx, d_stage + off[j], in[j]->blocks, in[j]->nblocks, nullptr));
    }
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(join_records_impl(ctx, side, ptrs[0], n[0], ptrs[1], n[1], &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = side[0].bytes + side[1].bytes;
    *out_items = n_out;
    return TG_OK;
}

int tg_exchange_records_select(tg_ctx* ctx, uint32_t mode, uint32_t item_bytes, uint32_t key_offset, uint32_t key_bytes,
                               const void* const* d_shards, const size_t* n_shards, uint32_t p, void* const* d_windows,
                               const size_t* window_bytes, uint64_t* out_counts) {
    if (!ctx || p < 1 || p > TG_MAX_RANKS || mode > 1 || !d_shards || !n_shards || !out_counts)
        return tg_set_error(ctx, TG_ERR_ARG, "exchange_records_select: p=%u, mode %u or a NULL argument", p, mode);
    const RecSide s = { item_bytes, key_offset, key_bytes };
    TG_TRY(check_side(ctx, "exchange_records_select", s));
    for (uint32_t w = 0; w < p; ++w) {
        if (n_shards[w] && !d_shards[w]) return tg_set_error(ctx, TG_ERR_ARG, "exchange_records_select: shard %u is NULL", w);
        if ((uintptr_t)d_shards[w] & 3) return tg_set_error(ctx, TG_ERR_ARG, "exchange_records_select: records must be 4-byte aligned");
    }
    for (uint32_t w = 0; w < p; ++w)
        if (n_shards[w] >= JOIN_LIMIT) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "exchange_records_select: shard %u has %zu records", w, n_shards[w]);
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const int P = (int)p;
    u32* h_mat = (u32*)ctx->pinned + 16384;          // (the pinned scratch's count matrix, as in xchg_counts)
    Pair* ptup;
    u32* d_tot;
    for (int w = 0; w < P; ++w) {
        TG_TRY(partition_record_tuples(ctx, d_shards[w], n_shards[w], s, p, &ptup, &d_tot));
        TG_CUDA(ctx, cudaMemcpyAsync(h_mat + w * P, d_tot, (size_t)P * 4, cudaMemcpyDeviceToHost, ctx->stream));
    }
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    TG_TRY(select_check(ctx, h_mat, P, item_bytes, d_windows, window_bytes, out_counts));
    if (!d_windows) return TG_OK;
    for (int w = 0; w < P; ++w) {
        // (the partition again: the next worker's overwrote it)
        TG_TRY(partition_record_tuples(ctx, d_shards[w], n_shards[w], s, p, &ptup, &d_tot));
        TG_TRY(exchange_store_records(ctx, (int)mode, true, d_shards[w], item_bytes, ptup, n_shards[w], h_mat, P, w, d_windows));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return TG_OK;
}

}  // extern "C"
