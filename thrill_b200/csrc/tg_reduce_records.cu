// tg_reduce_records.cu — ReduceByKey on records (api::ReduceByKey, api/reduce_by_key.hpp:312-363; ReduceNode :100-211): DIAs of
// fixed-size records reduced by an unsigned integer key field, field by field, on H100s.  The reduce function is a list of field
// runs (consecutive 8-byte fields, each folded by one TG_OP_*); every other byte of an output comes from the group's first record.
//
// One local reduce of n records (p = 1: the operator; p > 1: the pre phase, and again on the received records):
//   1. tuples {key, position} of the records, stably sorted by the key (sort_record_tuples, shared with InnerJoin on records)
//   2. rr_heads_kernel: the group heads of each tile of T sorted tuples (a head = a key that differs from its predecessor), then
//      the tile scan (join_scan_tiles_kernel) -> each tile's first output slot and the output size m
//   3. rr_reduce_kernel, one CTA per tile: gathers only the run words of the tile's records into shared memory (consecutive
//      threads on consecutive words of a record), folds each field over each group inside the tile in a fixed order (a
//      sequential fold per chunk of C items, then a segmented Hillis-Steele scan over the chunks), and writes every group headed
//      in the tile: the head record's words with the folded fields in place.  A group cut by the tile's end is written with the
//      tile's partial; the items before the tile's first head (the piece of a group headed in an earlier tile) leave one partial
//      per field in lpart.
//   4. rr_cut_kernel, one CTA per cut group: folds the group's pieces (the lpart of the following tiles up to the first one that
//      heads a group) in tile order, every thread a contiguous run of pieces and then an in-order tree, into the written partial.
// T follows from the field count F so that the tile's values fit in shared memory (T * F <= 4096, T <= 2048); the bracketing of
// every fold depends on positions and these fixed sizes only, so the result is bitwise reproducible.
//
// With p > 1 (DESIGN.md §6): the local reduce of the input, the owner partition of its result's tuples (partition_record_tuples,
// Hash128to64(0, key) % p), the count matrix, the records into the owners' windows (exchange_store_records), then the local
// reduce of the received records.  They lie grouped by source rank, so the stable sort keeps a group's globally first record first.
#include <algorithm>

#include "tg_exchange.cuh"
#include "tg_tile_scan.cuh"
#include "tg_records.cuh"
#include "tg_reduce_ops.cuh"

using namespace tgp;

namespace {

typedef ulonglong2 Pair;
constexpr int RR_THREADS = 256;
constexpr u64 RR_LIMIT = 1ull << 30;
constexpr u32 RR_MAX_RUNS = 8;
constexpr u32 RR_VALUES = 4096;           // T * F: values a tile holds in shared memory
constexpr u32 RR_MAX_TILE = 2048;
constexpr size_t RR_MAX_SMEM = 64 << 10;

// what the kernels know of the descriptor and the tile geometry
struct RRDesc {
    u32 rw, nf, nruns;                     // record words, fields, runs
    u32 run_word[RR_MAX_RUNS];             // first record word of run r
    u32 run_f0[RR_MAX_RUNS + 1];           // first field of run r; run_f0[nruns] = nf
    u32 run_op[RR_MAX_RUNS];
    u32 T, nch, lc, fs;                    // tile items, chunks per tile, log2 of the chunk length C = T / nch, field stride
    u32 inv_g, inv_o;                      // gather_reciprocal(2 * nf), gather_reciprocal(rw) (0: divide)
};

__device__ __forceinline__ u32 run_of(const RRDesc& d, u32 f) {
    u32 r = 0;
#pragma unroll
    for (u32 q = 1; q < RR_MAX_RUNS; ++q)
        if (q < d.nruns && f >= d.run_f0[q]) r = q;
    return r;
}

// the value of item i of field f lives at v[f * fs + i + i / C]: the skew keeps the chunks' sequential folds on distinct banks
__device__ __forceinline__ u32 vslot(const RRDesc& d, u32 f, u32 i) { return f * d.fs + i + (i >> d.lc); }

__device__ __forceinline__ bool is_head(const Pair* __restrict__ tup, u32 g, u64 key) { return g == 0 || tup[g - 1].x != key; }

// tile_sum[t] = the group heads among the T sorted tuples of tile t
__global__ void __launch_bounds__(RR_THREADS)
rr_heads_kernel(const Pair* __restrict__ tup, u32 n, u32 T, u64* __restrict__ tile_sum) {
    __shared__ u32 wc[RR_THREADS / 32];
    const u32 g0 = blockIdx.x * T, g1 = min(g0 + T, n);
    u32 c = 0;
    for (u32 g = g0 + threadIdx.x; g < g1; g += RR_THREADS) c += is_head(tup, g, tup[g].x);
#pragma unroll
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane_id() == 0) wc[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 s = 0;
#pragma unroll
        for (int w = 0; w < RR_THREADS / 32; ++w) s += wc[w];
        tile_sum[blockIdx.x] = s;
    }
}

// One CTA per tile (steps 3 of the file comment).  Dynamic shared memory: see rr_smem_bytes.
__global__ void __launch_bounds__(RR_THREADS)
rr_reduce_kernel(const Pair* __restrict__ tup, u32 n, const u32* __restrict__ rec, const u64* __restrict__ tile_base, const RRDesc d,
                 u64* __restrict__ lpart, u32* __restrict__ out) {
    extern __shared__ u64 sm[];
    const u32 T = d.T, F = d.nf, nch = d.nch, nw = T / 32;
    u64* v = sm;                                   // F x fs values
    u64* pre = v + (size_t)F * d.fs;               // per (field, chunk): the fold before the chunk's first head
    u64* sv = pre + RR_THREADS;                    // per (field, chunk): the scan's value ...
    int* shp = (int*)(sv + RR_THREADS);            // ... and head (the last head at or before the chunk's end, -1: none)
    u32* pos = (u32*)(shp + RR_THREADS);           // T record positions
    u32* hmask = pos + T;                          // head bits, one word per 32 items
    u32* wpre = hmask + nw;                        // heads before each word of hmask; wpre[nw] = the tile's heads
    unsigned short* hidx = (unsigned short*)(wpre + nw + 1);    // item of the tile's j-th head
    unsigned short* wkind = hidx + T;              // record word w: 0xffff = copied from the head record, else 2 * field + half
    unsigned short* gword = wkind + d.rw;          // gathered word k (2 * field + half) -> record word
    const u32 g0 = blockIdx.x * T, nt = min(T, n - g0);

    for (u32 w = threadIdx.x; w < d.rw; w += RR_THREADS) {
        u32 k = 0xffff;
        for (u32 r = 0; r < d.nruns; ++r)
            if (w >= d.run_word[r] && w < d.run_word[r] + 2 * (d.run_f0[r + 1] - d.run_f0[r])) k = 2 * d.run_f0[r] + (w - d.run_word[r]);
        wkind[w] = (unsigned short)k;
    }
    for (u32 k = threadIdx.x; k < 2 * F; k += RR_THREADS) {
        const u32 f = k >> 1, r = run_of(d, f);
        gword[k] = (unsigned short)(d.run_word[r] + 2 * (f - d.run_f0[r]) + (k & 1));
    }
    for (u32 i = threadIdx.x; i < T; i += RR_THREADS) {
        bool h = false;
        if (i < nt) {
            const Pair t = tup[g0 + i];
            pos[i] = (u32)(t.y >> 32);
            h = is_head(tup, g0 + i, t.x);
        }
        const u32 m = __ballot_sync(0xffffffffu, h);
        if (lane_id() == 0) hmask[i >> 5] = m;
    }
    __syncthreads();
    if (threadIdx.x < 32) {                        // exclusive scan of the words' head counts (nw <= 64: two words per lane)
        const u32 l = threadIdx.x;
        const u32 c0 = 2 * l < nw ? __popc(hmask[2 * l]) : 0, c1 = 2 * l + 1 < nw ? __popc(hmask[2 * l + 1]) : 0;
        u32 x = c0 + c1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const u32 y = __shfl_up_sync(0xffffffffu, x, o);
            if ((int)l >= o) x += y;
        }
        if (2 * l < nw) wpre[2 * l] = x - c0 - c1;
        if (2 * l + 1 < nw) wpre[2 * l + 1] = x - c1;
        if (l == 31) wpre[nw] = x;
    }
    __syncthreads();
    for (u32 i = threadIdx.x; i < nt; i += RR_THREADS) {
        const u32 m = hmask[i >> 5], b = i & 31;
        if ((m >> b) & 1) hidx[wpre[i >> 5] + __popc(m & ((1u << b) - 1))] = (unsigned short)i;
    }
    if (F) {
        // the run words of the tile's records: word lt -> (item, gathered word) by a multiply-high (2F >= 2, lt < 2 * RR_VALUES)
        u32* v32 = (u32*)v;
        const u32 gw = 2 * F, words = nt * gw;
#pragma unroll 4
        for (u32 lt = threadIdx.x; lt < words; lt += RR_THREADS) {
            const u32 t = __umulhi(lt, d.inv_g), k = lt - t * gw;
            v32[2 * vslot(d, k >> 1, t) + (k & 1)] = rec[(size_t)pos[t] * d.rw + gword[k]];
        }
        __syncthreads();
        // one (field, chunk) per thread (F * nch <= RR_THREADS): the sequential fold of the chunk's C items.  A group headed
        // and ended inside the chunk is complete: its value goes to its head's slot.
        const u32 e = threadIdx.x, C = T / nch;
        const bool act = e < F * nch;
        const u32 f = act ? e / nch : 0, c = e & (nch - 1);
        const int op = (int)d.run_op[run_of(d, f)];
        const u64 ident = op_identity(op);
        u64 acc = ident;
        int lh = -1;
        if (act) {
            const u32 i0 = c * C, i1 = min(i0 + C, nt);
            for (u32 i = i0; i < i1; ++i) {
                if ((hmask[i >> 5] >> (i & 31)) & 1) {
                    if (lh >= 0) v[vslot(d, f, lh)] = acc;
                    else pre[e] = acc;
                    lh = (int)i;
                    acc = ident;
                }
                acc = op_combine(op, acc, v[vslot(d, f, i)]);
            }
            sv[e] = acc;
            shp[e] = lh;
        }
        // segmented inclusive scan over the chunks of each field: S_c = (last head at or before chunk c's end, the fold from it)
        const bool had = lh >= 0;
        u64 mv = acc;
        int mh = lh;
        for (u32 s = 1; s < nch; s <<= 1) {
            __syncthreads();
            const bool take = act && c >= s && mh < 0;
            u64 lv = 0;
            int lhp = -1;
            if (take) { lv = sv[e - s]; lhp = shp[e - s]; }
            __syncthreads();
            if (take) {
                mv = op_combine(op, lv, mv);
                mh = lhp;
                sv[e] = mv;
                shp[e] = mh;
            }
        }
        __syncthreads();
        if (act) {
            // the group that ends in this chunk, before its first head: headed in an earlier chunk, or in an earlier tile
            if (had) {
                const u64 val = c ? op_combine(op, sv[e - 1], pre[e]) : pre[e];
                const int ph = c ? shp[e - 1] : -1;
                if (ph >= 0) v[vslot(d, f, (u32)ph)] = val;
                else lpart[(size_t)blockIdx.x * F + f] = val;
            }
            // the tile's last group (complete, or cut by the tile's end), or the whole tile when it heads no group
            if (c == nch - 1) {
                if (mh >= 0) v[vslot(d, f, (u32)mh)] = mv;
                else lpart[(size_t)blockIdx.x * F + f] = mv;
            }
        }
    }
    __syncthreads();
    // the groups headed in the tile: rw words each, the head record's with the folded fields in place
    const u32 rw = d.rw, words = wpre[nw] * rw;
    u32* dst = out + tile_base[blockIdx.x] * rw;
    const u32* v32 = (const u32*)v;
#pragma unroll 4
    for (u32 lt = threadIdx.x; lt < words; lt += RR_THREADS) {
        const u32 j = d.inv_o ? __umulhi(lt, d.inv_o) : lt / rw, w = lt - j * rw;
        const u32 i = hidx[j], k = wkind[w];
        dst[lt] = k == 0xffff ? rec[(size_t)pos[i] * rw + w] : v32[2 * vslot(d, k >> 1, i) + (k & 1)];
    }
}

// One CTA per tile t < ntiles - 1: if t's last group runs on into tile t + 1, fold its pieces (lpart of tiles t + 1 .. b, b the
// first later tile that heads a group, or the last tile) in tile order into the partial rr_reduce_kernel wrote for it.
__global__ void __launch_bounds__(RR_THREADS)
rr_cut_kernel(const Pair* __restrict__ tup, u32 n, const u64* __restrict__ tile_sum, const u64* __restrict__ tile_base, u32 ntiles,
              const RRDesc d, const u64* __restrict__ lpart, u32* __restrict__ out) {
    __shared__ u64 red[RR_THREADS];
    __shared__ u32 sb;
    const u32 t = blockIdx.x, g = (t + 1) * d.T;
    if (tile_sum[t] == 0 || g >= n || tup[g].x != tup[g - 1].x) return;
    if (threadIdx.x == 0) sb = ntiles - 1;
    __syncthreads();
    for (u32 base = t + 1; base < ntiles; base += RR_THREADS) {
        const u32 u = base + threadIdx.x;
        const bool h = u < ntiles && tile_sum[u] != 0;
        if (h) atomicMin(&sb, u);
        if (__syncthreads_or(h)) break;
    }
    const u32 b = sb, R = (b - t + RR_THREADS - 1) / RR_THREADS;
    const u32 p0 = t + 1 + threadIdx.x * R, p1 = min(p0 + R, b + 1);
    u32* o = out + (tile_base[t] + tile_sum[t] - 1) * d.rw;
    for (u32 f = 0; f < d.nf; ++f) {
        const u32 r = run_of(d, f), wf = d.run_word[r] + 2 * (f - d.run_f0[r]);
        const int op = (int)d.run_op[r];
        u64 acc = op_identity(op);
        for (u32 q = p0; q < p1; ++q) acc = op_combine(op, acc, lpart[(size_t)q * d.nf + f]);
        red[threadIdx.x] = acc;
        __syncthreads();
        for (u32 s = 1; s < RR_THREADS; s <<= 1) {
            if ((threadIdx.x & (2 * s - 1)) == 0) red[threadIdx.x] = op_combine(op, red[threadIdx.x], red[threadIdx.x + s]);
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            const u64 x = op_combine(op, (u64)o[wf] | ((u64)o[wf + 1] << 32), red[0]);
            o[wf] = (u32)x;
            o[wf + 1] = (u32)(x >> 32);
        }
        __syncthreads();
    }
}

u32 pow2_floor(u32 x) { return x ? 1u << (31 - __builtin_clz(x)) : 0; }

size_t rr_smem_bytes(const RRDesc& d) {
    return (size_t)d.nf * d.fs * 8 + RR_THREADS * (8 + 8 + 4) + (size_t)d.T * 4 + (size_t)(2 * (d.T / 32) + 1) * 4 + (size_t)d.T * 2 +
           (size_t)d.rw * 2 + (size_t)d.nf * 4;
}

int check_reduce_records_args(tg_ctx* ctx, const tg_reduce_records_desc* dsc, RRDesc* d, RecSide* side) {
    if (!ctx || !dsc) return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records: NULL argument");
    *side = { dsc->item_bytes, dsc->key_offset, dsc->key_bytes };
    TG_TRY(check_side(ctx, "reduce_by_key_records", *side));
    if (ctx->nranks > TG_MAX_RANKS) return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records: at most 16 ranks");
    if (dsc->nruns > RR_MAX_RUNS) return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records: %u field runs (at most 8)", dsc->nruns);
    memset(d, 0, sizeof(*d));
    const u64 kb = dsc->key_offset, ke = kb + dsc->key_bytes;
    u32 nf = 0;
    for (u32 r = 0; r < dsc->nruns; ++r) {
        const tg_field_run& a = dsc->runs[r];
        const u64 b = a.offset, e = b + 8ull * a.count;
        if (a.count == 0 || a.op > TG_OP_MAX_F64 || a.offset % 4 || e > dsc->item_bytes)
            return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records: run %u {offset %u, count %u, op %u}: 1 or more 8-byte fields at "
                                "an offset that is a multiple of 4, inside the %u-byte item, op one of TG_OP_SUM_F64..TG_OP_MAX_F64",
                                r, a.offset, a.count, a.op, dsc->item_bytes);
        if (b < ke && kb < e) return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records: run %u overlaps the key", r);
        for (u32 q = 0; q < r; ++q) {
            const u64 qb = dsc->runs[q].offset, qe = qb + 8ull * dsc->runs[q].count;
            if (b < qe && qb < e) return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records: runs %u and %u overlap", q, r);
        }
        d->run_word[r] = a.offset / 4;
        d->run_f0[r] = nf;
        d->run_op[r] = a.op;
        nf += a.count;
    }
    d->run_f0[dsc->nruns] = nf;
    d->nruns = dsc->nruns;
    d->nf = nf;
    d->rw = dsc->item_bytes / 4;
    // nf <= 127 (the fields and a key of at least one byte fit in 1024 bytes): T >= 32, nf * nch <= RR_THREADS
    d->T = nf ? std::min(RR_MAX_TILE, pow2_floor(RR_VALUES / nf)) : RR_MAX_TILE;
    d->nch = nf ? std::min(d->T, pow2_floor(RR_THREADS / nf)) : 1;
    d->lc = __builtin_ctz(d->T / d->nch);
    d->fs = d->T + d->nch + 1;
    d->inv_g = nf ? gather_reciprocal(2 * nf) : 0;
    d->inv_o = gather_reciprocal(d->rw);
    return TG_OK;
}

// One local reduce of the n < 2^30 records at rec into WS_RR_OUT: *out, *m = its item count (one host read when n > 0)
int local_reduce(tg_ctx* ctx, const RRDesc& d, const RecSide& side, const void* rec, u64 n, void** out, u64* m) {
    TG_TRY(tg_ws_get(ctx, WS_RR_OUT, n * side.bytes + 16, out));
    *m = 0;
    if (!n) return TG_OK;
    const Pair* tup;
    TG_TRY(sort_record_tuples(ctx, WS_RR_TUP, rec, n, side, &tup));
    // scratch: the output size | tile sums | tile bases | the pieces' partials (ntiles x nf)
    const u32 ntiles = (u32)((n + d.T - 1) / d.T);
    u64* aux;
    TG_TRY(tg_ws_get(ctx, WS_RR_AUX, (2 + 2 * ((size_t)ntiles + 1) + (size_t)ntiles * d.nf) * 8, (void**)&aux));
    u64 *d_m = aux, *tile_sum = aux + 2, *tile_base = tile_sum + ntiles + 1, *lpart = tile_base + ntiles + 1;
    const size_t smem = rr_smem_bytes(d);
    if (ctx->kernel_cfg.find((const void*)rr_reduce_kernel) == ctx->kernel_cfg.end()) {
        TG_CUDA(ctx, cudaFuncSetAttribute(rr_reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RR_MAX_SMEM));
        ctx->kernel_cfg[(const void*)rr_reduce_kernel] = 1;
    }
    TG_LAUNCH_T(ctx, TG_K_REDUCE_RECORDS, rr_heads_kernel, ntiles, RR_THREADS, 0, tup, (u32)n, d.T, tile_sum);
    TG_LAUNCH_T(ctx, TG_K_REDUCE_RECORDS, join_scan_tiles_kernel, 1, JS_THREADS, 0, (const u64*)tile_sum, ntiles, tile_base, d_m);
    TG_LAUNCH_T(ctx, TG_K_REDUCE_RECORDS, rr_reduce_kernel, ntiles, RR_THREADS, smem, tup, (u32)n, (const u32*)rec,
                (const u64*)tile_base, d, lpart, (u32*)*out);
    if (ntiles > 1 && d.nf)
        TG_LAUNCH_T(ctx, TG_K_REDUCE_RECORDS, rr_cut_kernel, ntiles - 1, RR_THREADS, 0, tup, (u32)n, (const u64*)tile_sum,
                    (const u64*)tile_base, ntiles, d, (const u64*)lpart, (u32*)*out);
    u64* h = (u64*)ctx->pinned + 65536;          // byte offset 512 KB of the pinned scratch
    TG_CUDA(ctx, cudaMemcpyAsync(h, d_m, 8, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *m = h[0];
    return TG_OK;
}

int reduce_records_impl(tg_ctx* ctx, const RRDesc& d, const RecSide& side, const void* d_in, size_t n_local, void** out_dptr,
                        size_t* out_n) {
    const int p = ctx->nranks;
    const bool too_large = n_local >= RR_LIMIT;
    // an input in a slot the local reduce writes (the un-detached result of an earlier reduce on records) is copied out of the way
    const void* rec = d_in;
    const size_t bytes = too_large ? 0 : n_local * side.bytes;
    const int dst = WS_RR_IN;
    TG_TRY(move_inputs_out_of_slots(ctx, &rec, &bytes, 1, { WS_RR_TUP, WS_RR_AUX, WS_RR_OUT }, &dst));
    void* out;
    u64 m;
    if (p == 1) {
        if (too_large) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "reduce_by_key_records: %zu items (limit 2^30 - 1)", n_local);
        TG_TRY(local_reduce(ctx, d, side, rec, n_local, &out, &m));
        *out_dptr = out;
        *out_n = (size_t)m;
        return TG_OK;
    }
    // pre phase: at most one record per local key goes into the exchange.  A worker of 2^30 or more items takes part with none
    // and reports 2^30 for worker 0, so that the count matrix gives TG_ERR_TOO_LARGE on every rank.
    TG_TRY(xwin_negotiate(ctx));
    void* pre = nullptr;
    u64 m_pre = 0;
    if (!too_large) TG_TRY(local_reduce(ctx, d, side, rec, n_local, &pre, &m_pre));
    Pair* ptup;
    u32* d_tot;
    TG_TRY(partition_record_tuples(ctx, pre, m_pre, side, (u32)p, &ptup, &d_tot));
    if (too_large) TG_CUDA(ctx, cudaMemsetAsync((char*)d_tot + 3, 0x40, 1, ctx->stream));     // totals[0] = 2^30
    XchgResult xr;
    u64 need = 0;
    TG_TRY(xchg_counts(ctx, d_tot, (int)side.bytes, &xr, &need));                  // (synchronises; uniform verdicts)
    TG_TRY(xwin_ensure(ctx, need));
    TG_TRY(exchange_store_records(ctx, ctx->xwin.mode, false, pre, side.bytes, ptup, m_pre, xchg_matrix(ctx), p, ctx->rank, ctx->xwin.peer));
    if (ctx->xwin.mode == 1) TG_TRY(xwin_barrier(ctx));
    // post phase: the received records (the pre phase's output in WS_RR_OUT has been read by the exchange)
    TG_TRY(local_reduce(ctx, d, side, ctx->xwin.base, xr.n_recv, &out, &m));
    *out_dptr = out;
    *out_n = (size_t)m;
    return TG_OK;
}

}  // namespace

extern "C" {

int tg_reduce_by_key_records(tg_ctx* ctx, const tg_reduce_records_desc* desc, const void* d_in, size_t n_local, void** out_dptr,
                             size_t* out_n) {
    RRDesc d;
    RecSide side;
    TG_TRY(check_reduce_records_args(ctx, desc, &d, &side));
    if (!out_dptr || !out_n || (!d_in && n_local)) return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records: NULL argument");
    if ((uintptr_t)d_in & 3) return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records: records must be 4-byte aligned");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return reduce_records_impl(ctx, d, side, d_in, n_local, out_dptr, out_n);
}

int tg_reduce_by_key_records_file(tg_ctx* ctx, const tg_reduce_records_desc* desc, const tg_merge_input* in, size_t* out_items) {
    RRDesc d;
    RecSide side;
    TG_TRY(check_reduce_records_args(ctx, desc, &d, &side));
    if (!in || !out_items) return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records_file: NULL argument");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const u32 s = side.bytes;
    const void* ptr = nullptr;
    size_t n = 0;
    if (in->dev) {
        // a device File is read in place
        const tg_dev_file& f = *in->dev;
        if (f.item_bytes != s || (!f.dptr && f.items) || ((uintptr_t)f.dptr & 3))
            return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records_file: the device File has item size %u, the descriptor says %u", f.item_bytes, s);
        ptr = f.dptr;
        n = f.items;
    }
    else {
        // a host File goes up into the staging buffer
        if (!in->blocks && in->nblocks) return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records_file: the input has no blocks");
        size_t bytes = 0;
        for (size_t i = 0; i < in->nblocks; ++i) bytes += in->blocks[i].bytes;
        if (bytes % s) return tg_set_error(ctx, TG_ERR_ARG, "reduce_by_key_records_file: %zu bytes is not a multiple of %u", bytes, s);
        n = bytes / s;
        // over the limit: nothing is uploaded (with p > 1 the worker still takes part in the exchange's count matrix, with no items)
        if (n >= RR_LIMIT && ctx->nranks == 1)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "reduce_by_key_records_file: %zu items (limit 2^30 - 1)", n);
        if (n && n < RR_LIMIT) {
            void* d_stage;
            TG_TRY(tg_ws_get(ctx, WS_IN, bytes + 16, &d_stage));
            TG_TRY(tg_upload_blocks(ctx, d_stage, in->blocks, in->nblocks, nullptr));
            ptr = d_stage;
        }
    }
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(reduce_records_impl(ctx, d, side, ptr, n, &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = s;
    *out_items = n_out;
    return TG_OK;
}

}  // extern "C"
