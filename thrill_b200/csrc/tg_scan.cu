// tg_scan.cu — PrefixSum / ExPrefixSum (PrefixSumNode, api/prefix_sum.hpp:28-128) and ZipWithIndex (ZipWithIndexNode,
// api/zip_with_index.hpp:40-110): every worker keeps its items in order and each output needs the fold of everything before it.
//
// PrefixSum is a reduce-then-scan with no CTA waiting on another:
//   1. scan_reduce_kernel   reads each tile once (16-byte loads) and writes one aggregate per tile
//   2. scan_prefix_kernel   one CTA: the worker's local total S = T() + agg_0 + ... (phase TOTAL, what the worker contributes to
//                           the all-gather), and, once the totals of all workers are in device memory, the carry
//                           carry_r = initial + (S_0 + ... + S_{r-1}) and the exclusive scan of the tile aggregates seeded with
//                           it (phase PREFIX)
//   3. scan_tiles_kernel    re-reads each tile and scans it in registers from its tile prefix: thread-sequential over the
//                           thread's 128 bytes, then warp shuffles, then across the warps; writes inclusive or exclusive outputs
// Traffic: 24 bytes per item for 8-byte items, 48 for pairs.  The bracketing of a double sum is fixed by the tile geometry, never
// by timing, so a result is bitwise identical from run to run (a decoupled look-back would make it depend on which tiles had
// published; it would also have CTAs spin on each other, DESIGN.md §10).
// The sum functions work on one 8-byte value: the whole item, or a pair's .second.  A pair's .first is positional: ScanSecond
// takes it from the right-hand operand, so an inclusive output keeps its item's .first and an exclusive one takes the previous
// item's (the carry's for the worker's first item).
// ZipWithIndex: zip_index_kernel reads 8 bytes and writes 16 per item; the base index is the sum of the lower ranks' sizes.
//
// The actions Sum / Min / Max / AllReduce (AllReduceNode, api/all_reduce.hpp:27-85) reuse the tile reduce and the record:
//   1. scan_reduce_kernel   one aggregate per tile (8 bytes per item read, 16 for pairs, nothing written but the aggregates)
//   2. action_fold_kernel   one CTA: phase TOTAL folds the aggregates in order into the worker's value and writes its record;
//                           phase RESULT folds the p records (all-gathered, or filled in place by _select) in rank order
// Min / Max on doubles are exact and not commutative (std::min(a, b) = b < a ? b : a keeps the earlier of two equal values, and
// a NaN first operand sticks).  Their tile reduce folds positions in order (each thread a contiguous run, then lanes and warps
// in order) with a NaN-skipping function, and the first operand of the stock fold is applied on its own in the fold kernel.
#include "tg_common.cuh"
#include "tg_fold.cuh"

namespace {

constexpr u64 SCAN_LIMIT = 1ull << 30;
constexpr int SC_THREADS = 256;                 // scan_reduce_kernel / scan_tiles_kernel
constexpr int SC_UNITS = 8;                     // 16-byte units per thread: 128 bytes
constexpr int TILE_UNITS = SC_THREADS * SC_UNITS;   // 32 KB: 4096 8-byte items or 2048 pairs
// a thread's row in shared memory: its 16 words and 4 words of padding, so that the 8 threads of a quarter-warp reading
// 16 bytes each at the same column hit 8 distinct 4-bank groups
constexpr int ROW_WORDS = 2 * SC_UNITS + 4;
constexpr int ST_THREADS = 512;                 // scan_prefix_kernel (one CTA)
constexpr int ST_PER = 8;                       // aggregates per thread and round
constexpr int ZIP_THREADS = 256, ZIP_PER = 4;

enum { STEP_REDUCE = 1, STEP_TOTAL = 2, STEP_PREFIX = 4, STEP_SCAN = 8, STEP_RESULT = 16 };

// what each worker contributes to the all-gather: its size and its local total S (for pairs: S.first = the .first of its
// last item, 0 if it has none)
struct ScanRec { u64 n, first, value, pad; };

// T(): the value-initialised item the stock node folds its local total from (+0.0, 0)
constexpr u64 T_VALUE = 0;

template <int OP>
__device__ __forceinline__ u64 warp_reduce(u64 v) {
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) v = combine<OP>(v, __shfl_down_sync(0xffffffffu, v, d));
    return v;                                   // (lane 0)
}
// the same with lane 0 holding the lanes' values folded in lane order
template <int OP>
__device__ __forceinline__ u64 warp_reduce_in_order(u64 v) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) v = combine<OP>(v, __shfl_down_sync(0xffffffffu, v, d));
    return v;                                   // (lane 0)
}

// inclusive scan over the lanes (left to right), and the exclusive value of each lane
template <int OP>
__device__ __forceinline__ u64 warp_scan(u64 v, u64* excl) {
    const u32 lane = lane_id();
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u64 o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= (u32)d) v = combine<OP>(o, v);
    }
    const u64 e = __shfl_up_sync(0xffffffffu, v, 1);
    *excl = lane ? e : ident<OP>();
    return v;
}

// pass 1: agg[tile] = the fold of the tile's values (in position order for in_order ops: thread t takes the units 8t..8t+7)
template <int OP, int IB>
__global__ void __launch_bounds__(SC_THREADS) scan_reduce_kernel(const ulonglong2* __restrict__ in, u64 n, u64* __restrict__ agg) {
    __shared__ u64 wsum[SC_THREADS / 32];
    const u64 tile = (u64)blockIdx.x * TILE_UNITS;
    ulonglong2 v[SC_UNITS];
#pragma unroll
    for (int j = 0; j < SC_UNITS; ++j)
        v[j] = load_unit<OP, IB>(in, in_order<OP>() ? tile + threadIdx.x * SC_UNITS + j : tile + threadIdx.x + (u64)j * SC_THREADS, n);
    u64 acc = IB == 16 ? v[0].y : combine<OP>(v[0].x, v[0].y);
#pragma unroll
    for (int j = 1; j < SC_UNITS; ++j) acc = IB == 16 ? combine<OP>(acc, v[j].y) : combine<OP>(combine<OP>(acc, v[j].x), v[j].y);
    acc = in_order<OP>() ? warp_reduce_in_order<OP>(acc) : warp_reduce<OP>(acc);
    if (lane_id() == 0) wsum[threadIdx.x / 32] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        u64 t = wsum[0];
#pragma unroll
        for (int w = 1; w < SC_THREADS / 32; ++w) t = combine<OP>(t, wsum[w]);
        agg[blockIdx.x] = t;
    }
}

// phase TOTAL: *my_rec = (n, last .first, T() + the fold of the aggregates).  Phase PREFIX: carry = initial for rank 0, else
// initial + (S_0 + ... + S_{rank-1}) from the gathered records, the inner fold left to right (net/flow_control_channel.hpp:
// 259-276); carry_out = (carry.first, carry.value); tile_prefix[t] = carry + (agg_0 + ... + agg_{t-1}).
template <int OP, int IB>
__global__ void __launch_bounds__(ST_THREADS) scan_prefix_kernel(const u64* __restrict__ agg, u32 ntiles, u32 steps,
                                                                 const ulonglong2* __restrict__ in, u64 n, ScanRec* my_rec,
                                                                 const ScanRec* __restrict__ recs, u32 rank, u64 init_first,
                                                                 u64 init_value, u64* __restrict__ tile_prefix, u64* carry_out) {
    __shared__ u64 wsum[ST_THREADS / 32];
    __shared__ u64 s_carry;
    const u32 tid = threadIdx.x, lane = lane_id(), warp = tid / 32;
    if ((steps & STEP_PREFIX) && tid == 0) {
        u64 c = init_value, cf = init_first;
        if (rank) {
            u64 inner = recs[0].value;
            for (u32 i = 1; i < rank; ++i) inner = combine<OP>(inner, recs[i].value);
            c = combine<OP>(init_value, inner);
            cf = recs[rank - 1].first;
        }
        carry_out[0] = cf;
        carry_out[1] = c;
        s_carry = c;
    }
    __syncthreads();
    u64 running = ident<OP>();
    for (u32 base = 0; base < ntiles; base += ST_THREADS * ST_PER) {
        u64 v[ST_PER];
        const u32 i0 = base + tid * ST_PER;
#pragma unroll
        for (int k = 0; k < ST_PER; ++k) v[k] = i0 + k < ntiles ? agg[i0 + k] : ident<OP>();
        u64 t = v[0];
#pragma unroll
        for (int k = 1; k < ST_PER; ++k) t = combine<OP>(t, v[k]);
        u64 lane_excl;
        const u64 incl = warp_scan<OP>(t, &lane_excl);
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        u64 wpre = ident<OP>(), chunk = ident<OP>();
        for (u32 w = 0; w < ST_THREADS / 32; ++w) {
            if (w == warp) wpre = chunk;
            chunk = combine<OP>(chunk, wsum[w]);
        }
        if (steps & STEP_PREFIX) {
            u64 e = combine<OP>(running, combine<OP>(wpre, lane_excl));
            const u64 c = s_carry;
#pragma unroll
            for (int k = 0; k < ST_PER; ++k) {
                if (i0 + k < ntiles) tile_prefix[i0 + k] = combine<OP>(c, e);
                e = combine<OP>(e, v[k]);
            }
        }
        running = combine<OP>(running, chunk);
        __syncthreads();
    }
    if ((steps & STEP_TOTAL) && tid == 0) {
        my_rec->n = n;
        my_rec->first = IB == 16 && n ? in[n - 1].x : 0;
        my_rec->value = combine<OP>(T_VALUE, running);
        my_rec->pad = 0;
    }
}

// pass 2: the tile scanned from tile_prefix[tile]; carry_in[0] = the .first an exclusive pair output 0 takes
template <int OP, int IB, bool INCL>
__global__ void __launch_bounds__(SC_THREADS, 2) scan_tiles_kernel(const ulonglong2* __restrict__ in, u64 n,
                                                                const u64* __restrict__ tile_prefix,
                                                                const u64* __restrict__ carry_in, ulonglong2* __restrict__ out) {
    constexpr int IPT = IB == 16 ? SC_UNITS : 2 * SC_UNITS;     // items per thread
    __shared__ __align__(16) u64 rows[SC_THREADS * ROW_WORDS];
    __shared__ u64 wsum[SC_THREADS / 32];
    const u32 tid = threadIdx.x, lane = lane_id(), warp = tid / 32;
    const u64 ubase = (u64)blockIdx.x * TILE_UNITS;
    // striped, coalesced 16-byte loads into the threads' rows
#pragma unroll
    for (int j = 0; j < SC_UNITS; ++j) {
        const u32 ul = j * SC_THREADS + tid;
        const ulonglong2 v = load_unit<OP, IB>(in, ubase + ul, n);
        *(ulonglong2*)&rows[(ul / SC_UNITS) * ROW_WORDS + 2 * (ul % SC_UNITS)] = v;
    }
    const u64 tprefix = tile_prefix[blockIdx.x];
    u64 prev_first = 0;
    if (IB == 16 && !INCL && tid == 0) prev_first = blockIdx.x ? in[ubase - 1].x : carry_in[0];
    __syncthreads();
    // this thread's 128 consecutive bytes
    u64 v[IPT], f[IB == 16 ? IPT : 1];
    const u64* row = &rows[tid * ROW_WORDS];
#pragma unroll
    for (int k = 0; k < IPT; ++k) {
        if (IB == 16) { f[k] = row[2 * k]; v[k] = row[2 * k + 1]; }
        else v[k] = row[k];
    }
    if (IB == 16 && !INCL && tid) prev_first = rows[(tid - 1) * ROW_WORDS + 2 * (SC_UNITS - 1)];
    u64 t = v[0];
#pragma unroll
    for (int k = 1; k < IPT; ++k) t = combine<OP>(t, v[k]);
    u64 lane_excl;
    const u64 incl = warp_scan<OP>(t, &lane_excl);
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();                            // (also: every row has been read before any is overwritten)
    u64 wpre = ident<OP>();
    for (u32 w = 0; w < warp; ++w) wpre = combine<OP>(wpre, wsum[w]);
    u64 run = combine<OP>(combine<OP>(tprefix, wpre), lane_excl);
#pragma unroll
    for (int k = 0; k < IPT; ++k) {
        if (INCL) { run = combine<OP>(run, v[k]); v[k] = run; }
        else { const u64 x = v[k]; v[k] = run; run = combine<OP>(run, x); }
    }
    u64* wrow = &rows[tid * ROW_WORDS];
#pragma unroll
    for (int k = 0; k < IPT; ++k) {
        if (IB == 16) {
            wrow[2 * k] = INCL ? f[k] : (k ? f[k - 1] : prev_first);
            wrow[2 * k + 1] = v[k];
        }
        else wrow[k] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < SC_UNITS; ++j) {
        const u32 ul = j * SC_THREADS + tid;
        const u64 u = ubase + ul;
        const ulonglong2 o = *(const ulonglong2*)&rows[(ul / SC_UNITS) * ROW_WORDS + 2 * (ul % SC_UNITS)];
        if (IB == 16) { if (u < n) out[u] = o; }
        else if (2 * u + 1 < n) out[u] = o;
        else if (2 * u < n) ((u64*)out)[2 * u] = o.x;
    }
}

// ZipWithIndex: out[i] = (base + i, in[i]) or (in[i], base + i)
template <bool INDEX_FIRST>
__global__ void __launch_bounds__(ZIP_THREADS) zip_index_kernel(const u64* __restrict__ in, u64 n, u64 base, ulonglong2* __restrict__ out) {
    const u64 i0 = (u64)blockIdx.x * (ZIP_THREADS * ZIP_PER) + threadIdx.x;
    u64 x[ZIP_PER];
#pragma unroll
    for (int k = 0; k < ZIP_PER; ++k) {
        const u64 i = i0 + (u64)k * ZIP_THREADS;
        x[k] = i < n ? in[i] : 0;
    }
#pragma unroll
    for (int k = 0; k < ZIP_PER; ++k) {
        const u64 i = i0 + (u64)k * ZIP_THREADS;
        if (i < n) out[i] = INDEX_FIRST ? make_ulonglong2(base + i, x[k]) : make_ulonglong2(x[k], base + i);
    }
}

// The actions.  Phase TOTAL: R = agg_0 + ... + agg_{ntiles-1} in order (each thread a contiguous run, then lanes and warps in
// order), and *my_rec = (n, .first of the last item, W) with the stock node's worker value (all_reduce.hpp:36-63, whose value
// starts as the initial value on every worker):
//   no items: the initial value if there is one (init & INIT_GIVEN), else T();  otherwise initial + R on the worker that folds
//   it (init & INIT_FOLD: worker 0), else R (the fold of every item from the first).  For Min / Max on doubles the first
//   operand, initial or x_0, goes through the stock function.
// Phase RESULT: out = (recs[p-1].first, recs[0] + ... + recs[p-1]) folded left to right with the stock function.
enum { INIT_GIVEN = 1, INIT_FOLD = 2 };
template <int OP, int IB>
__global__ void __launch_bounds__(ST_THREADS) action_fold_kernel(const u64* __restrict__ agg, u32 ntiles, u32 steps,
                                                                 const ulonglong2* __restrict__ in, u64 n, int init,
                                                                 u64 init_first, u64 init_value, ScanRec* my_rec,
                                                                 const ScanRec* recs, u32 p, u64* out) {
    __shared__ u64 wsum[ST_THREADS / 32];
    const u32 tid = threadIdx.x;
    if (steps & STEP_TOTAL) {
        const u32 per = (ntiles + ST_THREADS - 1) / ST_THREADS, b = tid * per, e = min(b + per, ntiles);
        u64 acc = ident<OP>();
        for (u32 i = b; i < e; ++i) acc = combine<OP>(acc, agg[i]);
        acc = warp_reduce_in_order<OP>(acc);
        if (lane_id() == 0) wsum[tid / 32] = acc;
        __syncthreads();
        if (tid == 0) {
            u64 r = wsum[0];
            for (int w = 1; w < ST_THREADS / 32; ++w) r = combine<OP>(r, wsum[w]);
            u64 first = 0, value = T_VALUE;
            const bool fold_init = init & INIT_FOLD;
            if (n) {
                first = IB == 16 ? in[n - 1].x : 0;
                if (in_order<OP>()) value = stock_fn<OP>(fold_init ? init_value : IB == 16 ? in[0].y : in[0].x, r);
                else value = fold_init ? combine<OP>(init_value, r) : r;
            }
            else if (init & INIT_GIVEN) { first = init_first; value = init_value; }
            *my_rec = ScanRec{ n, first, value, 0 };
        }
    }
    if ((steps & STEP_RESULT) && tid == 0) {
        u64 v = recs[0].value;
        for (u32 r = 1; r < p; ++r) v = stock_fn<OP>(v, recs[r].value);
        out[0] = recs[p - 1].first;
        out[1] = v;
    }
}

// ---- host side ---------------------------------------------------------------------------------------------------------------

// one scan on one worker.  The WS_SCAN_AUX workspace holds, in this order: carry (2 words), this worker's record, the p
// gathered records, then the tile aggregates and the tile prefixes.
constexpr size_t AUX_CARRY = 0, AUX_REC = 64, AUX_RECS = 128, AUX_TILES = AUX_RECS + TG_MAX_RANKS * sizeof(ScanRec);
struct ScanJob {
    uint32_t op = 0, ib = 8;
    const void* in = nullptr;
    u64 n = 0;
    int inclusive = 1;
    u64 init_first = 0, init_value = 0;
    u32 rank = 0;
    char* aux = nullptr;
    void* out = nullptr;
    u32 ntiles() const { return (u32)((n * ib + TILE_UNITS * 16 - 1) / (TILE_UNITS * 16)); }
    u64* agg() const { return (u64*)(aux + AUX_TILES); }
    u64* prefix() const { return agg() + ((ntiles() + 1) & ~1u); }
    ScanRec* my_rec() const { return (ScanRec*)(aux + AUX_REC); }
    ScanRec* recs() const { return (ScanRec*)(aux + AUX_RECS); }
    u64* carry() const { return (u64*)(aux + AUX_CARRY); }
};

template <int OP, int IB>
int scan_steps(tg_ctx* ctx, const ScanJob& j, int steps) {
    const u32 nt = j.ntiles();
    const ulonglong2* in = (const ulonglong2*)j.in;
    if ((steps & STEP_REDUCE) && nt)
        TG_LAUNCH_T(ctx, TG_K_SCAN, (scan_reduce_kernel<OP, IB>), nt, SC_THREADS, 0, in, j.n, j.agg());
    if (steps & (STEP_TOTAL | STEP_PREFIX))
        TG_LAUNCH_T(ctx, TG_K_SCAN, (scan_prefix_kernel<OP, IB>), 1, ST_THREADS, 0, (const u64*)j.agg(), nt,
                    (u32)(steps & (STEP_TOTAL | STEP_PREFIX)), in, j.n, j.my_rec(), (const ScanRec*)j.recs(), j.rank,
                    j.init_first, j.init_value, j.prefix(), j.carry());
    if ((steps & STEP_SCAN) && nt) {
        if (j.inclusive)
            TG_LAUNCH_T(ctx, TG_K_SCAN, (scan_tiles_kernel<OP, IB, true>), nt, SC_THREADS, 0, in, j.n, (const u64*)j.prefix(),
                        (const u64*)j.carry(), (ulonglong2*)j.out);
        else
            TG_LAUNCH_T(ctx, TG_K_SCAN, (scan_tiles_kernel<OP, IB, false>), nt, SC_THREADS, 0, in, j.n, (const u64*)j.prefix(),
                        (const u64*)j.carry(), (ulonglong2*)j.out);
    }
    return TG_OK;
}

template <int OP>
int scan_steps_ib(tg_ctx* ctx, const ScanJob& j, int steps) {
    return j.ib == 16 ? scan_steps<OP, 16>(ctx, j, steps) : scan_steps<OP, 8>(ctx, j, steps);
}

int scan_run(tg_ctx* ctx, const ScanJob& j, int steps) {
    switch (j.op) {
    case TG_OP_SUM_F64: return scan_steps_ib<TG_OP_SUM_F64>(ctx, j, steps);
    case TG_OP_SUM_U64: return scan_steps_ib<TG_OP_SUM_U64>(ctx, j, steps);
    case TG_OP_MIN_U64: return scan_steps_ib<TG_OP_MIN_U64>(ctx, j, steps);
    default: return scan_steps_ib<TG_OP_MAX_U64>(ctx, j, steps);
    }
}

int check_desc(tg_ctx* ctx, const tg_scan_desc* desc) {
    if (!desc) return tg_set_error(ctx, TG_ERR_ARG, "prefix_sum: NULL descriptor");
    if (desc->item_bytes != 8 && desc->item_bytes != 16)
        return tg_set_error(ctx, TG_ERR_ARG, "prefix_sum: %u-byte items (8: uint64_t / double, 16: pair<uint64_t, V>)", desc->item_bytes);
    if (desc->op != TG_OP_SUM_F64 && desc->op != TG_OP_SUM_U64 && desc->op != TG_OP_MIN_U64 && desc->op != TG_OP_MAX_U64)
        return tg_set_error(ctx, TG_ERR_ARG, "prefix_sum: op %u (std::plus<double>, std::plus<uint64_t>, MinU64 and MaxU64 only)", desc->op);
    return TG_OK;
}

// the job's aux workspace (records, aggregates, prefixes) for n items
int prepare_aux(tg_ctx* ctx, ScanJob* j, u64 n) {
    n = n < SCAN_LIMIT ? n : 0;                         // (an input over the limit is only counted, never read)
    const u64 nt = (n * j->ib + TILE_UNITS * 16 - 1) / (TILE_UNITS * 16);
    void* aux;
    TG_TRY(tg_ws_get(ctx, WS_SCAN_AUX, AUX_TILES + (nt + 2) * 16, &aux));
    j->aux = (char*)aux;
    return TG_OK;
}

// ... and the output of n items of out_bytes
int prepare(tg_ctx* ctx, ScanJob* j, uint32_t out_bytes) {
    const u64 n = j->n < SCAN_LIMIT ? j->n : 0;
    TG_TRY(prepare_aux(ctx, j, j->n));
    void* out;
    TG_TRY(tg_ws_get(ctx, WS_SCAN_OUT, n * out_bytes + 16, &out));
    j->out = out;
    return TG_OK;
}

void set_initial(ScanJob* j, const void* initial_item) {
    u64 w[2] = { 0, 0 };
    if (initial_item) memcpy(w, initial_item, j->ib);
    if (j->ib == 16) { j->init_first = w[0]; j->init_value = w[1]; }
    else { j->init_first = 0; j->init_value = w[0]; }
}

// p > 1: this worker's record into the all-gather, then one host read of the gathered sizes (the verdict on the limit is the
// same on every rank); the gathered records stay in device memory for the carry fold
int gather_records(tg_ctx* ctx, const ScanJob& j, bool with_total, const char* what, u64* sizes) {
    const int p = ctx->nranks;
    if (j.n >= SCAN_LIMIT || !with_total) {
        ScanRec* hr = (ScanRec*)ctx->pinned;
        *hr = ScanRec{ j.n, 0, 0, 0 };
        TG_CUDA(ctx, cudaMemcpyAsync(j.my_rec(), hr, sizeof(ScanRec), cudaMemcpyHostToDevice, ctx->stream));
    }
    TG_NCCL(ctx, ncclAllGather(j.my_rec(), j.recs(), sizeof(ScanRec) / 8, ncclUint64, ctx->comm, ctx->stream));
    ScanRec* hrecs = (ScanRec*)((char*)ctx->pinned + 4096);
    TG_CUDA(ctx, cudaMemcpyAsync(hrecs, j.recs(), p * sizeof(ScanRec), cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int r = 0; r < p; ++r) {
        sizes[r] = hrecs[r].n;
        if (hrecs[r].n >= SCAN_LIMIT)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "%s: worker %d holds %llu items (limit 2^30 - 1)", what, r,
                                (unsigned long long)hrecs[r].n);
    }
    return TG_OK;
}

int prefix_sum_impl(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n_local, const void* initial_item,
                    int inclusive, void** out_dptr, size_t* out_n) {
    const int p = ctx->nranks;
    if (p == 1 && n_local >= SCAN_LIMIT)
        return tg_set_error(ctx, TG_ERR_TOO_LARGE, "prefix_sum: n_local=%zu (limit 2^30 - 1)", n_local);
    ScanJob j;
    j.op = desc->op; j.ib = desc->item_bytes; j.in = d_in; j.n = n_local; j.inclusive = inclusive; j.rank = (u32)ctx->rank;
    set_initial(&j, initial_item);
    TG_TRY(prepare(ctx, &j, j.ib));
    if (p == 1) TG_TRY(scan_run(ctx, j, STEP_REDUCE | STEP_PREFIX | STEP_SCAN));
    else {
        if (n_local < SCAN_LIMIT) TG_TRY(scan_run(ctx, j, STEP_REDUCE | STEP_TOTAL));
        u64 sizes[TG_MAX_RANKS];
        TG_TRY(gather_records(ctx, j, true, "prefix_sum", sizes));
        TG_TRY(scan_run(ctx, j, STEP_PREFIX | STEP_SCAN));
    }
    *out_dptr = j.out;
    *out_n = n_local;
    return TG_OK;
}

int zip_launch(tg_ctx* ctx, const void* d_in, u64 n, u64 base, int index_first, void* out) {
    if (!n) return TG_OK;
    const u64 grid = (n + ZIP_THREADS * ZIP_PER - 1) / (ZIP_THREADS * ZIP_PER);
    if (index_first) TG_LAUNCH_T(ctx, TG_K_SCAN, zip_index_kernel<true>, grid, ZIP_THREADS, 0, (const u64*)d_in, n, base, (ulonglong2*)out);
    else TG_LAUNCH_T(ctx, TG_K_SCAN, zip_index_kernel<false>, grid, ZIP_THREADS, 0, (const u64*)d_in, n, base, (ulonglong2*)out);
    return TG_OK;
}

int zip_impl(tg_ctx* ctx, const void* d_in, size_t n_local, int index_first, void** out_dptr, size_t* out_n) {
    const int p = ctx->nranks;
    if (p == 1 && n_local >= SCAN_LIMIT)
        return tg_set_error(ctx, TG_ERR_TOO_LARGE, "zip_with_index: n_local=%zu (limit 2^30 - 1)", n_local);
    ScanJob j;
    j.ib = 8; j.in = d_in; j.n = n_local; j.rank = (u32)ctx->rank;
    TG_TRY(prepare(ctx, &j, 16));
    u64 base = 0;
    if (p > 1) {
        u64 sizes[TG_MAX_RANKS];
        TG_TRY(gather_records(ctx, j, false, "zip_with_index", sizes));
        for (int r = 0; r < ctx->rank; ++r) base += sizes[r];
    }
    TG_TRY(zip_launch(ctx, d_in, n_local, base, index_first, j.out));
    *out_dptr = j.out;
    *out_n = n_local;
    return TG_OK;
}

int check_ranks(tg_ctx* ctx) {
    if (ctx->nranks > TG_MAX_RANKS) return tg_set_error(ctx, TG_ERR_ARG, "scan: at most 16 ranks");
    return TG_OK;
}

// a host File goes up into the WS_IN staging buffer, a device File is read where it is
int stage_input(tg_ctx* ctx, const tg_merge_input* in, uint32_t item_bytes, const void** d_in, size_t* n) {
    if (in->dev) {
        if (in->dev->item_bytes != item_bytes || (!in->dev->dptr && in->dev->items))
            return tg_set_error(ctx, TG_ERR_ARG, "scan_file: the device File has item size %u, the operator takes %u",
                                in->dev->item_bytes, item_bytes);
        *d_in = in->dev->dptr;
        *n = in->dev->items;
        return TG_OK;
    }
    if (!in->blocks && in->nblocks) return tg_set_error(ctx, TG_ERR_ARG, "scan_file: the input has no blocks");
    size_t bytes = 0;
    for (size_t i = 0; i < in->nblocks; ++i) bytes += in->blocks[i].bytes;
    if (bytes % item_bytes) return tg_set_error(ctx, TG_ERR_ARG, "scan_file: %zu bytes is not a multiple of %u", bytes, item_bytes);
    *n = bytes / item_bytes;
    *d_in = nullptr;
    if (bytes) {
        void* d;
        TG_TRY(tg_ws_get(ctx, WS_IN, bytes + 16, &d));
        TG_TRY(tg_upload_blocks(ctx, d, in->blocks, in->nblocks, nullptr));
        *d_in = d;
    }
    return TG_OK;
}

// ---- the actions ------------------------------------------------------------------------------------------------------------

int check_action_desc(tg_ctx* ctx, const tg_scan_desc* desc) {
    if (!desc) return tg_set_error(ctx, TG_ERR_ARG, "all_reduce: NULL descriptor");
    if (desc->item_bytes != 8 && desc->item_bytes != 16)
        return tg_set_error(ctx, TG_ERR_ARG, "all_reduce: %u-byte items (8: uint64_t / double, 16: pair<uint64_t, V>)", desc->item_bytes);
    if (desc->op > TG_OP_MAX_F64)
        return tg_set_error(ctx, TG_ERR_ARG, "all_reduce: op %u (sum, min and max of uint64_t and double only)", desc->op);
    return TG_OK;
}

// steps of one worker (STEP_REDUCE | STEP_TOTAL into *rec) and / or the fold of the p records at j.recs() (STEP_RESULT into
// j.carry()); init: INIT_GIVEN | INIT_FOLD flags of this worker
template <int OP, int IB>
int action_steps(tg_ctx* ctx, const ScanJob& j, int steps, int init, ScanRec* rec, u32 p) {
    const u32 nt = j.ntiles();
    const ulonglong2* in = (const ulonglong2*)j.in;
    if ((steps & STEP_REDUCE) && nt)
        TG_LAUNCH_T(ctx, TG_K_SCAN, (scan_reduce_kernel<OP, IB>), nt, SC_THREADS, 0, in, j.n, j.agg());
    if (steps & (STEP_TOTAL | STEP_RESULT))
        TG_LAUNCH_T(ctx, TG_K_SCAN, (action_fold_kernel<OP, IB>), 1, ST_THREADS, 0, (const u64*)j.agg(), nt,
                    (u32)(steps & (STEP_TOTAL | STEP_RESULT)), in, j.n, init, j.init_first, j.init_value, rec,
                    (const ScanRec*)j.recs(), p, j.carry());
    return TG_OK;
}

template <int OP>
int action_steps_ib(tg_ctx* ctx, const ScanJob& j, int steps, int init, ScanRec* rec, u32 p) {
    return j.ib == 16 ? action_steps<OP, 16>(ctx, j, steps, init, rec, p) : action_steps<OP, 8>(ctx, j, steps, init, rec, p);
}

int action_run(tg_ctx* ctx, const ScanJob& j, int steps, int init, ScanRec* rec, u32 p) {
    switch (j.op) {
    case TG_OP_SUM_F64: return action_steps_ib<TG_OP_SUM_F64>(ctx, j, steps, init, rec, p);
    case TG_OP_SUM_U64: return action_steps_ib<TG_OP_SUM_U64>(ctx, j, steps, init, rec, p);
    case TG_OP_MIN_U64: return action_steps_ib<TG_OP_MIN_U64>(ctx, j, steps, init, rec, p);
    case TG_OP_MAX_U64: return action_steps_ib<TG_OP_MAX_U64>(ctx, j, steps, init, rec, p);
    case TG_OP_MIN_F64: return action_steps_ib<TG_OP_MIN_F64>(ctx, j, steps, init, rec, p);
    default: return action_steps_ib<TG_OP_MAX_F64>(ctx, j, steps, init, rec, p);
    }
}

// the one host read: the result words and the p records (aux bytes [0, AUX_RECS + p records)), then the verdict on the limit
// (the same on every rank) and the result item
int action_finish(tg_ctx* ctx, const ScanJob& j, u32 p, const char* what, void* out_item) {
    char* h = (char*)ctx->pinned;
    TG_CUDA(ctx, cudaMemcpyAsync(h, j.aux, AUX_RECS + p * sizeof(ScanRec), cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const ScanRec* recs = (const ScanRec*)(h + AUX_RECS);
    for (u32 r = 0; r < p; ++r)
        if (recs[r].n >= SCAN_LIMIT)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "%s: worker %u holds %llu items (limit 2^30 - 1)", what, r,
                                (unsigned long long)recs[r].n);
    const u64* res = (const u64*)(h + AUX_CARRY);
    if (j.ib == 16) memcpy(out_item, res, 16);
    else memcpy(out_item, &res[1], 8);
    return TG_OK;
}

// p = 1: the reduce and both fold phases, one host read.  p > 1: this worker's record (written from the host if it is over the
// limit: only its size is read), one ncclAllGather of the records into device memory, the fold, one host read.
int all_reduce_impl(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n_local, const void* initial_item,
                    void* out_item) {
    const int p = ctx->nranks;
    if (p == 1 && n_local >= SCAN_LIMIT)
        return tg_set_error(ctx, TG_ERR_TOO_LARGE, "all_reduce: n_local=%zu (limit 2^30 - 1)", n_local);
    ScanJob j;
    j.op = desc->op; j.ib = desc->item_bytes; j.in = d_in; j.n = n_local; j.rank = (u32)ctx->rank;
    set_initial(&j, initial_item);
    const int init = initial_item ? INIT_GIVEN | (ctx->rank == 0 ? INIT_FOLD : 0) : 0;
    TG_TRY(prepare_aux(ctx, &j, j.n));
    if (p == 1) TG_TRY(action_run(ctx, j, STEP_REDUCE | STEP_TOTAL | STEP_RESULT, init, j.recs(), 1));
    else {
        if (n_local < SCAN_LIMIT) TG_TRY(action_run(ctx, j, STEP_REDUCE | STEP_TOTAL, init, j.my_rec(), p));
        else {
            ScanRec* hr = (ScanRec*)ctx->pinned;
            *hr = ScanRec{ j.n, 0, 0, 0 };
            TG_CUDA(ctx, cudaMemcpyAsync(j.my_rec(), hr, sizeof(ScanRec), cudaMemcpyHostToDevice, ctx->stream));
        }
        TG_NCCL(ctx, ncclAllGather(j.my_rec(), j.recs(), sizeof(ScanRec) / 8, ncclUint64, ctx->comm, ctx->stream));
        TG_TRY(action_run(ctx, j, STEP_RESULT, 0, nullptr, p));
    }
    return action_finish(ctx, j, p, "all_reduce", out_item);
}

}  // namespace

extern "C" {

int tg_prefix_sum(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n_local, const void* initial_item,
                  int inclusive, void** out_dptr, size_t* out_n) {
    if (!ctx || !out_dptr || !out_n || (!d_in && n_local)) return tg_set_error(ctx, TG_ERR_ARG, "prefix_sum: NULL argument");
    TG_TRY(check_desc(ctx, desc));
    TG_TRY(check_ranks(ctx));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return prefix_sum_impl(ctx, desc, d_in, n_local, initial_item, inclusive, out_dptr, out_n);
}

int tg_prefix_sum_file(tg_ctx* ctx, const tg_scan_desc* desc, const tg_merge_input* in, const void* initial_item, int inclusive,
                       size_t* out_items) {
    if (!ctx || !in || !out_items) return tg_set_error(ctx, TG_ERR_ARG, "prefix_sum_file: NULL argument");
    TG_TRY(check_desc(ctx, desc));
    TG_TRY(check_ranks(ctx));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* d_in;
    size_t n;
    TG_TRY(stage_input(ctx, in, desc->item_bytes, &d_in, &n));
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(prefix_sum_impl(ctx, desc, d_in, n, initial_item, inclusive, &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = desc->item_bytes;
    *out_items = n_out;
    return TG_OK;
}

int tg_zip_with_index(tg_ctx* ctx, const void* d_in, size_t n_local, int index_first, void** out_dptr, size_t* out_n) {
    if (!ctx || !out_dptr || !out_n || (!d_in && n_local)) return tg_set_error(ctx, TG_ERR_ARG, "zip_with_index: NULL argument");
    TG_TRY(check_ranks(ctx));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return zip_impl(ctx, d_in, n_local, index_first, out_dptr, out_n);
}

int tg_zip_with_index_file(tg_ctx* ctx, const tg_merge_input* in, int index_first, size_t* out_items) {
    if (!ctx || !in || !out_items) return tg_set_error(ctx, TG_ERR_ARG, "zip_with_index_file: NULL argument");
    TG_TRY(check_ranks(ctx));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* d_in;
    size_t n;
    TG_TRY(stage_input(ctx, in, 8, &d_in, &n));
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(zip_impl(ctx, d_in, n, index_first, &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = 16;
    *out_items = n_out;
    return TG_OK;
}

int tg_scan_local_total(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n, void* out_total_item) {
    if (!ctx || !out_total_item || (!d_in && n)) return tg_set_error(ctx, TG_ERR_ARG, "scan_local_total: NULL argument");
    TG_TRY(check_desc(ctx, desc));
    if (n >= SCAN_LIMIT) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "scan_local_total: n=%zu (limit 2^30 - 1)", n);
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    ScanJob j;
    j.op = desc->op; j.ib = desc->item_bytes; j.in = d_in; j.n = n;
    TG_TRY(prepare(ctx, &j, j.ib));
    TG_TRY(scan_run(ctx, j, STEP_REDUCE | STEP_TOTAL));
    ScanRec* hr = (ScanRec*)ctx->pinned;
    TG_CUDA(ctx, cudaMemcpyAsync(hr, j.my_rec(), sizeof(ScanRec), cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const u64 w[2] = { hr->first, hr->value };
    if (j.ib == 16) memcpy(out_total_item, w, 16);
    else memcpy(out_total_item, &w[1], 8);
    return TG_OK;
}

int tg_prefix_sum_select(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n_local, uint32_t rank, uint32_t p,
                         const void* totals, const void* initial_item, int inclusive, void** out_dptr, size_t* out_n) {
    if (!ctx || !totals || !out_dptr || !out_n || (!d_in && n_local) || p == 0 || p > TG_MAX_RANKS || rank >= p)
        return tg_set_error(ctx, TG_ERR_ARG, "prefix_sum_select: rank=%u p=%u or a NULL argument", rank, p);
    TG_TRY(check_desc(ctx, desc));
    if (n_local >= SCAN_LIMIT) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "prefix_sum_select: n_local=%zu (limit 2^30 - 1)", n_local);
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    ScanJob j;
    j.op = desc->op; j.ib = desc->item_bytes; j.in = d_in; j.n = n_local; j.inclusive = inclusive; j.rank = rank;
    set_initial(&j, initial_item);
    TG_TRY(prepare(ctx, &j, j.ib));
    // the records the all-gather would have delivered
    ScanRec* hr = (ScanRec*)ctx->pinned;
    const u64* t = (const u64*)totals;
    for (uint32_t r = 0; r < p; ++r)
        hr[r] = j.ib == 16 ? ScanRec{ 0, t[2 * r], t[2 * r + 1], 0 } : ScanRec{ 0, 0, t[r], 0 };
    TG_CUDA(ctx, cudaMemcpyAsync(j.recs(), hr, p * sizeof(ScanRec), cudaMemcpyHostToDevice, ctx->stream));
    TG_TRY(scan_run(ctx, j, STEP_REDUCE | STEP_PREFIX | STEP_SCAN));
    *out_dptr = j.out;
    *out_n = n_local;
    return TG_OK;
}

int tg_zip_with_index_select(tg_ctx* ctx, const void* d_in, size_t n_local, uint32_t rank, uint32_t p, const uint64_t* sizes,
                             int index_first, void** out_dptr, size_t* out_n) {
    if (!ctx || !sizes || !out_dptr || !out_n || (!d_in && n_local) || p == 0 || p > TG_MAX_RANKS || rank >= p)
        return tg_set_error(ctx, TG_ERR_ARG, "zip_with_index_select: rank=%u p=%u or a NULL argument", rank, p);
    if (n_local >= SCAN_LIMIT) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "zip_with_index_select: n_local=%zu (limit 2^30 - 1)", n_local);
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    ScanJob j;
    j.ib = 8; j.in = d_in; j.n = n_local;
    TG_TRY(prepare(ctx, &j, 16));
    u64 base = 0;
    for (uint32_t r = 0; r < rank; ++r) base += sizes[r];
    TG_TRY(zip_launch(ctx, d_in, n_local, base, index_first, j.out));
    *out_dptr = j.out;
    *out_n = n_local;
    return TG_OK;
}

int tg_all_reduce(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n_local, const void* initial_item,
                  void* out_item) {
    if (!ctx || !out_item || (!d_in && n_local)) return tg_set_error(ctx, TG_ERR_ARG, "all_reduce: NULL argument");
    TG_TRY(check_action_desc(ctx, desc));
    TG_TRY(check_ranks(ctx));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return all_reduce_impl(ctx, desc, d_in, n_local, initial_item, out_item);
}

int tg_all_reduce_file(tg_ctx* ctx, const tg_scan_desc* desc, const tg_merge_input* in, const void* initial_item, void* out_item) {
    if (!ctx || !in || !out_item) return tg_set_error(ctx, TG_ERR_ARG, "all_reduce_file: NULL argument");
    TG_TRY(check_action_desc(ctx, desc));
    TG_TRY(check_ranks(ctx));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* d_in;
    size_t n;
    TG_TRY(stage_input(ctx, in, desc->item_bytes, &d_in, &n));
    return all_reduce_impl(ctx, desc, d_in, n, initial_item, out_item);
}

int tg_all_reduce_select(tg_ctx* ctx, const tg_scan_desc* desc, const void* const* d_shards, const size_t* n_shards, uint32_t p,
                         const void* initial_item, void* out_item) {
    if (!ctx || !d_shards || !n_shards || !out_item || p == 0 || p > TG_MAX_RANKS)
        return tg_set_error(ctx, TG_ERR_ARG, "all_reduce_select: p=%u or a NULL argument", p);
    TG_TRY(check_action_desc(ctx, desc));
    u64 largest = 0;
    for (uint32_t w = 0; w < p; ++w) {
        if (!d_shards[w] && n_shards[w]) return tg_set_error(ctx, TG_ERR_ARG, "all_reduce_select: shard %u is NULL", w);
        if (n_shards[w] >= SCAN_LIMIT)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "all_reduce_select: shard %u holds %zu items (limit 2^30 - 1)", w, n_shards[w]);
        largest = n_shards[w] > largest ? n_shards[w] : largest;
    }
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    ScanJob j;
    j.op = desc->op; j.ib = desc->item_bytes;
    set_initial(&j, initial_item);
    TG_TRY(prepare_aux(ctx, &j, largest));
    // worker w's record into the slot the all-gather fills
    for (uint32_t w = 0; w < p; ++w) {
        j.in = d_shards[w]; j.n = n_shards[w]; j.rank = w;
        TG_TRY(action_run(ctx, j, STEP_REDUCE | STEP_TOTAL, initial_item ? INIT_GIVEN | (w == 0 ? INIT_FOLD : 0) : 0,
                          j.recs() + w, p));
    }
    TG_TRY(action_run(ctx, j, STEP_RESULT, 0, nullptr, p));
    return action_finish(ctx, j, p, "all_reduce_select", out_item);
}

}  // extern "C"
