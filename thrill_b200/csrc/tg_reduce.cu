// tg_reduce.cu — the hash-aggregate operator of Thrill's ReduceNode (ReduceByKey / ReducePair) on H100s.
//
// Reference path replaced: ReducePrePhase::Insert -> ReduceProbingHashTable::Insert (open addressing,
// linear probing, Key()==0 sentinel in a side slot; core/reduce_probing_hash_table.hpp:190-268), FlushAll
// -> ReducePrePhaseEmitter::Emit into the writer of worker Hash128to64(0,key) % p
// (core/reduce_pre_phase.hpp:57-61, core/reduce_functional.hpp:60-72), the MixStream exchange
// (api/reduce_by_key.hpp:109-114), and ReduceByHashPostPhase (core/reduce_by_hash_post_phase.hpp:44-281).
//
// GPU formulation (same result set; output order is table order = unspecified in the reference too):
//   pre phase   : local aggregation of the worker's records ("partitioned aggregation", below): two stable partition
//                 passes by two bytes of the key hash, then shared-memory probing tables over runs of whole segments
//   partition   : stable partition pass with digit = Hash128to64(0,key) % p              (p > 1 only)
//   exchange    : NCCL Alltoallv of the p contiguous groups                              (p > 1 only)
//   post phase  : the same aggregation over the received partial aggregates             (p > 1 only)
// Inputs below 2^18 records, and the pieces of segments that had to be split, go through an open-addressing table in
// HBM (16-byte slots, atomicCAS on the key, native atomics on the value) + compaction of the used slots.
#include <algorithm>
#include <vector>

#include "tg_partition.cuh"
#include "tg_segmented.cuh"
#include "tg_exchange.cuh"
#include "tg_reduce_ops.cuh"

using namespace tgp;

namespace {

// atomically fold `val` into *slot_val; `claimed` = this thread created the slot (needed for FIRST)
__device__ __forceinline__ void op_apply(int op, u64* slot_val, u64 val, bool claimed) {
    switch (op) {
    case TG_OP_SUM_F64: atomicAdd((double*)slot_val, __longlong_as_double((long long)val)); break;
    case TG_OP_SUM_U64: atomicAdd(slot_val, val); break;
    case TG_OP_MIN_U64: atomicMin(slot_val, val); break;
    case TG_OP_MAX_U64: atomicMax(slot_val, val); break;
    case TG_OP_MIN_F64:
    case TG_OP_MAX_F64: {
        u64 old = *(volatile u64*)slot_val;
        while (true) {
            if (!f64_better(op, val, old)) break;
            u64 prev = atomicCAS(slot_val, old, val);
            if (prev == old) break;
            old = prev;
        }
        break;
    }
    default:      // TG_OP_FIRST: the value that created the slot stays
        if (claimed) atomicExch(slot_val, val);
        break;
    }
}

__device__ __forceinline__ u64 key_hash(u64 key) { return hash128to64_dev(0, key); }

// ---- output reservation shared by the table kernels --------------------------------------------------------------
// append items to the global output: ONE atomic on the global cursor per CTA per call (a cursor bumped per
// warp is a single hot L2 address: ~4M serialized atomics per 1.25e8 records, measured 3-4 ms).  All threads of
// the CTA must call it; NITEMS items per thread; `scratch` = 34 u32 of shared memory.
template <int NITEMS>
__device__ __forceinline__ void emit_block(ulonglong2* __restrict__ out, u64* cursor, const u64 (&key)[NITEMS],
                                           const u64 (&val)[NITEMS], const bool (&has)[NITEMS], u32* scratch) {
    const u32 lane = lane_id(), warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    u32 mine = 0;
#pragma unroll
    for (int i = 0; i < NITEMS; ++i) mine += has[i] ? 1u : 0u;
    // exclusive scan of `mine` inside the warp
    u32 incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        u32 v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) scratch[warp] = incl;
    __syncthreads();
    u64* base_slot = reinterpret_cast<u64*>(scratch + 32);      // 8-byte aligned: scratch is 8-byte aligned
    if (warp == 0) {
        u32 w = lane < nwarps ? scratch[lane] : 0;
        u32 winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            u32 v = __shfl_up_sync(0xffffffffu, winc, o);
            if (lane >= o) winc += v;
        }
        scratch[lane] = winc - w;                                // exclusive offsets of the warps
        u32 total = __shfl_sync(0xffffffffu, winc, 31);
        if (lane == 0) *base_slot = total ? atomicAdd(cursor, (u64)total) : 0ull;
    }
    __syncthreads();
    u64 pos = *base_slot + scratch[warp] + (incl - mine);
#pragma unroll
    for (int i = 0; i < NITEMS; ++i)
        if (has[i]) out[pos++] = make_ulonglong2(key[i], val[i]);
    __syncthreads();                                             // scratch is reused by the next call
}

// ---- post phase: open addressing in HBM ------------------------------------------------------------------------
__global__ void table_init_kernel(ulonglong2* __restrict__ tab, u64 cap, u64 ident) {
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += stride) tab[i] = make_ulonglong2(0, ident);
}

__global__ void __launch_bounds__(512)
aggregate_kernel(const ulonglong2* __restrict__ in, u64 n, int op, ulonglong2* __restrict__ tab, u64 cap,
                 u64* __restrict__ zero_slot) {
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        ulonglong2 kv = in[i];
        if (kv.x == 0) {
            u64 prev = atomicCAS(&zero_slot[0], 0ull, 1ull);
            op_apply(op, &zero_slot[1], kv.y, prev == 0);
            continue;
        }
        u64 slot = __umul64hi(key_hash(kv.x), cap);       // uniform hash -> [0, cap)
        while (true) {
            u64* kp = &tab[slot].x;
            u64 prev = *(volatile u64*)kp;
            if (prev == 0) prev = atomicCAS(kp, 0ull, kv.x);
            if (prev == 0 || prev == kv.x) {
                op_apply(op, &tab[slot].y, kv.y, prev == 0);
                break;
            }
            if (++slot == cap) slot = 0;
        }
    }
}

__global__ void __launch_bounds__(512)
compact_kernel(const ulonglong2* __restrict__ tab, u64 cap, ulonglong2* __restrict__ out, u64* __restrict__ cursor,
               const u64* __restrict__ zero_slot) {
    __shared__ __align__(8) u32 scratch[36];
    constexpr int CI = 8;
    const u64 stride = (u64)gridDim.x * blockDim.x * CI;
    const u64 rounds = (cap + stride - 1) / stride;
    for (u64 r = 0; r < rounds; ++r) {
        u64 key[CI], val[CI];
        bool has[CI];
#pragma unroll
        for (int j = 0; j < CI; ++j) {
            u64 i = r * stride + ((u64)blockIdx.x * CI + j) * blockDim.x + threadIdx.x;
            ulonglong2 e = i < cap ? tab[i] : make_ulonglong2(0, 0);
            key[j] = e.x; val[j] = e.y; has[j] = e.x != 0;
        }
        emit_block<CI>(out, cursor, key, val, has, scratch);
    }
    if (blockIdx.x == 0) {
        u64 key[1] = { 0 }, val[1] = { zero_slot[1] };
        bool has[1] = { threadIdx.x == 0 && zero_slot[0] != 0 };
        emit_block<1>(out, cursor, key, val, has, scratch);
    }
}

struct ReduceScratch {
    u64* cursor;        // [0] output cursor
    u64* zero_slot;     // [0] flag, [1] value
};

int get_scratch(tg_ctx* ctx, int op, ReduceScratch* sc) {
    u64* d;
    TG_TRY(tg_ws_get(ctx, WS_MISC, 1 << 16, (void**)&d));
    sc->cursor = d + 4096;
    sc->zero_slot = d + 4100;
    u64 init[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    init[5] = op_identity(op);        // zero_slot[1]
    u64* h = (u64*)ctx->pinned + 1024;
    memcpy(h, init, sizeof(init));
    TG_CUDA(ctx, cudaMemcpyAsync(sc->cursor, h, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    return TG_OK;
}

int read_cursor(tg_ctx* ctx, const ReduceScratch& sc, u64* out) {
    u64* h = (u64*)ctx->pinned + 2048;
    TG_CUDA(ctx, cudaMemcpyAsync(h, sc.cursor, 8, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *out = h[0];
    return TG_OK;
}

// post phase: m (partial) items -> distinct keys in d_out (capacity m)
int run_aggregate(tg_ctx* ctx, int op, const void* d_in, u64 m, void* d_out, u64* out_distinct) {
    ReduceScratch sc;
    TG_TRY(get_scratch(ctx, op, &sc));
    if (m == 0) { *out_distinct = 0; return TG_OK; }
    u64 cap = m + m / 2 + 64;                     // load factor <= 2/3
    ulonglong2* tab;
    TG_TRY(tg_ws_get(ctx, WS_TABLE, cap * 16, (void**)&tab));
    const u64 ident = op_identity(op);
    if (ident == 0) TG_CUDA(ctx, cudaMemsetAsync(tab, 0, cap * 16, ctx->stream));
    else TG_LAUNCH(ctx, table_init_kernel, ctx->sm_count * 8, 512, 0, tab, cap, ident);
    TG_LAUNCH_T(ctx, TG_K_AGGREGATE, aggregate_kernel, ctx->sm_count * 4, 512, 0, (const ulonglong2*)d_in, m, op, tab, cap, sc.zero_slot);
    TG_LAUNCH_T(ctx, TG_K_COMPACT, compact_kernel, ctx->sm_count * 4, 512, 0, (const ulonglong2*)tab, cap, (ulonglong2*)d_out, sc.cursor, sc.zero_slot);
    return read_cursor(ctx, sc, out_distinct);
}

// ---- partitioned aggregation -------------------------------------------------------------------------------------
// An open-addressing table in HBM makes one random 32-byte sector access (plus an L2 atomic) per record: several times
// more sector traffic than useful data.  Shared memory is the only place where the probing and the
// reduce function are cheap, so the records are first brought into an order in which every CTA sees few distinct keys:
//   two stable partition passes by two 8-bit digits of Hash128to64(0,key) (chunked + segmented, tg_segmented.cuh)
//   -> 65536 segments with disjoint key sets, ~n/65536 records each
//   -> "units" of whole consecutive segments (<= AGG_UNIT records) are reduced in a shared-memory probing table
//      (ReduceProbingHashTable::Insert, core/reduce_probing_hash_table.hpp:190-268, one table per unit) and emitted;
//      a segment longer than a unit (a hot key) is cut into pieces whose partial aggregates are merged afterwards by the
//      HBM table (few items).
// The hash bits used here (24..51) are not the ones that pick the destination worker (hash % p).
constexpr int AGG_THREADS = 256;
constexpr int AGG_RPT = 8;                         // records per thread
constexpr int AGG_UNIT = AGG_THREADS * AGG_RPT;    // 2048 records
constexpr u32 AGG_SLOTS = 2 * AGG_UNIT;            // load factor <= 1/2
constexpr u32 AGG_TAGS = 1024;                     // per-warp tag bytes of the in-warp leader election (agg_units_kernel)
constexpr int AGG_SHIFT1 = 24, AGG_SHIFT2 = 32, AGG_SHIFT_SLOT = 40;
constexpr size_t AGG_MIN_ITEMS = 1u << 18;         // below: the HBM table alone

struct HashLevelDigit {
    int shift;
    static constexpr bool kStoreDigit = true;
    static constexpr bool kHasDrop = false;
    static constexpr int kScratch = 0;
    __device__ __forceinline__ void init() {}
    __device__ __forceinline__ u32 operator()(const ulonglong2& v, u32) const { return (u32)(key_hash(v.x) >> shift) & (RADIX - 1); }
};

constexpr u32 AGG_MAX_UNIT = 1u << 16;             // longer segments are cut (their pieces are merged afterwards)
constexpr u32 AGG_FLUSH_FILL = AGG_SLOTS * 7 / 8;  // the table is emitted early rather than filled beyond this

// One unit = a run of records whose keys occur in no other unit (whole segments), or a piece of a very long segment
// (`partial`: its aggregates are merged afterwards).  The unit is streamed through the table in rounds of AGG_UNIT
// records; if the table would get too full it is emitted as partial aggregates and cleared (FlushPartition,
// reduce_probing_hash_table.hpp:372-377).
template <int OP>
__global__ void __launch_bounds__(AGG_THREADS, 3)
agg_units_kernel(const ulonglong2* __restrict__ in, const uint2* __restrict__ units /* {first record, records | long << 30 | partial << 31} */,
                 u32 max_units, u32* __restrict__ nunits_ptr /* build_units_kernel's counters */, u64 ident, ulonglong2* __restrict__ out, u64* __restrict__ cursor,
                 ulonglong2* __restrict__ dup_out, u64* __restrict__ dup_cursor, u64* __restrict__ zero_slot) {
    extern __shared__ __align__(16) unsigned char agg_smem[];
    u64* const keys = reinterpret_cast<u64*>(agg_smem);
    u64* const vals = keys + AGG_SLOTS;
    u32* const scratch = reinterpret_cast<u32*>(vals + AGG_SLOTS);      // [0..31] warp totals of the emit scan
    u32* const fill = scratch + 32;                                      // used slots of the table
    u64* const out_base = reinterpret_cast<u64*>(scratch + 34);          // reserved output position (8-byte aligned)
    uint4* const next_unit = reinterpret_cast<uint4*>(scratch + 36);     // [2] {unit id, first record, records|flags, -}, double buffered
    unsigned char* const wtag = reinterpret_cast<unsigned char*>(next_unit + 2) + (threadIdx.x >> 5) * AGG_TAGS;   // [warps][AGG_TAGS] leader election
    const u32 lane = lane_id(), warp = threadIdx.x >> 5;
    constexpr int op = OP;             // compile-time: the reduce function's switch folds away
    constexpr int EI = AGG_SLOTS / AGG_THREADS;
    const u32 nbig = nunits_ptr[0], nunits = nbig + nunits_ptr[2];
    u32* const work = nunits_ptr + 1;           // dynamic scheduling: work ids below nbig are the long units
    auto unit_at = [&](u32 w) -> uint2 { return __ldg(&units[w < nbig ? w : max_units - 1 - (w - nbig)]); };

    // Thread 0 fetches the id and the descriptor of a unit into next_unit[b] in three steps spread over the work of the
    // unit before it, so that neither L2 round trip (the work counter, the descriptor) is waited for: fetch_id at the start
    // of an emit, fetch_desc before the rows of the following round, fetch_store before that round's barrier.  Readers read
    // next_unit[b] after that barrier.
    u32 pend_id = 0xffffffffu;
    uint2 pend_desc = make_uint2(0, 0);
    int pend_buf = -1;
    auto fetch_id = [&](int b) { pend_id = atomicAdd(work, 1u); pend_buf = b; };
    auto fetch_desc = [&]() { if (pend_buf >= 0) pend_desc = pend_id < nunits ? unit_at(pend_id) : make_uint2(0, 0); };
    auto fetch_store = [&]() {
        if (pend_buf >= 0) { next_unit[pend_buf] = make_uint4(pend_id, pend_desc.x, pend_desc.y, 0); pend_buf = -1; }
    };
    u64 key[AGG_RPT], val[AGG_RPT];
    bool valid[AGG_RPT];
    auto load_round = [&](u32 first, u32 rl) {
#pragma unroll
        for (int r = 0; r < AGG_RPT; ++r) {
            const u32 i = r * AGG_THREADS + threadIdx.x;
            valid[r] = i < rl;
            ulonglong2 kv = valid[r] ? in[(size_t)first + i] : make_ulonglong2(0, 0);
            key[r] = kv.x; val[r] = kv.y;
        }
    };
    // Emit the table and clear it in the same sweep (FlushPartitionEmit, reduce_probing_hash_table.hpp:443-482).  The
    // number of used slots is known (`fill`): the output range is reserved first and the L2 round trip of that atomic
    // overlaps the sweep.  fetch >= 0: thread 0 also starts fetching the unit after the next one into next_unit[fetch].  All
    // threads call it after a barrier that follows the last insert; it ends with a barrier.
    auto emit_and_clear = [&](bool partial, int fetch) {
        u64 base_reg = 0;
        if (threadIdx.x == 0) {
            const u32 cnt = *(volatile u32*)fill;
            if (cnt) base_reg = atomicAdd(partial ? dup_cursor : cursor, (u64)cnt);
            if (fetch >= 0) fetch_id(fetch);
        }
        u32 mine = 0;
#pragma unroll
        for (int j = 0; j < EI; ++j) mine += keys[j * AGG_THREADS + threadIdx.x] != 0 ? 1u : 0u;
        u32 incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            u32 t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= (u32)o) incl += t;
        }
        if (lane == 31) scratch[warp] = incl;
        if (threadIdx.x == 0) { *out_base = base_reg; *fill = 0; }
        __syncthreads();
        u32 before = incl - mine;
        for (u32 w = 0; w < warp; ++w) before += scratch[w];
        ulonglong2* dst = (partial ? dup_out : out) + *out_base + before;
#pragma unroll
        for (int j = 0; j < EI; ++j) {
            const u32 i = j * AGG_THREADS + threadIdx.x;
            const u64 k = keys[i];
            if (k != 0) {
                *dst++ = make_ulonglong2(k, vals[i]);
                keys[i] = 0;
                vals[i] = ident;
            }
        }
        __syncthreads();
    };

    for (u32 i = threadIdx.x; i < AGG_SLOTS; i += AGG_THREADS) { keys[i] = 0; vals[i] = ident; }
    if (threadIdx.x == 0) { *fill = 0; fetch_id(0); fetch_desc(); fetch_store(); }
    __syncthreads();
    uint4 cur = next_unit[0];
    if (threadIdx.x == 0) fetch_id(1);                         // (stored before, read after the first round's barrier)
    if (cur.x < nunits) load_round(cur.y, (cur.z & 0x3fffffffu) < (u32)AGG_UNIT ? (cur.z & 0x3fffffffu) : (u32)AGG_UNIT);
    int nb = 1;                                                 // buffer that holds the next unit
    while (cur.x < nunits) {
        const u32 start = cur.y, len = cur.z & 0x3fffffffu;
        bool partial = (cur.z >> 31) != 0;
        for (u32 off = 0; off < len; off += AGG_UNIT) {
            if (off) {
                // every thread reads the fill count of the finished rounds between two barriers: a uniform decision
                const u32 filled = *(volatile u32*)fill;
                __syncthreads();
                const u32 rlen = len - off < (u32)AGG_UNIT ? len - off : (u32)AGG_UNIT;
                if (filled + rlen > AGG_FLUSH_FILL) {          // this round could take the table beyond 3/4 full
                    emit_and_clear(true, -1);
                    partial = true;
                }
                load_round(start + off, rlen);
            }
            u32 claims = 0;            // slots this thread claimed in this round (one shared atomic per warp at its end)
            if (threadIdx.x == 0) fetch_desc();
#pragma unroll
            for (int r = 0; r < AGG_RPT; ++r) {
                u64 v = val[r];
                bool mine = valid[r];
                if (!__any_sync(0xffffffffu, mine)) continue;          // (a unit rarely fills all rows: skip the empty ones)
                const u32 home = (u32)(key_hash(key[r]) >> AGG_SHIFT_SLOT) & (AGG_SLOTS - 1);
                // Lanes of the warp that carry the same key are reduced in registers first and one lane touches the table:
                // records of a popular key sit next to each other here (their segment holds little else), and several lanes on
                // one shared-memory CAS are replayed one after the other (measured: 5x the kernel time on Zipf keys).  Equal keys
                // have equal home slots.  A leader per home slot is elected through a small warp-private tag array (every lane
                // stores its lane id at tag[home mod AGG_TAGS], then reads the survivor back): when every lane is its own leader
                // — nearly every row of well-spread keys — nothing else is needed; otherwise the lanes are grouped by their
                // leader's lane id (5 ballots), the leader speaks for the lanes that really have its key, and all groups are
                // reduced at once by pointer jumping along their lanes.
                u32 peers = __ballot_sync(0xffffffffu, mine);
                if (!mine) peers = 0;
                u32 win = lane;
                if (mine) {
                    wtag[home & (AGG_TAGS - 1)] = (unsigned char)lane;
                }
                __syncwarp();
                if (mine) win = wtag[home & (AGG_TAGS - 1)];
                __syncwarp();
                bool leads = mine;
                if (__any_sync(0xffffffffu, win != lane)) {
                    // crowded row: group the lanes by their leader (5 ballots on its lane id)
#pragma unroll
                    for (int bit = 0; bit < 5; ++bit) {
                        const bool one = (win >> bit) & 1u;
                        const u32 m = __ballot_sync(0xffffffffu, one);
                        peers &= one ? m : ~m;
                    }
                    const int leader = mine ? __ffs(peers) - 1 : (int)lane;
                    const u64 kl = __shfl_sync(0xffffffffu, key[r], leader);
                    const bool follows = mine && key[r] == kl;             // (a lane with another key in the same tag slot: on its own)
                    const u32 samekey = __ballot_sync(0xffffffffu, follows);
                    const u32 group = follows ? (peers & samekey) : (mine ? (1u << lane) : 0u);
                    leads = mine && ((group & ((1u << lane) - 1)) == 0);
                    if (__any_sync(0xffffffffu, (group & (group - 1)) != 0)) {
                        const u32 above = group & ~((2u << lane) - 1u);
                        int nxt = above ? __ffs(above) - 1 : -1;
#pragma unroll
                        for (int step = 0; step < 5; ++step) {
                            const int src = nxt < 0 ? (int)lane : nxt;
                            const u64 other = __shfl_sync(0xffffffffu, v, src);
                            const int nn = __shfl_sync(0xffffffffu, nxt, src);
                            if (nxt >= 0) { v = op_combine(op, v, other); nxt = nn; }
                        }
                    }
                }
                if (!leads) continue;
                if (key[r] == 0) {
                    // Key() == 0: reduced in a side slot, never probed (reduce_probing_hash_table.hpp:195-218)
                    u64 prev = atomicCAS(&zero_slot[0], 0ull, 1ull);
                    op_apply(op, &zero_slot[1], v, prev == 0);
                    continue;
                }
                // find (or claim) the key's slot: linear probing from the home slot (:229-248)
                u32 slot = home;
                bool claimed = false;
                while (true) {
                    u64 k = *(volatile u64*)&keys[slot];
                    if (k == 0) {
                        k = atomicCAS(&keys[slot], 0ull, key[r]);
                        claimed = k == 0;
                        if (claimed) { ++claims; break; }
                    }
                    if (k == key[r]) break;
                    slot = (slot + 1) & (AGG_SLOTS - 1);
                }
                // (the compiler's shared-memory 64-bit atomics are the hardware-assisted ATOMS.CAST.SPIN form: a hand-written
                // ld/atom.cas loop in PTX measured 2x slower for the whole kernel)
                op_apply(op, &vals[slot], v, claimed);
            }
            claims = __reduce_add_sync(0xffffffffu, claims);
            if (lane == 0 && claims) atomicAdd(fill, claims);
            if (threadIdx.x == 0) fetch_store();
            __syncthreads();
        }
        // the next unit's descriptor was fetched a whole unit ago: its first records are requested now and arrive while this
        // unit's table is emitted; thread 0 fetches the unit after that during the emit
        const uint4 nxt_unit = next_unit[nb];
        if (nxt_unit.x < nunits)
            load_round(nxt_unit.y, (nxt_unit.z & 0x3fffffffu) < (u32)AGG_UNIT ? (nxt_unit.z & 0x3fffffffu) : (u32)AGG_UNIT);
        emit_and_clear(partial, nb ^ 1);
        cur = nxt_unit;
        nb ^= 1;
    }
}

// ---- popular keys: reduced where the records are first read ------------------------------------------------------------
// Under a skewed key distribution (Zipf s = 1: the 1000 most frequent of 6.7e7 keys carry 40 % of the records) most of the
// traffic of the two partition passes moves records whose keys could have been folded on first sight — what the
// reference's pre-phase table does for every key it can hold (core/reduce_pre_phase.hpp:167).  Here: a sample of the
// input (HOT_SAMPLES records) is counted in a small HBM table, the keys seen at least 4 times (at most HOT_CAP, the most
// frequent first) form the HOT TABLE; the counting read of the first pass (hot_hist_kernel) folds every record of a hot key
// into CTA-private shared-memory accumulators, flushed to the table's accumulators at its end, and the first pass leaves
// those records out (HotLevelDigit: digit RADIX-1 = drop).  The hot keys are appended to the result at the end.  Inputs
// without popular keys (uniform keys over a large universe) find an empty table and skip the probing.
constexpr u32 HOT_SLOTS = 4096, HOT_CAP = 1024, HOT_SAMPLES = 65536, HOT_STAB = 131072, HOT_MIN_COUNT = 4;
constexpr u32 HOT_SUPER = 64;        // the most frequent hot keys get warp-private accumulators in the counting read
constexpr int HOT_SHIFT = 52;
constexpr int HOT_HIST_THREADS = 512;
struct HotTable {
    u64 keys[HOT_SLOTS];            // open addressing, linear probing (load <= 1/4), 0 = empty (the key 0 is never hot)
    u64 hashes[HOT_SLOTS];          // Hash128to64(0, key) of the slot's key: the hash is a bijection of the key (odd multiplications
                                    // and xor-shifts), so probing compares hashes — which every record has computed anyway; 0 = empty
    u64 acc[HOT_SLOTS];
    u32 super_slot[HOT_SUPER];      // slot of super-hot key j
    unsigned char super_idx[HOT_SLOTS];   // 0xff, or j: this slot holds super-hot key j
    u32 nhot, threshold, nsuper, super_threshold;
    u32 sample_distinct, pad0, pad1, pad2;      // distinct keys among the HOT_SAMPLES sampled records
};

// slot of the key with hash h in a hot table (hashes in shared memory), or -1.  Two probes without a branch back (at load
// 1/4 nearly every search ends there, and the lanes of a warp stay together), then the general loop.
__device__ __forceinline__ int hot_find(const u64* __restrict__ hashes, u64 h) {
    u32 slot = (u32)(h >> HOT_SHIFT) & (HOT_SLOTS - 1);
    const u64 k0 = hashes[slot], k1 = hashes[(slot + 1) & (HOT_SLOTS - 1)];
    if (k0 == h) return (int)slot;
    if (k0 == 0) return -1;
    if (k1 == h) return (int)((slot + 1) & (HOT_SLOTS - 1));
    if (k1 == 0) return -1;
    slot = (slot + 2) & (HOT_SLOTS - 1);
    while (true) {
        const u64 k = hashes[slot];
        if (k == h) return (int)slot;
        if (k == 0) return -1;
        slot = (slot + 1) & (HOT_SLOTS - 1);
    }
}

__global__ void hot_sample_kernel(const ulonglong2* __restrict__ in, u64 n, u64* __restrict__ skeys, u32* __restrict__ scnt) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= HOT_SAMPLES) return;
    const u64 key = in[(u64)i * n / HOT_SAMPLES].x;
    if (key == 0) return;
    u32 slot = (u32)(key_hash(key) >> 40) & (HOT_STAB - 1);
    while (true) {
        u64 k = skeys[slot];
        if (k == 0) k = atomicCAS(&skeys[slot], 0ull, key);
        if (k == 0 || k == key) { atomicAdd(&scnt[slot], 1u); return; }
        slot = (slot + 1) & (HOT_STAB - 1);
    }
}

// one CTA: threshold = smallest count >= HOT_MIN_COUNT that leaves at most HOT_CAP keys (HOT_SUPER for the super-hot ones);
// those keys into the hot table
__global__ void __launch_bounds__(1024) hot_select_kernel(const u64* __restrict__ skeys, const u32* __restrict__ scnt, HotTable* ht, u64 ident) {
    __shared__ u32 hist[256];
    __shared__ u32 thr, thr2;
    for (int i = threadIdx.x; i < 256; i += 1024) hist[i] = 0;
    for (u32 s = threadIdx.x; s < HOT_SLOTS; s += 1024) ht->super_idx[s] = 0xff;
    __syncthreads();
    u32 seen = 0;
    for (u32 s = threadIdx.x; s < HOT_STAB; s += 1024) {
        const u32 c = scnt[s];
        seen += c ? 1u : 0u;
        if (c >= HOT_MIN_COUNT) atomicAdd(&hist[c < 255 ? c : 255], 1u);
    }
    seen = __reduce_add_sync(0xffffffffu, seen);
    if ((threadIdx.x & 31) == 0 && seen) atomicAdd(&ht->sample_distinct, seen);
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 acc = 0, t = 256, t2 = 255;        // (t2: if even the keys seen >= 255 times outnumber HOT_SUPER, the first HOT_SUPER of them)
        for (int c = 255; c >= (int)HOT_MIN_COUNT; --c) {
            if (acc + hist[c] > HOT_CAP) break;
            acc += hist[c];
            t = (u32)c;
            if (acc <= HOT_SUPER) t2 = (u32)c;
        }
        thr = t; thr2 = t2;
        ht->threshold = t;
        ht->super_threshold = t2;
    }
    __syncthreads();
    const u32 t = thr, t2 = thr2;
    for (u32 s = threadIdx.x; s < HOT_STAB; s += 1024) {
        const u32 c = scnt[s];
        if (c < t) continue;
        const u64 key = skeys[s];
        u32 slot = (u32)(key_hash(key) >> HOT_SHIFT) & (HOT_SLOTS - 1);
        while (atomicCAS(&ht->keys[slot], 0ull, key) != 0) slot = (slot + 1) & (HOT_SLOTS - 1);
        ht->hashes[slot] = key_hash(key);
        ht->acc[slot] = ident;
        atomicAdd(&ht->nhot, 1u);
        if (c >= t2) {
            const u32 j = atomicAdd(&ht->nsuper, 1u);
            if (j < HOT_SUPER) {
                ht->super_slot[j] = slot;
                ht->super_idx[slot] = (unsigned char)j;
            }
        }
    }
}

// digit of the first pass: values 0..254 of the hash byte (rescaled), or RADIX-1 = a record of a hot key, which the counting
// read has folded: dropped.  The counting read leaves every record's digit in `dig` (one byte per record: 0.8 % of the pass's
// traffic), so the pass itself neither hashes nor probes.
struct HotLevelDigit {
    int shift;
    const HotTable* ht;
    const unsigned char* dig;
    u32 nhot;
    static constexpr bool kStoreDigit = true;
    static constexpr bool kHasDrop = true;
    static constexpr int kScratch = 0;
    __device__ __forceinline__ void init() { nhot = ht->nhot; }
    __device__ __forceinline__ u32 level(u64 h) const { return (((u32)(h >> shift) & (RADIX - 1)) * (RADIX - 1)) >> RADIX_BITS; }
    __device__ __forceinline__ u32 operator()(const ulonglong2&, u32 pos) const { return __ldg(&dig[pos]); }
};

// counting read of the first pass (the chunk_hist_kernel of tg_segmented.cuh) that also folds the records of hot keys:
// chunkcount[chunk][d] for d < RADIX-1 = records of the chunk that the pass will move, [RADIX-1] = records folded here; every
// record's digit goes to dig[].  Hot keys are accumulated in shared memory: the HOT_SUPER most frequent ones in warp-private
// accumulators (a key with 5 % of the records would otherwise serialise the whole CTA on one shared-memory word), the others in
// one table per CTA; everything is flushed to the hot table's accumulators at the end.
constexpr int HOT_HIST_SMEM = HOT_SLOTS * 16 + (HOT_HIST_THREADS / 32) * HOT_SUPER * 8 + HOT_SLOTS + RADIX * 4;
__global__ void __launch_bounds__(HOT_HIST_THREADS) hot_hist_kernel(const ulonglong2* __restrict__ in, u32 n, u32 chunk_items, HotLevelDigit fn,
                                                                    int op, u64 ident, HotTable* ht, u32* __restrict__ chunkcount,
                                                                    unsigned char* __restrict__ dig) {
    constexpr int U = 4, NW = HOT_HIST_THREADS / 32;
    extern __shared__ __align__(16) unsigned char hot_smem[];
    u64* const hhash = reinterpret_cast<u64*>(hot_smem);                    // [HOT_SLOTS]
    u64* const hacc = hhash + HOT_SLOTS;                                    // [HOT_SLOTS]
    u64* const wacc = hacc + HOT_SLOTS;                                     // [NW][HOT_SUPER]
    unsigned char* const hsuper = reinterpret_cast<unsigned char*>(wacc + NW * HOT_SUPER);    // [HOT_SLOTS]
    u32* const sh = reinterpret_cast<u32*>(hsuper + HOT_SLOTS);             // [RADIX]
    fn.init();
    const bool hot = fn.nhot != 0;
    const u32 warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < RADIX; i += blockDim.x) sh[i] = 0;
    if (hot) {
        for (int i = threadIdx.x; i < (int)HOT_SLOTS; i += blockDim.x) { hhash[i] = ht->hashes[i]; hacc[i] = ident; hsuper[i] = ht->super_idx[i]; }
        for (int i = threadIdx.x; i < NW * (int)HOT_SUPER; i += blockDim.x) wacc[i] = ident;
    }
    __syncthreads();
    const u32 lo = blockIdx.x * chunk_items;
    const u32 hi = (n - lo < chunk_items) ? n : lo + chunk_items;
    for (u32 base = lo; base < hi; base += blockDim.x * U) {
        ulonglong2 v[U];
        bool valid[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const u32 i = base + u * blockDim.x + threadIdx.x;
            valid[u] = i < hi;
            if (valid[u]) v[u] = in[i];
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const u32 i = base + u * blockDim.x + threadIdx.x;
            int slot = -1;
            u64 h = 0;
            if (valid[u]) {
                h = key_hash(v[u].x);
                if (hot && v[u].x != 0) slot = hot_find(hhash, h);
            }
            if (!valid[u]) continue;
            const u32 d = slot >= 0 ? (u32)(RADIX - 1) : fn.level(h);
            dig[i] = (unsigned char)d;
            if (slot >= 0) {
                const u32 sj = hsuper[slot];
                op_apply(op, sj != 0xffu ? &wacc[warp * HOT_SUPER + sj] : &hacc[slot], v[u].y, false);
            }
            atomicAdd(&sh[d], 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < RADIX; i += blockDim.x) chunkcount[(size_t)blockIdx.x * RADIX + i] = sh[i];
    if (hot) {
        for (int i = threadIdx.x; i < (int)HOT_SLOTS; i += blockDim.x)
            if (hhash[i] != 0 && hacc[i] != ident) op_apply(op, &ht->acc[i], hacc[i], false);
        if (threadIdx.x < (ht->nsuper < HOT_SUPER ? ht->nsuper : HOT_SUPER)) {
            u64 a = ident;
            for (int w = 0; w < NW; ++w) a = op_combine(op, a, wacc[w * HOT_SUPER + threadIdx.x]);
            if (a != ident) op_apply(op, &ht->acc[ht->super_slot[threadIdx.x]], a, false);
        }
    }
}

// the hot keys and their folded values appended to the output
__global__ void __launch_bounds__(1024) hot_emit_kernel(const HotTable* ht, ulonglong2* __restrict__ out, u64* cursor) {
    for (u32 s = threadIdx.x; s < HOT_SLOTS; s += 1024) {
        const u64 k = ht->keys[s];
        if (k != 0) out[atomicAdd(cursor, 1ull)] = make_ulonglong2(k, ht->acc[s]);
    }
}

// Units straight from the segment tables (the segments lie back to back in table order; segstart[s] = position of segment s):
// 2^group_log2 consecutive segments form a unit; a unit of more than AGG_UNIT records is streamed in rounds with the intra-warp
// reduction switched on (dominated by popular keys), one of more than AGG_MAX_UNIT records is cut into partial pieces.  The
// long units are listed from the front of `units` (they are scheduled first), the short ones from its back; one thread per
// group, positions by atomic counters: ctr[0] = long entries, ctr[1] = work counter of the aggregation, ctr[2] = short entries.
__global__ void __launch_bounds__(256) build_units_kernel(const u32* __restrict__ segcount, const u32* __restrict__ segstart, int nseg,
                                                           int group_log2, uint2* __restrict__ units, u32 max_units, u32* __restrict__ ctr) {
    const int ngroups = nseg >> group_log2, gsz = 1 << group_log2;
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ngroups) return;
    u32 len = 0;
    for (int i = 0; i < gsz; ++i) len += segcount[(size_t)g * gsz + i];
    if (len == 0) return;
    const u32 pos = segstart[(size_t)g * gsz];
    if (len <= (u32)AGG_UNIT) units[max_units - 1 - atomicAdd(&ctr[2], 1u)] = make_uint2(pos, len);
    else if (len <= AGG_MAX_UNIT) units[atomicAdd(&ctr[0], 1u)] = make_uint2(pos, len | 0x40000000u);
    else {
        const u32 pieces = (len + AGG_MAX_UNIT - 1) / AGG_MAX_UNIT;
        u32 at = atomicAdd(&ctr[0], pieces);
        for (u32 off = 0; off < len; off += AGG_MAX_UNIT) {
            const u32 l = len - off < AGG_MAX_UNIT ? len - off : AGG_MAX_UNIT;
            units[at++] = make_uint2(pos + off, l | 0xC0000000u);
        }
    }
}

int run_aggregate(tg_ctx* ctx, int op, const void* d_in, u64 m, void* d_out, u64* out_distinct);

// The aggregation does not depend on the order of the records inside a segment (the reduce functions are commutative and
// associative as far as the reference's own arrival order is concerned): the two hash passes rank with the cheaper unstable
// atomic ranking (TG_REDUCE_UNSTABLE=0 switches it off).
bool reduce_unstable() {
    static int on = -1;
    if (on < 0) { const char* e = getenv("TG_REDUCE_UNSTABLE"); on = e ? atoi(e) : 1; }
    return on != 0;
}

// n records -> distinct keys in d_out (capacity n + 1)
int run_partitioned_aggregate(tg_ctx* ctx, int op, const void* d_in, u64 n, void* d_out, u64* out_distinct) {
    if (n < AGG_MIN_ITEMS || n >= (1u << 30) || getenv("TG_REDUCE_HBM_TABLE")) return run_aggregate(ctx, op, d_in, n, d_out, out_distinct);
    const u64 ident = op_identity(op);
    void *bufA, *bufB;
    TG_TRY(tg_ws_get(ctx, WS_AUX, (n + 2) * 16, &bufA));
    TG_TRY(tg_ws_get(ctx, WS_AUX2, (n + 2) * 16, &bufB));
    // (0) popular keys: sample, hot table (FIRST keeps the value of one arbitrary record: nothing to fold early)
    const bool use_hot = op != TG_OP_FIRST && !getenv("TG_REDUCE_NO_HOT");
    unsigned char* d_hot;
    const size_t hot_fixed = (sizeof(HotTable) + 255) / 256 * 256 + (size_t)HOT_STAB * 12;
    TG_TRY(tg_ws_get(ctx, WS_HOT, hot_fixed + n + 64, (void**)&d_hot));
    HotTable* ht = (HotTable*)d_hot;
    u64* skeys = (u64*)(d_hot + (sizeof(HotTable) + 255) / 256 * 256);
    u32* scnt = (u32*)(skeys + HOT_STAB);
    unsigned char* hot_dig = (unsigned char*)(scnt + HOT_STAB);      // one byte per record: its first-pass digit (RADIX-1: folded)
    TG_CUDA(ctx, cudaMemsetAsync(d_hot, 0, hot_fixed, ctx->stream));
    if (use_hot) {
        TG_LAUNCH(ctx, hot_sample_kernel, HOT_SAMPLES / 256, 256, 0, (const ulonglong2*)d_in, n, skeys, scnt);
        TG_LAUNCH(ctx, hot_select_kernel, 1, 1024, 0, (const u64*)skeys, (const u32*)scnt, ht, ident);
    }
    // (1) first hash digit: chunked pass; its counting read folds the records of the hot keys, the pass drops them
    u32 *d_tot1, *d_gbase1;
    HotLevelDigit fn1 = { AGG_SHIFT1, ht, hot_dig, 0 };
    {
        const ChunkGeom g = chunk_geometry<2>(ctx, n);
        const size_t cw = (size_t)g.nchunks * RADIX;
        u32* tab;
        TG_TRY(tg_ws_get(ctx, WS_SORT_HIST2, (2 * cw + 2 * RADIX + 16) * 4, (void**)&tab));
        u32* chunkcount = tab;
        u32* chunkbase = tab + cw;
        d_tot1 = chunkbase + cw;
        d_gbase1 = d_tot1 + RADIX;
        if (ctx->kernel_cfg.find((const void*)hot_hist_kernel) == ctx->kernel_cfg.end()) {
            TG_CUDA(ctx, cudaFuncSetAttribute(hot_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, HOT_HIST_SMEM));
            ctx->kernel_cfg[(const void*)hot_hist_kernel] = 2;
        }
        TG_LAUNCH_T(ctx, TG_K_PREAGG, hot_hist_kernel, g.nchunks, HOT_HIST_THREADS, HOT_HIST_SMEM, (const ulonglong2*)d_in, (u32)n, g.chunk_items, fn1, op,
                    ident, ht, chunkcount, hot_dig);
        TG_LAUNCH(ctx, chunk_scan_kernel, 1, 4 * RADIX, 0, chunkcount, g.nchunks, d_tot1, d_gbase1, chunkbase);
        std::vector<u32> chunk_size(g.nchunks, g.chunk_items);
        chunk_size[g.nchunks - 1] = (u32)(n - (size_t)(g.nchunks - 1) * g.chunk_items);
        uint4* d_ctiles;
        u32 ctotal = 0;
        TG_TRY(build_tile_list(ctx, g.nchunks, chunk_size.data(), tile_items<2>(), 0, WS_SEG_TILES2, &d_ctiles, &ctotal));
        u32* cstatus;
        TG_TRY(tg_ws_get(ctx, WS_SORT_STATUS, (size_t)ctotal * RADIX * 4, (void**)&cstatus));
        TG_CUDA(ctx, cudaMemsetAsync(cstatus, 0, (size_t)ctotal * RADIX * 4, ctx->stream));
        SegList csl = { d_ctiles, chunkbase, ctotal, nullptr };
        if (reduce_unstable()) TG_TRY((launch_partition_seg_unstable<2, HotLevelDigit>(ctx, d_in, bufA, (u32)n, fn1, cstatus, csl)));
        else TG_TRY((launch_partition_seg<2, HotLevelDigit>(ctx, d_in, bufA, (u32)n, fn1, cstatus, csl)));
    }
    u32* h_tot1 = (u32*)ctx->pinned;
    u32* h_hot = h_tot1 + RADIX;              // nhot, threshold, nsuper, super_threshold, sample_distinct
    TG_CUDA(ctx, cudaMemcpyAsync(h_tot1, d_tot1, RADIX * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(h_hot, &ht->nhot, 32, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const u64 n_hot = h_tot1[RADIX - 1];          // records folded by the counting read; the first pass left them out
    h_tot1[RADIX - 1] = 0;
    const u64 n_rest = n - n_hot;
    ctx->hot_records += n_hot;
    // (2) second hash digit inside the buckets of the first: segmented pass
    uint4* d_tiles;
    u32 total = 0;
    TG_TRY(build_tile_list(ctx, RADIX, h_tot1, tile_items<2>(), 1, WS_SEG_TILES, &d_tiles, &total));
    u32* tables;       // segcount [seg][RADIX] | segbase [seg][RADIX]
    const size_t table_words = (size_t)RADIX * RADIX;
    TG_TRY(tg_ws_get(ctx, WS_SEG_TABLES, 2 * table_words * 4, (void**)&tables));
    u32* segcount = tables;
    u32* segbase = tables + table_words;
    u32* status;
    TG_TRY(tg_ws_get(ctx, WS_SORT_STATUS2, (size_t)total * RADIX * 4, (void**)&status));
    TG_CUDA(ctx, cudaMemsetAsync(segcount, 0, table_words * 4, ctx->stream));
    TG_CUDA(ctx, cudaMemsetAsync(status, 0, (size_t)total * RADIX * 4, ctx->stream));
    SegList sl = { d_tiles, segbase, total, nullptr };
    DigitList<HashLevelDigit> dl;
    dl.n = 1;
    for (int i = 0; i < 4; ++i) dl.fn[i] = HashLevelDigit{ AGG_SHIFT2 };
    TG_TRY((launch_seg_count<2, HashLevelDigit>(ctx, bufA, sl, dl, segcount)));
    TG_LAUNCH(ctx, seg_scan_kernel, dim3(RADIX, 1), RADIX, 0, segcount, d_gbase1, 1, RADIX, segbase);
    if (reduce_unstable()) TG_TRY((launch_partition_seg_unstable<2, HashLevelDigit>(ctx, bufA, bufB, (u32)n, dl.fn[0], status, sl)));
    else TG_TRY((launch_partition_seg<2, HashLevelDigit>(ctx, bufA, bufB, (u32)n, dl.fn[0], status, sl)));
    // (3) units of whole segments, built on the device from the segment table
    int group_log2 = 0;
    while (group_log2 < 16 && ((u64)(n_rest ? n_rest : 1) << (group_log2 + 1)) / (RADIX * RADIX) <= (u64)AGG_UNIT / 2) ++group_log2;
    // Skewed inputs: a segment holds far fewer distinct keys than records, and a unit's cost is dominated by the sweep of its
    // 4096-slot table and its barriers.  The sample tells how many distinct keys to expect (its distinct ratio overestimates the
    // ratio inside a segment by about 2x: keys repeat more over 1167 records than over a 65536-record sample of 1.25e8): group
    // segments until a unit is expected to hold ~1400 distinct keys (measured: groups of 2 segments 1.33 -> 1.16 ms, groups of 4 start
    // to flush partial aggregates) (TG_REDUCE_GROUP=0 switches it off).
    static const bool regroup = !(getenv("TG_REDUCE_GROUP") && atoi(getenv("TG_REDUCE_GROUP")) == 0);
    if (regroup && use_hot && h_hot[4] > 0 && n_rest > 0) {
        const double est_ratio = 0.6 * (double)h_hot[4] / (double)HOT_SAMPLES;
        double target = 1400.0 / (est_ratio > 0.05 ? est_ratio : 0.05);
        if (target > 4.0 * AGG_UNIT) target = 4.0 * AGG_UNIT;
        const double per_seg = (double)n_rest / (double)(RADIX * RADIX);
        while (group_log2 < 6 && per_seg * (double)(2u << group_log2) <= target) ++group_log2;
    }
    const size_t max_units = (table_words >> group_log2) + n / AGG_MAX_UNIT + 2;
    uint2* d_units;
    TG_TRY(tg_ws_get(ctx, WS_SEG_TILES2, max_units * sizeof(uint2) + 64, (void**)&d_units));
    u32* d_nunits = (u32*)(d_units + max_units);
    TG_CUDA(ctx, cudaMemsetAsync(d_nunits, 0, 16, ctx->stream));
    TG_LAUNCH(ctx, build_units_kernel, ((int)(table_words >> group_log2) + 255) / 256, 256, 0, segcount, (const u32*)segbase, RADIX * RADIX, group_log2,
              d_units, (u32)max_units, d_nunits);
    ReduceScratch sc;
    TG_TRY(get_scratch(ctx, op, &sc));
    u64* dup_cursor = sc.cursor + 1;
    ulonglong2* d_dup = (ulonglong2*)bufA;                     // the first pass's output is dead: reuse it for the partial aggregates
    const int agrid = ctx->sm_count * 3;
    constexpr int AGG_SMEM = AGG_SLOTS * 16 + 36 * 4 + 2 * 16 + (AGG_THREADS / 32) * AGG_TAGS + 32;
#define TG_AGG_LAUNCH(OPC)                                                                                              \
    case OPC: {                                                                                                         \
        auto kern = agg_units_kernel<OPC>;                                                                              \
        if (ctx->kernel_cfg.find((const void*)kern) == ctx->kernel_cfg.end()) {                                         \
            TG_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, AGG_SMEM));            \
            ctx->kernel_cfg[(const void*)kern] = 3;                                                                     \
        }                                                                                                               \
        TG_LAUNCH_T(ctx, TG_K_AGGREGATE, kern, agrid, AGG_THREADS, AGG_SMEM, (const ulonglong2*)bufB, (const uint2*)d_units, \
                    (u32)max_units, d_nunits, ident, (ulonglong2*)d_out, sc.cursor, d_dup, dup_cursor, sc.zero_slot);                     \
        break;                                                                                                          \
    }
    switch (op) {
        TG_AGG_LAUNCH(TG_OP_SUM_F64)
        TG_AGG_LAUNCH(TG_OP_SUM_U64)
        TG_AGG_LAUNCH(TG_OP_MIN_U64)
        TG_AGG_LAUNCH(TG_OP_MAX_U64)
        TG_AGG_LAUNCH(TG_OP_MIN_F64)
        TG_AGG_LAUNCH(TG_OP_MAX_F64)
        TG_AGG_LAUNCH(TG_OP_FIRST)
    default: return tg_set_error(ctx, TG_ERR_ARG, "reduce: op %d", op);
    }
#undef TG_AGG_LAUNCH
    u64* h = (u64*)ctx->pinned + 2048;
    TG_CUDA(ctx, cudaMemcpyAsync(h, sc.cursor, 16, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const u64 ndup = h[1];
    if (getenv("TG_DEBUG_REDUCE")) fprintf(stderr, "[tg_reduce] n=%llu hot records=%llu group_log2=%d emitted=%llu partial aggregates=%llu\n", (unsigned long long)n, (unsigned long long)n_hot, group_log2, (unsigned long long)h[0], (unsigned long long)ndup);
    // (4) merge the pieces of the long segments (and emit the zero key) through the HBM table, appended to d_out
    u64 cap = ndup ? ndup + ndup / 2 + 64 : 0;
    ulonglong2* tab = nullptr;
    if (ndup) {
        TG_TRY(tg_ws_get(ctx, WS_TABLE, cap * 16, (void**)&tab));
        TG_LAUNCH(ctx, table_init_kernel, ctx->sm_count * 4, 512, 0, tab, cap, ident);
        TG_LAUNCH_T(ctx, TG_K_AGGREGATE, aggregate_kernel, ctx->sm_count * 4, 512, 0, (const ulonglong2*)d_dup, ndup, op, tab, cap, sc.zero_slot);
    }
    TG_LAUNCH_T(ctx, TG_K_COMPACT, compact_kernel, ndup ? ctx->sm_count * 4 : 1, ndup ? 512 : 32, 0, (const ulonglong2*)tab, cap,
                (ulonglong2*)d_out, sc.cursor, sc.zero_slot);
    if (n_hot) TG_LAUNCH(ctx, hot_emit_kernel, 1, 1024, 0, (const HotTable*)ht, (ulonglong2*)d_out, sc.cursor);
    return read_cursor(ctx, sc, out_distinct);
}

// ---- ReduceToIndex: the dense result (the range partition is RangeDigit, tg_exchange.cuh; out-of-range indices are reported
// by the dense scatter) ----------------------------------------------------------------------------------------------------
__global__ void fill_dense_kernel(ulonglong2* __restrict__ out, u64 n, ulonglong2 neutral) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = neutral;
}

// every index occurs at most once in `in` (it has been aggregated): plain stores
__global__ void scatter_dense_kernel(const ulonglong2* __restrict__ in, u64 m, u64 begin, u64 count, ulonglong2* __restrict__ out,
                                     u32* __restrict__ bad) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const ulonglong2 kv = in[i];
        if (kv.x < begin || kv.x - begin >= count) { *bad = 1; continue; }
        out[kv.x - begin] = kv;
    }
}

int check_kv(tg_ctx* ctx, const tg_kv_desc* d) {
    if (!ctx || !d || d->item_bytes != 16 || d->op > TG_OP_FIRST)
        return tg_set_error(ctx, TG_ERR_ARG, "reduce: only 16-byte (u64 key, 8-byte value) items and TG_OP_* are supported");
    return TG_OK;
}

}  // namespace

extern "C" {

int tg_hash_aggregate(tg_ctx* ctx, const tg_kv_desc* desc, const void* d_in, size_t n, void* d_out, uint64_t* out_distinct) {
    TG_TRY(check_kv(ctx, desc));
    if (n >= (1u << 30)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "hash_aggregate: n=%zu", n);
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    u64 distinct = 0;
    TG_TRY(run_partitioned_aggregate(ctx, (int)desc->op, d_in, n, d_out, &distinct));
    *out_distinct = distinct;
    return TG_OK;
}

int tg_hash_partition(tg_ctx* ctx, const tg_kv_desc* desc, const void* d_in, size_t n, uint32_t p, void* d_out, uint64_t* out_counts) {
    TG_TRY(check_kv(ctx, desc));
    if (p == 0 || p > RADIX) return tg_set_error(ctx, TG_ERR_ARG, "hash_partition: p=%u", p);
    if (n >= (1u << 30)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "hash_partition: n=%zu", n);
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    HashDigit fn = { p };
    u32* d_counts = nullptr;
    TG_TRY((partition_chunked<2, HashDigit>(ctx, d_in, d_out, n, fn, &d_counts, nullptr)));
    u32* hc = (u32*)ctx->pinned;
    TG_CUDA(ctx, cudaMemcpyAsync(hc, d_counts, RADIX * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (uint32_t r = 0; r < p; ++r) out_counts[r] = hc[r];
    return TG_OK;
}

int tg_reduce_by_key(tg_ctx* ctx, const tg_kv_desc* desc, const void* d_in, size_t n_local, void** out_dptr, size_t* out_n) {
    TG_TRY(check_kv(ctx, desc));
    if (!out_dptr || !out_n) return TG_ERR_ARG;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const int op = (int)desc->op;
    const int p = ctx->nranks, me = ctx->rank;
    // n_local >= 2^30: with several workers, the exchange reports it to every rank (a uniform TG_ERR_TOO_LARGE)
    const bool too_large = n_local >= (1u << 30);
    if (too_large && p == 1) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "reduce_by_key: n_local=%zu", n_local);
    // pre phase (ReducePrePhase, StartPreOp..StopPreOp: api/reduce_by_key.hpp:142-168): the local aggregation; with one
    // worker it is already the result
    void* d_pre = nullptr;
    u64 m = n_local;
    if (!too_large) {
        TG_TRY(tg_ws_get(ctx, WS_OUT, (n_local + 2) * 16, &d_pre));
        TG_TRY(run_partitioned_aggregate(ctx, op, d_in, n_local, d_pre, &m));
    }
    if (p == 1) {
        *out_dptr = d_pre;
        *out_n = (size_t)m;
        return TG_OK;
    }
    // partition by Hash128to64(0,key) % p and exchange (replaces the MixStream writers, :109-114): one pass that stores every
    // partial aggregate into its owner's exchange window
    HashDigit fn = { (u32)p };
    XchgResult xr;
    TG_TRY((exchange_scatter<2, HashDigit>(ctx, d_pre, m, fn, &xr)));
    const void* d_post_in = xr.d_recv;
    const u64 m_post = xr.n_recv;
    // post phase (ReduceByHashPostPhase, ProcessChannel + PushData: api/reduce_by_key.hpp:176-211)
    void* d_out;
    TG_TRY(tg_ws_get(ctx, WS_OUT, (m_post + 2) * 16, &d_out));      // (the pre phase's output was consumed by the partition)
    u64 distinct = 0;
    TG_TRY(run_partitioned_aggregate(ctx, op, d_post_in, m_post, d_out, &distinct));
    *out_dptr = d_out;
    *out_n = (size_t)distinct;
    return TG_OK;
}

int tg_reduce_to_index(tg_ctx* ctx, const tg_kv_desc* desc, const void* d_in, size_t n_local, uint64_t result_size,
                       const void* neutral_item16, void** out_dptr, size_t* out_n, uint64_t* out_begin) {
    TG_TRY(check_kv(ctx, desc));
    if (!out_dptr || !out_n || !out_begin || !neutral_item16) return TG_ERR_ARG;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const int op = (int)desc->op;
    const int p = ctx->nranks, me = ctx->rank;
    // the index range of this worker: Range(0, size).Partition(me, p) (common/math.hpp:85-94).  The limit is checked on the
    // largest range of any worker, so that every rank returns the same verdict.
    const u64 begin = range_begin(me, result_size, p), count = range_begin(me + 1, result_size, p) - begin;
    u64 max_count = 0;
    for (int r = 0; r < p; ++r) max_count = std::max(max_count, range_begin(r + 1, result_size, p) - range_begin(r, result_size, p));
    if (max_count >= (1ull << 31)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "reduce_to_index: %llu indices per worker", (unsigned long long)max_count);
    // n_local >= 2^30: with several workers, the exchange reports it to every rank (a uniform TG_ERR_TOO_LARGE)
    const bool too_large = n_local >= (1u << 30);
    if (too_large && p == 1) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "reduce_to_index: n_local=%zu", n_local);
    // pre phase: local aggregation by index
    void* d_pre = nullptr;
    u64 m = n_local;
    if (!too_large) {
        TG_TRY(tg_ws_get(ctx, WS_OUT, (n_local + 2) * 16, &d_pre));
        TG_TRY(run_partitioned_aggregate(ctx, op, d_in, n_local, d_pre, &m));
    }
    const void* d_post = d_pre;
    u64 m_post = m;
    if (p > 1) {
        RangeDigit fn = { result_size, (u32)p };
        XchgResult xr;
        TG_TRY((exchange_scatter<2, RangeDigit>(ctx, d_pre, m, fn, &xr)));
        const ulonglong2* d_recv = (const ulonglong2*)xr.d_recv;
        const u64 n_recv = xr.n_recv;
        // post phase, first half: one item per index
        void* d_agg;
        TG_TRY(tg_ws_get(ctx, WS_OUT, (n_recv + 2) * 16, &d_agg));
        u64 distinct = 0;
        TG_TRY(run_partitioned_aggregate(ctx, op, d_recv, n_recv, d_agg, &distinct));
        d_post = d_agg;
        m_post = distinct;
    }
    // post phase, second half: the dense table filled with the neutral element (reduce_by_index_post_phase.hpp:141-160)
    ulonglong2* d_dense;
    TG_TRY(tg_ws_get(ctx, WS_DENSE, (count + 2) * 16, (void**)&d_dense));
    ulonglong2 neutral;
    memcpy(&neutral, neutral_item16, 16);
    u32* d_bad;
    TG_TRY(tg_ws_get(ctx, WS_MISC, 1 << 16, (void**)&d_bad));
    d_bad += 12288;       // (48 KB into the scratch: behind the cursors of get_scratch at 32 KB)
    TG_CUDA(ctx, cudaMemsetAsync(d_bad, 0, 4, ctx->stream));
    if (count) TG_LAUNCH(ctx, fill_dense_kernel, ctx->sm_count * 8, 256, 0, d_dense, count, neutral);
    if (m_post) TG_LAUNCH(ctx, scatter_dense_kernel, ctx->sm_count * 8, 256, 0, (const ulonglong2*)d_post, m_post, begin, count, d_dense, d_bad);
    u32* hb = (u32*)ctx->pinned;
    TG_CUDA(ctx, cudaMemcpyAsync(hb, d_bad, 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*hb) return tg_set_error(ctx, TG_ERR_ARG, "reduce_to_index: an index is not below result_size=%llu", (unsigned long long)result_size);
    *out_dptr = d_dense;
    *out_n = (size_t)count;
    *out_begin = begin;
    return TG_OK;
}

int tg_reduce_to_index_file(tg_ctx* ctx, const tg_kv_desc* desc, const tg_block* in_blocks, size_t n_in_blocks,
                            uint64_t result_size, const void* neutral_item16, size_t* out_items, uint64_t* out_begin) {
    TG_TRY(check_kv(ctx, desc));
    if (!out_items || !out_begin) return TG_ERR_ARG;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    size_t bytes = 0;
    for (size_t i = 0; i < n_in_blocks; ++i) bytes += in_blocks[i].bytes;
    if (bytes % 16) return tg_set_error(ctx, TG_ERR_ARG, "reduce_to_index_file: %zu bytes is not a multiple of 16", bytes);
    void* d_in;
    TG_TRY(tg_ws_get(ctx, WS_IN, bytes + 16, &d_in));
    TG_TRY(tg_upload_blocks(ctx, d_in, in_blocks, n_in_blocks, nullptr));
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(tg_reduce_to_index(ctx, desc, d_in, bytes / 16, result_size, neutral_item16, &out, &n_out, out_begin));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = 16;
    *out_items = n_out;
    return TG_OK;
}

int tg_reduce_file(tg_ctx* ctx, const tg_kv_desc* desc, const tg_block* in_blocks, size_t n_in_blocks, size_t* out_items) {
    TG_TRY(check_kv(ctx, desc));
    if (!out_items) return TG_ERR_ARG;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    size_t bytes = 0;
    for (size_t i = 0; i < n_in_blocks; ++i) bytes += in_blocks[i].bytes;
    if (bytes % 16) return tg_set_error(ctx, TG_ERR_ARG, "reduce_file: %zu bytes is not a multiple of 16", bytes);
    void* d_in;
    TG_TRY(tg_ws_get(ctx, WS_IN, bytes + 16, &d_in));
    TG_TRY(tg_upload_blocks(ctx, d_in, in_blocks, n_in_blocks, nullptr));
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(tg_reduce_by_key(ctx, desc, d_in, bytes / 16, &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = 16;
    *out_items = n_out;
    return TG_OK;
}

}  // extern "C"
