// tg_sample_sort.cu — the sample-sort operator of Thrill's SortNode on H100s (one GPU per worker).
//
// Reference path replaced (api/sort.hpp): OnPreOpFile sampling (:151-175), MainOp (:537-663) =
// ExPrefixSumTotal (:541), samples -> FindAndSendSplitters (:337-378), TreeBuilder + TransmitItems
// classification with the global-index tie-break (:380-426, :434-535), the MixStream exchange (:615-641),
// ReceiveItems/SortAndWriteToFile local sort (:665-742) and the multiway merge of PushData (:216-271,
// core/multiway_merge.hpp:30-116).
//
// GPU formulations (same output contract, SURVEY.md §8a):
//   default, the reference's own order: classify + stable scatter by the splitters (one chunked partition pass with the
//     (key, global index) tie-break) -> NCCL Alltoallv -> local sort of what was received;
//   TG_SORT_PIPELINE=merge, the "sorted runs" form named in the north star: local sort -> splitter bucket boundaries
//     (classification of a sorted, stable shard is a set of p-1 positions: lower_bound by key + the number of equal-key
//     items with global index <= the splitter's index) -> NCCL Alltoallv of the p contiguous ranges -> k-way merge of the p
//     received runs.
// The stand-alone classify+scatter (tg_classify_scatter, the literal TransmitItems) is exported for parity tests and ncu
// captures; the k-way merge (tg_kway_merge) lives in tg_merge.cu.
#include <algorithm>
#include <cmath>

#include "tg_partition.cuh"
#include "tg_keys.cuh"
#include "tg_segmented.cuh"
#include "tg_exchange.cuh"
#include "tg_records.cuh"

using namespace tgp;

int tg_radix_sort_items(tg_ctx* ctx, const tg_key_desc* desc, void* d_items, void* d_tmp, size_t n, void** result);

namespace {

// ---- classification by splitters: bucket = #splitters (key, idx) < (item key, item global index) ----
// == TransmitItems' tree descent + EqualSampleGreaterIndex walk (api/sort.hpp:478-502); the padded
// sentinel splitters (:607-609) and the writer swap (:460) only exist to make the tree a power of two.
struct SplitterDigit {
    const CanonIdx* spl;
    u32 nspl;
    u64 gbase;
    KeyView kv;
    const u64* gbase_dev;          // if set: the worker's global index base, written by select_splitters_kernel
    const unsigned char* lut;      // if set: [256] lower | [256] upper bucket bounds by the most significant key byte (splitter_lut_kernel)
    const CanonIdx* s_spl;         // shared-memory copies (init_shared)
    const unsigned char* s_lut;
    static constexpr bool kStoreDigit = true;
    static constexpr bool kHasDrop = false;
    static constexpr int kScratch = TG_MAX_RANKS * 24 + 512;
    __device__ __forceinline__ void init() { if (gbase_dev) gbase = *gbase_dev; s_spl = spl; s_lut = nullptr; }
    // the splitters and the lookup table into the CTA's shared memory (called by every thread before the kernel's first barrier)
    __device__ __forceinline__ void init_shared(unsigned char* scratch, int tid, int nthreads) {
        if (!lut) return;
        u64* w = reinterpret_cast<u64*>(scratch);
        const u64* g = reinterpret_cast<const u64*>(spl);
        for (int i = tid; i < (int)nspl * 3; i += nthreads) w[i] = g[i];
        unsigned char* l = scratch + TG_MAX_RANKS * 24;
        for (int i = tid; i < 512; i += nthreads) l[i] = lut[i];
        s_spl = reinterpret_cast<const CanonIdx*>(scratch);
        s_lut = l;
    }
    template <class Item>
    __device__ __forceinline__ u32 operator()(const Item& v, u32 pos) const {
        const bool int_key = kv.kind == TG_KEY_UINT_LE && kv.bytes == 8 && (kv.off & 7) == 0;
        Canon k;
        // (the same canonical key as canon_key: a descending key complements hi as well, as the splitters' keys do)
        if (int_key) { k.hi = kv.desc ? ~0ull : 0ull; k.lo = item_word(v, (int)(kv.off >> 3)); if (kv.desc) k.lo = ~k.lo; }
        else k = canon_key(v, kv);
        u32 lo = 0, hi = nspl;
        if (s_lut) {
            // most keys fall into a byte range that holds no splitter: one shared-memory byte decides
            const u32 tb = canon_top_byte(k, kv);
            lo = s_lut[tb]; hi = s_lut[256 + tb];
            if (lo == hi) return lo;
        }
        const CanonIdx me = { k.hi, k.lo, gbase + pos };
        while (lo < hi) {
            const u32 mid = (lo + hi) >> 1;
            const CanonIdx s = s_spl[mid];
            if (canonidx_less(s, me)) lo = mid + 1; else hi = mid;
        }
        return lo;
    }
};

// lut[b] = number of splitters whose most significant key byte is < b, lut[256 + b] = ... <= b: a key with top byte b belongs to
// a bucket in [lut[b], lut[256 + b]]
__global__ void splitter_lut_kernel(const CanonIdx* __restrict__ spl, u32 nspl, KeyView kv, unsigned char* __restrict__ lut) {
    const u32 b = threadIdx.x;
    u32 lt = 0, le = 0;
    for (u32 j = 0; j < nspl; ++j) {
        const Canon c = { spl[j].hi, spl[j].lo };
        const u32 t = canon_top_byte(c, kv);
        lt += t < b ? 1u : 0u;
        le += t <= b ? 1u : 0u;
    }
    lut[b] = (unsigned char)lt;
    lut[256 + b] = (unsigned char)le;
}

// ---- sampling: gather items at pseudo-random positions (OnPreOpFile, api/sort.hpp:162-170) --------------
template <int WORDS>
__global__ void draw_samples_kernel(const typename ItemT<WORDS>::type* __restrict__ in, u64 n, u64 gbase, u64 seed,
                                    u32 nsamples, KeyView kv, typename ItemT<WORDS>::type* __restrict__ out_items,
                                    CanonIdx* __restrict__ out_canon) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nsamples) return;
    u64 index = splitmix64_dev(seed + i) % n;
    typename ItemT<WORDS>::type v = in[index];
    if (out_items) out_items[i] = v;
    Canon c = canon_key(v, kv);
    CanonIdx ci = { c.hi, c.lo, gbase + index };
    out_canon[i] = ci;
}

// ---- the sample of a worker, drawn and ordered on the device -------------------------------------------------------
// One slot per worker travels in the sample all-gather: a header and up to SAMPLE_MAX (key, LOCAL index) pairs in
// LessSampleIndex order (api/sort.hpp:419-422; the global index base is added by the reader, which knows every n_local).
constexpr u32 SAMPLE_MAX = 3008;             // >= tg_sample_size(2^30 - 1) = 2999
struct SampleHdr { u64 n_local, ns, pad0, pad1; };
constexpr size_t SAMPLE_SLOT_BYTES = sizeof(SampleHdr) + (size_t)SAMPLE_MAX * sizeof(CanonIdx);
constexpr int SRANK_THREADS = 1024;

// every CTA gathers all ns samples (items at positions rng % n: OnPreOpFile's reservoir stand-in, api/sort.hpp:162-170)
// into shared memory; warp w of CTA b ranks samples b*32+w, +grid*32, ... by counting (ties of identical pairs by draw
// order) and stores each at its rank
template <int WORDS>
__global__ void __launch_bounds__(SRANK_THREADS)
sample_rank_kernel(const typename ItemT<WORDS>::type* __restrict__ in, u64 n, u64 seed, u32 ns, KeyView kv,
                   unsigned char* __restrict__ slot) {
    extern __shared__ __align__(16) unsigned char srank_smem[];
    CanonIdx* const sm = reinterpret_cast<CanonIdx*>(srank_smem);
    for (u32 i = threadIdx.x; i < ns; i += SRANK_THREADS) {
        const u64 index = splitmix64_dev(seed + i) % n;
        const Canon c = canon_key(in[index], kv);
        sm[i] = CanonIdx{ c.hi, c.lo, index };
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *reinterpret_cast<SampleHdr*>(slot) = SampleHdr{ n, ns, 0, 0 };
    __syncthreads();
    CanonIdx* const out = reinterpret_cast<CanonIdx*>(slot + sizeof(SampleHdr));
    const u32 lane = lane_id(), warp = threadIdx.x >> 5;
    for (u32 j = blockIdx.x * (SRANK_THREADS / 32) + warp; j < ns; j += gridDim.x * (SRANK_THREADS / 32)) {
        const CanonIdx me = sm[j];
        u32 cnt = 0;
        for (u32 x = lane; x < ns; x += 32) {
            const CanonIdx o = sm[x];
            const bool eq = o.hi == me.hi && o.lo == me.lo && o.idx == me.idx;
            cnt += (canonidx_less(o, me) || (eq && x < j)) ? 1u : 0u;
        }
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (lane == 0) out[cnt] = me;
    }
}

// Splitters from the p gathered, ordered samples (FindAndSendSplitters, api/sort.hpp:337-378): sample (q, j) has global
// rank j + sum over the other workers of the number of their samples below it (global indices of different workers are
// disjoint: no ties across lists); the sample whose rank is floor(i * S / p) is splitter i.  Every rank runs this on the
// same bytes and gets the same splitters.  ctl[0] = this worker's global index base, ctl[1] = total items, ctl[2] = S.
__global__ void __launch_bounds__(256)
select_splitters_kernel(const unsigned char* __restrict__ slots, int p, int me, CanonIdx* __restrict__ spl, u64* __restrict__ ctl) {
    __shared__ u64 prefix[TG_MAX_RANKS + 1];
    __shared__ u32 ns_of[TG_MAX_RANKS];
    __shared__ u64 total_s;
    if (threadIdx.x == 0) {
        u64 acc = 0, S = 0;
        for (int q = 0; q < p; ++q) {
            const SampleHdr h = *reinterpret_cast<const SampleHdr*>(slots + (size_t)q * SAMPLE_SLOT_BYTES);
            prefix[q] = acc;
            acc += h.n_local;
            ns_of[q] = (u32)h.ns;
            S += h.ns;
        }
        prefix[p] = acc;
        total_s = S;
        if (blockIdx.x == 0) { ctl[0] = prefix[me]; ctl[1] = acc; ctl[2] = S; }
    }
    __syncthreads();
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    const int q = (int)(t / SAMPLE_MAX);
    const u32 j = t % SAMPLE_MAX;
    if (q >= p || j >= ns_of[q]) return;
    auto list = [&](int w) { return reinterpret_cast<const CanonIdx*>(slots + (size_t)w * SAMPLE_SLOT_BYTES + sizeof(SampleHdr)); };
    CanonIdx mine = list(q)[j];
    mine.idx += prefix[q];
    u64 rank = j;
    for (int w = 0; w < p; ++w) {
        if (w == q) continue;
        const CanonIdx* l = list(w);
        u32 lo = 0, hi = ns_of[w];
        while (lo < hi) {
            const u32 mid = (lo + hi) >> 1;
            CanonIdx o = l[mid];
            o.idx += prefix[w];
            if (canonidx_less(o, mine)) lo = mid + 1; else hi = mid;
        }
        rank += lo;
    }
    const double splitting_size = (double)total_s / (double)p;
    for (int i = 1; i < p; ++i)
        if ((u64)((double)i * splitting_size) == rank) spl[i - 1] = mine;
}

// ---- number of local items equal to splitter j's key with global index <= splitter j's index ------------
template <int WORDS>
__global__ void tie_count_kernel(const typename ItemT<WORDS>::type* __restrict__ in, u32 n, u64 gbase, KeyView kv,
                                 const CanonIdx* __restrict__ spl, u32 nspl, u32* __restrict__ tie) {
    u32 stride = gridDim.x * blockDim.x;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        Canon k = canon_key(in[i], kv);
        u32 lo = 0, hi = nspl;
        while (lo < hi) {           // first splitter with key >= k
            u32 mid = (lo + hi) >> 1;
            Canon s = { spl[mid].hi, spl[mid].lo };
            if (canon_less(s, k)) lo = mid + 1; else hi = mid;
        }
        while (lo < nspl) {
            CanonIdx s = spl[lo];
            Canon sk = { s.hi, s.lo };
            if (!canon_eq(sk, k)) break;
            if (gbase + i <= s.idx) atomicAdd(&tie[lo], 1u);
            ++lo;
        }
    }
}

// bnd[j] = lower_bound(sorted, splitter j key) + tie[j]   (one thread per splitter)
template <int WORDS>
__global__ void boundaries_kernel(const typename ItemT<WORDS>::type* __restrict__ sorted, u32 n, KeyView kv,
                                  const CanonIdx* __restrict__ spl, u32 nspl, const u32* __restrict__ tie,
                                  u64* __restrict__ bnd) {
    u32 j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nspl) return;
    Canon s = { spl[j].hi, spl[j].lo };
    u32 lo = 0, hi = n;
    while (lo < hi) {
        u32 mid = lo + ((hi - lo) >> 1);
        if (canon_less(canon_key(sorted[mid], kv), s)) lo = mid + 1; else hi = mid;
    }
    bnd[j] = (u64)lo + tie[j];
}

void canon_splitters_from_packed(const tg_key_desc* desc, const KeyView& kv, const void* packed, uint32_t nspl,
                                 std::vector<CanonIdx>* out) {
    const unsigned char* p = (const unsigned char*)packed;
    size_t s = desc->item_bytes + 8;
    out->resize(nspl);
    for (uint32_t j = 0; j < nspl; ++j) {
        Canon c = canon_key_host(p + j * s, kv);
        u64 idx;
        memcpy(&idx, p + j * s + desc->item_bytes, 8);
        (*out)[j] = { c.hi, c.lo, idx };
    }
}

// order of the multi-worker pipeline: classify/scatter -> exchange -> sort (default, the reference's order), or
// TG_SORT_PIPELINE=merge: sort -> boundaries -> exchange -> merge of the received runs
bool classify_first() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("TG_SORT_PIPELINE"); v = (e && !strcmp(e, "merge")) ? 0 : 1; }
    return v != 0;
}

// The sample workspace of p workers (WS_SAMPLES): [p] gathered slots | this worker's slot | splitters | ctl | LUT.
// ctl = { this worker's global index base, total items, total samples, status flags }.
struct SampleWs {
    unsigned char* slots;
    unsigned char* mine;
    CanonIdx* spl;
    u64* ctl;
    unsigned char* lut;
};
int sample_workspace(tg_ctx* ctx, int p, SampleWs* ws) {
    unsigned char* d_samp;
    TG_TRY(tg_ws_get(ctx, WS_SAMPLES, (size_t)(p + 1) * SAMPLE_SLOT_BYTES + 8192, (void**)&d_samp));
    ws->slots = d_samp;
    ws->mine = d_samp + (size_t)p * SAMPLE_SLOT_BYTES;
    ws->spl = reinterpret_cast<CanonIdx*>(ws->mine + SAMPLE_SLOT_BYTES);
    ws->ctl = reinterpret_cast<u64*>(ws->spl + TG_MAX_RANKS);
    ws->lut = reinterpret_cast<unsigned char*>(ws->ctl + 8);
    return TG_OK;
}

// the sample slot of worker `me` at d_slot: its header and its sample in LessSampleIndex order, drawn with the operator's seed.
// `items` are WORDS-word items whose canonical key is described by kv; too_large: an empty slot that reports the limit.
template <int WORDS>
int draw_sample_slot(tg_ctx* ctx, const KeyView& kv, const void* d_items, size_t n_local, uint64_t rng_seed, int me, bool too_large,
                     unsigned char* d_slot) {
    typedef typename ItemT<WORDS>::type Item;
    const u64 n_eff = too_large ? 0 : n_local;
    const u64 want = n_eff ? tg_sample_size(n_eff) : 0;
    const u32 ns = (u32)(want < n_eff ? want : n_eff);
    if (ns) {
        auto kern = sample_rank_kernel<WORDS>;
        const size_t smem = (size_t)ns * sizeof(CanonIdx);
        if (ctx->kernel_cfg.find((const void*)kern) == ctx->kernel_cfg.end()) {
            TG_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(SAMPLE_MAX * sizeof(CanonIdx))));
            ctx->kernel_cfg[(const void*)kern] = 1;
        }
        const int grid = (int)((ns + 31) / 32) < ctx->sm_count ? (int)((ns + 31) / 32) : ctx->sm_count;
        TG_LAUNCH(ctx, kern, grid, SRANK_THREADS, smem, (const Item*)d_items, (u64)n_eff,
                  rng_seed * 0x9E3779B97F4A7C15ull + (u64)me * 0x100000000ull, ns, kv, d_slot);
    }
    else {
        SampleHdr* h = (SampleHdr*)((u64*)ctx->pinned + 2560);        // (pinned scratch, byte offset 20 KB)
        *h = SampleHdr{ 0, 0, too_large ? 1ull : 0ull, 0 };
        TG_CUDA(ctx, cudaMemcpyAsync(d_slot, h, sizeof(SampleHdr), cudaMemcpyHostToDevice, ctx->stream));
    }
    return TG_OK;
}

// splitters, ctl and LUT of worker `me` from the p gathered slots (every worker computes the same splitters; ctl[0] is its own)
int splitters_from_slots(tg_ctx* ctx, const KeyView& kv, const SampleWs& ws, int p, int me) {
    TG_LAUNCH(ctx, select_splitters_kernel, (p * SAMPLE_MAX + 255) / 256, 256, 0, (const unsigned char*)ws.slots, p, me, ws.spl, ws.ctl);
    TG_LAUNCH(ctx, splitter_lut_kernel, 1, 256, 0, (const CanonIdx*)ws.spl, (u32)(p - 1), kv, ws.lut);
    return TG_OK;
}

// samples of every worker and the splitters, all on the device (no host round trip): d_spl[p-1] in LessSampleIndex order,
// d_ctl as in SampleWs.  Collective (one ncclAllGather).
template <int WORDS>
int device_splitters(tg_ctx* ctx, const KeyView& kv, const void* d_items, size_t n_local, uint64_t rng_seed, bool too_large,
                     CanonIdx** d_spl_out, u64** d_ctl_out, unsigned char** d_lut_out = nullptr) {
    const int p = ctx->nranks, me = ctx->rank;
    SampleWs ws;
    TG_TRY(sample_workspace(ctx, p, &ws));
    TG_TRY(draw_sample_slot<WORDS>(ctx, kv, d_items, n_local, rng_seed, me, too_large, ws.mine));
    TG_NCCL(ctx, ncclAllGather(ws.mine, ws.slots, SAMPLE_SLOT_BYTES, ncclUint8, ctx->comm, ctx->stream));
    TG_TRY(splitters_from_slots(ctx, kv, ws, p, me));
    if (d_lut_out) *d_lut_out = ws.lut;
    *d_spl_out = ws.spl;
    *d_ctl_out = ws.ctl;
    return TG_OK;
}

// The merge pipeline's bucket boundaries of one shard: the per-splitter tie counts on the unsorted shard (item i has global
// index gbase + i), the stable local sort (d_in or d_tmp ends up holding it: *d_sorted), then bnd[j] = lower_bound(sorted,
// splitter j's key) + tie[j].  d_tie: 4 KiB of device scratch.
template <int WORDS>
int shard_boundaries(tg_ctx* ctx, const tg_key_desc* desc, const KeyView& kv, void* d_in, void* d_tmp, size_t n_local, u64 gbase,
                     const CanonIdx* d_spl, u32 nspl, u32* d_tie, u64* d_bnd, void** d_sorted) {
    typedef typename ItemT<WORDS>::type Item;
    TG_CUDA(ctx, cudaMemsetAsync(d_tie, 0, 4096, ctx->stream));
    if (n_local && nspl)
        TG_LAUNCH(ctx, tie_count_kernel<WORDS>, ctx->sm_count * 4, 512, 0, (const Item*)d_in, (u32)n_local, gbase, kv, d_spl, nspl, d_tie);
    TG_TRY(tg_radix_sort_items(ctx, desc, d_in, d_tmp, n_local, d_sorted));
    if (nspl) TG_LAUNCH(ctx, boundaries_kernel<WORDS>, (nspl + 63) / 64, 64, 0, (const Item*)*d_sorted, (u32)n_local, kv, d_spl, nspl, d_tie, d_bnd);
    return TG_OK;
}

// an operator input that lies inside the exchange window (the previous collective operator's result) is moved out of
// the peers' way first
int evacuate_window_input(tg_ctx* ctx, void** d_in, size_t bytes) {
    const char* b = (const char*)ctx->xwin.base;
    if (!b || (const char*)*d_in < b || (const char*)*d_in >= b + ctx->xwin.cap) return TG_OK;
    void* d;
    TG_TRY(tg_ws_get(ctx, WS_IN, bytes + 16, &d));
    if (d != *d_in) TG_CUDA(ctx, cudaMemcpyAsync(d, *d_in, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    *d_in = d;
    return TG_OK;
}

template <int WORDS>
int sort_multi_impl(tg_ctx* ctx, const tg_key_desc* desc, const KeyView& kv, void* d_in, size_t n_local,
                    uint64_t rng_seed, void** out_dptr, size_t* out_n) {
    typedef typename ItemT<WORDS>::type Item;
    const int p = ctx->nranks, me = ctx->rank;
    const size_t s = sizeof(Item);
    u64* h = (u64*)ctx->pinned;                      // host scratch (pinned, 1 MiB)
    const bool too_large = n_local >= (1u << 30);    // reported to every rank through the sample header: a uniform error
    TG_TRY(evacuate_window_input(ctx, &d_in, n_local * s));

    // (1) + (2) ExPrefixSumTotal(local_items_) (api/sort.hpp:541), samples (:151-175) and FindAndSendSplitters (:337-378):
    // one all-gather, splitters selected on the device by every rank
    CanonIdx* d_spl;
    u64* d_ctl;
    unsigned char* d_lut;
    TG_TRY((device_splitters<WORDS>(ctx, kv, d_in, n_local, rng_seed, too_large, &d_spl, &d_ctl, &d_lut)));
    const u32 nspl = (u32)(p - 1);
    u64* h_ctl = h + 3072;                           // byte offset 24 KB: ctl[4] | splitters
    CanonIdx* h_spl = (CanonIdx*)(h_ctl + 4);
    TG_CUDA(ctx, cudaMemcpyAsync(h_ctl, d_ctl, 32, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(h_spl, d_spl, nspl * sizeof(CanonIdx), cudaMemcpyDeviceToHost, ctx->stream));

    if (classify_first()) {
        // The reference's own order (api/sort.hpp:615-742): classify + scatter by the splitters (TransmitItems) and the exchange
        // — here one kernel that stores every item into its destination worker's window — then sort what was received.
        SplitterDigit fn = { d_spl, nspl, 0, kv, d_ctl, d_lut, nullptr, nullptr };
        XchgResult xr;
        TG_TRY((exchange_scatter<WORDS, SplitterDigit>(ctx, d_in, too_large ? 0 : n_local, fn, &xr)));      // (synchronises once)
        if (h_ctl[3]) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "sort: a worker holds 2^30 or more items");
        if (h_ctl[1] == 0) { *out_dptr = nullptr; *out_n = 0; return TG_OK; }                           // :550-559
        // ReceiveItems + SortAndWriteToFile (:665-742): the received items arrive grouped by source worker in worker order, each
        // group in input order: the stable local sort leaves equal keys in global input order
        const u64 n_recv = xr.n_recv;
        void* d_tmp2;
        TG_TRY(tg_ws_get(ctx, WS_SORT_TMP, (n_recv + 2) * s, &d_tmp2));
        // this worker's keys lie between its two splitters: the most significant bit in which they can differ
        const int saved_top = ctx->spec_top_bit;
        if (kv.kind == TG_KEY_UINT_LE && !kv.desc && kv.bytes == 8 && (kv.off & 7) == 0 && h_ctl[2] > 0) {
            const u64 lo = me > 0 ? h_spl[me - 1].lo : 0ull, hi = me < p - 1 ? h_spl[me].lo : ~0ull;
            const u64 x = lo ^ hi;
            ctx->spec_top_bit = x ? 64 - __builtin_clzll(x) : 8;
        }
        void* d_res = xr.d_recv;
        const int st = tg_radix_sort_items(ctx, desc, xr.d_recv, d_tmp2, n_recv, &d_res);
        ctx->spec_top_bit = saved_top;
        TG_TRY(st);
        *out_dptr = d_res;
        *out_n = (size_t)n_recv;
        return TG_OK;
    }

    // ---- TG_SORT_PIPELINE=merge (tests only): sorted runs -> boundaries -> NCCL Alltoallv -> merge of the received runs
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h_ctl[3]) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "sort: a worker holds 2^30 or more items");
    if (h_ctl[1] == 0) { *out_dptr = nullptr; *out_n = 0; return TG_OK; }
    const u64 prefix = h_ctl[0];
    u64* d_ctl2;                                     // device control-plane scratch
    TG_TRY(tg_ws_get(ctx, WS_MISC, 1 << 16, (void**)&d_ctl2));
    u64* d_ctl_old = d_ctl; (void)d_ctl_old;
    d_ctl = d_ctl2;
    // (3) per-splitter tie counts on the unsorted shard, (4) local radix sort, (5) bucket boundaries
    u32* d_tie = (u32*)(d_ctl + 1024);
    u64* d_bnd = d_ctl + 2048;
    void* d_tmp;
    TG_TRY(tg_ws_get(ctx, WS_SORT_TMP, n_local * s, &d_tmp));
    void* d_sorted;      // d_in or d_tmp, whichever the last pass wrote
    TG_TRY(shard_boundaries<WORDS>(ctx, desc, kv, d_in, d_tmp, n_local, prefix, d_spl, nspl, d_tie, d_bnd, &d_sorted));
    TG_CUDA(ctx, cudaMemcpyAsync(h, d_bnd, 8 * nspl, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::vector<u64> send_cnt(p), send_off(p + 1, 0);
    {
        u64 prev = 0;
        for (int r = 0; r < p; ++r) {
            u64 b = (r < p - 1) ? h[r] : n_local;
            send_cnt[r] = b - prev;
            prev = b;
            send_off[r + 1] = send_off[r] + send_cnt[r];
        }
    }
    // (6) count exchange: all-gather the p send counts of every rank (what the 29-byte block headers carry
    // in the reference, data/multiplexer_header.hpp:36-72), then the Alltoallv itself
    for (int r = 0; r < p; ++r) h[r] = send_cnt[r];
    TG_CUDA(ctx, cudaMemcpyAsync(d_ctl, h, 8 * p, cudaMemcpyHostToDevice, ctx->stream));
    TG_NCCL(ctx, ncclAllGather(d_ctl, d_ctl + 64, p, ncclUint64, ctx->comm, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(h, d_ctl + 64, 8 * p * p, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::vector<u64> recv_cnt(p), recv_off(p + 1, 0);
    for (int r = 0; r < p; ++r) { recv_cnt[r] = h[(size_t)r * p + me]; recv_off[r + 1] = recv_off[r] + recv_cnt[r]; }
    const u64 n_recv = recv_off[p];
    Item* d_recv;
    TG_TRY(tg_ws_get(ctx, WS_XCHG_RECV, (n_recv + 1) * s, (void**)&d_recv));
    const int xprof_ = ctx->profile ? tg_prof_begin(ctx, TG_K_EXCHANGE) : -1;
        TG_NCCL(ctx, ncclGroupStart());
    for (int r = 0; r < p; ++r) {
        if (send_cnt[r]) TG_NCCL(ctx, ncclSend((const Item*)d_sorted + send_off[r], send_cnt[r] * s, ncclUint8, r, ctx->comm, ctx->stream));
        if (recv_cnt[r]) TG_NCCL(ctx, ncclRecv(d_recv + recv_off[r], recv_cnt[r] * s, ncclUint8, r, ctx->comm, ctx->stream));
    }
    TG_NCCL(ctx, ncclGroupEnd());
        if (xprof_ >= 0) tg_prof_end(ctx, xprof_);

    // (7) merge the p received sorted runs (source order = worker order: stable)
    Item* d_out;
    TG_TRY(tg_ws_get(ctx, WS_OUT, (n_recv + 1) * s, (void**)&d_out));
    void* d_mtmp;        // (WS_SORT_TMP may still be the send buffer of the exchange)
    TG_TRY(tg_ws_get(ctx, WS_AUX2, (n_recv + 1) * s, &d_mtmp));
    const void* runs[TG_MAX_RANKS];
    for (int r = 0; r < p; ++r) runs[r] = d_recv + recv_off[r];
    TG_TRY(merge_runs(ctx, kv, (uint32_t)s, runs, (const uint64_t*)recv_cnt.data(), (uint32_t)p, d_out, d_mtmp));
    *out_dptr = d_out;
    *out_n = (size_t)n_recv;
    return TG_OK;
}


// tg_sort_select: the operator's non-collective steps for p simulated workers on one device.  Worker w's sample slot is drawn
// where the all-gather would put it; then, worker by worker, the splitters with me = w (its global index base lands in ctl[0])
// and the classification pass that the P2P exchange runs, storing locally.
template <int WORDS>
int sort_select_impl(tg_ctx* ctx, const tg_key_desc* desc, const KeyView& kv, const void* const* d_shards, const size_t* n_shards,
                     int p, uint64_t rng_seed, void* out_splitters, void* const* d_out, uint64_t* out_counts, uint64_t* out_merge_bounds) {
    typedef typename ItemT<WORDS>::type Item;
    const size_t s = sizeof(Item);
    const u32 nspl = (u32)(p - 1);
    SampleWs ws;
    TG_TRY(sample_workspace(ctx, p, &ws));
    u64 prefix[TG_MAX_RANKS + 1] = { 0 };
    // (the header of an empty shard is staged in the same pinned words for every worker: the bytes are the same each time)
    for (int w = 0; w < p; ++w) {
        prefix[w + 1] = prefix[w] + n_shards[w];
        TG_TRY(draw_sample_slot<WORDS>(ctx, kv, d_shards[w], n_shards[w], rng_seed, w, false, ws.slots + (size_t)w * SAMPLE_SLOT_BYTES));
    }
    u64* h = (u64*)ctx->pinned + 3072;               // byte offset 24 KB: splitters | counts | bounds | splitter items
    CanonIdx* h_spl = (CanonIdx*)h;
    u32* h_cnt = (u32*)(h_spl + TG_MAX_RANKS);
    u64* h_bnd = (u64*)(h_cnt + RADIX);
    for (int w = 0; w < p; ++w) {
        TG_TRY(splitters_from_slots(ctx, kv, ws, p, w));
        SplitterDigit fn = { ws.spl, nspl, 0, kv, ws.ctl, ws.lut, nullptr, nullptr };
        u32* d_tot = nullptr;
        TG_TRY((partition_chunked<WORDS, SplitterDigit>(ctx, d_shards[w], d_out[w], n_shards[w], fn, &d_tot, nullptr)));
        TG_CUDA(ctx, cudaMemcpyAsync(h_cnt, d_tot, (size_t)p * 4, cudaMemcpyDeviceToHost, ctx->stream));
        if (w == 0) TG_CUDA(ctx, cudaMemcpyAsync(h_spl, ws.spl, nspl * sizeof(CanonIdx), cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int d = 0; d < p; ++d) out_counts[(size_t)w * p + d] = h_cnt[d];
    }
    // the splitters as tg_select_splitters packs them: the sampled item, then its global index (no items: no sample, zeros)
    unsigned char* o = (unsigned char*)out_splitters;
    unsigned char* h_item = (unsigned char*)(h_bnd + TG_MAX_RANKS);
    memset(o, 0, nspl * (s + 8));
    if (prefix[p]) {
        for (u32 j = 0; j < nspl; ++j) {
            const u64 g = h_spl[j].idx;
            memset(h_item + j * s, 0, s);
            if (g >= prefix[p]) continue;                // (not a sampled position: reported as is, with a zero item)
            int w = 0;
            while (g >= prefix[w + 1]) ++w;
            TG_CUDA(ctx, cudaMemcpyAsync(h_item + j * s, (const char*)d_shards[w] + (g - prefix[w]) * s, s, cudaMemcpyDeviceToHost, ctx->stream));
        }
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (u32 j = 0; j < nspl; ++j) {
            memcpy(o + j * (s + 8), h_item + j * s, s);
            memcpy(o + j * (s + 8) + s, &h_spl[j].idx, 8);
        }
    }
    if (!out_merge_bounds) return TG_OK;
    u64* d_misc;
    TG_TRY(tg_ws_get(ctx, WS_MISC, 1 << 16, (void**)&d_misc));
    for (int w = 0; w < p; ++w) {
        const size_t n = n_shards[w];
        void *d_copy, *d_tmp, *d_sorted;
        TG_TRY(tg_ws_get(ctx, WS_AUX, (n + 1) * s, &d_copy));
        TG_TRY(tg_ws_get(ctx, WS_SORT_TMP, (n + 1) * s, &d_tmp));
        if (n) TG_CUDA(ctx, cudaMemcpyAsync(d_copy, d_shards[w], n * s, cudaMemcpyDeviceToDevice, ctx->stream));
        TG_TRY(shard_boundaries<WORDS>(ctx, desc, kv, d_copy, d_tmp, n, prefix[w], ws.spl, nspl, (u32*)(d_misc + 1024), d_misc + 2048, &d_sorted));
        TG_CUDA(ctx, cudaMemcpyAsync(h_bnd, d_misc + 2048, nspl * 8, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (u32 j = 0; j < nspl; ++j) out_merge_bounds[(size_t)w * nspl + j] = h_bnd[j];
    }
    return TG_OK;
}

// ---- records with payload (TeraSort: Record{uint8 key[10]; uint8 value[90]}, examples/terasort/terasort.cpp:31-42) ----
// Sorted through 16-byte tuples {key bytes (<= 12, zero padded), u32 position}: build (reads only the sectors that hold the
// keys, writes 16), radix sort of the tuples (stable, so equal keys keep input order), one gather pass of the s-byte records.
// Records are a multiple of 4 bytes long and 4-byte aligned: every access below is a 32-bit word, consecutive threads on
// consecutive words.

// out record j = rec[tuples[j].position]: a CTA moves REC_BATCH consecutive output records per step, thread t the words
// t, t + 256, ... of the batch (coalesced stores; the words of a record are read by consecutive threads).  Word index lt ->
// (record, word) by a multiply-high with inv = gather_reciprocal(rec_words), or by a division (DIV) where that is 0.
constexpr u32 REC_BATCH = 1024;
template <bool DIV>
__global__ void __launch_bounds__(256) gather_records_kernel(const u32* __restrict__ rec, const ulonglong2* __restrict__ tuples,
                                                              u32 n, u32 rec_words, u32 inv, u32* __restrict__ out) {
    for (u32 r0 = blockIdx.x * REC_BATCH; r0 < n; r0 += gridDim.x * REC_BATCH) {
        const u32 nrec = n - r0 < REC_BATCH ? n - r0 : REC_BATCH, words = nrec * rec_words;
        u32* const o = out + (size_t)r0 * rec_words;
#pragma unroll 4
        for (u32 lt = threadIdx.x; lt < words; lt += 256) {
            const u32 j = DIV ? lt / rec_words : __umulhi(lt, inv), w = lt - j * rec_words;
            const u32 src = (u32)(__ldg(&tuples[r0 + j].y) >> 32);
            o[lt] = rec[(size_t)src * rec_words + w];
        }
    }
}

// The exchange of the records, one launch per destination worker: tuple first + j of the destination-partitioned tuple array
// names the record that becomes record j of this worker's share in the destination's window (mapped peer memory, or the local
// send buffer).  The share is a contiguous stream of cnt * rec_words 32-bit words starting at a 4-byte-aligned address:
// a thread assembles one 16-byte-aligned group of four stream words (they may come from two records) and issues ONE 128-bit
// store — NVLink moves 16-byte stores at about twice the rate of 4-byte ones; only the first and last group of a stream are
// written word by word.
__global__ void __launch_bounds__(256) scatter_records_kernel(const u32* __restrict__ rec, const ulonglong2* __restrict__ ptuples,
                                                               u32 cnt, u32 rec_words, u32 inv, u32* __restrict__ dst) {
    const u32 a = (u32)(((uintptr_t)dst >> 2) & 3u);             // stream word 0 sits at word `a` of its 16-byte group
    uint4* const dst4 = reinterpret_cast<uint4*>(dst - a);
    const u64 nwords = (u64)cnt * rec_words;
    const u64 ngroups = (nwords + a + 3) / 4;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x; c < ngroups; c += stride) {
        u32 val[4];
        bool ok[4];
        // (record, word) of the group's first stream word by one division, of the following ones by stepping
        const u64 wfirst = 4 * c >= a ? 4 * c - a : 0;
        u32 j = (u32)(wfirst / rec_words), ww = (u32)(wfirst - (u64)j * rec_words);
        u32 src = j < cnt ? (u32)(__ldg(&ptuples[j].y) >> 32) : 0u;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const u64 w = 4 * c + k;
            ok[k] = w >= a && w - a < nwords;
            val[k] = 0;
            if (ok[k]) {
                val[k] = rec[(size_t)src * rec_words + ww];
                if (++ww == rec_words) { ww = 0; ++j; src = j < cnt ? (u32)(__ldg(&ptuples[j].y) >> 32) : 0u; }
            }
        }
        if (ok[0] && ok[3]) dst4[c] = make_uint4(val[0], val[1], val[2], val[3]);
        else {
            u32* q = reinterpret_cast<u32*>(dst4 + c);
#pragma unroll
            for (int k = 0; k < 4; ++k) if (ok[k]) q[k] = val[k];
        }
    }
    (void)inv;
}

int sort_records_local(tg_ctx* ctx, const tg_key_desc* desc, const tg_key_desc& tdesc, const void* d_rec, size_t n, void** out_dptr) {
    const u32 rb = desc->item_bytes;
    ulonglong2* d_tup;
    void* d_tmp;
    TG_TRY(tg_ws_get(ctx, WS_AUX, (n + 1) * 16, (void**)&d_tup));
    TG_TRY(tg_ws_get(ctx, WS_SORT_TMP, (n + 1) * 16, &d_tmp));
    unsigned char* d_out;
    TG_TRY(tg_ws_get(ctx, WS_OUT, (n + 1) * (size_t)rb, (void**)&d_out));
    *out_dptr = d_out;
    if (!n) return TG_OK;
    TG_LAUNCH_T(ctx, TG_K_OTHER, make_tuples_kernel, ctx->sm_count * 8, 256, 0, (const u32*)d_rec, (u32)n, rb / 4, desc->key_offset, desc->key_bytes, d_tup);
    void* d_stup;
    TG_TRY(tg_radix_sort_items(ctx, &tdesc, d_tup, d_tmp, n, &d_stup));
    const u32 inv = gather_reciprocal(rb / 4);
    if (inv)
        TG_LAUNCH_T(ctx, TG_K_MERGE, gather_records_kernel<false>, ctx->sm_count * 8, 256, 0, (const u32*)d_rec, (const ulonglong2*)d_stup, (u32)n, rb / 4, inv, (u32*)d_out);
    else
        TG_LAUNCH_T(ctx, TG_K_MERGE, gather_records_kernel<true>, ctx->sm_count * 8, 256, 0, (const u32*)d_rec, (const ulonglong2*)d_stup, (u32)n, rb / 4, 0u, (u32*)d_out);
    return TG_OK;
}

int sort_records_impl(tg_ctx* ctx, const tg_key_desc* desc, void* d_in, size_t n_local, uint64_t rng_seed,
                      void** out_dptr, size_t* out_n) {
    const u32 rb = desc->item_bytes;
    if (rb % 4 || desc->key_kind != TG_KEY_BYTES_BE || desc->key_bytes > 12 || desc->descending)
        return tg_set_error(ctx, TG_ERR_ARG, "sort: records need item_bytes %% 4 == 0 and an ascending byte-string key of <= 12 bytes");
    if (((uintptr_t)d_in) & 3) return tg_set_error(ctx, TG_ERR_ARG, "sort: records must be 4-byte aligned");
    const int p = ctx->nranks, me = ctx->rank;
    tg_key_desc tdesc = { 16, 0, desc->key_bytes, TG_KEY_BYTES_BE, 0, 1 };
    KeyView tkv = { 0, desc->key_bytes, TG_KEY_BYTES_BE, 0 };
    if (p == 1) {
        // workers_algo = 1 (api/sort.hpp:575-579): the local sort is the result
        if (n_local >= (1u << 30)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "sort: n_local=%zu", n_local);
        TG_TRY(sort_records_local(ctx, desc, tdesc, d_in, n_local, out_dptr));
        *out_n = n_local;
        return TG_OK;
    }
    // the reference's order (api/sort.hpp:615-742): classify by the splitters, exchange, sort what was received
    const bool too_large = n_local >= (1u << 30);
    const size_t n = too_large ? 0 : n_local;
    TG_TRY(evacuate_window_input(ctx, &d_in, n * rb));
    ulonglong2 *d_tup, *d_ptup;
    TG_TRY(tg_ws_get(ctx, WS_AUX, (n + 1) * 16, (void**)&d_tup));
    TG_TRY(tg_ws_get(ctx, WS_AUX2, (n + 1) * 16, (void**)&d_ptup));
    if (n) TG_LAUNCH(ctx, make_tuples_kernel, ctx->sm_count * 8, 256, 0, (const u32*)d_in, (u32)n, rb / 4, desc->key_offset, desc->key_bytes, d_tup);
    CanonIdx* d_spl;
    u64* d_ctl;
    unsigned char* d_lut;
    TG_TRY((device_splitters<2>(ctx, tkv, d_tup, n_local, rng_seed, too_large, &d_spl, &d_ctl, &d_lut)));
    u64* h_ctl = (u64*)ctx->pinned + 3072;
    TG_CUDA(ctx, cudaMemcpyAsync(h_ctl, d_ctl, 32, cudaMemcpyDeviceToHost, ctx->stream));
    SplitterDigit fn = { d_spl, (u32)(p - 1), 0, tkv, d_ctl, d_lut, nullptr, nullptr };
    TG_TRY(xwin_negotiate(ctx));
    // destination histogram and the stable partition of the TUPLES by destination (local), then the records follow them
    u32 *d_tot = nullptr, *d_gb = nullptr;
    TG_TRY((partition_chunked<2, SplitterDigit>(ctx, d_tup, d_ptup, n, fn, &d_tot, &d_gb)));
    XchgResult xr;
    u64 need = 0;
    TG_TRY(xchg_counts(ctx, d_tot, (int)rb, &xr, &need));                    // (synchronises; uniform verdicts)
    if (h_ctl[3]) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "sort: a worker holds 2^30 or more records");
    if (h_ctl[1] == 0) { *out_dptr = nullptr; *out_n = 0; return TG_OK; }
    TG_TRY(xwin_ensure(ctx, need));
    TG_TRY(exchange_store_records(ctx, ctx->xwin.mode, false, d_in, rb, d_ptup, n, xchg_matrix(ctx), p, me, ctx->xwin.peer));
    if (ctx->xwin.mode == 1) TG_TRY(xwin_barrier(ctx));
    // ReceiveItems + SortAndWriteToFile (:665-742) on the received records (grouped by source worker in worker order)
    TG_TRY(sort_records_local(ctx, desc, tdesc, ctx->xwin.base, xr.n_recv, out_dptr));
    *out_n = (size_t)xr.n_recv;
    return TG_OK;
}

// ---- tg_exchange_select: one exchange for p simulated workers, one after another on the ctx's stream ----------------------------
// (never two workers' passes at once: the look-back of the partition pass sizes its grid assuming every CTA is resident)

// 8- or 16-byte items by fn; prep(w) sets up worker w's state of fn (the splitters) before each of its steps
template <int WORDS, class DigitFn, class Prep>
int select_items(tg_ctx* ctx, int mode, const void* const* d_shards, const size_t* n_shards, int p, const DigitFn& fn, Prep prep,
                 void* const* d_windows, const size_t* window_bytes, uint64_t* out_counts) {
    u32* h_mat = (u32*)ctx->pinned + 16384;          // (the pinned scratch's count matrix, as in xchg_counts)
    XchgLocal xl;
    for (int w = 0; w < p; ++w) {
        TG_TRY(prep(w));
        TG_TRY((exchange_count<WORDS, DigitFn>(ctx, d_shards[w], n_shards[w], fn, &xl)));
        TG_CUDA(ctx, cudaMemcpyAsync(h_mat + w * p, xl.totals, (size_t)p * 4, cudaMemcpyDeviceToHost, ctx->stream));
    }
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    TG_TRY(select_check(ctx, h_mat, p, 8 * WORDS, d_windows, window_bytes, out_counts));
    if (!d_windows) return TG_OK;
    for (int w = 0; w < p; ++w) {
        // (the count step again: its chunk bases were overwritten by the next worker's)
        TG_TRY(prep(w));
        TG_TRY((exchange_count<WORDS, DigitFn>(ctx, d_shards[w], n_shards[w], fn, &xl)));
        TG_TRY((exchange_store<WORDS, DigitFn>(ctx, mode, true, d_shards[w], xl, fn, h_mat, p, w, d_windows)));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));        // (the pinned staging of the destination pointers is reused)
    }
    return TG_OK;
}

// records: worker w's tuples, sample and splitters as in sort_records_impl, then the records' store step
int select_records(tg_ctx* ctx, int mode, const tg_key_desc* desc, uint64_t rng_seed, const void* const* d_shards, const size_t* n_shards,
                   int p, void* const* d_windows, const size_t* window_bytes, uint64_t* out_counts) {
    const u32 rb = desc->item_bytes;
    const KeyView tkv = { 0, desc->key_bytes, TG_KEY_BYTES_BE, 0 };
    SampleWs ws;
    TG_TRY(sample_workspace(ctx, p, &ws));
    SplitterDigit fn = { ws.spl, (u32)(p - 1), 0, tkv, ws.ctl, ws.lut, nullptr, nullptr };
    auto tuples = [&](int w, ulonglong2** d_tup) -> int {
        TG_TRY(tg_ws_get(ctx, WS_AUX, (n_shards[w] + 1) * 16, (void**)d_tup));
        if (n_shards[w])
            TG_LAUNCH(ctx, make_tuples_kernel, ctx->sm_count * 8, 256, 0, (const u32*)d_shards[w], (u32)n_shards[w], rb / 4,
                      desc->key_offset, desc->key_bytes, *d_tup);
        return TG_OK;
    };
    // worker w's tuples partitioned by destination into WS_AUX2 (*d_tot: its per-destination counts)
    auto partition = [&](int w, ulonglong2** d_ptup, u32** d_tot) -> int {
        ulonglong2* d_tup;
        TG_TRY(tuples(w, &d_tup));
        TG_TRY(splitters_from_slots(ctx, tkv, ws, p, w));
        TG_TRY(tg_ws_get(ctx, WS_AUX2, (n_shards[w] + 1) * 16, (void**)d_ptup));
        return partition_chunked<2, SplitterDigit>(ctx, d_tup, *d_ptup, n_shards[w], fn, d_tot, nullptr);
    };
    for (int w = 0; w < p; ++w) {
        ulonglong2* d_tup;
        TG_TRY(tuples(w, &d_tup));
        TG_TRY(draw_sample_slot<2>(ctx, tkv, d_tup, n_shards[w], rng_seed, w, false, ws.slots + (size_t)w * SAMPLE_SLOT_BYTES));
    }
    u32* h_mat = (u32*)ctx->pinned + 16384;
    ulonglong2* d_ptup;
    u32* d_tot;
    for (int w = 0; w < p; ++w) {
        TG_TRY(partition(w, &d_ptup, &d_tot));
        TG_CUDA(ctx, cudaMemcpyAsync(h_mat + w * p, d_tot, (size_t)p * 4, cudaMemcpyDeviceToHost, ctx->stream));
    }
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    TG_TRY(select_check(ctx, h_mat, p, rb, d_windows, window_bytes, out_counts));
    if (!d_windows) return TG_OK;
    for (int w = 0; w < p; ++w) {
        TG_TRY(partition(w, &d_ptup, &d_tot));
        TG_TRY(exchange_store_records(ctx, mode, true, d_shards[w], rb, d_ptup, n_shards[w], h_mat, p, w, d_windows));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return TG_OK;
}

}  // namespace

namespace tgp {

// Store step of the records' exchange for worker `me` of p: d_ptup = its n tuples partitioned by destination, counts = the p x p
// count matrix (host), windows[d] = worker d's window.  Mode 1 stores the records straight into the windows, mode 0 into the
// local send buffer (WS_XCHG_SEND) followed by the transfers (xchg_transfer).
int exchange_store_records(tg_ctx* ctx, int mode, bool simulated, const void* d_in, u32 rb, const ulonglong2* d_ptup, size_t n,
                           const u32* counts, int p, int me, void* const* windows) {
    u64 before[TG_MAX_RANKS], send_cnt[TG_MAX_RANKS], rc[TG_MAX_RANKS], nr, worst;
    tg_exchange_plan((u32)p, (u32)me, counts, (uint64_t*)send_cnt, (uint64_t*)rc, (uint64_t*)before, (uint64_t*)&nr, (uint64_t*)&worst);
    u64 first[TG_MAX_RANKS + 1];                 // first tuple of every destination in the partitioned tuple array
    first[0] = 0;
    for (int d = 0; d < TG_MAX_RANKS; ++d) first[d + 1] = first[d] + (d < p ? send_cnt[d] : 0);
    const int xprof = ctx->profile ? tg_prof_begin(ctx, TG_K_EXCHANGE) : -1;
    if (mode == 1) {
        // one launch per destination, every worker starting with its right-hand neighbour: at any time each window is written by
        // one peer (all workers going through the destinations in the same order would queue up on one NVLink ingress after the other)
        for (int k = 0; k < p; ++k) {
            const int d = (me + 1 + k) % p;
            u32* dst = (u32*)((char*)windows[d] + before[d] * rb);
            if (send_cnt[d])
                TG_LAUNCH(ctx, scatter_records_kernel, ctx->sm_count * 8, 256, 0, (const u32*)d_in, d_ptup + first[d],
                          (u32)send_cnt[d], rb / 4, 0u, dst);
        }
    }
    else {
        char* d_send;
        TG_TRY(tg_ws_get(ctx, WS_XCHG_SEND, (n + 1) * (size_t)rb, (void**)&d_send));
        for (int d = 0; d < p; ++d)
            if (send_cnt[d])
                TG_LAUNCH(ctx, scatter_records_kernel, ctx->sm_count * 8, 256, 0, (const u32*)d_in, d_ptup + first[d],
                          (u32)send_cnt[d], rb / 4, 0u, (u32*)(d_send + (size_t)first[d] * rb));
        TG_TRY(xchg_transfer(ctx, simulated, d_send, rb, counts, p, me, windows));
    }
    if (xprof >= 0) tg_prof_end(ctx, xprof);
    return TG_OK;
}

// after the count steps: out_counts, the receive limit and the windows' sizes, before any store
int select_check(tg_ctx* ctx, const u32* h_mat, int p, size_t s, void* const* d_windows, const size_t* window_bytes, uint64_t* out_counts) {
    for (int i = 0; i < p * p; ++i) out_counts[i] = h_mat[i];
    u64 sc[TG_MAX_RANKS], rc[TG_MAX_RANKS], before[TG_MAX_RANKS], nr, worst;
    tg_exchange_plan((u32)p, 0, h_mat, (uint64_t*)sc, (uint64_t*)rc, (uint64_t*)before, (uint64_t*)&nr, (uint64_t*)&worst);
    if (worst >= (1u << 30))
        return tg_set_error(ctx, TG_ERR_TOO_LARGE, "exchange_select: a worker would receive %llu items (limit 2^30 - 1)", (unsigned long long)worst);
    if (!d_windows) return TG_OK;
    if (!window_bytes) return tg_set_error(ctx, TG_ERR_ARG, "exchange_select: windows without their sizes");
    for (int d = 0; d < p; ++d) {
        u64 recv = 0;
        for (int src = 0; src < p; ++src) recv += h_mat[src * p + d];
        if ((recv && !d_windows[d]) || window_bytes[d] < recv * s)
            return tg_set_error(ctx, TG_ERR_ARG, "exchange_select: window %d holds %zu bytes, receives %llu", d, window_bytes[d],
                                (unsigned long long)(recv * s));
    }
    return TG_OK;
}

}  // namespace tgp

extern "C" {

// common/reservoir_sampling.hpp:270-275 with desired_imbalance = 0.1 (api/sort.hpp:298); note
// 1/(0.1*0.1) == 99.99999999999999 in double, exactly as the reference computes it
uint64_t tg_sample_size(uint64_t local_items) {
    const double imbalance = 0.1;
    uint64_t s = (uint64_t)(std::log2((double)local_items) * (1.0 / (imbalance * imbalance)));
    return s > 1 ? s : 1;
}

int tg_select_splitters(const tg_key_desc* desc, void* samples, uint64_t nsamples, uint32_t p, void* out_splitters) {
    KeyView kv;
    if (make_key_view(desc, &kv) != TG_OK || !samples || p == 0) return TG_ERR_ARG;
    if (nsamples == 0) return TG_OK;
    const size_t s = desc->item_bytes + 8;
    unsigned char* base = (unsigned char*)samples;
    struct Ent { CanonIdx c; uint64_t src; };
    std::vector<Ent> v(nsamples);
    for (uint64_t i = 0; i < nsamples; ++i) {
        Canon c = canon_key_host(base + i * s, kv);
        u64 idx;
        memcpy(&idx, base + i * s + desc->item_bytes, 8);
        v[i] = { { c.hi, c.lo, idx }, i };
    }
    std::stable_sort(v.begin(), v.end(), [](const Ent& a, const Ent& b) { return canonidx_less(a.c, b.c); });
    std::vector<unsigned char> sorted(nsamples * s);
    for (uint64_t i = 0; i < nsamples; ++i) memcpy(&sorted[i * s], base + v[i].src * s, s);
    memcpy(base, sorted.data(), sorted.size());
    double splitting_size = (double)nsamples / (double)p;
    for (uint32_t i = 1; i < p; ++i)
        memcpy((unsigned char*)out_splitters + (size_t)(i - 1) * s, base + (size_t)((double)i * splitting_size) * s, s);
    return TG_OK;
}

int tg_draw_samples(tg_ctx* ctx, const tg_key_desc* desc, const void* d_items, size_t n, uint64_t global_index_base,
                    uint64_t rng_seed, void* out_samples_host, uint64_t* out_nsamples) {
    KeyView kv;
    if (!ctx || make_key_view(desc, &kv) != TG_OK || (desc->item_bytes != 8 && desc->item_bytes != 16))
        return tg_set_error(ctx, TG_ERR_ARG, "draw_samples: unsupported descriptor");
    uint64_t want = n ? tg_sample_size(n) : 0;
    u32 ns = (u32)(want < n ? want : n);
    *out_nsamples = ns;
    if (!ns) return TG_OK;
    unsigned char* d;
    size_t ib = desc->item_bytes;
    TG_TRY(tg_ws_get(ctx, WS_SAMPLES, (size_t)ns * (ib + sizeof(CanonIdx)) + 4096, (void**)&d));
    CanonIdx* d_canon = (CanonIdx*)d;
    unsigned char* d_items_out = d + (((size_t)ns * sizeof(CanonIdx) + 255) & ~(size_t)255);
    if (ib == 8)
        TG_LAUNCH(ctx, draw_samples_kernel<1>, (ns + 255) / 256, 256, 0, (const u64*)d_items, (u64)n, global_index_base, rng_seed, ns, kv, (u64*)d_items_out, d_canon);
    else
        TG_LAUNCH(ctx, draw_samples_kernel<2>, (ns + 255) / 256, 256, 0, (const ulonglong2*)d_items, (u64)n, global_index_base, rng_seed, ns, kv, (ulonglong2*)d_items_out, d_canon);
    std::vector<CanonIdx> canon(ns);
    std::vector<unsigned char> items((size_t)ns * ib);
    TG_CUDA(ctx, cudaMemcpyAsync(canon.data(), d_canon, ns * sizeof(CanonIdx), cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(items.data(), d_items_out, (size_t)ns * ib, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    unsigned char* o = (unsigned char*)out_samples_host;
    for (u32 i = 0; i < ns; ++i) {
        memcpy(o + (size_t)i * (ib + 8), &items[(size_t)i * ib], ib);
        memcpy(o + (size_t)i * (ib + 8) + ib, &canon[i].idx, 8);
    }
    return TG_OK;
}

int tg_classify_scatter(tg_ctx* ctx, const tg_key_desc* desc, const void* d_in, size_t n, uint64_t global_index_base,
                        const void* splitters_host, uint32_t p, void* d_out, uint64_t* out_counts) {
    KeyView kv;
    if (!ctx || make_key_view(desc, &kv) != TG_OK || (desc->item_bytes != 8 && desc->item_bytes != 16) || p == 0 || p > RADIX)
        return tg_set_error(ctx, TG_ERR_ARG, "classify_scatter: unsupported descriptor or p");
    if (n >= (1u << 30)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "classify_scatter: n=%zu", n);
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<CanonIdx> spl;
    canon_splitters_from_packed(desc, kv, splitters_host, p - 1, &spl);
    CanonIdx* d_spl;
    TG_TRY(tg_ws_get(ctx, WS_SAMPLES, (size_t)p * sizeof(CanonIdx) + 256, (void**)&d_spl));
    if (p > 1) TG_CUDA(ctx, cudaMemcpyAsync(d_spl, spl.data(), (p - 1) * sizeof(CanonIdx), cudaMemcpyHostToDevice, ctx->stream));
    SplitterDigit fn = { d_spl, p - 1, global_index_base, kv, nullptr, nullptr, nullptr, nullptr };
    u32* d_counts = nullptr;
    if (desc->item_bytes == 8) TG_TRY((partition_chunked<1, SplitterDigit>(ctx, d_in, d_out, n, fn, &d_counts, nullptr)));
    else TG_TRY((partition_chunked<2, SplitterDigit>(ctx, d_in, d_out, n, fn, &d_counts, nullptr)));
    u32* hc = (u32*)ctx->pinned;
    TG_CUDA(ctx, cudaMemcpyAsync(hc, d_counts, RADIX * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (uint32_t r = 0; r < p; ++r) out_counts[r] = hc[r];
    return TG_OK;
}

int tg_sort_select(tg_ctx* ctx, const tg_key_desc* desc, const void* const* d_shards, const size_t* n_shards, uint32_t p,
                   uint64_t rng_seed, void* out_splitters, void* const* d_out, uint64_t* out_counts, uint64_t* out_merge_bounds) {
    KeyView kv;
    if (!ctx || make_key_view(desc, &kv) != TG_OK || (desc->item_bytes != 8 && desc->item_bytes != 16))
        return tg_set_error(ctx, TG_ERR_ARG, "sort_select: unsupported descriptor (8- or 16-byte items)");
    if (p < 2 || p > TG_MAX_RANKS || !d_shards || !n_shards || !out_splitters || !d_out || !out_counts)
        return tg_set_error(ctx, TG_ERR_ARG, "sort_select: p=%u or a NULL argument", p);
    for (uint32_t w = 0; w < p; ++w)
        if (n_shards[w] && (!d_shards[w] || !d_out[w])) return tg_set_error(ctx, TG_ERR_ARG, "sort_select: shard %u is NULL", w);
    for (uint32_t w = 0; w < p; ++w)
        if (n_shards[w] >= (1u << 30)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "sort_select: shard %u has %zu items", w, n_shards[w]);
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return desc->item_bytes == 8
               ? sort_select_impl<1>(ctx, desc, kv, d_shards, n_shards, (int)p, rng_seed, out_splitters, d_out, out_counts, out_merge_bounds)
               : sort_select_impl<2>(ctx, desc, kv, d_shards, n_shards, (int)p, rng_seed, out_splitters, d_out, out_counts, out_merge_bounds);
}

int tg_exchange_select(tg_ctx* ctx, uint32_t route, uint32_t mode, const tg_key_desc* desc, uint64_t rng_seed, uint64_t result_size,
                       const void* const* d_shards, const size_t* n_shards, uint32_t p, void* const* d_windows,
                       const size_t* window_bytes, uint64_t* out_counts) {
    if (!ctx || p < 2 || p > TG_MAX_RANKS || !d_shards || !n_shards || !out_counts)
        return tg_set_error(ctx, TG_ERR_ARG, "exchange_select: p=%u or a NULL argument", p);
    if (route > TG_ROUTE_SPLITTERS || mode > 1) return tg_set_error(ctx, TG_ERR_ARG, "exchange_select: route %u, mode %u", route, mode);
    for (uint32_t w = 0; w < p; ++w)
        if (n_shards[w] && !d_shards[w]) return tg_set_error(ctx, TG_ERR_ARG, "exchange_select: shard %u is NULL", w);
    KeyView kv = {};
    bool records = false;
    if (route == TG_ROUTE_SPLITTERS) {
        if (make_key_view(desc, &kv) != TG_OK) return tg_set_error(ctx, TG_ERR_ARG, "exchange_select: unsupported descriptor");
        records = desc->item_bytes != 8 && desc->item_bytes != 16;
        if (records && (desc->item_bytes % 4 || desc->key_kind != TG_KEY_BYTES_BE || desc->key_bytes > 12 || desc->descending))
            return tg_set_error(ctx, TG_ERR_ARG, "exchange_select: records need item_bytes %% 4 == 0 and an ascending byte-string key of <= 12 bytes");
        for (uint32_t w = 0; w < p && records; ++w) {
            if (((uintptr_t)d_shards[w]) & 3) return tg_set_error(ctx, TG_ERR_ARG, "exchange_select: records must be 4-byte aligned");
            if (n_shards[w] >= (1u << 30)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "exchange_select: shard %u has %zu records", w, n_shards[w]);
        }
    }
    if (route == TG_ROUTE_RANGE && result_size && result_size - 1 > ~0ull / p)
        return tg_set_error(ctx, TG_ERR_ARG, "exchange_select: k * p overflows for result_size=%llu", (unsigned long long)result_size);
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const int P = (int)p, M = (int)mode;
    auto none = [](int) { return TG_OK; };
    switch (route) {
    case TG_ROUTE_HASH:
        return select_items<2>(ctx, M, d_shards, n_shards, P, HashDigit{ p }, none, d_windows, window_bytes, out_counts);
    case TG_ROUTE_MOD:
        return select_items<2>(ctx, M, d_shards, n_shards, P, ModDigit::make(p), none, d_windows, window_bytes, out_counts);
    case TG_ROUTE_RANGE:
        return select_items<2>(ctx, M, d_shards, n_shards, P, RangeDigit{ result_size, p }, none, d_windows, window_bytes, out_counts);
    default:
        break;
    }
    if (records) return select_records(ctx, M, desc, rng_seed, d_shards, n_shards, P, d_windows, window_bytes, out_counts);
    // the sample slots of every worker where the all-gather puts them, then worker w's splitters before each of its steps
    SampleWs ws;
    TG_TRY(sample_workspace(ctx, P, &ws));
    for (int w = 0; w < P; ++w) {
        const bool too_large = n_shards[w] >= (1u << 30);
        if (desc->item_bytes == 8) TG_TRY(draw_sample_slot<1>(ctx, kv, d_shards[w], n_shards[w], rng_seed, w, too_large, ws.slots + (size_t)w * SAMPLE_SLOT_BYTES));
        else TG_TRY(draw_sample_slot<2>(ctx, kv, d_shards[w], n_shards[w], rng_seed, w, too_large, ws.slots + (size_t)w * SAMPLE_SLOT_BYTES));
    }
    const SplitterDigit fn = { ws.spl, p - 1, 0, kv, ws.ctl, ws.lut, nullptr, nullptr };
    auto prep = [&](int w) { return splitters_from_slots(ctx, kv, ws, P, w); };
    return desc->item_bytes == 8 ? select_items<1>(ctx, M, d_shards, n_shards, P, fn, prep, d_windows, window_bytes, out_counts)
                                 : select_items<2>(ctx, M, d_shards, n_shards, P, fn, prep, d_windows, window_bytes, out_counts);
}

int tg_sort(tg_ctx* ctx, const tg_key_desc* desc, void* d_in, size_t n_local, uint64_t rng_seed, void** out_dptr, size_t* out_n) {
    KeyView kv;
    if (!ctx || !out_dptr || !out_n || make_key_view(desc, &kv) != TG_OK)
        return tg_set_error(ctx, TG_ERR_ARG, "sort: unsupported descriptor");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (desc->item_bytes != 8 && desc->item_bytes != 16)
        return sort_records_impl(ctx, desc, d_in, n_local, rng_seed, out_dptr, out_n);
    if (ctx->nranks == 1) {
        // workers_algo = 1: zero splitters, everything lands in bucket 0 (api/sort.hpp:575-579): local sort only
        void* d_tmp;
        TG_TRY(tg_ws_get(ctx, WS_SORT_TMP, n_local * desc->item_bytes, &d_tmp));
        void* d_sorted;
        TG_TRY(tg_radix_sort_items(ctx, desc, d_in, d_tmp, n_local, &d_sorted));
        *out_dptr = d_sorted;        // d_in or the ctx-owned sort buffer
        *out_n = n_local;
        return TG_OK;
    }
    if (ctx->nranks > 16) return tg_set_error(ctx, TG_ERR_ARG, "sort: at most 16 ranks");
    return desc->item_bytes == 8 ? sort_multi_impl<1>(ctx, desc, kv, d_in, n_local, rng_seed, out_dptr, out_n)
                                 : sort_multi_impl<2>(ctx, desc, kv, d_in, n_local, rng_seed, out_dptr, out_n);
}

int tg_sort_file(tg_ctx* ctx, const tg_key_desc* desc, const tg_block* in_blocks, size_t n_in_blocks, uint64_t rng_seed,
                 size_t* out_items) {
    if (!ctx || !desc || !out_items) return TG_ERR_ARG;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    size_t bytes = 0;
    for (size_t i = 0; i < n_in_blocks; ++i) bytes += in_blocks[i].bytes;
    if (bytes % desc->item_bytes) return tg_set_error(ctx, TG_ERR_ARG, "sort_file: %zu bytes is not a multiple of the item size", bytes);
    void* d_in;
    TG_TRY(tg_ws_get(ctx, WS_IN, bytes + 16, &d_in));
    TG_TRY(tg_upload_blocks(ctx, d_in, in_blocks, n_in_blocks, nullptr));
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(tg_sort(ctx, desc, d_in, bytes / desc->item_bytes, rng_seed, &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = desc->item_bytes;
    *out_items = n_out;
    return TG_OK;
}

int tg_fetch_output(tg_ctx* ctx, const tg_block_mut* out_blocks, size_t n_out_blocks) {
    if (!ctx) return TG_ERR_ARG;
    size_t bytes = 0;
    for (size_t i = 0; i < n_out_blocks; ++i) bytes += out_blocks[i].bytes;
    if (bytes != ctx->out_items * ctx->out_item_bytes)
        return tg_set_error(ctx, TG_ERR_ARG, "fetch_output: blocks hold %zu bytes, result has %zu", bytes, ctx->out_items * ctx->out_item_bytes);
    if (bytes) TG_TRY(tg_download_blocks(ctx, ctx->out_ptr, out_blocks, n_out_blocks));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->out_ptr = nullptr; ctx->out_items = 0;
    return TG_OK;
}

}  // extern "C"
