// tg_merge.cu — the merge of sorted runs on H100s: the k-way merge behind Sort's TG_SORT_PIPELINE=merge and tg_kway_merge,
// and the Merge operator (DIA::Merge / api::Merge, api/merge.hpp:75-721) of k globally sorted DIAs.
//
// Merge operator, p workers (DESIGN.md §6):
//   1. all-gather of every worker's k shard sizes: global totals, targets t_d = ceil(d * N / p), the size verdict
//   2. exact multi-sequence selection on the device: K_d = key of the item at merged rank t_d, found one key byte per round
//      (most significant first): each round counts, for the 255 candidate values of the byte, the items below the candidate
//      in every local run (binary searches), sums the counts over the workers (one ncclAllReduce) and keeps the largest
//      candidate whose count is <= t_d.  key_bytes rounds (<= 8 for 8-byte keys, <= 16 for 16-byte byte keys), no host sync.
//   3. per run, the items below K_d and equal to K_d; one all-gather gives every worker the whole matrix (one host sync)
//   4. tg_merge_plan (host): the first position of every run that goes to worker d, equal keys assigned in (input, worker)
//      order, so that the merged order is (key, input index, global position within the input)
//   5. exchange of the pieces into the receivers' windows, input-major (input j's pieces of workers 0..p-1 back to back form
//      one sorted run), and the local merge of the k runs.
// The local merge is a tree of stable 2-way merge-path passes: ceil(log2 k) passes, ties to the lower run index.
#include <algorithm>

#include "tg_keys.cuh"
#include "tg_exchange.cuh"

using namespace tgp;

namespace {

// ---- 2-way merge (merge path), stable: ties take from A (the run with the lower index) --------------------
constexpr int MG_THREADS = 256;
template <int WORDS> struct MergeCfg { static constexpr int VT = 16 / WORDS; static constexpr int TILE = MG_THREADS * VT; };

// split[t] = number of A items among the first min(t * TILE, na + nb) outputs, t = 0..ntiles.  On sorted runs the splits
// partition A and B; on unsorted ones they may not, and *bad is set: the merge then concatenates A and B instead, so that
// its output is still a permutation of its input.
template <int WORDS>
__global__ void merge_splits_kernel(const typename ItemT<WORDS>::type* __restrict__ A, u32 na,
                                    const typename ItemT<WORDS>::type* __restrict__ B, u32 nb, u32 ntiles,
                                    u32* __restrict__ split, u32* __restrict__ bad, KeyView kv) {
    constexpr u32 TILE = MergeCfg<WORDS>::TILE;
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t > ntiles) return;
    const u32 total = na + nb;
    const u32 o0 = t * TILE < total ? t * TILE : total;
    const u32 a0 = merge_path_search(A, na, B, nb, o0, kv);
    split[t] = a0;
    if (t < ntiles) {
        const u32 o1 = o0 + TILE < total ? o0 + TILE : total;
        const u32 a1 = merge_path_search(A, na, B, nb, o1, kv);
        if (a1 < a0 || o1 - a1 < o0 - a0) atomicOr(bad, 1u);
    }
}

template <int WORDS>
__global__ void __launch_bounds__(MG_THREADS)
merge2_kernel(const typename ItemT<WORDS>::type* __restrict__ A, u32 na, const typename ItemT<WORDS>::type* __restrict__ B,
              u32 nb, const u32* __restrict__ split, const u32* __restrict__ bad, typename ItemT<WORDS>::type* __restrict__ out,
              KeyView kv) {
    typedef typename ItemT<WORDS>::type Item;
    constexpr int VT = MergeCfg<WORDS>::VT, TILE = MergeCfg<WORDS>::TILE;
    __shared__ Item sm[TILE + 1];
    __shared__ u32 tsplit[MG_THREADS + 1];
    const u32 total = na + nb;
    const u32 o0 = blockIdx.x * TILE;
    const u32 o1 = o0 + TILE < total ? o0 + TILE : total;
    const bool cat = *bad != 0;
    const u32 a0 = cat ? (o0 < na ? o0 : na) : split[blockIdx.x];
    const u32 a1 = cat ? (o1 < na ? o1 : na) : split[blockIdx.x + 1];
    const u32 b0 = o0 - a0, b1 = o1 - a1;
    const u32 la = a1 - a0, lb = b1 - b0;
    for (u32 i = threadIdx.x; i < la; i += MG_THREADS) sm[i] = A[a0 + i];
    for (u32 i = threadIdx.x; i < lb; i += MG_THREADS) sm[la + i] = B[b0 + i];
    __syncthreads();
    const Item* sa = sm;
    const Item* sb = sm + la;
    const u32 len = la + lb;
    u32 diag = threadIdx.x * VT;
    if (diag > len) diag = len;
    u32 ai = cat ? 0 : merge_path_search(sa, la, sb, lb, diag, kv);
    tsplit[threadIdx.x] = ai;
    if (threadIdx.x == 0) tsplit[MG_THREADS] = la;
    __syncthreads();
    // thread t merges exactly A[tsplit[t], tsplit[t+1]) and B[diag_t - tsplit[t], diag_{t+1} - tsplit[t+1]): on sorted
    // runs that is what the merge path gives it; if the splits of this tile do not partition it (unsorted runs), the tile is
    // written as it was loaded
    u32 dnext = diag + VT > len ? len : diag + VT;
    const u32 aend = tsplit[threadIdx.x + 1], bend = dnext - aend;
    u32 bi = diag - ai;
    const bool tile_bad = __syncthreads_or(cat || aend < ai || bend < bi);
    if (tile_bad) {
        for (u32 i = threadIdx.x; i < len; i += MG_THREADS) out[o0 + i] = sm[i];
        return;
    }
    Item r[VT];
#pragma unroll
    for (int i = 0; i < VT; ++i) {
        bool take_a;
        if (ai >= aend) take_a = false;
        else if (bi >= bend) take_a = true;
        else take_a = !canon_less(canon_key(sb[bi], kv), canon_key(sa[ai], kv));
        if (ai < aend || bi < bend) r[i] = take_a ? sa[ai] : sb[bi];
        if (take_a) ++ai; else ++bi;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < VT; ++i)
        if (threadIdx.x * VT + i < len) sm[threadIdx.x * VT + i] = r[i];
    __syncthreads();
    for (u32 i = threadIdx.x; i < len; i += MG_THREADS) out[o0 + i] = sm[i];
}

// Stable merge of k sorted runs (run r: run_items[r] items at runs[r]) into d_out, through d_tmp (>= the total): a tree of
// 2-way merges, ceil(log2 k) passes; the last pass writes d_out.  Empty runs are dropped (as SortNode never creates them,
// api/sort.hpp:696-704).
template <int WORDS>
int merge_runs_impl(tg_ctx* ctx, const KeyView& kv, const void* const* runs, const uint64_t* run_items, uint32_t k,
                    void* d_out, void* d_tmp) {
    typedef typename ItemT<WORDS>::type Item;
    constexpr int TILE = MergeCfg<WORDS>::TILE;
    struct Run { const Item* ptr; size_t len; };
    std::vector<Run> cur;
    size_t total = 0;
    for (uint32_t r = 0; r < k; ++r) {
        total += run_items[r];
        if (run_items[r]) cur.push_back({ (const Item*)runs[r], (size_t)run_items[r] });
    }
    if (total >= (1ull << 31)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "merge: %zu items", total);
    if (cur.empty()) return TG_OK;
    int levels = 0;
    for (size_t c = cur.size(); c > 1; c = (c + 1) / 2) ++levels;
    if (levels == 0) {
        TG_CUDA(ctx, cudaMemcpyAsync(d_out, cur[0].ptr, cur[0].len * sizeof(Item), cudaMemcpyDeviceToDevice, ctx->stream));
        return TG_OK;
    }
    // splits of every merge of a level, and one flag per merge
    const size_t npairs = cur.size() / 2;
    u32* d_split;
    TG_TRY(tg_ws_get(ctx, WS_SEG_TABLES, (total / TILE + 2 * npairs + 2) * 4 + npairs * 4 + 256, (void**)&d_split));
    u32* d_bad = d_split + total / TILE + 2 * npairs + 2;
    // ping-pong so that the last level lands in d_out: level l writes bufs[(levels - 1 - l) % 2]
    Item* bufs[2] = { (Item*)d_out, (Item*)d_tmp };
    for (int l = 0; l < levels; ++l) {
        Item* dst = bufs[(levels - 1 - l) % 2];
        TG_CUDA(ctx, cudaMemsetAsync(d_bad, 0, (cur.size() / 2) * 4 + 4, ctx->stream));
        std::vector<Run> next;
        size_t woff = 0, soff = 0;
        for (size_t i = 0; i < cur.size(); i += 2) {
            if (i + 1 < cur.size()) {
                const size_t len = cur[i].len + cur[i + 1].len;
                const u32 ntiles = (u32)((len + TILE - 1) / TILE);
                u32* split = d_split + soff;
                u32* bad = d_bad + i / 2;
                TG_LAUNCH_T(ctx, TG_K_MERGE, merge_splits_kernel<WORDS>, (ntiles + 1 + 127) / 128, 128, 0, cur[i].ptr,
                            (u32)cur[i].len, cur[i + 1].ptr, (u32)cur[i + 1].len, ntiles, split, bad, kv);
                TG_LAUNCH_T(ctx, TG_K_MERGE, merge2_kernel<WORDS>, ntiles, MG_THREADS, 0, cur[i].ptr, (u32)cur[i].len,
                            cur[i + 1].ptr, (u32)cur[i + 1].len, (const u32*)split, (const u32*)bad, dst + woff, kv);
                soff += ntiles + 1;
                next.push_back({ dst + woff, len });
                woff += len;
            }
            else {
                TG_CUDA(ctx, cudaMemcpyAsync(dst + woff, cur[i].ptr, cur[i].len * sizeof(Item), cudaMemcpyDeviceToDevice, ctx->stream));
                next.push_back({ dst + woff, cur[i].len });
                woff += cur[i].len;
            }
        }
        cur.swap(next);
    }
    return TG_OK;
}

// ---- multi-sequence selection ---------------------------------------------------------------------------------------
struct MergeRun { const void* ptr; u64 n; };
constexpr u32 SEL_DIGITS = 256;

// bit position of key byte r (0 = most significant) inside the canonical key
__host__ __device__ inline void key_byte_pos(const KeyView& kv, u32 r, bool* in_hi, u32* shift) {
    if (kv.kind == TG_KEY_UINT_LE) { *in_hi = false; *shift = 8 * (kv.bytes - 1 - r); }
    else if (r < 8) { *in_hi = true; *shift = 8 * (7 - r); }
    else { *in_hi = false; *shift = 8 * (15 - r); }
}
__host__ __device__ inline Canon with_key_byte(Canon c, const KeyView& kv, u32 r, u32 b) {
    bool in_hi;
    u32 sh;
    key_byte_pos(kv, r, &in_hi, &sh);
    if (in_hi) c.hi |= (u64)b << sh; else c.lo |= (u64)b << sh;
    return c;
}
// the smallest canonical key of the descriptor: the key bytes zero, the other bits as canon_key leaves them (complemented
// for descending descriptors)
Canon select_base(const KeyView& kv) {
    Canon m = { 0, 0 };
    for (u32 r = 0; r < kv.bytes; ++r) m = with_key_byte(m, kv, r, 0xffu);
    return kv.desc ? Canon{ ~m.hi, ~m.lo } : Canon{ 0, 0 };
}

template <class Item>
__device__ __forceinline__ u64 lower_bound_key(const Item* a, u64 n, const Canon& c, const KeyView& kv) {
    u64 lo = 0, hi = n;
    while (lo < hi) {
        const u64 mid = (lo + hi) >> 1;
        if (canon_less(canon_key(a[mid], kv), c)) lo = mid + 1; else hi = mid;
    }
    return lo;
}
template <class Item>
__device__ __forceinline__ u64 upper_bound_key(const Item* a, u64 n, const Canon& c, const KeyView& kv) {
    u64 lo = 0, hi = n;
    while (lo < hi) {
        const u64 mid = (lo + hi) >> 1;
        if (!canon_less(c, canon_key(a[mid], kv))) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// CTA (boundary d, run): thread b adds the number of the run's items below prefix[d] with key byte `round` = b
template <int WORDS>
__global__ void __launch_bounds__(SEL_DIGITS)
select_count_kernel(const MergeRun* __restrict__ runs, const Canon* __restrict__ prefix, u32 round, KeyView kv,
                    unsigned long long* __restrict__ counts) {
    typedef typename ItemT<WORDS>::type Item;
    const u32 d = blockIdx.x, b = threadIdx.x;
    const MergeRun r = runs[blockIdx.y];
    if (b == 0 || r.n == 0) return;
    const u64 c = lower_bound_key((const Item*)r.ptr, r.n, with_key_byte(prefix[d], kv, round, b), kv);
    if (c) atomicAdd(&counts[(size_t)d * SEL_DIGITS + b], (unsigned long long)c);
}

// key byte `round` of K_d: the largest b whose count (summed over every run of every worker) is <= t_d
__global__ void select_narrow_kernel(const unsigned long long* __restrict__ counts, const u64* __restrict__ targets, u32 nb,
                                     u32 round, KeyView kv, Canon* __restrict__ prefix) {
    const u32 d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= nb) return;
    u32 best = 0;
    for (u32 b = 1; b < SEL_DIGITS; ++b)
        if (counts[(size_t)d * SEL_DIGITS + b] <= targets[d]) best = b;
    prefix[d] = with_key_byte(prefix[d], kv, round, best);
}

// less[run * nb + d] / equal[...] = items of the run below / equal to K_d
template <int WORDS>
__global__ void select_bounds_kernel(const MergeRun* __restrict__ runs, u32 nruns, const Canon* __restrict__ keys, u32 nb,
                                     KeyView kv, u64* __restrict__ less, u64* __restrict__ equal) {
    typedef typename ItemT<WORDS>::type Item;
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nruns * nb) return;
    const MergeRun r = runs[t / nb];
    const Canon c = keys[t % nb];
    const u64 lo = lower_bound_key((const Item*)r.ptr, r.n, c, kv);
    less[t] = lo;
    equal[t] = upper_bound_key((const Item*)r.ptr, r.n, c, kv) - lo;
}

// device scratch of the selection (WS_SAMPLES): runs | targets | keys | counts | less | equal | gather (the all-gathers)
struct SelScratch {
    MergeRun* runs; u64* targets; Canon* keys; unsigned long long* counts; u64* less; u64* equal; u64* gather;
};
constexpr u32 SEL_MAX_RUNS = TG_MAX_RANKS * 16;
int sel_scratch(tg_ctx* ctx, SelScratch* s) {
    const size_t nb = TG_MAX_RANKS;
    unsigned char* d;
    const size_t bytes = SEL_MAX_RUNS * sizeof(MergeRun) + nb * 8 + nb * sizeof(Canon) + nb * SEL_DIGITS * 8 + 4 * SEL_MAX_RUNS * nb * 8;
    TG_TRY(tg_ws_get(ctx, WS_SAMPLES, bytes + 256, (void**)&d));
    s->runs = (MergeRun*)d;              d += SEL_MAX_RUNS * sizeof(MergeRun);
    s->targets = (u64*)d;                d += nb * 8;
    s->keys = (Canon*)d;                 d += nb * sizeof(Canon);
    s->counts = (unsigned long long*)d;  d += nb * SEL_DIGITS * 8;
    s->less = (u64*)d;                   d += SEL_MAX_RUNS * nb * 8;
    s->equal = (u64*)d;                 d += SEL_MAX_RUNS * nb * 8;
    s->gather = (u64*)d;
    return TG_OK;
}

// K_d of the nb = p - 1 inner boundaries over `nruns` runs (already in s.runs, targets in s.targets), then less / equal of
// every run at them.  collective: the counts are summed over the workers by an ncclAllReduce in every round; otherwise the
// runs are those of every (simulated) worker and the count kernel sums them itself.
template <int WORDS>
int select_keys(tg_ctx* ctx, const KeyView& kv, const SelScratch& s, u32 nruns, u32 nb, bool collective) {
    std::vector<Canon> base(nb, select_base(kv));
    TG_CUDA(ctx, cudaMemcpyAsync(s.keys, base.data(), nb * sizeof(Canon), cudaMemcpyHostToDevice, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));     // (base lives on this host stack)
    for (u32 r = 0; r < kv.bytes; ++r) {
        TG_CUDA(ctx, cudaMemsetAsync(s.counts, 0, (size_t)nb * SEL_DIGITS * 8, ctx->stream));
        if (nruns) TG_LAUNCH(ctx, select_count_kernel<WORDS>, dim3(nb, nruns), SEL_DIGITS, 0, (const MergeRun*)s.runs,
                             (const Canon*)s.keys, r, kv, s.counts);
        if (collective)
            TG_NCCL(ctx, ncclAllReduce(s.counts, s.counts, (size_t)nb * SEL_DIGITS, ncclUint64, ncclSum, ctx->comm, ctx->stream));
        TG_LAUNCH(ctx, select_narrow_kernel, 1, 32, 0, (const unsigned long long*)s.counts, (const u64*)s.targets, nb, r, kv, s.keys);
    }
    if (nruns)
        TG_LAUNCH(ctx, select_bounds_kernel<WORDS>, (nruns * nb + 127) / 128, 128, 0, (const MergeRun*)s.runs, nruns,
                  (const Canon*)s.keys, nb, kv, s.less, s.equal);
    return TG_OK;
}

// bounds of every run from the (less, equal) counts at the inner boundaries (layout [run][d], run = w * k + j); where those
// are inconsistent (unsorted input: the result is unspecified) the runs are cut as if every key were equal
int plan_bounds(u32 p, u32 k, const uint64_t* sizes, const uint64_t* targets, const uint64_t* less_in, const uint64_t* equal_in,
                uint64_t* bounds) {
    const u32 nruns = p * k, nb = p - 1;
    std::vector<uint64_t> less((size_t)nruns * (p + 1)), equal((size_t)nruns * (p + 1));
    for (u32 r = 0; r < nruns; ++r) {
        for (u32 d = 0; d <= p; ++d) {
            uint64_t& l = less[(size_t)r * (p + 1) + d];
            uint64_t& e = equal[(size_t)r * (p + 1) + d];
            if (d == 0) { l = 0; e = 0; }
            else if (d == p) { l = sizes[r]; e = 0; }
            else { l = less_in[(size_t)r * nb + d - 1]; e = equal_in[(size_t)r * nb + d - 1]; }
        }
    }
    if (tg_merge_plan(p, k, targets, less.data(), equal.data(), bounds) == TG_OK) return TG_OK;
    for (u32 r = 0; r < nruns; ++r)
        for (u32 d = 0; d <= p; ++d) {
            less[(size_t)r * (p + 1) + d] = 0;
            equal[(size_t)r * (p + 1) + d] = d == p ? 0 : sizes[r];
            if (d == p) less[(size_t)r * (p + 1) + d] = sizes[r];
        }
    return tg_merge_plan(p, k, targets, less.data(), equal.data(), bounds);
}

void merge_targets(u32 p, uint64_t total, uint64_t* targets) {
    for (u32 d = 0; d <= p; ++d) targets[d] = ((u64)d * total + p - 1) / p;
}

int check_merge_args(tg_ctx* ctx, const tg_key_desc* desc, KeyView* kv, uint32_t k) {
    if (!ctx || make_key_view(desc, kv) != TG_OK || (desc->item_bytes != 8 && desc->item_bytes != 16))
        return tg_set_error(ctx, TG_ERR_ARG, "merge: 8- or 16-byte items with a supported key descriptor");
    if (k < 2 || k > 16) return tg_set_error(ctx, TG_ERR_ARG, "merge: %u inputs (2..16)", k);
    return TG_OK;
}

// 8-byte words from src to dst (8-byte aligned) with 16-byte stores wherever dst allows: the exchange of the pieces into the
// peers' windows (NVLink moves 16-byte stores at about twice the rate of 8-byte ones)
__global__ void __launch_bounds__(256) copy_words_kernel(const u64* __restrict__ src, u64 words, u64* __restrict__ dst) {
    const u32 a = (u32)(((uintptr_t)dst >> 3) & 1u);        // dst word 0 sits at word `a` of its 16-byte group
    uint4* const dst4 = reinterpret_cast<uint4*>(dst - a);
    const u64 ngroups = (words + a + 1) / 2;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x; c < ngroups; c += stride) {
        const u64 w0 = 2 * c, w1 = 2 * c + 1;
        const bool ok0 = w0 >= a && w0 - a < words, ok1 = w1 - a < words;
        const u64 v0 = ok0 ? src[w0 - a] : 0, v1 = ok1 ? src[w1 - a] : 0;
        if (ok0 && ok1) dst4[c] = make_uint4((u32)v0, (u32)(v0 >> 32), (u32)v1, (u32)(v1 >> 32));
        else {
            u64* q = reinterpret_cast<u64*>(dst4 + c);
            if (ok0) q[0] = v0;
            if (ok1) q[1] = v1;
        }
    }
}

template <int WORDS>
int merge_multi_impl(tg_ctx* ctx, const KeyView& kv, const void* const* d_inputs, const size_t* n_inputs, uint32_t k,
                     void** out_dptr, size_t* out_n) {
    typedef typename ItemT<WORDS>::type Item;
    const u32 p = (u32)ctx->nranks, me = (u32)ctx->rank, nb = p - 1;
    const size_t s = sizeof(Item);
    const void* in[16];
    size_t in_bytes[16];
    for (u32 j = 0; j < k; ++j) { in[j] = d_inputs[j]; in_bytes[j] = n_inputs[j] * s; }
    TG_TRY(xwin_negotiate(ctx));
    TG_TRY(evacuate_window_inputs(ctx, in, in_bytes, k));
    // (1) the k shard sizes of every worker
    SelScratch sc;
    TG_TRY(sel_scratch(ctx, &sc));
    u64* h = (u64*)ctx->pinned + 32768;          // byte offset 256 KB of the pinned scratch: sizes | less | equal
    u64* d_sizes = sc.gather;
    for (u32 j = 0; j < 16; ++j) h[j] = j < k ? n_inputs[j] : 0;
    TG_CUDA(ctx, cudaMemcpyAsync(d_sizes, h, 16 * 8, cudaMemcpyHostToDevice, ctx->stream));
    TG_NCCL(ctx, ncclAllGather(d_sizes, d_sizes + 16, 16, ncclUint64, ctx->comm, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(h + 16, d_sizes + 16, (size_t)p * 16 * 8, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::vector<uint64_t> sizes((size_t)p * k);
    uint64_t total = 0, worst_shard = 0;
    for (u32 w = 0; w < p; ++w) {
        uint64_t mine = 0;
        for (u32 j = 0; j < k; ++j) { sizes[(size_t)w * k + j] = h[16 + w * 16 + j]; mine += h[16 + w * 16 + j]; }
        total += mine;
        worst_shard = std::max(worst_shard, mine);
    }
    std::vector<uint64_t> targets(p + 1);
    merge_targets(p, total, targets.data());
    uint64_t worst_share = 0;
    for (u32 d = 0; d < p; ++d) worst_share = std::max(worst_share, targets[d + 1] - targets[d]);
    if (worst_shard >= (1u << 30) || worst_share >= (1u << 30))        // (the same verdict on every rank)
        return tg_set_error(ctx, TG_ERR_TOO_LARGE, "merge: a worker holds or receives 2^30 or more items");
    Item* d_out;
    void* d_tmp;
    TG_TRY(tg_ws_get(ctx, WS_OUT, (targets[me + 1] - targets[me] + 1) * s, (void**)&d_out));
    TG_TRY(tg_ws_get(ctx, WS_AUX2, (targets[me + 1] - targets[me] + 1) * s, &d_tmp));
    *out_dptr = d_out;
    *out_n = (size_t)(targets[me + 1] - targets[me]);
    if (total == 0) return TG_OK;
    // (2) the boundary keys, (3) less / equal of the local runs at them, all-gathered
    MergeRun runs[16];
    for (u32 j = 0; j < k; ++j) runs[j] = MergeRun{ in[j], n_inputs[j] };
    TG_CUDA(ctx, cudaMemcpyAsync(sc.runs, runs, k * sizeof(MergeRun), cudaMemcpyHostToDevice, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(sc.targets, targets.data() + 1, nb * 8, cudaMemcpyHostToDevice, ctx->stream));
    TG_TRY(select_keys<WORDS>(ctx, kv, sc, k, nb, true));
    const size_t mine = (size_t)k * nb;           // less | equal of this worker's runs, gathered into [w][less | equal]
    u64* d_le = sc.gather;                        // [less | equal] of this worker, then those of every worker
    TG_CUDA(ctx, cudaMemcpyAsync(d_le, sc.less, mine * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(d_le + mine, sc.equal, mine * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    TG_NCCL(ctx, ncclAllGather(d_le, d_le + 2 * mine, 2 * mine, ncclUint64, ctx->comm, ctx->stream));
    u64* h_le = h + 512;
    TG_CUDA(ctx, cudaMemcpyAsync(h_le, d_le + 2 * mine, (size_t)p * 2 * mine * 8, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::vector<uint64_t> less((size_t)p * mine), equal((size_t)p * mine);
    for (u32 w = 0; w < p; ++w)
        for (size_t i = 0; i < mine; ++i) {
            less[w * mine + i] = h_le[w * 2 * mine + i];
            equal[w * mine + i] = h_le[w * 2 * mine + mine + i];
        }
    // (4) the plan: every rank derives the same one
    std::vector<uint64_t> bounds((size_t)p * k * (p + 1));
    if (plan_bounds(p, k, sizes.data(), targets.data(), less.data(), equal.data(), bounds.data()) != TG_OK)
        return tg_set_error(ctx, TG_ERR_ARG, "merge: inconsistent plan");
    auto piece = [&](u32 w, u32 j, u32 d) {
        const uint64_t* b = &bounds[((size_t)w * k + j) * (p + 1)];
        return b[d + 1] - b[d];
    };
    // where piece (w, j) lands in worker d's window: after the pieces of the inputs below j, and of input j's lower workers
    auto landing = [&](u32 w, u32 j, u32 d) {
        u64 off = 0;
        for (u32 jj = 0; jj < k; ++jj)
            for (u32 ww = 0; ww < p; ++ww) {
                if (jj == j && ww == w) return off;
                off += piece(ww, jj, d);
            }
        return off;
    };
    TG_TRY(xwin_ensure(ctx, (worst_share + 4) * s));
    // (5) the exchange: piece (me, j, d) = input j's items [bounds[d], bounds[d + 1]) into worker d's window
    const int xprof = ctx->profile ? tg_prof_begin(ctx, TG_K_EXCHANGE) : -1;
    if (ctx->xwin.mode == 1) {
        // every worker starts with its right-hand neighbour: at any time each window is written by one peer
        for (u32 q = 0; q < p; ++q) {
            const u32 d = (me + 1 + q) % p;
            for (u32 j = 0; j < k; ++j) {
                const u64 n = piece(me, j, d);
                if (!n) continue;
                const u64 first = bounds[((size_t)me * k + j) * (p + 1) + d];
                u64* dst = (u64*)((char*)ctx->xwin.peer[d] + landing(me, j, d) * s);
                const u64 words = n * (s / 8);
                const u32 grid = (u32)std::min<u64>((words / 2 + 256) / 256, (u64)ctx->sm_count * 8);
                TG_LAUNCH(ctx, copy_words_kernel, grid, 256, 0, (const u64*)((const char*)in[j] + first * s), words, dst);
            }
        }
        TG_TRY(xwin_barrier(ctx));
    }
    else {
        // pieces packed per destination in input order, one send per peer; received per source worker into a staging buffer,
        // then laid out input-major in the window
        size_t send_total = 0;
        for (u32 j = 0; j < k; ++j) send_total += n_inputs[j];
        char *d_send, *d_stage;
        TG_TRY(tg_ws_get(ctx, WS_XCHG_SEND, (send_total + 1) * s, (void**)&d_send));
        TG_TRY(tg_ws_get(ctx, WS_XCHG_RECV, (*out_n + 1) * s, (void**)&d_stage));
        std::vector<uint64_t> soff(p + 1, 0), roff(p + 1, 0);
        for (u32 d = 0; d < p; ++d) {
            soff[d + 1] = soff[d];
            roff[d + 1] = roff[d];
            for (u32 j = 0; j < k; ++j) {
                const u64 n = piece(me, j, d);
                if (n) TG_CUDA(ctx, cudaMemcpyAsync(d_send + soff[d + 1] * s, (const char*)in[j] + bounds[((size_t)me * k + j) * (p + 1) + d] * s,
                                                    n * s, cudaMemcpyDeviceToDevice, ctx->stream));
                soff[d + 1] += n;
                roff[d + 1] += piece(d, j, me);
            }
        }
        TG_NCCL(ctx, ncclGroupStart());
        for (u32 r = 0; r < p; ++r) {
            if (soff[r + 1] > soff[r]) TG_NCCL(ctx, ncclSend(d_send + soff[r] * s, (soff[r + 1] - soff[r]) * s, ncclUint8, r, ctx->comm, ctx->stream));
            if (roff[r + 1] > roff[r]) TG_NCCL(ctx, ncclRecv(d_stage + roff[r] * s, (roff[r + 1] - roff[r]) * s, ncclUint8, r, ctx->comm, ctx->stream));
        }
        TG_NCCL(ctx, ncclGroupEnd());
        for (u32 w = 0; w < p; ++w) {
            u64 o = roff[w];
            for (u32 j = 0; j < k; ++j) {
                const u64 n = piece(w, j, me);
                if (n) TG_CUDA(ctx, cudaMemcpyAsync((char*)ctx->xwin.base + landing(w, j, me) * s, d_stage + o * s, n * s,
                                                    cudaMemcpyDeviceToDevice, ctx->stream));
                o += n;
            }
        }
    }
    if (xprof >= 0) tg_prof_end(ctx, xprof);
    // the local merge of the k received runs
    const void* rp[16];
    uint64_t rn[16];
    for (u32 j = 0; j < k; ++j) {
        rp[j] = (const char*)ctx->xwin.base + landing(0, j, me) * s;
        rn[j] = 0;
        for (u32 w = 0; w < p; ++w) rn[j] += piece(w, j, me);
    }
    return merge_runs_impl<WORDS>(ctx, kv, rp, rn, k, d_out, d_tmp);
}

}  // namespace

namespace tgp {
// the merge of the received runs of Sort's TG_SORT_PIPELINE=merge (tg_sample_sort.cu)
int merge_runs(tg_ctx* ctx, const KeyView& kv, uint32_t item_bytes, const void* const* runs, const uint64_t* run_items,
               uint32_t k, void* d_out, void* d_tmp) {
    return item_bytes == 8 ? merge_runs_impl<1>(ctx, kv, runs, run_items, k, d_out, d_tmp)
                           : merge_runs_impl<2>(ctx, kv, runs, run_items, k, d_out, d_tmp);
}
}  // namespace tgp

extern "C" {

int tg_kway_merge(tg_ctx* ctx, const tg_key_desc* desc, const void* d_runs, const uint64_t* run_items, uint32_t k,
                  void* d_out, void* d_tmp) {
    KeyView kv;
    if (!ctx || make_key_view(desc, &kv) != TG_OK || (desc->item_bytes != 8 && desc->item_bytes != 16))
        return tg_set_error(ctx, TG_ERR_ARG, "kway_merge: unsupported descriptor");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<const void*> runs(k);
    size_t off = 0;
    for (uint32_t r = 0; r < k; ++r) { runs[r] = (const char*)d_runs + off * desc->item_bytes; off += run_items[r]; }
    return merge_runs(ctx, kv, desc->item_bytes, runs.data(), run_items, k, d_out, d_tmp);
}

int tg_merge_plan(uint32_t p, uint32_t k, const uint64_t* targets, const uint64_t* less, const uint64_t* equal,
                  uint64_t* out_bounds) {
    if (p == 0 || p > TG_MAX_RANKS || k == 0 || k > 16 || !targets || !less || !equal || !out_bounds) return TG_ERR_ARG;
    const u32 nruns = p * k;
    for (u32 d = 0; d <= p; ++d) {
        if (d && targets[d] < targets[d - 1]) return TG_ERR_ARG;
        u64 sl = 0, se = 0;
        for (u32 r = 0; r < nruns; ++r) { sl += less[(size_t)r * (p + 1) + d]; se += equal[(size_t)r * (p + 1) + d]; }
        if (targets[d] < sl || targets[d] - sl > se) return TG_ERR_ARG;
        // the items equal to K_d that precede rank t_d: in (input, worker) order
        u64 rem = targets[d] - sl;
        for (u32 j = 0; j < k; ++j)
            for (u32 w = 0; w < p; ++w) {
                const size_t i = ((size_t)w * k + j) * (p + 1) + d;
                const u64 take = rem < equal[i] ? rem : equal[i];
                out_bounds[i] = less[i] + take;
                rem -= take;
            }
    }
    for (u32 r = 0; r < nruns; ++r)
        for (u32 d = 1; d <= p; ++d)
            if (out_bounds[(size_t)r * (p + 1) + d] < out_bounds[(size_t)r * (p + 1) + d - 1]) return TG_ERR_ARG;
    return TG_OK;
}

int tg_merge_select(tg_ctx* ctx, const tg_key_desc* desc, const void* const* d_runs, const size_t* n_runs, uint32_t p,
                    uint32_t k, uint64_t* out_bounds) {
    KeyView kv;
    TG_TRY(check_merge_args(ctx, desc, &kv, k));
    if (p == 0 || p > TG_MAX_RANKS || !d_runs || !n_runs || !out_bounds) return tg_set_error(ctx, TG_ERR_ARG, "merge_select: arguments");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const u32 nruns = p * k, nb = p - 1;
    std::vector<uint64_t> sizes(nruns), targets(p + 1);
    u64 total = 0;
    for (u32 r = 0; r < nruns; ++r) {
        if (!d_runs[r] && n_runs[r]) return tg_set_error(ctx, TG_ERR_ARG, "merge_select: run %u is NULL", r);
        sizes[r] = n_runs[r];
        total += n_runs[r];
    }
    if (total >= (1u << 30)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "merge_select: %llu items", (unsigned long long)total);
    merge_targets(p, total, targets.data());
    std::vector<uint64_t> less((size_t)nruns * nb), equal((size_t)nruns * nb);
    if (nb) {
        SelScratch sc;
        TG_TRY(sel_scratch(ctx, &sc));
        std::vector<MergeRun> runs(nruns);
        for (u32 r = 0; r < nruns; ++r) runs[r] = MergeRun{ d_runs[r], n_runs[r] };
        TG_CUDA(ctx, cudaMemcpyAsync(sc.runs, runs.data(), nruns * sizeof(MergeRun), cudaMemcpyHostToDevice, ctx->stream));
        TG_CUDA(ctx, cudaMemcpyAsync(sc.targets, targets.data() + 1, nb * 8, cudaMemcpyHostToDevice, ctx->stream));
        if (desc->item_bytes == 8) TG_TRY(select_keys<1>(ctx, kv, sc, nruns, nb, false));
        else TG_TRY(select_keys<2>(ctx, kv, sc, nruns, nb, false));
        TG_CUDA(ctx, cudaMemcpyAsync(less.data(), sc.less, less.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaMemcpyAsync(equal.data(), sc.equal, equal.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (plan_bounds(p, k, sizes.data(), targets.data(), less.data(), equal.data(), out_bounds) != TG_OK)
        return tg_set_error(ctx, TG_ERR_ARG, "merge_select: inconsistent plan");
    return TG_OK;
}

int tg_merge(tg_ctx* ctx, const tg_key_desc* desc, const void* const* d_inputs, const size_t* n_inputs, uint32_t k,
             void** out_dptr, size_t* out_n) {
    KeyView kv;
    TG_TRY(check_merge_args(ctx, desc, &kv, k));
    if (!d_inputs || !n_inputs || !out_dptr || !out_n) return tg_set_error(ctx, TG_ERR_ARG, "merge: NULL argument");
    for (u32 j = 0; j < k; ++j)
        if (!d_inputs[j] && n_inputs[j]) return tg_set_error(ctx, TG_ERR_ARG, "merge: input %u is NULL", j);
    if (ctx->nranks > TG_MAX_RANKS) return tg_set_error(ctx, TG_ERR_ARG, "merge: at most 16 ranks");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t s = desc->item_bytes;
    if (ctx->nranks == 1) {
        // no selection and no exchange: the local merge of the k inputs
        size_t total = 0;
        for (u32 j = 0; j < k; ++j) total += n_inputs[j];
        if (total >= (1u << 30)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "merge: %zu items (limit 2^30 - 1)", total);
        void *d_out, *d_tmp;
        TG_TRY(tg_ws_get(ctx, WS_OUT, (total + 1) * s, &d_out));
        TG_TRY(tg_ws_get(ctx, WS_AUX2, (total + 1) * s, &d_tmp));
        uint64_t n[16];
        for (u32 j = 0; j < k; ++j) n[j] = n_inputs[j];
        TG_TRY(merge_runs(ctx, kv, desc->item_bytes, d_inputs, n, k, d_out, d_tmp));
        *out_dptr = d_out;
        *out_n = total;
        return TG_OK;
    }
    return s == 8 ? merge_multi_impl<1>(ctx, kv, d_inputs, n_inputs, k, out_dptr, out_n)
                  : merge_multi_impl<2>(ctx, kv, d_inputs, n_inputs, k, out_dptr, out_n);
}

int tg_merge_file(tg_ctx* ctx, const tg_key_desc* desc, const tg_merge_input* inputs, uint32_t k, size_t* out_items) {
    KeyView kv;
    TG_TRY(check_merge_args(ctx, desc, &kv, k));
    if (!inputs || !out_items) return tg_set_error(ctx, TG_ERR_ARG, "merge_file: NULL argument");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t s = desc->item_bytes;
    // host Files go up into one staging buffer (each at a 16-byte aligned offset), device Files are read where they are
    size_t n[16], off[16], staged = 0;
    for (u32 j = 0; j < k; ++j) {
        const tg_merge_input& in = inputs[j];
        if (in.dev) {
            if (in.dev->item_bytes != s || (!in.dev->dptr && in.dev->items))
                return tg_set_error(ctx, TG_ERR_ARG, "merge_file: device File %u has item size %u, the descriptor %zu", j, in.dev->item_bytes, s);
            n[j] = in.dev->items;
            continue;
        }
        if (!in.blocks && in.nblocks) return tg_set_error(ctx, TG_ERR_ARG, "merge_file: input %u has no blocks", j);
        size_t bytes = 0;
        for (size_t i = 0; i < in.nblocks; ++i) bytes += in.blocks[i].bytes;
        if (bytes % s) return tg_set_error(ctx, TG_ERR_ARG, "merge_file: input %u: %zu bytes is not a multiple of the item size", j, bytes);
        n[j] = bytes / s;
        off[j] = staged;
        staged += (bytes + 15) & ~(size_t)15;
    }
    char* d_stage = nullptr;
    if (staged) TG_TRY(tg_ws_get(ctx, WS_IN, staged + 16, (void**)&d_stage));
    const void* ptrs[16];
    for (u32 j = 0; j < k; ++j) {
        if (inputs[j].dev) { ptrs[j] = inputs[j].dev->dptr; continue; }
        ptrs[j] = d_stage ? d_stage + off[j] : nullptr;
        if (n[j]) TG_TRY(tg_upload_blocks(ctx, d_stage + off[j], inputs[j].blocks, inputs[j].nblocks, nullptr));
    }
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(tg_merge(ctx, desc, ptrs, n, k, &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = desc->item_bytes;
    *out_items = n_out;
    return TG_OK;
}

}  // extern "C"
