// tg_sample.cu — Sample (SampleNode, api/sample.hpp:37-140) and BernoulliSample (api/bernoulli_sample.hpp:27-77) by global
// position: position g has the 64-bit key key(seed, g) = mix(mix(seed) + (g + 1) * 0x9e3779b97f4a7c15), mix the SplitMix64
// output function (splitmix64_dev(x) = mix(x + gamma), so key = splitmix64_dev(mix(seed) + g * gamma)).  Keys of distinct
// positions are distinct, and no item is read to find which positions are kept:
//   Sample(s), 0 < s < N     K = the s-th smallest key of all N positions, found one digit per round (most significant first:
//                            12, 12, 12, 12, 12, 4 bits), keep key <= K: exactly s items
//   BernoulliSample(p)       keep (key >> 11) < ceil(p * 2^53)
// Selection: round 1 hashes every local position into a 4096-bin histogram of the top 12 bits (summed over the workers by one
// ncclAllReduce), a one-CTA kernel picks the digit and the remaining rank; round 2 hashes again and appends the keys of the chosen
// bin to a candidate buffer (about n / 4096 keys, but sized n so no overflow path exists); rounds 3-6 histogram the candidates
// only.  The state stays on the device: no host synchronisation between rounds.
// Compaction (both operators): keep a position iff its key < T (T = K + 1, or ceil(p * 2^53) << 11): a count kernel per tile of
// 4096 positions, the join's exclusive tile scan (tg_tile_scan.cuh), then a write kernel that hashes again and copies the kept
// items in input order.  The write loads only the kept items' words: Sample(10) of 1e8 items reads ten items.
#include "tg_tile_scan.cuh"

namespace {

constexpr u64 SP_LIMIT = 1ull << 30;
constexpr u64 GAMMA = 0x9E3779B97F4A7C15ull;
constexpr int SC_THREADS = 256;                 // count / write: 16 consecutive positions per thread
constexpr u32 SC_PER = 16;
constexpr u32 SC_TILE = SC_THREADS * SC_PER;
constexpr int SH_THREADS = 512;                 // histograms: grid-stride, a private 4096-bin histogram per CTA
constexpr u32 SH_BINS = 4096;
constexpr int SP_THREADS = 1024;                // the one-CTA digit pick: 4 bins per thread
constexpr int SEL_ROUNDS = 6;
constexpr u32 SEL_SHIFT[SEL_ROUNDS] = { 52, 40, 28, 16, 4, 0 };
constexpr u32 SEL_BITS[SEL_ROUNDS] = { 12, 12, 12, 12, 12, 4 };

// aux workspace, in u64 words: the histogram, the selection state, the output count, this worker's record and the p gathered
// records, then the tile counts and tile bases
enum { AUX_HIST = 0, AUX_STATE = SH_BINS, AUX_TOTAL = SH_BINS + 4, AUX_REC = SH_BINS + 8, AUX_TILES = AUX_REC + 4 * (TG_MAX_RANKS + 1) };
// selection state: the key prefix chosen so far, the rank still to find within it, T = K + 1, the candidates
enum { ST_PREFIX = 0, ST_RANK = 1, ST_THR = 2, ST_CAND = 3 };

// the all-gathered record of a worker: its size, its seed and the operator's parameter (s, or the bits of p)
struct Rec { u64 n, seed, param, pad; };

u64 mix_host(u64 z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// bit j set iff position i0 + j (< n) has a key below thr; z0 = mix(seed) + f * gamma for a worker starting at position f
__device__ __forceinline__ u32 keep_mask(u64 z0, u64 i0, u64 n, u64 thr) {
    u32 m = 0;
    u64 z = z0 + i0 * GAMMA;
#pragma unroll
    for (u32 j = 0; j < SC_PER; ++j) {
        if (i0 + j < n && splitmix64_dev(z) < thr) m |= 1u << j;
        z += GAMMA;
    }
    return m;
}

__device__ __forceinline__ void flush_hist(const u32* h, u32 nb, u64* hist) {
    __syncthreads();
    for (u32 b = threadIdx.x; b < nb; b += blockDim.x)
        if (h[b]) atomicAdd((unsigned long long*)&hist[b], (unsigned long long)h[b]);
}

// round 1: the top 12 bits of the keys of positions [0, n)
__global__ void __launch_bounds__(SH_THREADS) sample_hist_kernel(u64 z0, u64 n, u64* __restrict__ hist) {
    __shared__ u32 h[SH_BINS];
    for (u32 b = threadIdx.x; b < SH_BINS; b += SH_THREADS) h[b] = 0;
    __syncthreads();
    for (u64 i = (u64)blockIdx.x * SH_THREADS + threadIdx.x; i < n; i += (u64)gridDim.x * SH_THREADS)
        atomicAdd(&h[splitmix64_dev(z0 + i * GAMMA) >> 52], 1u);
    flush_hist(h, SH_BINS, hist);
}

// round 2: the keys whose top 12 bits are the chosen digit, appended to the candidates (order is irrelevant: only their
// histograms are taken)
__global__ void __launch_bounds__(SH_THREADS)
sample_gather_kernel(u64 z0, u64 n, u64* __restrict__ state, u64* __restrict__ cand) {
    const u64 top = state[ST_PREFIX] >> 52;
    for (u64 i = (u64)blockIdx.x * SH_THREADS + threadIdx.x; i < n; i += (u64)gridDim.x * SH_THREADS) {
        const u64 k = splitmix64_dev(z0 + i * GAMMA);
        if (k >> 52 == top) cand[atomicAdd((unsigned long long*)&state[ST_CAND], 1ull)] = k;
    }
}

// rounds 2-6: digit (k >> shift) & (2^bits - 1) of the candidates that agree with the prefix above it
__global__ void __launch_bounds__(SH_THREADS)
sample_cand_hist_kernel(const u64* __restrict__ cand, const u64* __restrict__ state, u32 shift, u32 bits, u64* __restrict__ hist) {
    __shared__ u32 h[SH_BINS];
    const u32 nb = 1u << bits, hi = shift + bits;
    const u64 top = state[ST_PREFIX] >> hi, nc = state[ST_CAND];
    for (u32 b = threadIdx.x; b < nb; b += SH_THREADS) h[b] = 0;
    __syncthreads();
    for (u64 c = (u64)blockIdx.x * SH_THREADS + threadIdx.x; c < nc; c += (u64)gridDim.x * SH_THREADS) {
        const u64 k = cand[c];
        if (k >> hi == top) atomicAdd(&h[(k >> shift) & (nb - 1)], 1u);
    }
    flush_hist(h, nb, hist);
}

// the digit holding the r-th smallest key of the current prefix (r = r0 in round 1, else the state's), the rank within it; T =
// K + 1 after the last digit.  Zeroes the histogram for the next round.
__global__ void __launch_bounds__(SP_THREADS) sample_pick_kernel(u64* __restrict__ hist, u64* __restrict__ state, u32 shift, u32 bits, u64 r0) {
    __shared__ u64 warp_tot[SP_THREADS / 32];
    const u32 nb = 1u << bits, b0 = threadIdx.x * 4;
    const u64 r = r0 ? r0 : state[ST_RANK];
    u64 c[4], sum = 0;
#pragma unroll
    for (u32 j = 0; j < 4; ++j) { c[j] = b0 + j < nb ? hist[b0 + j] : 0; sum += c[j]; }
    u64 tot;
    u64 before = block_excl_scan_u64<SP_THREADS>(sum, warp_tot, &tot);
    if (before < r && r <= before + sum) {
        for (u32 j = 0; j < 4; ++j) {
            if (r <= before + c[j]) {
                const u64 prefix = state[ST_PREFIX] | ((u64)(b0 + j) << shift);
                state[ST_PREFIX] = prefix;
                state[ST_RANK] = r - before;
                if (shift == 0) state[ST_THR] = prefix + 1;
                break;
            }
            before += c[j];
        }
    }
    for (u32 b = threadIdx.x; b < nb; b += SP_THREADS) hist[b] = 0;
}

// kept positions per tile of SC_TILE positions
__global__ void __launch_bounds__(SC_THREADS)
sample_count_kernel(u64 z0, u64 n, const u64* __restrict__ d_thr, u64 thr_v, u64* __restrict__ tile_cnt) {
    __shared__ u64 warp_tot[SC_THREADS / 32];
    const u64 thr = d_thr ? *d_thr : thr_v;
    const u32 m = keep_mask(z0, (u64)blockIdx.x * SC_TILE + threadIdx.x * SC_PER, n, thr);
    u64 tot;
    block_excl_scan_u64<SC_THREADS>(__popc(m), warp_tot, &tot);
    if (threadIdx.x == 0) tile_cnt[blockIdx.x] = tot;
}

// the kept items of a tile, in order, from output index tile_base[tile]: the kept positions are listed in shared memory, then
// the CTA copies their words (units of U bytes, w units per item) so that only kept items are loaded
template <typename U>
__global__ void __launch_bounds__(SC_THREADS)
sample_write_kernel(const U* __restrict__ in, u64 z0, u64 n, const u64* __restrict__ d_thr, u64 thr_v,
                    const u64* __restrict__ tile_base, u32 w, U* __restrict__ out) {
    __shared__ u32 idx[SC_TILE];
    __shared__ u64 warp_tot[SC_THREADS / 32];
    const u64 thr = d_thr ? *d_thr : thr_v;
    const u64 t0 = (u64)blockIdx.x * SC_TILE;
    u32 m = keep_mask(z0, t0 + threadIdx.x * SC_PER, n, thr);
    u64 tot;
    u32 o = (u32)block_excl_scan_u64<SC_THREADS>(__popc(m), warp_tot, &tot);
    while (m) {
        idx[o++] = threadIdx.x * SC_PER + __ffs(m) - 1;
        m &= m - 1;
    }
    __syncthreads();
    const U* src = in + t0 * w;
    U* dst = out + tile_base[blockIdx.x] * w;
    const u32 units = (u32)tot * w;
    for (u32 u = threadIdx.x; u < units; u += SC_THREADS) {
        const u32 item = u / w;
        dst[u] = src[(u64)idx[item] * w + (u - item * w)];
    }
}

// ---- host side ---------------------------------------------------------------------------------------------------------------

int check_item_bytes(tg_ctx* ctx, const char* what, uint32_t ib) {
    if (ib < 4 || ib > 256 || ib % 4)
        return tg_set_error(ctx, TG_ERR_ARG, "%s: %u-byte items (a multiple of 4 bytes from 4 to 256)", what, ib);
    return TG_OK;
}

int check_ranks(tg_ctx* ctx, const char* what) {
    if (ctx->nranks > TG_MAX_RANKS) return tg_set_error(ctx, TG_ERR_ARG, "%s: at most 16 ranks", what);
    return TG_OK;
}

double p_of(u64 bits) {
    double p;
    memcpy(&p, &bits, 8);
    return p;
}

// the verdict from every worker's record (the same on every rank): the limits, then the parameter all ranks must share
int verdict(tg_ctx* ctx, const char* what, bool bern, const Rec* recs, u32 p) {
    for (u32 w = 0; w < p; ++w)
        if (recs[w].n >= SP_LIMIT)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "%s: worker %u holds %llu items (limit 2^30 - 1)", what, w,
                                (unsigned long long)recs[w].n);
    for (u32 w = 1; w < p; ++w)
        if (recs[w].param != recs[0].param)
            return tg_set_error(ctx, TG_ERR_ARG, "%s: worker %u's %s differs from worker 0's", what, w,
                                bern ? "probability" : "sample size");
    if (bern) {
        const double pv = p_of(recs[0].param);
        if (!(pv >= 0.0 && pv <= 1.0)) return tg_set_error(ctx, TG_ERR_ARG, "%s: probability %g (0..1)", what, pv);
    }
    return TG_OK;
}

// the aux workspace with room for the tiles of n positions (none when n is over the limit: the verdict refuses it)
int prepare_aux(tg_ctx* ctx, u64 n, u64** aux) {
    const u64 nt = n < SP_LIMIT ? (n + SC_TILE - 1) / SC_TILE : 0;
    return tg_ws_get(ctx, WS_SAMPLE_AUX, (AUX_TILES + 2 * nt + 2) * 8, (void**)aux);
}

u32 hash_grid(tg_ctx* ctx, u64 n) {
    const u64 g = (n + SH_THREADS - 1) / SH_THREADS, cap = 2 * (u64)ctx->sm_count;
    return (u32)(g < cap ? g : cap);
}

// T = K + 1 into state[ST_THR], K the s-th smallest key of the positions [fs[w], fs[w] + ns[w]) of the nw workers: the
// worker's own range with the histograms all-reduced (collective), or every simulated worker into the same histogram
int select_threshold(tg_ctx* ctx, u64 ms, const u64* fs, const u64* ns, u32 nw, bool collective, u64 s, u64* aux) {
    u64* hist = aux + AUX_HIST;
    u64* state = aux + AUX_STATE;
    u64 nc = 0;
    for (u32 w = 0; w < nw; ++w) nc += ns[w];
    u64* cand;
    TG_TRY(tg_ws_get(ctx, WS_SAMPLE_CAND, nc * 8 + 16, (void**)&cand));
    TG_CUDA(ctx, cudaMemsetAsync(aux, 0, (SH_BINS + 4) * 8, ctx->stream));
    for (int r = 0; r < SEL_ROUNDS; ++r) {
        if (r == 0) {
            for (u32 w = 0; w < nw; ++w)
                if (ns[w]) TG_LAUNCH_T(ctx, TG_K_SAMPLE, sample_hist_kernel, hash_grid(ctx, ns[w]), SH_THREADS, 0, ms + fs[w] * GAMMA, ns[w], hist);
        }
        else {
            if (r == 1)
                for (u32 w = 0; w < nw; ++w)
                    if (ns[w]) TG_LAUNCH_T(ctx, TG_K_SAMPLE, sample_gather_kernel, hash_grid(ctx, ns[w]), SH_THREADS, 0, ms + fs[w] * GAMMA, ns[w], state, cand);
            TG_LAUNCH_T(ctx, TG_K_SAMPLE, sample_cand_hist_kernel, ctx->sm_count, SH_THREADS, 0, (const u64*)cand, (const u64*)state,
                        SEL_SHIFT[r], SEL_BITS[r], hist);
        }
        if (collective) TG_NCCL(ctx, ncclAllReduce(hist, hist, 1u << SEL_BITS[r], ncclUint64, ncclSum, ctx->comm, ctx->stream));
        TG_LAUNCH_T(ctx, TG_K_SAMPLE, sample_pick_kernel, 1, SP_THREADS, 0, hist, state, SEL_SHIFT[r], SEL_BITS[r], r == 0 ? s : 0ull);
    }
    return TG_OK;
}

template <typename U>
int launch_write(tg_ctx* ctx, u32 nt, const void* d_in, u64 z0, u64 n, const u64* d_thr, u64 thr, const u64* tile_base, u32 ib,
                 void* out) {
    TG_LAUNCH_T(ctx, TG_K_SAMPLE, sample_write_kernel<U>, nt, SC_THREADS, 0, (const U*)d_in, z0, n, d_thr, thr, tile_base,
                ib / (u32)sizeof(U), (U*)out);
    return TG_OK;
}

// the worker's n items at positions z0's, kept iff key < T (*d_thr on the device, or thr): count, scan, then the output size
// (known = the count when the caller knows it, else one host read) and the write
int compact(tg_ctx* ctx, u32 ib, const void* d_in, u64 n, u64 z0, const u64* d_thr, u64 thr, const u64* known, u64* aux,
            void** out_dptr, u64* out_n) {
    const u32 nt = (u32)((n + SC_TILE - 1) / SC_TILE);
    u64* tile_cnt = aux + AUX_TILES;
    u64* tile_base = tile_cnt + nt;
    u64 m = 0;
    if (n) {
        TG_LAUNCH_T(ctx, TG_K_SAMPLE, sample_count_kernel, nt, SC_THREADS, 0, z0, n, d_thr, thr, tile_cnt);
        TG_LAUNCH_T(ctx, TG_K_SAMPLE, join_scan_tiles_kernel, 1, JS_THREADS, 0, (const u64*)tile_cnt, nt, tile_base, aux + AUX_TOTAL);
        if (known) m = *known;
        else {
            u64* h = (u64*)((char*)ctx->pinned + 8192);
            TG_CUDA(ctx, cudaMemcpyAsync(h, aux + AUX_TOTAL, 8, cudaMemcpyDeviceToHost, ctx->stream));
            TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            m = *h;
        }
    }
    void* out;
    TG_TRY(tg_ws_get(ctx, WS_SAMPLE_OUT, m * ib + 16, &out));
    if (m) {
        if (ib % 16 == 0) TG_TRY(launch_write<uint4>(ctx, nt, d_in, z0, n, d_thr, thr, tile_base, ib, out));
        else if (ib % 8 == 0) TG_TRY(launch_write<uint2>(ctx, nt, d_in, z0, n, d_thr, thr, tile_base, ib, out));
        else TG_TRY(launch_write<u32>(ctx, nt, d_in, z0, n, d_thr, thr, tile_base, ib, out));
    }
    *out_dptr = out;
    *out_n = m;
    return TG_OK;
}

// every item of the worker (s >= N, or p = 1), or none
int take_all(tg_ctx* ctx, u32 ib, const void* d_in, u64 n, void** out_dptr, u64* out_n) {
    void* out;
    TG_TRY(tg_ws_get(ctx, WS_SAMPLE_OUT, n * ib + 16, &out));
    if (n) TG_CUDA(ctx, cudaMemcpyAsync(out, d_in, n * ib, cudaMemcpyDeviceToDevice, ctx->stream));
    *out_dptr = out;
    *out_n = n;
    return TG_OK;
}

// worker `rank` of p once every worker's record is on the host: the verdict, then the selection (collective: this worker's
// positions, histograms all-reduced; otherwise every worker's positions on this device: one worker, or p simulated ones) and
// the compaction of d_in
int sample_run(tg_ctx* ctx, const char* what, bool bern, u32 ib, const void* d_in, const Rec* recs, u32 p, u32 rank,
               bool collective, void** out_dptr, size_t* out_n) {
    TG_TRY(verdict(ctx, what, bern, recs, p));
    u64 fs[TG_MAX_RANKS], ns[TG_MAX_RANKS], N = 0;
    for (u32 w = 0; w < p; ++w) { fs[w] = N; ns[w] = recs[w].n; N += recs[w].n; }
    const u64 n = ns[rank], ms = mix_host(recs[0].seed), z0 = ms + fs[rank] * GAMMA, param = recs[0].param;
    u64* aux;
    TG_TRY(prepare_aux(ctx, n, &aux));
    u64 m = 0;
    void* out;
    if (!bern) {
        if (param >= N) TG_TRY(take_all(ctx, ib, d_in, n, &out, &m));
        else if (param == 0) TG_TRY(take_all(ctx, ib, d_in, 0, &out, &m));
        else {
            if (collective) TG_TRY(select_threshold(ctx, ms, fs + rank, ns + rank, 1, true, param, aux));
            else TG_TRY(select_threshold(ctx, ms, fs, ns, p, false, param, aux));
            // one worker keeps exactly s: no read of its count
            TG_TRY(compact(ctx, ib, d_in, n, z0, aux + AUX_STATE + ST_THR, 0, p == 1 ? &param : nullptr, aux, &out, &m));
        }
    }
    else {
        const double pv = p_of(param);
        if (pv == 1.0) TG_TRY(take_all(ctx, ib, d_in, n, &out, &m));
        else if (pv == 0.0) TG_TRY(take_all(ctx, ib, d_in, 0, &out, &m));
        else {
            // p * 2^53 is exact (a power-of-two scaling), so is its ceiling; < 2^53 for p < 1
            const u64 t = (u64)ceil(ldexp(pv, 53));
            TG_TRY(compact(ctx, ib, d_in, n, z0, nullptr, t << 11, nullptr, aux, &out, &m));
        }
    }
    *out_dptr = out;
    *out_n = (size_t)m;
    return TG_OK;
}

// p = 1: no collective.  p > 1: this worker's record into one ncclAllGather, one host read of the records, then sample_run.
int sample_impl(tg_ctx* ctx, const char* what, bool bern, u32 ib, const void* d_in, size_t n_local, u64 param, u64 seed,
                void** out_dptr, size_t* out_n) {
    const u32 p = (u32)ctx->nranks;
    Rec recs[TG_MAX_RANKS];
    if (p == 1) recs[0] = Rec{ n_local, seed, param, 0 };
    else {
        u64* aux;
        TG_TRY(prepare_aux(ctx, n_local, &aux));
        Rec* h = (Rec*)ctx->pinned;
        h[0] = Rec{ n_local, seed, param, 0 };
        TG_CUDA(ctx, cudaMemcpyAsync(aux + AUX_REC, h, sizeof(Rec), cudaMemcpyHostToDevice, ctx->stream));
        TG_NCCL(ctx, ncclAllGather(aux + AUX_REC, aux + AUX_REC + 4, sizeof(Rec), ncclUint8, ctx->comm, ctx->stream));
        Rec* hs = (Rec*)((char*)ctx->pinned + 4096);
        TG_CUDA(ctx, cudaMemcpyAsync(hs, aux + AUX_REC + 4, p * sizeof(Rec), cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (u32 w = 0; w < p; ++w) recs[w] = hs[w];
    }
    return sample_run(ctx, what, bern, ib, d_in, recs, p, (u32)ctx->rank, p > 1, out_dptr, out_n);
}

// a host File goes up into the WS_IN staging buffer, a device File is read where it is
int stage_input(tg_ctx* ctx, const char* what, const tg_merge_input* in, uint32_t item_bytes, const void** d_in, size_t* n) {
    if (in->dev) {
        if (in->dev->item_bytes != item_bytes || (!in->dev->dptr && in->dev->items))
            return tg_set_error(ctx, TG_ERR_ARG, "%s: the device File has item size %u, the operator takes %u", what,
                                in->dev->item_bytes, item_bytes);
        *d_in = in->dev->dptr;
        *n = in->dev->items;
        return TG_OK;
    }
    if (!in->blocks && in->nblocks) return tg_set_error(ctx, TG_ERR_ARG, "%s: the input has no blocks", what);
    size_t bytes = 0;
    for (size_t i = 0; i < in->nblocks; ++i) bytes += in->blocks[i].bytes;
    if (bytes % item_bytes) return tg_set_error(ctx, TG_ERR_ARG, "%s: %zu bytes is not a multiple of %u", what, bytes, item_bytes);
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

int device_call(tg_ctx* ctx, const char* what, bool bern, uint32_t ib, const void* d_in, size_t n_local, u64 param, u64 seed,
                void** out_dptr, size_t* out_n) {
    if (!ctx || !out_dptr || !out_n || (!d_in && n_local)) return tg_set_error(ctx, TG_ERR_ARG, "%s: NULL argument", what);
    TG_TRY(check_item_bytes(ctx, what, ib));
    TG_TRY(check_ranks(ctx, what));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return sample_impl(ctx, what, bern, ib, d_in, n_local, param, seed, out_dptr, out_n);
}

int file_call(tg_ctx* ctx, const char* what, bool bern, uint32_t ib, const tg_merge_input* in, u64 param, u64 seed,
              size_t* out_items) {
    if (!ctx || !in || !out_items) return tg_set_error(ctx, TG_ERR_ARG, "%s: NULL argument", what);
    TG_TRY(check_item_bytes(ctx, what, ib));
    TG_TRY(check_ranks(ctx, what));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* d_in;
    size_t n;
    TG_TRY(stage_input(ctx, what, in, ib, &d_in, &n));
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(sample_impl(ctx, what, bern, ib, d_in, n, param, seed, &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = ib;
    *out_items = n_out;
    return TG_OK;
}

int select_call(tg_ctx* ctx, const char* what, bool bern, uint32_t ib, const void* const* d_shards, const size_t* n_shards,
                uint32_t p, uint32_t rank, const uint64_t* params, const uint64_t* seeds, void** out_dptr, size_t* out_n) {
    if (!ctx || !d_shards || !n_shards || !params || !seeds || !out_dptr || !out_n || p == 0 || p > TG_MAX_RANKS || rank >= p)
        return tg_set_error(ctx, TG_ERR_ARG, "%s: rank=%u p=%u or a NULL argument", what, rank, p);
    TG_TRY(check_item_bytes(ctx, what, ib));
    Rec recs[TG_MAX_RANKS];
    for (uint32_t w = 0; w < p; ++w) {
        if (!d_shards[w] && n_shards[w]) return tg_set_error(ctx, TG_ERR_ARG, "%s: shard %u is NULL", what, w);
        recs[w] = Rec{ n_shards[w], seeds[w], params[w], 0 };
    }
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return sample_run(ctx, what, bern, ib, d_shards[rank], recs, p, rank, false, out_dptr, out_n);
}

u64 bits_of(double p) {
    u64 b;
    memcpy(&b, &p, 8);
    return b;
}

}  // namespace

extern "C" {

int tg_sample(tg_ctx* ctx, uint32_t item_bytes, const void* d_in, size_t n_local, uint64_t sample_size, uint64_t seed,
              void** out_dptr, size_t* out_n) {
    return device_call(ctx, "sample", false, item_bytes, d_in, n_local, sample_size, seed, out_dptr, out_n);
}

int tg_bernoulli_sample(tg_ctx* ctx, uint32_t item_bytes, const void* d_in, size_t n_local, double p, uint64_t seed,
                        void** out_dptr, size_t* out_n) {
    return device_call(ctx, "bernoulli_sample", true, item_bytes, d_in, n_local, bits_of(p), seed, out_dptr, out_n);
}

int tg_sample_file(tg_ctx* ctx, uint32_t item_bytes, const tg_merge_input* in, uint64_t sample_size, uint64_t seed,
                   size_t* out_items) {
    return file_call(ctx, "sample_file", false, item_bytes, in, sample_size, seed, out_items);
}

int tg_bernoulli_sample_file(tg_ctx* ctx, uint32_t item_bytes, const tg_merge_input* in, double p, uint64_t seed,
                             size_t* out_items) {
    return file_call(ctx, "bernoulli_sample_file", true, item_bytes, in, bits_of(p), seed, out_items);
}

int tg_sample_select(tg_ctx* ctx, uint32_t item_bytes, const void* const* d_shards, const size_t* n_shards, uint32_t p_workers,
                     uint32_t rank, const uint64_t* sample_sizes, const uint64_t* seeds, void** out_dptr, size_t* out_n) {
    return select_call(ctx, "sample_select", false, item_bytes, d_shards, n_shards, p_workers, rank, sample_sizes, seeds,
                       out_dptr, out_n);
}

int tg_bernoulli_sample_select(tg_ctx* ctx, uint32_t item_bytes, const void* const* d_shards, const size_t* n_shards,
                               uint32_t p_workers, uint32_t rank, const double* ps, const uint64_t* seeds, void** out_dptr,
                               size_t* out_n) {
    if (!ps) return tg_set_error(ctx, TG_ERR_ARG, "bernoulli_sample_select: NULL argument");
    uint64_t bits[TG_MAX_RANKS];
    for (uint32_t w = 0; w < p_workers && w < TG_MAX_RANKS; ++w) bits[w] = bits_of(ps[w]);
    return select_call(ctx, "bernoulli_sample_select", true, item_bytes, d_shards, n_shards, p_workers, rank, bits, seeds,
                       out_dptr, out_n);
}

}  // extern "C"
