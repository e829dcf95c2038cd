// tg_hll.cu — HyperLogLog (HyperLogLogNode, api/hyperloglog.hpp:26-72; HyperLogLogRegisters<p>, core/hyperloglog.cpp:1715-1768):
// every item is hashed with SipHash-2-4 (key bytes 0..15, tlx/siphash.hpp:248-270) and raises one of 2^p one-byte registers:
//   index = h >> (64 - p),  w = h << p,  value = (w == 0 ? 64 - p : clz(w)) + 1,  register = max of its values.
// The registers of the workers merge by per-register max.  Max is commutative and associative, so the registers depend on the
// multiset of items only: not on the sharding, the tile order, or which CTA saw an item first.
//
//   hll_update_kernel<IB, SHARED>   persistent CTAs, grid-stride over 32 KB tiles (256 threads x 8 coalesced 16-byte loads), SipHash
//                                   in registers.  Registers are bytes packed four to a 32-bit word.  A thread reads the word
//                                   (a plain load) and only where its value is larger raises the byte: a compare-and-swap loop
//                                   on the word with a per-byte max.  After the first few thousand items almost no item raises
//                                   a register, so the atomic is the cold path.
//     SHARED (p <= 17)              a private register array per CTA in shared memory (2^p bytes: 128 KB at p = 17), flushed into
//                                   the worker's global array once at the end with the same per-byte max, zero words skipped
//     !SHARED (p = 18)              256 KB does not fit in shared memory: the CTAs work on the worker's global array directly.
//                                   It stays in L2; a stale cached word can only be smaller than the current one (registers
//                                   never decrease), so the filter lets through an update too many, never one too few
//   hll_merge_kernel                _select only: the per-register max over the simulated workers' arrays, what the all-reduce does
// No CTA waits on another and nothing depends on launch order.
#include "tg_common.cuh"

namespace {

constexpr u64 HLL_LIMIT = 1ull << 30;
constexpr int HL_THREADS = 256;
constexpr int HL_UNITS = 8;                         // 16-byte units per thread and tile
constexpr int HL_TILE_UNITS = HL_THREADS * HL_UNITS;    // 32 KB: 4096 8-byte items or 2048 pairs
constexpr u32 HL_SHARED_MAX_P = 17;
constexpr int HL_MAX_SMEM = 1 << HL_SHARED_MAX_P;
constexpr size_t HL_SLOT_PAD = 16;                  // a worker's array: 2^p register bytes, the over-the-limit flag byte, padding

__device__ __forceinline__ u64 rotl64(u64 x, int r) {       // r <= 32: two funnel shifts (a swap of the halves at 32)
    const u32 lo = (u32)x, hi = (u32)(x >> 32);
    if (r == 32) return ((u64)lo << 32) | hi;
    return ((u64)__funnelshift_l(lo, hi, r) << 32) | __funnelshift_l(hi, lo, r);
}

#define HL_SIPROUND()                                                               \
    do {                                                                            \
        v0 += v1; v1 = rotl64(v1, 13); v1 ^= v0; v0 = rotl64(v0, 32);               \
        v2 += v3; v3 = rotl64(v3, 16); v3 ^= v2;                                    \
        v0 += v3; v3 = rotl64(v3, 21); v3 ^= v0;                                    \
        v2 += v1; v1 = rotl64(v1, 17); v1 ^= v2; v2 = rotl64(v2, 32);               \
    } while (0)

// SipHash-2-4 of an IB-byte message (m0, and m1 for 16 bytes) under the key k0 = 0x0706050403020100, k1 = 0x0f0e0d0c0b0a0908:
// two rounds per message word, the length in the top byte of the last word, 0xff into v2, four rounds
template <int IB>
__device__ __forceinline__ u64 siphash24(u64 m0, u64 m1) {
    constexpr u64 k0 = 0x0706050403020100ull, k1 = 0x0f0e0d0c0b0a0908ull;
    u64 v0 = k0 ^ 0x736f6d6570736575ull, v1 = k1 ^ 0x646f72616e646f6dull;
    u64 v2 = k0 ^ 0x6c7967656e657261ull, v3 = k1 ^ 0x7465646279746573ull;
    v3 ^= m0; HL_SIPROUND(); HL_SIPROUND(); v0 ^= m0;
    if (IB == 16) { v3 ^= m1; HL_SIPROUND(); HL_SIPROUND(); v0 ^= m1; }
    constexpr u64 last = (u64)IB << 56;
    v3 ^= last; HL_SIPROUND(); HL_SIPROUND(); v0 ^= last;
    v2 ^= 0xff;
    HL_SIPROUND(); HL_SIPROUND(); HL_SIPROUND(); HL_SIPROUND();
    return v0 ^ v1 ^ v2 ^ v3;
}

// word = per-byte max(word, vals), given the value `old` just read from it
__device__ __forceinline__ void raise_word(u32* word, u32 old, u32 vals) {
    for (;;) {
        const u32 want = __vmaxu4(old, vals);
        if (want == old) return;
        const u32 seen = atomicCAS(word, old, want);
        if (seen == old) return;
        old = seen;
    }
}

// clz(h << p) is 64 where the low 64 - p bits of h are all zero, and at most 63 - p otherwise: the min is the stock rule
__device__ __forceinline__ void hll_insert(u32* regs, u64 h, u32 p) {
    const u32 idx = (u32)(h >> (64 - p));
    const u32 val = min((u32)__clzll((long long)(h << p)), 64u - p) + 1u;
    const u32 shift = (idx & 3u) * 8u;
    u32* word = regs + (idx >> 2);
    const u32 old = *word;
    if (((old >> shift) & 0xffu) < val) raise_word(word, old, val << shift);
}

// unit u of the input: a pair, or two 8-byte items (one if the input's last item is its first half); nothing past the end
template <int IB>
__device__ __forceinline__ ulonglong2 load_unit(const ulonglong2* __restrict__ in, u64 u, u64 n, u64 units) {
    if (u >= units) return make_ulonglong2(0, 0);
    if (IB == 16 || 2 * u + 1 < n) return in[u];
    return make_ulonglong2(((const u64*)in)[2 * u], 0);
}

template <int IB, bool SHARED>
__global__ void __launch_bounds__(HL_THREADS) hll_update_kernel(const ulonglong2* __restrict__ in, u64 n, u32 p, u32 ntiles,
                                                                u32* regs) {
    extern __shared__ u32 sregs[];
    const u32 words = (1u << p) / 4;
    u32* mine = SHARED ? sregs : regs;
    if (SHARED) {
        for (u32 i = threadIdx.x; i < words; i += HL_THREADS) sregs[i] = 0;
        __syncthreads();
    }
    // The unit loop is not unrolled: SipHash is a few hundred instructions per item, and eight inlined copies of it (64 KB of code
    // for 8-byte items) run out of the instruction cache.  The next unit is loaded before the current one is hashed.
    const u64 units = IB == 16 ? n : (n + 1) / 2;
    for (u32 tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        u64 u = (u64)tile * HL_TILE_UNITS + threadIdx.x;
        ulonglong2 cur = load_unit<IB>(in, u, n, units);
#pragma unroll 1
        for (int j = 0; j < HL_UNITS && u < units; ++j, u += HL_THREADS) {
            const ulonglong2 next = j + 1 < HL_UNITS ? load_unit<IB>(in, u + HL_THREADS, n, units) : make_ulonglong2(0, 0);
            if (IB == 16) hll_insert(mine, siphash24<16>(cur.x, cur.y), p);
            else {
                hll_insert(mine, siphash24<8>(cur.x, 0), p);
                if (2 * u + 1 < n) hll_insert(mine, siphash24<8>(cur.y, 0), p);
            }
            cur = next;
        }
    }
    if (SHARED) {
        __syncthreads();
        for (u32 i = threadIdx.x; i < words; i += HL_THREADS) {
            const u32 s = sregs[i];
            if (s) raise_word(regs + i, regs[i], s);
        }
    }
}

// out = the per-register max of the nslots arrays at slots + w * stride (words; the flag byte's word included)
__global__ void hll_merge_kernel(const u32* __restrict__ slots, u32 nslots, u32 stride, u32 words, u32* __restrict__ out) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= words) return;
    u32 m = 0;
    for (u32 w = 0; w < nslots; ++w) m = __vmaxu4(m, slots[(size_t)w * stride + i]);
    out[i] = m;
}

int check_args(tg_ctx* ctx, const char* what, uint32_t item_bytes, uint32_t precision) {
    if (item_bytes != 8 && item_bytes != 16)
        return tg_set_error(ctx, TG_ERR_ARG, "%s: %u-byte items (8: uint64_t / double, 16: pair<uint64_t, V>)", what, item_bytes);
    if (precision < 4 || precision > 18) return tg_set_error(ctx, TG_ERR_ARG, "%s: precision %u (4..18)", what, precision);
    return TG_OK;
}

size_t slot_bytes(u32 p) { return ((size_t)1 << p) + HL_SLOT_PAD; }

template <int IB, bool SHARED>
int launch_update(tg_ctx* ctx, const void* d_in, u64 n, u32 p, u32* regs) {
    auto kern = hll_update_kernel<IB, SHARED>;
    const size_t smem = SHARED ? (size_t)1 << p : 0;
    if (SHARED && ctx->kernel_cfg.find((const void*)kern) == ctx->kernel_cfg.end()) {
        TG_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, HL_MAX_SMEM));
        ctx->kernel_cfg[(const void*)kern] = 1;
    }
    int ctas_per_sm = 0;
    TG_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, kern, HL_THREADS, smem));
    if (ctas_per_sm < 1) return tg_set_error(ctx, TG_ERR_CUDA, "hyperloglog: the update kernel does not fit on an SM");
    const u64 ntiles = (n * IB + HL_TILE_UNITS * 16 - 1) / (HL_TILE_UNITS * 16);
    const u64 resident = (u64)ctas_per_sm * ctx->sm_count;
    TG_LAUNCH_T(ctx, TG_K_HLL, kern, (u32)(ntiles < resident ? ntiles : resident), HL_THREADS, smem, (const ulonglong2*)d_in, n, p,
                (u32)ntiles, regs);
    return TG_OK;
}

// one worker's registers into `regs` (2^p bytes and the flag byte, cleared here): a worker with no items launches nothing, a
// worker over the limit reads nothing and sets the flag
int worker_registers(tg_ctx* ctx, uint32_t ib, u32 p, const void* d_in, u64 n, u32* regs) {
    TG_CUDA(ctx, cudaMemsetAsync(regs, 0, slot_bytes(p), ctx->stream));
    if (n >= HLL_LIMIT) {
        TG_CUDA(ctx, cudaMemsetAsync((char*)regs + ((size_t)1 << p), 1, 1, ctx->stream));
        return TG_OK;
    }
    if (!n) return TG_OK;
    if (p <= HL_SHARED_MAX_P) return ib == 16 ? launch_update<16, true>(ctx, d_in, n, p, regs) : launch_update<8, true>(ctx, d_in, n, p, regs);
    return ib == 16 ? launch_update<16, false>(ctx, d_in, n, p, regs) : launch_update<8, false>(ctx, d_in, n, p, regs);
}

// the one host read: the merged registers and the flag byte behind them
int finish(tg_ctx* ctx, const char* what, u32 p, const u32* regs, uint8_t* out_registers) {
    const size_t m = (size_t)1 << p;
    uint8_t* h = (uint8_t*)ctx->pinned;
    TG_CUDA(ctx, cudaMemcpyAsync(h, regs, m + 1, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h[m]) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "%s: a worker holds 2^30 or more items (limit 2^30 - 1)", what);
    memcpy(out_registers, h, m);
    return TG_OK;
}

// p = 1: the update and one host read.  p > 1: one ncclAllReduce(max) over the register bytes and the flag byte (so every rank
// sees a worker over the limit, from the same collective), then the host read.
int hll_impl(tg_ctx* ctx, uint32_t ib, u32 p, const void* d_in, size_t n_local, uint8_t* out_registers) {
    if (ctx->nranks == 1 && n_local >= HLL_LIMIT)
        return tg_set_error(ctx, TG_ERR_TOO_LARGE, "hyperloglog: n_local=%zu (limit 2^30 - 1)", n_local);
    void* regs;
    TG_TRY(tg_ws_get(ctx, WS_HLL, slot_bytes(p), &regs));
    TG_TRY(worker_registers(ctx, ib, p, d_in, n_local, (u32*)regs));
    if (ctx->nranks > 1)
        TG_NCCL(ctx, ncclAllReduce(regs, regs, ((size_t)1 << p) + 1, ncclUint8, ncclMax, ctx->comm, ctx->stream));
    return finish(ctx, "hyperloglog", p, (const u32*)regs, out_registers);
}

// a host File goes up into the WS_IN staging buffer, a device File is read where it is
int stage_input(tg_ctx* ctx, const tg_merge_input* in, uint32_t item_bytes, const void** d_in, size_t* n) {
    if (in->dev) {
        if (in->dev->item_bytes != item_bytes || (!in->dev->dptr && in->dev->items))
            return tg_set_error(ctx, TG_ERR_ARG, "hyperloglog_file: the device File has item size %u, the call says %u",
                                in->dev->item_bytes, item_bytes);
        *d_in = in->dev->dptr;
        *n = in->dev->items;
        return TG_OK;
    }
    if (!in->blocks && in->nblocks) return tg_set_error(ctx, TG_ERR_ARG, "hyperloglog_file: the input has no blocks");
    size_t bytes = 0;
    for (size_t i = 0; i < in->nblocks; ++i) bytes += in->blocks[i].bytes;
    if (bytes % item_bytes) return tg_set_error(ctx, TG_ERR_ARG, "hyperloglog_file: %zu bytes is not a multiple of %u", bytes, item_bytes);
    *n = bytes / item_bytes;
    *d_in = nullptr;
    if (bytes && *n < HLL_LIMIT) {                      // (an input over the limit is only counted, never read)
        void* d;
        TG_TRY(tg_ws_get(ctx, WS_IN, bytes + 16, &d));
        TG_TRY(tg_upload_blocks(ctx, d, in->blocks, in->nblocks, nullptr));
        *d_in = d;
    }
    return TG_OK;
}

}  // namespace

extern "C" {

int tg_hyperloglog(tg_ctx* ctx, uint32_t item_bytes, uint32_t precision, const void* d_in, size_t n_local, uint8_t* out_registers) {
    if (!ctx || !out_registers || (!d_in && n_local)) return tg_set_error(ctx, TG_ERR_ARG, "hyperloglog: NULL argument");
    TG_TRY(check_args(ctx, "hyperloglog", item_bytes, precision));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return hll_impl(ctx, item_bytes, precision, d_in, n_local, out_registers);
}

int tg_hyperloglog_file(tg_ctx* ctx, uint32_t item_bytes, uint32_t precision, const tg_merge_input* in, uint8_t* out_registers) {
    if (!ctx || !in || !out_registers) return tg_set_error(ctx, TG_ERR_ARG, "hyperloglog_file: NULL argument");
    TG_TRY(check_args(ctx, "hyperloglog_file", item_bytes, precision));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* d_in;
    size_t n;
    TG_TRY(stage_input(ctx, in, item_bytes, &d_in, &n));
    return hll_impl(ctx, item_bytes, precision, d_in, n, out_registers);
}

int tg_hyperloglog_select(tg_ctx* ctx, uint32_t item_bytes, uint32_t precision, const void* const* d_shards, const size_t* n_shards,
                          uint32_t p_workers, uint8_t* out_registers) {
    if (!ctx || !d_shards || !n_shards || !out_registers || p_workers == 0 || p_workers > TG_MAX_RANKS)
        return tg_set_error(ctx, TG_ERR_ARG, "hyperloglog_select: p_workers=%u or a NULL argument", p_workers);
    TG_TRY(check_args(ctx, "hyperloglog_select", item_bytes, precision));
    for (uint32_t w = 0; w < p_workers; ++w) {
        if (!d_shards[w] && n_shards[w]) return tg_set_error(ctx, TG_ERR_ARG, "hyperloglog_select: shard %u is NULL", w);
        if (n_shards[w] >= HLL_LIMIT)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "hyperloglog_select: shard %u holds %zu items (limit 2^30 - 1)", w, n_shards[w]);
    }
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    // slot w is worker w's array, as the all-reduce would find it; one more slot takes their max
    const size_t slot = slot_bytes(precision);
    void* base;
    TG_TRY(tg_ws_get(ctx, WS_HLL, (p_workers + 1) * slot, &base));
    for (uint32_t w = 0; w < p_workers; ++w)
        TG_TRY(worker_registers(ctx, item_bytes, precision, d_shards[w], n_shards[w], (u32*)((char*)base + (w + 1) * slot)));
    const u32 words = (u32)(slot / 4);
    TG_LAUNCH_T(ctx, TG_K_HLL, hll_merge_kernel, (words + 255) / 256, 256, 0, (const u32*)((char*)base + slot), p_workers, words, words,
                (u32*)base);
    return finish(ctx, "hyperloglog_select", precision, (const u32*)base, out_registers);
}

}  // extern "C"
