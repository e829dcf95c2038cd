// tg_common.cuh — shared declarations of libthrill_gpu.so (sm_90a only; no other target is built)
#pragma once

#include <cuda_runtime.h>
#include <nccl.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <vector>

#include "../../include/thrill_gpu.h"

typedef unsigned long long u64;
typedef unsigned int u32;

#define TG_NUM_WS 37
#define TG_MAX_RANKS 16

struct tg_ctx {
    int device = 0, rank = 0, nranks = 1;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    ncclComm_t comm = nullptr;
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
    char err[512] = { 0 };
    uint64_t launches = 0;
    std::map<void*, size_t> allocs;             // tg_alloc'd buffers
    void* ws[TG_NUM_WS] = { nullptr };          // cached workspaces, grown on demand
    size_t ws_bytes[TG_NUM_WS] = { 0 };
    void* pinned = nullptr;                     // small pinned staging area (control-plane scalars)
    size_t pinned_bytes = 0;
    void* pinned_list[2] = { nullptr, nullptr };       // pinned staging of host-built tile / unit lists (tg_pinned_list)
    size_t pinned_list_bytes[2] = { 0, 0 };
    // per-device kernel attributes already applied by this ctx (cudaFuncSetAttribute is per device, and one
    // process may drive several GPUs: Thrill runs its workers as threads): kernel -> resident CTAs per SM
    std::map<const void*, int> kernel_cfg;
    // prefix sort (tg_radix_sort.cu): sorts to skip after a failed attempt, and how often it fell back
    int prefix_sort_penalty = 0;
    int prefix_spec_penalty = 0;               // ... after the speculative fast path guessed the wrong top digit
    uint64_t prefix_sort_fallbacks = 0;
    // optional per-kernel-class timing (tg_profile_*)
    bool profile = false;
    struct ProfEv { int cls; cudaEvent_t a, b; };
    std::vector<ProfEv> prof_events;
    std::vector<cudaEvent_t> prof_pool;
    // exchange window (tg_exchange.cu): the buffer the peers of a collective operator store this worker's share of the
    // Alltoallv into, directly over NVLink (P2P stores from the partition kernel).  peer[r] = rank r's window as mapped
    // into this process (CUDA IPC between processes, the raw pointer + peer access between worker threads of one process).
    struct XWin {
        void* base = nullptr;
        size_t cap = 0;                        // bytes; the same on every rank (grown collectively)
        void* peer[TG_MAX_RANKS] = { nullptr };
        bool ipc_open[TG_MAX_RANKS] = { false };
        int mode = -1;                         // -1 not negotiated yet, 0 = NCCL send/recv, 1 = P2P stores
    } xwin;
    uint64_t hot_records = 0;                    // records folded by the counting reads of the aggregations (tg_hot_records)
    uint64_t bytes_h2d = 0, bytes_d2h = 0;       // through tg_upload(_blocks) / tg_download(_blocks)
    int spec_top_bit = 64;                     // prefix sort: expected position of the most significant varying key bit
    // result of the last *_file operator, fetched by tg_fetch_output
    void* out_ptr = nullptr;
    size_t out_items = 0;
    uint32_t out_item_bytes = 0;
};

// workspace slots
enum { WS_SORT_TMP = 0, WS_SORT_STATUS = 1, WS_SORT_HIST = 2, WS_XCHG_SEND = 3, WS_XCHG_RECV = 4,
       WS_MISC = 5, WS_TABLE = 6, WS_OUT = 7, WS_IN = 8, WS_AUX = 9, WS_AUX2 = 10, WS_SAMPLES = 11,
       WS_SEG_TILES = 12, WS_SEG_TABLES = 13, WS_SORT_STATUS2 = 14,
       WS_SORT_HIST2 = 15, WS_SEG_TILES2 = 16, WS_DENSE = 17, WS_XCTL = 18, WS_REC = 19, WS_HOT = 20,
       // InnerJoin (tg_join.cu): the sorted sides (items + sort scratch each), counts / offsets / splits, the output.
       // GroupByKey / GroupToIndex (tg_group.cu) sort into WS_JOIN_L: their result is the sorted items
       WS_JOIN_L = 21, WS_JOIN_R = 22, WS_JOIN_AUX = 23, WS_JOIN_OUT = 24,
       // PrefixSum / ExPrefixSum / ZipWithIndex (tg_scan.cu): tile aggregates, prefixes and the gathered records; the output
       WS_SCAN_AUX = 25, WS_SCAN_OUT = 26,
       // HyperLogLog (tg_hll.cu): the worker's registers (one array per simulated worker in _select)
       WS_HLL = 27,
       // Window (tg_window.cu): the all-gathered records and the halo; the output
       WS_WIN_AUX = 28, WS_WIN_OUT = 29,
       // Sample / BernoulliSample (tg_sample.cu): histogram, selection state, records and tile counts; the candidate keys; the output
       WS_SAMPLE_AUX = 30, WS_SAMPLE_CAND = 31, WS_SAMPLE_OUT = 32,
       // InnerJoin on records (tg_join.cu): p > 1, the left side's received records, out of the exchange window's way; an input
       // that lies in a slot the join writes (an un-detached join or GroupByKey result), copied out of the way (left, right)
       WS_JOIN_LREC = 33, WS_JOIN_IN_L = 34, WS_JOIN_IN_R = 35,
       // radix sort (tg_radix_sort.cu): one bit per item, the group heads claimed by the fused finishing pass's repair kernel
       WS_FINISH = 36 };

int tg_set_error(tg_ctx* ctx, int status, const char* fmt, ...);
int tg_ws_get(tg_ctx* ctx, int slot, size_t bytes, void** out);
int tg_pinned_list(tg_ctx* ctx, int which, size_t bytes, void** out);      // two buffers, grown on demand, owned by the ctx

#define TG_CUDA(ctx, call)                                                                         \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
            return tg_set_error((ctx), TG_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call,   \
                                cudaGetErrorString(e_));                                           \
    } while (0)

#define TG_NCCL(ctx, call)                                                                         \
    do {                                                                                           \
        ncclResult_t r_ = (call);                                                                  \
        if (r_ != ncclSuccess)                                                                     \
            return tg_set_error((ctx), TG_ERR_NCCL, "%s:%d %s -> %s", __FILE__, __LINE__, #call,   \
                                ncclGetErrorString(r_));                                           \
    } while (0)

#define TG_TRY(call)                      \
    do {                                  \
        int s_ = (call);                  \
        if (s_ != TG_OK) return s_;       \
    } while (0)

int tg_prof_begin(tg_ctx* ctx, int cls);
void tg_prof_end(tg_ctx* ctx, int slot);

// every kernel launch goes through these so tg_launch_count() is honest; TG_LAUNCH_T also times the
// launch with CUDA events when profiling is enabled
#define TG_LAUNCH(ctx, kernel, grid, block, smem, ...) TG_LAUNCH_T(ctx, TG_K_OTHER, kernel, grid, block, smem, __VA_ARGS__)
#define TG_LAUNCH_T(ctx, cls, kernel, grid, block, smem, ...)                                      \
    do {                                                                                           \
        int ps_ = (ctx)->profile ? tg_prof_begin((ctx), (cls)) : -1;                               \
        kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);                           \
        if (ps_ >= 0) tg_prof_end((ctx), ps_);                                                     \
        (ctx)->launches++;                                                                         \
        cudaError_t e_ = cudaGetLastError();                                                       \
        if (e_ != cudaSuccess)                                                                     \
            return tg_set_error((ctx), TG_ERR_CUDA, "%s:%d launch %s -> %s", __FILE__, __LINE__,   \
                                #kernel, cudaGetErrorString(e_));                                  \
    } while (0)

// ---- device helpers -------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ u32 smem_u32(const void* p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ u32 lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ u32 lanemask_lt() {
    u32 m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}
__device__ __forceinline__ u64 splitmix64_dev(u64 x) {
    x += 0x9E3779B97F4A7C15ull;
    u64 z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
// common/hash.hpp:64-73
__device__ __forceinline__ u64 hash128to64_dev(u64 upper, u64 lower) {
    const u64 k = 0x9DDFEA08EB382D69ull;
    u64 a = (lower ^ upper) * k;
    a ^= (a >> 47);
    u64 b = (upper ^ a) * k;
    b ^= (b >> 47);
    b *= k;
    return b;
}

// mbarrier + 1-D bulk async copy (TMA unit, SASS UBLKCP)
__device__ __forceinline__ void mbar_init(u64* bar, u32 count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(u64* bar, u32 bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(u64* bar, u32 parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, u32 bytes, u64* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ u32 ld_relaxed_u32(const u32* p) {
    u32 v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u32(u32* p, u32 v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
#endif
