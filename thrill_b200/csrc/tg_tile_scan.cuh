// tg_tile_scan.cuh — the exclusive scan of per-tile u64 counts shared by InnerJoin (tg_join.cu: match counts) and Sample /
// BernoulliSample (tg_sample.cu: kept items per tile)
#pragma once

#include "tg_common.cuh"

namespace {

constexpr int JS_THREADS = 1024;      // the one-CTA scan of the tile sums

// exclusive scan of one u64 per thread over the CTA; *total = the sum.  warp_tot: NT / 32 words of shared memory.
template <int NT>
__device__ __forceinline__ u64 block_excl_scan_u64(u64 v, u64* warp_tot, u64* total) {
    const u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    u64 x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const u64 y = __shfl_up_sync(0xffffffffu, x, o);
        if ((int)lane >= o) x += y;
    }
    if (lane == 31) warp_tot[w] = x;
    __syncthreads();
    if (w == 0) {
        u64 t = lane < NT / 32 ? warp_tot[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const u64 y = __shfl_up_sync(0xffffffffu, t, o);
            if ((int)lane >= o) t += y;
        }
        if (lane < NT / 32) warp_tot[lane] = t;
    }
    __syncthreads();
    const u64 before = w ? warp_tot[w - 1] : 0;
    *total = warp_tot[NT / 32 - 1];
    __syncthreads();                       // (warp_tot is reused by the next call)
    return before + x - v;
}

// exclusive scan of the nt tile sums (one CTA: thread t scans a contiguous run of tiles); *d_total = the sum of all
__global__ void __launch_bounds__(JS_THREADS)
join_scan_tiles_kernel(const u64* __restrict__ tile_sum, u32 nt, u64* __restrict__ tile_base, u64* __restrict__ d_total) {
    __shared__ u64 warp_tot[JS_THREADS / 32];
    const u32 per = (nt + JS_THREADS - 1) / JS_THREADS;
    const u32 t0 = min(threadIdx.x * per, nt), t1 = min(t0 + per, nt);
    u64 s = 0;
    for (u32 t = t0; t < t1; ++t) s += tile_sum[t];
    u64 tot;
    u64 base = block_excl_scan_u64<JS_THREADS>(s, warp_tot, &tot);
    for (u32 t = t0; t < t1; ++t) {
        tile_base[t] = base;
        base += tile_sum[t];
    }
    if (threadIdx.x == 0) *d_total = tot;
}

}  // namespace
