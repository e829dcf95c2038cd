// tg_exchange.cu — exchange windows of the collective operators (see tg_exchange.cuh): allocation, mapping into the peers
// (CUDA IPC / peer access), the count matrix of one exchange and the destination pointers of its peer-store pass.
#include <stdlib.h>
#include <unistd.h>

#include "tg_exchange.cuh"

int tg_radix_sort_items(tg_ctx* ctx, const tg_key_desc* desc, void* d_items, void* d_tmp, size_t n, void** result);

namespace tgp {

namespace {

// what a rank publishes about its window (all-gathered through NCCL, 128 bytes per rank)
struct WinInfo {
    cudaIpcMemHandle_t handle;      // 64 bytes
    u64 ptr, cap, pid, host;
    int device, can_p2p, pad[2];
    char fill[16];
};
static_assert(sizeof(WinInfo) == 128, "WinInfo is exchanged as 128 raw bytes");

u64 host_hash() {
    char name[256] = { 0 };
    gethostname(name, sizeof(name) - 1);
    u64 h = 1469598103934665603ull;
    for (const char* c = name; *c; ++c) h = (h ^ (unsigned char)*c) * 1099511628211ull;
    // the boot id distinguishes containers that share a hostname
    if (FILE* f = fopen("/proc/sys/kernel/random/boot_id", "r")) {
        char b[64] = { 0 };
        if (fgets(b, sizeof(b), f)) for (const char* c = b; *c; ++c) h = (h ^ (unsigned char)*c) * 1099511628211ull;
        fclose(f);
    }
    return h;
}

// all-gather `bytes` host bytes per rank through the communicator (control plane of the window setup: rare)
int allgather_host(tg_ctx* ctx, const void* mine, void* all, size_t bytes) {
    char* d;
    TG_TRY(tg_ws_get(ctx, WS_XCTL, 1 << 17, (void**)&d));
    const int p = ctx->nranks;
    if (bytes * (size_t)(p + 1) > (1 << 15)) return tg_set_error(ctx, TG_ERR_ARG, "allgather_host: %zu bytes", bytes);
    TG_CUDA(ctx, cudaMemcpyAsync(d, mine, bytes, cudaMemcpyHostToDevice, ctx->stream));
    TG_NCCL(ctx, ncclAllGather(d, d + (1 << 15), bytes, ncclUint8, ctx->comm, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(all, d + (1 << 15), bytes * p, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return TG_OK;
}

void unmap_peers(tg_ctx* ctx) {
    for (int r = 0; r < TG_MAX_RANKS; ++r) {
        if (ctx->xwin.ipc_open[r] && ctx->xwin.peer[r]) cudaIpcCloseMemHandle(ctx->xwin.peer[r]);
        ctx->xwin.ipc_open[r] = false;
        ctx->xwin.peer[r] = nullptr;
    }
}

// (re)allocate this rank's window with `cap` bytes and map every peer's; decides the mode on first use.  Collective.
int remap(tg_ctx* ctx, size_t cap) {
    const int p = ctx->nranks, me = ctx->rank;
    tg_ctx::XWin& w = ctx->xwin;
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    // every rank unmaps its peers before anybody frees (the all-gather below is the barrier in between)
    unmap_peers(ctx);
    {
        u64 token = 0, all[TG_MAX_RANKS];
        TG_TRY(allgather_host(ctx, &token, all, 8));
    }
    if (w.base) { TG_CUDA(ctx, cudaFree(w.base)); w.base = nullptr; w.cap = 0; }
    cudaError_t e = cudaMalloc(&w.base, cap);
    if (e != cudaSuccess) { cudaGetLastError(); w.base = nullptr; }
    WinInfo mine;
    memset(&mine, 0, sizeof(mine));
    mine.ptr = (u64)(uintptr_t)w.base;
    mine.cap = w.base ? cap : 0;
    mine.pid = (u64)getpid();
    mine.host = host_hash();
    mine.device = ctx->device;
    mine.can_p2p = (w.mode != 0 && w.base) ? 1 : 0;
    if (mine.can_p2p && cudaIpcGetMemHandle(&mine.handle, w.base) != cudaSuccess) { cudaGetLastError(); mine.can_p2p = 0; }
    WinInfo all[TG_MAX_RANKS];
    TG_TRY(allgather_host(ctx, &mine, all, sizeof(WinInfo)));
    bool alloc_ok = true, p2p = w.mode != 0;
    for (int r = 0; r < p; ++r) { alloc_ok = alloc_ok && all[r].cap >= cap; p2p = p2p && all[r].can_p2p; }
    if (!alloc_ok) return tg_set_error(ctx, TG_ERR_OOM, "exchange window: a rank could not allocate %zu bytes", cap);   // (uniform)
    w.cap = cap;
    int ok = 1;
    if (p2p) {
        for (int r = 0; r < p && ok; ++r) {
            if (r == me) { w.peer[r] = w.base; continue; }
            if (all[r].host != mine.host) { ok = 0; break; }
            if (all[r].pid == mine.pid) {
                // a worker thread of this process (Thrill runs its workers as threads): the pointer is valid as it is
                int can = 0;
                if (cudaDeviceCanAccessPeer(&can, ctx->device, all[r].device) != cudaSuccess || !can) { cudaGetLastError(); ok = 0; break; }
                cudaError_t pe = cudaDeviceEnablePeerAccess(all[r].device, 0);
                if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); ok = 0; break; }
                cudaGetLastError();
                w.peer[r] = (void*)(uintptr_t)all[r].ptr;
            }
            else {
                void* q = nullptr;
                if (cudaIpcOpenMemHandle(&q, all[r].handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = 0; break; }
                w.peer[r] = q;
                w.ipc_open[r] = true;
            }
        }
    }
    else ok = 0;
    // the mode must be the same everywhere: P2P only if every rank mapped every peer
    u64 okw = (u64)ok, oks[TG_MAX_RANKS];
    TG_TRY(allgather_host(ctx, &okw, oks, 8));
    bool all_ok = true;
    for (int r = 0; r < p; ++r) all_ok = all_ok && oks[r] != 0;
    if (!all_ok) {
        unmap_peers(ctx);
        w.peer[me] = w.base;
    }
    if (w.mode < 0) {
        w.mode = all_ok ? 1 : 0;
        if (getenv("TG_DEBUG_EXCHANGE") && me == 0)
            fprintf(stderr, "[tg_exchange] %d ranks: %s\n", p, w.mode ? "P2P stores into mapped peer windows" : "NCCL send/recv (peers cannot be mapped)");
    }
    else if (w.mode == 1 && !all_ok)
        return tg_set_error(ctx, TG_ERR_CUDA, "exchange window: a peer window could not be mapped after growth");       // (uniform)
    return TG_OK;
}

}  // namespace

int xwin_negotiate(tg_ctx* ctx) {
    tg_ctx::XWin& w = ctx->xwin;
    if (w.mode >= 0) return TG_OK;
    const char* e = getenv("TG_EXCHANGE");
    if (e && !strcmp(e, "nccl")) w.mode = 0;
    return remap(ctx, (size_t)1 << 20);
}

int xwin_ensure(tg_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->xwin.cap) return TG_OK;          // (`bytes` is the maximum over all ranks: a uniform decision)
    return remap(ctx, bytes + (bytes >> 2) + ((size_t)1 << 20));
}

int xwin_barrier(tg_ctx* ctx) {
    u32* d;
    TG_TRY(tg_ws_get(ctx, WS_XCTL, 1 << 17, (void**)&d));
    d += (96 << 10) / 4;              // byte offset 96 KB of the control scratch
    TG_NCCL(ctx, ncclAllReduce(d, d + 64, 1, ncclUint32, ncclSum, ctx->comm, ctx->stream));
    return TG_OK;
}

// all-gather the p per-destination counts of every rank; fills send/recv counts; *need_bytes_max = largest receive size
// of any rank in bytes (plus slack for the 16-byte granule reads of the kernels that consume the window)
int xchg_counts(tg_ctx* ctx, const u32* d_totals, int item_bytes, XchgResult* res, u64* need_bytes_max) {
    const int p = ctx->nranks, me = ctx->rank;
    u32* d;
    TG_TRY(tg_ws_get(ctx, WS_XCTL, 1 << 17, (void**)&d));
    u32* d_mat = d + (1 << 14);           // byte offset 64 KB: p x p u32 (p <= 16: 1 KB)
    u32* h_mat = (u32*)ctx->pinned + 16384;     // byte offset 64 KB of the pinned scratch (the operators use the first 32 KB)
    TG_NCCL(ctx, ncclAllGather(d_totals, d_mat, p, ncclUint32, ctx->comm, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(h_mat, d_mat, (size_t)p * p * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    u64 worst = 0, before[TG_MAX_RANKS];
    tg_exchange_plan((u32)p, (u32)me, h_mat, (uint64_t*)res->send_cnt, (uint64_t*)res->recv_cnt, (uint64_t*)before, (uint64_t*)&res->n_recv, (uint64_t*)&worst);
    if (worst >= (1u << 30))          // the same verdict on every rank: nobody is left waiting in a collective
        return tg_set_error(ctx, TG_ERR_TOO_LARGE, "exchange: a worker would receive %llu items (limit 2^30 - 1)", (unsigned long long)worst);
    *need_bytes_max = (worst + 4) * (u64)item_bytes;
    return TG_OK;
}

const u32* xchg_matrix(tg_ctx* ctx) { return (const u32*)ctx->pinned + 16384; }

// destination pointers of the peer-store pass.  Bucket d of the local partition would start at gbase[d] = sum of the
// send counts below d; in worker d's window this worker's items start after those of the lower ranks.  dbase[d] is biased
// by -gbase[d] so that the pass can use the positions it computes for a local output.  Staged through the pinned scratch
// (byte offset 72 KB) into the control workspace (byte offset 80 KB): the next upload must wait for this one's copy.
int xchg_upload_dest(tg_ctx* ctx, const u32* counts, int p, int me, int item_bytes, void* const* windows, void*** d_dbase_out) {
    u64* h_ptr = (u64*)ctx->pinned + 9216;
    char* d;
    TG_TRY(tg_ws_get(ctx, WS_XCTL, 1 << 17, (void**)&d));
    void** d_dbase = (void**)(d + (80 << 10));
    u64 gbase = 0, before[TG_MAX_RANKS], sc[TG_MAX_RANKS], rc[TG_MAX_RANKS], nr, worst;
    tg_exchange_plan((u32)p, (u32)me, counts, (uint64_t*)sc, (uint64_t*)rc, (uint64_t*)before, (uint64_t*)&nr, (uint64_t*)&worst);
    for (int d = 0; d < PEER_MAX; ++d) {
        if (d >= p) { h_ptr[d] = 0; continue; }
        h_ptr[d] = (u64)(uintptr_t)windows[d] + (before[d] - gbase) * (u64)item_bytes;   // (64-bit: wraps like the pass's positions)
        gbase += sc[d];
    }
    TG_CUDA(ctx, cudaMemcpyAsync(d_dbase, h_ptr, PEER_MAX * sizeof(void*), cudaMemcpyHostToDevice, ctx->stream));
    *d_dbase_out = d_dbase;
    return TG_OK;
}

int xchg_transfer(tg_ctx* ctx, bool simulated, const void* d_part, size_t s, const u32* counts, int p, int me, void* const* windows) {
    u64 before[TG_MAX_RANKS], sc[TG_MAX_RANKS], rc[TG_MAX_RANKS], nr, worst;
    tg_exchange_plan((u32)p, (u32)me, counts, (uint64_t*)sc, (uint64_t*)rc, (uint64_t*)before, (uint64_t*)&nr, (uint64_t*)&worst);
    u64 soff = 0, roff = 0;
    if (simulated) {
        // what ncclSend(segment d) / ncclRecv on worker d put there: the same bytes at the same place of worker d's window
        for (int d = 0; d < p; ++d) {
            if (sc[d]) TG_CUDA(ctx, cudaMemcpyAsync((char*)windows[d] + before[d] * s, (const char*)d_part + soff * s, sc[d] * s,
                                                    cudaMemcpyDeviceToDevice, ctx->stream));
            soff += sc[d];
        }
        return TG_OK;
    }
    TG_NCCL(ctx, ncclGroupStart());
    for (int r = 0; r < p; ++r) {
        if (sc[r]) TG_NCCL(ctx, ncclSend((const char*)d_part + soff * s, sc[r] * s, ncclUint8, r, ctx->comm, ctx->stream));
        if (rc[r]) TG_NCCL(ctx, ncclRecv((char*)ctx->xwin.base + roff * s, rc[r] * s, ncclUint8, r, ctx->comm, ctx->stream));
        soff += sc[r];
        roff += rc[r];
    }
    TG_NCCL(ctx, ncclGroupEnd());
    return TG_OK;
}

int evacuate_window_inputs(tg_ctx* ctx, const void** in, const size_t* bytes, uint32_t k) {
    const char* b = (const char*)ctx->xwin.base;
    if (!b) return TG_OK;
    const char *lo = nullptr, *hi = nullptr;
    for (uint32_t j = 0; j < k; ++j) {
        const char* q = (const char*)in[j];
        if (!bytes[j] || q < b || q >= b + ctx->xwin.cap) continue;
        if (!lo || q < lo) lo = q;
        if (!hi || q + bytes[j] > hi) hi = q + bytes[j];
    }
    if (!lo) return TG_OK;
    char* d;
    TG_TRY(tg_ws_get(ctx, WS_AUX, (size_t)(hi - lo) + 16, (void**)&d));
    TG_CUDA(ctx, cudaMemcpyAsync(d, lo, (size_t)(hi - lo), cudaMemcpyDeviceToDevice, ctx->stream));
    for (uint32_t j = 0; j < k; ++j) {
        const char* q = (const char*)in[j];
        if (bytes[j] && q >= lo && q < hi) in[j] = d + (q - lo);
    }
    return TG_OK;
}

int sort_pairs_into(tg_ctx* ctx, int slot, const void* src, u64 n, const ulonglong2** sorted) {
    ulonglong2* buf;
    TG_TRY(tg_ws_get(ctx, slot, (2 * n + 2) * 16, (void**)&buf));
    if (n) TG_CUDA(ctx, cudaMemcpyAsync(buf, src, n * 16, cudaMemcpyDeviceToDevice, ctx->stream));
    const tg_key_desc sd = { 16, 0, 8, TG_KEY_UINT_LE, 0, 1 };
    void* res = buf;
    TG_TRY(tg_radix_sort_items(ctx, &sd, buf, buf + n + 1, n, &res));
    *sorted = (const ulonglong2*)res;
    return TG_OK;
}

void xwin_release(tg_ctx* ctx) {
    unmap_peers(ctx);
    if (ctx->xwin.base) cudaFree(ctx->xwin.base);
    ctx->xwin = tg_ctx::XWin();
}

}  // namespace tgp

extern "C" int tg_exchange_plan(uint32_t p, uint32_t me, const uint32_t* counts, uint64_t* send_cnt, uint64_t* recv_cnt,
                                uint64_t* recv_before, uint64_t* n_recv, uint64_t* worst) {
    if (p == 0 || p > TG_MAX_RANKS || me >= p || !counts) return TG_ERR_ARG;
    u64 w = 0, nr = 0;
    for (u32 dst = 0; dst < p; ++dst) {
        u64 tot = 0, before = 0;
        for (u32 src = 0; src < p; ++src) {
            if (src < me) before += counts[src * p + dst];
            tot += counts[src * p + dst];
        }
        if (tot > w) w = tot;
        if (recv_before) recv_before[dst] = before;
        if (send_cnt) send_cnt[dst] = counts[me * p + dst];
        if (recv_cnt) recv_cnt[dst] = counts[dst * p + me];
        nr += counts[dst * p + me];
    }
    if (n_recv) *n_recv = nr;
    if (worst) *worst = w;
    return TG_OK;
}
