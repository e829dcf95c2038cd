// tg_group.cu — the device half of GroupByKey (api/group_by_key.hpp:46-377) and GroupToIndex (api/group_to_index.hpp:36-255)
// on DIAs of 16-byte (u64 key, 8-byte value) pairs grouped by the key.  The reference's nodes do their work in two halves: MainOp
// exchanges the items to the key's owner and sorts each worker's share by the key (:348-376, :234-254); PushData walks the
// sorted items and calls the user's group function once per group (:204-331, :116-215).  The first half runs here, per worker:
//   1. p > 1: one exchange_scatter<2, DigitFn> to the owner: ModDigit (key % p) for GroupByKey, RangeDigit (k * p / size, the
//      range partition of ReduceToIndex) for GroupToIndex
//   2. the stable local radix sort of the received items by the key (the sort behind tg_radix_sort_local)
// The second half, with the arbitrary group function and output type, stays on the host (GpuGroupNode, thrill_gpu_nodes.hpp).
// The result is ordered by (key, global position): the exchange and the sort are stable.  The input is read, never modified.
// GroupToIndex: an index >= result_size is TG_ERR_ARG on every rank: such items sort last on the last worker, one kernel reads
// the last key, and with p > 1 an all-reduce of that verdict reaches every rank.
#include "tg_exchange.cuh"

using namespace tgp;

namespace {

constexpr u64 GROUP_LIMIT = 1ull << 30;

// *bad = 1 if the largest key of the sorted items is not below size
__global__ void group_index_check_kernel(const ulonglong2* __restrict__ sorted, u64 n, u64 size, u32* __restrict__ bad) {
    *bad = n && sorted[n - 1].x >= size ? 1u : 0u;
}

int group_impl(tg_ctx* ctx, const void* d_in, size_t n_local, bool to_index, u64 result_size, void** out_dptr, size_t* out_n) {
    const int p = ctx->nranks;
    const char* what = to_index ? "group_to_index" : "group_by_key";
    const ulonglong2* sorted;
    u64 n;
    if (p == 1) {
        if (n_local >= GROUP_LIMIT)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "%s: n_local=%zu (limit 2^30 - 1)", what, n_local);
        n = n_local;
        TG_TRY(sort_pairs_into(ctx, WS_JOIN_L, d_in, n, &sorted));
    }
    else {
        // (an input inside the exchange window is moved out of the peers' way first; n_local >= 2^30 is reported to every
        // rank by the exchange's count matrix)
        const void* in[1] = { d_in };
        const size_t bytes[1] = { n_local < GROUP_LIMIT ? n_local * 16 : 0 };
        TG_TRY(xwin_negotiate(ctx));
        TG_TRY(evacuate_window_inputs(ctx, in, bytes, 1));
        if (to_index) TG_TRY(exchange_sort_pairs(ctx, WS_JOIN_L, in[0], n_local, RangeDigit{ result_size, (u32)p }, &sorted, &n));
        else TG_TRY(exchange_sort_pairs(ctx, WS_JOIN_L, in[0], n_local, ModDigit::make((u32)p), &sorted, &n));
    }
    if (to_index && (p > 1 || n)) {
        u32* d_bad;
        TG_TRY(tg_ws_get(ctx, WS_MISC, 1 << 16, (void**)&d_bad));
        d_bad += 12288;       // (48 KB into the scratch: behind the cursors of get_scratch at 32 KB)
        TG_LAUNCH(ctx, group_index_check_kernel, 1, 1, 0, sorted, n, result_size, d_bad);
        if (p > 1) TG_NCCL(ctx, ncclAllReduce(d_bad, d_bad, 1, ncclUint32, ncclMax, ctx->comm, ctx->stream));
        u32* hb = (u32*)ctx->pinned;
        TG_CUDA(ctx, cudaMemcpyAsync(hb, d_bad, 4, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (*hb) return tg_set_error(ctx, TG_ERR_ARG, "group_to_index: an index is not below result_size=%llu", (unsigned long long)result_size);
    }
    *out_dptr = (void*)sorted;
    *out_n = (size_t)n;
    return TG_OK;
}

int check_result_size(tg_ctx* ctx, u64 result_size) {
    const u64 p = (u64)ctx->nranks;
    if (result_size && result_size - 1 > ~0ull / p)
        return tg_set_error(ctx, TG_ERR_ARG, "group_to_index: k * p overflows for result_size=%llu", (unsigned long long)result_size);
    return TG_OK;
}

int check_ranks(tg_ctx* ctx) {
    if (ctx->nranks > TG_MAX_RANKS) return tg_set_error(ctx, TG_ERR_ARG, "group: at most 16 ranks");
    return TG_OK;
}

// a host File goes up into the WS_IN staging buffer, a device File is read where it is
int stage_input(tg_ctx* ctx, const tg_merge_input* in, const void** d_in, size_t* n) {
    if (in->dev) {
        if (in->dev->item_bytes != 16 || (!in->dev->dptr && in->dev->items))
            return tg_set_error(ctx, TG_ERR_ARG, "group_file: the device File has item size %u, the operator takes 16", in->dev->item_bytes);
        *d_in = in->dev->dptr;
        *n = in->dev->items;
        return TG_OK;
    }
    if (!in->blocks && in->nblocks) return tg_set_error(ctx, TG_ERR_ARG, "group_file: the input has no blocks");
    size_t bytes = 0;
    for (size_t i = 0; i < in->nblocks; ++i) bytes += in->blocks[i].bytes;
    if (bytes % 16) return tg_set_error(ctx, TG_ERR_ARG, "group_file: %zu bytes is not a multiple of 16", bytes);
    *n = bytes / 16;
    *d_in = nullptr;
    if (bytes) {
        void* d;
        TG_TRY(tg_ws_get(ctx, WS_IN, bytes + 16, &d));
        TG_TRY(tg_upload_blocks(ctx, d, in->blocks, in->nblocks, nullptr));
        *d_in = d;
    }
    return TG_OK;
}

}  // namespace

extern "C" {

int tg_group_by_key(tg_ctx* ctx, const void* d_in, size_t n_local, void** out_dptr, size_t* out_n) {
    if (!ctx || !out_dptr || !out_n || (!d_in && n_local)) return tg_set_error(ctx, TG_ERR_ARG, "group_by_key: NULL argument");
    TG_TRY(check_ranks(ctx));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return group_impl(ctx, d_in, n_local, false, 0, out_dptr, out_n);
}

int tg_group_by_key_file(tg_ctx* ctx, const tg_merge_input* in, size_t* out_items) {
    if (!ctx || !in || !out_items) return tg_set_error(ctx, TG_ERR_ARG, "group_by_key_file: NULL argument");
    TG_TRY(check_ranks(ctx));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* d_in;
    size_t n;
    TG_TRY(stage_input(ctx, in, &d_in, &n));
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(group_impl(ctx, d_in, n, false, 0, &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = 16;
    *out_items = n_out;
    return TG_OK;
}

int tg_group_to_index(tg_ctx* ctx, const void* d_in, size_t n_local, uint64_t result_size, void** out_dptr, size_t* out_n,
                      uint64_t* out_begin, uint64_t* out_end) {
    if (!ctx || !out_dptr || !out_n || !out_begin || !out_end || (!d_in && n_local))
        return tg_set_error(ctx, TG_ERR_ARG, "group_to_index: NULL argument");
    TG_TRY(check_ranks(ctx));
    TG_TRY(check_result_size(ctx, result_size));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    TG_TRY(group_impl(ctx, d_in, n_local, true, result_size, out_dptr, out_n));
    *out_begin = range_begin(ctx->rank, result_size, ctx->nranks);
    *out_end = range_begin(ctx->rank + 1, result_size, ctx->nranks);
    return TG_OK;
}

int tg_group_to_index_file(tg_ctx* ctx, const tg_merge_input* in, uint64_t result_size, size_t* out_items,
                           uint64_t* out_begin, uint64_t* out_end) {
    if (!ctx || !in || !out_items || !out_begin || !out_end) return tg_set_error(ctx, TG_ERR_ARG, "group_to_index_file: NULL argument");
    TG_TRY(check_ranks(ctx));
    TG_TRY(check_result_size(ctx, result_size));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* d_in;
    size_t n;
    TG_TRY(stage_input(ctx, in, &d_in, &n));
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(group_impl(ctx, d_in, n, true, result_size, &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = 16;
    *out_items = n_out;
    *out_begin = range_begin(ctx->rank, result_size, ctx->nranks);
    *out_end = range_begin(ctx->rank + 1, result_size, ctx->nranks);
    return TG_OK;
}

}  // extern "C"
