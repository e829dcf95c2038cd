// tg_window.cu — Window (OverlapWindowNode, api/window.hpp:140-246; DisjointWindowNode, :387-503) with the closed set of fold
// functions of tg_fold.cuh: every output is the left fold of k consecutive items (or of the trailing ones) by global position.
//
// Van Herk / Gil-Werman: the global sequence is cut into blocks of k items starting at multiples of k from position 0.  Within a
// block, P_o is the fold of the block's items up to o and S_o the fold from o to the block's end (operands kept in order:
// x_o + (x_{o+1} + ...)).  Then every output is one combine, whatever k is:
//   the overlapping window [i, i+k-1]      S_i + P_{i+k-1}, or S_i alone when i starts a block
//   a disjoint block                       S at the block's start
//   a partial suffix [j, N-1]              S_j (the block cut at N-1), + P_{N-1} when N-1 lies in the next block
// In-block folds: a block is cut into runs of R items from its start (R = max(16, 2^ceil(ceil(log2 k) / 2)), J = ceil(k / R)
// runs).  Each run is folded sequentially (its aggregate A_j), the aggregates are folded sequentially per block (E_j = A_0 + ...
// + A_{j-1} left to right, F_j = A_{j+1} + (... + A_{J-1}) right to left), and then P_o = E_j + (run prefix to o), S_o = (run
// suffix from o) + F_j.  The bracketing of a double sum is a function of global positions and k only: the same bits for every
// sharding, worker count and placement.  A summand goes through at most D = min(k - 1, R + J - 1) additions
// (include/thrill_gpu.h states the bound).
//
// window_kernel: a CTA owns m = max(1, 4096 / k) whole blocks; it stages them (and the following block, whose P its windows
// need) in shared memory, reading global position g from the halo when g < f_r and from the input otherwise (the input is never
// copied).  Reads (1 + 1/m) x s B per item, writes s B per output (s / k for disjoint windows).
// The halo is the k - 1 items before the worker's first: with p > 1 each worker all-gathers a record of its size and its last
// min(n, k - 1) items, and copies the halo out of the predecessors' records (several when they hold fewer than k - 1 items:
// FlowControlChannel::Predecessor, net/flow_control_channel.hpp:712-763).
#include "tg_common.cuh"
#include "tg_fold.cuh"

namespace {

constexpr u64 WIN_LIMIT = 1ull << 30;
constexpr u32 WIN_MAX_K = 4096;
constexpr int WN_THREADS = 256;
constexpr u32 WN_TILE = 4096;                   // items of a CTA's own blocks when k <= 2048 (32 KB of 8-byte values)
constexpr u32 WN_MAX_RUNS = 512;                // (m + 1) * J for J >= 2: at most 482 (k = 17)
// staged values and prefixes: 2 x (8192 + 8192 / 64 + 1) words at k = 4096
constexpr size_t WN_MAX_SMEM = 2 * (2 * WIN_MAX_K + 2 * WIN_MAX_K / 64 + 1) * 8;

struct WinArgs {
    const void* in;             // the worker's n items: global positions [f, f + n)
    const void* halo;           // global positions [lo, f)
    void* out;
    u64 f, n, lo, N;
    u64 b0;                     // the first block of CTA 0
    u64 out_extra;              // partial suffixes on the last worker: the output index of the first
    u32 k, m, R, logR, J;
    int last;                   // rank p - 1
};

__device__ __forceinline__ bool is_nan_bits(u64 x) { return (x & 0x7fffffffffffffffull) > 0x7ff0000000000000ull; }

// the item at global position g, lo <= g < f + n (an 8-byte item in .y)
template <int IB>
__device__ __forceinline__ ulonglong2 item_at(const WinArgs& a, u64 g) {
    const char* p = g < a.f ? (const char*)a.halo + (g - a.lo) * IB : (const char*)a.in + (g - a.f) * IB;
    if (IB == 16) return *(const ulonglong2*)p;
    return make_ulonglong2(0, *(const u64*)p);
}

template <int IB>
__device__ __forceinline__ void store_out(const WinArgs& a, u64 o, u64 first, u64 value) {
    if (IB == 16) ((ulonglong2*)a.out)[o] = make_ulonglong2(first, value);
    else ((u64*)a.out)[o] = value;
}

// The output of a window starting at i with its stored S_i: for Min / Max on doubles the stock fold keeps a NaN first item (S_i
// holds it then), otherwise the NaN-skipping fold is the stock one
template <int OP>
__device__ __forceinline__ u64 finish(u64 s, u64 p) {
    if (in_order<OP>() && is_nan_bits(s)) return s;
    return combine<OP>(s, p);
}

template <int OP, int IB, int MODE>
__global__ void __launch_bounds__(WN_THREADS) window_kernel(const WinArgs a) {
    extern __shared__ __align__(16) u64 wsm[];
    __shared__ u64 agg[WN_MAX_RUNS], epre[WN_MAX_RUNS], esuf[WN_MAX_RUNS];
    constexpr bool DISJ = MODE == TG_WINDOW_DISJOINT;
    const u32 k = a.k, R = a.R, J = a.J, lr = a.logR;
    const u32 own = a.m * k;
    const u32 Q = own + (DISJ ? 0 : k);
    // one padding word per run of R words, so that the lanes walking their runs hit distinct banks
    u64* v = wsm;
    u64* pre = wsm + Q + (Q >> lr) + 1;
#define WIDX(q) ((q) + ((q) >> lr))
    const u64 s0 = (a.b0 + (u64)blockIdx.x * a.m) * k;
    const u64 L = a.f + a.n;
    for (u32 q = threadIdx.x; q < Q; q += WN_THREADS) {
        const u64 g = s0 + q;
        v[WIDX(q)] = g >= a.lo && g < L ? item_at<IB>(a, g).y : ident<OP>();
    }
    __syncthreads();
    const u32 nblk = Q / k, nruns = nblk * J;
    if (J > 1) {
        for (u32 r = threadIdx.x; r < nruns; r += WN_THREADS) {
            const u32 j = r % J, q0 = (r / J) * k + j * R, len = min(R, k - j * R);
            if (DISJ && j == 0) continue;
            u64 acc = v[WIDX(q0)];
            for (u32 q = q0 + 1; q < q0 + len; ++q) acc = combine<OP>(acc, v[WIDX(q)]);
            agg[r] = acc;
        }
        __syncthreads();
        for (u32 b = threadIdx.x; b < nblk; b += WN_THREADS) {
            const u32 r0 = b * J;
            if (!DISJ) {
                u64 e = agg[r0];
                epre[r0 + 1] = e;
                for (u32 j = 2; j < J; ++j) { e = combine<OP>(e, agg[r0 + j - 1]); epre[r0 + j] = e; }
            }
            u64 s = agg[r0 + J - 1];
            esuf[r0 + J - 2] = s;
            if (DISJ) { for (u32 j = J - 2; j >= 1; --j) s = combine<OP>(agg[r0 + j], s); esuf[r0] = s; }
            else for (u32 j = J - 2; j >= 1; --j) { s = combine<OP>(agg[r0 + j], s); esuf[r0 + j - 1] = s; }
        }
        __syncthreads();
    }
    // P (not for disjoint windows) and S of every staged position, each run by one thread; S overwrites the values
    for (u32 r = threadIdx.x; r < nruns; r += WN_THREADS) {
        const u32 j = r % J, q0 = (r / J) * k + j * R, len = min(R, k - j * R);
        if (DISJ && j != 0) continue;
        if (!DISJ) {
            u64 acc = v[WIDX(q0)];
            pre[WIDX(q0)] = j ? combine<OP>(epre[r], acc) : acc;
            for (u32 q = q0 + 1; q < q0 + len; ++q) {
                acc = combine<OP>(acc, v[WIDX(q)]);
                pre[WIDX(q)] = j ? combine<OP>(epre[r], acc) : acc;
            }
        }
        u64 acc = 0;
        for (u32 t = len; t-- > 0;) {
            const u32 q = q0 + t;
            const u64 x = v[WIDX(q)];
            acc = t == len - 1 ? x : combine<OP>(x, acc);
            u64 s = j + 1 < J ? combine<OP>(acc, esuf[r]) : acc;
            if (in_order<OP>() && is_nan_bits(x)) s = x;
            v[WIDX(q)] = s;
        }
    }
    __syncthreads();
    const u64 own_end = s0 + own;
    if (!DISJ) {
        // the full windows starting in the CTA's blocks: output i - lo
        const u64 i_lo = s0 > a.lo ? s0 : a.lo;
        const u64 i_hi = L >= k ? (own_end < L - k + 1 ? own_end : L - k + 1) : 0;
        for (u64 i = i_lo + threadIdx.x; i < i_hi; i += WN_THREADS) {
            const u32 q = (u32)(i - s0);
            u64 s = v[WIDX(q)];
            if (q % k) s = finish<OP>(s, pre[WIDX(q + k - 1)]);
            store_out<IB>(a, i - a.lo, IB == 16 ? item_at<IB>(a, i + k - 1).x : 0, s);
        }
        if (MODE == TG_WINDOW_PARTIAL && a.last) {
            // the suffixes [j, N-1], j = max(0, N-k+1) ... N-1, after the full windows
            const u64 N = a.N, j0 = N + 1 >= k ? N + 1 - k : 0;
            const u64 jl = s0 > j0 ? s0 : j0, jh = own_end < N ? own_end : N;
            const u64 first = IB == 16 && jl < jh ? item_at<IB>(a, N - 1).x : 0;
            for (u64 j = jl + threadIdx.x; j < jh; j += WN_THREADS) {
                const u32 q = (u32)(j - s0);
                u64 s = v[WIDX(q)];
                if ((N - 1) / k != j / k) s = finish<OP>(s, pre[WIDX((u32)(N - 1 - s0))]);
                store_out<IB>(a, a.out_extra + (j - j0), first, s);
            }
        }
    }
    else {
        // block b's output goes to the worker that holds its last item, output b - floor(f / k); the trailing N mod k items to
        // the last worker
        for (u32 bl = threadIdx.x; bl < a.m; bl += WN_THREADS) {
            const u64 bs = s0 + (u64)bl * k, g = bs + k - 1;
            const bool full = g >= a.f && g < L;
            const bool trail = a.last && a.N % k && bs == a.N - a.N % k;
            if (!full && !trail) continue;
            store_out<IB>(a, bs / k - a.f / k, IB == 16 ? item_at<IB>(a, full ? g : a.N - 1).x : 0, v[WIDX(bl * k)]);
        }
    }
#undef WIDX
}

// ---- host side ---------------------------------------------------------------------------------------------------------------

// the outputs of a worker holding [f, f + n) of N items
u64 out_count(u32 mode, u64 k, u64 f, u64 n, u64 N, bool last) {
    const u64 L = f + n;
    if (mode == TG_WINDOW_DISJOINT) return L / k - f / k + (last && N % k ? 1 : 0);
    const u64 start = f > k - 1 ? f : k - 1;
    u64 c = L > start ? L - start : 0;
    if (mode == TG_WINDOW_PARTIAL && last) c += N < k - 1 ? N : k - 1;
    return c;
}

// all-gathered record: n, then the worker's last min(n, k - 1) items
size_t rec_bytes(u32 k, u32 ib) { return (16 + (size_t)(k - 1) * ib + 15) & ~(size_t)15; }

int check_args(tg_ctx* ctx, const char* what, const tg_scan_desc* desc, uint32_t k, uint32_t mode) {
    if (!desc) return tg_set_error(ctx, TG_ERR_ARG, "%s: NULL descriptor", what);
    if (desc->item_bytes != 8 && desc->item_bytes != 16)
        return tg_set_error(ctx, TG_ERR_ARG, "%s: %u-byte items (8: uint64_t / double, 16: pair<uint64_t, V>)", what, desc->item_bytes);
    if (desc->op > TG_OP_MAX_F64)
        return tg_set_error(ctx, TG_ERR_ARG, "%s: op %u (sum, min and max of uint64_t and double only)", what, desc->op);
    if (k < 2 || k > WIN_MAX_K) return tg_set_error(ctx, TG_ERR_ARG, "%s: window size %u (2..4096)", what, k);
    if (mode > TG_WINDOW_DISJOINT) return tg_set_error(ctx, TG_ERR_ARG, "%s: mode %u", what, mode);
    return TG_OK;
}

// rec <- (n, the last min(n, k - 1) items of d_in); hdr: 16 bytes of page-locked memory, not reused before the stream syncs.
// A worker over the limit writes its size only.
int write_record(tg_ctx* ctx, char* rec, const void* d_in, u64 n, u32 k, u32 ib, u64* hdr) {
    hdr[0] = n; hdr[1] = 0;
    TG_CUDA(ctx, cudaMemcpyAsync(rec, hdr, 16, cudaMemcpyHostToDevice, ctx->stream));
    const u64 t = n < k - 1 ? n : k - 1;
    if (n < WIN_LIMIT && t)
        TG_CUDA(ctx, cudaMemcpyAsync(rec + 16, (const char*)d_in + (n - t) * ib, t * ib, cudaMemcpyDeviceToDevice, ctx->stream));
    return TG_OK;
}

template <int OP, int IB, int MODE>
int launch(tg_ctx* ctx, const WinArgs& a, u32 grid) {
    auto kern = window_kernel<OP, IB, MODE>;
    if (ctx->kernel_cfg.find((const void*)kern) == ctx->kernel_cfg.end()) {
        TG_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WN_MAX_SMEM));
        ctx->kernel_cfg[(const void*)kern] = 1;
    }
    const u32 Q = (a.m + (MODE == TG_WINDOW_DISJOINT ? 0 : 1)) * a.k;
    const size_t smem = (MODE == TG_WINDOW_DISJOINT ? 1 : 2) * (size_t)(Q + (Q >> a.logR) + 1) * 8;
    TG_LAUNCH_T(ctx, TG_K_WINDOW, kern, grid, WN_THREADS, smem, a);
    return TG_OK;
}

template <int OP, int IB>
int launch_mode(tg_ctx* ctx, u32 mode, const WinArgs& a, u32 grid) {
    if (mode == TG_WINDOW_FULL) return launch<OP, IB, TG_WINDOW_FULL>(ctx, a, grid);
    if (mode == TG_WINDOW_PARTIAL) return launch<OP, IB, TG_WINDOW_PARTIAL>(ctx, a, grid);
    return launch<OP, IB, TG_WINDOW_DISJOINT>(ctx, a, grid);
}

template <int OP>
int launch_ib(tg_ctx* ctx, u32 ib, u32 mode, const WinArgs& a, u32 grid) {
    return ib == 16 ? launch_mode<OP, 16>(ctx, mode, a, grid) : launch_mode<OP, 8>(ctx, mode, a, grid);
}

int launch_op(tg_ctx* ctx, const tg_scan_desc* d, u32 mode, const WinArgs& a, u32 grid) {
    switch (d->op) {
    case TG_OP_SUM_F64: return launch_ib<TG_OP_SUM_F64>(ctx, d->item_bytes, mode, a, grid);
    case TG_OP_SUM_U64: return launch_ib<TG_OP_SUM_U64>(ctx, d->item_bytes, mode, a, grid);
    case TG_OP_MIN_U64: return launch_ib<TG_OP_MIN_U64>(ctx, d->item_bytes, mode, a, grid);
    case TG_OP_MAX_U64: return launch_ib<TG_OP_MAX_U64>(ctx, d->item_bytes, mode, a, grid);
    case TG_OP_MIN_F64: return launch_ib<TG_OP_MIN_F64>(ctx, d->item_bytes, mode, a, grid);
    default: return launch_ib<TG_OP_MAX_F64>(ctx, d->item_bytes, mode, a, grid);
    }
}

// The window aux workspace: this worker's record, the p gathered records, then the halo
int prepare_aux(tg_ctx* ctx, u32 k, u32 ib, u32 p, char** aux) {
    void* d;
    TG_TRY(tg_ws_get(ctx, WS_WIN_AUX, (p + 1) * rec_bytes(k, ib) + (size_t)k * ib + 16, &d));
    *aux = (char*)d;
    return TG_OK;
}

// the verdict on the limits from every worker's size (the same on every rank): no worker over 2^30 - 1 items or outputs
int check_limits(tg_ctx* ctx, const char* what, u32 k, u32 mode, const u64* sizes, u32 p, u32 rank, u64* f_out, u64* N_out,
                 u64* n_out) {
    u64 N = 0, f = 0;
    for (u32 w = 0; w < p; ++w) {
        if (sizes[w] >= WIN_LIMIT)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "%s: worker %u holds %llu items (limit 2^30 - 1)", what, w,
                                (unsigned long long)sizes[w]);
        if (w < rank) f += sizes[w];
        N += sizes[w];
    }
    u64 fw = 0;
    for (u32 w = 0; w < p; fw += sizes[w], ++w) {
        const u64 c = out_count(mode, k, fw, sizes[w], N, w == p - 1);
        if (c >= WIN_LIMIT)
            return tg_set_error(ctx, TG_ERR_TOO_LARGE, "%s: worker %u would emit %llu items (limit 2^30 - 1)", what, w,
                                (unsigned long long)c);
        if (w == rank) *n_out = c;
    }
    *f_out = f;
    *N_out = N;
    return TG_OK;
}

// Worker `rank` of p once every worker's size is known on the host and, with p > 1, the records are in device memory
// (aux + rec_bytes, one per worker): the verdict on the limits, the halo out of the predecessors' records, the kernel
int window_run(tg_ctx* ctx, const tg_scan_desc* desc, u32 k, u32 mode, const void* d_in, const u64* sizes, u32 p, u32 rank,
               char* aux, const char* what, void** out_dptr, size_t* out_n) {
    const u32 ib = desc->item_bytes;
    u64 f, N, n_out;
    TG_TRY(check_limits(ctx, what, k, mode, sizes, p, rank, &f, &N, &n_out));
    const u64 n = sizes[rank];
    const u64 h = f < k - 1 ? f : k - 1;
    const size_t rb = rec_bytes(k, ib);
    char* halo = aux + (p + 1) * rb;
    // positions [f - h, f): from the tails of ranks rank-1, rank-2, ... (rank q's tail holds [f_q + n_q - t_q, f_q + n_q))
    u64 need_end = f;
    for (int q = (int)rank - 1; q >= 0 && need_end > f - h; --q) {
        const u64 nq = sizes[q], end_q = need_end, tq = nq < k - 1 ? nq : k - 1;
        const u64 beg = end_q - tq > f - h ? end_q - tq : f - h;
        if (end_q > beg)
            TG_CUDA(ctx, cudaMemcpyAsync(halo + (beg - (f - h)) * ib, aux + (q + 1) * rb + 16 + (beg - (end_q - tq)) * ib,
                                         (end_q - beg) * ib, cudaMemcpyDeviceToDevice, ctx->stream));
        need_end -= nq;
    }
    void* out;
    TG_TRY(tg_ws_get(ctx, WS_WIN_OUT, n_out * ib + 16, &out));
    if (n_out) {
        WinArgs a;
        a.in = d_in; a.halo = halo; a.out = out;
        a.f = f; a.n = n; a.lo = f - h; a.N = N;
        a.k = k;
        a.m = WN_TILE / k > 1 ? WN_TILE / k : 1;
        u32 lg = 0;
        while ((1u << lg) < k) ++lg;
        a.logR = (lg + 1) / 2 > 4 ? (lg + 1) / 2 : 4;
        a.R = 1u << a.logR;
        a.J = (k + a.R - 1) / a.R;
        a.b0 = a.lo / k;
        a.out_extra = out_count(TG_WINDOW_FULL, k, f, n, N, false);
        a.last = rank == p - 1;
        const u64 nblocks = (f + n - 1) / k + 1 - a.b0;
        TG_TRY(launch_op(ctx, desc, mode, a, (u32)((nblocks + a.m - 1) / a.m)));
    }
    *out_dptr = out;
    *out_n = n_out;
    return TG_OK;
}

// p = 1: no collective and no host round trip.  p > 1: this worker's record into one ncclAllGather, one host read of the
// gathered sizes, then window_run.
int window_impl(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n_local, uint32_t k, uint32_t mode,
                void** out_dptr, size_t* out_n) {
    const u32 p = (u32)ctx->nranks, ib = desc->item_bytes;
    if (p == 1 && n_local >= WIN_LIMIT)
        return tg_set_error(ctx, TG_ERR_TOO_LARGE, "window: n_local=%zu (limit 2^30 - 1)", n_local);
    char* aux;
    TG_TRY(prepare_aux(ctx, k, ib, p, &aux));
    u64 sizes[TG_MAX_RANKS];
    if (p == 1) sizes[0] = n_local;
    else {
        const size_t rb = rec_bytes(k, ib);
        TG_TRY(write_record(ctx, aux, d_in, n_local, k, ib, (u64*)ctx->pinned));
        TG_NCCL(ctx, ncclAllGather(aux, aux + rb, rb, ncclUint8, ctx->comm, ctx->stream));
        u64* hs = (u64*)((char*)ctx->pinned + 4096);
        TG_CUDA(ctx, cudaMemcpy2DAsync(hs, 8, aux + rb, rb, 8, p, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (u32 w = 0; w < p; ++w) sizes[w] = hs[w];
    }
    return window_run(ctx, desc, k, mode, d_in, sizes, p, (u32)ctx->rank, aux, "window", out_dptr, out_n);
}

int check_ranks(tg_ctx* ctx) {
    if (ctx->nranks > TG_MAX_RANKS) return tg_set_error(ctx, TG_ERR_ARG, "window: at most 16 ranks");
    return TG_OK;
}

// a host File goes up into the WS_IN staging buffer, a device File is read where it is
int stage_input(tg_ctx* ctx, const tg_merge_input* in, uint32_t item_bytes, const void** d_in, size_t* n) {
    if (in->dev) {
        if (in->dev->item_bytes != item_bytes || (!in->dev->dptr && in->dev->items))
            return tg_set_error(ctx, TG_ERR_ARG, "window_file: the device File has item size %u, the operator takes %u",
                                in->dev->item_bytes, item_bytes);
        *d_in = in->dev->dptr;
        *n = in->dev->items;
        return TG_OK;
    }
    if (!in->blocks && in->nblocks) return tg_set_error(ctx, TG_ERR_ARG, "window_file: the input has no blocks");
    size_t bytes = 0;
    for (size_t i = 0; i < in->nblocks; ++i) bytes += in->blocks[i].bytes;
    if (bytes % item_bytes) return tg_set_error(ctx, TG_ERR_ARG, "window_file: %zu bytes is not a multiple of %u", bytes, item_bytes);
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

}  // namespace

extern "C" {

int tg_window(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n_local, uint32_t k, uint32_t mode,
              void** out_dptr, size_t* out_n) {
    if (!ctx || !out_dptr || !out_n || (!d_in && n_local)) return tg_set_error(ctx, TG_ERR_ARG, "window: NULL argument");
    TG_TRY(check_args(ctx, "window", desc, k, mode));
    TG_TRY(check_ranks(ctx));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return window_impl(ctx, desc, d_in, n_local, k, mode, out_dptr, out_n);
}

int tg_window_file(tg_ctx* ctx, const tg_scan_desc* desc, const tg_merge_input* in, uint32_t k, uint32_t mode, size_t* out_items) {
    if (!ctx || !in || !out_items) return tg_set_error(ctx, TG_ERR_ARG, "window_file: NULL argument");
    TG_TRY(check_args(ctx, "window_file", desc, k, mode));
    TG_TRY(check_ranks(ctx));
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const void* d_in;
    size_t n;
    TG_TRY(stage_input(ctx, in, desc->item_bytes, &d_in, &n));
    void* out = nullptr;
    size_t n_out = 0;
    TG_TRY(window_impl(ctx, desc, d_in, n, k, mode, &out, &n_out));
    ctx->out_ptr = out; ctx->out_items = n_out; ctx->out_item_bytes = desc->item_bytes;
    *out_items = n_out;
    return TG_OK;
}

int tg_window_select(tg_ctx* ctx, const tg_scan_desc* desc, const void* const* d_shards, const size_t* n_shards, uint32_t p,
                     uint32_t rank, uint32_t k, uint32_t mode, void** out_dptr, size_t* out_n) {
    if (!ctx || !d_shards || !n_shards || !out_dptr || !out_n || p == 0 || p > TG_MAX_RANKS || rank >= p)
        return tg_set_error(ctx, TG_ERR_ARG, "window_select: rank=%u p=%u or a NULL argument", rank, p);
    TG_TRY(check_args(ctx, "window_select", desc, k, mode));
    u64 sizes[TG_MAX_RANKS];
    for (uint32_t w = 0; w < p; ++w) {
        if (!d_shards[w] && n_shards[w]) return tg_set_error(ctx, TG_ERR_ARG, "window_select: shard %u is NULL", w);
        sizes[w] = n_shards[w];
    }
    u64 f, N, n_out;
    TG_TRY(check_limits(ctx, "window_select", k, mode, sizes, p, rank, &f, &N, &n_out));       // (before any tail is read)
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const u32 ib = desc->item_bytes;
    char* aux;
    TG_TRY(prepare_aux(ctx, k, ib, p, &aux));
    // worker w's record into the slot the all-gather fills
    const size_t rb = rec_bytes(k, ib);
    if (p > 1) {
        for (uint32_t w = 0; w < p; ++w)
            TG_TRY(write_record(ctx, aux + (w + 1) * rb, d_shards[w], sizes[w], k, ib, (u64*)ctx->pinned + 2 * w));
        // the headers are copied out of ctx->pinned asynchronously: done before the host may write there again
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return window_run(ctx, desc, k, mode, d_shards[rank], sizes, p, rank, aux, "window_select", out_dptr, out_n);
}

}  // extern "C"
