// tg_radix_sort.cu — LSB radix sort of fixed-size items on one H100 (sm_90a).
//
// Replaces the local sort of the reference's sample sort: SortNode::SortAndWriteToFile ->
// sort_algorithm_(begin,end,cmp) = std::sort (api/sort.hpp:696-742, :789-796).
//
// Prefix sort (the fast path, prefix_sort_fast): one counting read (chunk histograms of the most significant key byte +
// OR/AND of all keys), the pass on that byte as a chunked pass, the next K-1 non-constant bytes as segmented passes inside
// its buckets (tg_segmented.cuh), and the finishing step that orders the short runs of equal K-byte prefixes by the full
// key: fused into the last of those passes plus a repair of the runs it cannot see whole (FusedFinish,
// finish_repair_kernel), or a separate pass (prefix_fixup_kernel); K = ceil((log2 n + 4) / 8).  8 + K*16 + 8 bytes per
// 8-byte key (+ 16 with the separate pass).
// General path (few non-constant bytes, long runs of equal prefixes, small inputs): one histogram kernel (all digit
// histograms from a single read), one tiny scan kernel, then one stable partition pass per non-constant 8-bit digit,
// least significant first (chained scan).  n*s for the histogram + per pass n*s read + n*s write (s = item bytes).
#include "tg_partition.cuh"
#include "tg_keys.cuh"
#include "tg_segmented.cuh"

#include <algorithm>

using namespace tgp;

namespace {

constexpr int MAX_PASSES = 16;

struct PassList {
    int npass;
    unsigned char word[MAX_PASSES];     // which u64 word of the item holds the digit
    unsigned char shift[MAX_PASSES];    // bit shift inside the word
    u32 flip;                           // RADIX-1 for descending order
};

// histogram of every digit position from one read of the input.  Four items per thread in flight; digit
// positions on which the whole warp agrees (constant high bytes, Zipf keys) are detected with two REDUX.OR per
// item word and cost one shared-memory atomic per warp instead of 32 conflicting ones.
template <int WORDS>
__global__ void __launch_bounds__(512) radix_hist_kernel(const typename ItemT<WORDS>::type* __restrict__ in, size_t n,
                                                         PassList pl, u32* __restrict__ ghist) {
    typedef typename ItemT<WORDS>::type Item;
    constexpr int U = 4;
    extern __shared__ u32 sh[];      // [npass][RADIX]
    for (int i = threadIdx.x; i < pl.npass * RADIX; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const size_t stride = (size_t)gridDim.x * blockDim.x * U;
    const u32 lane = lane_id();
    for (size_t base = (size_t)blockIdx.x * blockDim.x * U; base < n; base += stride) {
        Item v[U];
        bool valid[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            size_t i = base + (size_t)u * blockDim.x + threadIdx.x;
            valid[u] = i < n;
            if (valid[u]) v[u] = in[i];
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (__all_sync(0xffffffffu, valid[u])) {
                u64 diff[WORDS];
#pragma unroll
                for (int w = 0; w < WORDS; ++w) {
                    u64 x = item_word(v[u], w);
                    u64 x0 = __shfl_sync(0xffffffffu, x, 0);
                    u64 d = x ^ x0;
                    u32 lo = __reduce_or_sync(0xffffffffu, (u32)d), hi = __reduce_or_sync(0xffffffffu, (u32)(d >> 32));
                    diff[w] = ((u64)hi << 32) | lo;
                }
#pragma unroll 1
                for (int p = 0; p < pl.npass; ++p) {
                    int w = pl.word[p], shf = pl.shift[p];
                    u32 d = ((u32)(item_word(v[u], w) >> shf) & (RADIX - 1)) ^ pl.flip;
                    bool uniform = (((WORDS == 2 && w) ? diff[WORDS - 1] : diff[0]) >> shf & 0xffull) == 0;
                    if (uniform) { if (lane == 0) atomicAdd(&sh[p * RADIX + d], 32u); }
                    else atomicAdd(&sh[p * RADIX + d], 1u);
                }
            }
            else if (valid[u]) {
#pragma unroll 1
                for (int p = 0; p < pl.npass; ++p) {
                    u32 d = ((u32)(item_word(v[u], pl.word[p]) >> pl.shift[p]) & (RADIX - 1)) ^ pl.flip;
                    atomicAdd(&sh[p * RADIX + d], 1u);
                }
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < pl.npass * RADIX; i += blockDim.x)
        if (sh[i]) atomicAdd(&ghist[i], sh[i]);
}

// fast path of the histogram for plain u64 keys (8 digits = the 8 bytes of the key): constant shifts, fully unrolled
__global__ void __launch_bounds__(512) radix_hist_u64_kernel(const u64* __restrict__ in, size_t n, u32 flip, u32* __restrict__ ghist) {
    constexpr int U = 4;
    __shared__ u32 sh[8 * RADIX];
    for (int i = threadIdx.x; i < 8 * RADIX; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const size_t stride = (size_t)gridDim.x * blockDim.x * U;
    const u32 lane = lane_id();
    for (size_t base = (size_t)blockIdx.x * blockDim.x * U; base < n; base += stride) {
        u64 v[U];
        bool valid[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            size_t i = base + (size_t)u * blockDim.x + threadIdx.x;
            valid[u] = i < n;
            v[u] = valid[u] ? in[i] : 0;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (__all_sync(0xffffffffu, valid[u])) {
                u64 x0 = __shfl_sync(0xffffffffu, v[u], 0);
                u64 df = v[u] ^ x0;
                u32 dlo = __reduce_or_sync(0xffffffffu, (u32)df), dhi = __reduce_or_sync(0xffffffffu, (u32)(df >> 32));
                u32 klo = (u32)v[u], khi = (u32)(v[u] >> 32);
#pragma unroll
                for (int p = 0; p < 8; ++p) {
                    u32 w = p < 4 ? klo : khi, dw = p < 4 ? dlo : dhi;
                    u32 d = ((w >> (8 * (p & 3))) & 0xffu) ^ flip;
                    if (((dw >> (8 * (p & 3))) & 0xffu) == 0) { if (lane == 0) atomicAdd(&sh[p * RADIX + d], 32u); }
                    else atomicAdd(&sh[p * RADIX + d], 1u);
                }
            }
            else if (valid[u]) {
#pragma unroll
                for (int p = 0; p < 8; ++p) atomicAdd(&sh[p * RADIX + (((u32)(v[u] >> (8 * p)) & 0xffu) ^ flip)], 1u);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 8 * RADIX; i += blockDim.x)
        if (sh[i]) atomicAdd(&ghist[i], sh[i]);
}

// ---- finishing pass of the prefix sort --------------------------------------------------------------------------
// After stable LSD passes over the most significant digits only, the items are ordered by a key PREFIX; items that
// share a prefix form short runs ("groups") that still have to be ordered by the rest of the key.  For n keys and a
// prefix of >= log2(n)+4 well-spread bits nearly every group is a single item, so one read + one write finishes the
// sort instead of one partition pass per remaining digit.  Every item looks at its neighbours in a shared-memory
// tile (with a halo of FIX_H items on both sides); members of a group of more than one item rank themselves by
// counting the group's smaller keys (ties by position: stable).  A group longer than FIX_H cannot be seen whole from
// every member's tile: the kernel raises *fail and the caller falls back to the plain LSD sort.
constexpr int FIX_H = 64;
constexpr int FIX_THREADS = 256;
constexpr int FIX_IPT = 8;
constexpr int FIX_TILE = FIX_THREADS * FIX_IPT;

struct PrefixMask {
    u64 hi, lo;
};

template <bool PLAIN, class Item>
__device__ __forceinline__ Canon fix_canon(const Item& v, const KeyView& kv) {
    if (PLAIN) {
        Canon c;
        c.hi = 0;
        c.lo = item_word(v, 0);
        return c;
    }
    return canon_key(v, kv);
}
template <bool PLAIN>
__device__ __forceinline__ bool same_prefix(const Canon& a, const Canon& b, const PrefixMask& m) {
    if (PLAIN) return ((a.lo ^ b.lo) & m.lo) == 0;
    return (((a.hi ^ b.hi) & m.hi) | ((a.lo ^ b.lo) & m.lo)) == 0;
}

// the members of a group of more than one item: bounds by scanning the shared tile, rank by counting
template <bool PLAIN, class Item>
__device__ __noinline__ void fixup_group_member(const Item* s, int li, long long first, u32 n, const KeyView& kv,
                                                const PrefixMask& pm, bool head, bool tail, Item* __restrict__ out,
                                                u32* __restrict__ fail) {
    const Item me = s[li];
    const Canon k = fix_canon<PLAIN>(me, kv);
    int lo = li, hi = li;
    bool bad = false;
    if (!head) {
        for (;;) {
            --lo;
            if (li - lo >= FIX_H) { bad = true; break; }
            if (first + lo == 0 || !same_prefix<PLAIN>(fix_canon<PLAIN>(s[lo - 1], kv), k, pm)) break;
        }
    }
    if (!tail && !bad) {
        for (;;) {
            ++hi;
            if (hi - lo >= FIX_H) { bad = true; break; }
            if (first + hi == (long long)n - 1 || !same_prefix<PLAIN>(fix_canon<PLAIN>(s[hi + 1], kv), k, pm)) break;
        }
    }
    if (bad) {
        *fail = 1;
        return;
    }
    u32 rank = 0;
    for (int x = lo; x <= hi; ++x) {
        const Canon c = fix_canon<PLAIN>(s[x], kv);
        rank += (canon_less(c, k) || (x < li && canon_eq(c, k))) ? 1u : 0u;
    }
    out[(u32)(first + lo) + rank] = me;
}

template <int WORDS, bool PLAIN>
__global__ void __launch_bounds__(FIX_THREADS) prefix_fixup_kernel(const typename ItemT<WORDS>::type* __restrict__ in,
                                                                   typename ItemT<WORDS>::type* __restrict__ out, u32 n,
                                                                   KeyView kv, PrefixMask pm, u32* __restrict__ fail) {
    typedef typename ItemT<WORDS>::type Item;
    __shared__ __align__(16) Item s[FIX_TILE + 2 * FIX_H];
    const u32 tile0 = blockIdx.x * FIX_TILE;                 // first owned position
    const long long first = (long long)tile0 - FIX_H;        // position of s[0]
    const bool interior = tile0 >= (u32)FIX_H && (size_t)tile0 + FIX_TILE + FIX_H <= n;
    if (interior) {
        // whole tile + halo in range: 16-byte loads (tile0 - FIX_H is a multiple of 64 items)
        constexpr int VEC = (FIX_TILE + 2 * FIX_H) * (int)sizeof(Item) / 16;
        const uint4* src = reinterpret_cast<const uint4*>(in + (tile0 - FIX_H));
        uint4* dst = reinterpret_cast<uint4*>(s);
#pragma unroll
        for (int j = 0; j < (VEC + FIX_THREADS - 1) / FIX_THREADS; ++j) {
            int q = j * FIX_THREADS + threadIdx.x;
            if (q < VEC) dst[q] = src[q];
        }
    }
    else {
        for (int j = threadIdx.x; j < FIX_TILE + 2 * FIX_H; j += FIX_THREADS) {
            long long g = first + j;
            if (g >= 0 && g < (long long)n) s[j] = in[g];
        }
    }
    __syncthreads();
    if (interior) {
#pragma unroll
        for (int r = 0; r < FIX_IPT; ++r) {
            const int li = FIX_H + r * FIX_THREADS + threadIdx.x;
            const Item me = s[li];
            const Canon k = fix_canon<PLAIN>(me, kv);
            const bool head = !same_prefix<PLAIN>(fix_canon<PLAIN>(s[li - 1], kv), k, pm);
            const bool tail = !same_prefix<PLAIN>(fix_canon<PLAIN>(s[li + 1], kv), k, pm);
            if (head && tail) out[tile0 + r * FIX_THREADS + threadIdx.x] = me;
            else fixup_group_member<PLAIN>(s, li, first, n, kv, pm, head, tail, out, fail);
        }
    }
    else {
#pragma unroll 1
        for (int r = 0; r < FIX_IPT; ++r) {
            const int li = FIX_H + r * FIX_THREADS + threadIdx.x;
            const u32 g = tile0 + r * FIX_THREADS + threadIdx.x;
            if (g >= n) continue;
            const Item me = s[li];
            const Canon k = fix_canon<PLAIN>(me, kv);
            const bool head = g == 0 || !same_prefix<PLAIN>(fix_canon<PLAIN>(s[li - 1], kv), k, pm);
            const bool tail = g == n - 1 || !same_prefix<PLAIN>(fix_canon<PLAIN>(s[li + 1], kv), k, pm);
            if (head && tail) out[g] = me;
            else fixup_group_member<PLAIN>(s, li, first, n, kv, pm, head, tail, out, fail);
        }
    }
}

// ---- the finishing pass fused into the last prefix pass -----------------------------------------------------------
// The last pass on a prefix digit holds each tile's items in prefix order in its exchange buffer (the tile lies inside one
// segment, which the earlier passes ordered by the lower prefix digits): every group of equal prefixes that lies inside an
// exchange round is a run of neighbours there.  Its write-out orders those runs the way fixup_group_member does (rank =
// smaller full keys, ties by position: stable), so the separate finishing pass, one more read and write of every item, is
// not needed.  Groups that cross a piece of a digit run — a boundary between two tiles' runs of the same digit, or the
// boundary between a tile's two exchange rounds — are ordered piece by piece; finish_repair_kernel then re-sorts them whole.
template <bool PLAIN>
struct FusedFinish {
    static constexpr bool kOn = true;
    KeyView kv;
    PrefixMask pm;
    u32* fail;

    template <class Item>
    __device__ __forceinline__ Canon full(const Item& v) const { return fix_canon<PLAIN>(v, kv); }
    // the key's prefix bits (PLAIN: in .lo only)
    template <class Item>
    __device__ __forceinline__ Canon prefix(const Item& v) const {
        const Canon c = full(v);
        Canon p;
        p.hi = PLAIN ? 0 : c.hi & pm.hi;
        p.lo = c.lo & pm.lo;
        return p;
    }
    __device__ __forceinline__ static bool eq(const Canon& a, const Canon& b) { return PLAIN ? a.lo == b.lo : canon_eq(a, b); }

    // an item of a group of more than one in xb[0, nr): its rank in the group -> dst[head + rank]; a group of more than FIX_H
    // items sets *fail (the same limit as prefix_fixup_kernel; every member finds it) and leaves its members where they are
    template <class Item>
    __device__ __forceinline__ void member(const Item* xb, u32 x, u32 nr, Item* dst) const {
        const Item me = xb[x];
        const Canon k = full(me), pk = prefix(me);
        u32 lo = x, hi = x;
        bool bad = false;
        while (lo > 0 && eq(prefix(xb[lo - 1]), pk)) {
            --lo;
            if (x - lo >= (u32)FIX_H) { bad = true; break; }
        }
        while (!bad && hi + 1 < nr && eq(prefix(xb[hi + 1]), pk)) {
            ++hi;
            if (hi - lo >= (u32)FIX_H) bad = true;
        }
        if (bad) {
            *fail = 1;
            dst[x] = me;
            return;
        }
        u32 rank = 0;
        for (u32 y = lo; y <= hi; ++y) {
            const Canon c = full(xb[y]);
            rank += (canon_less(c, k) || (y < x && canon_eq(c, k))) ? 1u : 0u;
        }
        dst[lo + rank] = me;
    }

    // write-out of one exchange round: xb[0, nr) holds tile positions [q0, q0 + nr); item x of digit d goes to
    // out[goff[d] + q0 + x].  Items whose neighbours have other prefixes (nearly all of them) are stored in the first loop,
    // as the plain write-out does; the group members are flagged and ordered after it, so that a warp branches once per
    // member it holds, not once per store.  The positions outside [0, nr) count as other prefixes.
    template <int THREADS, int IT, class Item, class DigitFn>
    __device__ __forceinline__ void write_out(const Item* xb, u32 nr, u32 q0, const u32* goff, const DigitFn& fn, Item* out,
                                              int tid) const {
        const u32 lane = (u32)tid & 31u;
        u32 mem = 0;         // bit i: the item at xb[i * THREADS + tid] is a group member
#pragma unroll
        for (int i = 0; i < IT; ++i) {
            const u32 x = (u32)(i * THREADS + tid);
            const Item v = xb[x];
            const Canon p = prefix(v);
            Canon pl, pr;          // the neighbours' prefixes
            bool has_l = x > 0, has_r = x + 1 < nr;
            if (PLAIN) {
                // plain keys: both neighbours from the buffer, no branch (the loads of all iterations can be issued together)
                pl = prefix(xb[x > 0 ? x - 1 : 0]);
                pr = prefix(xb[x + 1 < (u32)(IT * THREADS) ? x + 1 : x]);
            }
            else {
                // canonical keys cost more to form: from the neighbouring lanes, lanes 0 and 31 from the buffer
                pl.lo = __shfl_up_sync(0xffffffffu, p.lo, 1);
                pr.lo = __shfl_down_sync(0xffffffffu, p.lo, 1);
                pl.hi = __shfl_up_sync(0xffffffffu, p.hi, 1);
                pr.hi = __shfl_down_sync(0xffffffffu, p.hi, 1);
                const u32 y = lane == 0 ? x - 1 : x + 1;      // (x - 1 wraps to >= nr at x = 0)
                bool edge = false;
                if ((lane == 0 || lane == 31) && y < nr) {
                    const Canon e = prefix(xb[y]);
                    if (lane == 0) pl = e; else pr = e;
                    edge = true;
                }
                if (lane == 0) has_l = edge;
                if (lane == 31) has_r = edge;
            }
            if (x < nr) {
                if ((has_l && eq(pl, p)) || (has_r && eq(pr, p))) mem |= 1u << i;
                else out[goff[fn(v, 0)] + q0 + x] = v;
            }
        }
        while (mem) {
            const int i = __ffs(mem) - 1;
            mem &= mem - 1;
            const u32 x = (u32)(i * THREADS + tid);
            member(xb, x, nr, out + goff[fn(xb[x], 0)] + q0);
        }
    }

    // finish_repair_kernel: is p (0 < p < n) inside a group of equal prefixes?  Then the thread that first claims the group's
    // head re-sorts the whole group in place by (full key, position): stable, since the pieces were ordered stably and lie in
    // input order.  The other threads that meet the group only read it, and every position of it holds one of its items at
    // any time, so they find the same head.
    template <class Item>
    __device__ __forceinline__ void repair(Item* out, u32 n, u32 p, u32* claim) const {
        const Canon pk = prefix(out[p]);
        if (!eq(prefix(out[p - 1]), pk)) return;
        u32 h = p - 1;
        while (h > 0 && eq(prefix(out[h - 1]), pk)) {
            --h;
            if (p - h >= (u32)FIX_H) { *fail = 1; return; }
        }
        const u32 bit = 1u << (h & 31);
        if (atomicOr(&claim[h >> 5], bit) & bit) return;
        u32 e = p;
        while (e + 1 < n && eq(prefix(out[e + 1]), pk)) {
            ++e;
            if (e - h >= (u32)FIX_H) { *fail = 1; return; }
        }
        const u32 len = e - h + 1;
        unsigned char rk[FIX_H];
        for (u32 x = 0; x < len; ++x) {
            const Canon k = full(out[h + x]);
            u32 r = 0;
            for (u32 y = 0; y < len; ++y) {
                const Canon c = full(out[h + y]);
                r += (canon_less(c, k) || (y < x && canon_eq(c, k))) ? 1u : 0u;
            }
            rk[x] = (unsigned char)r;
        }
        u64 placed = 0;      // apply the permutation x -> rk[x] cycle by cycle
        for (u32 x = 0; x < len; ++x) {
            if ((placed >> x) & 1u) continue;
            Item v = out[h + x];
            u32 y = rk[x];
            placed |= 1ull << x;
            while (y != x) {
                const Item w = out[h + y];
                out[h + y] = v;
                v = w;
                placed |= 1ull << y;
                y = rk[y];
            }
            out[h + x] = v;
        }
    }
};

// After a fused last pass: one CTA per tile of its tile list, one thread per digit.  The boundaries where a group can be cut
// are the start of every nonempty run of a digit (its position follows from the pass's final inclusive status rows and
// segbase) and the position of a tile's second exchange round inside the digit run that holds it.  Each is checked once.
// claim: one zeroed bit per position (a group's head, taken by the one thread that re-sorts it).
template <int WORDS, bool PLAIN>
__global__ void __launch_bounds__(RADIX) finish_repair_kernel(typename ItemT<WORDS>::type* out, u32 n, const SegList sl,
                                                              const u32* __restrict__ status, u32* __restrict__ claim,
                                                              const FusedFinish<PLAIN> fin) {
    constexpr u32 HALF = (u32)PartCfg<WORDS>::HALF;
    __shared__ u32 warp_tot[RADIX / 32];
    if (blockIdx.x >= seg_num_tiles(sl)) return;
    const uint4 t = __ldg(&sl.tiles[blockIdx.x]);
    const u32 len = t.y, row = t.z, idx = t.w & 0xfffffu, seg = t.w >> 20;
    const u32 d = threadIdx.x, lane = d & 31;
    const u32 incl = __ldg(&status[(size_t)row * RADIX + d]) & VALUE_MASK;
    const u32 excl = idx > 0 ? __ldg(&status[(size_t)(row - 1) * RADIX + d]) & VALUE_MASK : 0u;
    const u32 cnt = incl - excl;
    const u32 p = __ldg(&sl.segbase[(size_t)seg * RADIX + d]) + excl;       // output position of the tile's run of d
    // tile-local start of the run: exclusive scan of the counts over the digits
    u32 sc = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const u32 v = __shfl_up_sync(0xffffffffu, sc, o);
        if (lane >= (u32)o) sc += v;
    }
    if (lane == 31) warp_tot[d >> 5] = sc;
    __syncthreads();
    u32 ls = sc - cnt;
    for (u32 w = 0; w < (d >> 5); ++w) ls += warp_tot[w];
    if (cnt > 0 && p > 0) fin.repair(out, n, p, claim);
    if (len > HALF && ls < HALF && HALF < ls + cnt) fin.repair(out, n, p + (HALF - ls), claim);
}

bool fused_finish_enabled() {
    static int on = -1;
    if (on < 0) { const char* e = getenv("TG_FUSED_FINISH"); on = e ? atoi(e) : 1; }
    return on != 0;
}

// digit passes of a key descriptor over the item's little-endian u64 words, least significant first
int build_pass_list(const tg_key_desc* d, PassList* pl) {
    if (d->item_bytes != 8 && d->item_bytes != 16) return TG_ERR_ARG;
    if (d->key_bytes == 0 || d->key_bytes > MAX_PASSES || d->key_offset + d->key_bytes > d->item_bytes) return TG_ERR_ARG;
    pl->npass = (int)d->key_bytes;
    pl->flip = d->descending ? (RADIX - 1) : 0;
    for (u32 j = 0; j < d->key_bytes; ++j) {
        u32 byte = (d->key_kind == TG_KEY_UINT_LE) ? d->key_offset + j : d->key_offset + d->key_bytes - 1 - j;
        pl->word[j] = (unsigned char)(byte / 8);
        pl->shift[j] = (unsigned char)(8 * (byte % 8));
    }
    return TG_OK;
}

// prefix mask (canonical key space) of the digit passes >= pass0: pass j is the j-th least significant key byte
PrefixMask prefix_mask(const tg_key_desc* d, int pass0) {
    PrefixMask m = { 0, 0 };
    const u32 kb = d->key_bytes;
    if (d->key_kind == TG_KEY_UINT_LE) {
        const u64 all = kb >= 8 ? ~0ull : ((1ull << (8 * kb)) - 1);
        m.lo = pass0 >= 8 ? 0 : (all & ~((1ull << (8 * pass0)) - 1));
    }
    else {
        const u32 top = kb - (u32)pass0;         // leading key bytes; the canonical form is left-aligned
        m.hi = top >= 8 ? ~0ull : (top ? ~0ull << (8 * (8 - top)) : 0);
        m.lo = top > 8 ? (top >= 16 ? ~0ull : ~0ull << (8 * (16 - top))) : 0;
    }
    return m;
}

// number of leading digits after which a group of equal prefixes is expected to be a single key
// (well-spread keys): 2^(8K) >= 16 n
int prefix_digits_for(size_t n) {
    int bits = 4;
    while (bits < 64 && ((size_t)1 << bits) < n * 16) ++bits;
    return (bits + 7) / 8;
}

bool prefix_sort_enabled() {
    static int on = -1;
    if (on < 0) { const char* e = getenv("TG_PREFIX_SORT"); on = e ? atoi(e) : 1; }
    return on != 0;
}

bool segmented_enabled() {
    static int on = -1;
    if (on < 0) { const char* e = getenv("TG_SEGMENTED"); on = e ? atoi(e) : 1; }
    return on != 0;
}

// The finishing pass of a prefix sort fused into its last prefix pass (FusedFinish): the key, the prefix, the flag that a group
// was too long (device word, zeroed by run_segmented_passes).
struct FinishArgs {
    const tg_key_desc* desc;
    bool plain_u64;
    PrefixMask pm;
    u32* fail;
};

// the last prefix pass with the fused finishing pass, then finish_repair_kernel (the attempt's one finishing launch)
template <int WORDS, bool PLAIN>
int launch_fused_last(tg_ctx* ctx, const FinishArgs& fa, const void* src, void* dst, u32 n, const RadixDigit& fn, u32* status,
                      const SegList& sl) {
    typedef typename ItemT<WORDS>::type Item;
    FusedFinish<PLAIN> fin;
    if (make_key_view(fa.desc, &fin.kv) != TG_OK) return tg_set_error(ctx, TG_ERR_ARG, "radix sort: unsupported key descriptor");
    fin.pm = fa.pm;
    fin.fail = fa.fail;
    u32* claim;
    const size_t claim_bytes = (((size_t)n + 31) / 32) * 4;
    TG_TRY(tg_ws_get(ctx, WS_FINISH, claim_bytes, (void**)&claim));
    TG_CUDA(ctx, cudaMemsetAsync(claim, 0, claim_bytes, ctx->stream));
    TG_CUDA(ctx, cudaMemsetAsync(fa.fail, 0, 4, ctx->stream));
    TG_TRY((launch_partition_v<WORDS, RadixDigit, true, false, false, FusedFinish<PLAIN>>(ctx, src, dst, n, fn, nullptr, status, sl,
                                                                                        nullptr, fin)));
    TG_LAUNCH_T(ctx, TG_K_FIXUP, (finish_repair_kernel<WORDS, PLAIN>), sl.num_tiles, RADIX, 0, (Item*)dst, n, sl, (const u32*)status,
                claim, fin);
    return TG_OK;
}

// `npos` stable passes (digit positions pos[0..npos), least significant first) inside the segments given by the
// histogram of the digit the items are currently partitioned by (seg_size on the host, seg_start on the device)
// first_unstable: the first of these passes orders by a digit below which nothing has been ordered yet, and the items are
// nothing but their key: it may run with the cheaper unstable ranking.
// seg_size == nullptr: the segment sizes are only known on the device (d_seg_size): the tile list is built there and nothing
// waits for the host.
// fin != nullptr: the last pass finishes the prefix sort (launch_fused_last); read fin->fail with finish_flag.
template <int WORDS>
int run_segmented_passes(tg_ctx* ctx, const PassList& pl, const int* pos, int npos, const u32* seg_size, const u32* d_seg_size,
                         const u32* d_seg_start, size_t n, void** src, void** dst, bool first_unstable = false,
                         const FinishArgs* fin = nullptr) {
    typedef typename ItemT<WORDS>::type Item;
    if (fin && npos == 0) return tg_set_error(ctx, TG_ERR_ARG, "segmented passes: a fused finishing pass needs a pass");
    if (npos == 0) return TG_OK;
    if (npos > 4) return tg_set_error(ctx, TG_ERR_ARG, "segmented passes: at most 4 digit positions");
    // (pinned staging buffer 1: the chunk list of the pass before this may still be in flight from buffer 0; every caller
    // has synchronised the stream since the previous use of buffer 1)
    uint4* d_tiles;
    u32 total = 0;
    const u32* d_total = nullptr;
    if (seg_size) TG_TRY(build_tile_list(ctx, RADIX, seg_size, tile_items<WORDS>(), 1, WS_SEG_TILES, &d_tiles, &total));
    else TG_TRY(build_seg_tiles_device(ctx, d_seg_size, d_seg_start, n, tile_items<WORDS>(), false, WS_SEG_TILES, &d_tiles, &d_total, &total));
    if (total == 0) return fin ? tg_set_error(ctx, TG_ERR_ARG, "segmented passes: a fused finishing pass needs items") : TG_OK;
    u32* tables;       // segcount [seg][npos][RADIX] | segbase [pos][seg][RADIX]
    const size_t table_words = (size_t)RADIX * npos * RADIX;
    TG_TRY(tg_ws_get(ctx, WS_SEG_TABLES, 2 * table_words * 4, (void**)&tables));
    u32* segcount = tables;
    u32* segbase = tables + table_words;
    u32* status;
    const size_t pass_status_words = (size_t)total * RADIX;
    TG_TRY(tg_ws_get(ctx, WS_SORT_STATUS2, (size_t)npos * pass_status_words * 4, (void**)&status));
    TG_CUDA(ctx, cudaMemsetAsync(segcount, 0, table_words * 4, ctx->stream));
    TG_CUDA(ctx, cudaMemsetAsync(status, 0, (size_t)npos * pass_status_words * 4, ctx->stream));
    SegList sl = { d_tiles, nullptr, total, d_total };
    DigitList<RadixDigit> dl;
    dl.n = npos;
    for (int i = 0; i < 4; ++i) {
        const int q = pos[i < npos ? i : 0];
        dl.fn[i] = RadixDigit{ (int)pl.word[q], (int)pl.shift[q], pl.flip };
    }
    TG_TRY((launch_seg_count<WORDS, RadixDigit>(ctx, *src, sl, dl, segcount)));
    TG_LAUNCH(ctx, seg_scan_kernel, dim3(RADIX, npos), RADIX, 0, segcount, d_seg_start, npos, RADIX, segbase);
    for (int i = 0; i < npos; ++i) {
        RadixDigit fn = { (int)pl.word[pos[i]], (int)pl.shift[pos[i]], pl.flip };
        sl.segbase = segbase + (size_t)i * RADIX * RADIX;
        if (i == 0 && first_unstable)
            TG_TRY((launch_partition_seg_unstable<WORDS, RadixDigit>(ctx, *src, *dst, (u32)n, fn, status + (size_t)i * pass_status_words, sl)));
        else if (fin && i == npos - 1) {
            if constexpr (WORDS == 1) {
                if (fin->plain_u64 && !fin->desc->descending)
                    TG_TRY((launch_fused_last<WORDS, true>(ctx, *fin, *src, *dst, (u32)n, fn, status + (size_t)i * pass_status_words, sl)));
                else
                    TG_TRY((launch_fused_last<WORDS, false>(ctx, *fin, *src, *dst, (u32)n, fn, status + (size_t)i * pass_status_words, sl)));
            }
            else TG_TRY((launch_fused_last<WORDS, false>(ctx, *fin, *src, *dst, (u32)n, fn, status + (size_t)i * pass_status_words, sl)));
        }
        else
            TG_TRY((launch_partition_seg<WORDS, RadixDigit>(ctx, *src, *dst, (u32)n, fn, status + (size_t)i * pass_status_words, sl)));
        void* t = *src; *src = *dst; *dst = t;
    }
    return TG_OK;
}

// *ok = the finishing pass (separate or fused) found no group too long; synchronises the stream
int finish_flag(tg_ctx* ctx, const u32* d_fail, bool* ok) {
    u32* h_fail = (u32*)ctx->pinned + 7168;       // (byte offset 28 KB of the pinned scratch: the callers keep the histogram / OR-AND words at its start)
    TG_CUDA(ctx, cudaMemcpyAsync(h_fail, d_fail, 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *ok = *h_fail == 0;
    return TG_OK;
}

// After the finishing pass: *src = the sorted items if `sorted`; otherwise a permutation of the input stably ordered by the
// prefix, what the general path expects: the last prefix pass's input after a fused finishing pass, its output otherwise.
inline void finish_swap(bool fused, bool sorted, void** src, void** dst) {
    if (sorted != fused) std::swap(*src, *dst);
}

// finishing pass of the prefix sort over src -> dst; *ok = no group was too long
template <int WORDS>
int run_fixup(tg_ctx* ctx, const tg_key_desc* desc, bool plain_u64, const PrefixMask& pm, const void* src, void* dst, size_t n, u32* d_fail,
              bool* ok) {
    typedef typename ItemT<WORDS>::type Item;
    KeyView kv;
    if (make_key_view(desc, &kv) != TG_OK) return tg_set_error(ctx, TG_ERR_ARG, "radix sort: unsupported key descriptor");
    const u32 grid = (u32)((n + FIX_TILE - 1) / FIX_TILE);
    TG_CUDA(ctx, cudaMemsetAsync(d_fail, 0, 4, ctx->stream));
    if (plain_u64 && !desc->descending)
        TG_LAUNCH_T(ctx, TG_K_FIXUP, (prefix_fixup_kernel<WORDS, true>), grid, FIX_THREADS, 0, (const Item*)src, (Item*)dst, (u32)n, kv, pm, d_fail);
    else
        TG_LAUNCH_T(ctx, TG_K_FIXUP, (prefix_fixup_kernel<WORDS, false>), grid, FIX_THREADS, 0, (const Item*)src, (Item*)dst, (u32)n, kv, pm, d_fail);
    return finish_flag(ctx, d_fail, ok);
}

// Speculative fast path of the prefix sort: assumes the position of the most significant varying key bit (ctx->spec_top_bit for
// integer keys held in one item word — a worker of a multi-GPU sort knows it from its splitters, a single worker learns it from
// the OR/AND of the previous sort — the most significant key byte otherwise) and that the digit below it has many values.  One
// read (chunk histograms of that digit + OR/AND of the keys), the pass on it as a segmented pass over the chunks, the other K-1
// prefix digits inside its buckets, the finishing pass.  *taken = the items in *src are sorted; otherwise *src holds a
// permutation of the input and the caller runs the general path.
template <int WORDS>
int prefix_sort_fast(tg_ctx* ctx, const tg_key_desc* desc, const PassList& pl, bool plain_u64, size_t n, void** src, void** dst,
                     bool* taken) {
    typedef typename ItemT<WORDS>::type Item;
    *taken = false;
    const int K = prefix_digits_for(n);
    if (!prefix_sort_enabled() || !segmented_enabled() || pl.npass < K + 2 || n < (1u << 15)) return TG_OK;
    if (ctx->prefix_sort_penalty > 0) return TG_OK;          // counted down by the general path
    if (ctx->prefix_spec_penalty > 0) { ctx->prefix_spec_penalty--; return TG_OK; }
    // integer key inside one item word: digits at bit granularity (a worker's key range need not start at a byte boundary)
    const bool bitwise = desc->key_kind == TG_KEY_UINT_LE && (desc->key_offset & 7) + desc->key_bytes <= 8;
    const int kb0 = 8 * (int)(desc->key_offset & 7), kbits = 8 * (int)desc->key_bytes;
    PassList pp = pl;                // the K prefix digits, least significant first (pp.npass = K)
    int tb = kbits;
    if (bitwise) {
        tb = ctx->spec_top_bit < kbits ? ctx->spec_top_bit : kbits;
        if ((tb + 7) / 8 < K + 2 || tb - 8 * K < 0) return TG_OK;          // few varying bits: plain LSD passes are as cheap
        pp.npass = K;
        for (int i = 0; i < K; ++i) {
            pp.word[i] = (unsigned char)(desc->key_offset / 8);
            pp.shift[i] = (unsigned char)(kb0 + tb - 8 * (K - i));
        }
    }
    const int top = bitwise ? K - 1 : pl.npass - 1;
    const u32 tile = tile_items<WORDS>();
    const ChunkGeom cg = chunk_geometry<WORDS>(ctx, n);
    const u32 chunk_items = cg.chunk_items;
    const int nchunks = cg.nchunks;

    u32* tab;      // chunkcount [nchunks][RADIX] | chunk segbase [nchunks][RADIX] | totals [RADIX] | gbase [RADIX] | orand u64[4] | fail
    const size_t cw = (size_t)nchunks * RADIX;
    TG_TRY(tg_ws_get(ctx, WS_SORT_HIST2, (2 * cw + 2 * RADIX + 16) * 4, (void**)&tab));
    u32* chunkcount = tab;
    u32* chunkbase = tab + cw;
    u32* totals = chunkbase + cw;
    u32* gbase_top = totals + RADIX;
    u64* orand = (u64*)(gbase_top + RADIX);
    u32* fail = (u32*)(orand + 4);
    u64* h_orand = (u64*)ctx->pinned;
    u32* h_totals = (u32*)(h_orand + 4);
    u64* h_init = h_orand + 512;                 // separate pinned words: read by the H2D copy below
    for (int w = 0; w < 2; ++w) { h_init[2 * w] = 0; h_init[2 * w + 1] = ~0ull; }
    TG_CUDA(ctx, cudaMemcpyAsync(orand, h_init, 32, cudaMemcpyHostToDevice, ctx->stream));
    const RadixDigit top_fn = { (int)pp.word[top], (int)pp.shift[top], pl.flip };
    TG_LAUNCH_T(ctx, TG_K_RADIX_HIST, (chunk_hist_kernel<WORDS, RadixDigit, true>), nchunks, 512, 0, (const Item*)*src, (u32)n, chunk_items,
                top_fn, chunkcount, orand);
    TG_LAUNCH(ctx, chunk_scan_kernel, 1, 4 * RADIX, 0, chunkcount, nchunks, totals, gbase_top, chunkbase);
    TG_CUDA(ctx, cudaMemcpyAsync(h_orand, orand, 32, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(h_totals, totals, RADIX * 4, cudaMemcpyDeviceToHost, ctx->stream));
    // the chunk tile list does not depend on the data: build and upload it while the histogram runs
    std::vector<u32> chunk_size(nchunks, chunk_items);
    chunk_size[nchunks - 1] = (u32)(n - (size_t)(nchunks - 1) * chunk_items);
    uint4* d_ctiles;
    u32 ctotal = 0;
    TG_TRY(build_tile_list(ctx, nchunks, chunk_size.data(), tile, 0, WS_SEG_TILES2, &d_ctiles, &ctotal));
    u32* cstatus;
    TG_TRY(tg_ws_get(ctx, WS_SORT_STATUS, (size_t)ctotal * RADIX * 4, (void**)&cstatus));
    TG_CUDA(ctx, cudaMemsetAsync(cstatus, 0, (size_t)ctotal * RADIX * 4, ctx->stream));
    // Items that are nothing but their key (equal keys are indistinguishable) need no stability from the pass on the most
    // significant digit nor from the first pass below it: the cheaper unstable ranking (TG_UNSTABLE_RANK=0 switches it off)
    static const bool unstable_ok = !(getenv("TG_UNSTABLE_RANK") && atoi(getenv("TG_UNSTABLE_RANK")) == 0);
    const bool key_only = unstable_ok && desc->key_bytes == desc->item_bytes && desc->key_offset == 0;
    static const bool optimistic = !(getenv("TG_SORT_OPTIMISTIC") && atoi(getenv("TG_SORT_OPTIMISTIC")) == 0);
    const bool fused = fused_finish_enabled();
    if (bitwise && optimistic) {
        // Integer keys: the digits are fixed by the assumed top bit, so everything can be queued without waiting for the histogram
        // — the pass on the top digit, the tile list of its buckets (built on the device), the passes inside them, the finishing
        // pass — and the host looks at the histogram, the OR/AND of the keys and the finishing pass's flag once, at the end.  A
        // wrong assumption (bits above the top digit vary, the digit has few values, a group was too long) leaves a permutation of
        // the input in *src for the general path, exactly as before.
        int ppos[MAX_PASSES];
        for (int i = 0; i < K - 1; ++i) ppos[i] = i;
        const u64 kmask = kbits >= 64 ? ~0ull : (((1ull << kbits) - 1) << kb0);
        PrefixMask pmo = { 0, (kmask >> kb0) & ~((1ull << (pp.shift[0] - kb0)) - 1) };
        {
            SegList sl = { d_ctiles, chunkbase, ctotal, nullptr };
            if (key_only) TG_TRY((launch_partition_seg_unstable<WORDS, RadixDigit>(ctx, *src, *dst, (u32)n, top_fn, cstatus, sl)));
            else TG_TRY((launch_partition_seg<WORDS, RadixDigit>(ctx, *src, *dst, (u32)n, top_fn, cstatus, sl)));
            void* t = *src; *src = *dst; *dst = t;
        }
        const FinishArgs fa = { desc, plain_u64, pmo, fail };
        TG_TRY((run_segmented_passes<WORDS>(ctx, pp, ppos, K - 1, nullptr, totals, gbase_top, n, src, dst, key_only, fused ? &fa : nullptr)));
        bool ok = false;
        if (fused) TG_TRY(finish_flag(ctx, fail, &ok));                                           // (the one synchronisation)
        else TG_TRY((run_fixup<WORDS>(ctx, desc, plain_u64, pmo, *src, *dst, n, fail, &ok)));
        int nonempty_o = 0;
        for (int d = 0; d < RADIX; ++d) nonempty_o += h_totals[d] ? 1 : 0;
        const int w = pp.word[0];
        const u64 diff = (h_orand[2 * w] ^ h_orand[2 * w + 1]) & kmask;
        const int tb_act = diff ? 64 - __builtin_clzll(diff) - kb0 : 0;          // most significant varying key bit + 1
        if (tb_act != tb) ctx->spec_top_bit = tb_act > 8 ? tb_act : 8;           // what the next sort on this ctx should assume
        if (tb_act > tb || nonempty_o < 32) {
            if (tb_act <= tb && (tb_act + 7) / 8 < K + 2) ctx->prefix_spec_penalty = 8;
            finish_swap(fused, false, src, dst);
            return TG_OK;                                                         // (*src: a permutation of the input)
        }
        finish_swap(fused, ok, src, dst);
        if (ok) *taken = true;
        else {
            ctx->prefix_sort_penalty = 8;
            ctx->prefix_sort_fallbacks++;
        }
        return TG_OK;
    }
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));

    int nonempty = 0;
    for (int d = 0; d < RADIX; ++d) nonempty += h_totals[d] ? 1 : 0;
    int prefix_pos[MAX_PASSES];      // indices into pp of the K-1 lower prefix digits, least significant first
    PrefixMask pm = { 0, 0 };
    if (bitwise) {
        const int w = pp.word[0];
        const u64 kmask = kbits >= 64 ? ~0ull : (((1ull << kbits) - 1) << kb0);
        const u64 diff = (h_orand[2 * w] ^ h_orand[2 * w + 1]) & kmask;
        const int tb_act = diff ? 64 - __builtin_clzll(diff) - kb0 : 0;          // most significant varying key bit + 1
        if (tb_act != tb) ctx->spec_top_bit = tb_act > 8 ? tb_act : 8;           // what the next sort on this ctx should assume
        if (tb_act > tb || nonempty < 32) {
            // bits above the assumed top digit vary (this is not a most-significant-digit pass), or the digit has few values
            if (tb_act > tb || (tb_act + 7) / 8 < K + 2) ctx->prefix_spec_penalty = tb_act > tb ? 0 : 8;
            return TG_OK;
        }
        for (int i = 0; i < K - 1; ++i) prefix_pos[i] = i;
        pm.lo = (kmask >> kb0) & ~((1ull << (pp.shift[0] - kb0)) - 1);            // canonical key = the key value (tg_keys.cuh)
    }
    else {
        // which digit positions are active (not constant over all keys), least significant first
        int active[MAX_PASSES], nactive = 0;
        for (int p = 0; p < pl.npass; ++p) {
            const u64 diff = h_orand[2 * pl.word[p]] ^ h_orand[2 * pl.word[p] + 1];
            if ((diff >> pl.shift[p]) & 0xffu) active[nactive++] = p;
        }
        if (nactive < K + 2 || active[nactive - 1] != top || nonempty < 32) {
            ctx->prefix_spec_penalty = 8;         // the guess was wrong for this kind of input: do not pay for it every time
            return TG_OK;
        }
        for (int i = 0; i < K - 1; ++i) prefix_pos[i] = active[nactive - K + i];
        pm = prefix_mask(desc, active[nactive - K]);
    }
    // (1) most significant digit: segmented pass over the chunks
    {
        SegList sl = { d_ctiles, chunkbase, ctotal, nullptr };
        if (key_only) TG_TRY((launch_partition_seg_unstable<WORDS, RadixDigit>(ctx, *src, *dst, (u32)n, top_fn, cstatus, sl)));
        else TG_TRY((launch_partition_seg<WORDS, RadixDigit>(ctx, *src, *dst, (u32)n, top_fn, cstatus, sl)));
        void* t = *src; *src = *dst; *dst = t;
    }
    // (2) the other K-1 prefix digits inside the buckets of (1), the last one with the finishing pass fused in
    const FinishArgs fa = { desc, plain_u64, pm, fail };
    TG_TRY((run_segmented_passes<WORDS>(ctx, pp, prefix_pos, K - 1, h_totals, nullptr, gbase_top, n, src, dst, key_only, fused ? &fa : nullptr)));
    // (3) finishing pass (separate, or the fused pass's flag)
    bool ok = false;
    if (fused) TG_TRY(finish_flag(ctx, fail, &ok));
    else TG_TRY((run_fixup<WORDS>(ctx, desc, plain_u64, pm, *src, *dst, n, fail, &ok)));
    finish_swap(fused, ok, src, dst);
    if (ok) *taken = true;
    else {
        ctx->prefix_sort_penalty = 8;
        ctx->prefix_sort_fallbacks++;
    }
    return TG_OK;
}

// The sorted items end up in *result (= d_items or d_tmp); result == nullptr asks for them in d_items.
template <int WORDS>
int radix_sort_impl(tg_ctx* ctx, const tg_key_desc* desc, const PassList& pl, void* d_items, void* d_tmp, size_t n,
                    void** result) {
    typedef typename ItemT<WORDS>::type Item;
    const u32 num_tiles = num_tiles_for<WORDS>(n);
    void* src = d_items;
    void* dst = d_tmp;
    bool plain_u64 = WORDS == 1 && pl.npass == 8;
    for (int p = 0; p < pl.npass && plain_u64; ++p) plain_u64 = pl.word[p] == 0 && pl.shift[p] == 8 * p;

    bool fast = false;
    TG_TRY((prefix_sort_fast<WORDS>(ctx, desc, pl, plain_u64, n, &src, &dst, &fast)));
    if (fast) {
        if (result) *result = src;
        else if (src != d_items)
            TG_LAUNCH(ctx, copy_items_kernel<WORDS>, ctx->sm_count * 8, 256, 0, (const Item*)src, (Item*)d_items, n);
        return TG_OK;
    }

    u32* hist;      // [npass][RADIX] counts | [npass][RADIX] bases | [npass] skip | fail flag
    size_t hist_words = (size_t)2 * pl.npass * RADIX + MAX_PASSES + 4;
    TG_TRY(tg_ws_get(ctx, WS_SORT_HIST, hist_words * 4, (void**)&hist));
    u32* gbase = hist + (size_t)pl.npass * RADIX;
    u32* skip = gbase + (size_t)pl.npass * RADIX;
    u32* fail = skip + MAX_PASSES;
    u32* status;
    const size_t pass_status_bytes = (size_t)num_tiles * RADIX * 4;
    size_t status_bytes = (size_t)pl.npass * pass_status_bytes;
    TG_TRY(tg_ws_get(ctx, WS_SORT_STATUS, status_bytes, (void**)&status));
    TG_CUDA(ctx, cudaMemsetAsync(hist, 0, hist_words * 4, ctx->stream));
    TG_CUDA(ctx, cudaMemsetAsync(status, 0, status_bytes, ctx->stream));

    if (plain_u64)
        TG_LAUNCH_T(ctx, TG_K_RADIX_HIST, radix_hist_u64_kernel, ctx->sm_count * 2, 512, 0, (const u64*)src, n, pl.flip, hist);
    else
        TG_LAUNCH_T(ctx, TG_K_RADIX_HIST, radix_hist_kernel<WORDS>, ctx->sm_count * 2, 512, pl.npass * RADIX * 4, (const Item*)src, n, pl, hist);
    TG_LAUNCH(ctx, scan_hist_kernel, 1, RADIX, 0, hist, gbase, skip, pl.npass, (u32)n);
    // skip flags and the digit histograms themselves (segment sizes of the segmented passes) to the host
    u32* h_skip = (u32*)ctx->pinned;
    u32* h_hist = h_skip + MAX_PASSES;
    TG_CUDA(ctx, cudaMemcpyAsync(h_skip, skip, pl.npass * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaMemcpyAsync(h_hist, hist, (size_t)pl.npass * RADIX * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));

    int active[MAX_PASSES], nactive = 0;      // digit positions where the keys differ, least significant first
    for (int p = 0; p < pl.npass; ++p)
        if (!h_skip[p]) active[nactive++] = p;

    auto run_pass = [&](int p) -> int {
        RadixDigit fn = { (int)pl.word[p], (int)pl.shift[p], pl.flip };
        TG_TRY((launch_partition<WORDS, RadixDigit>(ctx, src, dst, (u32)n, fn, gbase + (size_t)p * RADIX,
                                                    status + (size_t)p * num_tiles * RADIX)));
        void* t = src; src = dst; dst = t;
        return TG_OK;
    };

    // ---- prefix sort: the K most significant active digits, then one finishing pass (see prefix_fixup_kernel)
    const int K = prefix_digits_for(n);
    bool done = false;
    if (prefix_sort_enabled() && nactive >= K + 2 && ctx->prefix_sort_penalty == 0) {
        const int top = active[nactive - 1];
        int nonempty = 0;
        for (int d = 0; d < RADIX; ++d) nonempty += h_hist[top * RADIX + d] ? 1 : 0;
        const PrefixMask pm = prefix_mask(desc, active[nactive - K]);
        bool fused = false;
        if (segmented_enabled() && K >= 2 && nonempty >= 32) {
            // most significant digit first (global pass), then the other K-1 digits inside its buckets, the last one with the
            // finishing pass fused in
            fused = fused_finish_enabled();
            const FinishArgs fa = { desc, plain_u64, pm, fail };
            TG_TRY(run_pass(top));
            TG_TRY((run_segmented_passes<WORDS>(ctx, pl, active + (nactive - K), K - 1, h_hist + top * RADIX, nullptr,
                                                 gbase + (size_t)top * RADIX, n, &src, &dst, false, fused ? &fa : nullptr)));
        }
        else
            for (int a = nactive - K; a < nactive; ++a) TG_TRY(run_pass(active[a]));
        bool ok = false;
        if (fused) TG_TRY(finish_flag(ctx, fail, &ok));
        else TG_TRY((run_fixup<WORDS>(ctx, desc, plain_u64, pm, src, dst, n, fail, &ok)));
        finish_swap(fused, ok, &src, &dst);
        if (ok) done = true;
        else {
            // a group of equal prefixes was longer than the finishing pass can see (heavy duplicates / clustered
            // keys): plain LSD over all active digits from the current permutation of the input; skip the attempt
            // for the next few sorts on this ctx
            ctx->prefix_sort_penalty = 8;
            ctx->prefix_sort_fallbacks++;
            for (int a = nactive - K; a < nactive; ++a)
                TG_CUDA(ctx, cudaMemsetAsync((char*)status + (size_t)active[a] * pass_status_bytes, 0, pass_status_bytes, ctx->stream));
        }
    }
    else if (ctx->prefix_sort_penalty > 0 && nactive >= K + 2) ctx->prefix_sort_penalty--;

    if (!done)
        for (int a = 0; a < nactive; ++a) TG_TRY(run_pass(active[a]));

    if (result) *result = src;
    else if (src != d_items)
        TG_LAUNCH(ctx, copy_items_kernel<WORDS>, ctx->sm_count * 8, 256, 0, (const Item*)src, (Item*)d_items, n);
    return TG_OK;
}

}  // namespace

// used by the operators (tg_sample_sort.cu): the sorted items are in *result (d_items or d_tmp), or in d_items if
// result == nullptr
int tg_radix_sort_items(tg_ctx* ctx, const tg_key_desc* desc, void* d_items, void* d_tmp, size_t n, void** result) {
    if (result) *result = d_items;
    if (n >= (1u << 30)) return tg_set_error(ctx, TG_ERR_TOO_LARGE, "radix sort: n=%zu >= 2^30", n);
    if (((uintptr_t)d_items | (uintptr_t)d_tmp) & 15) return tg_set_error(ctx, TG_ERR_ARG, "buffers must be 16-byte aligned");
    PassList pl;
    if (build_pass_list(desc, &pl) != TG_OK) return tg_set_error(ctx, TG_ERR_ARG, "radix sort: unsupported key descriptor");
    if (n < 2) return TG_OK;
    return desc->item_bytes == 8 ? radix_sort_impl<1>(ctx, desc, pl, d_items, d_tmp, n, result)
                                 : radix_sort_impl<2>(ctx, desc, pl, d_items, d_tmp, n, result);
}

extern "C" int tg_radix_sort_local(tg_ctx* ctx, const tg_key_desc* desc, void* d_items, void* d_tmp, size_t n) {
    if (!ctx || !desc) return TG_ERR_ARG;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    return tg_radix_sort_items(ctx, desc, d_items, d_tmp, n, nullptr);
}
