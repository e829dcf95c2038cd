// tg_keys.cuh — canonical keys of a tg_key_desc: (hi, lo) compared as an unsigned 128-bit number is the order of the
// reference comparator (std::less on the integer key / lexicographic compare of the key bytes,
// examples/terasort/terasort.cpp:35-37), descending descriptors are complemented.
#pragma once
#include "tg_partition.cuh"

namespace tgp {

// ---- canonical keys: (hi, lo) compared as unsigned 128-bit == the reference comparator's order ----------
struct KeyView {
    u32 off, bytes, kind, desc;
};

struct Canon {
    u64 hi, lo;
};
struct CanonIdx {
    u64 hi, lo, idx;
};

__host__ __device__ inline bool canon_less(const Canon& a, const Canon& b) {
    return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo);
}
__host__ __device__ inline bool canon_eq(const Canon& a, const Canon& b) { return a.hi == b.hi && a.lo == b.lo; }
// LessSampleIndex (api/sort.hpp:419-422) on canonical keys
__host__ __device__ inline bool canonidx_less(const CanonIdx& a, const CanonIdx& b) {
    if (a.hi != b.hi) return a.hi < b.hi;
    if (a.lo != b.lo) return a.lo < b.lo;
    return a.idx < b.idx;
}

// most significant byte of a canonical key (the order of the top bytes is the order of the keys' first byte-ranges)
__host__ __device__ inline u32 canon_top_byte(const Canon& c, const KeyView& kv) {
    if (kv.kind == TG_KEY_UINT_LE) return (u32)(c.lo >> (8 * (kv.bytes > 8 ? 8 : kv.bytes) - 8)) & 0xffu;
    return (u32)(c.hi >> 56);
}

// byte j of an item held as little-endian u64 words
template <class Item>
__device__ __forceinline__ u32 item_byte(const Item& v, u32 j) {
    return (u32)(item_word(v, (int)(j >> 3)) >> (8 * (j & 7))) & 0xffu;
}

template <class Item>
__device__ __forceinline__ Canon canon_key(const Item& v, const KeyView& kv) {
    Canon c;
    c.hi = 0; c.lo = 0;
    if (kv.kind == TG_KEY_UINT_LE) {
        if (kv.bytes == 8 && (kv.off & 7) == 0) c.lo = item_word(v, (int)(kv.off >> 3));
        else
            for (u32 j = 0; j < kv.bytes; ++j) c.lo |= (u64)item_byte(v, kv.off + j) << (8 * j);
    }
    else {
        for (u32 j = 0; j < kv.bytes && j < 8; ++j) c.hi |= (u64)item_byte(v, kv.off + j) << (8 * (7 - j));
        for (u32 j = 8; j < kv.bytes; ++j) c.lo |= (u64)item_byte(v, kv.off + j) << (8 * (15 - j));
    }
    if (kv.desc) { c.hi = ~c.hi; c.lo = ~c.lo; }
    return c;
}

inline Canon canon_key_host(const unsigned char* item, const KeyView& kv) {
    Canon c;
    c.hi = 0; c.lo = 0;
    if (kv.kind == TG_KEY_UINT_LE) {
        for (u32 j = 0; j < kv.bytes; ++j) c.lo |= (u64)item[kv.off + j] << (8 * j);
    }
    else {
        for (u32 j = 0; j < kv.bytes && j < 8; ++j) c.hi |= (u64)item[kv.off + j] << (8 * (7 - j));
        for (u32 j = 8; j < kv.bytes; ++j) c.lo |= (u64)item[kv.off + j] << (8 * (15 - j));
    }
    if (kv.desc) { c.hi = ~c.hi; c.lo = ~c.lo; }
    return c;
}

inline int make_key_view(const tg_key_desc* d, KeyView* kv) {
    if (!d) return TG_ERR_ARG;
    if (d->key_bytes == 0 || d->key_offset + d->key_bytes > d->item_bytes) return TG_ERR_ARG;
    if (d->key_kind == TG_KEY_UINT_LE && d->key_bytes > 8) return TG_ERR_ARG;
    if (d->key_kind == TG_KEY_BYTES_BE && d->key_bytes > 16) return TG_ERR_ARG;
    if (d->key_kind != TG_KEY_UINT_LE && d->key_kind != TG_KEY_BYTES_BE) return TG_ERR_ARG;
    kv->off = d->key_offset; kv->bytes = d->key_bytes; kv->kind = d->key_kind; kv->desc = d->descending;
    return TG_OK;
}

// merge path of sorted A and B: the number of A items among the first `diag` merged outputs, ties to A (stable).  Used by the
// merges (tg_merge.cu) and by the join's co-ranks (tg_join.cu).
template <class Item>
__device__ __forceinline__ u32 merge_path_search(const Item* A, u32 na, const Item* B, u32 nb, u32 diag, const KeyView& kv) {
    u32 lo = diag > nb ? diag - nb : 0, hi = diag < na ? diag : na;
    while (lo < hi) {
        u32 mid = (lo + hi) >> 1;            // take mid+1 items from A?
        Canon a = canon_key(A[mid], kv);
        Canon b = canon_key(B[diag - 1 - mid], kv);
        if (canon_less(b, a)) hi = mid; else lo = mid + 1;      // A[mid] <= B[..] -> A first (stable)
    }
    return lo;
}

// tg_merge.cu: stable merge of k sorted runs of 8- or 16-byte items into d_out (d_tmp: scratch of the same size), ties to the
// lower run index
int merge_runs(tg_ctx* ctx, const KeyView& kv, uint32_t item_bytes, const void* const* runs, const uint64_t* run_items,
               uint32_t k, void* d_out, void* d_tmp);

}  // namespace tgp
