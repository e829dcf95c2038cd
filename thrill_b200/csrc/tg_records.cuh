// tg_records.cuh — fixed-size records handled through 16-byte tuples {key bytes, u32 position}: Sort's record path
// (tg_sample_sort.cu), InnerJoin on records (tg_join.cu) and ReduceByKey on records (tg_reduce_records.cu).  Records are a
// multiple of 4 bytes long and 4-byte aligned.
#pragma once
#include <initializer_list>

#include "tg_common.cuh"

namespace {

// tuple i = { key bytes of record i, i }: one thread per record, the key read as the (<= 4) aligned words that cover it.
// For a key of at most 8 bytes, .x is the key's bytes as a little-endian integer, zero-extended, and .y = i << 32.
__global__ void make_tuples_kernel(const u32* __restrict__ rec, u32 n, u32 rec_words, u32 key_off, u32 key_bytes,
                                   ulonglong2* __restrict__ tuples) {
    const u32 stride = gridDim.x * blockDim.x;
    const u32 w0 = key_off >> 2, sh = 8 * (key_off & 3), nw = (sh ? 1 : 0) + (key_bytes + 3) / 4;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const u32* r = rec + (size_t)i * rec_words + w0;
        u32 x[5] = { 0, 0, 0, 0, 0 };
#pragma unroll
        for (u32 j = 0; j < 4; ++j)
            if (j < nw && w0 + j < rec_words) x[j] = r[j];
        u32 k[3];
#pragma unroll
        for (u32 j = 0; j < 3; ++j) k[j] = sh ? __funnelshift_r(x[j], x[j + 1], sh) : x[j];
        // zero the bytes beyond the key
        if (key_bytes < 12) {
            const u32 full = key_bytes >> 2, rem = key_bytes & 3;
#pragma unroll
            for (u32 j = 0; j < 3; ++j) {
                if (j > full || (j == full && rem == 0)) k[j] = 0;
                else if (j == full) k[j] &= (1u << (8 * rem)) - 1;
            }
        }
        tuples[i] = make_ulonglong2(((u64)k[1] << 32) | k[0], ((u64)i << 32) | k[2]);
    }
}

// Word index lt of a batch -> (record, word) by a multiply-high with inv = gather_reciprocal(rec_words), or by a division where
// that is 0.  inv = floor((2^32 - 1) / d) + 1 = (2^32 + e) / d with 0 <= e < d, so __umulhi(lt, inv) == lt / d whenever
// lt * (d - 1) < 2^32: for every word index of a batch of 1024 records (lt < 1024 * d) that holds up to d = 2048.  d = 1 would
// need inv = 2^32, which does not fit: 4-byte records, and records of more than 8 KiB, take the division.
inline u32 gather_reciprocal(u32 rec_words) {
    return rec_words >= 2 && rec_words <= 2048 ? 0xffffffffu / rec_words + 1 : 0u;
}

}  // namespace

namespace tgp {

// a record type: item size, and its key field (an unsigned little-endian integer of key_bytes = 1..8 bytes at byte offset key_off)
struct RecSide {
    u32 bytes, key_off, key_bytes;
};

// TG_ERR_ARG unless the size is a multiple of 4 in 4..1024 and the key is 1..8 bytes inside the item (`what` heads the message)
int check_side(tg_ctx* ctx, const char* what, const RecSide& s);

// the n records' tuples in workspace `slot` (tuples | sort scratch), stably sorted by the key: *sorted  (tg_join.cu)
int sort_record_tuples(tg_ctx* ctx, int slot, const void* rec, u64 n, const RecSide& s, const ulonglong2** sorted);

// worker w's n records: their tuples into WS_JOIN_L, partitioned by the owner Hash128to64(0, key) % p into *ptup (WS_JOIN_R);
// *d_tot = the per-destination counts (device)  (tg_join.cu)
int partition_record_tuples(tg_ctx* ctx, const void* rec, size_t n, const RecSide& s, u32 p, ulonglong2** ptup, u32** d_tot);

// An operator's k inputs (rec[j], bytes[j] bytes) that lie in a workspace slot it writes (`slots`: an un-detached result of an
// earlier operator) are copied out of the way first, input j into dst_slots[j]; rec[j] is updated.  An input that is the same
// span as input 0 stays one copy.  (tg_join.cu)
int move_inputs_out_of_slots(tg_ctx* ctx, const void** rec, const size_t* bytes, int k, std::initializer_list<int> slots,
                             const int* dst_slots);

// Store step of the records' exchange for worker `me` of p: d_ptup = its n tuples partitioned by destination, counts = the p x p
// count matrix (host), windows[d] = worker d's window.  Mode 1 stores the records straight into the windows, mode 0 into the
// local send buffer (WS_XCHG_SEND) followed by the transfers (xchg_transfer).  (tg_sample_sort.cu)
int exchange_store_records(tg_ctx* ctx, int mode, bool simulated, const void* d_in, u32 rb, const ulonglong2* d_ptup, size_t n,
                           const u32* counts, int p, int me, void* const* windows);

// The checks of the simulated exchanges after their count steps: out_counts, the receive limit and the windows' sizes (s bytes
// per item), before any store.  (tg_sample_sort.cu)
int select_check(tg_ctx* ctx, const u32* h_mat, int p, size_t s, void* const* d_windows, const size_t* window_bytes, uint64_t* out_counts);

}  // namespace tgp
