// tg_reduce_ops.cuh — the reduce functions the host shim recognises (TG_OP_*), as identities and register-level folds: shared by
// ReduceByKey on pairs (tg_reduce.cu) and on records (tg_reduce_records.cu)
#pragma once
#include "tg_common.cuh"

namespace {

// Every table slot, accumulator and side slot starts at op_identity(op), and folding a key's first record into it must give
// that record back bit for bit, as the reference stores a key's first record as is (core/reduce_probing_hash_table.hpp:201,
// :251).  Sums of doubles start at -0.0 (-0.0 + x == x for every x, +0.0 + -0.0 == +0.0 would lose the sign), min/max of
// doubles at a NaN that every value replaces (f64_better).  The identity of FIRST is never read.
__host__ __device__ inline u64 op_identity(int op) {
    switch (op) {
    case TG_OP_SUM_F64: return 0x8000000000000000ull;          // -0.0
    case TG_OP_MIN_U64: return ~0ull;
    case TG_OP_MIN_F64:
    case TG_OP_MAX_F64: return 0x7FF8000000000000ull;          // NaN
    default: return 0ull;
    }
}

// min/max of doubles (bit patterns): v replaces the accumulated o if it is smaller (larger), if o is the identity, or if o is
// a NaN of the input and v a number.  A NaN never replaces a number, nor a NaN of the input, and the identity replaces
// nothing: an accumulator that has seen a record holds one of the input's bit patterns, whatever unused accumulators
// (still the identity) are folded into it.
__device__ __forceinline__ bool f64_better(int op, u64 vb, u64 ob) {
    const double v = __longlong_as_double((long long)vb), o = __longlong_as_double((long long)ob);
    return (op == TG_OP_MIN_F64 ? v < o : o < v) || (isnan(o) && (!isnan(v) || ob == op_identity(op)));
}

// register-level reduce function (the warp-uniform fast path)
__device__ __forceinline__ u64 op_combine(int op, u64 a, u64 b) {
    switch (op) {
    case TG_OP_SUM_F64: return (u64)__double_as_longlong(__longlong_as_double((long long)a) + __longlong_as_double((long long)b));
    case TG_OP_SUM_U64: return a + b;
    case TG_OP_MIN_U64: return a < b ? a : b;
    case TG_OP_MAX_U64: return a > b ? a : b;
    case TG_OP_MIN_F64:
    case TG_OP_MAX_F64: return f64_better(op, b, a) ? b : a;
    default: return a;          // TG_OP_FIRST
    }
}

}  // namespace
