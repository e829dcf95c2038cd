// tg_fold.cuh — the closed set of fold functions on one 8-byte value (the whole item, or a pair's .second), shared by the scans
// and actions (tg_scan.cu) and Window (tg_window.cu).  Everything is in an anonymous namespace: each translation unit gets its
// own copies, so the kernels that include it compile exactly as if the functions were written in their file.
#pragma once

#include "tg_common.cuh"

namespace {

// Min / Max on doubles: partial folds must keep positions in order
template <int OP>
__host__ __device__ constexpr bool in_order() { return OP == TG_OP_MIN_F64 || OP == TG_OP_MAX_F64; }

// the one combine function of the sum functions on the 8-byte value, used by every kernel and by the carry fold.  For Min / Max
// on doubles it skips a NaN operand (a NaN is its identity) and keeps the left operand of two equal values; the stock function,
// whose NaN first operand sticks, is stock_fn.
template <int OP>
__device__ __forceinline__ u64 combine(u64 a, u64 b) {
    if (OP == TG_OP_SUM_F64) return (u64)__double_as_longlong(__longlong_as_double((long long)a) + __longlong_as_double((long long)b));
    if (OP == TG_OP_SUM_U64) return a + b;
    if (OP == TG_OP_MIN_U64) return b < a ? b : a;
    if (in_order<OP>()) {
        const double x = __longlong_as_double((long long)a), y = __longlong_as_double((long long)b);
        if (x != x) return b;
        return (OP == TG_OP_MIN_F64 ? y < x : x < y) ? b : a;
    }
    return a < b ? b : a;                       // TG_OP_MAX_U64
}
// the stock function: common::minimum / maximum (std::min / std::max) on doubles, combine otherwise
template <int OP>
__device__ __forceinline__ u64 stock_fn(u64 a, u64 b) {
    if (!in_order<OP>()) return combine<OP>(a, b);
    const double x = __longlong_as_double((long long)a), y = __longlong_as_double((long long)b);
    return (OP == TG_OP_MIN_F64 ? y < x : x < y) ? b : a;
}
// the exact identity of the partial folds (-0.0 for double sums: x + -0.0 == x for every x, including -0.0; a quiet NaN for
// Min / Max on doubles)
template <int OP>
__device__ __forceinline__ u64 ident() {
    return OP == TG_OP_SUM_F64 ? 0x8000000000000000ull : OP == TG_OP_MIN_U64 ? ~0ull
         : in_order<OP>() ? 0x7ff8000000000000ull : 0ull;
}

// unit u of the input: a pair, or two 8-byte items; past the end the value is the identity
template <int OP, int IB>
__device__ __forceinline__ ulonglong2 load_unit(const ulonglong2* __restrict__ in, u64 u, u64 n) {
    if (IB == 16) return u < n ? in[u] : make_ulonglong2(0, ident<OP>());
    if (2 * u + 1 < n) return in[u];
    return make_ulonglong2(2 * u < n ? ((const u64*)in)[2 * u] : ident<OP>(), ident<OP>());
}

}  // namespace
