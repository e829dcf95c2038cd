/*******************************************************************************
 * tests/host/gpu_join_records_test.cpp — InnerJoin on records of the drop-in INSIDE the unmodified reference.
 *
 * A real Thrill job (api::Run, mock network, THRILL_WORKERS_PER_HOST = number of GPUs): the same DIAs of fixed-size records go
 * through the stock api::InnerJoin(l, r, KeyField<L>(), KeyField<R>(), JoinPair<L, R>()) and through thrill_gpu::InnerJoin with
 * the same functors (GpuJoinNode of thrill_b200/host/thrill_gpu_nodes.hpp with tg_join_records_desc).  The stock operator leaves
 * the placement and the order of equal keys open, so the gathered results are compared sorted.  Shapes: a 4-byte item that is
 * its key, a 2-byte key at offset 5 of 12 bytes, a 5-byte key at offset 3 of 24 bytes, a key at the very end of its item,
 * TPC-H-shaped 176 / 152-byte items, pair<uint64_t, V> with KeyFirst, one hot key, an empty side, a self-join, and
 * Size(InnerJoin(...)) over device-resident parents, which moves nothing over PCIe (tg_transfer_bytes).
 * Prints "PASS ..." lines and exits non-zero on any mismatch.
 ******************************************************************************/
#include <thrill/api/all_gather.hpp>
#include <thrill/api/cache.hpp>
#include <thrill/api/generate.hpp>
#include <thrill/api/inner_join.hpp>
#include <thrill/api/reduce_by_key.hpp>
#include <thrill/api/size.hpp>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <tuple>
#include <utility>
#include <vector>

#include "../../thrill_b200/host/thrill_gpu_nodes.hpp"

using namespace thrill; // NOLINT

static inline uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    uint64_t z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

//! a record of N bytes compared by its bytes; fields filled from splitmix64(global index, seed), the key field set after
template <size_t N>
struct Bytes {
    uint8_t b[N];
    static Bytes Make(size_t g, uint64_t seed) {
        Bytes r;
        for (size_t i = 0; i < N; i += 8) {
            uint64_t w = splitmix64(g * 1000003 + i + seed);
            std::memcpy(r.b + i, &w, std::min<size_t>(8, N - i));
        }
        return r;
    }
    Bytes& SetKey(size_t off, size_t nb, uint64_t key) { std::memcpy(b + off, &key, nb); return *this; }
    friend bool operator < (const Bytes& x, const Bytes& y) { return std::memcmp(x.b, y.b, N) < 0; }
    friend bool operator == (const Bytes& x, const Bytes& y) { return std::memcmp(x.b, y.b, N) == 0; }
};
struct Rec4 : Bytes<4> { };
struct Rec12 : Bytes<12> { };
struct Rec24 : Bytes<24> { };
struct RecEnd : Bytes<16> { };
struct LineItem : Bytes<176> { };
struct Order : Bytes<152> { };
using Pair = std::pair<uint64_t, uint64_t>;
struct V24 {
    uint64_t a, b, c;
    friend bool operator < (const V24& x, const V24& y) { return std::tie(x.a, x.b, x.c) < std::tie(y.a, y.b, y.c); }
    friend bool operator == (const V24& x, const V24& y) { return x.a == y.a && x.b == y.b && x.c == y.c; }
};
using PairV24 = std::pair<uint64_t, V24>;

namespace thrill_gpu {
template <> struct UintKeyTraits<Rec4> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 0, key_bytes = 4; };
template <> struct UintKeyTraits<Rec12> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 5, key_bytes = 2; };
template <> struct UintKeyTraits<Rec24> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 3, key_bytes = 5; };
template <> struct UintKeyTraits<RecEnd> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 12, key_bytes = 4; };
template <> struct UintKeyTraits<LineItem> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 0, key_bytes = 8; };
template <> struct UintKeyTraits<Order> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 0, key_bytes = 8; };
}  // namespace thrill_gpu

using thrill_gpu::JoinPair;
using thrill_gpu::KeyField;
using thrill_gpu::KeyFirst;

static std::atomic<int> g_failures { 0 };

static void Report(api::Context& ctx, bool ok, const char* what, size_t n) {
    ok = ctx.net.AllReduce(static_cast<size_t>(ok ? 0 : 1)) == 0;
    if (ctx.my_rank() == 0) printf("%s InnerJoin records %s n=%zu workers=%zu\n", ok ? "PASS" : "FAIL", what, n, ctx.num_workers());
    if (!ok && ctx.my_rank() == 0) g_failures++;
}

template <typename T>
static std::vector<T> Sorted(std::vector<T> v) {
    std::sort(v.begin(), v.end());
    return v;
}

template <typename T>
static auto Side(api::Context& ctx, size_t n, uint64_t seed, uint64_t universe) {
    using K = thrill_gpu::UintKeyTraits<T>;
    return api::Generate(ctx, n, [=](size_t g) {
        T r;
        static_cast<Bytes<sizeof(T)>&>(r) = Bytes<sizeof(T)>::Make(g, seed);
        r.SetKey(K::key_offset, K::key_bytes, splitmix64(g + 77 * seed) % universe);
        return r;
    }).Cache().Keep(2);
}

//! the stock and the GPU join of two record DIAs on KeyField, gathered and sorted
template <typename L, typename R, typename LD, typename RD>
static void Compare(api::Context& ctx, const LD& a, const RD& b, const char* what, size_t n, bool nonempty = true) {
    auto cpu = Sorted(api::InnerJoin(a, b, KeyField<L>(), KeyField<R>(), JoinPair<L, R>()).AllGather());
    auto gpu = Sorted(thrill_gpu::InnerJoin(a, b, KeyField<L>(), KeyField<R>(), JoinPair<L, R>()).AllGather());
    Report(ctx, cpu == gpu && (!nonempty || !cpu.empty()), what, n);
}

int main(int argc, char** argv) {
    size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 9999;
    int rc = api::Run(
        [&](api::Context& ctx) {
            Compare<Rec4, Rec4>(ctx, Side<Rec4>(ctx, n, 1, 3000), Side<Rec4>(ctx, n / 2, 2, 3000), "4-byte items that are their keys", n);
            Compare<Rec12, Rec24>(ctx, Side<Rec12>(ctx, n, 3, 1000), Side<Rec24>(ctx, n, 4, 1000),
                                  "12-byte (2-byte key at 5) x 24-byte (5-byte key at 3)", n);
            Compare<RecEnd, Rec4>(ctx, Side<RecEnd>(ctx, n, 5, 2000), Side<Rec4>(ctx, n / 3, 6, 2000), "a key at the end of its item", n);
            Compare<LineItem, Order>(ctx, Side<LineItem>(ctx, n, 7, n / 4 + 1), Side<Order>(ctx, n / 4, 8, n / 4 + 1),
                                     "TPC-H-shaped 176 x 152 bytes", n);
            Compare<Rec24, Rec12>(ctx, Side<Rec24>(ctx, 300, 9, 1), Side<Rec12>(ctx, 200, 10, 1), "300 x 200 on one key", 300);
            Compare<Rec24, Rec12>(ctx, Side<Rec24>(ctx, n, 11, 100), Side<Rec12>(ctx, 0, 12, 100), "an empty side", n, false);
            {
                auto a = Side<Rec24>(ctx, n, 13, 2000);
                Compare<Rec24, Rec24>(ctx, a, a, "InnerJoin(a, a)", n);
            }
            // pair<uint64_t, V> with KeyFirst on the GPU side, the stock side with lambdas
            {
                auto a = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i) % 3000, i); }).Cache().Keep(2);
                auto b = api::Generate(ctx, n / 2, [](size_t i) { return PairV24(splitmix64(i + 5) % 3000, V24 { i, 2 * i, 3 * i }); })
                         .Cache().Keep(2);
                auto cpu = Sorted(api::InnerJoin(a, b, [](const Pair& p) { return p.first; }, [](const PairV24& p) { return p.first; },
                                                 [](const Pair& l, const PairV24& r) { return std::make_pair(l, r); }).AllGather());
                auto gpu = Sorted(thrill_gpu::InnerJoin(a, b, KeyFirst(), KeyFirst(), JoinPair<Pair, PairV24>()).AllGather());
                Report(ctx, cpu == gpu && !cpu.empty(), "pair<u64, 8 B> x pair<u64, 24 B> on .first", n);
            }
            // device-resident parents: ReducePair -> InnerJoin(JoinPair) -> Size downloads nothing
            {
                auto x = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i + 3) % 3000, i % 1000); }).Cache().Keep(2);
                auto y = api::Generate(ctx, n / 2 + 7, [](size_t i) { return Pair(splitmix64(i + 4) % 3000, i % 977); }).Cache().Keep(2);
                auto plus = std::plus<uint64_t>();
                auto key_of = [](const Pair& p) { return p.first; };
                const size_t cpu = api::InnerJoin(x.ReducePair(plus), y.ReducePair(plus), key_of, key_of,
                                                  [](const Pair& l, const Pair& r) { return std::make_pair(l, r); }).Size();
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                const size_t gpu = thrill_gpu::Size(thrill_gpu::InnerJoin(thrill_gpu::ReducePair(x, plus), thrill_gpu::ReducePair(y, plus),
                                                                          KeyFirst(), KeyFirst(), JoinPair<Pair, Pair>()));
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers();
                // only this worker's two input shares went up; nothing came down
                Report(ctx, cpu == gpu && cpu > 0 && d1 == d0 && h1 - h0 <= 16 * ((n + n / 2 + 7) / p + 2),
                       "Size(InnerJoin(ReducePair, ReducePair)) device-resident", n);
            }
        });
    if (rc != 0) return rc;
    return g_failures.load() ? 1 : 0;
}
