/*******************************************************************************
 * tests/host/gpu_reduce_records_test.cpp — ReduceByKey on records of the drop-in INSIDE the unmodified reference.
 *
 * A real Thrill job (api::Run, mock network, THRILL_WORKERS_PER_HOST = number of GPUs): the same DIAs of fixed-size records go
 * through the stock dia.ReduceByKey(KeyField<T>(), FieldReduce<T>()) and through thrill_gpu::ReduceByKey with the same functors
 * (GpuReduceNode of thrill_b200/host/thrill_gpu_nodes.hpp with tg_reduce_records_desc).  Doubles are integer-valued, so every
 * bracketing gives the same sums; the stock operator leaves the placement and the order open, so the gathered results are compared
 * sorted.  Shapes: the k-means ClosestCentroid (40 bytes, D = 3) and its count-only second reduce, a 176-byte line item with a
 * 1-byte key and four runs (MIN / MAX among them), pair<uint64_t, 24-byte V> with KeyFirst, one hot key, and the chain
 * thrill_gpu::InnerJoin(line items, orders, JoinPair) -> thrill_gpu::ReduceByKey on the 328-byte result, which moves nothing over
 * PCIe between the two nodes (tg_transfer_bytes).  Prints "PASS ..." lines and exits non-zero on any mismatch.
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

//! items compared by their bytes
template <typename T>
static bool BytesLess(const T& x, const T& y) { return std::memcmp(&x, &y, sizeof(T)) < 0; }
template <typename T>
static bool BytesEqual(const std::vector<T>& a, const std::vector<T>& b) {
    return a.size() == b.size() && (a.empty() || std::memcmp(a.data(), b.data(), a.size() * sizeof(T)) == 0);
}

//! k-means: ClosestCentroid<Vector<3, double>> = {size_t cluster_id; {double p[3]; size_t count}}
struct CC3 { uint64_t cluster_id; double p[3]; uint64_t count; };
struct CC3Count : CC3 { };                         // the second reduce: the count only, a's coordinates kept
//! a line item: 1-byte key at 0, then quantity (u64), price, discount, tax (double), two min / max u64 fields, payload
struct LineItem { uint8_t b[176]; };
struct Order { uint8_t b[152]; };
using Joined = std::pair<LineItem, Order>;
struct V24 { uint64_t a, b; double c; };
using PairV24 = std::pair<uint64_t, V24>;

namespace thrill_gpu {
template <> struct UintKeyTraits<CC3> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 0, key_bytes = 8; };
template <> struct UintKeyTraits<CC3Count> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 0, key_bytes = 8; };
template <> struct UintKeyTraits<LineItem> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 0, key_bytes = 1; };
template <> struct UintKeyTraits<Order> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 0, key_bytes = 1; };
template <> struct UintKeyTraits<Joined> { static constexpr bool is_uint_key = true; static constexpr uint32_t key_offset = 0, key_bytes = 1; };
template <> struct ReduceFieldsTraits<CC3> {
    static constexpr bool is_reduce_fields = true;
    static std::vector<tg_field_run> runs() { return { { 8, 3, TG_OP_SUM_F64 }, { 32, 1, TG_OP_SUM_U64 } }; }
};
template <> struct ReduceFieldsTraits<CC3Count> {
    static constexpr bool is_reduce_fields = true;
    static std::vector<tg_field_run> runs() { return { { 32, 1, TG_OP_SUM_U64 } }; }
};
template <> struct ReduceFieldsTraits<LineItem> {
    static constexpr bool is_reduce_fields = true;
    static std::vector<tg_field_run> runs() {
        return { { 8, 1, TG_OP_SUM_U64 }, { 16, 3, TG_OP_SUM_F64 }, { 40, 1, TG_OP_MIN_U64 }, { 48, 1, TG_OP_MAX_F64 } };
    }
};
template <> struct ReduceFieldsTraits<Joined> {         // the line item's quantity and prices, the order's first field
    static constexpr bool is_reduce_fields = true;
    static std::vector<tg_field_run> runs() { return { { 8, 1, TG_OP_SUM_U64 }, { 16, 3, TG_OP_SUM_F64 }, { 184, 1, TG_OP_MAX_U64 } }; }
};
template <> struct ReduceFieldsTraits<PairV24> {
    static constexpr bool is_reduce_fields = true;
    static std::vector<tg_field_run> runs() { return { { 8, 2, TG_OP_SUM_U64 }, { 24, 1, TG_OP_MIN_F64 } }; }
};
}  // namespace thrill_gpu

using thrill_gpu::FieldReduce;
using thrill_gpu::KeyField;
using thrill_gpu::KeyFirst;

static std::atomic<int> g_failures { 0 };

static void Report(api::Context& ctx, bool ok, const char* what, size_t n) {
    ok = ctx.net.AllReduce(static_cast<size_t>(ok ? 0 : 1)) == 0;
    if (ctx.my_rank() == 0) printf("%s ReduceByKey records %s n=%zu workers=%zu\n", ok ? "PASS" : "FAIL", what, n, ctx.num_workers());
    if (!ok && ctx.my_rank() == 0) g_failures++;
}

template <typename T>
static std::vector<T> Sorted(std::vector<T> v) {
    std::sort(v.begin(), v.end(), BytesLess<T>);
    return v;
}

static CC3 MakeCC3(size_t g, uint64_t keys) {
    CC3 c;
    c.cluster_id = splitmix64(g) % keys;
    for (int d = 0; d < 3; ++d) c.p[d] = static_cast<double>(static_cast<int64_t>(splitmix64(g * 3 + d + 11) % 2000001) - 1000000);
    c.count = 1;
    return c;
}

template <typename Rec>
static Rec MakeRecord(size_t g, uint64_t seed, uint64_t keys) {
    Rec r;
    for (size_t i = 0; i < sizeof(Rec); i += 8) {
        uint64_t w = splitmix64(g * 1000003 + i + seed);
        std::memcpy(r.b + i, &w, std::min<size_t>(8, sizeof(Rec) - i));
    }
    r.b[0] = static_cast<uint8_t>(splitmix64(g + 7 * seed) % keys);
    uint64_t q = splitmix64(g + 1) % 50;
    std::memcpy(r.b + 8, &q, 8);
    for (int d = 0; d < 3; ++d) {
        double x = static_cast<double>(splitmix64(g * 5 + d + seed) % 100000);
        std::memcpy(r.b + 16 + 8 * d, &x, 8);
    }
    double y = static_cast<double>(static_cast<int64_t>(splitmix64(g + 99) % 1001) - 500);
    std::memcpy(r.b + 48, &y, 8);
    return r;
}

//! the stock and the GPU reduce of one DIA, gathered and sorted (stock_key: the same key for the stock operator, which needs a
//! key extractor with one operator())
template <typename T, typename DIAType, typename KeyEx, typename StockKey>
static void Compare(api::Context& ctx, const DIAType& a, const KeyEx& key, const StockKey& stock_key, const char* what, size_t n) {
    auto cpu = Sorted(a.ReduceByKey(stock_key, FieldReduce<T>()).AllGather());
    auto gpu = Sorted(thrill_gpu::ReduceByKey(a, key, FieldReduce<T>()).AllGather());
    Report(ctx, BytesEqual(cpu, gpu) && !cpu.empty(), what, n);
}

int main(int argc, char** argv) {
    size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 99999;
    int rc = api::Run(
        [&](api::Context& ctx) {
            for (uint64_t keys : { 16, 1024 }) {
                auto pts = api::Generate(ctx, n, [=](size_t g) { return MakeCC3(g, keys); }).Cache().Keep(2);
                Compare<CC3>(ctx, pts, KeyField<CC3>(), KeyField<CC3>(), keys == 16 ? "k-means ClosestCentroid, 16 keys" : "k-means ClosestCentroid, 1024 keys", n);
            }
            {
                auto pts = api::Generate(ctx, n, [](size_t g) { CC3Count c; static_cast<CC3&>(c) = MakeCC3(g, 64); return c; }).Cache().Keep(2);
                Compare<CC3Count>(ctx, pts, KeyField<CC3Count>(), KeyField<CC3Count>(), "k-means count-only second reduce", n);
            }
            {
                auto li = api::Generate(ctx, n, [](size_t g) { return MakeRecord<LineItem>(g, 3, 4); }).Cache().Keep(2);
                Compare<LineItem>(ctx, li, KeyField<LineItem>(), KeyField<LineItem>(), "176-byte line items, 1-byte key, four runs", n);
                auto hot = api::Generate(ctx, n, [](size_t g) { return MakeRecord<LineItem>(g, 5, 1); }).Cache().Keep(2);
                Compare<LineItem>(ctx, hot, KeyField<LineItem>(), KeyField<LineItem>(), "one hot key", n);
            }
            {
                auto pv = api::Generate(ctx, n, [](size_t g) {
                    return PairV24(splitmix64(g) % 3000, V24 { g, 2 * g, static_cast<double>(splitmix64(g + 3) % 1000) - 500.0 });
                }).Cache().Keep(2);
                Compare<PairV24>(ctx, pv, KeyFirst(), [](const PairV24& x) { return x.first; }, "pair<u64, 24 B> with KeyFirst", n);
            }
            // the chain: InnerJoin(JoinPair) -> ReduceByKey on the 328-byte result, device-resident in between
            {
                // the stock join emits a key's pairs in an order of its own, so every byte outside the runs is made a function of
                // the key (one order per key): then the first item of a group is the same record for both
                auto li = api::Generate(ctx, n, [](size_t g) {
                    const uint64_t k = splitmix64(g + 21) % 200;
                    LineItem r = MakeRecord<LineItem>(k, 7, 256), v = MakeRecord<LineItem>(g, 9, 256);
                    r.b[0] = static_cast<uint8_t>(k);
                    std::memcpy(r.b + 8, v.b + 8, 32);              // quantity and prices vary by item
                    return r;
                }).Cache().Keep(2);
                auto od = api::Generate(ctx, 200, [](size_t g) { Order o = MakeRecord<Order>(g, 8, 200); o.b[0] = static_cast<uint8_t>(g); return o; })
                          .Cache().Keep(2);
                auto cpu = Sorted(api::InnerJoin(li, od, KeyField<LineItem>(), KeyField<Order>(), thrill_gpu::JoinPair<LineItem, Order>())
                                  .ReduceByKey(KeyField<Joined>(), FieldReduce<Joined>()).AllGather());
                auto joined = thrill_gpu::InnerJoin(li, od, KeyField<LineItem>(), KeyField<Order>(), thrill_gpu::JoinPair<LineItem, Order>());
                auto reduced = thrill_gpu::ReduceByKey(joined, KeyField<Joined>(), FieldReduce<Joined>());
                reduced.Keep();
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                const size_t m = thrill_gpu::Size(reduced);       // runs the join and the reduce; Size downloads nothing
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                auto gpu = Sorted(reduced.AllGather());
                const size_t p = ctx.num_workers();
                // only this worker's two input shares went up; nothing came down between the join and the reduce
                const bool same = BytesEqual(cpu, gpu), pcie = d1 == d0 && h1 - h0 <= 176 * (n / p + 2) + 152 * (200 / p + 2);
                if (!same || !pcie || m != gpu.size())
                    printf("chain: equal %d, sizes %zu / %zu / %zu, h2d %llu, d2h %llu\n", (int)same, cpu.size(), gpu.size(), m,
                           (unsigned long long)(h1 - h0), (unsigned long long)(d1 - d0));
                Report(ctx, same && pcie && m == gpu.size() && !cpu.empty(),
                       "InnerJoin(JoinPair) -> ReduceByKey, 328-byte records, no PCIe in between", n);
            }
        });
    if (rc != 0) return rc;
    return g_failures.load() ? 1 : 0;
}
