/*******************************************************************************
 * tests/host/gpu_join_test.cpp — InnerJoin of the drop-in INSIDE the unmodified reference.
 *
 * A real Thrill job (api::Run, mock network, THRILL_WORKERS_PER_HOST = number of GPUs): the same DIAs go through the stock
 * api::InnerJoin and through thrill_gpu::InnerJoin (GpuJoinNode of thrill_b200/host/thrill_gpu_nodes.hpp).  The stock operator
 * leaves the placement and the order of equal keys open, so the gathered results are compared as multisets.  Mirrors
 * tests/api/join_test.cpp of the reference.  Prints "PASS ..." lines and exits non-zero on any mismatch.
 ******************************************************************************/
#include <thrill/api/all_gather.hpp>
#include <thrill/api/generate.hpp>
#include <thrill/api/inner_join.hpp>
#include <thrill/api/reduce_by_key.hpp>
#include <thrill/api/size.hpp>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <tuple>
#include <utility>
#include <vector>

#include "../../thrill_b200/host/thrill_gpu_nodes.hpp"

using namespace thrill; // NOLINT

using Pair = std::pair<uint64_t, uint64_t>;
using Triple = std::tuple<uint64_t, uint64_t, uint64_t>;

static inline uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    uint64_t z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

static std::atomic<int> g_failures { 0 };

static void Report(api::Context& ctx, bool ok, const char* what, size_t n) {
    // every worker's verdict counts: a mismatch on any worker fails the line
    ok = ctx.net.AllReduce(static_cast<size_t>(ok ? 0 : 1)) == 0;
    if (ctx.my_rank() == 0) printf("%s InnerJoin %s n=%zu workers=%zu\n", ok ? "PASS" : "FAIL", what, n, ctx.num_workers());
    if (!ok && ctx.my_rank() == 0) g_failures++;
}

template <typename T>
static std::vector<T> Sorted(std::vector<T> v) {
    std::sort(v.begin(), v.end());
    return v;
}

static auto key_of = [](const Pair& p) { return p.first; };
static auto stock_kv = [](const Pair& a, const Pair& b) { return Triple(a.first, a.second, b.second); };
static auto stock_v = [](const Pair& a, const Pair& b) { return Pair(a.second, b.second); };

int main(int argc, char** argv) {
    size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 9999;
    int rc = api::Run(
        [&](api::Context& ctx) {
            using thrill_gpu::KeyFirst;
            // ---- the shapes of the reference's tests/api/join_test.cpp the descriptor set expresses ----
            {
                // identity keys, both join functions
                auto a = api::Generate(ctx, n, [](size_t i) { return Pair(i, i * i); }).Cache().Keep(4);
                auto b = api::Generate(ctx, n, [](size_t i) { return Pair(i, i * i * i); }).Cache().Keep(4);
                auto cpu = Sorted(api::InnerJoin(a, b, key_of, key_of, stock_kv).AllGather());
                auto gpu = Sorted(thrill_gpu::InnerJoin(a, b, KeyFirst(), KeyFirst(), thrill_gpu::JoinKeyValues()).AllGather());
                Report(ctx, cpu == gpu && cpu.size() == n, "identity keys (key, v1, v2)", n);
                auto cpu2 = Sorted(api::InnerJoin(a, b, key_of, key_of, stock_v).AllGather());
                auto gpu2 = Sorted(thrill_gpu::InnerJoin(a, b, KeyFirst(), KeyFirst(), thrill_gpu::JoinValues()).AllGather());
                Report(ctx, cpu2 == gpu2 && cpu2.size() == n, "identity keys (v1, v2)", n);
            }
            {
                // every item on one key: 333 x 333 outputs
                auto a = api::Generate(ctx, 333, [](size_t i) { return Pair(1, i); }).Cache().Keep(2);
                auto b = api::Generate(ctx, 333, [](size_t i) { return Pair(1, i + 1000); }).Cache().Keep(2);
                auto cpu = Sorted(api::InnerJoin(a, b, key_of, key_of, stock_kv).AllGather());
                auto gpu = Sorted(thrill_gpu::InnerJoin(a, b, KeyFirst(), KeyFirst(), thrill_gpu::JoinKeyValues()).AllGather());
                Report(ctx, cpu == gpu && cpu.size() == 333 * 333, "333 x 333 on one key", 333);
            }
            {
                // 100 x 333 on small keys
                auto a = api::Generate(ctx, 100, [](size_t i) { return Pair(i % 10, i); }).Cache().Keep(2);
                auto b = api::Generate(ctx, 333, [](size_t i) { return Pair(i % 7, i * 3); }).Cache().Keep(2);
                auto cpu = Sorted(api::InnerJoin(a, b, key_of, key_of, stock_kv).AllGather());
                auto gpu = Sorted(thrill_gpu::InnerJoin(a, b, KeyFirst(), KeyFirst(), thrill_gpu::JoinKeyValues()).AllGather());
                Report(ctx, cpu == gpu && !cpu.empty(), "100 x 333", 433);
            }
            // ---- a self-join: one parent on both edges ----
            {
                auto a = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i) % 2000, i); }).Cache().Keep(2);
                auto cpu = Sorted(api::InnerJoin(a, a, key_of, key_of, stock_kv).AllGather());
                auto gpu = Sorted(thrill_gpu::InnerJoin(a, a, KeyFirst(), KeyFirst(), thrill_gpu::JoinKeyValues()).AllGather());
                Report(ctx, cpu == gpu, "InnerJoin(a, a)", n);
            }
            // ---- a host child reading the 24-byte tuples ----
            {
                auto a = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i + 1) % 5000, i); }).Cache().Keep(2);
                auto b = api::Generate(ctx, n / 2, [](size_t i) { return Pair(splitmix64(i + 2) % 5000, 7 * i); }).Cache().Keep(2);
                auto sum = [](const Triple& t) { return std::get<0>(t) + 3 * std::get<1>(t) + 5 * std::get<2>(t); };
                auto cpu = Sorted(api::InnerJoin(a, b, key_of, key_of, stock_kv).Map(sum).AllGather());
                auto gpu = Sorted(thrill_gpu::InnerJoin(a, b, KeyFirst(), KeyFirst(), thrill_gpu::JoinKeyValues()).Map(sum).AllGather());
                Report(ctx, cpu == gpu && !cpu.empty(), "host Map child of the (key, v1, v2) tuples", n);
            }
            // ---- ReducePair -> InnerJoin(JoinValues) -> ReducePair: nothing crosses PCIe between the nodes ----
            {
                auto x = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i + 3) % 3000, i % 1000); }).Cache().Keep(2);
                auto y = api::Generate(ctx, n / 2 + 7, [](size_t i) { return Pair(splitmix64(i + 4) % 3000, i % 977); }).Cache().Keep(2);
                auto plus = std::plus<uint64_t>();
                auto red = [](const Pair& a, const Pair& b) { return Pair(a.first, a.second + b.second); };
                auto cpu_j = api::InnerJoin(x.ReducePair(plus), y.ReducePair(plus), key_of, key_of, stock_v);
                auto cpu = Sorted(cpu_j.ReduceByKey(key_of, red).AllGather());
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                auto j = thrill_gpu::InnerJoin(thrill_gpu::ReducePair(x, plus), thrill_gpu::ReducePair(y, plus), KeyFirst(), KeyFirst(),
                                               thrill_gpu::JoinValues());
                auto out = thrill_gpu::ReducePair(j, plus);
                std::vector<Pair> gpu = Sorted(out.AllGather());
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers();
                // this worker's two input shares went up once, its share of the final result came down once
                bool lean = h1 - h0 <= 16 * ((n + n / 2 + 7) / p + 2) && d1 - d0 <= 16 * gpu.size();
                Report(ctx, cpu == gpu && lean && !cpu.empty(), "ReducePair -> InnerJoin -> ReducePair (device-resident in between)", n);
            }
        });
    if (rc != 0) return rc;
    return g_failures.load() ? 1 : 0;
}
