/*******************************************************************************
 * tests/host/gpu_group_test.cpp — GroupByKey / GroupToIndex of the drop-in INSIDE the unmodified reference.
 *
 * A real Thrill job (api::Run, mock network, THRILL_WORKERS_PER_HOST = number of GPUs): the same pair DIAs go through the stock
 * DIA::GroupByKey / DIA::GroupToIndex (key extractor .first) and through thrill_gpu::GroupByKey / GroupToIndex (GpuGroupNode of
 * thrill_b200/host/thrill_gpu_nodes.hpp).  Placement and key order agree, so for group functions that do not depend on the order
 * inside a group the gathered results are compared EQUAL, not only as multisets.  Mirrors tests/api/groupby_node_test.cpp of
 * the reference.  Prints "PASS ..." lines and exits non-zero on any mismatch.
 ******************************************************************************/
#include <thrill/api/all_gather.hpp>
#include <thrill/api/cache.hpp>
#include <thrill/api/generate.hpp>
#include <thrill/api/group_by_key.hpp>
#include <thrill/api/group_to_index.hpp>
#include <thrill/api/reduce_by_key.hpp>
#include <thrill/api/size.hpp>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <utility>
#include <vector>

#include "../../thrill_b200/host/thrill_gpu_nodes.hpp"

using namespace thrill; // NOLINT

using Pair = std::pair<uint64_t, uint64_t>;

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
    if (ctx.my_rank() == 0) printf("%s Group %s n=%zu workers=%zu\n", ok ? "PASS" : "FAIL", what, n, ctx.num_workers());
    if (!ok && ctx.my_rank() == 0) g_failures++;
}

template <typename T>
static std::vector<T> Sorted(std::vector<T> v) {
    std::sort(v.begin(), v.end());
    return v;
}

static auto key_of = [](const Pair& p) { return p.first; };

int main(int argc, char** argv) {
    size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 9999;
    int rc = api::Run(
        [&](api::Context& ctx) {
            using thrill_gpu::KeyFirst;
            // the sum of a group (groupby_node_test.cpp: GroupBySum), with the key
            auto sum_fn = [](auto& r, const uint64_t& key) {
                uint64_t s = 0;
                while (r.HasNext()) s += r.Next().second;
                return Pair(key, s);
            };
            // the median of a group (groupby_node_test.cpp: GroupByMedian): the middle of the sorted values
            auto median_fn = [](auto& r, const uint64_t& /* key */) {
                std::vector<uint64_t> all;
                while (r.HasNext()) all.push_back(r.Next().second);
                std::sort(all.begin(), all.end());
                return all[all.size() / 2];
            };
            // ---- the groupby_node_test.cpp shapes, mapped to pairs ----
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return Pair(i % 100, i); }).Cache().Keep(8);
                auto cpu = in.GroupByKey<Pair>(key_of, sum_fn).AllGather();
                auto gpu = thrill_gpu::GroupByKey<Pair>(in, KeyFirst(), sum_fn).AllGather();
                Report(ctx, cpu == gpu && cpu.size() == 100, "GroupByKey sum of i % 100", n);
                auto cpu_m = in.GroupByKey<uint64_t>(key_of, median_fn).AllGather();
                auto gpu_m = thrill_gpu::GroupByKey<uint64_t>(in, KeyFirst(), median_fn).AllGather();
                Report(ctx, cpu_m == gpu_m && cpu_m.size() == 100, "GroupByKey median of i % 100", n);
                // GroupToIndex over 2 * 100 indices: every second one has no items
                auto by2 = in.Map([](const Pair& p) { return Pair(2 * p.first, p.second); }).Cache().Keep(8);
                const Pair neutral(~0ull, 0);
                auto cpu_i = by2.GroupToIndex<Pair>(key_of, sum_fn, 200, neutral).AllGather();
                auto gpu_i = thrill_gpu::GroupToIndex<Pair>(by2, KeyFirst(), sum_fn, 200, neutral).AllGather();
                const size_t size = thrill_gpu::GroupToIndex<Pair>(by2, KeyFirst(), sum_fn, 200, neutral).Size();
                Report(ctx, cpu_i == gpu_i && cpu_i.size() == 200 && size == 200, "GroupToIndex sum, missing indices, size", n);
            }
            // ---- PageRank's link lists: GroupToIndex into std::vector<uint64_t> (a non-POD output type) ----
            {
                const size_t nodes = 1000;
                auto edges = api::Generate(ctx, n, [nodes](size_t i) {
                    return Pair(splitmix64(i) % nodes, splitmix64(i + 7) % nodes); }).Cache().Keep(8);
                using Links = std::vector<uint64_t>;
                auto links_fn = [](auto& r, const uint64_t&) {
                    Links out;
                    while (r.HasNext()) out.push_back(r.Next().second);
                    std::sort(out.begin(), out.end());
                    return out;
                };
                auto cpu = edges.GroupToIndex<Links>(key_of, links_fn, nodes).AllGather();
                auto gpu = thrill_gpu::GroupToIndex<Links>(edges, KeyFirst(), links_fn, nodes).AllGather();
                Report(ctx, cpu == gpu && cpu.size() == nodes, "GroupToIndex link lists (std::vector)", n);
                auto cpu_k = edges.GroupByKey<Links>(key_of, links_fn).AllGather();
                auto gpu_k = thrill_gpu::GroupByKey<Links>(edges, KeyFirst(), links_fn).AllGather();
                Report(ctx, cpu_k == gpu_k && !cpu_k.empty(), "GroupByKey link lists (std::vector)", n);
            }
            // ---- a function that stops before the end of its group: called again with the rest ----
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i) % 50, i); }).Cache().Keep(8);
                auto part = [](auto& r, const uint64_t& key) {
                    uint64_t read = 0;
                    while (read < 3 && r.HasNext()) { r.Next(); ++read; }
                    return Pair(key, read);
                };
                auto cpu = Sorted(in.GroupByKey<Pair>(key_of, part).AllGather());
                auto gpu = Sorted(thrill_gpu::GroupByKey<Pair>(in, KeyFirst(), part).AllGather());
                Report(ctx, cpu == gpu && cpu.size() >= n / 3, "GroupByKey partial function (multiset of (key, items read))", n);
            }
            // ---- a host Map child of the results ----
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i + 1) % 3000, i); }).Cache().Keep(8);
                auto f = [](const Pair& p) { return p.first * 3 + p.second; };
                auto cpu = in.GroupByKey<Pair>(key_of, sum_fn).Map(f).AllGather();
                auto gpu = thrill_gpu::GroupByKey<Pair>(in, KeyFirst(), sum_fn).Map(f).AllGather();
                Report(ctx, cpu == gpu && !cpu.empty(), "host Map child of GroupByKey", n);
            }
            // ---- ReducePair -> GroupByKey: the input goes up once, only the grouped items come down ----
            {
                auto x = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i + 3) % 4000, i % 1000); }).Cache().Keep(8);
                auto plus = std::plus<uint64_t>();
                auto count_fn = [](auto& r, const uint64_t& key) {
                    uint64_t s = 0, c = 0;
                    while (r.HasNext()) { s += r.Next().second; ++c; }
                    return Pair(key, s * 16 + c);
                };
                auto by_mod = [](const Pair& p) { return Pair(p.first % 97, p.second); };
                auto cpu = x.ReducePair(plus).Map(by_mod).Cache().GroupByKey<Pair>(key_of, count_fn).AllGather();
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                auto red = thrill_gpu::ReducePair(x, plus);
                auto g = thrill_gpu::GroupByKey<Pair>(red, KeyFirst(), count_fn);
                std::vector<Pair> gpu_direct = g.AllGather();
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers();
                // this worker's input share went up once; its grouped items came down once (ReducePair leaves one item per key,
                // so the workers' grouped items are as many as the groups)
                bool lean = h1 - h0 <= 16 * (n / p + 2) && d1 - d0 <= 16 * gpu_direct.size();
                auto cpu_direct = x.ReducePair(plus).GroupByKey<Pair>(key_of, count_fn).AllGather();
                auto gpu_mod = thrill_gpu::GroupByKey<Pair>(thrill_gpu::ReducePair(x, plus).Map(by_mod), KeyFirst(), count_fn).AllGather();
                Report(ctx, cpu_direct == gpu_direct && cpu == gpu_mod && lean && !cpu.empty(),
                       "ReducePair -> GroupByKey (device-resident in between)", n);
            }
        });
    if (rc != 0) return rc;
    return g_failures.load() ? 1 : 0;
}
