/*******************************************************************************
 * tests/host/gpu_merge_test.cpp — Merge of the drop-in INSIDE the unmodified reference.
 *
 * A real Thrill job (api::Run, mock network, THRILL_WORKERS_PER_HOST = number of GPUs): the same sorted DIAs go through
 * the stock api::Merge and through thrill_gpu::Merge (GpuMergeNode of thrill_b200/host/thrill_gpu_nodes.hpp); the gathered
 * results must be identical.  Where the stock operator leaves the order of equal items open (pairs compared by key), the
 * results are compared per key as multisets.  Mirrors tests/api/merge_node_test.cpp of the reference.  Prints "PASS ..."
 * lines and exits non-zero on any mismatch.
 ******************************************************************************/
#include <thrill/api/all_gather.hpp>
#include <thrill/api/generate.hpp>
#include <thrill/api/merge.hpp>
#include <thrill/api/size.hpp>
#include <thrill/api/sort.hpp>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <ostream>
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

static std::atomic<int> g_failures { 0 };

//! pair<uint64_t, uint64_t> as a POD, for the stock operator (which serializes and logs its pivots)
struct PodPair {
    uint64_t first, second;
    friend std::ostream& operator << (std::ostream& os, const PodPair& p) { return os << '(' << p.first << ',' << p.second << ')'; }
};

static void Report(api::Context& ctx, bool ok, const char* what, size_t n) {
    // every worker's verdict counts: a mismatch on any worker fails the line
    ok = ctx.net.AllReduce(static_cast<size_t>(ok ? 0 : 1)) == 0;
    if (ctx.my_rank() == 0) printf("%s Merge %s n=%zu workers=%zu\n", ok ? "PASS" : "FAIL", what, n, ctx.num_workers());
    if (!ok && ctx.my_rank() == 0) g_failures++;
}

//! the result gathered, and this worker's share within the balance the reference's test allows (merge_node_test.cpp:51)
template <typename DIAType>
static std::vector<typename DIAType::ValueType> GatherBalanced(api::Context& ctx, const DIAType& dia, bool* balanced) {
    using T = typename DIAType::ValueType;
    size_t count = 0;
    std::vector<T> all = dia.Map([&count](const T& x) { ++count; return x; }).AllGather();
    const size_t expect = all.size() / ctx.num_workers();
    *balanced = (count > expect ? count - expect : expect - count) <= ctx.num_workers() + 50;
    return all;
}

int main(int argc, char** argv) {
    size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 1000000;
    int rc = api::Run(
        [&](api::Context& ctx) {
            using Less = std::less<uint64_t>;
            // ---- the four shapes of the reference's tests/api/merge_node_test.cpp, at n items per input ----
            for (int shape = 0; shape < 4; ++shape) {
                const char* names[] = { "two balanced", "four balanced", "two imbalanced", "different sizes" };
                auto a = api::Generate(ctx, n, [shape](size_t i) -> uint64_t { return shape == 1 ? 4 * i : shape == 0 ? 2 * i : i; })
                         .Cache().Keep(4);
                std::vector<uint64_t> cpu, gpu;
                bool bal = false;
                if (shape == 0) {
                    auto b = a.Map([](uint64_t x) { return x + 1; }).Cache().Keep(2);
                    cpu = api::Merge(Less(), a, b).AllGather();
                    gpu = GatherBalanced(ctx, thrill_gpu::Merge(Less(), a, b), &bal);
                }
                else if (shape == 1) {
                    auto b = a.Map([](uint64_t x) { return x + 1; }).Cache().Keep(2);
                    auto c = a.Map([](uint64_t x) { return x + 2; }).Cache().Keep(2);
                    auto d = a.Map([](uint64_t x) { return x + 3; }).Cache().Keep(2);
                    cpu = api::Merge(Less(), a, b, c, d).AllGather();
                    gpu = GatherBalanced(ctx, thrill_gpu::Merge(Less(), a, b, c, d), &bal);
                }
                else if (shape == 2) {
                    auto b = a.Map([n](uint64_t x) { return x + 2 * n; }).Cache().Keep(2);
                    cpu = api::Merge(Less(), a, b).AllGather();
                    gpu = GatherBalanced(ctx, thrill_gpu::Merge(Less(), a, b), &bal);
                }
                else {
                    auto b = api::Generate(ctx, 2 * n, [n](size_t i) -> uint64_t { return i + n / 2; }).Cache().Keep(2);
                    cpu = api::Merge(Less(), a, b).AllGather();
                    gpu = GatherBalanced(ctx, thrill_gpu::Merge(Less(), a, b), &bal);
                }
                Report(ctx, cpu == gpu && bal && std::is_sorted(gpu.begin(), gpu.end()), names[shape], n);
            }
            // ---- GPU Sort -> GPU Merge: nothing crosses PCIe between the nodes ----
            {
                auto gen = [](uint64_t seed) { return [seed](size_t i) -> uint64_t { return splitmix64(i + seed) >> 8; }; };
                auto x = api::Generate(ctx, n, gen(1)).Cache().Keep(2);
                auto y = api::Generate(ctx, n / 2 + 7, gen(2)).Cache().Keep(2);
                std::vector<uint64_t> cpu = api::Merge(Less(), x.Sort(), y.Sort()).AllGather();
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                auto m = thrill_gpu::Merge(Less(), thrill_gpu::Sort(x), thrill_gpu::Sort(y));
                std::vector<uint64_t> gpu = m.AllGather();
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers(), local_in = (n + n / 2 + 7) / p + 2;
                // this worker's two input shares went up once, its share of the merged result came down once
                bool lean = h1 - h0 <= 8 * local_in && d1 - d0 <= 8 * ((n + n / 2 + 7) / p + 1);
                Report(ctx, cpu == gpu && lean, "GPU Sort -> GPU Merge (device-resident in between)", n);
            }
            // ---- Merge(cmp, a, a): one GPU parent feeding both inputs ----
            {
                auto x = api::Generate(ctx, n / 2, [](size_t i) -> uint64_t { return splitmix64(i + 5) % 100000; }).Cache().Keep(2);
                std::vector<uint64_t> cpu_sorted = x.Sort().AllGather();
                std::vector<uint64_t> cpu;
                for (uint64_t v : cpu_sorted) { cpu.push_back(v); cpu.push_back(v); }
                auto s = thrill_gpu::Sort(x);
                std::vector<uint64_t> gpu = thrill_gpu::Merge(Less(), s, s).AllGather();
                Report(ctx, cpu == gpu, "Merge(cmp, a, a)", n / 2);
            }
            // ---- one GPU parent and one CPU (Generate / Map) parent ----
            {
                auto x = api::Generate(ctx, n, [](size_t i) -> uint64_t { return splitmix64(i + 9) >> 4; }).Cache().Keep(2);
                auto y = api::Generate(ctx, n / 3, [](size_t i) -> uint64_t { return 3 * i; }).Map([](uint64_t v) { return v + 1; });
                auto y2 = api::Generate(ctx, n / 3, [](size_t i) -> uint64_t { return 3 * i; }).Map([](uint64_t v) { return v + 1; });
                std::vector<uint64_t> cpu = api::Merge(Less(), x.Sort(), y).AllGather();
                std::vector<uint64_t> gpu = thrill_gpu::Merge(Less(), thrill_gpu::Sort(x), y2).AllGather();
                Report(ctx, cpu == gpu, "GPU parent + CPU parent", n);
            }
            // ---- pairs by LessFirst: the stock order of equal keys is unspecified, so per key as multisets ----
            {
                using Pair = std::pair<uint64_t, uint64_t>;
                auto by_first = [](const Pair& a, const Pair& b) { return a.first < b.first; };
                auto x = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i + 1) % 5000, i); }).Cache().Keep(2);
                auto y = api::Generate(ctx, n / 2, [](size_t i) { return Pair(splitmix64(i + 2) % 5000, 1000000000 + i); }).Cache().Keep(2);
                auto xs = x.SortStable(by_first).Cache().Keep(2);
                auto ys = y.SortStable(by_first).Cache().Keep(2);
                // (the stock operator's pivots of std::pair items do not serialize: its side runs on a POD copy of the pairs)
                using Pod = PodPair;
                auto pod_first = [](const Pod& a, const Pod& b) { return a.first < b.first; };
                auto to_pod = [](const Pair& q) { return Pod { q.first, q.second }; };
                std::vector<Pod> cpu_pod = api::Merge(pod_first, xs.Map(to_pod), ys.Map(to_pod)).AllGather();
                std::vector<Pair> cpu;
                for (const Pod& q : cpu_pod) cpu.emplace_back(q.first, q.second);
                std::vector<Pair> gpu = thrill_gpu::Merge(thrill_gpu::LessFirst(), xs, ys).AllGather();
                bool keys = cpu.size() == gpu.size();
                for (size_t i = 0; keys && i < cpu.size(); ++i) keys = cpu[i].first == gpu[i].first;
                // the GPU order is exact: within a key, input 0 (values < 10^9) before input 1, each in position order
                bool order = std::is_sorted(gpu.begin(), gpu.end());
                std::sort(cpu.begin(), cpu.end());
                std::vector<Pair> g2 = gpu;
                std::sort(g2.begin(), g2.end());
                Report(ctx, keys && order && cpu == g2, "pairs by LessFirst", n);
            }
        });
    if (rc != 0) return rc;
    return g_failures.load() ? 1 : 0;
}
