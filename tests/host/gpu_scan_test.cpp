/*******************************************************************************
 * tests/host/gpu_scan_test.cpp — PrefixSum / ExPrefixSum / ZipWithIndex of the drop-in INSIDE the unmodified reference.
 *
 * A real Thrill job (api::Run, mock network, THRILL_WORKERS_PER_HOST = number of GPUs): the same DIAs go through the stock
 * DIA::PrefixSum / ExPrefixSum / ZipWithIndex and through thrill_gpu::PrefixSum / ExPrefixSum / ZipWithIndex (GpuScanNode of
 * thrill_b200/host/thrill_gpu_nodes.hpp) with the same functors, and the gathered results are compared EQUAL (integer sums, and
 * double sums of integer values, which every bracketing gives exactly).  Two chains check with the transfer counters that
 * nothing crosses PCIe between GPU nodes: SortStable -> ZipWithIndex(IndexFirst) -> ReducePair and
 * Sort -> PrefixSum(ScanSecond<MaxU64>).  Mirrors the PrefixSum and ZipWithIndex tests of tests/api/operations_test.cpp and
 * zip_node_test.cpp of the reference.  Prints "PASS ..." lines and exits non-zero on any mismatch.
 ******************************************************************************/
#include <thrill/api/all_gather.hpp>
#include <thrill/api/cache.hpp>
#include <thrill/api/ex_prefix_sum.hpp>
#include <thrill/api/generate.hpp>
#include <thrill/api/prefix_sum.hpp>
#include <thrill/api/reduce_by_key.hpp>
#include <thrill/api/sort.hpp>
#include <thrill/api/zip_with_index.hpp>

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
using PairD = std::pair<uint64_t, double>;

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
    if (ctx.my_rank() == 0) printf("%s Scan %s n=%zu workers=%zu\n", ok ? "PASS" : "FAIL", what, n, ctx.num_workers());
    if (!ok && ctx.my_rank() == 0) g_failures++;
}

template <typename T>
static std::vector<T> Sorted(std::vector<T> v) {
    std::sort(v.begin(), v.end());
    return v;
}

int main(int argc, char** argv) {
    size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 9999;
    int rc = api::Run(
        [&](api::Context& ctx) {
            using thrill_gpu::MaxU64;
            using thrill_gpu::MinU64;
            using thrill_gpu::ScanSecond;
            // ---- uint64_t and double items ----
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return splitmix64(i) >> 3; }).Cache().Keep(8);
                auto plus = std::plus<uint64_t>();
                Report(ctx, in.PrefixSum(plus, 12345).AllGather() == thrill_gpu::PrefixSum(in, plus, uint64_t(12345)).AllGather(),
                       "PrefixSum std::plus<uint64_t> (wraps), initial 12345", n);
                Report(ctx, in.ExPrefixSum(MinU64(), ~0ull).AllGather() == thrill_gpu::ExPrefixSum(in, MinU64(), ~0ull).AllGather(),
                       "ExPrefixSum MinU64, initial ~0", n);
                Report(ctx, in.PrefixSum(MaxU64()).AllGather() == thrill_gpu::PrefixSum(in, MaxU64()).AllGather(),
                       "PrefixSum MaxU64", n);
                auto d = api::Generate(ctx, n, [](size_t i) { return double(int64_t(splitmix64(i) % 2000001) - 1000000); })
                         .Cache().Keep(8);
                auto dplus = std::plus<double>();
                Report(ctx, d.ExPrefixSum(dplus, -0.5).AllGather() == thrill_gpu::ExPrefixSum(d, dplus, -0.5).AllGather(),
                       "ExPrefixSum std::plus<double> of integer values", n);
            }
            // ---- pairs: prefix doubling's names, and a double sum on .second ----
            {
                auto names = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i), splitmix64(i + 1) % 4 ? 0 : i + 1); })
                             .Cache().Keep(8);
                ScanSecond<MaxU64> mx;
                Report(ctx, names.PrefixSum(mx).AllGather() == thrill_gpu::PrefixSum(names, mx).AllGather() &&
                       names.ExPrefixSum(mx, Pair(7, 3)).AllGather() == thrill_gpu::ExPrefixSum(names, mx, Pair(7, 3)).AllGather(),
                       "PrefixSum / ExPrefixSum ScanSecond<MaxU64>", n);
                auto pd = api::Generate(ctx, n, [](size_t i) { return PairD(i, double(splitmix64(i) % 1001) - 500.0); })
                          .Cache().Keep(8);
                ScanSecond<std::plus<double> > sd;
                Report(ctx, pd.ExPrefixSum(sd, PairD(5, 0.25)).AllGather() == thrill_gpu::ExPrefixSum(pd, sd, PairD(5, 0.25)).AllGather(),
                       "ExPrefixSum ScanSecond<std::plus<double>> of integer values", n);
            }
            // ---- ZipWithIndex, both forms ----
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return splitmix64(i + 9); }).Cache().Keep(8);
                auto first = in.ZipWithIndex([](const uint64_t& x, const size_t& i) { return Pair(i, x); }).AllGather();
                auto second = in.ZipWithIndex([](const uint64_t& x, const size_t& i) { return Pair(x, i); }).AllGather();
                Report(ctx, first == thrill_gpu::ZipWithIndex(in, thrill_gpu::IndexFirst()).AllGather() &&
                       second == thrill_gpu::ZipWithIndex(in, thrill_gpu::IndexSecond()).AllGather(),
                       "ZipWithIndex IndexFirst and IndexSecond", n);
            }
            // ---- SortStable -> ZipWithIndex(IndexFirst) -> ReducePair: device-resident in between ----
            {
                auto x = api::Generate(ctx, n, [](size_t i) { return splitmix64(i + 3) % 5000; }).Cache().Keep(8);
                auto plus = std::plus<uint64_t>();
                auto cpu = Sorted(x.SortStable().ZipWithIndex([](const uint64_t& v, const size_t& i) { return Pair(i / 3, v); })
                                  .ReducePair(plus).AllGather());
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                auto z = thrill_gpu::ZipWithIndex(thrill_gpu::SortStable(x), thrill_gpu::IndexFirst());
                auto r = thrill_gpu::ReducePair(z, plus);
                std::vector<Pair> gpu = r.AllGather();
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers();
                // this worker's input went up once; only the reduced items came down
                bool lean = h1 - h0 <= 8 * (n / p + 2) && d1 - d0 <= 16 * (gpu.size() + 2);
                auto cpu_direct = Sorted(x.SortStable().ZipWithIndex([](const uint64_t& v, const size_t& i) { return Pair(i, v); })
                                         .ReducePair(plus).AllGather());
                Report(ctx, Sorted(gpu) == cpu_direct && lean && cpu.size() == (n + 2) / 3,
                       "SortStable -> ZipWithIndex(IndexFirst) -> ReducePair (device-resident in between)", n);
            }
            // ---- Sort -> PrefixSum(ScanSecond<MaxU64>): device-resident in between ----
            {
                // distinct keys (an odd multiplier permutes 2^64), so every sort gives the same order
                auto x = api::Generate(ctx, n, [](size_t i) {
                    return Pair(uint64_t(i) * 0x9E3779B97F4A7C15ull, splitmix64(i) % 3 ? 0 : i); }).Cache().Keep(8);
                ScanSecond<MaxU64> mx;
                auto cpu = x.Sort([](const Pair& a, const Pair& b) { return a.first < b.first; }).PrefixSum(mx).AllGather();
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                auto gpu = thrill_gpu::PrefixSum(thrill_gpu::Sort(x, thrill_gpu::LessFirst()), mx).AllGather();
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers();
                bool lean = h1 - h0 <= 16 * (n / p + 2) && d1 - d0 <= 16 * n;
                Report(ctx, cpu == gpu && lean && cpu.size() == n, "Sort -> PrefixSum(ScanSecond<MaxU64>) (device-resident in between)", n);
            }
        });
    if (rc != 0) return rc;
    return g_failures.load() ? 1 : 0;
}
