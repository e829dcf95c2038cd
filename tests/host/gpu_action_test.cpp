/*******************************************************************************
 * tests/host/gpu_action_test.cpp — Sum / Min / Max / AllReduce / Size of the drop-in INSIDE the unmodified reference.
 *
 * A real Thrill job (api::Run, mock network, THRILL_WORKERS_PER_HOST = number of GPUs): the same DIAs go through the stock
 * DIA::Sum / Min / Max / AllReduce / Size and through thrill_gpu::Sum / Min / Max / AllReduce / Size (GpuAllReduceNode and
 * GpuSizeNode of thrill_b200/host/thrill_gpu_nodes.hpp) with the same functors, and the results are compared EQUAL: integer
 * functions, Min / Max on doubles bit for bit (a NaN first item, +-0 ties, later NaNs), and double sums of integer values, which
 * every bracketing gives exactly.  Two chains check with the transfer counters that no File is fetched to the host:
 * Sort -> Size and ReducePair -> Sum(ScanSecond<std::plus<double>>).  Prints "PASS ..." lines and exits non-zero on any mismatch.
 ******************************************************************************/
#include <thrill/api/all_reduce.hpp>
#include <thrill/api/cache.hpp>
#include <thrill/api/generate.hpp>
#include <thrill/api/max.hpp>
#include <thrill/api/min.hpp>
#include <thrill/api/reduce_by_key.hpp>
#include <thrill/api/size.hpp>
#include <thrill/api/sort.hpp>
#include <thrill/api/sum.hpp>

#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <limits>
#include <utility>

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

static bool Same(double a, double b) { return memcmp(&a, &b, 8) == 0; }
static bool Same(const PairD& a, const PairD& b) { return a.first == b.first && Same(a.second, b.second); }

static double Payload() {
    uint64_t u = 0x7FF8000000012345ull;
    double d;
    memcpy(&d, &u, 8);
    return d;
}

static std::atomic<int> g_failures { 0 };

static void Report(api::Context& ctx, bool ok, const char* what, size_t n) {
    // every worker's verdict counts: a mismatch on any worker fails the line
    ok = ctx.net.AllReduce(static_cast<size_t>(ok ? 0 : 1)) == 0;
    if (ctx.my_rank() == 0) printf("%s Action %s n=%zu workers=%zu\n", ok ? "PASS" : "FAIL", what, n, ctx.num_workers());
    if (!ok && ctx.my_rank() == 0) g_failures++;
}

int main(int argc, char** argv) {
    size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 9999;
    int rc = api::Run(
        [&](api::Context& ctx) {
            using thrill_gpu::MaxU64;
            using thrill_gpu::MinU64;
            using thrill_gpu::ScanSecond;
            // ---- uint64_t items ----
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return splitmix64(i) >> 1; }).Cache().Keep(16);
                auto plus = std::plus<uint64_t>();
                bool ok = in.Sum() == thrill_gpu::Sum(in) && in.Sum(plus, ~0ull) == thrill_gpu::Sum(in, plus, ~0ull) &&
                          in.Min() == thrill_gpu::Min(in) && in.Min(uint64_t(5)) == thrill_gpu::Min(in, uint64_t(5)) &&
                          in.Max() == thrill_gpu::Max(in) && in.Max(~0ull) == thrill_gpu::Max(in, ~0ull) &&
                          in.AllReduce(MinU64()) == thrill_gpu::AllReduce(in, MinU64()) &&
                          in.AllReduce(MaxU64(), uint64_t(3)) == thrill_gpu::AllReduce(in, MaxU64(), uint64_t(3));
                auto f = thrill_gpu::SumFuture(in);
                ok = ok && f.get() == in.Sum() && thrill_gpu::MinFuture(in).get() == in.Min();
                Report(ctx, ok, "uint64_t Sum (wraps) / Min / Max / AllReduce, with and without initial", n);
            }
            // ---- doubles: Min / Max bit for bit, Sum of integer values ----
            {
                const double nan = Payload();
                auto d = api::Generate(ctx, n, [nan](size_t i) {
                    if (i % 7 == 3) return -0.0;
                    if (i % 11 == 5) return 0.0;
                    if (i % 13 == 6) return nan;
                    return double(int64_t(splitmix64(i) % 2001) - 1000);
                }).Cache().Keep(16);
                auto pos = api::Generate(ctx, n, [nan](size_t i) {
                    if (i == 0) return nan;                                 // a NaN first item sticks
                    if (i % 5 == 2) return (i / 5) % 2 ? 0.0 : -0.0;         // +-0 ties in both orders
                    return double(1 + splitmix64(i) % 1000);
                }).Cache().Keep(16);
                auto dplus = std::plus<double>();
                auto ints = api::Generate(ctx, n, [](size_t i) { return double(int64_t(splitmix64(i) % 2000001) - 1000000); })
                            .Cache().Keep(4);
                bool ok = Same(d.Min(), thrill_gpu::Min(d)) && Same(d.Max(), thrill_gpu::Max(d)) &&
                          Same(d.Min(0.5), thrill_gpu::Min(d, 0.5)) && Same(d.Max(nan), thrill_gpu::Max(d, nan)) &&
                          Same(pos.Min(), thrill_gpu::Min(pos)) && Same(pos.Max(-1.0), thrill_gpu::Max(pos, -1.0)) &&
                          Same(ints.Sum(), thrill_gpu::Sum(ints)) && Same(ints.Sum(dplus, -0.5), thrill_gpu::Sum(ints, dplus, -0.5));
                Report(ctx, ok, "double Min / Max bit for bit (NaN, +-0), Sum of integer values", n);
            }
            // ---- pairs ----
            {
                auto names = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i), splitmix64(i + 1) % 4 ? 0 : i + 1); })
                             .Cache().Keep(4);
                auto pd = api::Generate(ctx, n, [](size_t i) { return PairD(i, double(splitmix64(i) % 1001) - 500.0); })
                          .Cache().Keep(8);
                ScanSecond<MaxU64> mx;
                ScanSecond<std::plus<uint64_t> > su;
                ScanSecond<common::minimum<double> > mnd;
                ScanSecond<std::plus<double> > sd;
                bool ok = names.AllReduce(mx) == thrill_gpu::AllReduce(names, mx) &&
                          names.AllReduce(su, Pair(7, 3)) == thrill_gpu::AllReduce(names, su, Pair(7, 3)) &&
                          Same(pd.AllReduce(mnd), thrill_gpu::AllReduce(pd, mnd)) &&
                          Same(pd.AllReduce(mnd, PairD(2, -1e9)), thrill_gpu::AllReduce(pd, mnd, PairD(2, -1e9))) &&
                          Same(pd.AllReduce(sd), thrill_gpu::AllReduce(pd, sd)) &&
                          Same(pd.AllReduce(sd, PairD(5, 0.25)), thrill_gpu::AllReduce(pd, sd, PairD(5, 0.25)));
                Report(ctx, ok, "pair AllReduce ScanSecond<F>, with and without initial", n);
            }
            // ---- Size: a whole File, the per-item PreOp (a Filter on the stack), SizeFuture ----
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return splitmix64(i); }).Cache().Keep(8);
                auto odd = in.Filter([](const uint64_t& x) { return x & 1; });
                bool ok = thrill_gpu::Size(in) == in.Size() && thrill_gpu::SizeFuture(in).get() == n &&
                          thrill_gpu::Size(odd) == odd.Size();
                Report(ctx, ok, "Size / SizeFuture (File and per-item paths)", n);
            }
            // ---- Sort -> Size: no File fetched to the host ----
            {
                auto x = api::Generate(ctx, n, [](size_t i) { return splitmix64(i + 3); }).Cache().Keep(4);
                const size_t cpu = x.Sort().Size();
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                const size_t gpu = thrill_gpu::Size(thrill_gpu::Sort(x));
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers();
                // this worker's input went up once; nothing came down
                Report(ctx, cpu == gpu && gpu == n && h1 - h0 <= 8 * (n / p + 2) && d1 == d0,
                       "Sort -> Size (no File fetched to the host)", n);
            }
            // ---- ReducePair -> Sum(ScanSecond<std::plus<double>>): no File fetched to the host ----
            {
                auto kv = api::Generate(ctx, n, [](size_t i) { return PairD(splitmix64(i) % 1000, double(i % 97) - 48.0); })
                          .Cache().Keep(4);
                ScanSecond<std::plus<double> > sd;
                auto dplus = std::plus<double>();
                const double cpu = kv.ReducePair(dplus).Sum(sd).second;
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                const PairD gpu = thrill_gpu::Sum(thrill_gpu::ReducePair(kv, dplus), sd);
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers();
                Report(ctx, Same(cpu, gpu.second) && h1 - h0 <= 16 * (n / p + 2) && d1 == d0,
                       "ReducePair -> Sum(ScanSecond<std::plus<double>>) (no File fetched to the host)", n);
            }
        });
    if (rc != 0) return rc;
    return g_failures.load() ? 1 : 0;
}
