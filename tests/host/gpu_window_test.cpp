/*******************************************************************************
 * tests/host/gpu_window_test.cpp — Window of the drop-in INSIDE the unmodified reference.
 *
 * A real Thrill job (api::Run, mock network, THRILL_WORKERS_PER_HOST = number of GPUs): the same DIAs go through the stock
 * DIA::Window(k, f), Window(k, f, partial_f) and Window(DisjointTag, k, f) and through thrill_gpu::Window (GpuWindowNode of
 * thrill_b200/host/thrill_gpu_nodes.hpp) with the same functors (WindowFold<F>, DisjointFold<F>), and the gathered outputs are
 * compared EQUAL: integer functions and Min / Max on doubles bit for bit (NaN first items, NaNs inside, +-0 ties), double sums
 * of integer values, which every bracketing gives exactly.  A Sort -> Window -> Sum chain checks with the transfer counters that
 * the input goes up once and nothing but the value comes down.  A window size outside 2..4096 (0, 1, 4097, 2^32) is a die() on
 * every rank when the node executes, through each front door.  Prints "PASS ..." lines and exits non-zero on any mismatch.
 ******************************************************************************/
#include <thrill/api/all_gather.hpp>
#include <thrill/api/cache.hpp>
#include <thrill/api/generate.hpp>
#include <thrill/api/size.hpp>
#include <thrill/api/sort.hpp>
#include <thrill/api/sum.hpp>
#include <thrill/api/window.hpp>

#include <tlx/die.hpp>

#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
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

template <typename T>
static bool SameBytes(const std::vector<T>& a, const std::vector<T>& b) {
    return a.size() == b.size() && (a.empty() || memcmp(a.data(), b.data(), a.size() * sizeof(T)) == 0);
}

static std::atomic<int> g_failures { 0 };

static void Report(api::Context& ctx, bool ok, const char* what, size_t n) {
    ok = ctx.net.AllReduce(static_cast<size_t>(ok ? 0 : 1)) == 0;
    if (ctx.my_rank() == 0) printf("%s Window %s n=%zu workers=%zu\n", ok ? "PASS" : "FAIL", what, n, ctx.num_workers());
    if (!ok && ctx.my_rank() == 0) g_failures++;
}

//! the three forms, stock and GPU, with the same functors; every output gathered in order
template <typename F, typename DIAType>
static bool AllForms(const DIAType& in, size_t k) {
    using thrill_gpu::DisjointFold;
    using thrill_gpu::WindowFold;
    bool ok = SameBytes(in.Window(k, WindowFold<F>()).AllGather(), thrill_gpu::Window(in, k, WindowFold<F>()).AllGather());
    ok = ok && SameBytes(in.Window(k, WindowFold<F>(), WindowFold<F>()).AllGather(),
                         thrill_gpu::Window(in, k, WindowFold<F>(), WindowFold<F>()).AllGather());
    ok = ok && SameBytes(in.Window(api::DisjointTag, k, DisjointFold<F>()).AllGather(),
                         thrill_gpu::Window(api::DisjointTag, in, k, DisjointFold<F>()).AllGather());
    return ok;
}

int main(int argc, char** argv) {
    size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 9999;
    int rc = api::Run(
        [&](api::Context& ctx) {
            using thrill_gpu::MaxU64;
            using thrill_gpu::MinU64;
            using thrill_gpu::ScanSecond;
            const size_t ks[] = { 2, 3, 64, 4096 };
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return i % 3 ? splitmix64(i) : splitmix64(i) % 50; }).Cache().Keep(64);
                bool ok = true;
                for (size_t k : ks)
                    ok = ok && AllForms<std::plus<uint64_t> >(in, k) && AllForms<MinU64>(in, k) &&
                         AllForms<common::maximum<uint64_t> >(in, k);
                Report(ctx, ok, "uint64_t std::plus (wraps) / MinU64 / common::maximum, k = 2, 3, 64, 4096", n);
            }
            {
                uint64_t u = 0x7FF8000000012345ull;
                double nan;
                memcpy(&nan, &u, 8);
                auto d = api::Generate(ctx, n, [nan](size_t i) {
                    if (i % 7 == 3) return -0.0;
                    if (i % 11 == 5) return 0.0;
                    if (i % 13 == 6) return nan;
                    return double(int64_t(splitmix64(i) % 2001) - 1000);
                }).Cache().Keep(64);
                bool ok = true;
                for (size_t k : ks)
                    ok = ok && AllForms<common::minimum<double> >(d, k) && AllForms<common::maximum<double> >(d, k);
                auto ints = api::Generate(ctx, n, [](size_t i) { return double(int64_t(splitmix64(i) % 2001) - 1000); }).Cache().Keep(16);
                for (size_t k : ks) ok = ok && AllForms<std::plus<double> >(ints, k);
                Report(ctx, ok, "double Min / Max bit for bit (NaN, +-0), Sum of integer values", n);
            }
            {
                auto pu = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i), splitmix64(i + 1) >> 3); }).Cache().Keep(16);
                auto pd = api::Generate(ctx, n, [](size_t i) { return PairD(i, double(splitmix64(i) % 1001) - 500.0); }).Cache().Keep(16);
                bool ok = true;
                for (size_t k : { size_t(5), size_t(64) })
                    ok = ok && AllForms<ScanSecond<MaxU64> >(pu, k) && AllForms<ScanSecond<std::plus<uint64_t> > >(pu, k) &&
                         AllForms<ScanSecond<common::minimum<double> > >(pd, k) && AllForms<ScanSecond<std::plus<double> > >(pd, k);
                Report(ctx, ok, "pair ScanSecond<F> (.first of the window's last item)", n);
            }
            {
                auto x = api::Generate(ctx, n, [](size_t i) { return splitmix64(i + 3) >> 20; }).Cache().Keep(4);
                thrill_gpu::WindowFold<std::plus<uint64_t> > wf;
                const uint64_t cpu = x.Sort().Window(64, wf).Sum();
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                const uint64_t gpu = thrill_gpu::Sum(thrill_gpu::Window(thrill_gpu::Sort(x), 64, wf));
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers();
                Report(ctx, cpu == gpu && h1 - h0 <= 8 * (n / p + 2) && d1 == d0,
                       "Sort -> Window -> Sum (the input up once, nothing but the value down)", n);
            }
            {
                // a bad window size: every front door dies on every rank (the library's TG_ERR_ARG), and the ctx keeps working
                // (a fresh parent for every call: no failed node stays a child of a DIA that is read again)
                auto fresh = [&ctx, n] { return api::Generate(ctx, n, [](size_t i) { return splitmix64(i); }); };
                thrill_gpu::WindowFold<std::plus<uint64_t> > wf;
                thrill_gpu::DisjointFold<std::plus<uint64_t> > df;
                auto dies = [](auto&& run) {
                    try { run(); }
                    catch (const tlx::DieException&) { return true; }
                    return false;
                };
                bool ok = true;
                for (size_t k : { size_t(0), size_t(1), size_t(4097), size_t(1) << 32 }) {
                    ok = dies([&] { thrill_gpu::Window(fresh(), k, wf).Size(); }) && ok;
                    ok = dies([&] { thrill_gpu::Window(fresh(), k, wf, wf).Size(); }) && ok;
                    ok = dies([&] { thrill_gpu::Window(api::DisjointTag, fresh(), k, df).Size(); }) && ok;
                }
                ok = ok && SameBytes(fresh().Window(2, wf).AllGather(), thrill_gpu::Window(fresh(), 2, wf).AllGather());
                Report(ctx, ok, "window sizes 0, 1, 4097 and 2^32 die on every rank through every front door", n);
            }
        });
    if (rc != 0) return rc;
    return g_failures.load() ? 1 : 0;
}
