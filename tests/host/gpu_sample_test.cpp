/*******************************************************************************
 * tests/host/gpu_sample_test.cpp — Sample and BernoulliSample of the drop-in INSIDE the unmodified reference.
 *
 * A real Thrill job (api::Run, mock network, THRILL_WORKERS_PER_HOST = number of GPUs) runs thrill_gpu::Sample and
 * thrill_gpu::BernoulliSample (GpuSampleNode of thrill_b200/host/thrill_gpu_nodes.hpp):
 *   - the stock Operations.Sample cases (tests/api/operations_test.cpp:840-879): 100 of 9999, 20000 of 9999 (everything) and
 *     100 of a filtered, unbalanced input, each with the sizes the stock test asserts and distinct items from the input;
 *   - seeded results equal to the model of include/thrill_gpu.h (key(seed, g), the s smallest keys / u < p), gathered in order;
 *   - points.Sample(10).AllGather() with a 24-byte point type;
 *   - Sort -> Sample -> Sum and Sort -> BernoulliSample -> Size, which move nothing over PCIe between the nodes (tg_transfer_bytes);
 *   - a probability outside [0, 1] or NaN is a die() on every rank when the node executes.
 * Prints "PASS ..." lines and exits non-zero on any mismatch.
 ******************************************************************************/
#include <thrill/api/all_gather.hpp>
#include <thrill/api/cache.hpp>
#include <thrill/api/generate.hpp>
#include <thrill/api/size.hpp>
#include <thrill/api/sort.hpp>
#include <thrill/api/sum.hpp>

#include <tlx/die.hpp>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <vector>

#include "../../thrill_b200/host/thrill_gpu_nodes.hpp"

using namespace thrill; // NOLINT

static constexpr uint64_t kGamma = 0x9E3779B97F4A7C15ull;

static inline uint64_t mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static inline uint64_t key(uint64_t seed, uint64_t g) { return mix(mix(seed) + (g + 1) * kGamma); }

//! the kept global positions of Sample(s) / BernoulliSample(p) of N items, ascending
static std::vector<size_t> KeptSample(uint64_t seed, size_t N, size_t s) {
    std::vector<size_t> out;
    if (s >= N) { for (size_t g = 0; g < N; ++g) out.push_back(g); return out; }
    if (s == 0) return out;
    std::vector<uint64_t> k(N);
    for (size_t g = 0; g < N; ++g) k[g] = key(seed, g);
    std::vector<uint64_t> t = k;
    std::nth_element(t.begin(), t.begin() + (s - 1), t.end());
    for (size_t g = 0; g < N; ++g) if (k[g] <= t[s - 1]) out.push_back(g);
    return out;
}
static std::vector<size_t> KeptBernoulli(uint64_t seed, size_t N, double p) {
    const uint64_t t = static_cast<uint64_t>(std::ceil(std::ldexp(p, 53)));
    std::vector<size_t> out;
    for (size_t g = 0; g < N; ++g) if ((key(seed, g) >> 11) < t) out.push_back(g);
    return out;
}

struct Point { double x, y, z; };

static std::atomic<int> g_failures { 0 };

static void Report(api::Context& ctx, bool ok, const char* what) {
    ok = ctx.net.AllReduce(static_cast<size_t>(ok ? 0 : 1)) == 0;
    if (ctx.my_rank() == 0) printf("%s Sample %s workers=%zu\n", ok ? "PASS" : "FAIL", what, ctx.num_workers());
    if (!ok && ctx.my_rank() == 0) g_failures++;
}

static bool Distinct(std::vector<size_t> v, size_t below) {
    std::sort(v.begin(), v.end());
    return std::adjacent_find(v.begin(), v.end()) == v.end() && (v.empty() || v.back() < below);
}

int main() {
    int rc = api::Run(
        [&](api::Context& ctx) {
            const size_t n = 9999;
            {
                auto a = thrill_gpu::Sample(api::Generate(ctx, n), 100);
                std::vector<size_t> va = a.AllGather();
                bool ok = a.Size() == 100 && va.size() == 100 && Distinct(va, n);
                auto b = thrill_gpu::Sample(api::Generate(ctx, n), 20000);
                std::vector<size_t> vb = b.AllGather();
                ok = ok && b.Size() == 9999 && vb.size() == 9999;
                for (size_t i = 0; ok && i < vb.size(); ++i) ok = vb[i] == i;           // everything, in input order
                auto c = thrill_gpu::Sample(api::Generate(ctx, 1000).Filter([](size_t i) { return i < 80 || i % 10 == 1; }), 100);
                std::vector<size_t> vc = c.AllGather();
                ok = ok && c.Size() == 100 && vc.size() == 100 && Distinct(vc, 1000);
                for (size_t x : vc) ok = ok && (x < 80 || x % 10 == 1);
                Report(ctx, ok, "the stock Operations.Sample cases: 100 of 9999, 20000 of 9999, 100 of a filtered input");
            }
            {
                bool ok = true;
                for (uint64_t seed : { uint64_t(0), uint64_t(12345), ~uint64_t(0) }) {
                    for (size_t s : { size_t(1), size_t(10), size_t(4097), n - 1 })
                        ok = ok && thrill_gpu::Sample(api::Generate(ctx, n), s, seed).AllGather() == KeptSample(seed, n, s);
                    for (double p : { 0.0, 0.05, 0.3, 1.0 })
                        ok = ok && thrill_gpu::BernoulliSample(api::Generate(ctx, n), p, seed).AllGather() == KeptBernoulli(seed, n, p);
                }
                // a filtered (unbalanced) input: the model's positions are those of the filtered DIA
                std::vector<size_t> f;
                for (size_t i = 0; i < 1000; ++i) if (i < 80 || i % 10 == 1) f.push_back(i);
                std::vector<size_t> want;
                for (size_t g : KeptSample(7, f.size(), 100)) want.push_back(f[g]);
                ok = ok && thrill_gpu::Sample(api::Generate(ctx, 1000).Filter([](size_t i) { return i < 80 || i % 10 == 1; }), 100, 7)
                               .AllGather() == want;
                Report(ctx, ok, "seeded Sample / BernoulliSample equal to the model");
            }
            {
                auto points = api::Generate(ctx, 5000, [](size_t i) { return Point { double(i), -double(i), 0.5 * double(i) }; }).Cache();
                std::vector<Point> v = thrill_gpu::Sample(points, 10).AllGather();
                bool ok = v.size() == 10;
                for (const Point& q : v) ok = ok && q.y == -q.x && q.z == 0.5 * q.x && q.x >= 0 && q.x < 5000;
                std::vector<Point> w = thrill_gpu::Sample(points, 10, 99).AllGather();
                std::vector<size_t> kept = KeptSample(99, 5000, 10);
                for (size_t i = 0; ok && i < kept.size(); ++i) ok = w.size() == 10 && w[i].x == double(kept[i]);
                Report(ctx, ok, "points.Sample(10).AllGather() of 24-byte points");
            }
            {
                const size_t m = 200000;
                auto x = api::Generate(ctx, m, [](size_t i) { return mix(i + 11) >> 20; }).Cache().Keep(4);
                std::vector<uint64_t> sorted = x.Sort().AllGather();
                uint64_t want = 0;
                for (size_t g : KeptSample(5, m, 1000)) want += sorted[g];
                const size_t want_n = KeptBernoulli(6, m, 0.01).size();
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                const uint64_t sum = thrill_gpu::Sum(thrill_gpu::Sample(thrill_gpu::Sort(x), 1000, 5));
                const size_t cnt = thrill_gpu::Size(thrill_gpu::BernoulliSample(thrill_gpu::Sort(x), 0.01, 6));
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers();
                Report(ctx, sum == want && cnt == want_n && h1 - h0 <= 2 * 8 * (m / p + 2) && d1 == d0,
                       "Sort -> Sample -> Sum and Sort -> BernoulliSample -> Size (the input up once per chain, nothing down)");
            }
            {
                auto fresh = [&ctx, n] { return api::Generate(ctx, n); };
                auto dies = [](auto&& run) {
                    try { run(); }
                    catch (const tlx::DieException&) { return true; }
                    return false;
                };
                bool ok = true;
                for (double p : { -0.5, 1.5, std::numeric_limits<double>::quiet_NaN(), std::numeric_limits<double>::infinity() })
                    ok = dies([&] { thrill_gpu::BernoulliSample(fresh(), p).Size(); }) && ok;
                ok = ok && thrill_gpu::BernoulliSample(fresh(), 1.0).Size() == n;
                Report(ctx, ok, "BernoulliSample with p outside [0, 1] or NaN dies on every rank");
            }
        });
    if (rc != 0) return rc;
    return g_failures.load() ? 1 : 0;
}
