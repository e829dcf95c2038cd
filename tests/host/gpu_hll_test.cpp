/*******************************************************************************
 * tests/host/gpu_hll_test.cpp — HyperLogLog of the drop-in INSIDE the unmodified reference.
 *
 * A real Thrill job (api::Run, mock network, THRILL_WORKERS_PER_HOST = number of GPUs): the same DIAs go through the stock
 * HyperLogLogNode (api/hyperloglog.hpp) and through thrill_gpu::HyperLogLog / HyperLogLogRegisters (GpuHyperLogLogNode of
 * thrill_b200/host/thrill_gpu_nodes.hpp).  The stock node's registers object tells which format it ended in:
 *   dense   the GPU node's object serializes to the same bytes, and thrill_gpu::HyperLogLog<p>(dia) == dia.HyperLogLog<p>() bit
 *           for bit
 *   sparse  the stock estimate is the sparse one and the GPU's the dense one: both must lie within 3 * 1.04 / sqrt(2^p) of the
 *           distinct count, which the inputs fix by construction; and the stock object made dense (toDense()) serializes to the
 *           GPU node's bytes: the registers are the same either way
 * Also: operator + of two GPU sketches equals the sketch of the union, and Sort -> HyperLogLog fetches no File to the host
 * (transfer counters).  Prints "PASS ..." lines and exits non-zero on any mismatch.
 ******************************************************************************/
#include <thrill/api/cache.hpp>
#include <thrill/api/generate.hpp>
#include <thrill/api/hyperloglog.hpp>
#include <thrill/api/size.hpp>
#include <thrill/api/sort.hpp>

#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
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

static std::atomic<int> g_failures { 0 };

static void Report(api::Context& ctx, bool ok, const std::string& what, size_t n) {
    // every worker's verdict counts: a mismatch on any worker fails the line
    ok = ctx.net.AllReduce(static_cast<size_t>(ok ? 0 : 1)) == 0;
    if (ctx.my_rank() == 0) printf("%s HyperLogLog %s n=%zu workers=%zu\n", ok ? "PASS" : "FAIL", what.c_str(), n, ctx.num_workers());
    if (!ok && ctx.my_rank() == 0) g_failures++;
}

//! the serialized form: the format, then the sparse lists or one uint64_t per register
template <size_t p>
static std::string Bytes(const core::HyperLogLogRegisters<p>& r) {
    net::BufferBuilder bb;
    data::Serialization<net::BufferBuilder, core::HyperLogLogRegisters<p> >::Serialize(r, bb);
    return std::string(reinterpret_cast<const char*>(bb.data()), bb.size());
}

template <size_t p>
static bool IsDense(const core::HyperLogLogRegisters<p>& r) {
    const std::string b = Bytes(r);
    core::HyperLogLogRegisterFormat f;
    memcpy(&f, b.data(), sizeof(f));
    return f == core::HyperLogLogRegisterFormat::DENSE;
}

//! the stock node's registers (DIA::HyperLogLog<p>() keeps only their result())
template <size_t p, typename ValueType, typename Stack>
static core::HyperLogLogRegisters<p> Stock(const api::DIA<ValueType, Stack>& dia) {
    auto node = tlx::make_counting<api::HyperLogLogNode<p, ValueType> >(dia, "HyperLogLog");
    node->RunScope();
    return node->result();
}

//! dia needs 4 uses left.  Returns the verdict; *dense says which comparison it was
template <size_t p, typename ValueType, typename Stack>
static bool Compare(const api::DIA<ValueType, Stack>& dia, double distinct, bool* dense) {
    core::HyperLogLogRegisters<p> stock = Stock<p>(dia);
    core::HyperLogLogRegisters<p> gpu = thrill_gpu::HyperLogLogRegisters<p>(dia);
    const double est_stock = dia.template HyperLogLog<p>(), est_gpu = thrill_gpu::HyperLogLog<p>(dia);
    *dense = IsDense(stock);
    if (!IsDense(gpu) || !Same(est_gpu, gpu.result())) return false;
    if (*dense) return Bytes(stock) == Bytes(gpu) && Same(est_stock, est_gpu);
    const double tol = 3 * 1.04 / std::sqrt(static_cast<double>(size_t(1) << p));
    stock.toDense();
    return Bytes(stock) == Bytes(gpu) && std::fabs(est_stock / distinct - 1) <= tol && std::fabs(est_gpu / distinct - 1) <= tol;
}

template <size_t p, typename ValueType, typename Stack>
static void Line(api::Context& ctx, const api::DIA<ValueType, Stack>& dia, double distinct, const char* what, size_t n) {
    bool dense = false;
    const bool ok = Compare<p>(dia, distinct, &dense);
    // the workers agree on the format: the sum is one object
    Report(ctx, ok, std::string(what) + " p=" + std::to_string(p) + (dense ? " (stock ends dense: bit for bit)"
                                                                          : " (stock ends sparse: registers equal, estimates near)"), n);
}

int main(int argc, char** argv) {
    size_t n = argc > 1 ? strtoull(argv[1], nullptr, 10) : 9999;
    int rc = api::Run(
        [&](api::Context& ctx) {
            // ---- uint64_t items, all distinct ----
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return splitmix64(i); }).Cache().Keep(24);
                Line<4>(ctx, in, double(n), "uint64_t distinct", n);
                Line<8>(ctx, in, double(n), "uint64_t distinct", n);
                Line<12>(ctx, in, double(n), "uint64_t distinct", n);
                Line<14>(ctx, in, double(n), "uint64_t distinct", n);
                Line<16>(ctx, in, double(n), "uint64_t distinct", n);
                Line<18>(ctx, in, double(n), "uint64_t distinct", n);
            }
            // ---- doubles with heavy duplicates: min(n, 1000) distinct values, hashed as their bits ----
            {
                auto d = api::Generate(ctx, n, [](size_t i) { return double(i % 1000) * 0.125 - 50.0; })
                         .Cache().Keep(8);
                const double distinct = double(n < 1000 ? n : 1000);
                Line<10>(ctx, d, distinct, "double, 1000 distinct", n);
                Line<17>(ctx, d, distinct, "double, 1000 distinct", n);
            }
            // ---- pairs: 16 message bytes ----
            {
                auto kv = api::Generate(ctx, n, [](size_t i) { return Pair(splitmix64(i), i % 3); }).Cache().Keep(8);
                auto kd = api::Generate(ctx, n, [](size_t i) { return PairD(i, double(i % 7) - 3.0); }).Cache().Keep(8);
                Line<12>(ctx, kv, double(n), "pair<uint64_t, uint64_t> distinct", n);
                Line<16>(ctx, kv, double(n), "pair<uint64_t, uint64_t> distinct", n);
                Line<9>(ctx, kd, double(n), "pair<uint64_t, double> distinct", n);
                Line<15>(ctx, kd, double(n), "pair<uint64_t, double> distinct", n);
            }
            // ---- the per-item PreOp (a Filter on the stack) ----
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return splitmix64(i + 11); }).Cache().Keep(5);
                auto odd = in.Filter([](const uint64_t& x) { return x & 1; });
                const double distinct = double(odd.Size());
                Line<11>(ctx, odd, distinct, "uint64_t through a Filter (per-item PreOp)", n);
            }
            // ---- operator + of two GPU sketches is the sketch of the union ----
            {
                auto in = api::Generate(ctx, n, [](size_t i) { return splitmix64(i + 5); }).Cache().Keep(3);
                auto lo = in.Filter([](const uint64_t& x) { return x % 3 == 0; });
                auto hi = in.Filter([](const uint64_t& x) { return x % 3 != 0; });
                auto sum = thrill_gpu::HyperLogLogRegisters<13>(lo) + thrill_gpu::HyperLogLogRegisters<13>(hi);
                auto all = thrill_gpu::HyperLogLogRegisters<13>(in);
                Report(ctx, Bytes(sum) == Bytes(all) && Same(sum.result(), all.result()), "operator + of two sketches = the union's", n);
            }
            // ---- Sort -> HyperLogLog: no File fetched to the host ----
            {
                auto x = api::Generate(ctx, n, [](size_t i) { return splitmix64(i + 3); }).Cache().Keep(2);
                auto stock = Stock<14>(x.Sort());
                if (!IsDense(stock)) stock.toDense();
                uint64_t h0 = 0, d0 = 0, h1 = 0, d1 = 0;
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h0, &d0);
                auto gpu = thrill_gpu::HyperLogLogRegisters<14>(thrill_gpu::Sort(x));
                tg_transfer_bytes(thrill_gpu::WorkerCtx(ctx), &h1, &d1);
                const size_t p = ctx.num_workers();
                // this worker's input went up once; no File came down
                Report(ctx, Bytes(stock) == Bytes(gpu) && h1 - h0 <= 8 * (n / p + 2) && d1 == d0,
                       "Sort -> HyperLogLog (no File fetched to the host)", n);
            }
        });
    if (rc != 0) return rc;
    return g_failures.load() ? 1 : 0;
}
