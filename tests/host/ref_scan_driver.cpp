/*******************************************************************************
 * tests/host/ref_scan_driver.cpp — TEST INFRASTRUCTURE: the stock DIA::PrefixSum / DIA::ExPrefixSum / DIA::ZipWithIndex of the
 * UNMODIFIED reference.
 *
 * Links the reference library built by oracle/ref/Makefile.  Every worker reads the whole binary input and places its own shard
 * with ConcatToDIA (api/concat_to_dia.hpp:77-84): worker r takes the count_r items after count_0 + ... + count_{r-1}, so the
 * caller chooses the per-worker sizes, empty workers included.  Then one operator runs on the DIA:
 *   sum_u64 / min_u64 / max_u64   uint64_t items, PrefixSum(fn, initial) (api/dia.hpp:1850) with std::plus<uint64_t>, min, max
 *   sum_f64                       double items, std::plus<double>
 *   pair_max / pair_sum_f64       pair<uint64_t, uint64_t> / pair<uint64_t, double> items with
 *                                 (a, b) -> (b.first, F(a.second, b.second)), F = max or std::plus<double>
 *   zip_first / zip_second        uint64_t items, ZipWithIndex (api/zip_with_index.hpp:140) giving (index, item) / (item, index)
 * incl|excl picks PrefixSum or ExPrefixSum (api/dia.hpp:1867).  A Map child writes each worker's rank beside its outputs and
 * Gather(0) keeps the worker order, so the output file holds rows of 3 uint64_t: (rank, first word, second word) of every output
 * item (an 8-byte item has first word 0; doubles are written as their bits).  Generates the fixtures of
 * tests/golden/make_golden_scan.py.
 *
 * usage: THRILL_NET=mock THRILL_LOCAL=1 THRILL_WORKERS_PER_HOST=W ref_scan_driver in.bin out.bin mode incl|excl init_first
 *        init_second count_0 ... count_{W-1}
 ******************************************************************************/
#include <thrill/api/collapse.hpp>
#include <thrill/api/concat_to_dia.hpp>
#include <thrill/api/ex_prefix_sum.hpp>
#include <thrill/api/gather.hpp>
#include <thrill/api/prefix_sum.hpp>
#include <thrill/api/zip_with_index.hpp>

#include <array>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <utility>
#include <vector>

using namespace thrill; // NOLINT

using Row = std::array<uint64_t, 3>;

struct MinU64 { uint64_t operator () (uint64_t a, uint64_t b) const { return b < a ? b : a; } };
struct MaxU64 { uint64_t operator () (uint64_t a, uint64_t b) const { return a < b ? b : a; } };
//! a plain functor (the stock node reads its argument type), as thrill_gpu::ScanSecond is
template <typename M> struct MemberResult;
template <typename R, typename C, typename... A>
struct MemberResult<R (C::*)(A...) const> { using type = R; };
template <typename F>
struct ScanSecond {
    using P = std::pair<uint64_t, typename MemberResult<decltype(&F::operator ())>::type>;
    F fn;
    P operator () (const P& a, const P& b) const { return P(b.first, fn(a.second, b.second)); }
};

static uint64_t bits(double d) { uint64_t u; memcpy(&u, &d, 8); return u; }
static double dbl(uint64_t u) { double d; memcpy(&d, &u, 8); return d; }

//! this worker's shard of the input (as words): counts[r] items of `words` words each
static std::vector<uint64_t> Shard(const std::vector<uint64_t>& all, const std::vector<size_t>& counts, size_t rank,
                                   size_t words) {
    size_t begin = 0;
    for (size_t r = 0; r < rank; ++r) begin += counts[r];
    return std::vector<uint64_t>(all.begin() + begin * words, all.begin() + (begin + counts[rank]) * words);
}

int main(int argc, char** argv) {
    if (argc < 8) {
        fprintf(stderr, "usage: %s in.bin out.bin mode incl|excl init_first init_second count_0 ... count_{W-1}\n", argv[0]);
        return 2;
    }
    const std::string in_path = argv[1], out_path = argv[2], mode = argv[3];
    const bool incl = !strcmp(argv[4], "incl");
    const uint64_t init_first = strtoull(argv[5], nullptr, 10), init_second = strtoull(argv[6], nullptr, 10);
    std::vector<size_t> counts;
    for (int i = 7; i < argc; ++i) counts.push_back(strtoull(argv[i], nullptr, 10));
    std::vector<uint64_t> words;
    {
        FILE* f = fopen(in_path.c_str(), "rb");
        if (!f) { perror("fopen in"); return 2; }
        uint64_t w;
        while (fread(&w, 8, 1, f) == 1) words.push_back(w);
        fclose(f);
    }
    return api::Run(
        [&](api::Context& ctx) {
            if (counts.size() != ctx.num_workers()) {
                fprintf(stderr, "%zu counts for %zu workers\n", counts.size(), ctx.num_workers());
                exit(2);
            }
            const size_t rank = ctx.my_rank();
            const bool pair = mode.compare(0, 5, "pair_") == 0;
            const std::vector<uint64_t> mine = Shard(words, counts, rank, pair ? 2 : 1);
            std::vector<Row> all;
            auto tag = [&ctx](Row r) { r[0] = ctx.my_rank(); return r; };
            auto scan = [&](auto dia, auto fn, auto initial, auto to_row) {
                auto res = incl ? dia.PrefixSum(fn, initial).Map(to_row).Collapse()
                                : dia.ExPrefixSum(fn, initial).Map(to_row).Collapse();
                return res.Map(tag).Gather(0);
            };
            if (mode == "sum_u64" || mode == "min_u64" || mode == "max_u64") {
                auto dia = api::ConcatToDIA(ctx, mine);
                auto to_row = [](const uint64_t& x) { return Row { { 0, 0, x } }; };
                if (mode == "sum_u64") all = scan(dia, std::plus<uint64_t>(), init_second, to_row);
                else if (mode == "min_u64") all = scan(dia, MinU64(), init_second, to_row);
                else all = scan(dia, MaxU64(), init_second, to_row);
            }
            else if (mode == "sum_f64") {
                std::vector<double> d;
                for (uint64_t w : mine) d.push_back(dbl(w));
                auto to_row = [](const double& x) { return Row { { 0, 0, bits(x) } }; };
                all = scan(api::ConcatToDIA(ctx, d), std::plus<double>(), dbl(init_second), to_row);
            }
            else if (mode == "pair_max") {
                using P = std::pair<uint64_t, uint64_t>;
                std::vector<P> v;
                for (size_t i = 0; i < mine.size(); i += 2) v.emplace_back(mine[i], mine[i + 1]);
                auto to_row = [](const P& x) { return Row { { 0, x.first, x.second } }; };
                all = scan(api::ConcatToDIA(ctx, v), ScanSecond<MaxU64>(), P(init_first, init_second), to_row);
            }
            else if (mode == "pair_sum_f64") {
                using P = std::pair<uint64_t, double>;
                std::vector<P> v;
                for (size_t i = 0; i < mine.size(); i += 2) v.emplace_back(mine[i], dbl(mine[i + 1]));
                auto to_row = [](const P& x) { return Row { { 0, x.first, bits(x.second) } }; };
                all = scan(api::ConcatToDIA(ctx, v), ScanSecond<std::plus<double> >(), P(init_first, dbl(init_second)), to_row);
            }
            else if (mode == "zip_first" || mode == "zip_second") {
                auto dia = api::ConcatToDIA(ctx, mine);
                if (mode == "zip_first")
                    all = dia.ZipWithIndex([](const uint64_t& x, const size_t& i) { return Row { { 0, i, x } }; }).Map(tag).Gather(0);
                else
                    all = dia.ZipWithIndex([](const uint64_t& x, const size_t& i) { return Row { { 0, x, i } }; }).Map(tag).Gather(0);
            }
            else {
                fprintf(stderr, "unknown mode %s\n", mode.c_str());
                exit(2);
            }
            if (rank != 0) return;
            FILE* f = fopen(out_path.c_str(), "wb");
            if (!f) { perror("fopen out"); exit(2); }
            for (const Row& r : all) fwrite(r.data(), sizeof(Row), 1, f);
            fclose(f);
            printf("SCAN rows=%zu workers=%zu\n", all.size(), ctx.num_workers());
        });
}
