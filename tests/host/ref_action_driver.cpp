/*******************************************************************************
 * tests/host/ref_action_driver.cpp — TEST INFRASTRUCTURE: the stock DIA::Sum / Min / Max / AllReduce of the UNMODIFIED reference.
 *
 * Links the reference library built by oracle/ref/Makefile.  Every worker reads the whole binary input and places its own shard
 * with ConcatToDIA (api/concat_to_dia.hpp:77-84): worker r takes the count_r items after count_0 + ... + count_{r-1}, so the
 * caller chooses the per-worker sizes, empty workers included.  Then one action runs on the DIA, mode = <type>_<fn>:
 *   u64_sum / u64_min / u64_max         uint64_t items: Sum() or Sum(std::plus, initial), Min([initial]), Max([initial])
 *                                       (api/sum.hpp, min.hpp, max.hpp: std::plus, common::minimum, common::maximum)
 *   f64_sum / f64_min / f64_max         double items, the same actions
 *   pair_u64_<fn> / pair_f64_<fn>       pair<uint64_t, uint64_t> / pair<uint64_t, double> items: AllReduce(ScanSecond<F>
 *                                       [, initial]) with F the function above, (a, b) -> (b.first, F(a.second, b.second))
 * init|none picks the form with or without the initial value.  Every worker checks that its result equals worker 0's (as bits),
 * and worker 0 writes the result as two uint64_t: (first word, second word) (an 8-byte item has first word 0; doubles are written
 * as their bits).  Generates the fixtures of tests/golden/make_golden_action.py.
 *
 * usage: THRILL_NET=mock THRILL_LOCAL=1 THRILL_WORKERS_PER_HOST=W ref_action_driver in.bin out.bin mode init|none init_first
 *        init_second count_0 ... count_{W-1}
 ******************************************************************************/
#include <thrill/api/all_reduce.hpp>
#include <thrill/api/concat_to_dia.hpp>
#include <thrill/api/max.hpp>
#include <thrill/api/min.hpp>
#include <thrill/api/sum.hpp>
#include <thrill/common/functional.hpp>

#include <array>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

using namespace thrill; // NOLINT

using Row = std::array<uint64_t, 2>;

//! a plain functor (the stock node reads its argument type), as thrill_gpu::ScanSecond is
template <typename M> struct MemberResult;
template <typename R, typename C, typename... A>
struct MemberResult<R (C::*)(A...) const> { using type = typename std::decay<R>::type; };
template <typename F>
struct ScanSecond {
    using P = std::pair<uint64_t, typename MemberResult<decltype(&F::operator ())>::type>;
    F fn;
    P operator () (const P& a, const P& b) const { return P(b.first, fn(a.second, b.second)); }
};

static uint64_t bits(double d) { uint64_t u; memcpy(&u, &d, 8); return u; }
static uint64_t bits(uint64_t u) { return u; }
static double dbl(uint64_t u) { double d; memcpy(&d, &u, 8); return d; }

//! this worker's shard of the input (as words): counts[r] items of `words` words each
static std::vector<uint64_t> Shard(const std::vector<uint64_t>& all, const std::vector<size_t>& counts, size_t rank,
                                   size_t words) {
    size_t begin = 0;
    for (size_t r = 0; r < rank; ++r) begin += counts[r];
    return std::vector<uint64_t>(all.begin() + begin * words, all.begin() + (begin + counts[rank]) * words);
}

//! the scalar actions on uint64_t or double items
template <typename T>
Row Scalar(api::Context& ctx, const std::vector<T>& mine, const std::string& fn, bool init, T initial) {
    auto dia = api::ConcatToDIA(ctx, mine);
    T r;
    if (fn == "sum") r = init ? dia.Sum(std::plus<T>(), initial) : dia.Sum();
    else if (fn == "min") r = init ? dia.Min(initial) : dia.Min();
    else r = init ? dia.Max(initial) : dia.Max();
    return Row { { 0, bits(r) } };
}

//! AllReduce(ScanSecond<F>) on pair<uint64_t, T> items
template <typename T, typename F>
Row Pair(api::Context& ctx, const std::vector<uint64_t>& mine, bool init, uint64_t init_first, T init_second) {
    using P = std::pair<uint64_t, T>;
    std::vector<P> v;
    for (size_t i = 0; i < mine.size(); i += 2) {
        T x;
        memcpy(&x, &mine[i + 1], 8);
        v.emplace_back(mine[i], x);
    }
    auto dia = api::ConcatToDIA(ctx, v);
    P r = init ? dia.AllReduce(ScanSecond<F>(), P(init_first, init_second)) : dia.AllReduce(ScanSecond<F>());
    return Row { { r.first, bits(r.second) } };
}

template <typename T>
Row PairFn(api::Context& ctx, const std::vector<uint64_t>& mine, const std::string& fn, bool init, uint64_t init_first,
           T init_second) {
    if (fn == "sum") return Pair<T, std::plus<T> >(ctx, mine, init, init_first, init_second);
    if (fn == "min") return Pair<T, common::minimum<T> >(ctx, mine, init, init_first, init_second);
    return Pair<T, common::maximum<T> >(ctx, mine, init, init_first, init_second);
}

int main(int argc, char** argv) {
    if (argc < 8) {
        fprintf(stderr, "usage: %s in.bin out.bin mode init|none init_first init_second count_0 ... count_{W-1}\n", argv[0]);
        return 2;
    }
    const std::string in_path = argv[1], out_path = argv[2], mode = argv[3];
    const bool init = !strcmp(argv[4], "init");
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
    const size_t us = mode.rfind('_');
    const std::string type = mode.substr(0, us), fn = mode.substr(us + 1);
    if ((type != "u64" && type != "f64" && type != "pair_u64" && type != "pair_f64") ||
        (fn != "sum" && fn != "min" && fn != "max")) {
        fprintf(stderr, "unknown mode %s\n", mode.c_str());
        return 2;
    }
    return api::Run(
        [&](api::Context& ctx) {
            if (counts.size() != ctx.num_workers()) {
                fprintf(stderr, "%zu counts for %zu workers\n", counts.size(), ctx.num_workers());
                exit(2);
            }
            const size_t rank = ctx.my_rank();
            const bool pair = type.compare(0, 5, "pair_") == 0;
            const std::vector<uint64_t> mine = Shard(words, counts, rank, pair ? 2 : 1);
            Row r;
            if (type == "u64") r = Scalar<uint64_t>(ctx, mine, fn, init, init_second);
            else if (type == "f64") {
                std::vector<double> d;
                for (uint64_t w : mine) d.push_back(dbl(w));
                r = Scalar<double>(ctx, d, fn, init, dbl(init_second));
            }
            else if (type == "pair_u64") r = PairFn<uint64_t>(ctx, mine, fn, init, init_first, init_second);
            else r = PairFn<double>(ctx, mine, fn, init, init_first, dbl(init_second));
            // every worker holds the same result
            const Row r0 = ctx.net.Broadcast(r, 0);
            if (r0 != r) {
                fprintf(stderr, "worker %zu: result differs from worker 0's\n", rank);
                exit(3);
            }
            if (rank != 0) return;
            FILE* f = fopen(out_path.c_str(), "wb");
            if (!f) { perror("fopen out"); exit(2); }
            fwrite(r.data(), sizeof(Row), 1, f);
            fclose(f);
            printf("ACTION %s workers=%zu\n", mode.c_str(), ctx.num_workers());
        });
}
