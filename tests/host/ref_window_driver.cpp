/*******************************************************************************
 * tests/host/ref_window_driver.cpp — TEST INFRASTRUCTURE: the stock DIA::Window of the UNMODIFIED reference.
 *
 * Links the reference library built by oracle/ref/Makefile.  Every worker reads the whole binary input and places its own shard
 * with ConcatToDIA (api/concat_to_dia.hpp:77-84): worker r takes the count_r items after count_0 + ... + count_{r-1}, so the
 * caller chooses the per-worker sizes, empty workers included.  Then one Window runs on the DIA, mode = <type>_<fn>, form:
 *   <type>  u64 / f64 (uint64_t / double items), pair_u64 / pair_f64 (pair<uint64_t, uint64_t> / pair<uint64_t, double> with
 *           ScanSecond<F>, (a, b) -> (b.first, F(a.second, b.second)))
 *   <fn>    sum / min / max: std::plus, common::minimum, common::maximum
 *   form    full: Window(k, WindowFold), partial: Window(k, WindowFold, WindowFold), disjoint: Window(DisjointTag, k, DisjointFold)
 * WindowFold / DisjointFold return the left fold of the window with F from its first item (what thrill_gpu::WindowFold<F> and
 * DisjointFold<F> do).  Worker r writes its outputs, in the order it emits them, to out.<r> as two uint64_t per item (first word,
 * second word; an 8-byte item has first word 0, doubles are written as their bits).  Generates the fixtures of
 * tests/golden/make_golden_window.py.
 *
 * usage: THRILL_NET=mock THRILL_LOCAL=1 THRILL_WORKERS_PER_HOST=W ref_window_driver in.bin out mode form k count_0 ... count_{W-1}
 ******************************************************************************/
#include <thrill/api/concat_to_dia.hpp>
#include <thrill/api/size.hpp>
#include <thrill/api/window.hpp>
#include <thrill/common/functional.hpp>
#include <thrill/common/ring_buffer.hpp>

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

template <typename M> struct MemberResult;
template <typename R, typename C, typename... A>
struct MemberResult<R (C::*)(A...) const> { using type = typename std::decay<R>::type; };
template <typename F>
struct ScanSecond {
    using P = std::pair<uint64_t, typename MemberResult<decltype(&F::operator ())>::type>;
    F fn;
    P operator () (const P& a, const P& b) const { return P(b.first, fn(a.second, b.second)); }
};
//! plain functors with one operator () each (the stock DIA::Window reads their argument types)
template <typename F>
struct WindowFold {
    using T = typename MemberResult<decltype(&F::operator ())>::type;
    F fn;
    T operator () (size_t, const common::RingBuffer<T>& w) const {
        T acc = w[0];
        for (size_t i = 1; i < w.size(); ++i) acc = fn(acc, w[i]);
        return acc;
    }
};
template <typename F>
struct DisjointFold {
    using T = typename MemberResult<decltype(&F::operator ())>::type;
    F fn;
    T operator () (size_t, const std::vector<T>& w) const {
        T acc = w[0];
        for (size_t i = 1; i < w.size(); ++i) acc = fn(acc, w[i]);
        return acc;
    }
};

static uint64_t bits(double d) { uint64_t u; memcpy(&u, &d, 8); return u; }
static uint64_t bits(uint64_t u) { return u; }
static Row row(uint64_t x) { return Row { { 0, x } }; }
static Row row(double x) { return Row { { 0, bits(x) } }; }
template <typename T>
static Row row(const std::pair<uint64_t, T>& x) { return Row { { x.first, bits(x.second) } }; }

//! this worker's shard: counts[r] items of `words` words each, as items of type T
template <typename T>
static std::vector<T> Shard(const std::vector<uint64_t>& all, const std::vector<size_t>& counts, size_t rank) {
    size_t begin = 0;
    for (size_t r = 0; r < rank; ++r) begin += counts[r];
    std::vector<T> v(counts[rank]);
    if (counts[rank]) memcpy(v.data(), all.data() + begin * (sizeof(T) / 8), counts[rank] * sizeof(T));
    return v;
}

template <typename F>
std::vector<Row> Run(api::Context& ctx, const std::vector<uint64_t>& words, const std::vector<size_t>& counts,
                     const std::string& form, size_t k) {
    using T = typename WindowFold<F>::T;
    auto dia = api::ConcatToDIA(ctx, Shard<T>(words, counts, ctx.my_rank()));
    std::vector<Row> out;
    auto collect = [&out](const T& x) { out.push_back(row(x)); return 0; };
    if (form == "full") dia.Window(k, WindowFold<F>()).Map(collect).Size();
    else if (form == "partial") dia.Window(k, WindowFold<F>(), WindowFold<F>()).Map(collect).Size();
    else dia.Window(api::DisjointTag, k, DisjointFold<F>()).Map(collect).Size();
    return out;
}

template <typename T>
std::vector<Row> RunFn(api::Context& ctx, bool pair, const std::string& fn, const std::vector<uint64_t>& words,
                       const std::vector<size_t>& counts, const std::string& form, size_t k) {
    if (pair) {
        if (fn == "sum") return Run<ScanSecond<std::plus<T> > >(ctx, words, counts, form, k);
        if (fn == "min") return Run<ScanSecond<common::minimum<T> > >(ctx, words, counts, form, k);
        return Run<ScanSecond<common::maximum<T> > >(ctx, words, counts, form, k);
    }
    if (fn == "sum") return Run<std::plus<T> >(ctx, words, counts, form, k);
    if (fn == "min") return Run<common::minimum<T> >(ctx, words, counts, form, k);
    return Run<common::maximum<T> >(ctx, words, counts, form, k);
}

int main(int argc, char** argv) {
    if (argc < 7) {
        fprintf(stderr, "usage: %s in.bin out mode full|partial|disjoint k count_0 ... count_{W-1}\n", argv[0]);
        return 2;
    }
    const std::string in_path = argv[1], out_path = argv[2], mode = argv[3], form = argv[4];
    const size_t k = strtoull(argv[5], nullptr, 10);
    std::vector<size_t> counts;
    for (int i = 6; i < argc; ++i) counts.push_back(strtoull(argv[i], nullptr, 10));
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
        (fn != "sum" && fn != "min" && fn != "max") || (form != "full" && form != "partial" && form != "disjoint") || k < 2) {
        fprintf(stderr, "unknown mode %s %s k=%zu\n", mode.c_str(), form.c_str(), k);
        return 2;
    }
    return api::Run(
        [&](api::Context& ctx) {
            if (counts.size() != ctx.num_workers()) {
                fprintf(stderr, "%zu counts for %zu workers\n", counts.size(), ctx.num_workers());
                exit(2);
            }
            const bool pair = type.compare(0, 5, "pair_") == 0;
            const bool f64 = type == "f64" || type == "pair_f64";
            std::vector<Row> out = f64 ? RunFn<double>(ctx, pair, fn, words, counts, form, k)
                                       : RunFn<uint64_t>(ctx, pair, fn, words, counts, form, k);
            const std::string path = out_path + "." + std::to_string(ctx.my_rank());
            FILE* f = fopen(path.c_str(), "wb");
            if (!f) { perror("fopen out"); exit(2); }
            if (!out.empty()) fwrite(out.data(), sizeof(Row), out.size(), f);
            fclose(f);
        });
}
