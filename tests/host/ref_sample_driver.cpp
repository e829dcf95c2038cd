/*******************************************************************************
 * tests/host/ref_sample_driver.cpp — TEST INFRASTRUCTURE: the stock DIA::Sample and DIA::BernoulliSample of the UNMODIFIED
 * reference.
 *
 * Links the reference library built by oracle/ref/Makefile.  The items are the global positions: worker r places the count_r
 * positions after count_0 + ... + count_{r-1} with ConcatToDIA (api/concat_to_dia.hpp:77-84), so the caller chooses the
 * per-worker sizes, empty workers included, and a sample names the positions it kept.  Then the operator runs `reps` times on
 * the same cached DIA, each with the stock node's own random seed:
 *   sample      dia.Sample(param)            (SampleNode, api/sample.hpp:37-140; rank 0 broadcasts a random_device draw)
 *   bernoulli   dia.BernoulliSample(param)   (api/bernoulli_sample.hpp:27-77; param < 0.1 takes the geometric skip path)
 * Worker r writes, for every rep in order, its output count and then its outputs as uint64_t in the order it emits them, to
 * out.<r>.  Generates the fixtures of tests/golden/make_golden_sample.py.
 *
 * usage: THRILL_NET=mock THRILL_LOCAL=1 THRILL_WORKERS_PER_HOST=W ref_sample_driver out sample|bernoulli param reps count_0 ... count_{W-1}
 ******************************************************************************/
#include <thrill/api/bernoulli_sample.hpp>
#include <thrill/api/cache.hpp>
#include <thrill/api/concat_to_dia.hpp>
#include <thrill/api/sample.hpp>
#include <thrill/api/size.hpp>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

using namespace thrill; // NOLINT

int main(int argc, char** argv) {
    if (argc < 6) {
        fprintf(stderr, "usage: %s out sample|bernoulli param reps count_0 ... count_{W-1}\n", argv[0]);
        return 2;
    }
    const std::string out_path = argv[1], mode = argv[2];
    const double param = strtod(argv[3], nullptr);
    const size_t reps = strtoull(argv[4], nullptr, 10);
    std::vector<size_t> counts;
    for (int i = 5; i < argc; ++i) counts.push_back(strtoull(argv[i], nullptr, 10));
    if (mode != "sample" && mode != "bernoulli") { fprintf(stderr, "unknown mode %s\n", mode.c_str()); return 2; }
    return api::Run(
        [&](api::Context& ctx) {
            if (counts.size() != ctx.num_workers()) {
                fprintf(stderr, "%zu counts for %zu workers\n", counts.size(), ctx.num_workers());
                exit(2);
            }
            uint64_t begin = 0;
            for (size_t r = 0; r < ctx.my_rank(); ++r) begin += counts[r];
            std::vector<uint64_t> shard(counts[ctx.my_rank()]);
            for (size_t i = 0; i < shard.size(); ++i) shard[i] = begin + i;
            auto dia = api::ConcatToDIA(ctx, shard).Cache();
            std::vector<uint64_t> out;
            for (size_t rep = 0; rep < reps; ++rep) {
                std::vector<uint64_t> mine;
                auto collect = [&mine](const uint64_t& x) { mine.push_back(x); return 0; };
                if (mode == "sample") dia.Sample(static_cast<size_t>(param)).Map(collect).Size();
                else dia.BernoulliSample(param).Map(collect).Size();
                out.push_back(mine.size());
                out.insert(out.end(), mine.begin(), mine.end());
            }
            const std::string path = out_path + "." + std::to_string(ctx.my_rank());
            FILE* f = fopen(path.c_str(), "wb");
            if (!f) { perror("fopen out"); exit(2); }
            if (!out.empty()) fwrite(out.data(), 8, out.size(), f);
            fclose(f);
        });
}
