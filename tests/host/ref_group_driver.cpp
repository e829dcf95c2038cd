/*******************************************************************************
 * tests/host/ref_group_driver.cpp — TEST INFRASTRUCTURE: the stock DIA::GroupByKey / DIA::GroupToIndex of the UNMODIFIED
 * reference.
 *
 * Links the reference library built by oracle/ref/Makefile and runs GroupByKey<Row>(.first, fn) (api/group_by_key.hpp:419-428)
 * or GroupToIndex<Row>(.first, fn, size, neutral) (api/group_to_index.hpp:257-290) on a binary file of pair<uint64_t,
 * uint64_t>.  The group functions do not depend on the order inside a group:
 *   stats    (key, count, sum of values, xor of splitmix64(value), min value, max value)
 *   partial  (key, items read): reads at most 3 items, so a larger group is handed to it again (GroupByKey only)
 * A Map child writes the worker's rank into word 0 of each row, and Gather(0) keeps the worker order, so the output (rows of 7
 * uint64_t: rank, key, count, sum, xor, min, max; GroupToIndex's neutral element has key ~0 and zeros) records which worker
 * produced what.  Generates the fixtures of tests/golden/make_golden_group.py.
 *
 * usage: THRILL_NET=mock THRILL_LOCAL=1 THRILL_WORKERS_PER_HOST=W ref_group_driver in.bin out.bin key|index stats|partial [size]
 ******************************************************************************/
#include <thrill/api/cache.hpp>
#include <thrill/api/gather.hpp>
#include <thrill/api/group_by_key.hpp>
#include <thrill/api/group_to_index.hpp>
#include <thrill/api/read_binary.hpp>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

using namespace thrill; // NOLINT

struct Row {
    uint64_t w[7];
};

static inline uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    uint64_t z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

int main(int argc, char** argv) {
    if (argc < 5) {
        fprintf(stderr, "usage: %s in.bin out.bin key|index stats|partial [size]\n", argv[0]);
        return 2;
    }
    const std::string in_path = argv[1], out_path = argv[2];
    const bool to_index = !strcmp(argv[3], "index");
    const bool partial = !strcmp(argv[4], "partial");
    const size_t size = argc > 5 ? strtoull(argv[5], nullptr, 10) : 0;
    return api::Run(
        [&](api::Context& ctx) {
            using P = std::pair<uint64_t, uint64_t>;
            auto stats = [](auto& r, const uint64_t& key) {
                Row o = { { 0, key, 0, 0, 0, ~0ull, 0 } };
                while (r.HasNext()) {
                    const P p = r.Next();
                    o.w[2]++;
                    o.w[3] += p.second;
                    o.w[4] ^= splitmix64(p.second);
                    o.w[5] = std::min(o.w[5], p.second);
                    o.w[6] = std::max(o.w[6], p.second);
                }
                return o;
            };
            auto part = [](auto& r, const uint64_t& key) {
                Row o = { { 0, key, 0, 0, 0, 0, 0 } };
                while (o.w[2] < 3 && r.HasNext()) {
                    r.Next();
                    o.w[2]++;
                }
                return o;
            };
            auto key_of = [](const P& p) { return p.first; };
            auto tag = [&ctx](const Row& x) { Row y = x; y.w[0] = ctx.my_rank(); return y; };
            auto in = api::ReadBinary<P>(ctx, in_path).Cache();
            std::vector<Row> all;
            if (to_index) {
                const Row neutral = { { 0, ~0ull, 0, 0, 0, 0, 0 } };
                all = in.GroupToIndex<Row>(key_of, stats, size, neutral).Map(tag).Gather(0);
            }
            else if (partial) {
                all = in.GroupByKey<Row>(key_of, part).Map(tag).Gather(0);
            }
            else {
                all = in.GroupByKey<Row>(key_of, stats).Map(tag).Gather(0);
            }
            if (ctx.my_rank() != 0) return;
            FILE* f = fopen(out_path.c_str(), "wb");
            if (!f) { perror("fopen out"); exit(2); }
            for (const Row& r : all) fwrite(r.w, sizeof(r.w), 1, f);
            fclose(f);
            printf("GROUP rows=%zu workers=%zu\n", all.size(), ctx.num_workers());
        });
}
