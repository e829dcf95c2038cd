/*******************************************************************************
 * tests/host/ref_join_driver.cpp — TEST INFRASTRUCTURE: the stock api::InnerJoin of the UNMODIFIED reference.
 *
 * Links the reference library built by oracle/ref/Makefile and runs api::InnerJoin(left, right, .first, .first,
 * (l, r) -> tuple(key, l.second, r.second)) (api/inner_join.hpp:700-827, tests/api/join_test.cpp:51-55) on two binary files
 * of pair<uint64_t, uint64_t>.  The gathered tuples are written as (key, v1, v2) rows of three uint64_t, member by member.
 * Generates the fixtures of tests/golden/make_golden_join.py.
 *
 * usage: THRILL_NET=mock THRILL_LOCAL=1 THRILL_WORKERS_PER_HOST=W ref_join_driver left.bin right.bin out.bin
 ******************************************************************************/
#include <thrill/api/gather.hpp>
#include <thrill/api/inner_join.hpp>
#include <thrill/api/read_binary.hpp>
#include <thrill/api/size.hpp>

#include <cstdint>
#include <cstdio>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

using namespace thrill; // NOLINT

int main(int argc, char** argv) {
    if (argc != 4) {
        fprintf(stderr, "usage: %s left.bin right.bin out.bin\n", argv[0]);
        return 2;
    }
    const std::string left_path = argv[1], right_path = argv[2], out_path = argv[3];
    return api::Run(
        [&](api::Context& ctx) {
            using P = std::pair<uint64_t, uint64_t>;
            using T = std::tuple<uint64_t, uint64_t, uint64_t>;
            auto left = api::ReadBinary<P>(ctx, left_path).Cache();
            auto right = api::ReadBinary<P>(ctx, right_path).Cache();
            std::vector<T> all = api::InnerJoin(
                left, right, [](const P& p) { return p.first; }, [](const P& p) { return p.first; },
                [](const P& a, const P& b) { return T(a.first, a.second, b.second); }).Gather(0);
            if (ctx.my_rank() != 0) return;
            FILE* f = fopen(out_path.c_str(), "wb");
            if (!f) { perror("fopen out"); exit(2); }
            for (const T& t : all) {
                const uint64_t row[3] = { std::get<0>(t), std::get<1>(t), std::get<2>(t) };
                fwrite(row, sizeof(row), 1, f);
            }
            fclose(f);
            printf("JOIN rows=%zu workers=%zu\n", all.size(), ctx.num_workers());
        });
}
