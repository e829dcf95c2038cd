/*******************************************************************************
 * tests/host/ref_join_records_driver.cpp — TEST INFRASTRUCTURE: the stock api::InnerJoin of the UNMODIFIED reference on records.
 *
 * Links the reference library built by oracle/ref/Makefile and runs api::InnerJoin(left, right, key field, key field,
 * (l, r) -> std::make_pair(l, r)) (api/inner_join.hpp:700-827) on two binary files of fixed-size records.  The key of a record
 * is the unsigned little-endian integer of its key field, zero-extended (or .first of a pair<uint64_t, V>).  The gathered pairs
 * are written as rows of the left item's bytes followed by the right item's.  Generates the fixtures of
 * tests/golden/make_golden_join_records.py.
 *
 * usage: THRILL_NET=mock THRILL_LOCAL=1 THRILL_WORKERS_PER_HOST=W ref_join_records_driver shape left.bin right.bin out.bin
 *   shape: w4 (4-byte items that are their keys), r12x24 (2-byte key at 5 of 12 bytes x 5-byte key at 3 of 24 bytes), r24x8
 *          (5-byte key at 3 of 24 bytes x 5-byte key at 3 of 8 bytes: the key ends the item), r176x152 (8-byte keys at 0),
 *          self24 (a 24-byte side with a 5-byte key at 3 joined with itself; right.bin is not read), pair8 (pair<u64, u64> x
 *          pair<u64, u64> on .first), pair24 (pair<u64, u64> x pair<u64, 24-byte POD> on .first)
 ******************************************************************************/
#include <thrill/api/cache.hpp>
#include <thrill/api/gather.hpp>
#include <thrill/api/inner_join.hpp>
#include <thrill/api/read_binary.hpp>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

using namespace thrill; // NOLINT

template <size_t N>
struct Rec {
    uint8_t b[N];
};
struct V24 {
    uint64_t a, b, c;
};

//! the key field of a record: kBytes bytes at kOffset, little-endian, zero-extended
template <size_t N, size_t kOffset, size_t kBytes>
struct FieldKey {
    uint64_t operator () (const Rec<N>& r) const {
        uint64_t k = 0;
        std::memcpy(&k, r.b + kOffset, kBytes);
        return k;
    }
};

template <typename T>
static void Put(std::vector<uint8_t>* out, const T& x) {
    const uint8_t* p = reinterpret_cast<const uint8_t*>(&x);
    out->insert(out->end(), p, p + sizeof(T));
}
template <typename V>
static void Put(std::vector<uint8_t>* out, const std::pair<uint64_t, V>& x) {   // member-wise, as Thrill serializes a pair
    Put(out, x.first);
    Put(out, x.second);
}

template <typename L, typename R>
static void Write(api::Context& ctx, const std::vector<std::pair<L, R> >& all, const std::string& op) {
    if (ctx.my_rank() != 0) return;
    std::vector<uint8_t> bytes;
    for (const auto& x : all) { Put(&bytes, x.first); Put(&bytes, x.second); }
    FILE* f = fopen(op.c_str(), "wb");
    if (!f) { perror("fopen out"); exit(2); }
    if (!bytes.empty()) fwrite(bytes.data(), 1, bytes.size(), f);
    fclose(f);
    printf("JOIN_RECORDS rows=%zu workers=%zu\n", all.size(), ctx.num_workers());
}

template <typename L, typename R, typename KL, typename KR>
static void Run(api::Context& ctx, const std::string& lp, const std::string& rp, const std::string& op) {
    auto left = api::ReadBinary<L>(ctx, lp).Cache();
    auto right = api::ReadBinary<R>(ctx, rp).Cache();
    Write(ctx, api::InnerJoin(left, right, KL(), KR(), [](const L& l, const R& r) { return std::make_pair(l, r); }).Gather(0), op);
}

//! a self-join: one DIA on both edges
template <typename L, typename K>
static void RunSelf(api::Context& ctx, const std::string& lp, const std::string& op) {
    auto left = api::ReadBinary<L>(ctx, lp).Cache();
    Write(ctx, api::InnerJoin(left, left, K(), K(), [](const L& l, const L& r) { return std::make_pair(l, r); }).Gather(0), op);
}

struct First8 {
    uint64_t operator () (const std::pair<uint64_t, uint64_t>& p) const { return p.first; }
};
struct First24 {
    uint64_t operator () (const std::pair<uint64_t, V24>& p) const { return p.first; }
};

int main(int argc, char** argv) {
    if (argc != 5) {
        fprintf(stderr, "usage: %s shape left.bin right.bin out.bin\n", argv[0]);
        return 2;
    }
    const std::string shape = argv[1], lp = argv[2], rp = argv[3], op = argv[4];
    return api::Run(
        [&](api::Context& ctx) {
            using P8 = std::pair<uint64_t, uint64_t>;
            using P24 = std::pair<uint64_t, V24>;
            if (shape == "w4") Run<Rec<4>, Rec<4>, FieldKey<4, 0, 4>, FieldKey<4, 0, 4> >(ctx, lp, rp, op);
            else if (shape == "r12x24") Run<Rec<12>, Rec<24>, FieldKey<12, 5, 2>, FieldKey<24, 3, 5> >(ctx, lp, rp, op);
            else if (shape == "r24x8") Run<Rec<24>, Rec<8>, FieldKey<24, 3, 5>, FieldKey<8, 3, 5> >(ctx, lp, rp, op);
            else if (shape == "r176x152") Run<Rec<176>, Rec<152>, FieldKey<176, 0, 8>, FieldKey<152, 0, 8> >(ctx, lp, rp, op);
            else if (shape == "self24") RunSelf<Rec<24>, FieldKey<24, 3, 5> >(ctx, lp, op);
            else if (shape == "pair8") Run<P8, P8, First8, First8>(ctx, lp, rp, op);
            else if (shape == "pair24") Run<P8, P24, First8, First24>(ctx, lp, rp, op);
            else { fprintf(stderr, "unknown shape %s\n", shape.c_str()); exit(2); }
        });
}
