/*******************************************************************************
 * tests/host/ref_hll_driver.cpp — TEST INFRASTRUCTURE: the stock core::HyperLogLogRegisters<p> of the UNMODIFIED reference.
 *
 * Links the reference library built by oracle/ref/Makefile.  What HyperLogLogNode does (api/hyperloglog.hpp:40-52) is plain
 * library code: every worker inserts its items into its own registers (registers_.insert(x) = insert_hash(tlx::siphash(x))) and
 * net.AllReduce adds the workers' registers with operator +.  The driver does the same without a Thrill job: worker r takes the
 * count_r items after count_0 + ... + count_{r-1}, and the workers' registers are added in rank order.  mode:
 *   u64    8-byte items, inserted as uint64_t (a double is hashed as its bits: the same 8 message bytes)
 *   pair   16-byte items, inserted as std::pair<uint64_t, uint64_t>
 *   hash   8-byte words given to insert_hash directly (no SipHash): pins the register rule on hashes no item search can reach
 * For every precision p in {4, 8, 12, 14, 16, 18} the output holds, in this order:
 *   (a) 2^p bytes   the dense registers of one object made dense up front (toDense() on the empty object) and fed every item
 *   (b) 2^p bytes   the registers of the natural path: every worker starts sparse, operator + in rank order, and toDense() at the
 *                   end only if the sum is still sparse
 *   1 uint64_t      the format of the natural path's sum before that final toDense(): 0 sparse, 1 dense
 *   2 doubles       result() of (a), result() of the natural path's sum as it stood (sparse or dense)
 * The registers are read through the public Serialization (core/hyperloglog.cpp:1887-1903): the format, then one uint64_t per
 * register.  Generates the fixtures of tests/golden/make_golden_hll.py.
 *
 * usage: ref_hll_driver in.bin out.bin u64|pair|hash count_0 ... count_{W-1}
 ******************************************************************************/
#include <thrill/core/hyperloglog.hpp>
#include <thrill/data/serialization.hpp>
#include <thrill/net/buffer_builder.hpp>
#include <thrill/net/buffer_reader.hpp>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

using namespace thrill; // NOLINT

enum Mode { U64, PAIR, HASH };

//! the format (1 = dense) and, if dense, the registers of x
template <size_t p>
static bool Registers(const core::HyperLogLogRegisters<p>& x, std::vector<uint8_t>* regs) {
    net::BufferBuilder bb;
    data::Serialization<net::BufferBuilder, core::HyperLogLogRegisters<p> >::Serialize(x, bb);
    net::BufferReader br(bb.data(), bb.size());
    const auto format = br.Get<core::HyperLogLogRegisterFormat>();
    if (format != core::HyperLogLogRegisterFormat::DENSE) return false;
    regs->resize(size_t(1) << p);
    for (size_t i = 0; i < regs->size(); ++i) (*regs)[i] = static_cast<uint8_t>(br.Get<uint64_t>());
    return true;
}

template <size_t p>
static void Insert(core::HyperLogLogRegisters<p>& r, Mode mode, const uint64_t* w) {
    if (mode == U64) r.insert(w[0]);
    else if (mode == PAIR) r.insert(std::pair<uint64_t, uint64_t>(w[0], w[1]));
    else r.insert_hash(w[0]);
}

template <size_t p>
static void Run(Mode mode, const std::vector<uint64_t>& words, const std::vector<size_t>& counts, FILE* out) {
    const size_t wpi = mode == PAIR ? 2 : 1, n = words.size() / wpi;
    // (a) dense from the first item on
    core::HyperLogLogRegisters<p> a;
    a.toDense();
    for (size_t i = 0; i < n; ++i) Insert(a, mode, &words[i * wpi]);
    // the natural path
    core::HyperLogLogRegisters<p> sum;
    size_t begin = 0;
    for (size_t r = 0; r < counts.size(); ++r) {
        core::HyperLogLogRegisters<p> mine;
        for (size_t i = begin; i < begin + counts[r]; ++i) Insert(mine, mode, &words[i * wpi]);
        begin += counts[r];
        sum = r == 0 ? mine : sum + mine;
    }
    std::vector<uint8_t> ra, rb;
    if (!Registers(a, &ra)) { fprintf(stderr, "p=%zu: (a) is not dense\n", p); exit(3); }
    core::HyperLogLogRegisters<p> natural = sum;      // result() of a sparse object merges its lists: on a copy
    const double est_a = a.result(), est_b = natural.result();
    const uint64_t dense = Registers(sum, &rb) ? 1 : 0;
    if (!dense) {
        sum.toDense();
        Registers(sum, &rb);
    }
    fwrite(ra.data(), 1, ra.size(), out);
    fwrite(rb.data(), 1, rb.size(), out);
    fwrite(&dense, 8, 1, out);
    fwrite(&est_a, 8, 1, out);
    fwrite(&est_b, 8, 1, out);
}

int main(int argc, char** argv) {
    if (argc < 5) {
        fprintf(stderr, "usage: %s in.bin out.bin u64|pair|hash count_0 ... count_{W-1}\n", argv[0]);
        return 2;
    }
    const std::string m = argv[3];
    if (m != "u64" && m != "pair" && m != "hash") { fprintf(stderr, "unknown mode %s\n", argv[3]); return 2; }
    const Mode mode = m == "u64" ? U64 : m == "pair" ? PAIR : HASH;
    std::vector<size_t> counts;
    size_t total = 0;
    for (int i = 4; i < argc; ++i) { counts.push_back(strtoull(argv[i], nullptr, 10)); total += counts.back(); }
    std::vector<uint64_t> words;
    {
        FILE* f = fopen(argv[1], "rb");
        if (!f) { perror("fopen in"); return 2; }
        uint64_t w;
        while (fread(&w, 8, 1, f) == 1) words.push_back(w);
        fclose(f);
    }
    if (total * (mode == PAIR ? 2 : 1) != words.size()) {
        fprintf(stderr, "the counts add up to %zu items, the input holds %zu words\n", total, words.size());
        return 2;
    }
    FILE* out = fopen(argv[2], "wb");
    if (!out) { perror("fopen out"); return 2; }
    Run<4>(mode, words, counts, out);
    Run<8>(mode, words, counts, out);
    Run<12>(mode, words, counts, out);
    Run<14>(mode, words, counts, out);
    Run<16>(mode, words, counts, out);
    Run<18>(mode, words, counts, out);
    fclose(out);
    printf("HLL %s workers=%zu items=%zu\n", argv[3], counts.size(), total);
    return 0;
}
