// sfu_test_math_test.cpp -- CPU driver over csrc/sfu_test_math.hpp for tests/test_sfu_test_cpu.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python test can hold the host arithmetic of
// b2dp_sfu_test against tests/sfu_test_oracle.py:
//   table <seed> <fmt> <tile>           -> the operand table, [slot][thread] words
//   guard <fn> <type> <ftz> <x> <r>     -> sf_guard on the bits: "<pass> <err>"
//   fold <n> <w0..wn-1>                 -> sf_fold
//   consensus <fmt> <n_cta> <seq> <dir> -> sf_consensus over <dir>/dumps.bin ([cta][tile][thread][word] u32),
//                                          <dir>/recs.bin (n_cta CtRecords) and <dir>/table.bin (kCtTiles tables):
//                                          "<arrived> <sm_ids> <no_consensus> <out_of_bound> <dissents> <flags>
//                                          <clean> <first_bad_sm> <first_bad_tile> <mask0..3>", and the consensus words
//                                          and checks to <dir>/words.bin and <dir>/check.bin
//   time <seed>                         -> milliseconds to build every table of every format
//   layout                              -> the constants the kernel and the harness share
#include <chrono>
#include <cstdio>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>

#include "sfu_test_math.hpp"

using namespace b2dp;

template <typename T>
static std::vector<T> read_file(const std::string& p) {
    std::ifstream f(p, std::ios::binary);
    std::vector<char> b((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    std::vector<T> v(b.size() / sizeof(T));
    std::memcpy(v.data(), b.data(), v.size() * sizeof(T));
    return v;
}
template <typename T>
static void write_file(const std::string& p, const std::vector<T>& v) {
    std::ofstream f(p, std::ios::binary);
    f.write(reinterpret_cast<const char*>(v.data()), (std::streamsize)(v.size() * sizeof(T)));
}

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op;
        in >> op;
        if (op == "table") {
            unsigned long long seed;
            int fmt, tile;
            in >> seed >> fmt >> tile;
            std::vector<uint32_t> t((size_t)kSfSlots[fmt] * kCtThreads);
            sf_build_table((uint32_t)seed, fmt, tile, t.data());
            for (size_t i = 0; i < t.size(); ++i) std::printf(i ? " %u" : "%u", t[i]);
            std::printf("\n");
        } else if (op == "guard") {
            int fn, type, ftz;
            unsigned long long x, r;
            in >> fn >> type >> ftz >> x >> r;
            double err = 0;
            const bool ok = sf_guard(fn, type, ftz != 0, x, r, &err);
            std::printf("%d %.17g\n", ok ? 1 : 0, err);
        } else if (op == "fold") {
            int n;
            in >> n;
            std::vector<uint32_t> w(n);
            for (auto& v : w) {
                unsigned long long u;
                in >> u;
                v = (uint32_t)u;
            }
            std::printf("%u\n", sf_fold(w.data(), n));
        } else if (op == "consensus") {
            int fmt, n;
            unsigned long long seq;
            std::string dir;
            in >> fmt >> n >> seq >> dir;
            const auto dumps = read_file<uint32_t>(dir + "/dumps.bin");
            const auto recs = read_file<CtRecord>(dir + "/recs.bin");
            const auto table = read_file<uint32_t>(dir + "/table.bin");
            SfConsensus c;
            sf_consensus(fmt, dumps.data(), recs.data(), n, seq, table.data(), c);
            write_file(dir + "/words.bin", c.words);
            write_file(dir + "/check.bin", c.check);
            std::printf("%d %d %llu %llu %llu %u %d %d %d %llu %llu %llu %llu\n", c.arrived, c.sm_ids, c.no_consensus,
                        c.out_of_bound, c.dissents, c.flags(), c.clean() ? 1 : 0, c.first_bad_sm, c.first_bad_tile,
                        (unsigned long long)c.bad_sm_mask[0], (unsigned long long)c.bad_sm_mask[1],
                        (unsigned long long)c.bad_sm_mask[2], (unsigned long long)c.bad_sm_mask[3]);
        } else if (op == "time") {
            unsigned long long seed;
            in >> seed;
            const auto t0 = std::chrono::steady_clock::now();
            std::vector<uint32_t> t((size_t)kSfMaxWords * kCtThreads);
            for (int f = 0; f < kSfFormats; ++f)
                for (int tile = 0; tile < kCtTiles; ++tile) sf_build_table((uint32_t)seed, f, tile, t.data());
            std::printf("%.3f\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
        } else if (op == "layout") {
            std::printf("%d %d %d %d %d %d %d %d %d %d\n", kSfN, kSfSlots[0], kSfSlots[1], kSfSlots[2], kSfWords[0],
                        kSfWords[1], kSfWords[2], kSfResults[0], kSfResults[1], kSfResults[2]);
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
