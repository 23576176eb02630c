// l1_test_math_test.cpp -- CPU driver over csrc/l1_test_math.hpp for tests/test_l1_test_cpu.py and
// tests/test_gpu_l1_test.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python tests can hold the host arithmetic of
// b2dp_l1_test against tests/l1_test_oracle.py and the device's DUMP:
//   tile <seed> <fmt> <tile>     -> the table (kL1TableWords), every thread's result words, then the kCtThreads checks
//   span <seed> <tile> <K> <c>   -> L1_DATA: every raw value CTA c's threads read in repetition 0, in DUMP order
//   image <seed> / bank <seed>   -> the texel image (row-major, four words a texel) / the constant bank
//   order <K>                    -> the blocks of the three read passes over K blocks
//   ok <fmt> <w0> <w1> <w2> <w3> -> 1 if l1_table_ok accepts the table
//   bounds                       -> the layout constants
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "l1_test_math.hpp"

using namespace b2dp;

static void print(const std::vector<uint32_t>& v) {
    std::string s;
    s.reserve(v.size() * 11);
    char buf[16];
    for (size_t i = 0; i < v.size(); ++i) {
        snprintf(buf, sizeof buf, i ? " %u" : "%u", v[i]);
        s += buf;
    }
    std::printf("%s\n", s.c_str());
}

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op;
        in >> op;
        if (op == "tile") {
            unsigned long long seed;
            int fmt, tile;
            in >> seed >> fmt >> tile;
            std::vector<uint32_t> table(kL1TableWords), words;
            uint32_t check[kCtThreads];
            l1_build_tile((uint32_t)seed, fmt, tile, table.data(), check, &words);
            table.insert(table.end(), words.begin(), words.end());
            table.insert(table.end(), check, check + kCtThreads);
            print(table);
        } else if (op == "span") {
            unsigned long long seed;
            int tile;
            unsigned K, c;
            in >> seed >> tile >> K >> c;
            uint32_t tab[kL1TableWords];
            l1_table((uint32_t)seed, L1_DATA, tile, tab);
            std::vector<uint32_t> out;
            for (int t = 0; t < kCtThreads; ++t)
                for (int p = 0; p < kL1Passes; ++p)
                    for (uint32_t s = 0; s < K; ++s)
                        for (int i = 0; i < 4; ++i)
                            out.push_back(l1_pattern(tab[0], tab[1], tab[2], c, K,
                                                     l1_data_block(p, s, K) * kL1BlockWords +
                                                         4u * (uint32_t)l1_data_writer(t, p) + (uint32_t)i));
            print(out);
        } else if (op == "image" || op == "bank") {
            unsigned long long seed;
            in >> seed;
            std::vector<uint32_t> v(op == "image" ? (size_t)kL1Texels * 4 : (size_t)kL1BankWords);
            if (op == "image") l1_tex_image((uint32_t)seed, v.data());
            else l1_bank((uint32_t)seed, v.data());
            print(v);
        } else if (op == "order") {
            unsigned K;
            in >> K;
            std::vector<uint32_t> v;
            for (int p = 0; p < kL1Passes; ++p)
                for (uint32_t s = 0; s < K; ++s) v.push_back(l1_data_block(p, s, K));
            print(v);
        } else if (op == "ok") {
            int fmt;
            uint32_t t[kL1TableWords];
            in >> fmt >> t[0] >> t[1] >> t[2] >> t[3];
            std::printf("%d\n", l1_table_ok(fmt, t) ? 1 : 0);
        } else if (op == "bounds") {
            for (int f = 0; f < kL1Formats; ++f)
                std::printf("%d %u %.0f ", l1_words(f), l1_table_bytes(f), l1_bytes_per_comparison(f, 1));
            std::printf("%u\n", l1_span_blocks(kL1DefaultSpan, 1));
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
