// sync_test_math_test.cpp -- CPU driver over csrc/sync_test_math.hpp for tests/test_sync_test_cpu.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python test can hold the host arithmetic of
// b2dp_sync_test against tests/sync_test_oracle.py:
//   tile <seed> <fmt> <tile>   -> the operand table ([slot][thread] words), then every thread's result words, then the
//                                 kCtThreads check values
//   fold <n> <w0..wn-1>        -> it_fold
//   bounds                     -> the layout constants
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>

#include "sync_test_math.hpp"

using namespace b2dp;

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
            std::vector<uint32_t> table(sy_table_bytes(fmt) / 4), words;
            uint32_t check[kCtThreads];
            sy_build_tile((uint32_t)seed, fmt, tile, table.data(), check, &words);
            for (size_t i = 0; i < table.size(); ++i) std::printf(i ? " %u" : "%u", table[i]);
            for (uint32_t w : words) std::printf(" %u", w);
            for (uint32_t c : check) std::printf(" %u", c);
            std::printf("\n");
        } else if (op == "fold") {
            int n;
            in >> n;
            std::vector<uint32_t> w(n);
            for (auto& v : w) {
                unsigned long long u;
                in >> u;
                v = (uint32_t)u;
            }
            std::printf("%u\n", it_fold(w.data(), n));
        } else if (op == "bounds") {
            for (int f = 0; f < kSyFormats; ++f)
                std::printf("%d %d %u %.0f ", kSySlots[f], kSyWords[f], sy_table_bytes(f), sy_ops_per_tile(f));
            std::printf("\n");
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
