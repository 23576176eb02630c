// smem_test_math_test.cpp -- CPU driver over csrc/smem_test_math.hpp for tests/test_smem_test_cpu.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python test can hold the host arithmetic of
// b2dp_smem_test against tests/smem_test_oracle.py:
//   tile <seed> <fmt> <tile>         -> the tile's table words, then its kCtThreads check values
//   reads <fmt> <kind> <key> <thread> -> every value the thread reads in one clean march, in order
//   pattern <kind> <key> <w0> <n>    -> P(w) for w in [w0, w0 + n)
//   rank_key <rank>                  -> R(rank)
//   layout                           -> the constants the kernel and the harness share
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "smem_test_math.hpp"

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
            uint32_t table[kShTableWords], check[kCtThreads];
            sh_build_tile((uint32_t)seed, fmt, tile, table, check);
            for (int i = 0; i < kShTableWords; ++i) std::printf(i ? " %u" : "%u", table[i]);
            for (int t = 0; t < kCtThreads; ++t) std::printf(" %u", check[t]);
            std::printf("\n");
        } else if (op == "reads") {
            int fmt, t;
            unsigned long long kind, key;
            in >> fmt >> kind >> key >> t;
            std::vector<uint32_t> r;
            sh_reads(fmt, (uint32_t)kind, (uint32_t)key, t, r);
            for (size_t i = 0; i < r.size(); ++i) std::printf(i ? " %u" : "%u", r[i]);
            std::printf("\n");
        } else if (op == "pattern") {
            unsigned long long kind, key, w0, n;
            in >> kind >> key >> w0 >> n;
            for (unsigned long long i = 0; i < n; ++i)
                std::printf(i ? " %u" : "%u", sh_pattern((uint32_t)kind, (uint32_t)key, (uint32_t)(w0 + i)));
            std::printf("\n");
        } else if (op == "rank_key") {
            unsigned r;
            in >> r;
            std::printf("%u\n", sh_rank_key(r));
        } else if (op == "layout") {
            std::printf("%u %d %d %d %d %d %d %d %u %u %d %d %d %d\n", kShBytes, kShWords, kShWordsPerThread, kShVecs,
                        kShVecsPerThread, kShVecTail, kShPairsPerThread, kShTableWords, kShHookWord, kShHookElement,
                        kShDumpWords, kShElements[0], kShElements[1], kShElements[2]);
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
