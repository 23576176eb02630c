// rf_test_math_test.cpp -- CPU driver over csrc/rf_test_math.hpp for tests/test_regfile_test_cpu.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python test can hold the host arithmetic of
// b2dp_regfile_test against tests/rf_test_oracle.py:
//   tile <seed> <fmt> <tile>           -> the tile's table words, then its kCtThreads check values
//   reads <fmt> <kind> <key> <thread>  -> every value the thread reads in one clean march, in order
//   pattern <kind> <key> <thread>      -> P(thread, j) for every held register j
//   gen <kind> <key> <thread>          -> the kernel's branch-free form of the same, from rf_gen_params
//   layout                             -> the constants the kernel and the harness share
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "rf_test_math.hpp"

using namespace b2dp;

static uint32_t rotl(uint32_t x, uint32_t s) { return s & 31u ? x << (s & 31u) | x >> (32u - (s & 31u)) : x; }

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
            uint32_t table[kRfTableWords], check[kCtThreads];
            rf_build_tile((uint32_t)seed, fmt, tile, table, check);
            for (int i = 0; i < kRfTableWords; ++i) std::printf(i ? " %u" : "%u", table[i]);
            for (int t = 0; t < kCtThreads; ++t) std::printf(" %u", check[t]);
            std::printf("\n");
        } else if (op == "reads") {
            int fmt, t;
            unsigned long long kind, key;
            in >> fmt >> kind >> key >> t;
            std::vector<uint32_t> r;
            rf_reads(fmt, (uint32_t)kind, (uint32_t)key, t, r);
            for (size_t i = 0; i < r.size(); ++i) std::printf(i ? " %u" : "%u", r[i]);
            std::printf("\n");
        } else if (op == "pattern" || op == "gen") {
            unsigned long long kind, key, t;
            in >> kind >> key >> t;
            const RfGenParams g = rf_gen_params((uint32_t)kind, (uint32_t)key);
            for (uint32_t j = 0; j < (uint32_t)kRfHeld; ++j) {
                const uint32_t v = op == "pattern"
                                       ? rf_pattern((uint32_t)kind, (uint32_t)key, (uint32_t)t, j)
                                       : ((uint32_t)t * (uint32_t)kRfHeld + j) * g.mul ^ ((j & 1u) ? g.odd : g.even) ^
                                             rotl(g.one, (uint32_t)t + j);
                std::printf(j ? " %u" : "%u", v);
            }
            std::printf("\n");
        } else if (op == "layout") {
            std::printf("%d %d %u %u %u %d %u %d %d %d %d %llu\n", kRfHeld, kRfTableWords, kRfHookReg, kRfHookElement,
                        kRfHookThread, kRfParamWords, kRfSmemBytes, kRfDumpWords, kRfElements[0], kRfElements[1],
                        kRfElements[2], kRfHoldNs);
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
