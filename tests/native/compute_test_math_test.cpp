// compute_test_math_test.cpp -- CPU driver over csrc/compute_test_math.hpp for tests/test_compute_test_cpu.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python test can hold the host arithmetic
// of b2dp_compute_test against tests/compute_test_oracle.py:
//   operand <seed> <fmt> <tile> <op>          -> scale exponent, then the rows x K operand values
//   encode <fmt> <e>                          -> the bits of every value in [lo, hi] times 2^e
//   scaled <seed> <fmt> <tile> <ea> <eb>      -> the exact result bits of the tile's operands scaled by 2^ea, 2^eb
//   tile <seed> <fmt> <tile>                  -> the exact result bits (M x N), then the kCtThreads check values
//   fold <x0..x63>                            -> ct_fold
//   verdict <ok> <n0> <n1> <n2> <records>     -> 1 / 0; records: n0 + n1 + n2 of <seq rounds comparisons mismatches>,
//                                                format by format; format f's launch carries seq f + 1
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>

#include "compute_test_math.hpp"

using namespace b2dp;

static void print_u32s(const uint32_t* v, size_t n) {
    for (size_t i = 0; i < n; ++i) std::printf(i ? " %u" : "%u", v[i]);
}

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op;
        in >> op;
        if (op == "operand") {
            unsigned long long seed;
            int fmt, tile, o;
            in >> seed >> fmt >> tile >> o;
            const std::vector<int> v = ct_operand((uint32_t)seed, fmt, tile, o);
            std::printf("%d", ct_scale_exp((uint32_t)seed, fmt, tile, o));
            for (int x : v) std::printf(" %d", x);
            std::printf("\n");
        } else if (op == "encode") {
            int fmt, e;
            in >> fmt >> e;
            for (int v = ct_lo(fmt); v <= ct_hi(fmt); ++v) std::printf(v == ct_lo(fmt) ? "%u" : " %u", ct_encode(fmt, v, e));
            std::printf("\n");
        } else if (op == "scaled") {
            unsigned long long seed;
            int fmt, tile, ea, eb;
            in >> seed >> fmt >> tile >> ea >> eb;
            const std::vector<uint32_t> d = ct_reference(fmt, ct_operand((uint32_t)seed, fmt, tile, 0),
                                                         ct_operand((uint32_t)seed, fmt, tile, 1), ea, eb);
            print_u32s(d.data(), d.size());
            std::printf("\n");
        } else if (op == "tile") {
            unsigned long long seed;
            int fmt, tile;
            in >> seed >> fmt >> tile;
            CtTile t;
            ct_build_tile((uint32_t)seed, fmt, tile, t);
            print_u32s(t.reference.data(), t.reference.size());
            std::printf(" ");
            print_u32s(t.check, kCtThreads);
            std::printf("\n");
        } else if (op == "fold") {
            uint32_t x[kCtAcc];
            for (auto& v : x) {
                unsigned long long u;
                in >> u;
                v = (uint32_t)u;
            }
            std::printf("%u\n", ct_fold(x));
        } else if (op == "verdict") {
            int ok, n[kCtFormats];
            in >> ok >> n[0] >> n[1] >> n[2];
            std::vector<CtRecord> recs[kCtFormats];
            unsigned long long seq[kCtFormats];
            for (int f = 0; f < kCtFormats; ++f) {
                seq[f] = (unsigned long long)(f + 1);
                for (int i = 0; i < n[f]; ++i) {
                    CtRecord r{};
                    in >> r.seq >> r.rounds >> r.comparisons >> r.mismatches;
                    recs[f].push_back(r);
                }
            }
            std::printf("%d\n", compute_test_healthy(ok != 0, recs, seq) ? 1 : 0);
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
