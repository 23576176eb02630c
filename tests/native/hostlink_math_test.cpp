// hostlink_math_test.cpp -- CPU driver over csrc/hostlink_math.hpp for tests/test_hostlink_test_cpu.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python test can hold the host arithmetic of
// b2dp_hostlink_test against tests/hostlink_oracle.py:
//   width <vec>                            -> bytes per store of that vector
//   link <gen> <width>                     -> per-direction GB/s (%.17g)
//   bytes <requested>                      -> the buffer size used (0 = rejected)
//   next <seed>                            -> the next round's seed
//   check <n_words> <seed> <idx mask>...   -> pattern(seed) with those words flipped, checked: "<bad> <first_bad>"
//   verdict <ok> <seq_ok> <cs_ok> <r0 r1 r2> <m0 m1 m2>  -> 1 Healthy / 0
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "hostlink_math.hpp"

using namespace b2dp;

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op;
        in >> op;
        if (op == "width") {
            unsigned long long v;
            in >> v;
            std::printf("%u\n", hl_store_width(v));
        } else if (op == "link") {
            int gen, width;
            in >> gen >> width;
            std::printf("%.17g\n", hl_link_gbs(gen, width));
        } else if (op == "bytes") {
            unsigned long long b;
            in >> b;
            std::printf("%llu\n", hl_buffer_bytes(b));
        } else if (op == "next") {
            unsigned long long s;
            in >> s;
            std::printf("%u\n", hl_next_seed((uint32_t)s));
        } else if (op == "check") {
            unsigned long long n, seed, idx, mask;
            in >> n >> seed;
            std::vector<uint32_t> p(n);
            hl_fill(p.data(), n, (uint32_t)seed);
            while (in >> idx >> mask) p[idx] ^= (uint32_t)mask;
            unsigned long long first = ~0ull;
            const unsigned long long bad = hl_check(p.data(), n, (uint32_t)seed, &first);
            std::printf("%llu %llu\n", bad, first);
        } else if (op == "verdict") {
            HlEvidence e;
            int ok, seq_ok, cs_ok;
            in >> ok >> seq_ok >> cs_ok;
            for (auto& r : e.rounds) in >> r;
            for (auto& m : e.mismatches) in >> m;
            e.calls_ok = ok;
            e.seq_ok = seq_ok;
            e.checksums_ok = cs_ok;
            std::printf("%d\n", hl_healthy(e) ? 1 : 0);
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
