// memtest_math_test.cpp -- CPU driver over csrc/memtest_math.hpp for tests/test_memtest_cpu.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python test can hold the host arithmetic
// of b2dp_memtest against tests/memtest_oracle.py on tables of inputs:
//   plan <free> <total> <reserve> <max>              -> segment sizes ("-" for none)
//   seed <seed> <g>                                  -> memtest_segment_seed
//   range <base> <n> <seed>                          -> range_checksum_host
//   expect <seed> <inv> <bytes...>                   -> memtest_expected_checksum
//   verdict <ok> <m0..m3> <c0..c3> <e0..e3> <unc> <remap_failed> <remap_pending>   -> 1 / 0
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>

#include "memtest_math.hpp"

using namespace b2dp;

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op;
        in >> op;
        if (op == "plan") {
            unsigned long long f, t, r, m;
            in >> f >> t >> r >> m;
            const std::vector<uint64_t> segs = memtest_plan(f, t, r, m);
            if (segs.empty()) std::printf("-");
            for (size_t i = 0; i < segs.size(); ++i) std::printf(i ? " %llu" : "%llu", (unsigned long long)segs[i]);
            std::printf("\n");
        } else if (op == "seed") {
            unsigned long long s, g;
            in >> s >> g;
            std::printf("%u\n", memtest_segment_seed((uint32_t)s, (uint32_t)g));
        } else if (op == "range") {
            unsigned long long b, n, s;
            in >> b >> n >> s;
            std::printf("%llu\n", range_checksum_host(b, n, (uint32_t)s));
        } else if (op == "expect") {
            unsigned long long s, inv, x;
            in >> s >> inv;
            std::vector<uint64_t> segs;
            while (in >> x) segs.push_back(x);
            std::printf("%llu\n", memtest_expected_checksum(segs, (uint32_t)s, (uint32_t)inv));
        } else if (op == "verdict") {
            MemtestEvidence e;
            int ok, rf, rp;
            in >> ok;
            for (auto& v : e.mismatches) in >> v;
            for (auto& v : e.checksum) in >> v;
            for (auto& v : e.expected) in >> v;
            in >> e.ecc_uncorrected >> rf >> rp;
            e.launch_ok = ok != 0;
            e.remap_failed = rf != 0;
            e.remap_pending = rp != 0;
            std::printf("%d\n", memtest_healthy(e) ? 1 : 0);
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
