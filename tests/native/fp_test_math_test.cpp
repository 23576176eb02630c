// fp_test_math_test.cpp -- CPU driver over csrc/fp_test_math.hpp for tests/test_fp_test_cpu.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python test can hold the host arithmetic of
// b2dp_fp_test against tests/fp_test_oracle.py:
//   tile <seed> <fmt> <tile>   -> the operand table ([slot][thread] values' bits), then every thread's result words,
//                                 then the kCtThreads check values
//   fma <fmt> <x> <a> <b>      -> ft_fma on the operands' bits (std::fmaf / std::fma), the host's reference
//   fold <n> <w0..wn-1>        -> ft_fold
//   time <seed>                -> milliseconds to build every tile of every format (what one b2dp_fp_test call builds)
//   bounds                     -> the constants the static_asserts bound
#include <chrono>
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>

#include "fp_test_math.hpp"

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
            FtTile t;
            ft_build_tile((uint32_t)seed, fmt, tile, t);
            const int vb = ft_value_bytes(fmt);
            for (size_t i = 0; i < t.table.size() / vb; ++i) {
                uint64_t v = 0;
                std::memcpy(&v, &t.table[i * vb], vb);
                std::printf(i ? " %llu" : "%llu", (unsigned long long)v);
            }
            for (uint32_t w : t.words) std::printf(" %u", w);
            for (uint32_t c : t.check) std::printf(" %u", c);
            std::printf("\n");
        } else if (op == "fma") {
            int fmt;
            unsigned long long x, a, b;
            in >> fmt >> x >> a >> b;
            std::printf("%llu\n", (unsigned long long)ft_fma(fmt, x, a, b));
        } else if (op == "fold") {
            int n;
            in >> n;
            std::vector<uint32_t> w(n);
            for (auto& v : w) {
                unsigned long long u;
                in >> u;
                v = (uint32_t)u;
            }
            std::printf("%u\n", ft_fold(w.data(), n));
        } else if (op == "time") {
            unsigned long long seed;
            in >> seed;
            const auto t0 = std::chrono::steady_clock::now();
            FtTile t;
            for (int f = 0; f < kFtFormats; ++f)
                for (int tile = 0; tile < kCtTiles; ++tile) ft_build_tile((uint32_t)seed, f, tile, t);
            std::printf("%.3f\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
        } else if (op == "bounds") {
            std::printf("%d %d %d %lld %d %d %d %d %d\n", kFtX, kFtAB, kFtDmmaK, kFtDmmaMax, kFtDmmaScaleExp,
                        kFtWords[FT_FP32], kFtWords[FT_FP64], kFtWords[FT_DMMA], kFtSubnormalXExp);
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
