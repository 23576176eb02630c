// compute_test_image_test.cpp -- CPU driver over csrc/compute_test_math.hpp for tests/test_compute_test_tables_cpu.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python test can hold the product's
// shared-memory image against tests/compute_test_tables.py:
//   image <seed> <fmt> <tile>                 -> the tile's shared-memory image, byte by byte (ct_build_tile)
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>

#include "compute_test_math.hpp"

using namespace b2dp;

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op;
        in >> op;
        if (op == "image") {
            unsigned long long seed;
            int fmt, tile;
            in >> seed >> fmt >> tile;
            CtTile t;
            ct_build_tile((uint32_t)seed, fmt, tile, t);
            for (size_t i = 0; i < t.image.size(); ++i) std::printf(i ? " %u" : "%u", (unsigned)t.image[i]);
            std::printf("\n");
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
