// l2_test_math_test.cpp -- CPU driver over csrc/l2_test_math.hpp for tests/test_l2_test_cpu.py.
//
// Reads one query per line from stdin and prints one answer line, so the Python test can hold the host arithmetic of
// b2dp_l2_test against tests/l2_test_oracle.py:
//   tile <seed> <fmt> <tile>   -> the tile table, then the kCtThreads check values
//   n <grid>                   -> l2_atom_n for every row
//   bounds                     -> the layout constants
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "l2_test_math.hpp"

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
            std::vector<uint32_t> table(l2_table_bytes(fmt) / 4);
            uint32_t check[kCtThreads];
            l2_build_tile((uint32_t)seed, fmt, tile, table.data(), check);
            for (size_t i = 0; i < table.size(); ++i) std::printf(i ? " %u" : "%u", table[i]);
            for (uint32_t c : check) std::printf(" %u", c);
            std::printf("\n");
        } else if (op == "n") {
            int grid;
            in >> grid;
            for (int r = 0; r < kL2AtomRows; ++r) std::printf(r ? " %d" : "%d", l2_atom_n(grid, r));
            std::printf("\n");
        } else if (op == "bounds") {
            std::printf("%d %d %d %d %d %d %d %d %d %d\n", kL2BlockWords, kL2Windows, kL2AtomSlots, kL2AtomRows,
                        kL2AtomMaxN, kL2AtomHotWords, kL2AtomTableWords, kL2TableWords, kL2DataOff, kL2MaxCtas);
        } else {
            std::printf("?\n");
        }
        std::fflush(stdout);
    }
    return 0;
}
