// rf_test_math.hpp -- host-side arithmetic of the on-demand register-file self-test (b2dp_regfile_test,
// rf_selftest.cuh).
//
// Pure C++ (no CUDA; the pattern is also compiled for the device), so the CPU tests compile it as it is
// (tests/native/rf_test_math_test.cpp) and compare it with the restatement in tests/rf_test_oracle.py:
//   - rf_pattern:     P(t, j), the value held register j of thread t carries under a tile's data background
//   - rf_reads:       format, tile, thread  ->  every value the thread reads from its held registers in one march, in
//                     the kernel's read order
//   - rf_build_tile:  a tile's table (kind, key, fault-hook register, element and thread) and its [thread] check values
// The per-CTA record (CtRecord), its completeness rule and the verdict are the tensor-core test's
// (compute_test_math.hpp); the pattern pieces are the shared-memory test's (smem_test_math.hpp).
//
// The register file: every thread holds kRfHeld 32-bit values in general registers across every element boundary of
// the march.  __launch_bounds__(128, 2) lets ptxas give each thread up to 255 registers, which the SM allocates as
// 256; two CTAs of four warps then take 2 x 4 x 32 x 256 = 65,536 registers, the SM's whole file.  Which physical cells
// a register index maps to is not published, and nothing is claimed about it.
//
// The marches (~P = P ^ 0xFFFFFFFF; a barrier separates the elements; ^ / v = j ascending / descending):
//   RF_ALU   w(P) by ld.shared.v4  ^r(P)w(~P)  ^r(~P)w(P)  vr(P)w(~P)  vr(~P)w(P)  ^r(P)      (March C-)
//            every w after the first is an in-place LOP3 (r ^= ~0): the ALU write-back port
//   RF_LOAD  w(P) by ld.shared.v4  ^r(P)w(~P) by ld.v4  ^r(~P)w(P) by ld.v2  ^r(P)w(~P) by ld.v2  ^r(~P)
//            every register is written by the load-return port, by a quad and by a pair load, each time with the
//            complement of what it held, so a dropped lane of a wide write reads wrong
//   RF_HOLD  w(P) by ld.shared.v4, held kRfHoldNs while the warps sleep, ^r(P)w(~P) (in-place LOP3), held again,
//            ^r(~P): a cell that loses its value while its SMSP idles.  Not a manufacturing-grade retention test: the
//            interval is fixed, short and at whatever voltage and temperature the card runs at.
// Every march writes P and ~P, so every bit of every held register is written and read back as 0 and as 1.
#pragma once
#include <cstdint>
#include <vector>

#include "compute_test_math.hpp"  // ct_stream_key, CtRecord, kCtThreads, kCtTiles, kCtReps
#include "smem_test_math.hpp"     // sh_pattern, kShPatternMul

#if defined(__CUDACC__)
#define B2DP_RF_HD __host__ __device__
#else
#define B2DP_RF_HD
#endif

namespace b2dp {

enum RfFormat { RF_ALU = 0, RF_LOAD = 1, RF_HOLD = 2 };
constexpr int kRfFormats = 3;
static_assert(kRfFormats == kCtFormats, "the verdict and the result struct are shared with the tensor-core test");

constexpr int kRfHeld = 204;                           // held registers per thread: the largest count with no spills
constexpr int kRfElements[kRfFormats] = {6, 5, 3};     // march elements per format
constexpr int kRfReads[kRfFormats] = {5, 4, 2};        // reads of every held register per march
constexpr int kRfWrites[kRfFormats] = {5, 4, 2};       // writes of every held register per march
constexpr unsigned long long kRfHoldNs = 100000;       // RF_HOLD: each value is held this long (100 us) ...
constexpr unsigned kRfSleepNs = 5000;                  // ... in nanosleep steps of this many ns
constexpr int kRfTableWords = 5;                       // a tile's table: kind, key, hook register, element, thread
constexpr uint32_t kRfHookReg = kRfHeld / 2;           // the held register the product's fault hook flips ...
constexpr uint32_t kRfHookElement = 0;                 // ... right after this element of the first comparison ...
constexpr uint32_t kRfHookThread = 0;                  // ... in this thread
constexpr int kRfImageWords = kRfHeld * kCtThreads;    // the shared-memory image the held values are loaded from
constexpr int kRfParamWords = 12;                      // shared memory ahead of the image: generator, mask, tallies
constexpr uint32_t kRfSmemBytes = 4u * (kRfParamWords + 2 * kCtThreads + kRfImageWords);  // + pin and check words
constexpr int kRfDumpWords = kRfImageWords + 2 * kCtThreads;  // DUMP, per CTA and tile: the registers, folds, errors
static_assert(kRfHeld % 4 == 0, "the held registers load as quads");
static_assert(2 * (kRfSmemBytes + 1024) <= 233472, "two CTAs must fit an SM's shared memory");

// Register bytes read and written by one CTA in one comparison (one march): the rate's numerator.
inline double rf_bytes_per_tile(int fmt) {
    return 4.0 * kRfHeld * kCtThreads * (kRfReads[fmt] + kRfWrites[fmt]);
}

// The kind of data background of tile t: 0 solid, 1 bit checkerboard (0x55555555 / 0xAAAAAAAA on even / odd
// registers), 2 alternating registers (0 / ~0), 3 walking one (rotl(1, t + j)), 4 (tiles 4..7) a distinct value per
// register of the CTA.
inline uint32_t rf_kind(int tile) { return tile < 4 ? (uint32_t)tile : 4u; }
inline uint32_t rf_key(uint32_t seed, int fmt, int tile) {
    return rf_kind(tile) == 4 ? ct_stream_key(seed, 6 + fmt, tile, 0) : 0u;
}

B2DP_RF_HD inline uint32_t rf_pattern(uint32_t kind, uint32_t key, uint32_t t, uint32_t j) {
    switch (kind) {
        case 2: return (j & 1u) ? ~0u : 0u;
        case 3: { const uint32_t s = (t + j) & 31u; return 1u << s; }
        case 4: return sh_pattern(4, key, t * (uint32_t)kRfHeld + j);
        default: return sh_pattern(kind, key, j);  // 0 solid, 1 bit checkerboard
    }
}

// The kernel's branch-free form of rf_pattern (and what it loads after every barrier): P(t, j) =
// (t * kRfHeld + j) * mul ^ (j odd ? odd : even) ^ rotl(one, t + j).
struct RfGenParams {
    uint32_t mul, even, odd, one;
};
B2DP_RF_HD inline RfGenParams rf_gen_params(uint32_t kind, uint32_t key) {
    RfGenParams p{0u, 0u, 0u, 0u};
    if (kind == 1) { p.even = 0x55555555u; p.odd = 0xAAAAAAAAu; }
    else if (kind == 2) p.odd = ~0u;
    else if (kind == 3) p.one = 1u;
    else if (kind >= 4) { p.mul = kShPatternMul; p.even = p.odd = key; }
    return p;
}

inline uint32_t rf_fold(const uint32_t* v, int n) { return sh_fold(v, n); }

// Every value thread t reads from its held registers in one march of format fmt, in the kernel's order.
inline void rf_reads(int fmt, uint32_t kind, uint32_t key, int t, std::vector<uint32_t>& out) {
    out.clear();
    auto pass = [&](bool down, uint32_t inv) {
        for (int k = 0; k < kRfHeld; ++k)
            out.push_back(rf_pattern(kind, key, (uint32_t)t, (uint32_t)(down ? kRfHeld - 1 - k : k)) ^ inv);
    };
    if (fmt == RF_ALU) {
        pass(false, 0u);
        pass(false, ~0u);
        pass(true, 0u);
        pass(true, ~0u);
        pass(false, 0u);
    } else if (fmt == RF_LOAD) {
        pass(false, 0u);
        pass(false, ~0u);
        pass(false, 0u);
        pass(false, ~0u);
    } else {
        pass(false, 0u);
        pass(false, ~0u);
    }
}

// One tile: its table (kind, key, the fault hook's register, element and thread) and every thread's check value.
inline void rf_build_tile(uint32_t seed, int fmt, int tile, uint32_t* table, uint32_t* check) {
    table[0] = rf_kind(tile);
    table[1] = rf_key(seed, fmt, tile);
    table[2] = kRfHookReg;
    table[3] = kRfHookElement;
    table[4] = kRfHookThread;
    std::vector<uint32_t> r;
    r.reserve((size_t)kRfHeld * 5);
    for (int t = 0; t < kCtThreads; ++t) {
        rf_reads(fmt, table[0], table[1], t, r);
        check[t] = rf_fold(r.data(), (int)r.size());
    }
}

}  // namespace b2dp
