// memtest_math.hpp -- host-side arithmetic of the on-demand memory test (b2dp_memtest, hbm_memtest.cuh).
//
// Pure C++ (no CUDA), so the CPU tests compile it as it is (tests/native/memtest_math_test.cpp) and compare it with the
// Python restatement in tests/memtest_oracle.py:
//   - memtest_plan:            free / total / reserve / max  ->  the segment sizes the test allocates
//   - memtest_segment_seed:    the pattern seed of segment g
//   - range_checksum_host:     closed-form checksum of the pattern over the word-index range [base, base + n)
//   - memtest_expected_checksum: the same over a list of segments (what every reading march element must sum to)
//   - memtest_healthy:         the verdict
#pragma once
#include <array>
#include <cstdint>
#include <vector>

#include "pattern_math.hpp"

namespace b2dp {

constexpr uint64_t kMemtestChunkBytes = 1ull << 30;  // every segment is one chunk, except that the last may be smaller
constexpr uint64_t kMemtestAlignBytes = 2ull << 20;  // segment sizes are multiples of 2 MiB: a whole number of tiles
constexpr int kMemtestMaxSegments = 256;             // 256 GiB; the segment table is a 3 KiB kernel parameter
constexpr int kMarchElements = 4;                    // E0 w(P), E1 r(P) w(~P), E2 r(~P) w(P), E3 r(P)

// Default reserve (reserve_bytes = 0): a tenth of the device's memory stays free for whoever allocates next.
inline uint64_t memtest_default_reserve(uint64_t total_bytes) { return total_bytes / 10; }

// Segment g of a test keyed with `seed` holds word(i, seed_g); the seed changes from segment to segment, so two
// segments that alias one physical page, or two words 2^32 indices (16 GiB) apart, never expect the same value.
inline uint32_t memtest_segment_seed(uint32_t seed, uint32_t g) { return seed ^ (uint32_t)(g * 0x9E3779B9u); }

// The sizes of the segments to allocate: min(max_bytes, free - reserve), rounded down to 2 MiB, cut into 1 GiB
// chunks with a smaller last one, and at most kMemtestMaxSegments of them.  max_bytes = 0 means no cap;
// reserve_bytes = 0 means memtest_default_reserve(total).
inline std::vector<uint64_t> memtest_plan(uint64_t free_bytes, uint64_t total_bytes, uint64_t reserve_bytes,
                                          uint64_t max_bytes) {
    const uint64_t reserve = reserve_bytes ? reserve_bytes : memtest_default_reserve(total_bytes);
    uint64_t budget = free_bytes > reserve ? free_bytes - reserve : 0;
    if (max_bytes && max_bytes < budget) budget = max_bytes;
    const uint64_t cap = kMemtestChunkBytes * (uint64_t)kMemtestMaxSegments;
    if (budget > cap) budget = cap;
    budget -= budget % kMemtestAlignBytes;
    std::vector<uint64_t> segs;
    while (budget) {
        const uint64_t s = budget < kMemtestChunkBytes ? budget : kMemtestChunkBytes;
        segs.push_back(s);
        budget -= s;
    }
    return segs;
}

// Bit counts of the pattern over [base, base + n): the difference of two prefix counts (pattern_math.hpp), which
// wrap at 2^32 words exactly like the kernels' uint32 index.
inline std::array<unsigned long long, 32> pattern_bit_counts_range(unsigned long long base, unsigned long long n) {
    std::array<unsigned long long, 32> hi = pattern_bit_counts_host(base + n);
    const std::array<unsigned long long, 32> lo = pattern_bit_counts_host(base);
    for (int b = 0; b < 32; ++b) hi[b] -= lo[b];
    return hi;
}

inline unsigned long long range_checksum_host(unsigned long long base, unsigned long long n, uint32_t seed) {
    return expected_checksum_from_counts(pattern_bit_counts_range(base, n), n, seed);
}

// Checksum of a clean march element that reads the segments `seg_bytes` (concatenated in order) under the seeds
// memtest_segment_seed(seed, g) ^ inv; inv = 0xFFFFFFFF is the complement pattern ~P.
inline unsigned long long memtest_expected_checksum(const std::vector<uint64_t>& seg_bytes, uint32_t seed, uint32_t inv) {
    unsigned long long sum = 0, base = 0;
    for (size_t g = 0; g < seg_bytes.size(); ++g) {
        const unsigned long long n = seg_bytes[g] / 4;
        sum += range_checksum_host(base, n, memtest_segment_seed(seed, (uint32_t)g) ^ inv);
        base += n;
    }
    return sum;
}

// What the verdict looks at.  Element 0 only writes; elements 1-3 read.
struct MemtestEvidence {
    bool launch_ok = false;                      // every launch succeeded and finished before the deadline
    unsigned long long mismatches[kMarchElements] = {};
    unsigned long long checksum[kMarchElements] = {};
    unsigned long long expected[kMarchElements] = {};
    unsigned long long ecc_uncorrected = 0;      // NVML volatile uncorrected-ECC delta over the test
    bool remap_failed = false, remap_pending = false;  // HBM row remapping (nvmlDeviceGetRemappedRows)
};

// Healthy iff the launches succeeded, every reading element verified every word and summed to the closed form (a
// kernel that skipped tiles cannot pass), no uncorrected ECC error appeared and no row remap failed or is pending.
// Corrected ECC errors are reported, not failed.
inline bool memtest_healthy(const MemtestEvidence& e) {
    if (!e.launch_ok || e.ecc_uncorrected != 0 || e.remap_failed || e.remap_pending) return false;
    for (int k = 1; k < kMarchElements; ++k)
        if (e.mismatches[k] != 0 || e.checksum[k] != e.expected[k]) return false;
    return true;
}

}  // namespace b2dp
