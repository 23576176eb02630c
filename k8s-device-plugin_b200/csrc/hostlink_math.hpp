// hostlink_math.hpp -- host arithmetic of the on-demand host-link self-test (b2dp_hostlink_test).
//
// Everything the test compares against is computed here, on the host, from the probe's pattern (hbm_probe.cuh,
// pattern_math.hpp): the words a buffer must hold, the store width the SM format uses for each vector, the capacity of
// the PCIe link NVML reports, the buffer size a caller may ask for, and the verdict.  No value comes from the device
// under test.  Oracle: tests/hostlink_oracle.py.
#pragma once
#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define B2DP_HL_HD __host__ __device__
#else
#define B2DP_HL_HD
#endif

namespace b2dp {

constexpr unsigned long long kHlDefaultBytes = 64ull << 20;  // per buffer (profiles/hostlink_size_sweep_h100.txt)
constexpr unsigned long long kHlMaxBytes = 1ull << 30;
constexpr int kHlFormats = 3;                                 // B2DP_HL_H2D, B2DP_HL_D2H, B2DP_HL_SM
constexpr int kHlStoreWidths = 5;

// The requested bytes per buffer: 0 = the default; otherwise a multiple of 16 no larger than 1 GiB, else 0 (invalid).
inline unsigned long long hl_buffer_bytes(unsigned long long requested) {
    if (requested == 0) return kHlDefaultBytes;
    if (requested % 16 != 0 || requested > kHlMaxBytes) return 0;
    return requested;
}

// Bytes per store the SM format uses for 16-byte vector `vec`: 16, 8, 4, 2, 1, 16, ... so every fifth vector crosses
// the link with each byte-enable shape.
B2DP_HL_HD constexpr unsigned hl_store_width(unsigned long long vec) {
    return 16u >> (unsigned)(vec % kHlStoreWidths);
}

// The probe's seed schedule: the next round's seed.
inline uint32_t hl_next_seed(uint32_t seed) { return seed * 1664525u + 1013904223u; }

// Per-direction capacity in GB/s of a PCIe link of generation `gen` and `width` lanes, before packet overhead:
// Gen1-2 carry 8 bits in 10 at 2.5 / 5 GT/s, Gen3-5 128 bits in 130 at 8 / 16 / 32 GT/s.  Anything else: 0.
inline double hl_link_gbs(int gen, int width) {
    if (width <= 0) return 0.0;
    double gts = 0.0, eff = 0.0;
    switch (gen) {
        case 1: gts = 2.5; eff = 8.0 / 10.0; break;
        case 2: gts = 5.0; eff = 8.0 / 10.0; break;
        case 3: gts = 8.0; eff = 128.0 / 130.0; break;
        case 4: gts = 16.0; eff = 128.0 / 130.0; break;
        case 5: gts = 32.0; eff = 128.0 / 130.0; break;
        default: return 0.0;
    }
    return gts * eff * width / 8.0;
}

// word(i, seed) = (uint32(i) * 2654435761) ^ seed, for i in [0, n_words)
inline void hl_fill(uint32_t* p, size_t n_words, uint32_t seed) {
    uint32_t m = 0;
    for (size_t i = 0; i < n_words; ++i, m += 2654435761u) p[i] = m ^ seed;
}

// Words of p that differ from the pattern; *first_bad = the lowest such index (left alone if there is none).
inline unsigned long long hl_check(const uint32_t* p, size_t n_words, uint32_t seed, unsigned long long* first_bad) {
    unsigned long long bad = 0;
    uint32_t m = 0;
    for (size_t i = 0; i < n_words; ++i, m += 2654435761u)
        if (p[i] != (m ^ seed)) {
            if (bad == 0 && i < *first_bad) *first_bad = i;
            ++bad;
        }
    return bad;
}

// What the verdict reads.
struct HlEvidence {
    bool calls_ok = true;                       // every CUDA call succeeded before the deadline
    unsigned long long rounds[kHlFormats] = {};
    bool seq_ok = true;                         // every ProbeOut sequence number echoed, every record arrived
    unsigned long long mismatches[kHlFormats] = {};
    bool checksums_ok = true;                   // every device checksum equals the host's closed form
};

inline bool hl_healthy(const HlEvidence& e) {
    if (!e.calls_ok || !e.seq_ok || !e.checksums_ok) return false;
    for (int f = 0; f < kHlFormats; ++f)
        if (e.rounds[f] == 0 || e.mismatches[f] != 0) return false;
    return true;
}

}  // namespace b2dp
