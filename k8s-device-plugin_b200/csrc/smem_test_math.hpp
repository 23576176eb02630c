// smem_test_math.hpp -- host-side arithmetic of the on-demand shared-memory self-test (b2dp_smem_test, smem_selftest.cuh).
//
// Pure C++ (no CUDA; the pattern and rank key are also compiled for the device), so the CPU tests compile it as it is
// (tests/native/smem_test_math_test.cpp) and compare it with the restatement in tests/smem_test_oracle.py:
//   - sh_pattern:     P(w), the value of word w under a tile's data background
//   - sh_rank_key:    R(rank), the constant the cells a DSMEM CTA owns also carry
//   - sh_reads:       format, tile, thread  ->  every value the thread reads in one march, in the kernel's read order,
//                     the DSMEM rank key XORed out
//   - sh_build_tile:  a tile's table (kind, key, fault-hook word and element) and its [thread] check values
// The per-CTA record (CtRecord), its completeness rule and the verdict are the tensor-core test's
// (compute_test_math.hpp).
//
// The array: every CTA takes kShBytes = 227 KiB of dynamic shared memory, the sm_90 opt-in maximum per block, so one
// CTA runs per SM and covers everything a CTA can address.  Thread t owns word t + 128 k (k < 454), 16-byte vector
// t + 128 k (k < 113, and k = 113 for t < 64: the 64-vector tail) and 8-byte pair t + 128 k (k < 227) -- a warp touches
// consecutive words, so no access has a bank conflict.  Not covered: the 1 KiB the runtime reserves per CTA, and the
// part of the SM's 256 KiB L1 / shared array outside the shared carve-out.  Nothing is claimed about how word
// addresses map to physical cells.
//
// The marches (^ = ascending k, v = descending k; ~P = P ^ 0xFFFFFFFF; a barrier separates the elements):
//   SH_WORD   (March C-, ld/st.shared.u32)  ^w(P)  ^r(P)w(~P)  ^r(~P)w(P)  vr(P)w(~P)  vr(~P)w(P)  ^r(P)
//   SH_BYTE   (mixed widths)                ^w(P) as st.u8 bytes 3,0,2,1 of each word
//                                           ^r(P) as ld.v4 per vector, w(~P) as two st.u16 per word
//                                           vr(~P) as ld.u8 of bytes 0..3 of each word, w(P) as st.v4
//                                           vr(P) as ld.v2 per pair
//   SH_DSMEM  (cluster of 2)                ^w(P) into the peer's array (st.shared::cluster)
//                                           ^r(P)w(~P) in the own array
//                                           ^r(~P)w(P) in the peer's array (ld/st.shared::cluster)
//                                           ^r(P) in the own array
//             every cell also carries R(owner's cluster rank): a write delivered to the wrong CTA reads wrong.
// Every march writes P and ~P, so every bit of every word is written and read back as 0 and as 1.  A read value is
// one element of a load: a word of ld.u32 / ld.v2 / ld.v4 (in lane order), a byte of ld.u8 (zero-extended).
#pragma once
#include <cstdint>
#include <vector>

#include "compute_test_math.hpp"  // ct_stream_key, CtRecord, kCtThreads, kCtTiles, kCtReps

#if defined(__CUDACC__)
#define B2DP_SH_HD __host__ __device__
#else
#define B2DP_SH_HD
#endif

namespace b2dp {

enum ShFormat { SH_WORD = 0, SH_BYTE = 1, SH_DSMEM = 2 };
constexpr int kShFormats = 3;
static_assert(kShFormats == kCtFormats, "the verdict and the result struct are shared with the tensor-core test");

constexpr uint32_t kShBytes = 232448;                   // 227 KiB: cudaDevAttrMaxSharedMemoryPerBlockOptin on sm_90
constexpr int kShWords = (int)(kShBytes / 4);           // 58,112
constexpr int kShWordsPerThread = kShWords / kCtThreads;
constexpr int kShVecs = (int)(kShBytes / 16);           // 14,528 16-byte vectors
constexpr int kShVecsPerThread = kShVecs / kCtThreads;  // every thread's vectors; threads < kShVecTail own one more
constexpr int kShVecTail = kShVecs % kCtThreads;
constexpr int kShPairs = (int)(kShBytes / 8);           // 29,056 8-byte pairs
constexpr int kShPairsPerThread = kShPairs / kCtThreads;
static_assert(kShWords == 58112 && kShWords % kCtThreads == 0 && kShWordsPerThread == 454, "454 words per thread");
static_assert(kShVecsPerThread == 113 && kShVecTail == 64, "113.5 vectors per thread: a 64-vector tail");
static_assert(kShPairs % kCtThreads == 0 && kShPairsPerThread == 227, "227 pairs per thread");

constexpr uint32_t kShPatternMul = 2654435761u;         // hbm_probe.cuh kPatternMul
constexpr int kShElements[kShFormats] = {6, 4, 4};      // march elements per format
constexpr int kShTableWords = 4;                        // a tile's table: kind, key, hook word, hook element
constexpr uint32_t kShHookWord = 4660;                  // the word the product's fault hook flips ...
constexpr uint32_t kShHookElement = 0;                  // ... right after this element of the first comparison
constexpr int kShDumpWords = kShWords + 2 * kCtThreads; // DUMP, per CTA and tile: the image, then folds and error counts
constexpr int kShMaxReads = 2734;                       // the most values one thread reads in one march (SH_BYTE, t < 64)

// Bytes read and written by one CTA in one comparison (one march over its array): the rate's numerator.
inline double sh_bytes_per_tile(int fmt) { return (double)kShBytes * (fmt == SH_WORD ? 10 : 6); }

// The kind of data background of tile t: 0 solid, 1 bit checkerboard, 2 alternating 128-byte bank rows,
// 3 walking one, 4 (tiles 4..7) a distinct value per word.
inline uint32_t sh_kind(int tile) { return tile < 4 ? (uint32_t)tile : 4u; }
inline uint32_t sh_key(uint32_t seed, int fmt, int tile) {
    return sh_kind(tile) == 4 ? ct_stream_key(seed, 3 + fmt, tile, 0) : 0u;
}

B2DP_SH_HD inline uint32_t sh_pattern(uint32_t kind, uint32_t key, uint32_t w) {
    switch (kind) {
        case 0: return 0u;
        case 1: return 0x55555555u ^ ((w & 1u) ? ~0u : 0u);
        case 2: return ((w >> 5) & 1u) ? ~0u : 0u;
        case 3: return 1u << ((w + (w >> 5)) & 31u);  // rotl(1, .): over 32 rows every bank holds it at every bit
        default: return (w * kShPatternMul) ^ key;
    }
}
B2DP_SH_HD inline uint32_t sh_rank_key(uint32_t rank) { return (rank + 1u) * 0x9E3779B9u; }

inline uint32_t sh_fold(const uint32_t* v, int n) {
    uint32_t h = 0;
    for (int j = 0; j < n; ++j) h += (2u * (uint32_t)j + 1u) * v[j];
    return h;
}

// Every value thread t reads in one march of format fmt over a clean array, in the kernel's order (for SH_DSMEM with
// the owner's rank key removed, so both ranks read the same sequence).
inline void sh_reads(int fmt, uint32_t kind, uint32_t key, int t, std::vector<uint32_t>& out) {
    out.clear();
    auto P = [&](uint32_t w) { return sh_pattern(kind, key, w); };
    auto words = [&](bool up, uint32_t inv) {
        for (int i = 0; i < kShWordsPerThread; ++i) {
            const int k = up ? i : kShWordsPerThread - 1 - i;
            out.push_back(P((uint32_t)(t + kCtThreads * k)) ^ inv);
        }
    };
    if (fmt == SH_WORD) {
        words(true, 0u);
        words(true, ~0u);
        words(false, 0u);
        words(false, ~0u);
        words(true, 0u);
    } else if (fmt == SH_DSMEM) {
        words(true, 0u);
        words(true, ~0u);
        words(true, 0u);
    } else {
        const int nv = kShVecsPerThread + (t < kShVecTail ? 1 : 0);
        for (int k = 0; k < nv; ++k)
            for (int i = 0; i < 4; ++i) out.push_back(P((uint32_t)(4 * (t + kCtThreads * k) + i)));
        for (int k = nv - 1; k >= 0; --k)
            for (int i = 0; i < 4; ++i)
                for (int b = 0; b < 4; ++b) out.push_back((~P((uint32_t)(4 * (t + kCtThreads * k) + i)) >> (8 * b)) & 0xFFu);
        for (int k = kShPairsPerThread - 1; k >= 0; --k)
            for (int i = 0; i < 2; ++i) out.push_back(P((uint32_t)(2 * (t + kCtThreads * k) + i)));
    }
}

// One tile: its table (kind, key, the fault hook's word and element) and every thread's check value.
inline void sh_build_tile(uint32_t seed, int fmt, int tile, uint32_t* table, uint32_t* check) {
    table[0] = sh_kind(tile);
    table[1] = sh_key(seed, fmt, tile);
    table[2] = kShHookWord;
    table[3] = kShHookElement;
    std::vector<uint32_t> r;
    r.reserve(kShMaxReads);
    for (int t = 0; t < kCtThreads; ++t) {
        sh_reads(fmt, table[0], table[1], t, r);
        check[t] = sh_fold(r.data(), (int)r.size());
    }
}

}  // namespace b2dp
