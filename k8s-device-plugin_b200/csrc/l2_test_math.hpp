// l2_test_math.hpp -- host-side arithmetic of the on-demand L2 self-test (b2dp_l2_test, l2_selftest.cuh).
//
// Pure C++ (no CUDA; the pattern, the mix and the scratch layout are also compiled for the device), so the CPU tests
// compile it as it is (tests/native/l2_test_math_test.cpp) and compare it with tests/l2_test_oracle.py:
//   - l2_pattern:      P(w), the value of word w of a window under a tile's data background
//   - l2_reads:        format, tile, thread  ->  every value the thread reads from one 2 KiB block in one march, in
//                      read order, with the block key removed
//   - l2_atom_*:       the L2_ATOM operands, final values and return folds for every count of contributors
//   - l2_build_tile:   a tile's table and its [thread] check values
// The per-CTA record (CtRecord), its completeness rule and the verdict are the tensor-core test's
// (compute_test_math.hpp).
//
// L2_WORD / L2_BYTE.  The span is K x G blocks of kL2BlockWords words (G = the cooperative grid, K >= 1 from the
// device's L2 size, l2_span_blocks); the buffer holds kL2Windows spans and round r marches window r % kL2Windows.  In
// element e, CTA c owns slice (c + e) % G: K consecutive blocks, and thread t owns 16-byte vector t of each.  A word
// written in element e is therefore read in element e + 1 by CTA c - 1, behind a grid barrier.
//   L2_WORD  (March C-, v4 ld/st.global.cg)  ^w(P)  ^r(P)w(~P)  ^r(~P)w(P)  vr(P)w(~P)  vr(~P)w(P)  ^r(P)
//   L2_BYTE  (mixed widths)                  ^w(P) as st.global.cg.u8, bytes 3,0,2,1 of each word
//                                            ^r(P) as ld.v4, w(~P) as two st.global.cg.u16 per word
//                                            vr(~P) as ld.v4, w(P) as st.u8 bytes 3,0,2,1
//                                            ^r(P) as ld.v4
// P(w) = sh_pattern(kind, key, w % 512) ^ (w / 512 + 1) * blockmul: the shared-memory test's data backgrounds on each
// block, and in the keyed tiles (blockmul != 0) a block key, so a write that lands in the wrong block reads wrong.
// A thread's fold takes every value it reads with the block key XORed out, weight 2j + 1 for the j-th value it reads
// from a block; over the K blocks of every element that is K x the host's check.
//
// L2_ATOM.  A hot block of kL2AtomSlots x kL2AtomRows x 32 words every CTA shares: warp g = 4 c + w (of 4 G) lane l
// targets word (slot, g % kL2AtomRows, l) of every slot, so n(row) = number of warps with g % rows == row, at most
// kL2AtomMaxN, contribute to each word, each with the operand of its rank q = g / kL2AtomRows.  Every op commutes, so
// the final value after n contributions is order-free; the host tabulates it for every n (l2_atom_final).  The
// returns of add / inc / dec / CAS are {f^i(init) : i < n}; for exch {returns} + {final} = {init} + {operands}.  Both
// enter order-free folds: the sum and the xor of l2_mix(value, lane) over the grid, tabulated per n over the 32 lanes.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#include "compute_test_math.hpp"  // CtRecord, kCtThreads, kCtTiles, kCtReps
#include "smem_test_math.hpp"     // sh_pattern, sh_kind

#if defined(__CUDACC__)
#define B2DP_L2_HD __host__ __device__
#else
#define B2DP_L2_HD
#endif

namespace b2dp {

enum L2Format { L2_WORD = 0, L2_BYTE = 1, L2_ATOM = 2 };
constexpr int kL2Formats = 3;
static_assert(kL2Formats == kCtFormats, "the verdict and the result struct are shared with the tensor-core test");

constexpr int kL2BlockWords = 4 * kCtThreads;      // one 16-byte vector per thread: 2 KiB
constexpr uint32_t kL2BlockBytes = 4u * kL2BlockWords;
constexpr int kL2Windows = 4;                      // the buffer is this many spans; round r marches window r % 4
constexpr int kL2SpanNum = 3, kL2SpanDen = 8;      // default span = 3/8 of cudaDevAttrL2CacheSize (DESIGN 4.12)
constexpr int kL2Elements[kL2Formats] = {6, 4, 0};
constexpr int kL2ReadElements[kL2Formats] = {5, 3, 0};
constexpr int kL2MaxCtas = 4096;                   // 16 resident CTAs x kCtMaxSmId SMs

// The scratch buffer (uint32_t words): a header, the per-CTA fold slots, then the data (the windows or the hot block).
constexpr int kL2HdrBlocks = 0;      // header: K, blocks per slice (host-written)
constexpr int kL2HdrDump = 1;        // header: word offset of the DUMP area (the harness only)
constexpr int kL2HdrCount = 8;       // grid barrier arrivals
constexpr int kL2HdrGen = 16;        // grid barrier generation (its own 32-byte sector)
constexpr int kL2HdrClaim = 24;      // the fault hook's claim
constexpr int kL2HdrStop = 32;       // CTA 0's stop decision for the round that just ended
constexpr int kL2HdrWords = 64;
constexpr int kL2FoldWords = 16;     // per CTA: sum and xor of each return op (L2_ATOM)
constexpr int kL2DataOff = kL2HdrWords + kL2FoldWords * kL2MaxCtas;
static_assert(kL2DataOff % 32 == 0, "the data starts on a 128-byte line");
constexpr unsigned long long kL2GraceNs = 2000000000ull;  // a grid-wide wait gives up this long past the deadline

// ---- L2_WORD / L2_BYTE --------------------------------------------------------------------------------------------
constexpr int kL2TableWords = 8;     // WORD / BYTE tile table: kind, key, blockmul, hook word, hook element
constexpr uint32_t kL2BlockMul = 0x9E3779B9u;
constexpr uint32_t kL2HookWord = 37;       // the word of the claimant's slice the fault hook flips ...
constexpr uint32_t kL2HookElement = 0;     // ... right after this element of the first comparison

B2DP_L2_HD inline uint32_t l2_pattern(uint32_t kind, uint32_t key, uint32_t blockmul, uint32_t w) {
    return sh_pattern(kind, key, w % (uint32_t)kL2BlockWords) ^ ((w / (uint32_t)kL2BlockWords + 1u) * blockmul);
}

// Blocks per CTA slice for a span of about span_bytes on a grid of G CTAs (at least one).
inline uint32_t l2_span_blocks(unsigned long long span_bytes, int grid) {
    const unsigned long long k = span_bytes / ((unsigned long long)grid * kL2BlockBytes);
    return k ? (uint32_t)k : 1u;
}
inline unsigned long long l2_default_span(unsigned long long l2_bytes) { return l2_bytes * kL2SpanNum / kL2SpanDen; }

// Bytes read and written by the whole grid in one comparison of a span of `span` bytes: the rate's numerator.
inline double l2_bytes_per_comparison(int fmt, double span) { return span * (fmt == L2_WORD ? 10 : 7); }

// Every value thread t reads from one block in one march (block key removed), in the kernel's order.
inline void l2_reads(int fmt, uint32_t kind, uint32_t key, int t, std::vector<uint32_t>& out) {
    out.clear();
    auto rd = [&](uint32_t inv) {
        for (int i = 0; i < 4; ++i) out.push_back(sh_pattern(kind, key, (uint32_t)(4 * t + i)) ^ inv);
    };
    if (fmt == L2_WORD) {
        rd(0u); rd(~0u); rd(0u); rd(~0u); rd(0u);
    } else if (fmt == L2_BYTE) {
        rd(0u); rd(~0u); rd(0u);
    }
}
inline uint32_t l2_fold(const uint32_t* v, int n) {
    uint32_t h = 0;
    for (int j = 0; j < n; ++j) h += (2u * (uint32_t)j + 1u) * v[j];
    return h;
}

// ---- L2_ATOM ------------------------------------------------------------------------------------------------------
enum L2AtomSlot {
    LA_ADD = 0, LA_INC, LA_DEC, LA_EXCH, LA_CAS32, LA_CAS64,  // LA_CAS64: two words, lo then hi
    LA_AND = 7, LA_OR, LA_XOR, LA_MIN_S, LA_MAX_S, LA_MIN_U, LA_MAX_U,
    LA_ADD64 = 14,                                             // two words
    LA_F32 = 16, LA_F64 = 17,                                  // LA_F64: two words
    LA_F16X2 = 19, LA_BF16X2, LA_V4RED = 21, LA_V4ATOM = 25,   // the v4 ops: four words each
    kL2AtomSlots = 29
};
constexpr int kL2AtomRows = 32;
constexpr int kL2AtomMaxN = 4 * kL2MaxCtas / kL2AtomRows;   // 512 warps per word at most
// inc / dec wrap bounds are 2 .. kL2WrapMax and the initial value is at most the bound, so a word crosses its bound
// whenever it takes more than kL2WrapMax contributions: on every grid of 8 x (kL2WrapMax + 1) CTAs or more.
constexpr uint32_t kL2WrapMax = 16;
constexpr int kL2WrapMinGrid = kL2AtomRows * ((int)kL2WrapMax + 1) / 4;
static_assert(kL2WrapMinGrid == 136, "an H100 runs 4 x 132 = 528 L2_ATOM CTAs: every word wraps");
constexpr int kL2AtomRet = 6;   // return ops, in this order: add, inc, dec, exch, cas32, cas64
constexpr int kL2AtomRetSlot[kL2AtomRet] = {LA_ADD, LA_INC, LA_DEC, LA_EXCH, LA_CAS32, LA_CAS64};
constexpr int kL2AtomHotWords = kL2AtomSlots * kL2AtomRows * 32;
// The tile table: operands [slot][q], finals [slot][n], return sums and xors [op][n].
constexpr int kL2AtomOpOff = 0;
constexpr int kL2AtomFinalOff = kL2AtomOpOff + kL2AtomSlots * kL2AtomMaxN;
constexpr int kL2AtomSumOff = kL2AtomFinalOff + kL2AtomSlots * (kL2AtomMaxN + 1);
constexpr int kL2AtomXorOff = kL2AtomSumOff + kL2AtomRet * (kL2AtomMaxN + 1);
constexpr int kL2AtomTableWords = (kL2AtomXorOff + kL2AtomRet * (kL2AtomMaxN + 1) + 3) & ~3;  // padded to 16 bytes
static_assert(kL2AtomTableWords % 4 == 0, "16-byte tile tables");
static_assert(kL2FoldWords >= 2 * kL2AtomRet, "the per-CTA fold slot holds a sum and a xor per return op");

// Float reductions take small integers, and every partial sum in every order must be exact (its magnitude at most
// the format's largest integer with every smaller one representable: 2^11 f16, 2^8 bf16, 2^24 f32, 2^53 f64).
constexpr int kL2F32Max = 1000, kL2F16Max = 3, kL2Bf16Max = 1;
constexpr long long kL2F64Max = 1ll << 40;
static_assert((long long)kL2F32Max * (kL2AtomMaxN + 1) < (1ll << 24), "f32 partial sums stay exact");
static_assert(kL2F16Max * (kL2AtomMaxN + 1) <= 2048, "f16 partial sums stay exact");
static_assert(kL2Bf16Max * (kL2AtomMaxN / 2) <= 256, "bf16: at most every second operand is nonzero, |sum| <= 256");
static_assert((double)kL2F64Max * (kL2AtomMaxN + 1) < 9007199254740992.0, "f64 partial sums stay exact");

// Hot word i: the slot whose value it follows, and its row and lane.  A one-word op's plane is [row][lane]; the
// 64-bit and v4 ops interleave their 2 or 4 words per (row, lane) over their 2 or 4 planes.
B2DP_L2_HD inline int l2_atom_word(int i, int& row, int& lane) {
    const int s = i / (kL2AtomRows * 32);
    int base = s, span = 1;
    if (s == LA_CAS64 || s == LA_CAS64 + 1) { base = LA_CAS64; span = 2; }
    else if (s == LA_ADD64 || s == LA_ADD64 + 1) { base = LA_ADD64; span = 2; }
    else if (s == LA_F64 || s == LA_F64 + 1) { base = LA_F64; span = 2; }
    else if (s >= LA_V4RED && s < LA_V4ATOM) { base = LA_V4RED; span = 4; }
    else if (s >= LA_V4ATOM) { base = LA_V4ATOM; span = 4; }
    const int j = i - base * kL2AtomRows * 32;
    row = (j / span) / 32;
    lane = (j / span) % 32;
    return base + j % span;
}

// Warps that target each word of row `row` on a grid of G CTAs.
B2DP_L2_HD inline int l2_atom_n(int grid, int row) {
    const int warps = 4 * grid;
    return row < warps ? (warps - 1 - row) / kL2AtomRows + 1 : 0;
}

// A bijective mix of a value, keyed by the lane whose word it came from (murmur3's finaliser).
B2DP_L2_HD inline uint32_t l2_mix(uint32_t v, uint32_t lane) {
    uint32_t h = v ^ ((lane + 1u) * 0x9E3779B9u);
    h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
    return h;
}
B2DP_L2_HD inline uint32_t l2_mix64(uint64_t v, uint32_t lane) {
    return l2_mix((uint32_t)v ^ l2_mix((uint32_t)(v >> 32), lane + 32u), lane);
}

inline uint32_t l2_rand(uint32_t seed, int tile, int a, int b) {
    return l2_mix(seed ^ l2_mix((uint32_t)tile * 0x632BE5ABu + (uint32_t)a * 0x85157AF5u + (uint32_t)b, 77u), 91u);
}
inline uint32_t l2_f32_bits(double v) { float f = (float)v; uint32_t u; memcpy(&u, &f, 4); return u; }
inline float l2_bits_f32(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
inline uint64_t l2_f64_bits(double v) { uint64_t u; memcpy(&u, &v, 8); return u; }
inline double l2_bits_f64(uint64_t u) { double d; memcpy(&d, &u, 8); return d; }
// An integer |i| <= 2048 as f16 bits, exactly; as bf16 bits (|i| <= 256).
inline uint32_t l2_f16_bits(int i) {
    if (i == 0) return 0;
    const uint32_t s = i < 0 ? 0x8000u : 0u, a = (uint32_t)(i < 0 ? -i : i);
    int e = 0;
    while ((a >> (e + 1)) != 0) ++e;
    const uint32_t m = e <= 10 ? (a << (10 - e)) & 0x3FFu : (a >> (e - 10)) & 0x3FFu;
    return s | ((uint32_t)(e + 15) << 10) | m;
}
inline int l2_f16_int(uint32_t b) {
    if ((b & 0x7FFFu) == 0) return 0;
    const int e = (int)((b >> 10) & 0x1Fu) - 15;
    const uint32_t m = (b & 0x3FFu) | 0x400u;
    const int a = e >= 10 ? (int)(m << (e - 10)) : (int)(m >> (10 - e));
    return (b & 0x8000u) ? -a : a;
}
inline uint32_t l2_bf16_bits(int i) { return l2_f32_bits((double)i) >> 16; }
inline int l2_bf16_int(uint32_t b) { return (int)l2_bits_f32(b << 16); }

// The operand word of slot s for the warp of rank q (ADD: 1, INC / DEC: their wrap bound, CAS: unused).
inline uint32_t l2_atom_operand(uint32_t seed, int tile, int s, int q) {
    const uint32_t r = l2_rand(seed, tile, 100 + s, q);
    const uint32_t b = l2_rand(seed, tile, 200 + s, 0);
    switch (s) {
        case LA_ADD: return 1u;
        case LA_INC: case LA_DEC: return 2u + b % (kL2WrapMax - 1u);
        case LA_EXCH: case LA_XOR: return r | 1u;
        case LA_CAS32: case LA_CAS64: case LA_CAS64 + 1: return 0u;
        case LA_AND: return ~(1u << (q & 31));
        case LA_OR: return 1u << (q & 31);
        case LA_ADD64: return r;
        case LA_ADD64 + 1: return r & 0xFFu;
        case LA_F32: return l2_f32_bits((double)((int)(r % (2 * kL2F32Max + 1)) - kL2F32Max));
        case LA_F64: case LA_F64 + 1: {
            const long long v = (long long)(((uint64_t)l2_rand(seed, tile, 100 + LA_F64, q) << 9) % (2ull * kL2F64Max + 1)) - kL2F64Max;
            const uint64_t u = l2_f64_bits((double)v);
            return s == LA_F64 ? (uint32_t)u : (uint32_t)(u >> 32);
        }
        case LA_F16X2: {
            const int lo = (int)(r % (2 * kL2F16Max + 1)) - kL2F16Max, hi = (int)((r >> 8) % (2 * kL2F16Max + 1)) - kL2F16Max;
            return l2_f16_bits(lo) | (l2_f16_bits(hi) << 16);
        }
        case LA_BF16X2: {
            if (q & 1) return 0u;
            const int lo = (r & 1) ? kL2Bf16Max : -kL2Bf16Max, hi = (r & 2) ? kL2Bf16Max : -kL2Bf16Max;
            return l2_bf16_bits(lo) | (l2_bf16_bits(hi) << 16);
        }
        default:  // LA_MIN_S .. LA_MAX_U, and the f32 lanes of the v4 ops
            if (s >= LA_V4RED) return l2_f32_bits((double)((int)(r % (2 * kL2F32Max + 1)) - kL2F32Max));
            return r;
    }
}

// The initial word of slot s (every lane and row holds it).
inline uint32_t l2_atom_init(uint32_t seed, int tile, int s) {
    const uint32_t r = l2_rand(seed, tile, 300 + s, 0);
    switch (s) {
        case LA_INC: case LA_DEC: return r % (l2_atom_operand(seed, tile, s, 0) + 1u);
        case LA_CAS64: return 0xFFFFFF00u + (r & 0x7Fu);   // the increments carry into the high word
        case LA_F32: return l2_f32_bits((double)((int)(r % 2001) - 1000));
        case LA_F64: case LA_F64 + 1: {
            const uint64_t u = l2_f64_bits((double)((long long)(l2_rand(seed, tile, 300 + LA_F64, 0) % 2001) - 1000));
            return s == LA_F64 ? (uint32_t)u : (uint32_t)(u >> 32);
        }
        case LA_F16X2: return l2_f16_bits((int)(r % 7) - 3) | (l2_f16_bits((int)((r >> 8) % 7) - 3) << 16);
        case LA_BF16X2: return 0u;
        default:
            if (s >= LA_V4RED) return l2_f32_bits((double)((int)(r % 2001) - 1000));
            return r;
    }
}

inline uint32_t l2_inc(uint32_t old, uint32_t b) { return old >= b ? 0u : old + 1u; }
inline uint32_t l2_dec(uint32_t old, uint32_t b) { return (old == 0u || old > b) ? b : old - 1u; }

// The host's tile of L2_ATOM: operands, every slot's final value after n = 0 .. kL2AtomMaxN contributions, and the
// return folds over the 32 lanes of a row for every n.
inline void l2_atom_build(uint32_t seed, int tile, uint32_t* tab) {
    uint32_t* op = tab + kL2AtomOpOff;
    uint32_t* fin = tab + kL2AtomFinalOff;
    for (int s = 0; s < kL2AtomSlots; ++s)
        for (int q = 0; q < kL2AtomMaxN; ++q) op[s * kL2AtomMaxN + q] = l2_atom_operand(seed, tile, s, q);
    auto X = [&](int s, int q) { return op[s * kL2AtomMaxN + q]; };
    auto F = [&](int s, int n) -> uint32_t& { return fin[s * (kL2AtomMaxN + 1) + n]; };
    uint32_t v[kL2AtomSlots];
    for (int s = 0; s < kL2AtomSlots; ++s) v[s] = l2_atom_init(seed, tile, s);
    for (int n = 0;; ++n) {
        for (int s = 0; s < kL2AtomSlots; ++s) F(s, n) = v[s];
        if (n == kL2AtomMaxN) break;
        const int q = n;  // contribution n is the warp of rank q = n: the order does not matter
        v[LA_ADD] += 1u;
        v[LA_INC] = l2_inc(v[LA_INC], X(LA_INC, q));
        v[LA_DEC] = l2_dec(v[LA_DEC], X(LA_DEC, q));
        v[LA_EXCH] = 0u;  // exch has no order-free final value: it enters the multiset fold
        v[LA_CAS32] += 1u;
        const uint64_t c64 = ((uint64_t)v[LA_CAS64 + 1] << 32 | v[LA_CAS64]) + 1u;
        v[LA_CAS64] = (uint32_t)c64; v[LA_CAS64 + 1] = (uint32_t)(c64 >> 32);
        v[LA_AND] &= X(LA_AND, q);
        v[LA_OR] |= X(LA_OR, q);
        v[LA_XOR] ^= X(LA_XOR, q);
        v[LA_MIN_S] = (uint32_t)std::min((int32_t)v[LA_MIN_S], (int32_t)X(LA_MIN_S, q));
        v[LA_MAX_S] = (uint32_t)std::max((int32_t)v[LA_MAX_S], (int32_t)X(LA_MAX_S, q));
        v[LA_MIN_U] = std::min(v[LA_MIN_U], X(LA_MIN_U, q));
        v[LA_MAX_U] = std::max(v[LA_MAX_U], X(LA_MAX_U, q));
        const uint64_t a64 = ((uint64_t)v[LA_ADD64 + 1] << 32 | v[LA_ADD64]) +
                             ((uint64_t)X(LA_ADD64 + 1, q) << 32 | X(LA_ADD64, q));
        v[LA_ADD64] = (uint32_t)a64; v[LA_ADD64 + 1] = (uint32_t)(a64 >> 32);
        v[LA_F32] = l2_f32_bits((double)l2_bits_f32(v[LA_F32]) + (double)l2_bits_f32(X(LA_F32, q)));
        const double f64 = l2_bits_f64((uint64_t)v[LA_F64 + 1] << 32 | v[LA_F64]) +
                           l2_bits_f64((uint64_t)X(LA_F64 + 1, q) << 32 | X(LA_F64, q));
        v[LA_F64] = (uint32_t)l2_f64_bits(f64); v[LA_F64 + 1] = (uint32_t)(l2_f64_bits(f64) >> 32);
        v[LA_F16X2] = l2_f16_bits(l2_f16_int(v[LA_F16X2] & 0xFFFFu) + l2_f16_int(X(LA_F16X2, q) & 0xFFFFu)) |
                      (l2_f16_bits(l2_f16_int(v[LA_F16X2] >> 16) + l2_f16_int(X(LA_F16X2, q) >> 16)) << 16);
        v[LA_BF16X2] = l2_bf16_bits(l2_bf16_int(v[LA_BF16X2] & 0xFFFFu) + l2_bf16_int(X(LA_BF16X2, q) & 0xFFFFu)) |
                       (l2_bf16_bits(l2_bf16_int(v[LA_BF16X2] >> 16) + l2_bf16_int(X(LA_BF16X2, q) >> 16)) << 16);
        for (int i = 0; i < 8; ++i)
            v[LA_V4RED + i] = l2_f32_bits((double)l2_bits_f32(v[LA_V4RED + i]) + (double)l2_bits_f32(X(LA_V4RED + i, q)));
    }
    // return folds: sum and xor over the lanes of l2_mix of every value a row's n contributions return
    uint32_t* sum = tab + kL2AtomSumOff;
    uint32_t* xr = tab + kL2AtomXorOff;
    for (int k = 0; k < kL2AtomRet; ++k) {
        const int s = kL2AtomRetSlot[k];
        // n = 0: exch's multiset is {init} (its final), the others return nothing
        const uint32_t init_exch = l2_atom_init(seed, tile, LA_EXCH);
        uint32_t sm = 0, x = 0;
        if (k == 3)
            for (uint32_t l = 0; l < 32; ++l) { sm += l2_mix(init_exch, l); x ^= l2_mix(init_exch, l); }
        sum[k * (kL2AtomMaxN + 1)] = sm;
        xr[k * (kL2AtomMaxN + 1)] = x;
        for (int n = 1; n <= kL2AtomMaxN; ++n) {
            for (uint32_t l = 0; l < 32; ++l) {
                uint32_t m;
                if (k == 3) m = l2_mix(X(LA_EXCH, n - 1), l);                         // an operand joins the multiset
                else if (k == 5) m = l2_mix64((uint64_t)F(s + 1, n - 1) << 32 | F(s, n - 1), l);
                else m = l2_mix(F(s, n - 1), l);                                    // the value before contribution n
                sm += m;
                x ^= m;
            }
            sum[k * (kL2AtomMaxN + 1) + n] = sm;
            xr[k * (kL2AtomMaxN + 1) + n] = x;
        }
    }
}

inline uint32_t l2_table_bytes(int fmt) {
    return 4u * (fmt == L2_ATOM ? (uint32_t)kL2AtomTableWords : (uint32_t)kL2TableWords);
}

// One tile: its table and every thread's check value (L2_ATOM: zero, the table carries every reference value).
inline void l2_build_tile(uint32_t seed, int fmt, int tile, uint32_t* table, uint32_t* check) {
    if (fmt == L2_ATOM) {
        l2_atom_build(seed, tile, table);
        for (int t = 0; t < kCtThreads; ++t) check[t] = 0;
        return;
    }
    memset(table, 0, 4 * kL2TableWords);
    table[0] = sh_kind(tile);
    table[1] = sh_key(seed, 3 + fmt, tile);
    table[2] = sh_kind(tile) == 4 ? kL2BlockMul : 0u;
    table[3] = kL2HookWord;
    table[4] = kL2HookElement;
    std::vector<uint32_t> r;
    for (int t = 0; t < kCtThreads; ++t) {
        l2_reads(fmt, table[0], table[1], t, r);
        check[t] = l2_fold(r.data(), (int)r.size());
    }
}

}  // namespace b2dp
