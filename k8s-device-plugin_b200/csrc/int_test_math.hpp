// int_test_math.hpp -- host-side arithmetic of the on-demand integer and warp-exchange self-test (b2dp_int_test,
// int_selftest.cuh).
//
// Pure C++ (no CUDA), so the CPU tests compile it as it is (tests/native/int_test_math_test.cpp) and compare it with the
// independent restatement in tests/int_test_oracle.py:
//   - it_operand / it_operands: seed, format, tile -> the operand table ([slot][thread] words), crafted classes included
//   - it_results:               the reference result words of every thread, in the kernel's word order
//   - it_fold:                  the per-thread comparison value
//   - it_build_tile:            the table a launch reads verbatim and the check values
// The per-CTA record (CtRecord), its completeness rule and the verdict are the tensor-core test's
// (compute_test_math.hpp): the kernel keeps that test's round / tile / repetition structure.
//
// Why the host can predict the device bit for bit: every op is two's-complement arithmetic, bit logic or a lane
// permutation, which the PTX ISA defines completely; nothing below uses a compiler builtin whose result for 0 is
// undefined, a signed overflow or a shift by the operand's width.
//
// Layout.  A thread's operands are kItSets[fmt] sets of kItSetSlots[fmt] words; slot = set * kItSetSlots + k.  Every op
// of the format runs on every set, and set s's result words are s * kItSetWords[fmt] + j, in the order of the ItMadWord /
// ItBitWord / ItWarpWord enums.  The low sets are crafted (it_operands), the rest random full-width words.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "compute_test_math.hpp"  // ct_mix, ct_hash, CtRecord, kCtThreads, kCtTiles, kCtReps

namespace b2dp {

enum ItFormat { IT_MAD = 0, IT_BIT = 1, IT_WARP = 2 };
constexpr int kItFormats = 3;
static_assert(kItFormats == kCtFormats, "the verdict and the result struct are shared with the tensor-core test");

constexpr int kItSets[kItFormats] = {20, 12, 12};
constexpr int kItSetSlots[kItFormats] = {4, 3, 7};
constexpr int kItSetWords[kItFormats] = {14, 23, 20};
constexpr int kItSlots[kItFormats] = {20 * 4, 12 * 3, 12 * 7};
constexpr int kItWords[kItFormats] = {20 * 14, 12 * 23, 12 * 20};
constexpr int kItMaxWords = 280;

// IT_MAD: slots a, b, c, d.  X = (b:a) and Y = (d:c) are the 64-bit operands of the carry pairs and Y mad.wide's addend.
enum ItMadWord {
    IM_MAD_LO = 0,   // mad.lo.u32 a, b, c
    IM_MULHI_U,      // mul.hi.u32 a, b
    IM_MULHI_S,      // mul.hi.s32 a, b
    IM_WIDE_U_LO,    // mad.wide.u32 a, b, Y
    IM_WIDE_U_HI,
    IM_WIDE_S_LO,    // mad.wide.s32 a, b, Y
    IM_WIDE_S_HI,
    IM_ADD_LO,       // add.cc.u32 a, c ; addc.u32 b, d
    IM_ADD_HI,
    IM_SUB_LO,       // sub.cc.u32 a, c ; subc.u32 b, d
    IM_SUB_HI,
    IM_DP4A_SS,      // dp4a.s32.s32 a, b, c
    IM_DP4A_SU,      // dp4a.s32.u32 a, b, c  (a's bytes signed, b's unsigned)
    IM_DP4A_UU,      // dp4a.u32.u32 a, b, c
};
// IT_BIT: slots a, b, c.
constexpr int kItLop3 = 8;
constexpr uint32_t kItLop3Imm[kItLop3] = {0x80, 0xFE, 0x96, 0xE8, 0xCA, 0x3C, 0x01, 0x69};
enum ItBitWord {
    IB_LOP3 = 0,     // lop3.b32 a, b, c, kItLop3Imm[0..7]: 8 words
    IB_SHF_L = 8,    // shf.l.wrap.b32 a (low), b (high), c
    IB_SHF_R,        // shf.r.wrap.b32 a, b, c
    IB_SHR_S,        // shr.s32 a, c
    IB_SHL,          // shl.b32 a, c
    IB_POPC,         // popc.b32 a
    IB_CLZ,          // clz.b32 b (on a, ptxas derives it from bfind.u32 a's FLO.U32 instead of running its own)
    IB_BFIND_U,      // bfind.u32 a
    IB_BFIND_S,      // bfind.s32 a
    IB_BREV,         // brev.b32 a
    IB_PRMT,         // prmt.b32 a, b, c
    IB_MIN_S,        // min.s32 a, b
    IB_MAX_S,
    IB_MIN_U,
    IB_MAX_U,
    IB_SAD,          // sad.u32 a, b, c
};
// IT_WARP: slots v (shfl data), b (source lane / delta / lane mask), c (shfl's c operand for idx / down / bfly; up
// takes c & 0x1f00), q (ballot predicate: q != 0), r (redux data), m (match.any data), m2 (match.all data).
enum ItWarpWord {
    IW_IDX = 0,      // shfl.sync.idx.b32 d|p: d, then p as 0 / 1
    IW_IDX_P,
    IW_UP,
    IW_UP_P,
    IW_DOWN,
    IW_DOWN_P,
    IW_BFLY,
    IW_BFLY_P,
    IW_BALLOT,       // vote.sync.ballot.b32 (q != 0)
    IW_ADD,          // redux.sync.add.u32 r
    IW_MIN_S,
    IW_MAX_S,
    IW_MIN_U,
    IW_MAX_U,
    IW_AND,
    IW_OR,
    IW_XOR,
    IW_MATCH_ANY,    // match.any.sync.b32 m
    IW_MATCH_ALL,    // match.all.sync.b32 d|p m2: d, then p
    IW_MATCH_ALL_P,
};

// operand table of one tile: [slot][thread] words, so a warp's loads of one slot are coalesced
inline uint32_t it_table_bytes(int fmt) { return (uint32_t)(kItSlots[fmt] * kCtThreads * 4); }
// Result words of one comparison (one repetition of one tile by one CTA); the rate counts every folded word.
inline double it_ops_per_tile(int fmt) { return (double)kCtThreads * kItWords[fmt]; }

// ---- the ops, per the PTX ISA ------------------------------------------------------------------------------------
inline uint32_t it_rotl(uint32_t x, int n) { n &= 31; return n ? x << n | x >> (32 - n) : x; }
inline uint64_t it_sext(uint32_t a) { return (uint64_t)(int64_t)(int32_t)a; }
inline uint32_t it_mulhi_u(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t it_mulhi_s(uint32_t a, uint32_t b) { return (uint32_t)((it_sext(a) * it_sext(b)) >> 32); }  // mod 2^64
inline uint64_t it_madwide_u(uint32_t a, uint32_t b, uint64_t y) { return (uint64_t)a * b + y; }
inline uint64_t it_madwide_s(uint32_t a, uint32_t b, uint64_t y) { return it_sext(a) * it_sext(b) + y; }
inline uint32_t it_dp4a(uint32_t a, uint32_t b, uint32_t c, bool sa, bool sb) {
    uint32_t s = c;
    for (int i = 0; i < 4; ++i) {
        const uint32_t xa = (a >> (8 * i)) & 0xFF, xb = (b >> (8 * i)) & 0xFF;
        const uint32_t ea = sa && (xa & 0x80) ? xa | 0xFFFFFF00u : xa, eb = sb && (xb & 0x80) ? xb | 0xFFFFFF00u : xb;
        s += ea * eb;  // mod 2^32: the low 32 bits of a product do not depend on signedness once extended
    }
    return s;
}
inline uint32_t it_lop3(uint32_t a, uint32_t b, uint32_t c, uint32_t imm) {
    uint32_t d = 0;
    for (int k = 0; k < 8; ++k)
        if (imm >> k & 1) d |= (k & 4 ? a : ~a) & (k & 2 ? b : ~b) & (k & 1 ? c : ~c);
    return d;
}
inline uint32_t it_shf_l_wrap(uint32_t lo, uint32_t hi, uint32_t c) {
    const int n = c & 31;
    return n ? hi << n | lo >> (32 - n) : hi;
}
inline uint32_t it_shf_r_wrap(uint32_t lo, uint32_t hi, uint32_t c) {
    const int n = c & 31;
    return n ? lo >> n | hi << (32 - n) : lo;
}
inline uint32_t it_shr_s32(uint32_t a, uint32_t c) {
    const uint32_t sign = a >> 31 ? ~0u : 0u;
    if (c >= 32) return sign;
    return c ? a >> c | sign << (32 - c) : a;
}
inline uint32_t it_shl(uint32_t a, uint32_t c) { return c >= 32 ? 0u : a << c; }
inline uint32_t it_popc(uint32_t a) {
    uint32_t n = 0;
    for (int i = 0; i < 32; ++i) n += a >> i & 1;
    return n;
}
inline uint32_t it_bfind_u(uint32_t a) {  // position of the most significant 1; 0xFFFFFFFF if none
    for (int i = 31; i >= 0; --i)
        if (a >> i & 1) return (uint32_t)i;
    return ~0u;
}
inline uint32_t it_bfind_s(uint32_t a) { return it_bfind_u(a >> 31 ? ~a : a); }  // of the most significant non-sign bit
inline uint32_t it_clz(uint32_t a) { return a ? 31u - it_bfind_u(a) : 32u; }
inline uint32_t it_brev(uint32_t a) {
    uint32_t d = 0;
    for (int i = 0; i < 32; ++i) d |= (a >> i & 1) << (31 - i);
    return d;
}
inline uint32_t it_prmt(uint32_t a, uint32_t b, uint32_t c) {  // default mode: bytes 0..3 of a, 4..7 of b
    const uint64_t src = (uint64_t)b << 32 | a;
    uint32_t d = 0;
    for (int i = 0; i < 4; ++i) {
        const uint32_t sel = c >> (4 * i) & 0xF;
        uint32_t byte = (uint32_t)(src >> (8 * (sel & 7))) & 0xFF;
        if (sel & 8) byte = byte & 0x80 ? 0xFF : 0x00;  // replicate the byte's sign
        d |= byte << (8 * i);
    }
    return d;
}
inline uint32_t it_min_s(uint32_t a, uint32_t b) { return (int32_t)a < (int32_t)b ? a : b; }
inline uint32_t it_max_s(uint32_t a, uint32_t b) { return (int32_t)a > (int32_t)b ? a : b; }
inline uint32_t it_min_u(uint32_t a, uint32_t b) { return a < b ? a : b; }
inline uint32_t it_max_u(uint32_t a, uint32_t b) { return a > b ? a : b; }
inline uint32_t it_sad_u(uint32_t a, uint32_t b, uint32_t c) { return c + (a < b ? b - a : a - b); }

// shfl.sync with the full member mask (PTX ISA "shfl.sync"): lane's own b and c choose its source lane j; out of range,
// the lane keeps its own value and p is false.
enum ItShfl { IT_SHFL_IDX, IT_SHFL_UP, IT_SHFL_DOWN, IT_SHFL_BFLY };
inline void it_shfl(int mode, const uint32_t* v, const uint32_t* b, const uint32_t* c, uint32_t* d, uint32_t* p) {
    for (int lane = 0; lane < 32; ++lane) {
        const int bval = b[lane] & 31, cval = c[lane] & 31, segmask = c[lane] >> 8 & 31;
        const int max_lane = (lane & segmask) | (cval & ~segmask & 31), min_lane = lane & segmask;
        int j;
        bool pv;
        switch (mode) {
            case IT_SHFL_UP: j = lane - bval; pv = j >= max_lane; break;
            case IT_SHFL_DOWN: j = lane + bval; pv = j <= max_lane; break;
            case IT_SHFL_BFLY: j = lane ^ bval; pv = j <= max_lane; break;
            default: j = min_lane | (bval & ~segmask & 31); pv = j <= max_lane; break;
        }
        if (!pv) j = lane;
        d[lane] = v[j];
        p[lane] = pv;
    }
}

// ---- the fold -----------------------------------------------------------------------------------------------------
// Four interleaved chains h_q <- rotl((h_q ^ w) * kItMul, kItFoldRot), word i to chain i % 4, combined by rotations.
// Each step is a bijection of h_q for a fixed w and of w for a fixed h_q (XOR, a multiplication by an odd number mod
// 2^32, a rotation), so one wrong word always changes its chain's final value and with it the check.  Two wrong words
// in one chain cancel only if the second word's error undoes the 32-bit state difference the first left; wrong words
// in different chains cancel only if the rotated final differences XOR to zero.  The rotation is what keeps two results
// that are both wrong in bit 31 from cancelling: 2^31 times an odd number is 2^31 again, so without it a bit-31 error
// stays a bit-31 state difference that the chain's next bit-31 error undoes, as in sum (2j + 1) w_j.
constexpr uint32_t kItMul = 2654435761u;  // kPatternMul
constexpr int kItFoldRot = 13;
constexpr uint32_t kItFoldInit[4] = {0x9E3779B1u, 0x85EBCA77u, 0xC2B2AE3Du, 0x27D4EB2Fu};
inline uint32_t it_fold(const uint32_t* w, int n) {
    uint32_t h[4] = {kItFoldInit[0], kItFoldInit[1], kItFoldInit[2], kItFoldInit[3]};
    for (int i = 0; i < n; ++i) h[i & 3] = it_rotl((h[i & 3] ^ w[i]) * kItMul, kItFoldRot);
    return h[0] ^ it_rotl(h[1], 8) ^ it_rotl(h[2], 16) ^ it_rotl(h[3], 24);
}

// ---- generator ------------------------------------------------------------------------------------------------------
inline uint32_t it_stream_key(uint32_t seed, int fmt, int tile) {
    return ct_mix(seed ^ (uint32_t)(fmt * 16 + tile + 1) * 0xC2B2AE3Du);
}
// the random word of slot `slot` of thread t (what a slot holds unless its set is crafted)
inline uint32_t it_operand(uint32_t seed, int fmt, int tile, int t, int slot) {
    return ct_hash(it_stream_key(seed, fmt, tile), (uint32_t)(t * 128 + slot));
}
// a word shared by the 32 lanes of warp w (IT_WARP's bases)
inline uint32_t it_warp_base(uint32_t seed, int tile, int w, int slot) {
    return ct_hash(it_stream_key(seed, IT_WARP, tile), (uint32_t)(0x10000 + w * 128 + slot));
}
constexpr uint32_t kItDistinctMul = 0x9E3779B1u;  // odd: (base ^ lane) * this is distinct in every lane
inline uint32_t it_shfl_c(int width) { return (uint32_t)(32 - width) << 8 | 0x1f; }

// The table of one tile: tab[slot * kCtThreads + t].
inline void it_operands(uint32_t seed, int fmt, int tile, uint32_t* tab) {
    const int SS = kItSetSlots[fmt];
    for (int t = 0; t < kCtThreads; ++t) {
        for (int s = 0; s < kItSlots[fmt]; ++s) tab[s * kCtThreads + t] = it_operand(seed, fmt, tile, t, s);
        auto at = [&](int set, int k) -> uint32_t& { return tab[(set * SS + k) * kCtThreads + t]; };
        const int i = t % 32, w = t / 32, j = w * 8 + tile;  // (i, j) covers 32 x 32 over a round's tiles and threads
        if (fmt == IT_MAD) {
            enum { A, B, C, D };
            at(0, A) = at(0, B) = ~0u;
            at(1, A) = at(1, B) = 0x80000000u;
            at(2, B) = 0;
            at(3, B) = 1;
            at(4, B) = ~0u;
            at(5, A) = 1u << i;  // one partial-product column alone
            at(5, B) = 1u << j;
            at(6, A) = 0x55555555u;
            at(6, B) = 0xAAAAAAAAu;
            at(6, C) = 0x2AAAAAAAu;  // a + c carries nowhere
            at(7, A) |= 1;           // the addend's low word carries into mad.wide's high word: lo(a * b) + c = 2^32
            at(7, B) |= 1;
            at(7, C) = 0u - at(7, A) * at(7, B);
            at(8, A) |= 0x80000000u;  // the addend wraps the full 64 bits of mad.wide.u32: a * b + Y = 2^64 + t
            at(8, B) |= 0x80000000u;
            const uint64_t y = (uint64_t)t - (uint64_t)at(8, A) * at(8, B);
            at(8, C) = (uint32_t)y;
            at(8, D) = (uint32_t)(y >> 32);
            const int k = (t + tile) % 32 + 1;  // a carry that runs k bits and stops
            at(9, A) = k == 32 ? ~0u : (1u << k) - 1;
            at(9, C) = 1;
            at(10, A) = ~0u;  // a carry through all 32 bits into the high word
            at(10, C) = 1;
            at(11, A) = 0;  // a borrow through all 32 bits
            at(11, C) = 1;
            const int lane = (t + tile) % 4;  // dp4a extremes in one byte lane alone
            at(12, A) = at(12, B) = 0x80u << (8 * lane);
            at(12, C) |= 0xFFFFC000u;  // + (-128)(-128) wraps
            at(13, A) = 0x80808080u;   // all four lanes: (-128)(-128), (-128)(255) and their unsigned readings
            at(13, B) = 0x80FF80FFu;
            at(13, C) = ~0u;
            at(14, A) = 0x80u << (8 * lane);
            at(14, B) = 0xFFu << (8 * lane);
            at(15, A) = at(15, B) = 0xFFu << (8 * lane);
            at(15, C) |= 0xFFFFFF00u;  // + 255 * 255 wraps
        } else if (fmt == IT_BIT) {
            enum { A, B, C };
            at(0, A) = it_rotl(0xF0F0F0F0u, i);  // every bit position meets all 8 input combinations
            at(0, B) = it_rotl(0xCCCCCCCCu, i);
            at(0, C) = it_rotl(0xAAAAAAAAu, i);
            at(1, A) = 1u << i;  // walking one, every amount 0..31
            at(1, B) = 1u << j;
            at(1, C) = (uint32_t)j;
            at(2, A) = ~(1u << i);  // walking zero, amounts 32..63
            at(2, B) = ~(1u << j);
            at(2, C) = 32u + (uint32_t)j;
            if (!(tile & 1)) at(3, C) &= 63;  // random word: amounts 0..63, or any 32-bit amount
            at(4, A) = 0;
            at(4, B) = ~0u;
            at(5, A) = at(5, B) = ~0u;
            uint32_t sel = at(6, C) & 0xFFFF0000u;  // every selector value in every position; the high half is ignored
            for (int p = 0; p < 4; ++p) sel |= (uint32_t)((t + 5 * p + tile) & 15) << (4 * p);
            at(6, C) = sel;
            at(7, A) = 0x80000000u;
            at(7, B) = 0x7FFFFFFFu;
            at(7, C) = ~0u;  // sad wraps
            at(8, B) = at(8, A);
            at(9, A) &= 0x7FFFFFFFu;  // a < b unsigned, a > b signed
            at(9, B) |= 0x80000000u;
            at(10, A) = ~0u;
            at(10, B) = 0;
        } else {
            enum { V, B, C, Q, R, M, M2 };
            const int L = (tile * 4 + w) % 32;  // the warp's lane of the tile: every lane over a round's tiles and warps
            const int mask = L % 31 + 1;        // bfly lane mask / rotation 1..31
            for (int s = 0; s < kItSets[IT_WARP]; ++s) {
                at(s, V) = (it_warp_base(seed, tile, w, s * 7 + V) ^ (uint32_t)i) * kItDistinctMul;
                at(s, C) = it_shfl_c(32);
                at(s, Q) &= 1;
                at(s, M) &= 3;
                if (!(s & 1)) at(s, M2) = it_warp_base(seed, tile, w, s * 7 + M2);
            }
            at(0, B) = (uint32_t)i;
            at(1, B) = 31u - (uint32_t)i;
            at(2, B) = (uint32_t)(i + mask) & 31;
            at(3, B) = (uint32_t)L;
            at(4, B) &= 31;
            at(5, B) |= 32;
            at(5, C) = it_shfl_c(16);
            at(6, B) = 31u - (uint32_t)L;
            at(7, B) = (uint32_t)L;
            at(7, C) = it_shfl_c(16);
            at(8, B) = (uint32_t)L;
            at(8, C) = it_shfl_c(8);
            at(9, V) = tile & 1 ? ~0u : 0u;
            at(9, B) = (uint32_t)mask;
            at(10, V) = i & 1 ? 0xAAAAAAAAu : 0x55555555u;
            at(10, B) = (uint32_t)mask;
            at(10, C) = it_shfl_c(16);
            at(11, V) = 1u << i;
            at(11, B) = (uint32_t)mask;
            at(11, C) = it_shfl_c(8);
            at(0, Q) = 0;
            at(1, Q) |= 1;
            at(2, Q) = i == L;
            at(3, Q) = i != L;
            at(0, R) = i == L ? 0x80000000u : 0x40000000u | at(0, R) >> 2;  // min.s32 / max.u32: the extreme in lane L
            at(1, R) = i == L ? 0x7FFFFFFFu : 0x80000000u | at(1, R) >> 2;  // max.s32 / min.u32
            at(2, R) |= 0xF0000000u;                                        // the sum wraps
            const uint32_t bit = 1u << ((3 * L + 1) % 32);                  // one lane differs in one bit
            at(3, R) = (it_warp_base(seed, tile, w, 3 * 7 + R) | bit) ^ (i == L ? bit : 0u);
            at(4, R) = (it_warp_base(seed, tile, w, 4 * 7 + R) & ~bit) ^ (i == L ? bit : 0u);
            at(0, M) = it_warp_base(seed, tile, w, 0 * 7 + M);
            at(1, M) = (it_warp_base(seed, tile, w, 1 * 7 + M) ^ (uint32_t)i) * kItDistinctMul;
            at(2, M) = it_warp_base(seed, tile, w, 2 * 7 + M) + (uint32_t)(i % 16);  // groups of 2
            at(3, M) = it_warp_base(seed, tile, w, 3 * 7 + M) + (uint32_t)(i % 8);   // of 4
            at(4, M) = it_warp_base(seed, tile, w, 4 * 7 + M) + (uint32_t)(i % 2);   // of 16
            at(1, M2) = it_warp_base(seed, tile, w, 1 * 7 + M2) ^ (i == L ? 1u << L : 0u);
        }
    }
}

// Reference result words of every thread: words[t * kItWords[fmt] + set * kItSetWords[fmt] + j].
inline void it_results(int fmt, const uint32_t* tab, uint32_t* words) {
    const int SS = kItSetSlots[fmt], SW = kItSetWords[fmt], W = kItWords[fmt];
    auto op = [&](int t, int set, int k) { return tab[(set * SS + k) * kCtThreads + t]; };
    for (int set = 0; set < kItSets[fmt]; ++set) {
        if (fmt == IT_MAD) {
            for (int t = 0; t < kCtThreads; ++t) {
                const uint32_t a = op(t, set, 0), b = op(t, set, 1), c = op(t, set, 2), d = op(t, set, 3);
                const uint64_t x = (uint64_t)b << 32 | a, y = (uint64_t)d << 32 | c;
                uint32_t* o = words + (size_t)t * W + set * SW;
                o[IM_MAD_LO] = a * b + c;
                o[IM_MULHI_U] = it_mulhi_u(a, b);
                o[IM_MULHI_S] = it_mulhi_s(a, b);
                const uint64_t wu = it_madwide_u(a, b, y), ws = it_madwide_s(a, b, y);
                o[IM_WIDE_U_LO] = (uint32_t)wu;
                o[IM_WIDE_U_HI] = (uint32_t)(wu >> 32);
                o[IM_WIDE_S_LO] = (uint32_t)ws;
                o[IM_WIDE_S_HI] = (uint32_t)(ws >> 32);
                o[IM_ADD_LO] = (uint32_t)(x + y);
                o[IM_ADD_HI] = (uint32_t)((x + y) >> 32);
                o[IM_SUB_LO] = (uint32_t)(x - y);
                o[IM_SUB_HI] = (uint32_t)((x - y) >> 32);
                o[IM_DP4A_SS] = it_dp4a(a, b, c, true, true);
                o[IM_DP4A_SU] = it_dp4a(a, b, c, true, false);
                o[IM_DP4A_UU] = it_dp4a(a, b, c, false, false);
            }
        } else if (fmt == IT_BIT) {
            for (int t = 0; t < kCtThreads; ++t) {
                const uint32_t a = op(t, set, 0), b = op(t, set, 1), c = op(t, set, 2);
                uint32_t* o = words + (size_t)t * W + set * SW;
                for (int k = 0; k < kItLop3; ++k) o[IB_LOP3 + k] = it_lop3(a, b, c, kItLop3Imm[k]);
                o[IB_SHF_L] = it_shf_l_wrap(a, b, c);
                o[IB_SHF_R] = it_shf_r_wrap(a, b, c);
                o[IB_SHR_S] = it_shr_s32(a, c);
                o[IB_SHL] = it_shl(a, c);
                o[IB_POPC] = it_popc(a);
                o[IB_CLZ] = it_clz(b);
                o[IB_BFIND_U] = it_bfind_u(a);
                o[IB_BFIND_S] = it_bfind_s(a);
                o[IB_BREV] = it_brev(a);
                o[IB_PRMT] = it_prmt(a, b, c);
                o[IB_MIN_S] = it_min_s(a, b);
                o[IB_MAX_S] = it_max_s(a, b);
                o[IB_MIN_U] = it_min_u(a, b);
                o[IB_MAX_U] = it_max_u(a, b);
                o[IB_SAD] = it_sad_u(a, b, c);
            }
        } else {
            for (int w = 0; w < kCtThreads / 32; ++w) {  // a lane's result depends on the other lanes' operands
                uint32_t s[7][32], d[32], p[32], cup[32];
                for (int k = 0; k < 7; ++k)
                    for (int l = 0; l < 32; ++l) s[k][l] = op(w * 32 + l, set, k);
                auto out = [&](int l, int j) -> uint32_t& { return words[(size_t)(w * 32 + l) * W + set * SW + j]; };
                for (int l = 0; l < 32; ++l) cup[l] = s[2][l] & 0x1f00u;
                for (int mode = 0; mode < 4; ++mode) {
                    it_shfl(mode, s[0], s[1], mode == IT_SHFL_UP ? cup : s[2], d, p);
                    for (int l = 0; l < 32; ++l) { out(l, 2 * mode) = d[l]; out(l, 2 * mode + 1) = p[l]; }
                }
                uint32_t ballot = 0, add = 0, mins = s[4][0], maxs = s[4][0], minu = s[4][0], maxu = s[4][0];
                uint32_t band = ~0u, bor = 0, bxor = 0;
                bool all = true;
                for (int l = 0; l < 32; ++l) {
                    const uint32_t r = s[4][l];
                    ballot |= (uint32_t)(s[3][l] != 0) << l;
                    add += r;
                    mins = it_min_s(mins, r); maxs = it_max_s(maxs, r);
                    minu = it_min_u(minu, r); maxu = it_max_u(maxu, r);
                    band &= r; bor |= r; bxor ^= r;
                    all = all && s[6][l] == s[6][0];
                }
                for (int l = 0; l < 32; ++l) {
                    uint32_t any = 0;
                    for (int k = 0; k < 32; ++k) any |= (uint32_t)(s[5][k] == s[5][l]) << k;
                    out(l, IW_BALLOT) = ballot;
                    out(l, IW_ADD) = add;
                    out(l, IW_MIN_S) = mins; out(l, IW_MAX_S) = maxs;
                    out(l, IW_MIN_U) = minu; out(l, IW_MAX_U) = maxu;
                    out(l, IW_AND) = band; out(l, IW_OR) = bor; out(l, IW_XOR) = bxor;
                    out(l, IW_MATCH_ANY) = any;
                    out(l, IW_MATCH_ALL) = all ? ~0u : 0u;
                    out(l, IW_MATCH_ALL_P) = all;
                }
            }
        }
    }
}

// table: it_table_bytes(fmt) bytes, copied verbatim to the device; check: kCtThreads comparison values; words
// (optional): [thread][kItWords[fmt]] reference results.
inline void it_build_tile(uint32_t seed, int fmt, int tile, uint32_t* table, uint32_t* check,
                          std::vector<uint32_t>* words = nullptr) {
    std::vector<uint32_t> own;
    std::vector<uint32_t>& w = words ? *words : own;
    w.assign((size_t)kCtThreads * kItWords[fmt], 0);
    it_operands(seed, fmt, tile, table);
    it_results(fmt, table, w.data());
    for (int t = 0; t < kCtThreads; ++t) check[t] = it_fold(&w[(size_t)t * kItWords[fmt]], kItWords[fmt]);
}

}  // namespace b2dp
