// fp_test_math.hpp -- host-side arithmetic of the on-demand FP32/FP64 self-test (b2dp_fp_test, fp_selftest.cuh).
//
// Pure C++ (no CUDA), so the CPU tests compile it as it is (tests/native/fp_test_math_test.cpp) and compare it with the
// exact restatement in tests/fp_test_oracle.py:
//   - ft_fma_operands:  seed, format, tile  ->  every thread's 8 x and 16 (a, b) operands, crafted classes included
//   - ft_dmma_operands: seed, tile          ->  every warp's integer A and B matrices and the tile's two scale exponents
//   - ft_fma_results / ft_dmma_results: the reference results, in the kernel's per-thread word order
//   - ft_fold:          the per-thread comparison value
//   - ft_build_tile:    the operand table a launch reads verbatim and the check values
// The per-CTA record (CtRecord), its completeness rule and the verdict are the tensor-core test's
// (compute_test_math.hpp): the kernel keeps that test's round / tile / repetition structure.
//
// Why the host can predict the device's result bit for bit:
//   - FP32 / FP64 FMA: IEEE 754 defines fma(x, a, b) = RN(x * a + b), one rounding to nearest-even of the exact value,
//     subnormals and signed zeros included; std::fmaf / std::fma compute exactly that on the host.  (Never x * a + b:
//     that rounds twice, or once if the compiler contracts it.)
//   - DMMA: every operand is an integer times a power of two shared by the tile's A (or B), and every partial sum of a
//     result element is an integer below 2^53 in magnitude times 2^(ea + eb), which binary64 holds exactly whatever the
//     order of accumulation.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "compute_test_math.hpp"  // ct_mix, ct_hash, ct_uniform, CtRecord, kCtThreads, kCtTiles, kCtReps

namespace b2dp {

enum FtFormat { FT_FP32 = 0, FT_FP64 = 1, FT_DMMA = 2 };
constexpr int kFtFormats = 3;
static_assert(kFtFormats == kCtFormats, "the verdict and the result struct are shared with the tensor-core test");

// ---- FFMA / DFMA ----------------------------------------------------------------------------------------------------
// Per tile each thread holds kFtX values x_i and kFtAB pairs (a_k, b_k) in registers and computes every
// r = fma(x_i, a_k, b_k): kFtResults independent FMAs per repetition, result j = k * kFtX + i.
constexpr int kFtX = 8, kFtAB = 16;
constexpr int kFtResults = kFtX * kFtAB;      // 128
constexpr int kFtSlots = kFtX + 2 * kFtAB;    // operand slots per thread: x_0..7, a_0..15, b_0..15
// Crafted classes: thread t's pair k = (2c + t) % 16 is built so that fma(x_{ft_class_x(c)}, a_k, b_k) falls in class c.
enum FtClass {
    FT_TIE_AWAY = 0,   // exact value halfway between two neighbours, rounded to the one of larger magnitude (even)
    FT_TIE_TOWARD,     // halfway, rounded to the one of smaller magnitude (even)
    FT_CANCEL,         // b = -RN(x * a): the result is the product's rounding error (>= 24 / 53 bits cancelled)
    FT_SUBNORMAL,      // x * a and b both below the normal range, same sign: a subnormal, nonzero result
    FT_ZERO_POS,       // x * a = -b exactly: +0
    FT_ZERO_NEG,       // x * a = -0 and b = -0: -0
    FT_STICKY,         // |b| > 2^M |x * a| and |x * a| in (ulp(b) / 2, ulp(b)): only the sticky bit says "round up"
    FT_SUB_OPERAND,    // a subnormal (top stored bit set), b normal in [2^EMIN, 2^(EMIN + 4)): every x_i * a moves the
                       // result off b, so a unit that reads a subnormal multiplicand as 0 gets all 8 results wrong
    kFtClasses
};
inline int ft_class_slot(int c, int t) { return (2 * c + t) % kFtAB; }
inline int ft_class_x(int c) {
    // x_0 has an odd significand, x_1 an even one that is not a power of two, x_2 the exponent -8, x_3 is random
    static const int x[kFtClasses] = {0, 1, 0, 2, 1, 3, 0, 3};
    return x[c];
}

// Binary formats.  M = stored mantissa bits, BIAS = exponent bias, EMIN = smallest normal exponent.
struct FtBin {
    int width, M, BIAS, EMIN;
    int x_exp, a_exp, b_spread;  // random x exponents in [-x_exp, x_exp], a in [-a_exp, a_exp], b = e(a) +- b_spread
};
constexpr FtBin kFtBin32 = {32, 23, 127, -126, 16, 40, 28};
constexpr FtBin kFtBin64 = {64, 52, 1023, -1022, 16, 300, 60};
inline const FtBin& ft_bin(int fmt) { return fmt == FT_FP32 ? kFtBin32 : kFtBin64; }
// every random or crafted operand stays normal (the subnormal class's b and the subnormal-operand class's a excepted)
// and every product below overflow
static_assert(kFtBin32.x_exp + kFtBin32.a_exp + kFtBin32.M + 2 < 127 &&
              kFtBin32.a_exp + kFtBin32.b_spread < 127 && -(kFtBin32.x_exp + kFtBin32.a_exp + kFtBin32.M + 1) > -126,
              "FP32 operand exponents stay in the normal range");
static_assert(kFtBin64.x_exp + kFtBin64.a_exp + kFtBin64.M + 2 < 1023 &&
              kFtBin64.a_exp + kFtBin64.b_spread < 1023 && -(kFtBin64.x_exp + kFtBin64.a_exp + kFtBin64.M + 1) > -1022,
              "FP64 operand exponents stay in the normal range");
constexpr int kFtSubnormalXExp = -8;  // x_2's exponent; the subnormal class's a has exponent EMIN + 3
static_assert(kFtSubnormalXExp + 3 + 2 <= 0 && kFtSubnormalXExp + 3 == -5,
              "the subnormal class's product x_2 * a lies in [2^(EMIN - 5), 2^(EMIN - 3)), below the normal range");

// ---- DMMA -----------------------------------------------------------------------------------------------------------
// mma.sync m16n8k16 .f64: per warp kFtDmmaSteps operand pairs (A_s 16 x 16, B_s 16 x 8, K x N) in registers and
// kFtDmmaSets independent accumulators; set c accumulates A_s * B_{(s + c) % steps} over s = 0..steps-1, so each of its
// 16 x 8 results sums K = 16 * steps products.
constexpr int kFtMmaM = 16, kFtMmaN = 8, kFtMmaK = 16;
constexpr int kFtDmmaSteps = 4, kFtDmmaSets = 4;
constexpr int kFtDmmaK = kFtMmaK * kFtDmmaSteps;  // 64
constexpr int kFtDmmaA = 8, kFtDmmaB = 4, kFtDmmaD = 4;                          // f64 registers per thread per mma
constexpr int kFtDmmaSlots = kFtDmmaSteps * (kFtDmmaA + kFtDmmaB);              // 48 operand slots per thread
constexpr long long kFtDmmaMax = 11863283;                                        // integers in [-max, max]
constexpr int kFtDmmaScaleExp = 480;  // a tile's A and B are scaled by 2^ea, 2^eb with |ea|, |eb| <= 480
static_assert(kFtDmmaK * kFtDmmaMax * kFtDmmaMax < (1ll << 53),
              "every DMMA partial sum is an integer below 2^53: binary64 holds it exactly");
static_assert((kFtDmmaK - 8) * kFtDmmaMax * kFtDmmaMax > (1ll << 52), "the extreme rows' sums exceed 2^52");
static_assert(2 * kFtDmmaScaleExp + 53 < 1024 && -2 * kFtDmmaScaleExp > -1022,
              "a scaled DMMA result stays a normal binary64 number");

// 32-bit words each thread folds per repetition (and DUMP writes per tile)
constexpr int kFtWords[kFtFormats] = {kFtResults, 2 * kFtResults, 2 * kFtDmmaSets * kFtDmmaD};
constexpr int kFtMaxWords = 2 * kFtResults;
inline int ft_slots(int fmt) { return fmt == FT_DMMA ? kFtDmmaSlots : kFtSlots; }
inline int ft_value_bytes(int fmt) { return fmt == FT_FP32 ? 4 : 8; }
// operand table of one tile: [slot][thread] values, so a warp's loads of one slot are coalesced
inline uint32_t ft_table_bytes(int fmt) { return (uint32_t)(ft_slots(fmt) * kCtThreads * ft_value_bytes(fmt)); }
// Multiply-adds of one comparison (one repetition of one tile by one CTA); 2 * this = its FLOPs.
inline double ft_macs_per_tile(int fmt) {
    return fmt == FT_DMMA ? (double)kCtThreads / 32 * kFtDmmaSteps * kFtDmmaSets * kFtMmaM * kFtMmaN * kFtMmaK
                          : (double)kCtThreads * kFtResults;
}

// ---- generator ------------------------------------------------------------------------------------------------------
inline uint32_t ft_stream_key(uint32_t seed, int fmt, int tile, int op) {
    return ct_mix(seed ^ (uint32_t)(((fmt * 16 + tile) * 4 + op) + 1) * 0x85EBCA77u);
}
// draw j of slot s of thread t
inline uint32_t ft_draw(uint32_t key, int t, int s, int j) { return ct_hash(key, (uint32_t)((t * 64 + s) * 4 + j)); }
inline uint64_t ft_draw64(uint32_t key, int t, int s) {
    return (uint64_t)ft_draw(key, t, s, 0) << 32 | ft_draw(key, t, s, 1);
}

// bits of sign * 1.mant * 2^e (normal), or sign * 0.mant * 2^EMIN with e = EMIN - 1 (subnormal or zero)
inline uint64_t ft_make(const FtBin& f, uint32_t sign, int e, uint64_t mant) {
    return (uint64_t)sign << (f.width - 1) | (uint64_t)(e + f.BIAS) << f.M | (mant & ((1ull << f.M) - 1));
}
inline int ft_exp(const FtBin& f, uint64_t bits) { return (int)((bits >> f.M) & ((1u << (f.width - f.M - 1)) - 1)) - f.BIAS; }
inline uint32_t ft_sign(const FtBin& f, uint64_t bits) { return (uint32_t)(bits >> (f.width - 1)) & 1u; }

inline float ft_f32(uint64_t b) { float x; uint32_t u = (uint32_t)b; std::memcpy(&x, &u, 4); return x; }
inline double ft_f64(uint64_t b) { double x; std::memcpy(&x, &b, 8); return x; }
inline uint64_t ft_bits(float x) { uint32_t u; std::memcpy(&u, &x, 4); return u; }
inline uint64_t ft_bits(double x) { uint64_t u; std::memcpy(&u, &x, 8); return u; }

// RN(x * a) and RN(x * a + b) in the format, on bits (std::fmaf / std::fma: one rounding, as IEEE 754 defines it)
inline uint64_t ft_mul(int fmt, uint64_t x, uint64_t a) {
    if (fmt == FT_FP32) return ft_bits((float)((double)ft_f32(x) * (double)ft_f32(a)));  // exact in double, one rounding
    return ft_bits(ft_f64(x) * ft_f64(a));
}
inline uint64_t ft_fma(int fmt, uint64_t x, uint64_t a, uint64_t b) {
    if (fmt == FT_FP32) return ft_bits(std::fmaf(ft_f32(x), ft_f32(a), ft_f32(b)));
    return ft_bits(std::fma(ft_f64(x), ft_f64(a), ft_f64(b)));
}

// Operands of one thread: x[8], a[16], b[16] as bits (FP32 in the low 32 bits).
struct FtFmaOperands {
    uint64_t x[kFtX], a[kFtAB], b[kFtAB];
};

inline void ft_fma_thread(uint32_t seed, int fmt, int tile, int t, FtFmaOperands& o) {
    const FtBin& f = ft_bin(fmt);
    const uint32_t key = ft_stream_key(seed, fmt, tile, 0);
    const uint64_t mmask = (1ull << f.M) - 1;
    for (int i = 0; i < kFtX; ++i) {
        const uint64_t r = ft_draw64(key, t, i);
        uint64_t mant = r & mmask;
        int e = ct_uniform(ft_draw(key, t, i, 2), -f.x_exp, f.x_exp);
        if (i == 0) mant |= 1;                // odd significand
        if (i == 1) mant = (mant & ~1ull) | 2;  // even, and not a power of two
        if (i == 2) e = kFtSubnormalXExp;
        o.x[i] = ft_make(f, (uint32_t)(r >> 63), e, mant);
    }
    for (int k = 0; k < kFtAB; ++k) {  // random pairs: b's exponent near a's, so x * a and b overlap in many ways
        const uint64_t ra = ft_draw64(key, t, kFtX + k), rb = ft_draw64(key, t, kFtX + kFtAB + k);
        const int ea = ct_uniform(ft_draw(key, t, kFtX + k, 2), -f.a_exp, f.a_exp);
        const int eb = ea + ct_uniform(ft_draw(key, t, kFtX + kFtAB + k, 2), -f.b_spread, f.b_spread);
        o.a[k] = ft_make(f, (uint32_t)(ra >> 63), ea, ra & mmask);
        o.b[k] = ft_make(f, (uint32_t)(rb >> 63), eb, rb & mmask);
    }
    for (int c = 0; c < kFtClasses; ++c) {
        const int k = ft_class_slot(c, t);
        const uint64_t x = o.x[ft_class_x(c)];
        const int ex = ft_exp(f, x);
        const uint32_t sa = (uint32_t)(o.a[k] >> (f.width - 1)) & 1u, sb = (uint32_t)(o.b[k] >> (f.width - 1)) & 1u;
        const int j = ft_exp(f, o.a[k]);             // a's random exponent
        const uint64_t pow2 = ft_make(f, sa, j, 0);  // +-2^j: x * a is exact
        const int q = ex + j;                        // exponent of x * 2^j
        const uint32_t sp = ft_sign(f, x) ^ sa;      // sign of x * a
        switch (c) {
            case FT_TIE_AWAY:    // b = ulp(x * a) / 2 with the product's sign: x_0's odd significand rounds up to even,
            case FT_TIE_TOWARD:  // x_1's even one stays
                o.a[k] = pow2;
                o.b[k] = ft_make(f, sp, q - f.M - 1, 0);
                break;
            case FT_CANCEL:  // a with an odd significand: the product of two odd significands needs 2M + 1 bits
                o.a[k] |= 1;
                o.b[k] = ft_mul(fmt, x, o.a[k]) ^ (1ull << (f.width - 1));
                break;
            case FT_SUBNORMAL:  // x_2 * a in [2^(EMIN - 5), 2^(EMIN - 3)); b subnormal below 2^(EMIN - 5), same sign
                o.a[k] = ft_make(f, sa, f.EMIN + 3, o.a[k]);
                o.b[k] = ft_make(f, sp, f.EMIN - 1, o.b[k] & ((1ull << (f.M - 5)) - 1));
                break;
            case FT_ZERO_POS:
                o.a[k] = pow2;
                o.b[k] = ft_mul(fmt, x, pow2) ^ (1ull << (f.width - 1));
                break;
            case FT_ZERO_NEG:  // x * a = -0, b = -0
                o.a[k] = (uint64_t)(ft_sign(f, x) ^ 1u) << (f.width - 1);
                o.b[k] = 1ull << (f.width - 1);
                break;
            case FT_STICKY:  // ulp(b) = 2^(q + 1); b's significand even, so a lost sticky bit would round to b
                o.a[k] = pow2;
                o.b[k] = ft_make(f, sb, q + f.M + 1, o.b[k] & ~1ull);
                break;
            case FT_SUB_OPERAND:  // |x_i * a| >= 2^(EMIN - 17) > ulp(b) / 2 = 2^(e(b) - M - 1) for every x_i
                o.a[k] = ft_make(f, sa, f.EMIN - 1, o.a[k] | 1ull << (f.M - 1));
                o.b[k] = ft_make(f, sb, ct_uniform(ft_draw(key, t, kFtX + kFtAB + k, 3), f.EMIN, f.EMIN + 3), o.b[k]);
                break;
        }
    }
}

// word w of the 2 * kFtResults (FP64) or kFtResults (FP32) words of the thread's results: result j's bits (FP32), or
// result j's low word at 2j and high word at 2j + 1 (FP64)
inline void ft_fma_results(int fmt, const FtFmaOperands& o, uint32_t* words) {
    for (int k = 0; k < kFtAB; ++k)
        for (int i = 0; i < kFtX; ++i) {
            const int j = k * kFtX + i;
            const uint64_t r = ft_fma(fmt, o.x[i], o.a[k], o.b[k]);
            if (fmt == FT_FP32) {
                words[j] = (uint32_t)r;
            } else {
                words[2 * j] = (uint32_t)r;
                words[2 * j + 1] = (uint32_t)(r >> 32);
            }
        }
}

// ---- DMMA operands, fragments and the exact product -------------------------------------------------------------------
// Integer matrices of warp w, step s: A (16 x 16, row-major M x K) and B (16 x 8, row-major K x N).  Random in
// [-max, max], except in warp tile % 4 (so every SM sub-partition meets them over a round): row 0 of every A_s and every
// B_s element with k != n hold -max, so row 0 of every result sums at least 56 of its 64 products max^2 (above 2^52).
inline int ft_dmma_scale_exp(uint32_t seed, int tile, int op) {
    return ct_uniform(ct_hash(ft_stream_key(seed, FT_DMMA, tile, 2), (uint32_t)op), -kFtDmmaScaleExp, kFtDmmaScaleExp);
}
inline long long ft_dmma_value(uint32_t seed, int tile, int op, int w, int s, int r, int c) {
    const bool extreme = w == tile % 4 && (op == 0 ? r == 0 : r != c);
    if (extreme) return -kFtDmmaMax;
    const uint32_t key = ft_stream_key(seed, FT_DMMA, tile, op);
    const int cols = op == 0 ? kFtMmaK : kFtMmaN;
    const uint32_t h = ct_hash(key, (uint32_t)(((w * kFtDmmaSteps + s) * kFtMmaK + r) * cols + c));
    return -kFtDmmaMax + (long long)(((uint64_t)h * (uint64_t)(2 * kFtDmmaMax + 1)) >> 32);
}
// Fragments of mma.sync.aligned.m16n8k16.row.col.f64 (PTX ISA, "Matrix fragments for mma.m16n8k16" .f64), lane l,
// groupID g = l / 4, threadID_in_group q = l % 4:
//   A register i (0..7): row g + 8 (i % 2), col q + 4 (i / 2);  B register i (0..3): k q + 4 i, n g;
//   D register i (0..3): row g + 8 (i / 2), col 2 q + i % 2.
inline int ft_a_row(int l, int i) { return l / 4 + 8 * (i % 2); }
inline int ft_a_col(int l, int i) { return l % 4 + 4 * (i / 2); }
inline int ft_b_k(int l, int i) { return l % 4 + 4 * i; }
inline int ft_b_n(int l, int /*i*/) { return l / 4; }
inline int ft_d_row(int l, int i) { return l / 4 + 8 * (i / 2); }
inline int ft_d_col(int l, int i) { return 2 * (l % 4) + i % 2; }

// Exact result of set c of warp w: D[m][n] = sum_s sum_kk A_s[m][kk] B_{(s + c) % steps}[kk][n], as an int64.
inline long long ft_dmma_exact(uint32_t seed, int tile, int w, int c, int m, int n) {
    long long sum = 0;
    for (int s = 0; s < kFtDmmaSteps; ++s)
        for (int kk = 0; kk < kFtMmaK; ++kk)
            sum += ft_dmma_value(seed, tile, 0, w, s, m, kk) *
                   ft_dmma_value(seed, tile, 1, w, (s + c) % kFtDmmaSteps, kk, n);
    return sum;
}

// ---- the fold and the tile ------------------------------------------------------------------------------------------
// sum_j (2j + 1) * w_j mod 2^32 over the thread's words.  Flipping bit b of one result changes one word (FP32, DMMA and
// FP64 alike: a binary64 result is two words) by +-2^b, so the sum by +-(2j + 1) * 2^b mod 2^32; an odd number times 2^b
// with b < 32 is never a multiple of 2^32, so no single flipped bit of any one result leaves the value unchanged.
inline uint32_t ft_fold(const uint32_t* w, int n) {
    uint32_t h = 0;
    for (int j = 0; j < n; ++j) h += (2u * (uint32_t)j + 1u) * w[j];
    return h;
}

struct FtTile {
    std::vector<uint8_t> table;     // ft_table_bytes(fmt): [slot][thread] operand values, copied verbatim to the device
    uint32_t check[kCtThreads];     // per-thread comparison values
    std::vector<uint32_t> words;    // [thread][kFtWords[fmt]] the reference results in the kernel's order
};

inline void ft_build_tile(uint32_t seed, int fmt, int tile, FtTile& out) {
    const int W = kFtWords[fmt], vb = ft_value_bytes(fmt);
    out.table.assign(ft_table_bytes(fmt), 0);
    out.words.assign((size_t)kCtThreads * W, 0);
    auto put = [&](int slot, int t, uint64_t bits) { std::memcpy(&out.table[((size_t)slot * kCtThreads + t) * vb], &bits, vb); };
    if (fmt != FT_DMMA) {
        FtFmaOperands o;
        for (int t = 0; t < kCtThreads; ++t) {
            ft_fma_thread(seed, fmt, tile, t, o);
            for (int i = 0; i < kFtX; ++i) put(i, t, o.x[i]);
            for (int k = 0; k < kFtAB; ++k) {
                put(kFtX + k, t, o.a[k]);
                put(kFtX + kFtAB + k, t, o.b[k]);
            }
            ft_fma_results(fmt, o, &out.words[(size_t)t * W]);
        }
    } else {
        const int ea = ft_dmma_scale_exp(seed, tile, 0), eb = ft_dmma_scale_exp(seed, tile, 1);
        for (int t = 0; t < kCtThreads; ++t) {
            const int w = t / 32, l = t % 32;
            for (int s = 0; s < kFtDmmaSteps; ++s) {
                for (int i = 0; i < kFtDmmaA; ++i)
                    put(s * kFtDmmaA + i, t,
                        ft_bits(std::ldexp((double)ft_dmma_value(seed, tile, 0, w, s, ft_a_row(l, i), ft_a_col(l, i)), ea)));
                for (int i = 0; i < kFtDmmaB; ++i)
                    put(kFtDmmaSteps * kFtDmmaA + s * kFtDmmaB + i, t,
                        ft_bits(std::ldexp((double)ft_dmma_value(seed, tile, 1, w, s, ft_b_k(l, i), ft_b_n(l, i)), eb)));
            }
            for (int c = 0; c < kFtDmmaSets; ++c)
                for (int i = 0; i < kFtDmmaD; ++i) {
                    const long long e = ft_dmma_exact(seed, tile, w, c, ft_d_row(l, i), ft_d_col(l, i));
                    const uint64_t r = e == 0 ? 0ull : ft_bits(std::ldexp((double)e, ea + eb));  // an exact zero is +0
                    uint32_t* dst = &out.words[(size_t)t * W + 2 * (c * kFtDmmaD + i)];
                    dst[0] = (uint32_t)r;
                    dst[1] = (uint32_t)(r >> 32);
                }
        }
    }
    for (int t = 0; t < kCtThreads; ++t) out.check[t] = ft_fold(&out.words[(size_t)t * W], W);
}

}  // namespace b2dp
