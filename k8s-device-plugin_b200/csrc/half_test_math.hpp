// half_test_math.hpp -- host-side arithmetic of the on-demand half-precision and conversion self-test (b2dp_half_test,
// half_selftest.cuh).
//
// Pure C++ (no CUDA), so the CPU tests compile it as it is (tests/native/half_test_math_test.cpp) and compare it with the
// independent restatement in tests/half_test_oracle.py:
//   - hp_operands:   seed, format, tile -> the operand table ([slot][thread] words), crafted classes included
//   - hp_results:    the reference result words of every thread, in the kernel's word order
//   - it_fold:       the per-thread comparison value (the integer test's fold, int_test_math.hpp)
//   - hp_build_tile: the table a launch reads verbatim and the check values
// The per-CTA record (CtRecord), its completeness rule and the verdict are the tensor-core test's.
//
// Why the host can predict the device bit for bit: every op under test is IEEE 754 or PTX-defined arithmetic with one
// rounding of the exact result.  Every result below is computed exactly (integers up to 128 bits times a power of two)
// and rounded once (hp_round); nothing goes through a host float operation.  (half)fmaf(a, b, c) would round twice, and
// the double-rounding class exists to catch a unit, or a reference, that does.  Infinite and NaN operands reach only the
// ops whose result bits the PTX ISA defines: min / max (canonical NaN 0x7FFF), .relu (NaN -> canonical NaN), .sat (NaN
// -> +0), .satfinite (NaN -> NaN, +-inf -> +-max finite) and float-to-integer conversion (NaN -> 0, saturating).
//
// Layout.  A thread's operands are kHpSets[fmt] sets of kHpSetSlots[fmt] words; slot = set * kHpSetSlots + k.  Every op
// of the format runs on every set, and set s's result words are s * kHpSetWords[fmt] + j, in the order of the HpF16Word
// / HpBf16Word / HpCvtWord enums.  The first kHpCrafted[fmt] sets are crafted, the rest random.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "compute_test_math.hpp"  // ct_mix, ct_hash, CtRecord, kCtThreads, kCtTiles, kCtReps
#include "int_test_math.hpp"      // it_fold

namespace b2dp {

enum HpFormat { HP_F16 = 0, HP_BF16 = 1, HP_CVT = 2 };
constexpr int kHpFormats = 3;
static_assert(kHpFormats == kCtFormats, "the verdict and the result struct are shared with the tensor-core test");

constexpr int kHpSets[kHpFormats] = {12, 12, 9};
constexpr int kHpCrafted[kHpFormats] = {6, 6, 8};
constexpr int kHpSetSlots[kHpFormats] = {6, 6, 13};
constexpr int kHpSetWords[kHpFormats] = {12, 9, 58};
constexpr int kHpSlots[kHpFormats] = {12 * 6, 12 * 6, 9 * 13};
constexpr int kHpWords[kHpFormats] = {12 * 12, 12 * 9, 9 * 58};
constexpr int kHpMaxWords = 9 * 58;

// HP_F16 / HP_BF16: slots a, b, c (finite: the rounding ops) and x, y, z (may be +-inf or NaN: the ops that define
// their result bits for them).  Every word holds two independent 16-bit lanes.
enum HpHalfSlot { HS_A = 0, HS_B, HS_C, HS_X, HS_Y, HS_Z };
enum HpF16Word {
    HF_FMA = 0,      // fma.rn.f16x2 a, b, c
    HF_FMA_RELU,     // fma.rn.relu.f16x2 x, y, z
    HF_FMA_SAT,      // fma.rn.sat.f16x2 x, y, z
    HF_FMA_FTZ,      // fma.rn.ftz.f16x2 a, b, c
    HF_ADD,          // add.rn.f16x2 a, b
    HF_SUB,          // sub.rn.f16x2 a, b
    HF_MUL,          // mul.rn.f16x2 a, b
    HF_MIN,          // min.f16x2 x, y
    HF_MAX,
    HF_MIN_NAN,      // min.NaN.f16x2 x, y
    HF_MAX_NAN,
    HF_MIN_XORSIGN,  // min.xorsign.abs.f16x2 a, b
};
enum HpBf16Word {
    HB_FMA = 0,      // fma.rn.bf16x2 a, b, c
    HB_FMA_RELU,     // fma.rn.relu.bf16x2 x, y, z
    HB_ADD,          // add.rn.bf16x2 a, b
    HB_SUB,
    HB_MUL,
    HB_MIN,          // min.bf16x2 x, y
    HB_MAX,
    HB_MIN_NAN,
    HB_MAX_NAN,
};
// HP_CVT slots: X, Y (finite f32), P, Q (f32, +-inf and NaN too), F (f32 for float-to-int), H (f16x2, +-inf too),
// E4 / E5 (an e4m3x2 / e5m2x2 pair in the low 16 bits, no NaN), I (s32), D (f64: lo, hi), L (64-bit integer: lo, hi).
enum HpCvtSlot { HC_X = 0, HC_Y, HC_P, HC_Q, HC_F, HC_H, HC_E4, HC_E5, HC_I, HC_DLO, HC_DHI, HC_LLO, HC_LHI };
enum HpCvtWord {
    HC_F16X2_RN = 0,   // cvt.rn.f16x2.f32 X, Y (X to the upper half)
    HC_F16X2_RZ,       // cvt.rz.f16x2.f32 X, Y
    HC_F16X2_RELU,     // cvt.rn.relu.f16x2.f32 P, Q
    HC_F16X2_SATF,     // cvt.rn.satfinite.f16x2.f32 P, Q
    HC_BF16X2_RN,      // cvt.rn.bf16x2.f32 X, Y
    HC_BF16X2_RZ,
    HC_BF16X2_RELU,    // P, Q
    HC_BF16X2_SATF,
    HC_E4M3_F32,       // cvt.rn.satfinite.e4m3x2.f32 P, Q (P to the upper byte)
    HC_E5M2_F32,       // cvt.rn.satfinite.e5m2x2.f32 X, Y
    HC_E4M3_F16,       // cvt.rn.satfinite.e4m3x2.f16x2 H
    HC_E5M2_F16,       // cvt.rn.satfinite.e5m2x2.f16x2 H
    HC_F16_E4M3,       // cvt.rn.f16x2.e4m3x2 E4
    HC_F16_E5M2,       // cvt.rn.f16x2.e5m2x2 E5
    HC_TF32,           // cvt.rn.tf32.f32 X
    HC_F16_RM,         // cvt.rm.f16.f32 X (zero-extended)
    HC_F16_RP,
    HC_BF16_RM,
    HC_BF16_RP,
    HC_S32 = 19,       // cvt.{rni,rzi,rmi,rpi}.s32.f32 F: 4 words
    HC_U32 = 23,       // cvt.{rni,rzi,rmi,rpi}.u32.f32 F: 4 words
    HC_S64 = 27,       // cvt.{rni,rzi,rmi,rpi}.s64.f64 D: 4 x (lo, hi)
    HC_I2F_S32 = 35,   // cvt.{rn,rz,rm,rp}.f32.s32 I: 4 words
    HC_I2F_U64 = 39,   // cvt.{rn,rz,rm,rp}.f32.u64 L: 4 words
    HC_I2F_S64 = 43,   // cvt.{rn,rz,rm,rp}.f64.s64 L: 4 x (lo, hi)
    HC_F32_F64 = 51,   // cvt.{rn,rz,rm,rp}.f32.f64 D: 4 words
    HC_FRND_F32 = 55,  // cvt.rni.f32.f32 X
    HC_FRND_F64 = 56,  // cvt.rmi.f64.f64 D: lo, hi
};
static_assert(HC_FRND_F64 + 2 == 58, "kHpSetWords[HP_CVT]");

// operand table of one tile: [slot][thread] words, so a warp's loads of one slot are coalesced
inline uint32_t hp_table_bytes(int fmt) { return (uint32_t)(kHpSlots[fmt] * kCtThreads * 4); }
// Result words of one comparison (one repetition of one tile by one CTA); the rate counts every folded word.
inline double hp_ops_per_tile(int fmt) { return (double)kCtThreads * kHpWords[fmt]; }

// ---- exact values and one rounding ----------------------------------------------------------------------------------
using hp_u128 = unsigned __int128;
enum HpMode { HP_RN = 0, HP_RZ = 1, HP_RM = 2, HP_RP = 3 };  // the order of .rn/.rz/.rm/.rp and .rni/.rzi/.rmi/.rpi
struct HpFmt { int ebits, mbits; bool has_inf; };  // has_inf = false: e4m3 (S.1111.111 is NaN, no infinity)
constexpr HpFmt kHpF16{5, 10, true}, kHpBf16{8, 7, true}, kHpF32{8, 23, true}, kHpF64{11, 52, true},
    kHpTf32{8, 10, true}, kHpE4m3{4, 3, false}, kHpE5m2{5, 2, true};
// (-1)^neg * m * 2^e, exactly; m < 2^120.  cls: 0 finite (zero included), 1 infinite, 2 NaN.
struct HpNum { bool neg; hp_u128 m; int e; int cls; };

inline int hp_msb(hp_u128 m) { int k = -1; while (m) { m >>= 1; ++k; } return k; }
inline uint64_t hp_sign_bit(HpFmt f) { return 1ull << (f.ebits + f.mbits); }
inline uint64_t hp_max_finite(HpFmt f) {
    const uint64_t top = (1ull << f.ebits) - 1;
    return f.has_inf ? (top - 1) << f.mbits | ((1ull << f.mbits) - 1) : top << f.mbits | ((1ull << f.mbits) - 2);
}
inline uint64_t hp_inf(HpFmt f) { return ((1ull << f.ebits) - 1) << f.mbits; }

inline HpNum hp_decode(uint64_t bits, HpFmt f) {
    const int bias = (1 << (f.ebits - 1)) - 1;
    const uint64_t mant = bits & ((1ull << f.mbits) - 1);
    const int ef = (int)(bits >> f.mbits & ((1ull << f.ebits) - 1));
    HpNum x{(bits & hp_sign_bit(f)) != 0, 0, 0, 0};
    if (ef == (1 << f.ebits) - 1 && (f.has_inf || mant == (1ull << f.mbits) - 1)) {
        x.cls = f.has_inf && mant == 0 ? 1 : 2;
        return x;
    }
    x.m = ef ? mant | 1ull << f.mbits : mant;
    x.e = (ef ? ef : 1) - bias - f.mbits;
    return x;
}

// The one rounding: the finite value x to format f under mode (ties to even for HP_RN).  The result is the nearest
// value in the direction the mode names with an unbounded exponent; a result beyond the largest finite value overflows
// to infinity (RN, and RM / RP away from zero) or to the largest finite value (RZ, RM / RP toward zero, .satfinite).
inline uint64_t hp_round(const HpNum& x, HpFmt f, int mode, bool satfinite = false) {
    const uint64_t sign = x.neg ? hp_sign_bit(f) : 0;
    if (x.m == 0) return sign;
    const int bias = (1 << (f.ebits - 1)) - 1, emin = 1 - bias;
    const int E = hp_msb(x.m) + x.e;
    int q = (E > emin ? E : emin) - f.mbits;  // the quantum's exponent
    hp_u128 n;
    int rest;  // the discarded part against half a quantum: -2 none, -1 below, 0 exactly half, 1 above
    if (x.e >= q) {
        n = x.m << (x.e - q);
        rest = -2;
    } else {
        const int s = q - x.e;
        if (s > hp_msb(x.m) + 1) {
            n = 0;
            rest = -1;
        } else {
            n = s >= 128 ? 0 : x.m >> s;
            const hp_u128 r = x.m - (n << s), half = (hp_u128)1 << (s - 1);
            rest = r == 0 ? -2 : r < half ? -1 : r == half ? 0 : 1;
        }
    }
    bool up = false;
    if (rest != -2) {
        if (mode == HP_RN) up = rest > 0 || (rest == 0 && (n & 1));
        else if (mode == HP_RM) up = x.neg;
        else if (mode == HP_RP) up = !x.neg;
    }
    n += up;
    if (n == 0) return sign;
    if (n >> (f.mbits + 1)) { n >>= 1; ++q; }
    uint64_t mag;
    if (n >> f.mbits == 0) mag = (uint64_t)n;  // subnormal (q is the least exponent)
    else {
        const long long ef = (long long)q + f.mbits + bias;
        mag = ef > (long long)((1ull << f.ebits) - 1) ? ~0ull : (uint64_t)ef << f.mbits | ((uint64_t)n & ((1ull << f.mbits) - 1));
    }
    if (mag > hp_max_finite(f)) {
        const bool to_max = satfinite || mode == HP_RZ || (mode == HP_RM && !x.neg) || (mode == HP_RP && x.neg);
        mag = to_max || !f.has_inf ? hp_max_finite(f) : hp_inf(f);
    }
    return sign | mag;
}

// a * b + c, exactly, for finite operands with m < 2^32 (the 16-bit formats).  When the exponents lie more than 80 bits
// apart the smaller term is replaced by one unit 80 bits below the larger: both lie strictly inside the same interval
// between points a rounding to at most 24 bits can land on, so they round alike in every mode.
inline HpNum hp_fma_exact(const HpNum& a, const HpNum& b, const HpNum& c) {
    HpNum p{a.neg != b.neg, a.m * b.m, a.e + b.e, 0};
    if (p.m == 0 && c.m == 0) return HpNum{p.neg && c.neg, 0, 0, 0};  // RN: -0 only for -0 + -0
    if (p.m == 0) return c;
    if (c.m == 0) return p;
    HpNum hi = p.e >= c.e ? p : c, lo = p.e >= c.e ? c : p;
    int e0;
    hp_u128 mh, ml;
    if (hi.e - lo.e > 80) { mh = hi.m << 80; ml = 1; e0 = hi.e - 80; }
    else { mh = hi.m << (hi.e - lo.e); ml = lo.m; e0 = lo.e; }
    if (hi.neg == lo.neg) return HpNum{hi.neg, mh + ml, e0, 0};
    if (mh == ml) return HpNum{false, 0, 0, 0};  // exact cancellation: +0 under RN
    return mh > ml ? HpNum{hi.neg, mh - ml, e0, 0} : HpNum{lo.neg, ml - mh, e0, 0};
}

// ---- the ops, per the PTX ISA (one 16-bit lane) -------------------------------------------------------------------
constexpr uint32_t kHpCanonicalNaN = 0x7FFF;  // f16 and bf16
enum HpFmaMod { HP_PLAIN = 0, HP_RELU, HP_SAT, HP_FTZ };
inline bool hp_is_sub(uint32_t h, HpFmt f) { return (h >> f.mbits & ((1u << f.ebits) - 1)) == 0 && (h & ((1u << f.mbits) - 1)); }
inline uint32_t hp_ftz(uint32_t h, HpFmt f) { return hp_is_sub(h, f) ? h & (uint32_t)hp_sign_bit(f) : h; }

// fma.rn{.relu,.sat,.ftz} of one lane (f = kHpF16 or kHpBf16)
inline uint32_t hp_fma(uint32_t a, uint32_t b, uint32_t c, HpFmt f, int mod = HP_PLAIN) {
    if (mod == HP_FTZ) { a = hp_ftz(a, f); b = hp_ftz(b, f); c = hp_ftz(c, f); }
    const HpNum x = hp_decode(a, f), y = hp_decode(b, f), z = hp_decode(c, f);
    const uint32_t one = (uint32_t)((1u << (f.ebits - 1)) - 1) << f.mbits;
    uint32_t r = 0;
    bool nan = false;
    if (x.cls == 2 || y.cls == 2 || z.cls == 2) nan = true;
    else if (x.cls == 1 || y.cls == 1) {
        const bool pneg = x.neg != y.neg;
        if ((x.cls != 1 && x.m == 0) || (y.cls != 1 && y.m == 0) || (z.cls == 1 && z.neg != pneg)) nan = true;
        else r = (uint32_t)(hp_inf(f) | (pneg ? hp_sign_bit(f) : 0));
    } else if (z.cls == 1) r = c;
    else r = (uint32_t)hp_round(hp_fma_exact(x, y, z), f, HP_RN);
    if (mod == HP_RELU) return nan ? kHpCanonicalNaN : (r & hp_sign_bit(f)) ? 0u : r;
    if (mod == HP_SAT) {
        if (nan || (r & hp_sign_bit(f))) return 0u;
        return r > one ? one : r;
    }
    if (mod == HP_FTZ) return hp_ftz(r, f);
    return nan ? kHpCanonicalNaN : r;  // not reached with the tables: a, b, c are finite
}
inline uint32_t hp_add(uint32_t a, uint32_t b, HpFmt f) { return hp_fma(a, (uint32_t)((1u << (f.ebits - 1)) - 1) << f.mbits, b, f); }
inline uint32_t hp_sub(uint32_t a, uint32_t b, HpFmt f) { return hp_add(a, b ^ (uint32_t)hp_sign_bit(f), f); }
inline uint32_t hp_mul(uint32_t a, uint32_t b, HpFmt f) { return hp_fma(a, b, (uint32_t)hp_sign_bit(f), f); }  // + (-0)
// a < b for non-NaN lanes, -0 below +0
inline bool hp_less(uint32_t a, uint32_t b, HpFmt f) {
    const uint32_t s = (uint32_t)hp_sign_bit(f);
    const int64_t ka = (a & s) ? -(int64_t)(a & (s - 1)) - 1 : (int64_t)a, kb = (b & s) ? -(int64_t)(b & (s - 1)) - 1 : (int64_t)b;
    return ka < kb;
}
inline bool hp_is_nan(uint32_t h, HpFmt f) { return hp_decode(h, f).cls == 2; }
// min / max: one NaN operand gives the other; two give the canonical NaN.  .NaN: any NaN gives the canonical NaN.
inline uint32_t hp_minmax(uint32_t a, uint32_t b, HpFmt f, bool is_max, bool nan_mode) {
    const bool na = hp_is_nan(a, f), nb = hp_is_nan(b, f);
    if (na && nb) return kHpCanonicalNaN;
    if (na || nb) return nan_mode ? kHpCanonicalNaN : na ? b : a;
    return hp_less(a, b, f) != is_max ? a : b;
}
// min.xorsign.abs: min(|a|, |b|) with the sign sign(a) ^ sign(b) (finite operands)
inline uint32_t hp_min_xorsign(uint32_t a, uint32_t b, HpFmt f) {
    const uint32_t s = (uint32_t)hp_sign_bit(f);
    const uint32_t m = (a & (s - 1)) < (b & (s - 1)) ? a & (s - 1) : b & (s - 1);
    return m | ((a ^ b) & s);
}

// ---- conversions --------------------------------------------------------------------------------------------------
// float (f32 / f16 bits) to a 16- or 8-bit format: satfinite maps NaN to NaN (0x7FFF / e4m3 0x7F) and +-inf to +-max;
// relu maps NaN to the canonical NaN and every negative result, -0 included, to +0.
inline uint32_t hp_cvt_float(uint64_t bits, HpFmt from, HpFmt to, int mode, bool satfinite, bool relu) {
    const HpNum x = hp_decode(bits, from);
    const uint64_t s = x.neg ? hp_sign_bit(to) : 0;
    uint64_t r;
    if (x.cls == 2) return to.has_inf ? kHpCanonicalNaN : 0x7Fu;  // NaN reaches only the f16 / bf16 / e4m3 targets
    if (x.cls == 1) r = satfinite || !to.has_inf ? s | hp_max_finite(to) : s | hp_inf(to);
    else r = hp_round(x, to, mode, satfinite);
    if (relu && (r & hp_sign_bit(to))) r = 0;
    return (uint32_t)r;
}
// cvt.rn.tf32.f32: the f32 bits with the lower 13 bits zero
inline uint32_t hp_tf32(uint32_t x) {
    const uint32_t r = (uint32_t)hp_round(hp_decode(x, kHpF32), kHpTf32, HP_RN);
    return (r & 0x40000u) << 13 | (r & 0x3FFFFu) << 13;
}
// round to an integer in mode; the magnitude and the sign
inline hp_u128 hp_round_int(const HpNum& x, int mode) {
    if (x.e >= 0) return hp_msb(x.m) + x.e > 100 ? (hp_u128)1 << 100 : x.m << x.e;  // past every integer width: saturates
    const int s = -x.e;
    if (s > hp_msb(x.m) + 1) return (mode == HP_RM && x.neg && x.m) || (mode == HP_RP && !x.neg && x.m) ? 1 : 0;
    const hp_u128 n = x.m >> s, r = x.m - (n << s), half = (hp_u128)1 << (s - 1);
    bool up = false;
    if (r) {
        if (mode == HP_RN) up = r > half || (r == half && (n & 1));
        else if (mode == HP_RM) up = x.neg;
        else if (mode == HP_RP) up = !x.neg;
    }
    return n + up;
}
// cvt.{rni,rzi,rmi,rpi}.{s32,u32,s64}.{f32,f64}: saturating, NaN -> 0
inline uint64_t hp_f2i(uint64_t bits, HpFmt from, int mode, int width, bool is_signed) {
    const HpNum x = hp_decode(bits, from);
    if (x.cls == 2) return 0;
    const hp_u128 lim_pos = is_signed ? ((hp_u128)1 << (width - 1)) - 1 : ((hp_u128)1 << width) - 1;
    const hp_u128 lim_neg = is_signed ? (hp_u128)1 << (width - 1) : 0;
    const uint64_t mask = width == 64 ? ~0ull : (1ull << width) - 1;
    hp_u128 n = x.cls == 1 ? ((hp_u128)1 << 100) : hp_round_int(x, mode);
    if (x.neg && n) {
        if (n > lim_neg) n = lim_neg;
        return (uint64_t)(0 - (uint64_t)n) & mask;
    }
    if (n > lim_pos) n = lim_pos;
    return (uint64_t)n & mask;
}
// cvt.{rn,rz,rm,rp}.{f32,f64}.{s32,u64,s64}
inline uint64_t hp_i2f(uint64_t v, int width, bool is_signed, HpFmt to, int mode) {
    const bool neg = is_signed && (v >> (width - 1) & 1);
    uint64_t mag = v;
    if (width == 32) mag &= 0xFFFFFFFFull;
    if (neg) mag = (width == 32 ? (uint64_t)(0u - (uint32_t)v) : 0 - v);
    return hp_round(HpNum{neg, mag, 0, 0}, to, mode);
}
// cvt.rni.f32.f32 / cvt.rmi.f64.f64: the integer in mode, with the operand's sign on a zero
inline uint64_t hp_frnd(uint64_t bits, HpFmt f, int mode) {
    const HpNum x = hp_decode(bits, f);
    if (x.e >= 0) return bits;  // already an integer
    const hp_u128 n = hp_round_int(x, mode);
    return hp_round(HpNum{x.neg, n, 0, 0}, f, HP_RN);
}

// ---- generator ------------------------------------------------------------------------------------------------------
inline uint32_t hp_stream_key(uint32_t seed, int fmt, int tile) {
    return ct_mix(seed ^ (uint32_t)(fmt * 16 + tile + 1) * 0x27D4EB2Fu);
}
inline uint32_t hp_hash(uint32_t seed, int fmt, int tile, int t, int slot, int k) {
    return ct_hash(hp_stream_key(seed, fmt, tile), (uint32_t)((t * 256 + slot) * 4 + k));
}
// Random finite values: sign, an exponent near 1 and a random significand.
inline uint32_t hp_rand_f16(uint32_t h) { return (h & 0x83FFu) | ((h >> 10) % 29 + 1) << 10; }
inline uint32_t hp_rand_bf16(uint32_t h) { return (h & 0x807Fu) | ((h >> 7) % 41 + 107) << 7; }
inline uint32_t hp_rand_f32(uint32_t h, uint32_t h2, int lo, int span) {
    return (h & 0x807FFFFFu) | (uint32_t)(lo + (int)(h2 % (uint32_t)span)) << 23;
}
inline uint32_t hp_rand_e4m3(uint32_t h) { return (h & 0x7F) == 0x7F ? h & 0xFE : h & 0xFF; }
inline uint32_t hp_rand_e5m2(uint32_t h) { return (h & 0x7F) > 0x7C ? (h & 0xFF) - 4 : h & 0xFF; }

// The crafted classes, one lane each: kHpAbc*[i] = {a, b, c}, kHpXyz*[i] = {x, y, z}.
constexpr int kHpHalfClasses = 12;  // = 2 lanes x kHpCrafted
constexpr uint16_t kHpAbcF16[kHpHalfClasses][3] = {
    {0x1000, 0x3C00, 0x3C00},  // tie, rounded down to even: 1 + 2^-11
    {0x1000, 0x3C00, 0x3C01},  // tie, rounded up to even: 1 + 2^-10 + 2^-11
    {0x3C01, 0x3C01, 0xBC02},  // cancellation: (1 + 2^-10)^2 - (1 + 2^-9) = 2^-20, a subnormal
    {0x0E55, 0x2E66, 0x8001},  // a subnormal result, rounded
    {0x0155, 0x4A00, 0x0003},  // a subnormal multiplicand and addend (both flushed under .ftz)
    {0x7800, 0x4000, 0x3C00},  // overflow to +inf
    {0xF800, 0x4000, 0x3C00},  // overflow to -inf
    {0x8000, 0x4500, 0x8000},  // -0 * 5 + -0 = -0
    {0x0000, 0xC500, 0x0000},  // -0 + +0 = +0
    {0x1001, 0x3C01, 0x3C00},  // one above a tie only through the sticky bits
    {0x3C01, 0x4200, 0x8001},  // double-rounding trap: 3 (1 + 2^-10) - 2^-24
    {0x0400, 0x3800, 0x0000},  // 2^-15: subnormal, flushed to +0 under .ftz
};
constexpr uint16_t kHpXyzF16[kHpHalfClasses][3] = {
    {0x4000, 0x4200, 0x3800},  // 6.5: .sat -> 1
    {0xC000, 0x4200, 0x3C00},  // -5: .sat and .relu -> +0
    {0x8000, 0x3C00, 0x8000},  // -0: .sat and .relu -> +0; min(-0, 1)
    {0x7E01, 0x4000, 0x3C00},  // one NaN
    {0xFE10, 0x7D00, 0x0000},  // two NaNs
    {0x7C00, 0x4000, 0xBC00},  // +inf: .sat -> 1
    {0x7C00, 0x3C00, 0xFC00},  // inf - inf = NaN
    {0x0000, 0x8000, 0x0000},  // min / max of +0 and -0
    {0x3800, 0x3A00, 0x3000},  // 0.5: inside [0, 1]
    {0x3C00, 0x3C00, 0x0000},  // exactly 1
    {0xFC00, 0x4000, 0x3C00},  // -inf
    {0x4500, 0xC500, 0x4E40},  // -25 + 25 = +0; min / max of equal magnitudes
};
constexpr uint16_t kHpAbcBf16[kHpHalfClasses][3] = {
    {0x3B80, 0x3F80, 0x3F80}, {0x3B80, 0x3F80, 0x3F81}, {0x3F81, 0x3F81, 0xBF82}, {0x1CD5, 0x21B3, 0x8001},
    {0x0055, 0x4140, 0x0003}, {0x7F00, 0x4000, 0x3F80}, {0xFF00, 0x4040, 0x3F80}, {0x8000, 0x40A0, 0x8000},
    {0x0000, 0xC0A0, 0x0000}, {0x3B81, 0x3F81, 0x3F80}, {0x3F81, 0x4040, 0xAB80}, {0x0080, 0x3F00, 0x0000},
};
constexpr uint16_t kHpXyzBf16[kHpHalfClasses][3] = {
    {0x4000, 0x4040, 0x3F00}, {0xC000, 0x4040, 0x3F80}, {0x8000, 0x3F80, 0x8000}, {0x7FC1, 0x4000, 0x3F80},
    {0xFFC2, 0x7F81, 0x0000}, {0x7F80, 0x4000, 0xBF80}, {0x7F80, 0x3F80, 0xFF80}, {0x0000, 0x8000, 0x0000},
    {0x3F00, 0x3F40, 0x3E00}, {0x3F80, 0x3F80, 0x0000}, {0xFF80, 0x4000, 0x3F80}, {0x40A0, 0xC0A0, 0x41C8},
};
// HP_CVT: per-lane lists (X / Y, P / Q, H, E4, E5: 16 lanes over the 8 crafted sets) and per-set lists (F, I, D, L).
constexpr uint32_t kHpCvtXY[16] = {
    0x3F801000u,  // 1 + 2^-11: f16 / tf32 tie, down to even
    0x3F803000u,  // 1 + 2^-10 + 2^-11: f16 / tf32 tie, up to even
    0x3F808000u,  // 1 + 2^-8: bf16 tie, down
    0x3F818000u,  // 1 + 2^-7 + 2^-8: bf16 tie, up
    0x477FF000u,  // 65520: f16 rn -> inf, rz -> 65504
    0xC7800000u,  // -65536
    0x35A12345u,  // an f16 subnormal result
    0x33000000u,  // 2^-25: half the least f16 subnormal, rn -> 0
    0x33000001u,  // just above it: rn -> 2^-24
    0xBF800001u,  // -(1 + 2^-23): rm / rp of a negative value
    0x47700000u,  // 61440: e5m2 tie at the top, .satfinite -> 57344
    0x47600000u,  // 57344: e5m2's largest finite value
    0x37000000u,  // 2^-17: half the least e5m2 subnormal -> 0
    0x36FFFFFFu,  // just below it
    0xC0200000u,  // -2.5: FRND to -2
    0x3FC00000u,  // 1.5: FRND to 2
};
constexpr uint32_t kHpCvtPQ[16] = {
    0x7F800000u, 0xFF800000u, 0x7FC00001u,  // +inf, -inf, NaN
    0x43E00000u,  // 448: e4m3's largest finite value
    0x43F00000u,  // 480: .satfinite -> 448
    0x43E80000u,  // 464: the tie above 448
    0x3B000000u,  // 2^-9: the least e4m3 subnormal
    0x3A800000u,  // 2^-10: half of it, rn -> 0
    0x3A800001u,  // just above: rn -> 2^-9
    0x3A7FFFFFu,  // just below
    0xBFC00000u,  // -1.5: .relu -> +0
    0x80000000u,  // -0: .relu -> +0
    0x477FF000u,  // 65520: .satfinite -> 65504 in f16
    0x7F7FFFFFu,  // the largest f32: bf16 .satfinite -> its largest finite value
    0xC3E80000u,  // -464
    0x3E2AAAABu,  // 1/6
};
constexpr uint16_t kHpCvtH[16] = {
    0x7C00, 0xFC00,  // +-inf: .satfinite -> +-max
    0x5F00, 0x5F80, 0x5F40,  // 448, 480, 464 (e4m3)
    0x7B00, 0x7B80,  // 57344, 61440 (e5m2)
    0x1800, 0x1400, 0x1401, 0x13FF,  // 2^-9, 2^-10 and its neighbours
    0x0100, 0x0080, 0x0081,  // 2^-16 (e5m2's least subnormal), half of it, just above
    0xBE00, 0x8000,  // -1.5, -0
};
constexpr uint8_t kHpCvtE4[16] = {0x01, 0x81, 0x7E, 0xFE, 0x08, 0x07, 0x00, 0x80,
                                  0x38, 0x3F, 0x77, 0xC5, 0x02, 0x40, 0x0F, 0x70};
constexpr uint8_t kHpCvtE5[16] = {0x01, 0x81, 0x7B, 0xFB, 0x7C, 0xFC, 0x04, 0x03,
                                  0x00, 0x80, 0x3C, 0x3F, 0x02, 0xC1, 0x5A, 0x43};
constexpr uint32_t kHpCvtF[8] = {
    0x4F000000u, 0xCF000000u, 0x4F800000u,  // 2^31, -2^31, 2^32: saturation
    0xBF000000u, 0x3F000000u, 0x3FC00000u, 0x40200000u,  // -0.5, 0.5, 1.5, 2.5
    0x7FC00000u,  // NaN -> 0
};
constexpr uint32_t kHpCvtI[8] = {0x01000001u, 0xFEFFFFFDu, 0x80000000u, 0x7FFFFFFFu,
                                 0x01000003u, 0x00000000u, 0xFFFFFFFFu, 0x00FFFFFFu};
constexpr uint64_t kHpCvtD[8] = {
    0x43E0000000000000ull,  // 2^63: s64 saturates
    0xC3E0000000000000ull,  // -2^63
    0x47F0000000000001ull,  // above f32's range: rz / rm -> max finite, rn / rp -> inf
    0xC7F0000000000001ull,
    0x3738000000000001ull,  // an f32 subnormal result
    0x3FF0000010000000ull,  // 1 + 2^-24: f32 tie
    0xC004000000000000ull,  // -2.5
    0x8000000000000001ull,  // -2^-1074: floor -> -1
};
constexpr uint64_t kHpCvtL[8] = {
    0x0020000000000001ull,  // 2^53 + 1
    0x8000010000000001ull,  // above 2^63 as u64
    0xFFFFFFFFFFFFFFFFull,  // u64 max / -1
    0x8000000000000000ull,
    0x7FFFFFFFFFFFFFFFull,
    0x0000000001000001ull,  // 2^24 + 1
    0xFFDFFFFFFFFFFFFFull,  // -(2^53 + 1)
    0x0020000000000003ull,  // 2^53 + 3
};

// The table of one tile: tab[slot * kCtThreads + t].  Crafted set s of thread t takes lane class (2s + L + t) % 16 (or
// % kHpHalfClasses) for lane L, and set class (s + t) % 8: every thread holds every class, and the two lanes of a word
// always hold different classes, so a lane swap shows.
inline void hp_operands(uint32_t seed, int fmt, int tile, uint32_t* tab) {
    const int SS = kHpSetSlots[fmt];
    for (int t = 0; t < kCtThreads; ++t) {
        auto at = [&](int set, int k) -> uint32_t& { return tab[(set * SS + k) * kCtThreads + t]; };
        auto h = [&](int set, int k, int i) { return hp_hash(seed, fmt, tile, t, set * SS + k, i); };
        for (int s = 0; s < kHpSets[fmt]; ++s) {
            const bool crafted = s < kHpCrafted[fmt];
            if (fmt != HP_CVT) {
                const bool f16 = fmt == HP_F16;
                for (int k = 0; k < 6; ++k) {
                    uint32_t w = 0;
                    for (int L = 0; L < 2; ++L) {
                        const int c = (2 * s + L + t) % kHpHalfClasses;
                        const uint32_t lane = !crafted ? (f16 ? hp_rand_f16(h(s, k, L)) : hp_rand_bf16(h(s, k, L)))
                                              : k < 3 ? (f16 ? kHpAbcF16 : kHpAbcBf16)[c][k]
                                                      : (f16 ? kHpXyzF16 : kHpXyzBf16)[c][k - 3];
                        w |= lane << (16 * L);
                    }
                    at(s, k) = w;
                }
                continue;
            }
            const int l0 = (2 * s + t) % 16, l1 = (2 * s + 1 + t) % 16, c = (s + t) % 8;
            if (crafted) {
                at(s, HC_X) = kHpCvtXY[l0];
                at(s, HC_Y) = kHpCvtXY[l1];
                at(s, HC_P) = kHpCvtPQ[l0];
                at(s, HC_Q) = kHpCvtPQ[l1];
                at(s, HC_F) = kHpCvtF[c];
                at(s, HC_H) = (uint32_t)kHpCvtH[l0] << 16 | kHpCvtH[l1];
                at(s, HC_E4) = (uint32_t)kHpCvtE4[l0] << 8 | kHpCvtE4[l1];
                at(s, HC_E5) = (uint32_t)kHpCvtE5[l0] << 8 | kHpCvtE5[l1];
                at(s, HC_I) = kHpCvtI[c];
                at(s, HC_DLO) = (uint32_t)kHpCvtD[c];
                at(s, HC_DHI) = (uint32_t)(kHpCvtD[c] >> 32);
                at(s, HC_LLO) = (uint32_t)kHpCvtL[c];
                at(s, HC_LHI) = (uint32_t)(kHpCvtL[c] >> 32);
            } else {
                at(s, HC_X) = hp_rand_f32(h(s, HC_X, 0), h(s, HC_X, 1), 97, 61);
                at(s, HC_Y) = hp_rand_f32(h(s, HC_Y, 0), h(s, HC_Y, 1), 97, 61);
                at(s, HC_P) = hp_rand_f32(h(s, HC_P, 0), h(s, HC_P, 1), 110, 30);
                at(s, HC_Q) = hp_rand_f32(h(s, HC_Q, 0), h(s, HC_Q, 1), 110, 30);
                at(s, HC_F) = hp_rand_f32(h(s, HC_F, 0), h(s, HC_F, 1), 123, 36);
                at(s, HC_H) = hp_rand_f16(h(s, HC_H, 0)) << 16 | hp_rand_f16(h(s, HC_H, 1));
                at(s, HC_E4) = hp_rand_e4m3(h(s, HC_E4, 0)) << 8 | hp_rand_e4m3(h(s, HC_E4, 1));
                at(s, HC_E5) = hp_rand_e5m2(h(s, HC_E5, 0)) << 8 | hp_rand_e5m2(h(s, HC_E5, 1));
                at(s, HC_I) = h(s, HC_I, 0);
                const uint32_t dh = h(s, HC_DHI, 0);
                at(s, HC_DLO) = h(s, HC_DLO, 0);
                at(s, HC_DHI) = (dh & 0x800FFFFFu) | (uint32_t)(1023 - 160 + (int)(h(s, HC_DHI, 1) % 321)) << 20;
                at(s, HC_LLO) = h(s, HC_LLO, 0);
                at(s, HC_LHI) = h(s, HC_LHI, 0) >> (h(s, HC_LHI, 1) % 32);  // magnitudes from 2^32 to 2^64
            }
        }
    }
}

// The result words of one set of HP_CVT; o receives kHpSetWords[HP_CVT] words.
inline void hp_cvt_set(const uint32_t* v, uint32_t* o) {
    const uint32_t X = v[HC_X], Y = v[HC_Y], P = v[HC_P], Q = v[HC_Q], F = v[HC_F], H = v[HC_H];
    const uint64_t D = (uint64_t)v[HC_DHI] << 32 | v[HC_DLO], L = (uint64_t)v[HC_LHI] << 32 | v[HC_LLO];
    auto pack16 = [](uint32_t hi, uint32_t lo) { return hi << 16 | lo; };
    auto f2h = [](uint32_t x, HpFmt to, int mode, bool sat, bool relu) { return hp_cvt_float(x, kHpF32, to, mode, sat, relu); };
    o[HC_F16X2_RN] = pack16(f2h(X, kHpF16, HP_RN, 0, 0), f2h(Y, kHpF16, HP_RN, 0, 0));
    o[HC_F16X2_RZ] = pack16(f2h(X, kHpF16, HP_RZ, 0, 0), f2h(Y, kHpF16, HP_RZ, 0, 0));
    o[HC_F16X2_RELU] = pack16(f2h(P, kHpF16, HP_RN, 0, 1), f2h(Q, kHpF16, HP_RN, 0, 1));
    o[HC_F16X2_SATF] = pack16(f2h(P, kHpF16, HP_RN, 1, 0), f2h(Q, kHpF16, HP_RN, 1, 0));
    o[HC_BF16X2_RN] = pack16(f2h(X, kHpBf16, HP_RN, 0, 0), f2h(Y, kHpBf16, HP_RN, 0, 0));
    o[HC_BF16X2_RZ] = pack16(f2h(X, kHpBf16, HP_RZ, 0, 0), f2h(Y, kHpBf16, HP_RZ, 0, 0));
    o[HC_BF16X2_RELU] = pack16(f2h(P, kHpBf16, HP_RN, 0, 1), f2h(Q, kHpBf16, HP_RN, 0, 1));
    o[HC_BF16X2_SATF] = pack16(f2h(P, kHpBf16, HP_RN, 1, 0), f2h(Q, kHpBf16, HP_RN, 1, 0));
    o[HC_E4M3_F32] = f2h(P, kHpE4m3, HP_RN, 1, 0) << 8 | f2h(Q, kHpE4m3, HP_RN, 1, 0);
    o[HC_E5M2_F32] = f2h(X, kHpE5m2, HP_RN, 1, 0) << 8 | f2h(Y, kHpE5m2, HP_RN, 1, 0);
    o[HC_E4M3_F16] = hp_cvt_float(H >> 16, kHpF16, kHpE4m3, HP_RN, 1, 0) << 8 | hp_cvt_float(H & 0xFFFF, kHpF16, kHpE4m3, HP_RN, 1, 0);
    o[HC_E5M2_F16] = hp_cvt_float(H >> 16, kHpF16, kHpE5m2, HP_RN, 1, 0) << 8 | hp_cvt_float(H & 0xFFFF, kHpF16, kHpE5m2, HP_RN, 1, 0);
    auto f8h = [](uint32_t b, HpFmt f) {
        const HpNum x = hp_decode(b, f);
        return x.cls == 1 ? (uint32_t)(hp_inf(kHpF16) | (x.neg ? 0x8000u : 0u)) : (uint32_t)hp_round(x, kHpF16, HP_RN);
    };
    o[HC_F16_E4M3] = pack16(f8h(v[HC_E4] >> 8 & 0xFF, kHpE4m3), f8h(v[HC_E4] & 0xFF, kHpE4m3));
    o[HC_F16_E5M2] = pack16(f8h(v[HC_E5] >> 8 & 0xFF, kHpE5m2), f8h(v[HC_E5] & 0xFF, kHpE5m2));
    o[HC_TF32] = hp_tf32(X);
    o[HC_F16_RM] = f2h(X, kHpF16, HP_RM, 0, 0);
    o[HC_F16_RP] = f2h(X, kHpF16, HP_RP, 0, 0);
    o[HC_BF16_RM] = f2h(X, kHpBf16, HP_RM, 0, 0);
    o[HC_BF16_RP] = f2h(X, kHpBf16, HP_RP, 0, 0);
    for (int m = 0; m < 4; ++m) {
        o[HC_S32 + m] = (uint32_t)hp_f2i(F, kHpF32, m, 32, true);
        o[HC_U32 + m] = (uint32_t)hp_f2i(F, kHpF32, m, 32, false);
        const uint64_t s64 = hp_f2i(D, kHpF64, m, 64, true);
        o[HC_S64 + 2 * m] = (uint32_t)s64;
        o[HC_S64 + 2 * m + 1] = (uint32_t)(s64 >> 32);
        o[HC_I2F_S32 + m] = (uint32_t)hp_i2f(v[HC_I], 32, true, kHpF32, m);
        o[HC_I2F_U64 + m] = (uint32_t)hp_i2f(L, 64, false, kHpF32, m);
        const uint64_t d = hp_i2f(L, 64, true, kHpF64, m);
        o[HC_I2F_S64 + 2 * m] = (uint32_t)d;
        o[HC_I2F_S64 + 2 * m + 1] = (uint32_t)(d >> 32);
        o[HC_F32_F64 + m] = hp_cvt_float(D, kHpF64, kHpF32, m, 0, 0);
    }
    o[HC_FRND_F32] = (uint32_t)hp_frnd(X, kHpF32, HP_RN);
    const uint64_t fl = hp_frnd(D, kHpF64, HP_RM);
    o[HC_FRND_F64] = (uint32_t)fl;
    o[HC_FRND_F64 + 1] = (uint32_t)(fl >> 32);
}

// Reference result words of every thread: words[t * kHpWords[fmt] + set * kHpSetWords[fmt] + j].
inline void hp_results(int fmt, const uint32_t* tab, uint32_t* words) {
    const int SS = kHpSetSlots[fmt], SW = kHpSetWords[fmt], W = kHpWords[fmt];
    for (int t = 0; t < kCtThreads; ++t)
        for (int set = 0; set < kHpSets[fmt]; ++set) {
            uint32_t v[13];
            for (int k = 0; k < SS; ++k) v[k] = tab[(set * SS + k) * kCtThreads + t];
            uint32_t* o = words + (size_t)t * W + set * SW;
            if (fmt == HP_CVT) { hp_cvt_set(v, o); continue; }
            const HpFmt f = fmt == HP_F16 ? kHpF16 : kHpBf16;
            auto lanes = [&](auto op) { return op(0) | op(16) << 16; };
            auto l = [&](int k, int sh) { return v[k] >> sh & 0xFFFF; };
            const uint32_t fma = lanes([&](int sh) { return hp_fma(l(HS_A, sh), l(HS_B, sh), l(HS_C, sh), f); });
            const uint32_t relu = lanes([&](int sh) { return hp_fma(l(HS_X, sh), l(HS_Y, sh), l(HS_Z, sh), f, HP_RELU); });
            const uint32_t add = lanes([&](int sh) { return hp_add(l(HS_A, sh), l(HS_B, sh), f); });
            const uint32_t sub = lanes([&](int sh) { return hp_sub(l(HS_A, sh), l(HS_B, sh), f); });
            const uint32_t mul = lanes([&](int sh) { return hp_mul(l(HS_A, sh), l(HS_B, sh), f); });
            auto mm = [&](bool mx, bool nan) {
                return lanes([&](int sh) { return hp_minmax(l(HS_X, sh), l(HS_Y, sh), f, mx, nan); });
            };
            if (fmt == HP_F16) {
                o[HF_FMA] = fma;
                o[HF_FMA_RELU] = relu;
                o[HF_FMA_SAT] = lanes([&](int sh) { return hp_fma(l(HS_X, sh), l(HS_Y, sh), l(HS_Z, sh), f, HP_SAT); });
                o[HF_FMA_FTZ] = lanes([&](int sh) { return hp_fma(l(HS_A, sh), l(HS_B, sh), l(HS_C, sh), f, HP_FTZ); });
                o[HF_ADD] = add;
                o[HF_SUB] = sub;
                o[HF_MUL] = mul;
                o[HF_MIN] = mm(false, false);
                o[HF_MAX] = mm(true, false);
                o[HF_MIN_NAN] = mm(false, true);
                o[HF_MAX_NAN] = mm(true, true);
                o[HF_MIN_XORSIGN] = lanes([&](int sh) { return hp_min_xorsign(l(HS_A, sh), l(HS_B, sh), f); });
            } else {
                o[HB_FMA] = fma;
                o[HB_FMA_RELU] = relu;
                o[HB_ADD] = add;
                o[HB_SUB] = sub;
                o[HB_MUL] = mul;
                o[HB_MIN] = mm(false, false);
                o[HB_MAX] = mm(true, false);
                o[HB_MIN_NAN] = mm(false, true);
                o[HB_MAX_NAN] = mm(true, true);
            }
        }
}

// table: hp_table_bytes(fmt) bytes, copied verbatim to the device; check: kCtThreads comparison values; words
// (optional): [thread][kHpWords[fmt]] reference results.
inline void hp_build_tile(uint32_t seed, int fmt, int tile, uint32_t* table, uint32_t* check,
                          std::vector<uint32_t>* words = nullptr) {
    std::vector<uint32_t> own;
    std::vector<uint32_t>& w = words ? *words : own;
    w.assign((size_t)kCtThreads * kHpWords[fmt], 0);
    hp_operands(seed, fmt, tile, table);
    hp_results(fmt, table, w.data());
    for (int t = 0; t < kCtThreads; ++t) check[t] = it_fold(&w[(size_t)t * kHpWords[fmt]], kHpWords[fmt]);
}

}  // namespace b2dp
