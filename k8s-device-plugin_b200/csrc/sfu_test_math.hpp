// sfu_test_math.hpp -- host-side arithmetic of the on-demand SFU self-test (b2dp_sfu_test, sfu_selftest.cuh).
//
// Pure C++ (no CUDA), so the CPU tests compile it as it is (tests/native/sfu_test_math_test.cpp) and compare it with the
// restatement in tests/sfu_test_oracle.py:
//   - sf_thread_operands: seed, format, tile, thread  ->  the thread's operand words, crafted classes included
//   - sf_build_table:     the operand table of one tile a launch reads verbatim ([slot][thread] words)
//   - sf_guard:           one result against a loose error bound of the exact function, or its specials class
//   - sf_consensus:       the reference dumps of every SM  ->  the majority words, the dissenting SMs, the guard
//   - sf_fold:            the per-thread comparison value the timed launch checks
// The per-CTA record (CtRecord), its completeness rule and the timed launch's verdict are the tensor-core test's
// (compute_test_math.hpp).
//
// Why the host cannot predict the results bit for bit, and what it checks instead: NVIDIA publishes no bit-level model
// of the special-function unit (MUFU), so the host can bound a result but not reproduce it.  The reference launch runs
// one CTA on every SM; each result word's majority value over the SMs is the reference, and any SM that disagrees with
// it is named.  No SM is ever judged against its own output.  The majority itself must lie within a loose bound of the
// exact function (computed in double with <cmath>), which catches a fault the whole device shares.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "compute_test_math.hpp"  // ct_mix, ct_hash, ct_uniform, CtRecord, kCtThreads, kCtTiles, kCtReps, kCtMaxSmId

namespace b2dp {

enum SfFormat { SF_F32 = 0, SF_ROOT = 1, SF_F16 = 2 };
constexpr int kSfFormats = 3;
static_assert(kSfFormats == kCtFormats, "the verdict and the result struct are shared with the tensor-core test");

// Operand groups: one PTX instruction each (sin and cos share their operands), kSfN operands per thread.
enum SfOp { SF_EX2, SF_LG2, SF_SINCOS, SF_TANH, SF_RCP, SF_RSQ, SF_SQRT, SF_RCP64, SF_RSQ64, SF_EX2H, SF_TANHH, kSfOps };
// The functions the guard evaluates (SF_SINCOS yields SF_FN_SIN and SF_FN_COS).
enum SfFn { SF_FN_EX2, SF_FN_LG2, SF_FN_SIN, SF_FN_COS, SF_FN_TANH, SF_FN_RCP, SF_FN_RSQ, SF_FN_SQRT, kSfFns };
enum SfType { SF_T32 = 0, SF_T64 = 1, SF_T16 = 2 };  // binary32, binary64 (two words), binary16 (half a word)

constexpr int kSfN = 16;  // operand words of one group per thread: 16 f32 / f64 values or 16 f16x2 pairs

struct SfOpInfo {
    const char* name;
    int fmt, type;
    bool ftz;          // the PTX form is .ftz: subnormal inputs and results are flushed to a signed zero
    int slot0, word0;  // first operand slot and first result word (SF_SINCOS: sin at word0 + i, cos at word0 + 16 + i)
    int fn0;           // SfFn of the (first) result
    int crafted;       // crafted classes (value v of thread t holds class (v - t) mod values when below this)
};
// Format SF_F32: ex2, lg2, sin + cos, tanh.  SF_ROOT: rcp, rsqrt, sqrt (f32), rcp, rsqrt (f64; two slots, two words
// per value, low word first).  SF_F16: ex2, tanh on f16x2 (value 2i is the low half of word i, 2i + 1 the high half).
constexpr SfOpInfo kSfOp[kSfOps] = {
    {"ex2", SF_F32, SF_T32, true, 0, 0, SF_FN_EX2, 11},      {"lg2", SF_F32, SF_T32, true, 16, 16, SF_FN_LG2, 11},
    {"sincos", SF_F32, SF_T32, true, 32, 32, SF_FN_SIN, 10}, {"tanh", SF_F32, SF_T32, false, 48, 64, SF_FN_TANH, 8},
    {"rcp", SF_ROOT, SF_T32, true, 0, 0, SF_FN_RCP, 10},     {"rsqrt", SF_ROOT, SF_T32, true, 16, 16, SF_FN_RSQ, 10},
    {"sqrt", SF_ROOT, SF_T32, true, 32, 32, SF_FN_SQRT, 10}, {"rcp64", SF_ROOT, SF_T64, true, 48, 48, SF_FN_RCP, 10},
    {"rsqrt64", SF_ROOT, SF_T64, true, 80, 80, SF_FN_RSQ, 10}, {"ex2h", SF_F16, SF_T16, false, 0, 0, SF_FN_EX2, 12},
    {"tanhh", SF_F16, SF_T16, false, 16, 16, SF_FN_TANH, 8},
};
constexpr int kSfSlots[kSfFormats] = {64, 112, 32};  // operand words per thread
constexpr int kSfWords[kSfFormats] = {80, 112, 32};  // result words per thread and repetition
constexpr int kSfMaxWords = 112;
// MUFU results per thread and repetition (one per f32 / f64 value, one per f16 half)
constexpr int kSfResults[kSfFormats] = {5 * kSfN, 5 * kSfN, 4 * kSfN};
inline int sf_values(int op) { return kSfOp[op].type == SF_T16 ? 2 * kSfN : kSfN; }
inline uint32_t sf_table_bytes(int fmt) { return (uint32_t)(kSfSlots[fmt] * kCtThreads * 4); }
inline double sf_results_per_tile(int fmt) { return (double)kCtThreads * kSfResults[fmt]; }

// Crafted classes (tests/sfu_test_oracle.py names them): per op the head classes of sf_operand's switch, then six
// specials every op shares -- a subnormal input (random sign), +0, -0, +inf, -inf and a quiet NaN.

// ---- bits ---------------------------------------------------------------------------------------------------------
struct SfBin {
    int width, M, BIAS;
};
constexpr SfBin kSfBin[3] = {{32, 23, 127}, {64, 52, 1023}, {16, 10, 15}};
inline uint64_t sf_mmask(int type) { return (1ull << kSfBin[type].M) - 1; }
// sign * 1.mant * 2^e (normal)
inline uint64_t sf_make(int type, uint32_t s, int e, uint64_t mant) {
    const SfBin& b = kSfBin[type];
    return (uint64_t)(s & 1u) << (b.width - 1) | (uint64_t)(e + b.BIAS) << b.M | (mant & sf_mmask(type));
}
inline uint64_t sf_sub(int type, uint32_t s, uint64_t mant) {  // a nonzero subnormal
    return (uint64_t)(s & 1u) << (kSfBin[type].width - 1) | (((mant & sf_mmask(type)) | 1ull));
}
inline uint64_t sf_zero(int type, uint32_t s) { return (uint64_t)(s & 1u) << (kSfBin[type].width - 1); }
inline uint64_t sf_inf(int type, uint32_t s) {
    const SfBin& b = kSfBin[type];
    return sf_zero(type, s) | (uint64_t)(2 * b.BIAS + 1) << b.M;
}
inline uint64_t sf_nan(int type) { return sf_inf(type, 0) | 1ull << (kSfBin[type].M - 1); }
// an integer k that the type holds exactly
inline uint64_t sf_int(int type, int k) {
    if (k == 0) return 0;
    const uint32_t s = k < 0;
    const uint64_t a = (uint64_t)(k < 0 ? -k : k);
    int e = 0;
    while ((a >> (e + 1)) != 0) ++e;
    return sf_make(type, s, e, (a << kSfBin[type].M >> e));
}
inline double sf_value(int type, uint64_t bits) {
    if (type == SF_T64) { double d; std::memcpy(&d, &bits, 8); return d; }
    if (type == SF_T32) { float f; uint32_t u = (uint32_t)bits; std::memcpy(&f, &u, 4); return (double)f; }
    const uint32_t s = (uint32_t)(bits >> 15) & 1u, e = (uint32_t)(bits >> 10) & 31u, m = (uint32_t)bits & 1023u;
    double v = e == 31 ? (m ? NAN : INFINITY) : e == 0 ? std::ldexp((double)m, -24) : std::ldexp(1024.0 + m, (int)e - 25);
    return s ? -v : v;
}
inline bool sf_is_subnormal(int type, uint64_t bits) {
    const SfBin& b = kSfBin[type];
    return ((bits >> b.M) & ((1ull << (b.width - 1 - b.M)) - 1)) == 0 && (bits & sf_mmask(type)) != 0;
}
inline double sf_min_normal(int type) { return std::ldexp(1.0, 1 - kSfBin[type].BIAS); }
inline double sf_max_finite(int type) {
    const SfBin& b = kSfBin[type];
    return std::ldexp(2.0 - std::ldexp(1.0, -b.M), b.BIAS);
}

// ---- generator ------------------------------------------------------------------------------------------------------
inline uint32_t sf_stream_key(uint32_t seed, int op, int tile) {
    return ct_mix(seed ^ (uint32_t)((tile * 16 + op) + 1) * 0x27D4EB2Fu);
}
// draw j (0..3) of value v of thread t
inline uint32_t sf_draw(uint32_t key, int t, int v, int j) { return ct_hash(key, (uint32_t)((t * 64 + v) * 4 + j)); }

// The random operand of each op: sign (-1 = random), and the exponent range of a full-mantissa value.
struct SfRandom {
    int sign, elo, ehi;
};
constexpr SfRandom kSfRandom[kSfOps] = {
    {-1, -20, 6},    {0, -126, 127}, {-1, -20, 2},     {-1, -20, 3},     {-1, -125, 124}, {0, -126, 127},
    {0, -126, 127},  {-1, -1021, 1020}, {0, -1022, 1023}, {-1, -10, 3}, {-1, -10, 2},
};

// Value v of op `op` for thread t: crafted class (v - t) mod values if that is below kSfOp[op].crafted, else random.
inline uint64_t sf_operand(uint32_t seed, int op, int tile, int t, int v) {
    const SfOpInfo& I = kSfOp[op];
    const int T = I.type, n = sf_values(op);
    const uint32_t key = sf_stream_key(seed, op, tile);
    const uint32_t d0 = sf_draw(key, t, v, 0), d1 = sf_draw(key, t, v, 1), d2 = sf_draw(key, t, v, 2),
                   d3 = sf_draw(key, t, v, 3);
    const uint64_t m = (uint64_t)d2 << 32 | d0;
    const uint32_t rs = d3 >> 31;
    const int c = ((v - t) % n + n) % n;
    const int nh = I.crafted - 6;
    if (c >= I.crafted) {
        const SfRandom& R = kSfRandom[op];
        return sf_make(T, R.sign < 0 ? rs : (uint32_t)R.sign, ct_uniform(d1, R.elo, R.ehi), m);
    }
    if (c >= nh) {
        switch (c - nh) {
            case 0: return sf_sub(T, rs, m);
            case 1: return sf_zero(T, 0);
            case 2: return sf_zero(T, 1);
            case 3: return sf_inf(T, 0);
            case 4: return sf_inf(T, 1);
            default: return sf_nan(T);
        }
    }
    const int EMAX = kSfBin[T].BIAS, EMIN = 1 - kSfBin[T].BIAS;
    switch (op) {
        case SF_EX2:
            switch (c) {
                case 0: return sf_int(T, ct_uniform(d1, -125, 127));  // 2^k: an exact point
                case 1: return 0x42FFFFFFu - (d0 & 63u);              // just below 128: 2^x just below 2^128
                case 2: return 0xC2FBFD00u - (d0 & 63u);              // -125.994..: 2^x 0.4 % above 2^-126
                case 3: return sf_int(T, 128 + (int)(d0 % 64u));      // +inf
                default: return sf_int(T, -(130 + (int)(d0 % 100u)));  // below 2^-129: flushed to +0
            }
        case SF_LG2:
            switch (c) {
                case 0: return sf_make(T, 0, ct_uniform(d1, EMIN, EMAX), 0);  // 2^k: an exact point
                case 1: return sf_make(T, 0, EMIN, m);
                case 2: return sf_make(T, 0, EMAX, m);
                case 3: return sf_make(T, 0, 0, d0 & 0xFFu);                   // 1 + a few ulp: a tiny result
                default: return sf_make(T, 1, ct_uniform(d1, EMIN, EMAX), m);  // NaN
            }
        case SF_SINCOS:
            switch (c) {
                case 0: return (uint64_t)rs << 31 | (0x41490FDAu - (d0 & 255u));  // |x| just below 4 pi
                case 1: return sf_make(T, rs, ct_uniform(d1, 4, 20), m);          // 16 <= |x| < 2^21
                case 2: return sf_make(T, rs, ct_uniform(d1, 60, EMAX), m);
                default: return sf_make(T, rs, ct_uniform(d1, EMIN, -60), m);
            }
        case SF_TANH:
        case SF_TANHH:
            if (c == 0) return sf_make(T, rs, ct_uniform(d1, T == SF_T16 ? 3 : 4, T == SF_T16 ? 15 : 20), m);  // +-1
            return sf_make(T, rs, ct_uniform(d1, EMIN, T == SF_T16 ? -5 : -20), m);
        case SF_RCP:
        case SF_RCP64:
        case SF_RSQ:
        case SF_SQRT:
        case SF_RSQ64: {
            const bool rcp = op == SF_RCP || op == SF_RCP64;
            const uint32_t s = rcp ? rs : 0u;
            switch (c) {
                case 0: return sf_make(T, s, 2 * ct_uniform(d1, -(EMAX / 2), EMAX / 2), 0);  // 4^k: an exact point
                case 1: return sf_make(T, s, EMIN, m);
                case 2: return rcp ? sf_make(T, s, EMAX - 2, m & sf_mmask(T) >> 1)  // 1 / x in (1.33, 2] * 2^EMIN
                                   : sf_make(T, s, EMAX, m);
                default: return rcp ? sf_make(T, s, EMAX, m)            // 1 / x below 2^EMIN: flushed to +-0
                                    : sf_make(T, 1, ct_uniform(d1, EMIN, EMAX), m);  // NaN
            }
        }
        default:  // SF_EX2H
            switch (c) {
                case 0: return sf_int(T, ct_uniform(d1, -14, 15));
                case 1: return 0x4BFFu - (d0 & 7u);                      // just below 16
                case 2: return 0xCAFFu - (d0 & 7u);                      // -13.99..: 2^x just above 2^-14
                case 3: return 0x4C00u + (d0 & 0x1FFu);                  // [16, 24): +inf
                case 4: return sf_int(T, -(15 + (int)(d0 % 9u)));         // 2^-15 .. 2^-23: a subnormal result
                default: return sf_int(T, -(25 + (int)(d0 % 40u)));      // below half the least subnormal
            }
    }
}

// The operand words of thread t ([slot]), as the kernel's registers hold them.
inline void sf_thread_operands(uint32_t seed, int fmt, int tile, int t, uint32_t* w) {
    for (int op = 0; op < kSfOps; ++op) {
        const SfOpInfo& I = kSfOp[op];
        if (I.fmt != fmt) continue;
        for (int v = 0; v < sf_values(op); ++v) {
            const uint64_t b = sf_operand(seed, op, tile, t, v);
            if (I.type == SF_T32) w[I.slot0 + v] = (uint32_t)b;
            else if (I.type == SF_T64) { w[I.slot0 + 2 * v] = (uint32_t)b; w[I.slot0 + 2 * v + 1] = (uint32_t)(b >> 32); }
            else if (v % 2 == 0) w[I.slot0 + v / 2] = (uint32_t)b;
            else w[I.slot0 + v / 2] |= (uint32_t)b << 16;
        }
    }
}

// Operand table of one tile: [slot][thread] words, so a warp's loads of one slot are coalesced.
inline void sf_build_table(uint32_t seed, int fmt, int tile, uint32_t* table) {
    uint32_t w[kSfMaxWords];
    for (int t = 0; t < kCtThreads; ++t) {
        sf_thread_operands(seed, fmt, tile, t, w);
        for (int s = 0; s < kSfSlots[fmt]; ++s) table[(size_t)s * kCtThreads + t] = w[s];
    }
}

// ---- the guard ------------------------------------------------------------------------------------------------------
// Error bound of each function per type: relative, except lg2, sin and cos (absolute).  Loose on purpose: it only
// has to catch a majority that is plainly wrong.
inline double sf_bound(int fn, int type) {
    if (type == SF_T16) return std::ldexp(1.0, -7);
    if (type == SF_T64) return std::ldexp(1.0, -16);
    if (fn == SF_FN_SIN || fn == SF_FN_COS) return std::ldexp(1.0, -16);
    if (fn == SF_FN_TANH) return std::ldexp(1.0, -8);
    return std::ldexp(1.0, -18);
}
inline bool sf_absolute(int fn) { return fn == SF_FN_LG2 || fn == SF_FN_SIN || fn == SF_FN_COS; }
// lg2's absolute bound grows with |e| beyond 16: 2^-18 is half an f32 ulp of a result in [64, 128), and an H100's
// lg2.approx.ftz.f32 is off by about one ulp there (DESIGN.md §4.8), so the bound is 2^-22 |e| above |e| = 16.
inline double sf_abs_bound(int fn, int type, double e) {
    const double B = sf_bound(fn, type);
    return fn == SF_FN_LG2 ? B * std::max(1.0, std::fabs(e) / 16) : B;
}
constexpr double kSfTrigGuarded = 4 * M_PI;  // sin, cos: bounded for |x| <= 4 pi, majority only beyond

inline double sf_exact(int fn, double x) {
    switch (fn) {
        case SF_FN_EX2: return std::exp2(x);
        case SF_FN_LG2: return std::log2(x);
        case SF_FN_SIN: return std::sin(x);
        case SF_FN_COS: return std::cos(x);
        case SF_FN_TANH: return std::tanh(x);
        case SF_FN_RCP: return 1.0 / x;
        case SF_FN_RSQ: return 1.0 / std::sqrt(x);
        default: return std::sqrt(x);
    }
}

// Does result r (bits) of fn on operand x (bits) pass the guard?  *err receives the error the bound was applied to (0
// where only the class was checked).  The exact value e is fn of x, with a subnormal x flushed to a signed zero for the
// .ftz forms.  Then:
//   - e NaN: r NaN.  e +-inf: r the same infinity.  e exactly +-0: r the same signed zero.
//   - lg2, sin, cos: |r - e| within the bound (sf_abs_bound; sin, cos only for |x| <= 4 pi, beyond that the majority
//     check alone).
//   - otherwise |r - e| / |e| within the bound, except at the ends of the type's range: where the bound reaches past
//     the largest finite value, r may be the infinity of e's sign; where it reaches below the smallest normal, only
//     the class is checked: r = +-0 for .ftz forms, r = +-0 or a subnormal of e's sign for the others.
inline bool sf_guard(int fn, int type, bool ftz, uint64_t xb, uint64_t rb, double* err = nullptr) {
    double x = sf_value(type, xb);
    if (ftz && sf_is_subnormal(type, xb)) x = std::copysign(0.0, x);
    const double e = sf_exact(fn, x), r = sf_value(type, rb);
    if (err) *err = 0;
    if (std::isnan(e)) return std::isnan(r);
    if (std::isnan(r)) return false;
    if (std::isinf(e)) return r == e;
    if (e == 0 && (x == 0 || std::isinf(x))) return r == 0 && std::signbit(r) == std::signbit(e);
    const double B = sf_bound(fn, type);
    if (sf_absolute(fn)) {
        if ((fn == SF_FN_SIN || fn == SF_FN_COS) && std::fabs(x) > kSfTrigGuarded) return true;
        if (std::isinf(r)) return false;
        const double d = std::fabs(r - e);
        if (err) *err = d;
        return d <= sf_abs_bound(fn, type, e);
    }
    const double ae = std::fabs(e), ar = std::fabs(r);
    if (ae * (1 - B) < sf_min_normal(type) && ar < sf_min_normal(type))
        return r == 0 || (!ftz && std::signbit(r) == std::signbit(e));
    if (std::signbit(r) != std::signbit(e)) return false;
    if (std::isinf(r)) return ae * (1 + B) > sf_max_finite(type);
    if (ftz && ar < sf_min_normal(type)) return false;
    const double d = std::fabs(ar - ae) / ae;
    if (err) *err = d;
    return d <= B;
}

// The guard over one thread's result words of one tile: the number of results that fail it, and the worst error per
// function (max with what worst[] holds).
inline int sf_guard_thread(int fmt, const uint32_t* ops, const uint32_t* words, double* worst = nullptr) {
    int bad = 0;
    for (int op = 0; op < kSfOps; ++op) {
        const SfOpInfo& I = kSfOp[op];
        if (I.fmt != fmt) continue;
        for (int v = 0; v < sf_values(op); ++v) {
            uint64_t x, r[2];
            int nr = 1;
            if (I.type == SF_T32) {
                x = ops[I.slot0 + v];
                r[0] = words[I.word0 + v];
                if (op == SF_SINCOS) { r[1] = words[I.word0 + kSfN + v]; nr = 2; }
            } else if (I.type == SF_T64) {
                x = (uint64_t)ops[I.slot0 + 2 * v + 1] << 32 | ops[I.slot0 + 2 * v];
                r[0] = (uint64_t)words[I.word0 + 2 * v + 1] << 32 | words[I.word0 + 2 * v];
            } else {
                x = (ops[I.slot0 + v / 2] >> (16 * (v % 2))) & 0xFFFFu;
                r[0] = (words[I.word0 + v / 2] >> (16 * (v % 2))) & 0xFFFFu;
            }
            for (int k = 0; k < nr; ++k) {
                const int fn = I.fn0 + k;
                double err = 0;
                if (!sf_guard(fn, I.type, I.ftz, x, r[k], &err)) ++bad;
                else if (worst && err > worst[fn * 3 + I.type]) worst[fn * 3 + I.type] = err;
            }
        }
    }
    return bad;
}

// ---- the fold -------------------------------------------------------------------------------------------------------
// sum_j (2j + 1) * w_j mod 2^32 over the thread's words: flipping bit b of one word changes it by +-(2j + 1) * 2^b,
// never a multiple of 2^32, so no single flipped bit of any one result leaves the value unchanged.
inline uint32_t sf_fold(const uint32_t* w, int n) {
    uint32_t h = 0;
    for (int j = 0; j < n; ++j) h += (2u * (uint32_t)j + 1u) * w[j];
    return h;
}

// ---- consensus over the reference launch --------------------------------------------------------------------------------
constexpr uint32_t kSfNoConsensus = 0x4u;  // B2DP_CT_NO_CONSENSUS in include/b200dp.h (cuda_backend.cu asserts it)
constexpr uint32_t kSfOutOfBound = 0x8u;   // B2DP_CT_OUT_OF_BOUND

struct SfConsensus {
    std::vector<uint32_t> words;          // [tile][thread][kSfWords[fmt]]: the majority (where none: the candidate)
    std::vector<uint32_t> check;          // [tile][thread]: sf_fold of the majority words, the timed launch's checks
    int ctas = 0, arrived = 0;            // reference CTAs launched / whose record arrived complete
    int sm_ids = 0;                       // distinct SM ids among them
    unsigned long long no_consensus = 0;  // words without a strict majority
    unsigned long long out_of_bound = 0;  // majority results that fail the guard
    unsigned long long dissents = 0;      // (CTA, tile) pairs in which a CTA differs from a majority word
    uint64_t bad_sm_mask[4] = {0, 0, 0, 0};
    int first_bad_sm = -1, first_bad_tile = -1;  // lowest dissenting SM id, and its CTA's first dissenting tile
    double worst[kSfFns * 3] = {};        // worst guarded error per [fn][type]
    uint32_t flags() const { return (no_consensus ? kSfNoConsensus : 0u) | (out_of_bound ? kSfOutOfBound : 0u); }
    // every record arrived, every word has a majority, no CTA dissents and every majority result passes the guard
    bool clean() const { return arrived == ctas && ctas > 0 && !no_consensus && !out_of_bound && !dissents; }
};

// dumps: [cta][tile][thread][W] result words of round 0, repetition 0; recs: one per CTA; table: kCtTiles operand
// tables of sf_table_bytes(fmt).  A CTA whose record is not complete (ct_record_complete) is left out of the vote.
inline void sf_consensus(int fmt, const uint32_t* dumps, const CtRecord* recs, int n_cta, unsigned long long seq,
                         const uint32_t* table, SfConsensus& out) {
    const int W = kSfWords[fmt];
    const size_t tile_words = (size_t)kCtThreads * W, per_cta = kCtTiles * tile_words;
    out = SfConsensus{};
    out.ctas = n_cta;
    out.words.assign(per_cta, 0);
    out.check.assign((size_t)kCtTiles * kCtThreads, 0);
    std::vector<int> in;
    std::vector<uint8_t> seen(kCtMaxSmId, 0);
    for (int c = 0; c < n_cta; ++c) {
        if (!ct_record_complete(recs[c], seq)) continue;
        in.push_back(c);
        if (recs[c].smid < (uint32_t)kCtMaxSmId && !seen[recs[c].smid]++) ++out.sm_ids;
    }
    out.arrived = (int)in.size();
    std::vector<uint32_t> cnt(tile_words);
    std::vector<uint8_t> has(tile_words);
    std::vector<int> first_bad(n_cta, -1);
    for (int tile = 0; tile < kCtTiles; ++tile) {
        uint32_t* cand = &out.words[tile * tile_words];
        std::fill(cnt.begin(), cnt.end(), 0u);
        for (int c : in) {  // Boyer-Moore majority vote, word by word
            const uint32_t* d = dumps + c * per_cta + tile * tile_words;
            for (size_t p = 0; p < tile_words; ++p) {
                if (cnt[p] == 0) { cand[p] = d[p]; cnt[p] = 1; }
                else cnt[p] += d[p] == cand[p] ? 1u : (uint32_t)-1;
            }
        }
        std::fill(cnt.begin(), cnt.end(), 0u);
        for (int c : in) {
            const uint32_t* d = dumps + c * per_cta + tile * tile_words;
            for (size_t p = 0; p < tile_words; ++p) cnt[p] += d[p] == cand[p];
        }
        for (size_t p = 0; p < tile_words; ++p) {
            has[p] = 2 * (size_t)cnt[p] > in.size();
            out.no_consensus += !has[p];
        }
        for (int c : in) {
            const uint32_t* d = dumps + c * per_cta + tile * tile_words;
            bool differs = false;
            for (size_t p = 0; p < tile_words && !differs; ++p) differs = has[p] && d[p] != cand[p];
            if (!differs) continue;
            ++out.dissents;
            if (first_bad[c] < 0) first_bad[c] = tile;
            const uint32_t s = recs[c].smid;
            if (s >= (uint32_t)kCtMaxSmId) continue;
            out.bad_sm_mask[s / 64] |= 1ull << (s % 64);
            if (out.first_bad_sm < 0 || (int)s < out.first_bad_sm) { out.first_bad_sm = (int)s; out.first_bad_tile = first_bad[c]; }
        }
        const uint32_t* tab = table + (size_t)tile * kSfSlots[fmt] * kCtThreads;
        uint32_t ops[kSfMaxWords];
        for (int t = 0; t < kCtThreads; ++t) {
            for (int s = 0; s < kSfSlots[fmt]; ++s) ops[s] = tab[(size_t)s * kCtThreads + t];
            const uint32_t* w = cand + (size_t)t * W;
            if (!in.empty()) out.out_of_bound += (unsigned)sf_guard_thread(fmt, ops, w, out.worst);
            out.check[tile * kCtThreads + t] = sf_fold(w, W);
        }
    }
}

}  // namespace b2dp
