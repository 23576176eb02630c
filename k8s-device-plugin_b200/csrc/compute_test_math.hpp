// compute_test_math.hpp -- host-side arithmetic of the on-demand tensor-core self-test (b2dp_compute_test,
// tc_selftest.cuh).
//
// Pure C++ (no CUDA), so the CPU tests compile it as it is (tests/native/compute_test_math_test.cpp) and compare it with
// the Python restatement in tests/compute_test_oracle.py:
//   - ct_operand / ct_scale_exp: seed, format, tile, operand  ->  the integer operand values (and the BF16 tile scale)
//   - ct_encode:                 an integer operand value      ->  its bf16 / e4m3 / s8 bits
//   - ct_reference:              the exact GEMM in int64, scaled and encoded to FP32 / s32 bits
//   - ct_fold / ct_thread_check: the per-thread comparison value, in the kernel's accumulator-fragment order
//   - ct_build_tile:             the shared-memory image of a tile the kernel copies verbatim, and its check values
//   - compute_test_healthy:      the verdict
//
// Why the host can predict the device's result bit for bit: every operand is an integer, or an integer times a power
// of two shared by the whole tile, so every partial sum of a result element is an integer times that power of two,
// and its magnitude stays below the bounds asserted here.  FP32 represents such a value exactly as long as the
// accumulator keeps that many bits, whatever the order of accumulation or the alignment of the addends.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace b2dp {

enum CtFormat { CT_BF16 = 0, CT_FP8 = 1, CT_INT8 = 2 };
constexpr int kCtFormats = 3;

constexpr int kCtM = 64, kCtN = 128;            // one warpgroup's wgmma result tile, m64n128
constexpr int kCtThreads = 128;                 // one warpgroup per CTA
constexpr int kCtAcc = kCtM * kCtN / kCtThreads;  // accumulator registers per thread (64)
constexpr int kCtTiles = 8;                     // distinct operand tiles per format
constexpr int kCtReps = 16;                     // each tile runs this many times per round; every repetition is compared
constexpr int kCtKStepBytes = 32;               // K bytes of one wgmma: k16 of bf16, k32 of e4m3 / s8
constexpr int kCtMaxSmId = 256;                 // per-SM tallies are sized for %nsmid <= 256

// Operand ranges and K per result tile.  "Worst case" is the largest |partial sum| of a result element.
constexpr int kCtBf16Max = 255;                 // integers in [-255, 255]: every significand bit of bf16
constexpr int kCtBf16K = 256;
constexpr int kCtBf16ScaleExp = 30;             // each BF16 tile's A and B are scaled by 2^a, 2^b with |a|, |b| <= 30
constexpr int kCtFp8Max = 15;                   // integers in [-15, 15]: the whole 4-bit significand of e4m3
constexpr int kCtFp8K = 32;
constexpr int kCtInt8Min = -128, kCtInt8Max = 127;
constexpr int kCtInt8K = 256;
static_assert((long long)kCtBf16K * kCtBf16Max * kCtBf16Max < (1ll << 24),
              "BF16 partial sums must fit the 24 bits an FP32 accumulator keeps");
static_assert(2 * kCtBf16ScaleExp + 24 < 127 && -2 * kCtBf16ScaleExp > -126,
              "a scaled BF16 result must stay a normal FP32 number");
static_assert(kCtFp8K * kCtFp8Max * kCtFp8Max < (1 << 13),
              "FP8 partial sums must fit the 14 bits publicly reported for Hopper's FP8 accumulator");
static_assert((long long)kCtInt8K * kCtInt8Min * kCtInt8Min <= (1ll << 22), "INT8 sums stay far inside s32");

inline int ct_k(int fmt) { return fmt == CT_BF16 ? kCtBf16K : fmt == CT_FP8 ? kCtFp8K : kCtInt8K; }
inline int ct_lo(int fmt) { return fmt == CT_BF16 ? -kCtBf16Max : fmt == CT_FP8 ? -kCtFp8Max : kCtInt8Min; }
inline int ct_hi(int fmt) { return fmt == CT_BF16 ? kCtBf16Max : fmt == CT_FP8 ? kCtFp8Max : kCtInt8Max; }
inline int ct_elem_bytes(int fmt) { return fmt == CT_BF16 ? 2 : 1; }
inline int ct_rows(int op) { return op ? kCtN : kCtM; }  // op 0 = A (M x K), op 1 = B (N x K); both K-major
inline uint32_t ct_operand_bytes(int fmt, int op) { return (uint32_t)(ct_rows(op) * ct_k(fmt) * ct_elem_bytes(fmt)); }
inline uint32_t ct_image_bytes(int fmt) { return ct_operand_bytes(fmt, 0) + ct_operand_bytes(fmt, 1); }
// Multiply-adds of one compared result tile (2 * this = its algorithmic FLOPs, or integer ops for INT8).
inline double ct_macs_per_tile(int fmt) { return (double)kCtM * kCtN * ct_k(fmt); }

// ---- operand generator ------------------------------------------------------------------------------------------
inline uint32_t ct_mix(uint32_t x) {  // a 32-bit integer hash with good avalanche
    x ^= x >> 16;
    x *= 0x7FEB352Du;
    x ^= x >> 15;
    x *= 0x846CA68Bu;
    x ^= x >> 16;
    return x;
}
inline uint32_t ct_stream_key(uint32_t seed, int fmt, int tile, int op) {
    return ct_mix(seed ^ (uint32_t)(((fmt * 16 + tile) * 2 + op) + 1) * 0x9E3779B9u);
}
inline uint32_t ct_hash(uint32_t key, uint32_t i) { return ct_mix(key + ct_mix(i)); }
inline int ct_uniform(uint32_t h, int lo, int hi) {
    return lo + (int)(((uint64_t)h * (uint64_t)(hi - lo + 1)) >> 32);
}

// The power-of-two exponent of a tile's operand (BF16 only; 0 for FP8 and INT8), uniform in [-30, 30].
inline int ct_scale_exp(uint32_t seed, int fmt, int tile, int op) {
    if (fmt != CT_BF16) return 0;
    return ct_uniform(ct_hash(ct_stream_key(seed, fmt, tile, op), 0xFFFFFFFFu), -kCtBf16ScaleExp, kCtBf16ScaleExp);
}

// Integer operand values, row-major rows x K.  Random in [lo, hi], except that row 0 of A and rows 0..7 of B hold
// the extreme value lo everywhere but (for B row n) at k = n: row 0 of the result then sums K - 1 products lo^2 plus
// one random one, which takes those sums to at least (K - 2) / K of the worst case (above 2^23.9 for BF16) and
// exercises every accumulator bit below the bound.
inline std::vector<int> ct_operand(uint32_t seed, int fmt, int tile, int op) {
    const int rows = ct_rows(op), K = ct_k(fmt), lo = ct_lo(fmt), hi = ct_hi(fmt);
    const uint32_t key = ct_stream_key(seed, fmt, tile, op);
    std::vector<int> v((size_t)rows * K);
    for (int r = 0; r < rows; ++r)
        for (int k = 0; k < K; ++k) {
            const uint32_t i = (uint32_t)(r * K + k);
            const bool extreme = op == 0 ? r == 0 : (r < 8 && k != r);
            v[i] = extreme ? lo : ct_uniform(ct_hash(key, i), lo, hi);
        }
    return v;
}

inline uint32_t ct_f32_bits(float f) {
    uint32_t u;
    std::memcpy(&u, &f, 4);
    return u;
}

// The bits of integer operand value v (times 2^e for BF16): bf16 = the top half of the exact FP32 value; e4m3 = sign,
// 4-bit exponent (bias 7), 3-bit mantissa; s8 = two's complement.  Every value in range is represented exactly.
inline uint32_t ct_encode(int fmt, int v, int e) {
    if (fmt == CT_BF16) return ct_f32_bits(std::ldexp((float)v, e)) >> 16;
    if (fmt == CT_INT8) return (uint32_t)(uint8_t)(int8_t)v;
    const uint32_t sign = v < 0 ? 0x80u : 0u;
    const uint32_t a = (uint32_t)(v < 0 ? -v : v);
    if (a == 0) return 0;
    int ex = 0;
    while ((a >> (ex + 1)) != 0) ++ex;  // floor(log2 a)
    return sign | (uint32_t)(ex + 7) << 3 | (((a << 3) >> ex) & 7u);
}

// ---- the exact GEMM -----------------------------------------------------------------------------------------------
// D[m][n] = sum_k A[m][k] * B[n][k] in int64, times 2^(ea + eb); returned as FP32 bits (BF16, FP8) or s32 bits (INT8),
// row-major M x N.  An exact zero is +0.
inline std::vector<uint32_t> ct_reference(int fmt, const std::vector<int>& A, const std::vector<int>& B, int ea, int eb) {
    const int K = ct_k(fmt);
    std::vector<uint32_t> d((size_t)kCtM * kCtN);
    for (int m = 0; m < kCtM; ++m)
        for (int n = 0; n < kCtN; ++n) {
            long long s = 0;
            for (int k = 0; k < K; ++k) s += (long long)A[(size_t)m * K + k] * B[(size_t)n * K + k];
            d[(size_t)m * kCtN + n] = fmt == CT_INT8 ? (uint32_t)(int32_t)s
                                      : s == 0     ? 0u
                                                   : ct_f32_bits(std::ldexp((float)s, ea + eb));
        }
    return d;
}

// ---- accumulator fragments and the comparison value ---------------------------------------------------------------
// Register j of thread t of the warpgroup holds D[ct_frag_row(t, j)][ct_frag_col(t, j)] after a wgmma m64nNk*
// (PTX ISA, "wgmma ... register fragment of the accumulator D").
inline int ct_frag_row(int t, int j) { return 16 * (t / 32) + (t % 32) / 4 + 8 * ((j / 2) % 2); }
inline int ct_frag_col(int t, int j) { return 8 * (j / 4) + 2 * (t % 4) + (j % 2); }

// sum_j (2j + 1) * x_j mod 2^32.  Flipping bit b of one element x_j changes the sum by +-(2j + 1) * 2^b mod 2^32, and
// an odd number times 2^b with b < 32 is never a multiple of 2^32: no single-bit error in any one element can leave the
// value unchanged.  (A 32-bit sum is one IMAD per element in the kernel; a 64-bit one would catch no more of them.)
inline uint32_t ct_fold(const uint32_t* x) {
    uint32_t h = 0;
    for (int j = 0; j < kCtAcc; ++j) h += (2u * (uint32_t)j + 1u) * x[j];
    return h;
}
inline uint32_t ct_thread_check(const std::vector<uint32_t>& d, int t) {
    uint32_t x[kCtAcc];
    for (int j = 0; j < kCtAcc; ++j) x[j] = d[(size_t)ct_frag_row(t, j) * kCtN + ct_frag_col(t, j)];
    return ct_fold(x);
}

// ---- the shared-memory image ----------------------------------------------------------------------------------------
// Both operands are K-major without swizzle, in the wgmma "core matrix" layout: 8 rows x 16 bytes stored as 128
// contiguous bytes.  For each wgmma of a tile (K step s, 32 bytes of K) the operand's block is rows x 32 bytes; in it
// the core matrix of row group g and K half c starts at g * 256 + c * 128.  So the descriptors carry LBO = 128 (next
// core matrix along K), SBO = 256 (next 8 rows), and advance by rows * 32 bytes per K step.
inline size_t ct_image_offset(int rows, int r, int kb) {
    return (size_t)(kb / kCtKStepBytes) * rows * kCtKStepBytes + (size_t)(r / 8) * 256 + (size_t)((kb % 32) / 16) * 128 +
           (size_t)(r % 8) * 16 + (size_t)(kb % 16);
}

struct CtTile {
    std::vector<uint8_t> image;         // A then B, ct_image_bytes(fmt) bytes, copied verbatim into shared memory
    uint32_t check[kCtThreads];         // per-thread comparison values of the exact result
    std::vector<uint32_t> reference;    // the exact result bits, row-major M x N
};

inline void ct_build_tile(uint32_t seed, int fmt, int tile, CtTile& out) {
    const int K = ct_k(fmt), eb = ct_elem_bytes(fmt);
    out.image.assign(ct_image_bytes(fmt), 0);
    std::vector<int> v[2];
    int ex[2];
    for (int op = 0; op < 2; ++op) {
        v[op] = ct_operand(seed, fmt, tile, op);
        ex[op] = ct_scale_exp(seed, fmt, tile, op);
        const int rows = ct_rows(op);
        uint8_t* base = out.image.data() + (op ? ct_operand_bytes(fmt, 0) : 0);
        for (int r = 0; r < rows; ++r)
            for (int k = 0; k < K; ++k) {
                const uint32_t bits = ct_encode(fmt, v[op][(size_t)r * K + k], ex[op]);
                const size_t o = ct_image_offset(rows, r, k * eb);
                base[o] = (uint8_t)bits;
                if (eb == 2) base[o + 1] = (uint8_t)(bits >> 8);  // little-endian bf16
            }
    }
    out.reference = ct_reference(fmt, v[0], v[1], ex[0], ex[1]);
    for (int t = 0; t < kCtThreads; ++t) out.check[t] = ct_thread_check(out.reference, t);
}

// ---- per-CTA record and verdict -----------------------------------------------------------------------------------
// Written by each CTA's thread 0 into pinned, device-mapped host memory when the CTA ends; seq last.
struct CtRecord {
    uint32_t smid, nsmid;               // %smid and %nsmid of the SM the CTA ran on
    unsigned long long rounds;          // rounds completed (each runs every tile kCtReps times)
    unsigned long long comparisons;     // (tile, repetition) results compared: rounds * kCtTiles * kCtReps
    unsigned long long mismatches;      // comparisons in which any thread's value differed from the host's
    int32_t first_bad_tile, first_bad_rep;  // of the first mismatching comparison; -1 if none
    unsigned long long seq;             // the launch's sequence number, written last
};
static_assert(sizeof(CtRecord) == 48, "CtRecord is shared by the kernel and the host");

// A CTA record is complete iff it arrived (seq), did at least one round and compared exactly what those rounds hold.
inline bool ct_record_complete(const CtRecord& r, unsigned long long seq) {
    return r.seq == seq && r.rounds >= 1 && r.comparisons == r.rounds * (unsigned long long)(kCtTiles * kCtReps);
}

// Healthy iff every launch succeeded before the deadline, and in every format every CTA's record is complete and has
// no mismatch.  Covering fewer SM ids than the device has is reported, not failed.
inline bool compute_test_healthy(bool launch_ok, const std::vector<CtRecord> (&recs)[kCtFormats],
                                 const unsigned long long (&seq)[kCtFormats]) {
    if (!launch_ok) return false;
    for (int f = 0; f < kCtFormats; ++f) {
        if (recs[f].empty()) return false;
        for (const CtRecord& r : recs[f])
            if (!ct_record_complete(r, seq[f]) || r.mismatches != 0) return false;
    }
    return true;
}

}  // namespace b2dp
