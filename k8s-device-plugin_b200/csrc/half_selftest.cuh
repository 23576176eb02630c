// half_selftest.cuh -- sm_90a self-test kernel of the on-demand half-precision and conversion self-test (b2dp_half_test).
//
// Four warps per CTA run the SM's 16-bit floating-point pipes and its type converters on operands the host generated,
// and compare against results the host computed exactly (half_test_math.hpp).  Every op under test is one inline-PTX
// statement and runs on every operand set of its format (12 / 12 / 9 sets per thread):
//     format  PTX under test, per set                                                       result words per set
//     F16     fma.rn / .relu / .sat / .ftz, add.rn, sub.rn, mul.rn, min, max, min.NaN, max.NaN,
//             min.xorsign.abs, all .f16x2                                                    12
//     BF16    fma.rn / .relu, add.rn, sub.rn, mul.rn, min, max, min.NaN, max.NaN, all .bf16x2  9
//     CVT     f32 -> f16x2 / bf16x2 (rn, rz, rn.relu, rn.satfinite), f32 / f16x2 -> e4m3x2 / e5m2x2 (rn.satfinite),
//             e4m3x2 / e5m2x2 -> f16x2, f32 -> tf32 (rn), f32 -> f16 / bf16 (rm, rp), f32 -> s32 / u32 and
//             f64 -> s64 (rni, rzi, rmi, rpi), s32 -> f32, u64 -> f32, s64 -> f64 and f64 -> f32 (rn, rz, rm, rp),
//             rni.f32.f32, rmi.f64.f64                                                       58
// The results are independent -- no result feeds another op under test -- and every result word enters the thread's
// fold (the integer test's ItSink / it_fold) as it is produced.
//
// The round / tile / repetition structure, the operand perturbation v ^ (rep & zero), the __syncthreads_or verdict, the
// CtRecord, the fault hook (round 0, tile 0, repetition 0, result word 0 of thread 0 on the SM fault_sm) and the DUMP
// contract (CTA 0 writes every result word of repetition 0 of every tile of round 0 to dump[tile][thread][word]) are
// int_selftest's.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "half_test_math.hpp"
#include "int_selftest.cuh"  // ItSink, globaltimer_ns

namespace b2dp {

#define B2DP_HP_OP3(NAME, PTX)                                                             \
    __device__ __forceinline__ uint32_t NAME(uint32_t a, uint32_t b, uint32_t c) {         \
        uint32_t d;                                                                        \
        asm volatile(PTX " %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));           \
        return d;                                                                          \
    }
#define B2DP_HP_OP2(NAME, PTX)                                                             \
    __device__ __forceinline__ uint32_t NAME(uint32_t a, uint32_t b) {                     \
        uint32_t d;                                                                        \
        asm volatile(PTX " %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));                       \
        return d;                                                                          \
    }
#define B2DP_HP_OP1(NAME, PTX)                                                             \
    __device__ __forceinline__ uint32_t NAME(uint32_t a) {                                 \
        uint32_t d;                                                                        \
        asm volatile(PTX " %0, %1;" : "=r"(d) : "r"(a));                                   \
        return d;                                                                          \
    }
// 16-bit results (f16 / bf16 / a pair of fp8), zero-extended
#define B2DP_HP_TO16_2(NAME, PTX)                                                          \
    __device__ __forceinline__ uint32_t NAME(uint32_t a, uint32_t b) {                     \
        unsigned short d;                                                                  \
        asm volatile(PTX " %0, %1, %2;" : "=h"(d) : "r"(a), "r"(b));                       \
        return d;                                                                          \
    }
#define B2DP_HP_TO16_1(NAME, PTX)                                                          \
    __device__ __forceinline__ uint32_t NAME(uint32_t a) {                                 \
        unsigned short d;                                                                  \
        asm volatile(PTX " %0, %1;" : "=h"(d) : "r"(a));                                   \
        return d;                                                                          \
    }
#define B2DP_HP_FROM16(NAME, PTX)                                                          \
    __device__ __forceinline__ uint32_t NAME(uint32_t a) {                                 \
        uint32_t d;                                                                        \
        asm volatile(PTX " %0, %1;" : "=r"(d) : "h"((unsigned short)a));                   \
        return d;                                                                          \
    }
#define B2DP_HP_F64_TO32(NAME, PTX)                                                        \
    __device__ __forceinline__ uint32_t NAME(unsigned long long a) {                       \
        uint32_t d;                                                                        \
        asm volatile(PTX " %0, %1;" : "=r"(d) : "l"(a));                                   \
        return d;                                                                          \
    }
#define B2DP_HP_64_TO64(NAME, PTX)                                                         \
    __device__ __forceinline__ unsigned long long NAME(unsigned long long a) {             \
        unsigned long long d;                                                              \
        asm volatile(PTX " %0, %1;" : "=l"(d) : "l"(a));                                   \
        return d;                                                                          \
    }
B2DP_HP_OP3(hp_fma_f16, "fma.rn.f16x2")
B2DP_HP_OP3(hp_fma_relu_f16, "fma.rn.relu.f16x2")
B2DP_HP_OP3(hp_fma_sat_f16, "fma.rn.sat.f16x2")
B2DP_HP_OP3(hp_fma_ftz_f16, "fma.rn.ftz.f16x2")
B2DP_HP_OP2(hp_add_f16, "add.rn.f16x2")
B2DP_HP_OP2(hp_sub_f16, "sub.rn.f16x2")
B2DP_HP_OP2(hp_mul_f16, "mul.rn.f16x2")
B2DP_HP_OP2(hp_min_f16, "min.f16x2")
B2DP_HP_OP2(hp_max_f16, "max.f16x2")
B2DP_HP_OP2(hp_min_nan_f16, "min.NaN.f16x2")
B2DP_HP_OP2(hp_max_nan_f16, "max.NaN.f16x2")
B2DP_HP_OP2(hp_min_xorsign_f16, "min.xorsign.abs.f16x2")
B2DP_HP_OP3(hp_fma_bf16, "fma.rn.bf16x2")
B2DP_HP_OP3(hp_fma_relu_bf16, "fma.rn.relu.bf16x2")
B2DP_HP_OP2(hp_add_bf16, "add.rn.bf16x2")
B2DP_HP_OP2(hp_sub_bf16, "sub.rn.bf16x2")
B2DP_HP_OP2(hp_mul_bf16, "mul.rn.bf16x2")
B2DP_HP_OP2(hp_min_bf16, "min.bf16x2")
B2DP_HP_OP2(hp_max_bf16, "max.bf16x2")
B2DP_HP_OP2(hp_min_nan_bf16, "min.NaN.bf16x2")
B2DP_HP_OP2(hp_max_nan_bf16, "max.NaN.bf16x2")
B2DP_HP_OP2(hp_cvt_f16x2_rn, "cvt.rn.f16x2.f32")
B2DP_HP_OP2(hp_cvt_f16x2_rz, "cvt.rz.f16x2.f32")
B2DP_HP_OP2(hp_cvt_f16x2_relu, "cvt.rn.relu.f16x2.f32")
B2DP_HP_OP2(hp_cvt_f16x2_satf, "cvt.rn.satfinite.f16x2.f32")
B2DP_HP_OP2(hp_cvt_bf16x2_rn, "cvt.rn.bf16x2.f32")
B2DP_HP_OP2(hp_cvt_bf16x2_rz, "cvt.rz.bf16x2.f32")
B2DP_HP_OP2(hp_cvt_bf16x2_relu, "cvt.rn.relu.bf16x2.f32")
B2DP_HP_OP2(hp_cvt_bf16x2_satf, "cvt.rn.satfinite.bf16x2.f32")
B2DP_HP_TO16_2(hp_cvt_e4m3_f32, "cvt.rn.satfinite.e4m3x2.f32")
B2DP_HP_TO16_2(hp_cvt_e5m2_f32, "cvt.rn.satfinite.e5m2x2.f32")
B2DP_HP_TO16_1(hp_cvt_e4m3_f16, "cvt.rn.satfinite.e4m3x2.f16x2")
B2DP_HP_TO16_1(hp_cvt_e5m2_f16, "cvt.rn.satfinite.e5m2x2.f16x2")
B2DP_HP_FROM16(hp_cvt_f16_e4m3, "cvt.rn.f16x2.e4m3x2")
B2DP_HP_FROM16(hp_cvt_f16_e5m2, "cvt.rn.f16x2.e5m2x2")
B2DP_HP_OP1(hp_cvt_tf32, "cvt.rn.tf32.f32")
B2DP_HP_TO16_1(hp_cvt_f16_rm, "cvt.rm.f16.f32")
B2DP_HP_TO16_1(hp_cvt_f16_rp, "cvt.rp.f16.f32")
B2DP_HP_TO16_1(hp_cvt_bf16_rm, "cvt.rm.bf16.f32")
B2DP_HP_TO16_1(hp_cvt_bf16_rp, "cvt.rp.bf16.f32")
B2DP_HP_OP1(hp_cvt_s32_rni, "cvt.rni.s32.f32")
B2DP_HP_OP1(hp_cvt_s32_rzi, "cvt.rzi.s32.f32")
B2DP_HP_OP1(hp_cvt_s32_rmi, "cvt.rmi.s32.f32")
B2DP_HP_OP1(hp_cvt_s32_rpi, "cvt.rpi.s32.f32")
B2DP_HP_OP1(hp_cvt_u32_rni, "cvt.rni.u32.f32")
B2DP_HP_OP1(hp_cvt_u32_rzi, "cvt.rzi.u32.f32")
B2DP_HP_OP1(hp_cvt_u32_rmi, "cvt.rmi.u32.f32")
B2DP_HP_OP1(hp_cvt_u32_rpi, "cvt.rpi.u32.f32")
B2DP_HP_64_TO64(hp_cvt_s64_rni, "cvt.rni.s64.f64")
B2DP_HP_64_TO64(hp_cvt_s64_rzi, "cvt.rzi.s64.f64")
B2DP_HP_64_TO64(hp_cvt_s64_rmi, "cvt.rmi.s64.f64")
B2DP_HP_64_TO64(hp_cvt_s64_rpi, "cvt.rpi.s64.f64")
B2DP_HP_OP1(hp_cvt_f32_s32_rn, "cvt.rn.f32.s32")
B2DP_HP_OP1(hp_cvt_f32_s32_rz, "cvt.rz.f32.s32")
B2DP_HP_OP1(hp_cvt_f32_s32_rm, "cvt.rm.f32.s32")
B2DP_HP_OP1(hp_cvt_f32_s32_rp, "cvt.rp.f32.s32")
B2DP_HP_F64_TO32(hp_cvt_f32_u64_rn, "cvt.rn.f32.u64")
B2DP_HP_F64_TO32(hp_cvt_f32_u64_rz, "cvt.rz.f32.u64")
B2DP_HP_F64_TO32(hp_cvt_f32_u64_rm, "cvt.rm.f32.u64")
B2DP_HP_F64_TO32(hp_cvt_f32_u64_rp, "cvt.rp.f32.u64")
B2DP_HP_64_TO64(hp_cvt_f64_s64_rn, "cvt.rn.f64.s64")
B2DP_HP_64_TO64(hp_cvt_f64_s64_rz, "cvt.rz.f64.s64")
B2DP_HP_64_TO64(hp_cvt_f64_s64_rm, "cvt.rm.f64.s64")
B2DP_HP_64_TO64(hp_cvt_f64_s64_rp, "cvt.rp.f64.s64")
B2DP_HP_F64_TO32(hp_cvt_f32_f64_rn, "cvt.rn.f32.f64")
B2DP_HP_F64_TO32(hp_cvt_f32_f64_rz, "cvt.rz.f32.f64")
B2DP_HP_F64_TO32(hp_cvt_f32_f64_rm, "cvt.rm.f32.f64")
B2DP_HP_F64_TO32(hp_cvt_f32_f64_rp, "cvt.rp.f32.f64")
B2DP_HP_OP1(hp_frnd_f32, "cvt.rni.f32.f32")
B2DP_HP_64_TO64(hp_frnd_f64, "cvt.rmi.f64.f64")
#undef B2DP_HP_OP1
#undef B2DP_HP_OP2
#undef B2DP_HP_OP3
#undef B2DP_HP_TO16_1
#undef B2DP_HP_TO16_2
#undef B2DP_HP_FROM16
#undef B2DP_HP_F64_TO32
#undef B2DP_HP_64_TO64

// Set S of format FMT on this repetition's operand words o[0 .. kHpSetSlots[FMT]), in half_test_math.hpp's word order.
template <int FMT, int S, bool DUMP>
__device__ __forceinline__ void hp_set(const uint32_t* o, ItSink<DUMP>& k) {
    constexpr int J = S * kHpSetWords[FMT];
    if constexpr (FMT == HP_F16) {
        const uint32_t a = o[HS_A], b = o[HS_B], c = o[HS_C], x = o[HS_X], y = o[HS_Y], z = o[HS_Z];
        k.template emit<J + HF_FMA>(hp_fma_f16(a, b, c));
        k.template emit<J + HF_FMA_RELU>(hp_fma_relu_f16(x, y, z));
        k.template emit<J + HF_FMA_SAT>(hp_fma_sat_f16(x, y, z));
        k.template emit<J + HF_FMA_FTZ>(hp_fma_ftz_f16(a, b, c));
        k.template emit<J + HF_ADD>(hp_add_f16(a, b));
        k.template emit<J + HF_SUB>(hp_sub_f16(a, b));
        k.template emit<J + HF_MUL>(hp_mul_f16(a, b));
        k.template emit<J + HF_MIN>(hp_min_f16(x, y));
        k.template emit<J + HF_MAX>(hp_max_f16(x, y));
        k.template emit<J + HF_MIN_NAN>(hp_min_nan_f16(x, y));
        k.template emit<J + HF_MAX_NAN>(hp_max_nan_f16(x, y));
        k.template emit<J + HF_MIN_XORSIGN>(hp_min_xorsign_f16(a, b));
    } else if constexpr (FMT == HP_BF16) {
        const uint32_t a = o[HS_A], b = o[HS_B], c = o[HS_C], x = o[HS_X], y = o[HS_Y], z = o[HS_Z];
        k.template emit<J + HB_FMA>(hp_fma_bf16(a, b, c));
        k.template emit<J + HB_FMA_RELU>(hp_fma_relu_bf16(x, y, z));
        k.template emit<J + HB_ADD>(hp_add_bf16(a, b));
        k.template emit<J + HB_SUB>(hp_sub_bf16(a, b));
        k.template emit<J + HB_MUL>(hp_mul_bf16(a, b));
        k.template emit<J + HB_MIN>(hp_min_bf16(x, y));
        k.template emit<J + HB_MAX>(hp_max_bf16(x, y));
        k.template emit<J + HB_MIN_NAN>(hp_min_nan_bf16(x, y));
        k.template emit<J + HB_MAX_NAN>(hp_max_nan_bf16(x, y));
    } else {
        const uint32_t X = o[HC_X], Y = o[HC_Y], P = o[HC_P], Q = o[HC_Q], F = o[HC_F], H = o[HC_H];
        const unsigned long long D = (unsigned long long)o[HC_DHI] << 32 | o[HC_DLO];
        const unsigned long long L = (unsigned long long)o[HC_LHI] << 32 | o[HC_LLO];
        unsigned long long r;
        k.template emit<J + HC_F16X2_RN>(hp_cvt_f16x2_rn(X, Y));
        k.template emit<J + HC_F16X2_RZ>(hp_cvt_f16x2_rz(X, Y));
        k.template emit<J + HC_F16X2_RELU>(hp_cvt_f16x2_relu(P, Q));
        k.template emit<J + HC_F16X2_SATF>(hp_cvt_f16x2_satf(P, Q));
        k.template emit<J + HC_BF16X2_RN>(hp_cvt_bf16x2_rn(X, Y));
        k.template emit<J + HC_BF16X2_RZ>(hp_cvt_bf16x2_rz(X, Y));
        k.template emit<J + HC_BF16X2_RELU>(hp_cvt_bf16x2_relu(P, Q));
        k.template emit<J + HC_BF16X2_SATF>(hp_cvt_bf16x2_satf(P, Q));
        k.template emit<J + HC_E4M3_F32>(hp_cvt_e4m3_f32(P, Q));
        k.template emit<J + HC_E5M2_F32>(hp_cvt_e5m2_f32(X, Y));
        k.template emit<J + HC_E4M3_F16>(hp_cvt_e4m3_f16(H));
        k.template emit<J + HC_E5M2_F16>(hp_cvt_e5m2_f16(H));
        k.template emit<J + HC_F16_E4M3>(hp_cvt_f16_e4m3(o[HC_E4]));
        k.template emit<J + HC_F16_E5M2>(hp_cvt_f16_e5m2(o[HC_E5]));
        k.template emit<J + HC_TF32>(hp_cvt_tf32(X));
        k.template emit<J + HC_F16_RM>(hp_cvt_f16_rm(X));
        k.template emit<J + HC_F16_RP>(hp_cvt_f16_rp(X));
        k.template emit<J + HC_BF16_RM>(hp_cvt_bf16_rm(X));
        k.template emit<J + HC_BF16_RP>(hp_cvt_bf16_rp(X));
        k.template emit<J + HC_S32 + 0>(hp_cvt_s32_rni(F));
        k.template emit<J + HC_S32 + 1>(hp_cvt_s32_rzi(F));
        k.template emit<J + HC_S32 + 2>(hp_cvt_s32_rmi(F));
        k.template emit<J + HC_S32 + 3>(hp_cvt_s32_rpi(F));
        k.template emit<J + HC_U32 + 0>(hp_cvt_u32_rni(F));
        k.template emit<J + HC_U32 + 1>(hp_cvt_u32_rzi(F));
        k.template emit<J + HC_U32 + 2>(hp_cvt_u32_rmi(F));
        k.template emit<J + HC_U32 + 3>(hp_cvt_u32_rpi(F));
        r = hp_cvt_s64_rni(D);
        k.template emit<J + HC_S64 + 0>((uint32_t)r);
        k.template emit<J + HC_S64 + 1>((uint32_t)(r >> 32));
        r = hp_cvt_s64_rzi(D);
        k.template emit<J + HC_S64 + 2>((uint32_t)r);
        k.template emit<J + HC_S64 + 3>((uint32_t)(r >> 32));
        r = hp_cvt_s64_rmi(D);
        k.template emit<J + HC_S64 + 4>((uint32_t)r);
        k.template emit<J + HC_S64 + 5>((uint32_t)(r >> 32));
        r = hp_cvt_s64_rpi(D);
        k.template emit<J + HC_S64 + 6>((uint32_t)r);
        k.template emit<J + HC_S64 + 7>((uint32_t)(r >> 32));
        k.template emit<J + HC_I2F_S32 + 0>(hp_cvt_f32_s32_rn(o[HC_I]));
        k.template emit<J + HC_I2F_S32 + 1>(hp_cvt_f32_s32_rz(o[HC_I]));
        k.template emit<J + HC_I2F_S32 + 2>(hp_cvt_f32_s32_rm(o[HC_I]));
        k.template emit<J + HC_I2F_S32 + 3>(hp_cvt_f32_s32_rp(o[HC_I]));
        k.template emit<J + HC_I2F_U64 + 0>(hp_cvt_f32_u64_rn(L));
        k.template emit<J + HC_I2F_U64 + 1>(hp_cvt_f32_u64_rz(L));
        k.template emit<J + HC_I2F_U64 + 2>(hp_cvt_f32_u64_rm(L));
        k.template emit<J + HC_I2F_U64 + 3>(hp_cvt_f32_u64_rp(L));
        r = hp_cvt_f64_s64_rn(L);
        k.template emit<J + HC_I2F_S64 + 0>((uint32_t)r);
        k.template emit<J + HC_I2F_S64 + 1>((uint32_t)(r >> 32));
        r = hp_cvt_f64_s64_rz(L);
        k.template emit<J + HC_I2F_S64 + 2>((uint32_t)r);
        k.template emit<J + HC_I2F_S64 + 3>((uint32_t)(r >> 32));
        r = hp_cvt_f64_s64_rm(L);
        k.template emit<J + HC_I2F_S64 + 4>((uint32_t)r);
        k.template emit<J + HC_I2F_S64 + 5>((uint32_t)(r >> 32));
        r = hp_cvt_f64_s64_rp(L);
        k.template emit<J + HC_I2F_S64 + 6>((uint32_t)r);
        k.template emit<J + HC_I2F_S64 + 7>((uint32_t)(r >> 32));
        k.template emit<J + HC_F32_F64 + 0>(hp_cvt_f32_f64_rn(D));
        k.template emit<J + HC_F32_F64 + 1>(hp_cvt_f32_f64_rz(D));
        k.template emit<J + HC_F32_F64 + 2>(hp_cvt_f32_f64_rm(D));
        k.template emit<J + HC_F32_F64 + 3>(hp_cvt_f32_f64_rp(D));
        k.template emit<J + HC_FRND_F32>(hp_frnd_f32(X));
        r = hp_frnd_f64(D);
        k.template emit<J + HC_FRND_F64>((uint32_t)r);
        k.template emit<J + HC_FRND_F64 + 1>((uint32_t)(r >> 32));
    }
}

template <int FMT, bool DUMP, int S = 0>
__device__ __forceinline__ void hp_sets(const uint32_t* w, ItSink<DUMP>& k) {
    if constexpr (S < kHpSets[FMT]) {
        constexpr int OFF = S * kHpSetSlots[FMT];
        hp_set<FMT, S, DUMP>(w + OFF, k);
        hp_sets<FMT, DUMP, S + 1>(w, k);
    }
}

// table: kCtTiles tables of hp_table_bytes(FMT) bytes; checks: [kCtTiles][kCtThreads]; rec: one per CTA.
// Block: kCtThreads threads, no dynamic shared memory.  Same signature as tc_selftest.
template <int FMT, bool DUMP>
__global__ void __launch_bounds__(kCtThreads)
half_selftest(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks, unsigned long long duration_ns,
              int fault_sm, uint32_t fault_mask, CtRecord* rec, unsigned long long seq, uint32_t* dump) {
    constexpr int SLOTS = kHpSlots[FMT];
    constexpr int W = kHpWords[FMT];
    const int tid = threadIdx.x;
    uint32_t smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned long long t_end = globaltimer_ns() + duration_ns;
    const uint32_t inj0 = (tid == 0 && (int)smid == fault_sm) ? fault_mask : 0u;
    // 0 at run time, but not provably so at compile time (int_selftest): no op leaves the repetition loop
    const uint32_t zero = smid < nsmid ? 0u : ~0u;
    uint32_t v[SLOTS], w[SLOTS];  // the tile's operand words; this repetition's
    unsigned long long rounds = 0, comparisons = 0, mismatches = 0;
    int bad_tile = -1, bad_rep = -1;
    for (;;) {
        for (int tile = 0; tile < kCtTiles; ++tile) {
            const uint32_t* tt = reinterpret_cast<const uint32_t*>(table) + (size_t)tile * SLOTS * kCtThreads + tid;
#pragma unroll
            for (int s = 0; s < SLOTS; ++s) v[s] = __ldg(tt + s * kCtThreads);
            const uint32_t want = __ldg(checks + tile * kCtThreads + tid);
            for (int rep = 0; rep < kCtReps; ++rep) {
#pragma unroll
                for (int s = 0; s < SLOTS; ++s) w[s] = v[s] ^ ((uint32_t)rep & zero);
                ItSink<DUMP> k;
                constexpr uint32_t i0 = kItFoldInit[0], i1 = kItFoldInit[1], i2 = kItFoldInit[2], i3 = kItFoldInit[3];
                k.h[0] = i0; k.h[1] = i1; k.h[2] = i2; k.h[3] = i3;
                k.inj = (rounds | (unsigned)tile | (unsigned)rep) == 0 ? inj0 : 0u;
                k.dump = (DUMP && blockIdx.x == 0 && rounds == 0 && rep == 0)
                             ? dump + ((size_t)tile * kCtThreads + tid) * W : nullptr;
                hp_sets<FMT, DUMP>(w, k);
                const int bad = __syncthreads_or(k.value() != want);
                ++comparisons;
                if (bad && mismatches++ == 0) { bad_tile = tile; bad_rep = rep; }
            }
        }
        ++rounds;
        if (__syncthreads_or(tid == 0 && globaltimer_ns() >= t_end)) break;
    }
    if (tid == 0) {
        volatile CtRecord* r = rec + blockIdx.x;
        r->smid = smid;
        r->nsmid = nsmid;
        r->rounds = rounds;
        r->comparisons = comparisons;
        r->mismatches = mismatches;
        r->first_bad_tile = bad_tile;
        r->first_bad_rep = bad_rep;
        __threadfence_system();
        r->seq = seq;
    }
}

}  // namespace b2dp
