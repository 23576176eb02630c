// sfu_selftest.cuh -- sm_90a self-test kernel of the on-demand SFU self-test (b2dp_sfu_test).
//
// Four warps per CTA run the special-function unit (MUFU) on operands the host generated (sfu_test_math.hpp).  Every
// checked result is the output of one MUFU instruction (the .ftz forms; without .ftz, ex2 and lg2 gain scaling code):
//     format  PTX -> SASS                                                                per thread and repetition
//     F32     ex2 / lg2 .approx.ftz.f32 -> MUFU.EX2 / MUFU.LG2                           16 each
//             sin / cos .approx.ftz.f32 -> one FMUL.RZ by 1/(2 pi), MUFU.SIN / MUFU.COS  16 operands, 16 each
//             tanh.approx.f32 -> MUFU.TANH                                               16
//     ROOT    rcp / rsqrt / sqrt .approx.ftz.f32 -> MUFU.RCP / MUFU.RSQ / MUFU.SQRT      16 each
//             rcp / rsqrt .approx.ftz.f64 -> MUFU.RCP64H / MUFU.RSQ64H                   16 each
//     F16     ex2 / tanh .approx.f16x2 -> two MUFU.EX2.F16 / MUFU.TANH.F16 per pair      16 pairs each
// The results are independent -- no chains, because a later op would hide an earlier wrong bit -- and every result
// word enters the thread's odd-weighted fold as soon as it is produced.
//
// The round / tile / repetition structure is tc_selftest's and fp_selftest's: a round runs each of the kCtTiles tiles
// kCtReps times, and a CTA repeats rounds until its %globaltimer deadline (at least one round).  Per tile every thread
// loads its operands from an L2-resident table ([slot][thread] words) into registers, and its comparison value; each
// repetition feeds the MUFU ops operands the compiler must treat as changed (sf_perturb), so no op leaves the
// repetition loop.  Every thread then compares its fold (sf_fold) with the host's; the CTA counts the repetition as one mismatch if any thread disagrees, and publishes one
// CtRecord.
//
// The host cannot compute MUFU's results, so the checks come from the device: the DUMP instantiation (the reference
// launch, one CTA on every SM) makes every CTA write every result word of round 0, repetition 0 of every tile to
// dump + blockIdx.x * kCtTiles * kCtThreads * kSfWords[FMT], as [tile][thread][word].  Launched with checks = nullptr
// it compares nothing (its records still count the repetitions).  The host takes each word's majority over the SMs,
// names every SM that disagrees, and folds the majority into the checks of the timed launch (sf_consensus).
//
// Test hook: as tc_selftest -- in round 0, thread 0 of a CTA whose %smid == fault_sm XORs fault_mask into its first
// result word of tile 0, repetition 0, before the fold (and before the dump).
#pragma once
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "hbm_probe.cuh"  // globaltimer_ns
#include "sfu_test_math.hpp"

namespace b2dp {

// The operand words of one repetition: v XOR (rep & zero), where zero is 0 at run time but not provably so at compile
// time (%smid < %nsmid, PTX ISA "Special registers").  An empty asm statement is not enough: it leaves no trace in the
// PTX, and ptxas then hoists the MUFU ops of loop-invariant operands out of the repetition loop.  One LOP3 per word.
__device__ __forceinline__ uint32_t sf_perturb(uint32_t v, int rep, uint32_t zero) { return v ^ ((uint32_t)rep & zero); }

#define B2DP_SF_F32_OP(NAME, PTX)                                              \
    __device__ __forceinline__ uint32_t NAME(uint32_t x) {                     \
        float r;                                                               \
        asm volatile(PTX " %0, %1;" : "=f"(r) : "f"(__uint_as_float(x)));      \
        return __float_as_uint(r);                                             \
    }
B2DP_SF_F32_OP(sf_ex2, "ex2.approx.ftz.f32")
B2DP_SF_F32_OP(sf_lg2, "lg2.approx.ftz.f32")
B2DP_SF_F32_OP(sf_sin, "sin.approx.ftz.f32")
B2DP_SF_F32_OP(sf_cos, "cos.approx.ftz.f32")
B2DP_SF_F32_OP(sf_tanh, "tanh.approx.f32")
B2DP_SF_F32_OP(sf_rcp, "rcp.approx.ftz.f32")
B2DP_SF_F32_OP(sf_rsq, "rsqrt.approx.ftz.f32")
B2DP_SF_F32_OP(sf_sqrt, "sqrt.approx.ftz.f32")
#undef B2DP_SF_F32_OP

__device__ __forceinline__ double sf_rcp64(double x) {
    double r;
    asm volatile("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    return r;
}
__device__ __forceinline__ double sf_rsq64(double x) {
    double r;
    asm volatile("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    return r;
}
__device__ __forceinline__ uint32_t sf_ex2h(uint32_t x) {
    uint32_t r;
    asm volatile("ex2.approx.f16x2 %0, %1;" : "=r"(r) : "r"(x));
    return r;
}
__device__ __forceinline__ uint32_t sf_tanhh(uint32_t x) {
    uint32_t r;
    asm volatile("tanh.approx.f16x2 %0, %1;" : "=r"(r) : "r"(x));
    return r;
}

// Result word j: the fault hook on word 0, the dump, and the fold.
template <bool DUMP>
__device__ __forceinline__ void sf_emit(uint32_t& h, int j, uint32_t w, uint32_t inj, uint32_t* dump) {
    if (j == 0) w ^= inj;
    if (DUMP && dump) dump[j] = w;
    h += (2u * (uint32_t)j + 1u) * w;
}

// One repetition of format FMT on the thread's operand words v: the fold of every result word, in sfu_test_math.hpp's
// word order (kSfOp[].word0).
template <int FMT, bool DUMP>
__device__ __forceinline__ uint32_t sf_rep(const uint32_t (&v)[kSfSlots[FMT]], uint32_t inj, uint32_t* dump) {
    uint32_t h = 0;
    if constexpr (FMT == SF_F32) {
#pragma unroll
        for (int i = 0; i < kSfN; ++i) sf_emit<DUMP>(h, i, sf_ex2(v[i]), inj, dump);
#pragma unroll
        for (int i = 0; i < kSfN; ++i) sf_emit<DUMP>(h, 16 + i, sf_lg2(v[16 + i]), inj, dump);
#pragma unroll
        for (int i = 0; i < kSfN; ++i) {
            sf_emit<DUMP>(h, 32 + i, sf_sin(v[32 + i]), inj, dump);
            sf_emit<DUMP>(h, 48 + i, sf_cos(v[32 + i]), inj, dump);
        }
#pragma unroll
        for (int i = 0; i < kSfN; ++i) sf_emit<DUMP>(h, 64 + i, sf_tanh(v[48 + i]), inj, dump);
    } else if constexpr (FMT == SF_ROOT) {
#pragma unroll
        for (int i = 0; i < kSfN; ++i) sf_emit<DUMP>(h, i, sf_rcp(v[i]), inj, dump);
#pragma unroll
        for (int i = 0; i < kSfN; ++i) sf_emit<DUMP>(h, 16 + i, sf_rsq(v[16 + i]), inj, dump);
#pragma unroll
        for (int i = 0; i < kSfN; ++i) sf_emit<DUMP>(h, 32 + i, sf_sqrt(v[32 + i]), inj, dump);
#pragma unroll
        for (int i = 0; i < kSfN; ++i) {
            const double r = sf_rcp64(__hiloint2double((int)v[49 + 2 * i], (int)v[48 + 2 * i]));
            sf_emit<DUMP>(h, 48 + 2 * i, (uint32_t)__double2loint(r), inj, dump);
            sf_emit<DUMP>(h, 49 + 2 * i, (uint32_t)__double2hiint(r), inj, dump);
        }
#pragma unroll
        for (int i = 0; i < kSfN; ++i) {
            const double r = sf_rsq64(__hiloint2double((int)v[81 + 2 * i], (int)v[80 + 2 * i]));
            sf_emit<DUMP>(h, 80 + 2 * i, (uint32_t)__double2loint(r), inj, dump);
            sf_emit<DUMP>(h, 81 + 2 * i, (uint32_t)__double2hiint(r), inj, dump);
        }
    } else {
#pragma unroll
        for (int i = 0; i < kSfN; ++i) sf_emit<DUMP>(h, i, sf_ex2h(v[i]), inj, dump);
#pragma unroll
        for (int i = 0; i < kSfN; ++i) sf_emit<DUMP>(h, 16 + i, sf_tanhh(v[16 + i]), inj, dump);
    }
    return h;
}

// table: kCtTiles tables of sf_table_bytes(FMT) bytes; checks: [kCtTiles][kCtThreads] (DUMP: may be null); rec: one
// per CTA.  Block: kCtThreads threads; the reference launch adds dynamic shared memory it does not use, so that one
// CTA runs per SM.  Same signature as tc_selftest.
template <int FMT, bool DUMP>
__global__ void __launch_bounds__(kCtThreads, 1)
sfu_selftest(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks, unsigned long long duration_ns,
             int fault_sm, uint32_t fault_mask, CtRecord* rec, unsigned long long seq, uint32_t* dump) {
    constexpr int SLOTS = kSfSlots[FMT];
    constexpr int W = kSfWords[FMT];
    const int tid = threadIdx.x;
    uint32_t smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned long long t_end = globaltimer_ns() + duration_ns;
    const uint32_t inj0 = (tid == 0 && (int)smid == fault_sm) ? fault_mask : 0u;
    const bool compare = !DUMP || checks != nullptr;
    const uint32_t zero = smid < nsmid ? 0u : ~0u;
    uint32_t v[SLOTS], w[SLOTS];  // the tile's operand words; this repetition's
    unsigned long long rounds = 0, comparisons = 0, mismatches = 0;
    int bad_tile = -1, bad_rep = -1;
    for (;;) {
        for (int tile = 0; tile < kCtTiles; ++tile) {
            const uint32_t* tt = reinterpret_cast<const uint32_t*>(table) + (size_t)tile * SLOTS * kCtThreads + tid;
#pragma unroll
            for (int s = 0; s < SLOTS; ++s) v[s] = __ldg(tt + s * kCtThreads);
            const uint32_t want = compare ? __ldg(checks + tile * kCtThreads + tid) : 0u;
            for (int rep = 0; rep < kCtReps; ++rep) {
#pragma unroll
                for (int s = 0; s < SLOTS; ++s) w[s] = sf_perturb(v[s], rep, zero);
                const uint32_t inj = (rounds | (unsigned)tile | (unsigned)rep) == 0 ? inj0 : 0u;
                uint32_t* dp = (DUMP && rounds == 0 && rep == 0)
                                   ? dump + ((size_t)blockIdx.x * kCtTiles * kCtThreads + (size_t)tile * kCtThreads + tid) * W
                                   : nullptr;
                const uint32_t h = sf_rep<FMT, DUMP>(w, inj, dp);
                const int bad = __syncthreads_or(compare && h != want);
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
