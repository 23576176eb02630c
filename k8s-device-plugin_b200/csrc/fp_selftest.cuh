// fp_selftest.cuh -- sm_90a FP32 / FP64 self-test kernel of the on-demand FP test (b2dp_fp_test).
//
// Four warps per CTA check the SMs' FMA units and FP64 tensor cores against values the host computed exactly
// (fp_test_math.hpp):
//     format  instruction (PTX -> SASS)                                     per thread and repetition
//     FP32    fma.rn.f32 -> FFMA (no .FTZ)                                  128 independent FMAs
//     FP64    fma.rn.f64 -> DFMA                                            128 independent FMAs
//     DMMA    mma.sync.aligned.m16n8k16.row.col.f64 -> DMMA.16x8x16       4 accumulator sets x 4 K steps (per warp)
// The round / tile / repetition structure is tc_selftest's: a round runs each of the kCtTiles tiles kCtReps times, and a
// CTA repeats rounds until its %globaltimer deadline (at least one round).  Per tile every thread loads its operands
// from an L2-resident table ([slot][thread], ft_build_tile) into registers, and its comparison value.  Per repetition:
//   - FP32 / FP64: every r = fma(x_i, a_k, b_k) enters the thread's weighted fold as soon as it is computed.  The FMAs
//     are independent on purpose: the last value of a dependent chain x <- fma(x, a, b) loses most single-bit errors
//     of its intermediate results (tests/test_fp_test_cpu.py keeps that experiment), so every result is compared.
//   - DMMA: partial sums are exact integers, so a chain over K loses nothing; each set's accumulators start at +0 and
//     are folded after the last K step.
// Every thread then compares its fold (ft_fold) with the host's; the CTA counts the repetition as one mismatch if any
// thread disagrees, and publishes one CtRecord like tc_selftest.
//
// The FMAs are inline PTX, so nvcc can neither contract nor reorder them, and each repetition starts from operands the
// compiler must treat as changed (ft_opaque), so none of the identical work is hoisted out of the repetition loop.
//
// Test hooks: as tc_selftest -- in round 0, thread 0 of a CTA whose %smid == fault_sm XORs fault_mask into its first
// result word of tile 0, repetition 0, before the fold.  DUMP (instantiated only by tests/native/fp_test_kernels.cu)
// makes CTA 0 write every result word of repetition 0 of every tile of round 0 to dump[tile][thread][kFtWords[FMT]].
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "fp_test_math.hpp"
#include "hbm_probe.cuh"  // globaltimer_ns

namespace b2dp {

// v, unchanged, through an instruction the compiler cannot see into (keeps loop-invariant work inside the loop)
__device__ __forceinline__ float ft_opaque(float v) { asm volatile("" : "+f"(v)); return v; }
__device__ __forceinline__ double ft_opaque(double v) { asm volatile("" : "+d"(v)); return v; }

__device__ __forceinline__ float ft_fma_dev(float x, float a, float b) {
    float r;
    asm volatile("fma.rn.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(x), "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ double ft_fma_dev(double x, double a, double b) {
    double r;
    asm volatile("fma.rn.f64 %0, %1, %2, %3;" : "=d"(r) : "d"(x), "d"(a), "d"(b));
    return r;
}

__device__ __forceinline__ void ft_dmma(double (&d)[kFtDmmaD], const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, "
                 "%11}, {%12, %13, %14, %15}, {%0, %1, %2, %3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]),
                   "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

__device__ __forceinline__ void ft_words(float r, uint32_t* w) { w[0] = __float_as_uint(r); }
__device__ __forceinline__ void ft_words(double r, uint32_t* w) {
    w[0] = (uint32_t)__double2loint(r);
    w[1] = (uint32_t)__double2hiint(r);
}

// One repetition of FP32 / FP64: the fold of every result (result j's words at j * NW ..).
template <typename T, bool DUMP>
__device__ __forceinline__ uint32_t ft_fma_rep(const T (&x)[kFtX], const T (&a)[kFtAB], const T (&b)[kFtAB],
                                               uint32_t inj, uint32_t* dump) {
    constexpr int NW = sizeof(T) / 4;
    uint32_t h = 0;
#pragma unroll
    for (int k = 0; k < kFtAB; ++k) {
#pragma unroll
        for (int i = 0; i < kFtX; ++i) {
            const int j = k * kFtX + i;
            uint32_t w[NW];
            ft_words(ft_fma_dev(x[i], a[k], b[k]), w);
            if (j == 0) w[0] ^= inj;
            if (DUMP && dump) {
#pragma unroll
                for (int q = 0; q < NW; ++q) dump[j * NW + q] = w[q];
            }
#pragma unroll
            for (int q = 0; q < NW; ++q) h += (2u * (uint32_t)(j * NW + q) + 1u) * w[q];
        }
    }
    return h;
}

// table: kCtTiles tables of ft_table_bytes(FMT) bytes; checks: [kCtTiles][kCtThreads]; rec: one per CTA.
// Block: kCtThreads threads, no dynamic shared memory.  Same signature as tc_selftest.  DUMP runs one CTA, so it may
// use every register (without the hint ptxas spills the DMMA DUMP at 128 registers).
template <int FMT, bool DUMP>
__global__ void __launch_bounds__(kCtThreads, DUMP ? 1 : 0)
fp_selftest(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks, unsigned long long duration_ns,
            int fault_sm, uint32_t fault_mask, CtRecord* rec, unsigned long long seq, uint32_t* dump) {
    using T = typename std::conditional<FMT == FT_FP32, float, double>::type;
    constexpr int SLOTS = FMT == FT_DMMA ? kFtDmmaSlots : kFtSlots;
    constexpr int W = kFtWords[FMT];
    const int tid = threadIdx.x;
    uint32_t smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned long long t_end = globaltimer_ns() + duration_ns;
    const uint32_t inj0 = (tid == 0 && (int)smid == fault_sm) ? fault_mask : 0u;
    T v[SLOTS];  // x, a, b (FP32 / FP64) or A_0..3, B_0..3 fragments (DMMA)
    unsigned long long rounds = 0, comparisons = 0, mismatches = 0;
    int bad_tile = -1, bad_rep = -1;
    for (;;) {
        for (int tile = 0; tile < kCtTiles; ++tile) {
            const T* tt = reinterpret_cast<const T*>(table) + (size_t)tile * SLOTS * kCtThreads + tid;
#pragma unroll
            for (int s = 0; s < SLOTS; ++s) v[s] = __ldg(tt + s * kCtThreads);
            const uint32_t want = __ldg(checks + tile * kCtThreads + tid);
            for (int rep = 0; rep < kCtReps; ++rep) {
#pragma unroll
                for (int s = 0; s < SLOTS; ++s) v[s] = ft_opaque(v[s]);
                const uint32_t inj = (rounds | (unsigned)tile | (unsigned)rep) == 0 ? inj0 : 0u;
                uint32_t* dp = (DUMP && blockIdx.x == 0 && rounds == 0 && rep == 0)
                                   ? dump + ((size_t)tile * kCtThreads + tid) * W : nullptr;
                uint32_t h;
                if constexpr (FMT != FT_DMMA) {
                    const T(&x)[kFtX] = *reinterpret_cast<const T(*)[kFtX]>(v);
                    const T(&a)[kFtAB] = *reinterpret_cast<const T(*)[kFtAB]>(v + kFtX);
                    const T(&b)[kFtAB] = *reinterpret_cast<const T(*)[kFtAB]>(v + kFtX + kFtAB);
                    h = ft_fma_rep<T, DUMP>(x, a, b, inj, dp);
                } else {
                    double d[kFtDmmaSets][kFtDmmaD];
#pragma unroll
                    for (int c = 0; c < kFtDmmaSets; ++c)
#pragma unroll
                        for (int i = 0; i < kFtDmmaD; ++i) d[c][i] = 0.0;
#pragma unroll
                    for (int s = 0; s < kFtDmmaSteps; ++s)
#pragma unroll
                        for (int c = 0; c < kFtDmmaSets; ++c)  // the sets are independent: they cover DMMA's latency
                            ft_dmma(d[c], v + s * kFtDmmaA,
                                    v + kFtDmmaSteps * kFtDmmaA + ((s + c) % kFtDmmaSteps) * kFtDmmaB);
                    h = 0;
#pragma unroll
                    for (int c = 0; c < kFtDmmaSets; ++c)
#pragma unroll
                        for (int i = 0; i < kFtDmmaD; ++i) {
                            const int j = 2 * (c * kFtDmmaD + i);
                            uint32_t w[2];
                            ft_words(d[c][i], w);
                            if (j == 0) w[0] ^= inj;
                            if (DUMP && dp) { dp[j] = w[0]; dp[j + 1] = w[1]; }
                            h += (2u * (uint32_t)j + 1u) * w[0] + (2u * (uint32_t)j + 3u) * w[1];
                        }
                }
                const int bad = __syncthreads_or(h != want);
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
