// tc_selftest.cuh -- sm_90a tensor-core self-test kernel of the on-demand compute test (b2dp_compute_test).
//
// One warpgroup per CTA runs warpgroup GEMMs (wgmma, SASS HGMMA / QGMMA / IGMMA) on operand tiles the host generated,
// and compares every result with values the host computed exactly (compute_test_math.hpp):
//     format  instruction                               K per result tile
//     BF16    wgmma m64n128k16.f32.bf16.bf16 (x16)      256
//     FP8     wgmma m64n128k32.f32.e4m3.e4m3 (x1)       32
//     INT8    wgmma m64n128k32.s32.s8.s8     (x8)       256
// A round runs each of the kCtTiles tiles kCtReps times; a CTA repeats rounds until its %globaltimer deadline (at
// least one round).  Per tile, thread 0 bulk-copies the tile's image (A then B, K-major, no swizzle; the layout is
// ct_image_offset) from an L2-resident table into shared memory, and each thread loads the host's comparison value of
// its accumulator fragment.  Per repetition every thread folds its 64 accumulators into ct_fold's weighted sum and
// compares it with that value; the CTA counts the repetition as one mismatch if any thread disagrees.
//
// Each CTA publishes one CtRecord (its %smid and %nsmid, rounds, comparisons, mismatches, first bad tile and
// repetition, seq last) through pinned, device-mapped host memory.
//
// Test hooks: in round 0, thread 0 of a CTA whose %smid == fault_sm XORs fault_mask into its first accumulator of tile
// 0, repetition 0, before the compare (fault_mask = 0: no effect).  DUMP (instantiated only by the test harness
// tests/native/compute_test_kernels.cu) makes CTA 0 write its raw accumulators of repetition 0 of every tile of round
// 0 to dump[tile][thread][64].
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "compute_test_math.hpp"
#include "hbm_probe.cuh"  // globaltimer_ns, smem_u32, mbar_*, bulk_g2s, fence_proxy_async_smem

namespace b2dp {

template <int FMT>
struct CtShape {
    static constexpr int K = FMT == CT_BF16 ? kCtBf16K : FMT == CT_FP8 ? kCtFp8K : kCtInt8K;
    static constexpr int EB = FMT == CT_BF16 ? 2 : 1;
    static constexpr uint32_t A_BYTES = kCtM * K * EB, B_BYTES = kCtN * K * EB;
    static constexpr uint32_t SMEM = A_BYTES + B_BYTES;
    static constexpr int STEPS = K * EB / kCtKStepBytes;  // wgmma instructions per result tile
};

// wgmma shared-memory matrix descriptor: start address, LBO = 128, SBO = 256 (all >> 4), no swizzle, base offset 0.
__device__ __forceinline__ uint64_t ct_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | (uint64_t)(128 >> 4) << 16 | (uint64_t)(256 >> 4) << 32;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define CT_D64                                                                                                        \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
    "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "  \
    "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define CT_OP8(c, i)                                                                                                  \
    c(d[i]), c(d[i + 1]), c(d[i + 2]), c(d[i + 3]), c(d[i + 4]), c(d[i + 5]), c(d[i + 6]), c(d[i + 7])
#define CT_OPS64(c)                                                                                                   \
    CT_OP8(c, 0), CT_OP8(c, 8), CT_OP8(c, 16), CT_OP8(c, 24), CT_OP8(c, 32), CT_OP8(c, 40), CT_OP8(c, 48), CT_OP8(c, 56)
// D (+)= A * B^T; accumulate = 0 overwrites D (the scale-d predicate)
#define CT_WGMMA(instr, tail, c)                                                                                      \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t" instr " " CT_D64 ", %64, %65, p" tail ";\n\t}"   \
                 : CT_OPS64(c) : "l"(da), "l"(db), "r"(accumulate))

template <int FMT>
struct CtMma;
template <>
struct CtMma<CT_BF16> {
    using Acc = float;
    static __device__ __forceinline__ void run(float (&d)[kCtAcc], uint64_t da, uint64_t db, int accumulate) {
        CT_WGMMA("wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16", ", 1, 1, 0, 0", "+f");
    }
};
template <>
struct CtMma<CT_FP8> {
    using Acc = float;
    static __device__ __forceinline__ void run(float (&d)[kCtAcc], uint64_t da, uint64_t db, int accumulate) {
        CT_WGMMA("wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3", ", 1, 1", "+f");
    }
};
template <>
struct CtMma<CT_INT8> {
    using Acc = uint32_t;
    static __device__ __forceinline__ void run(uint32_t (&d)[kCtAcc], uint64_t da, uint64_t db, int accumulate) {
        CT_WGMMA("wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8", "", "+r");
    }
};
#undef CT_WGMMA
#undef CT_OPS64
#undef CT_OP8
#undef CT_D64

__device__ __forceinline__ uint32_t ct_bits(float x) { return __float_as_uint(x); }
__device__ __forceinline__ uint32_t ct_bits(uint32_t x) { return x; }

// images: kCtTiles images of CtShape<FMT>::SMEM bytes; checks: [kCtTiles][kCtThreads]; rec: one per CTA.
// Dynamic shared memory: CtShape<FMT>::SMEM bytes.  Block: kCtThreads threads.
template <int FMT, bool DUMP>
__global__ void __launch_bounds__(kCtThreads)
tc_selftest(const uint8_t* __restrict__ images, const uint32_t* __restrict__ checks, unsigned long long duration_ns,
            int fault_sm, uint32_t fault_mask, CtRecord* rec, unsigned long long seq, uint32_t* dump) {
    using S = CtShape<FMT>;
    using Acc = typename CtMma<FMT>::Acc;
    extern __shared__ __align__(128) unsigned char ct_smem[];
    __shared__ uint64_t bar;
    const int tid = threadIdx.x;
    uint32_t smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned long long t_end = globaltimer_ns() + duration_ns;
    if (tid == 0) {
        mbar_init(&bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async_smem();
    }
    __syncthreads();
    const uint64_t da = ct_desc(smem_u32(ct_smem)), db = ct_desc(smem_u32(ct_smem + S::A_BYTES));
    const uint32_t inj0 = (tid == 0 && (int)smid == fault_sm) ? fault_mask : 0u;
    Acc d[kCtAcc];
#pragma unroll
    for (int j = 0; j < kCtAcc; ++j) d[j] = Acc(0);
    unsigned long long rounds = 0, comparisons = 0, mismatches = 0;
    int bad_tile = -1, bad_rep = -1;
    uint32_t phase = 0;
    for (;;) {
        for (int tile = 0; tile < kCtTiles; ++tile) {
            // The previous tile's wgmmas have completed: every thread waited for them before the last barrier below.
            if (tid == 0) {
                mbar_expect_tx(&bar, S::SMEM);
                bulk_g2s(ct_smem, images + (size_t)tile * S::SMEM, S::SMEM, &bar);
            }
            const uint32_t want = __ldg(checks + tile * kCtThreads + tid);
            mbar_wait(&bar, phase);
            phase ^= 1u;
            for (int rep = 0; rep < kCtReps; ++rep) {
                wgmma_fence();
#pragma unroll
                for (int s = 0; s < S::STEPS; ++s)  // descriptor addresses are in 16-byte units
                    CtMma<FMT>::run(d, da + (uint64_t)(s * kCtM * kCtKStepBytes / 16),
                                    db + (uint64_t)(s * kCtN * kCtKStepBytes / 16), s);
                wgmma_commit();
                wgmma_wait_all();
                if (DUMP && blockIdx.x == 0 && rounds == 0 && rep == 0) {
#pragma unroll
                    for (int j = 0; j < kCtAcc; ++j) dump[((size_t)tile * kCtThreads + tid) * kCtAcc + j] = ct_bits(d[j]);
                }
                // ct_fold: any single flipped bit of any one element changes h (see compute_test_math.hpp)
                uint32_t h = ct_bits(d[0]) ^ ((rounds | (unsigned)tile | (unsigned)rep) == 0 ? inj0 : 0u);
#pragma unroll
                for (int j = 1; j < kCtAcc; ++j) h += (2u * j + 1u) * ct_bits(d[j]);
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
