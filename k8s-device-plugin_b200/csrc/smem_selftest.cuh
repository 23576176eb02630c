// smem_selftest.cuh -- sm_90a self-test kernel of the on-demand shared-memory self-test (b2dp_smem_test).
//
// One CTA per SM marches its whole addressable shared memory (kShBytes = 227 KiB, the sm_90 opt-in maximum, so no SM
// holds two) with the marches of smem_test_math.hpp:
//     format    accesses (inline PTX inside the repetition loop)                 SASS
//     SH_WORD   March C-, ld/st.shared.u32                                       LDS / STS
//     SH_BYTE   st.shared.u8, ld.shared.v4 + st.shared.u16, ld.shared.u8 +       STS.U8, LDS.128, STS.U16, LDS.U8,
//               st.shared.v4, ld.shared.v2                                       STS.128, LDS.64
//     SH_DSMEM  a cluster of 2: ld/st.shared::cluster into the peer's window     ST.E / LD.E, UCGABAR_ARV / _WAIT
//               (mapa.shared::cluster), ld/st.shared.u32 into the own array
// Every thread keeps 8 or more independent loads in flight.
//
// The round / tile / repetition structure is the other self-tests': a round runs each of the kCtTiles tiles kCtReps
// times, and a CTA repeats rounds until its %globaltimer deadline (at least one round).  A tile is a data background
// (its table: kind, key).  One comparison is one (tile, repetition): a whole march over the CTA's array.  It is a
// mismatch if, for any thread,
//   (a) a value read differs from P or ~P, which the kernel computes from the tile table (sh_gen; for SH_DSMEM with
//       the owner's rank key), or
//   (b) the thread's fold of every value it read, in read order, differs from the host's check (sh_reads, sh_fold).
// (a) is what catches a stuck bit: March C- reads it wrong twice, and at bit 31 two such errors cancel in the fold
// (their weights sum to an even number).  (b) keeps the host the source of every reference value.
//
// SH_DSMEM: the two CTAs of a cluster must run the same number of rounds, or one would wait at a cluster barrier for
// ever, so rank 0 alone reads %globaltimer and publishes its decision to rank 1 behind the barrier that ends the round.
// Each CTA also writes its repetition's "bad" bit into the peer behind that barrier, so a mismatch seen by either CTA
// counts in both records.  Both exchanges use word kShXWord of the peer's array after the last read element; every
// repetition starts with a cluster barrier, after which the first element overwrites that word.  A DSMEM fault cannot
// be pinned to one SM of the pair, so both are named; SH_WORD and SH_BYTE show whether one of them also fails alone.
//
// Fault hook: in the first comparison (round 0, tile 0, repetition 0), after element table[3] of tile 0, thread 0 of
// a CTA whose %smid == fault_sm XORs fault_mask into word table[2] of its own array (the product: word kShHookWord
// after element 0).  Every CTA then passes one more barrier (a cluster barrier for SH_DSMEM), so the two CTAs of a
// cluster stay in step.
//
// DUMP (the test harness only): round 0, repetition 0 of every tile writes the final array image, then every thread's
// fold and direct-compare error count, to dump + (blockIdx.x * kCtTiles + tile) * kShDumpWords.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "hbm_probe.cuh"  // globaltimer_ns
#include "smem_test_math.hpp"

namespace b2dp {

constexpr uint32_t kShXWord = 0;  // SH_DSMEM: the peer's word that carries the bad bit and rank 0's stop decision

__device__ __forceinline__ uint32_t sh_ld32(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sh_st32(uint32_t a, uint32_t v) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t sh_ld8(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sh_st8(uint32_t a, uint32_t v) {
    asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
// .volatile: ptxas would otherwise merge the halves of a word, and neighbouring words, into one wider store
__device__ __forceinline__ void sh_st16(uint32_t a, uint32_t v) {
    asm volatile("st.volatile.shared.u16 [%0], %1;" ::"r"(a), "h"((unsigned short)v) : "memory");
}
__device__ __forceinline__ uint4 sh_ld128(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a)
                 : "memory");
    return v;
}
__device__ __forceinline__ void sh_st128(uint32_t a, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}
__device__ __forceinline__ uint2 sh_ld64(uint32_t a) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t sh_ld32_cluster(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sh_st32_cluster(uint32_t a, uint32_t v) {
    asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void sh_cluster_sync() {
    asm volatile("barrier.cluster.arrive;\n\tbarrier.cluster.wait;" ::: "memory");
}

// P(w) of smem_test_math.hpp without a branch: (w * mul) ^ key ^ (alt if bit `sh` of w) ^ rotl(one, w + (w >> 5)).
struct ShGen {
    uint32_t mul, key, sh, alt, one;
    __device__ __forceinline__ uint32_t operator()(uint32_t w) const {
        return (w * mul) ^ key ^ ((0u - ((w >> sh) & 1u)) & alt) ^ __funnelshift_l(one, one, w + (w >> 5));
    }
};
__device__ __forceinline__ ShGen sh_gen(uint32_t kind, uint32_t key) {
    ShGen g{0u, 0u, 0u, 0u, 0u};
    if (kind == 1) { g.key = 0x55555555u; g.alt = ~0u; }
    else if (kind == 2) { g.sh = 5; g.alt = ~0u; }
    else if (kind == 3) g.one = 1u;
    else if (kind >= 4) { g.mul = kShPatternMul; g.key = key; }
    return g;
}

// A thread's fold over four accumulators (read j enters accumulator j % 4 with weight 2j + 1) and its count of reads
// that differ from what the pattern says.
struct ShAcc {
    uint32_t h[4] = {0u, 0u, 0u, 0u};
    uint32_t wt = 1u, err = 0u;
    __device__ __forceinline__ void take(int i, uint32_t v, uint32_t want) {  // i: a constant once unrolled
        h[i & 3] += wt * v;
        wt += 2u;
        err += v != want;
    }
    __device__ __forceinline__ uint32_t fold() const { return h[0] + h[1] + h[2] + h[3]; }
};

enum ShMode { SH_W, SH_RW, SH_R };

// N words t + 128 k of one element (k = k0, k0 +- 1, ...): all N loads first, then the checks and stores.  The array
// is at `base` (the own array, or the peer's window when REMOTE); reads must equal P ^ xr, writes store P ^ xw, and a
// read value enters the fold XOR fk (the owner's rank key).
template <int N, bool UP, int MODE, bool REMOTE>
__device__ __forceinline__ void sh_words(uint32_t base, int t, int k0, const ShGen& g, uint32_t xr, uint32_t xw,
                                         uint32_t fk, ShAcc& a) {
    uint32_t v[N];
    if constexpr (MODE != SH_W) {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const uint32_t addr = base + 4u * (uint32_t)(t + kCtThreads * (UP ? k0 + i : k0 - i));
            v[i] = REMOTE ? sh_ld32_cluster(addr) : sh_ld32(addr);
        }
    }
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const uint32_t w = (uint32_t)(t + kCtThreads * (UP ? k0 + i : k0 - i));
        const uint32_t p = g(w);
        if constexpr (MODE != SH_W) a.take(i, v[i] ^ fk, p ^ xr ^ fk);
        if constexpr (MODE != SH_R) {
            if constexpr (REMOTE) sh_st32_cluster(base + 4u * w, p ^ xw);
            else sh_st32(base + 4u * w, p ^ xw);
        }
    }
}

// One word element over all kShWordsPerThread (454 = 56 x 8 + 6) words of the thread.
template <bool UP, int MODE, bool REMOTE>
__device__ __forceinline__ void sh_word_element(uint32_t base, int t, const ShGen& g, uint32_t xr, uint32_t xw,
                                                uint32_t fk, ShAcc& a) {
    constexpr int kFull = kShWordsPerThread / 8, kRest = kShWordsPerThread % 8;
#pragma unroll 1
    for (int c = 0; c < kFull; ++c)
        sh_words<8, UP, MODE, REMOTE>(base, t, UP ? 8 * c : kShWordsPerThread - 1 - 8 * c, g, xr, xw, fk, a);
    sh_words<kRest, UP, MODE, REMOTE>(base, t, UP ? 8 * kFull : kRest - 1, g, xr, xw, fk, a);
}

// SH_BYTE element 0: each of 8 words written as four st.u8 in byte order 3, 0, 2, 1.
__device__ __forceinline__ void sh_bytes_w(uint32_t base, int t, int k0, int n, const ShGen& g) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        if (i < n) {
            const uint32_t w = (uint32_t)(t + kCtThreads * (k0 + i));
            const uint32_t p = g(w), a = base + 4u * w;
            sh_st8(a + 3, p >> 24);
            sh_st8(a + 0, p);
            sh_st8(a + 2, p >> 16);
            sh_st8(a + 1, p >> 8);
        }
    }
}

// SH_BYTE element 1 on N vectors t + 128 k, k = k0 ...: ld.v4 reads P, then two st.u16 per word write ~P.
template <int N>
__device__ __forceinline__ void sh_vec_r4_w16(uint32_t base, int t, int k0, const ShGen& g, ShAcc& a) {
    uint4 v[N];
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = sh_ld128(base + 16u * (uint32_t)(t + kCtThreads * (k0 + i)));
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const uint32_t w0 = 4u * (uint32_t)(t + kCtThreads * (k0 + i));
        const uint32_t got[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t p = g(w0 + j);
            a.take(4 * i + j, got[j], p);
            sh_st16(base + 4u * (w0 + j), ~p);
            sh_st16(base + 4u * (w0 + j) + 2u, ~p >> 16);
        }
    }
}

// SH_BYTE element 2 on vector t + 128 k: 16 ld.u8 (words in order, bytes 0..3) read ~P, then st.v4 writes P.
__device__ __forceinline__ void sh_vec_r8_w128(uint32_t base, int t, int k, const ShGen& g, ShAcc& a) {
    const uint32_t w0 = 4u * (uint32_t)(t + kCtThreads * k);
    uint32_t v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = sh_ld8(base + 4u * w0 + (uint32_t)i);
    uint32_t p[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        p[j] = g(w0 + j);
#pragma unroll
        for (int b = 0; b < 4; ++b) a.take(4 * j + b, v[4 * j + b], (~p[j] >> (8 * b)) & 0xFFu);
    }
    sh_st128(base + 4u * w0, make_uint4(p[0], p[1], p[2], p[3]));
}

// SH_BYTE element 3 on N pairs t + 128 k, k = k0, k0 - 1, ...: ld.v2 reads P.
template <int N>
__device__ __forceinline__ void sh_pair_r64(uint32_t base, int t, int k0, const ShGen& g, ShAcc& a) {
    uint2 v[N];
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = sh_ld64(base + 8u * (uint32_t)(t + kCtThreads * (k0 - i)));
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const uint32_t w0 = 2u * (uint32_t)(t + kCtThreads * (k0 - i));
        a.take(2 * i, v[i].x, g(w0));
        a.take(2 * i + 1, v[i].y, g(w0 + 1));
    }
}

template <int FMT>
__device__ __forceinline__ void sh_sync() {
    if constexpr (FMT == SH_DSMEM) sh_cluster_sync();
    else __syncthreads();
}

// table: kCtTiles tables of kShTableWords words; checks: [kCtTiles][kCtThreads] (DUMP: may be null); rec: one per CTA.
// Block: kCtThreads threads, kShBytes of dynamic shared memory.  Same signature as tc_selftest.
template <int FMT, bool DUMP>
__device__ __forceinline__ void smem_selftest_body(const uint8_t* __restrict__ table,
                                                   const uint32_t* __restrict__ checks, unsigned long long duration_ns,
                                                   int fault_sm, uint32_t fault_mask, CtRecord* rec,
                                                   unsigned long long seq, uint32_t* dump) {
    extern __shared__ __align__(16) uint32_t sh_array[];
    const int tid = threadIdx.x;
    uint32_t smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const uint32_t base = (uint32_t)__cvta_generic_to_shared(sh_array);
    uint32_t rank = 0, peer = base, rk_own = 0, rk_peer = 0;
    if constexpr (FMT == SH_DSMEM) {
        asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer) : "r"(base), "r"(rank ^ 1u));
        rk_own = sh_rank_key(rank);
        rk_peer = sh_rank_key(rank ^ 1u);
    }
    const unsigned long long t_end = globaltimer_ns() + duration_ns;
    const bool compare = !DUMP || checks != nullptr;
    const uint32_t* tab = reinterpret_cast<const uint32_t*>(table);
    const uint32_t hook_word = __ldg(tab + 2), hook_elem = __ldg(tab + 3);
    const bool hook_here = (int)smid == fault_sm && hook_word < (uint32_t)kShWords;
    unsigned long long rounds = 0, comparisons = 0, mismatches = 0;
    int bad_tile = -1, bad_rep = -1;
    for (;;) {
        int stop = 0;
        for (int tile = 0; tile < kCtTiles; ++tile) {
            const ShGen g = sh_gen(__ldg(tab + tile * kShTableWords), __ldg(tab + tile * kShTableWords + 1));
            const uint32_t want = compare ? __ldg(checks + tile * kCtThreads + tid) : 0u;
            for (int rep = 0; rep < kCtReps; ++rep) {
                const bool first = (rounds | (unsigned)tile | (unsigned)rep) == 0;
                // after every element: a barrier, and in the first comparison the fault hook and one more barrier
                auto sep = [&](uint32_t e) {
                    sh_sync<FMT>();
                    if (first && e == hook_elem) {
                        if (tid == 0 && hook_here) sh_st32(base + 4u * hook_word, sh_ld32(base + 4u * hook_word) ^ fault_mask);
                        sh_sync<FMT>();
                    }
                };
                ShAcc a;
                if constexpr (FMT == SH_WORD) {
                    sh_word_element<true, SH_W, false>(base, tid, g, 0u, 0u, 0u, a);
                    sep(0);
                    sh_word_element<true, SH_RW, false>(base, tid, g, 0u, ~0u, 0u, a);
                    sep(1);
                    sh_word_element<true, SH_RW, false>(base, tid, g, ~0u, 0u, 0u, a);
                    sep(2);
                    sh_word_element<false, SH_RW, false>(base, tid, g, 0u, ~0u, 0u, a);
                    sep(3);
                    sh_word_element<false, SH_RW, false>(base, tid, g, ~0u, 0u, 0u, a);
                    sep(4);
                    sh_word_element<true, SH_R, false>(base, tid, g, 0u, 0u, 0u, a);
                    sep(5);
                } else if constexpr (FMT == SH_BYTE) {
                    const int nv = kShVecsPerThread + (tid < kShVecTail ? 1 : 0);
#pragma unroll 1
                    for (int k = 0; k < kShWordsPerThread; k += 8) sh_bytes_w(base, tid, k, kShWordsPerThread - k, g);
                    sep(0);
#pragma unroll 1
                    for (int k = 0; k + 8 <= kShVecsPerThread; k += 8) sh_vec_r4_w16<8>(base, tid, k, g, a);
#pragma unroll 1
                    for (int k = kShVecsPerThread / 8 * 8; k < nv; ++k) sh_vec_r4_w16<1>(base, tid, k, g, a);
                    sep(1);
#pragma unroll 1
                    for (int k = nv - 1; k >= 0; --k) sh_vec_r8_w128(base, tid, k, g, a);
                    sep(2);
                    constexpr int kFull = kShPairsPerThread / 8, kRest = kShPairsPerThread % 8;
#pragma unroll 1
                    for (int c = 0; c < kFull; ++c) sh_pair_r64<8>(base, tid, kShPairsPerThread - 1 - 8 * c, g, a);
                    sh_pair_r64<kRest>(base, tid, kRest - 1, g, a);
                    sep(3);
                } else {
                    sh_cluster_sync();  // the peer has started, and has read the exchange word of the last repetition
                    sh_word_element<true, SH_W, true>(peer, tid, g, 0u, rk_peer, 0u, a);
                    sep(0);
                    sh_word_element<true, SH_RW, false>(base, tid, g, rk_own, ~rk_own, rk_own, a);
                    sep(1);
                    sh_word_element<true, SH_RW, true>(peer, tid, g, ~rk_peer, rk_peer, rk_peer, a);
                    sep(2);
                    sh_word_element<true, SH_R, false>(base, tid, g, rk_own, 0u, rk_own, a);
                    sep(3);
                }
                const uint32_t h = a.fold();
                if (DUMP && rounds == 0 && rep == 0) {
                    uint32_t* d = dump + ((size_t)blockIdx.x * kCtTiles + tile) * kShDumpWords;
                    for (int w = tid; w < kShWords; w += kCtThreads) d[w] = sh_array[w];
                    d[kShWords + tid] = h;
                    d[kShWords + kCtThreads + tid] = a.err;
                    sh_sync<FMT>();  // SH_DSMEM: the peer's exchange store below must not race the image
                }
                int bad = __syncthreads_or(compare && (a.err != 0 || h != want));
                if constexpr (FMT == SH_DSMEM) {
                    if (rank == 0 && tile == kCtTiles - 1 && rep == kCtReps - 1)
                        stop = __syncthreads_or(tid == 0 && globaltimer_ns() >= t_end);
                    if (tid == 0) sh_st32_cluster(peer + 4u * kShXWord, (uint32_t)bad | ((uint32_t)stop << 1));
                    sh_cluster_sync();
                    const uint32_t x = sh_ld32(base + 4u * kShXWord);
                    bad |= (int)(x & 1u);
                    if (rank == 1) stop = (int)((x >> 1) & 1u);
                }
                ++comparisons;
                if (bad && mismatches++ == 0) { bad_tile = tile; bad_rep = rep; }
            }
        }
        ++rounds;
        if constexpr (FMT == SH_DSMEM) {
            if (stop) break;
        } else {
            if (__syncthreads_or(tid == 0 && globaltimer_ns() >= t_end)) break;
        }
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

template <int FMT, bool DUMP>
__global__ void __launch_bounds__(kCtThreads, 1)
smem_selftest(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks, unsigned long long duration_ns,
              int fault_sm, uint32_t fault_mask, CtRecord* rec, unsigned long long seq, uint32_t* dump) {
    smem_selftest_body<FMT, DUMP>(table, checks, duration_ns, fault_sm, fault_mask, rec, seq, dump);
}
// SH_DSMEM runs as clusters of two CTAs on two SMs.
template <>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kCtThreads, 1)
smem_selftest<SH_DSMEM, false>(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks,
                               unsigned long long duration_ns, int fault_sm, uint32_t fault_mask, CtRecord* rec,
                               unsigned long long seq, uint32_t* dump) {
    smem_selftest_body<SH_DSMEM, false>(table, checks, duration_ns, fault_sm, fault_mask, rec, seq, dump);
}
template <>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kCtThreads, 1)
smem_selftest<SH_DSMEM, true>(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks,
                              unsigned long long duration_ns, int fault_sm, uint32_t fault_mask, CtRecord* rec,
                              unsigned long long seq, uint32_t* dump) {
    smem_selftest_body<SH_DSMEM, true>(table, checks, duration_ns, fault_sm, fault_mask, rec, seq, dump);
}

}  // namespace b2dp
