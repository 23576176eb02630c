// hostlink_selftest.cuh -- sm_90a kernel of the on-demand host-link self-test's SM format (b2dp_hostlink_test).
//
// The H2D and D2H formats move the probe's pattern with the copy engines and verify it with hbm_probe_r128.  This
// kernel moves it with the SMs alone: it reads a pinned, device-mapped host buffer with 16-byte loads across PCIe,
// verifies every word with the probe's check4 (same mismatches, first bad word and checksum, published by the probe's
// finish), and writes the re-keyed vector to a second mapped host buffer.  No copy engine takes part.
//
// Stores: vector i is written with hl_store_width(i) bytes per store -- 16, 8, 4, 2, 1, 16, ... -- so writes of every
// byte-enable shape cross the link.  Nothing here depends on how the root complex packs them.
//
// Every CTA leaves one HlRecord (%smid, vectors verified, mismatches, then the launch's sequence number) in mapped host
// memory; the driver derives SM coverage and the bad-SM mask from them.  No access reaches past n_vec vectors of
// either buffer: host memory past them belongs to someone else.
//
// Fault hook (tests, b2dp_hostlink_opts.fault_word / fault_mask): the thread that reads word fault_word XORs
// fault_mask into the value it read, before the check.  The kernel counts that word once, and the re-keyed word it
// stores is wrong, so the host's check of the destination sees it too.
#pragma once
#include <cstdint>

#include "hbm_probe.cuh"
#include "hostlink_math.hpp"

namespace b2dp {

struct HlRecord {                    // one per CTA, in mapped host memory
    unsigned long long seq;          // the launch's sequence number, stored last
    unsigned long long vectors;      // 16-byte vectors this CTA verified
    unsigned long long mismatches;   // words among them that differed from the pattern
    unsigned int smid, nsmid;
};

constexpr int kHlThreads = 256, kHlUnroll = 4;   // 4 x 16 B loads in flight per thread

__device__ __forceinline__ uint4 hl_load(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// Store v at p with hl_store_width(vec) bytes per store, in address order.
__device__ __forceinline__ void hl_store(uint4* p, const uint4& v, unsigned long long vec) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    char* b = reinterpret_cast<char*>(p);
    switch (hl_store_width(vec)) {
        case 16:
            asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(b), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3])
                         : "memory");
            break;
        case 8:
#pragma unroll
            for (int k = 0; k < 2; ++k)
                asm volatile("st.global.v2.u32 [%0], {%1,%2};" :: "l"(b + 8 * k), "r"(w[2 * k]), "r"(w[2 * k + 1])
                             : "memory");
            break;
        case 4:
#pragma unroll
            for (int k = 0; k < 4; ++k) asm volatile("st.global.u32 [%0], %1;" :: "l"(b + 4 * k), "r"(w[k]) : "memory");
            break;
        case 2:
#pragma unroll
            for (int k = 0; k < 8; ++k)
                asm volatile("st.global.u16 [%0], %1;" :: "l"(b + 2 * k), "r"(w[k / 2] >> (16 * (k % 2))) : "memory");
            break;
        default:
#pragma unroll
            for (int k = 0; k < 16; ++k)
                asm volatile("st.global.u8 [%0], %1;" :: "l"(b + k), "r"(w[k / 4] >> (8 * (k % 4))) : "memory");
            break;
    }
}

__device__ __forceinline__ void hl_inject(uint4& v, unsigned long long vec, unsigned long long fault_vec,
                                          unsigned int lane, uint32_t mask) {
    if (vec != fault_vec) return;
    v.x ^= lane == 0 ? mask : 0u;
    v.y ^= lane == 1 ? mask : 0u;
    v.z ^= lane == 2 ? mask : 0u;
    v.w ^= lane == 3 ? mask : 0u;
}

// One pass over n_vec vectors: src (word(i, seed)) -> check4 -> dst (re-keyed by delta).  Persistent grid-stride over
// chunks of THREADS * UNROLL vectors, as hbm_probe_r128, then a plain grid-stride over the ragged tail.
// fault_mask = 0: no injection.
template <int THREADS, int UNROLL>
__global__ void __launch_bounds__(THREADS)
hostlink_sm(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned long long n_vec, uint32_t seed,
            uint32_t delta, unsigned long long fault_word, uint32_t fault_mask, ProbeCtl* ctl, ProbeOut* out,
            unsigned long long seq, HlRecord* rec) {
    __shared__ unsigned long long s_vec, s_bad;
    if (threadIdx.x == 0) { s_vec = 0; s_bad = 0; }
    __syncthreads();
    const unsigned long long t0 = globaltimer_ns();
    const unsigned long long fault_vec = fault_mask ? fault_word / 4 : ~0ull;
    const unsigned int fault_lane = (unsigned int)(fault_word % 4);
    Acc a;
    unsigned long long done = 0;
    const unsigned long long chunk = (unsigned long long)THREADS * UNROLL;
    const unsigned long long n_full = n_vec / chunk;
    for (unsigned long long c = blockIdx.x; c < n_full; c += gridDim.x) {
        const unsigned long long base = c * chunk + threadIdx.x;
        uint4 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) v[u] = hl_load(src + base + (unsigned long long)u * THREADS);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const unsigned long long i = base + (unsigned long long)u * THREADS;
            hl_inject(v[u], i, fault_vec, fault_lane, fault_mask);
            check4(v[u], i, seed, delta, a);
            hl_store(dst + i, v[u], i);
        }
        done += UNROLL;
    }
    for (unsigned long long i = n_full * chunk + (unsigned long long)blockIdx.x * THREADS + threadIdx.x; i < n_vec;
         i += (unsigned long long)gridDim.x * THREADS) {
        uint4 v = hl_load(src + i);
        hl_inject(v, i, fault_vec, fault_lane, fault_mask);
        check4(v, i, seed, delta, a);
        hl_store(dst + i, v, i);
        ++done;
    }
    if (done) atomicAdd(&s_vec, done);
    if (a.bad) atomicAdd(&s_bad, (unsigned long long)a.bad);
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned int smid, nsmid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
        HlRecord* r = rec + blockIdx.x;
        r->vectors = s_vec;
        r->mismatches = s_bad;
        r->smid = smid;
        r->nsmid = nsmid;
        __threadfence_system();
        *((volatile unsigned long long*)&r->seq) = seq;
    }
    finish<THREADS>(a, ctl, out, seq, t0);
}

}  // namespace b2dp
