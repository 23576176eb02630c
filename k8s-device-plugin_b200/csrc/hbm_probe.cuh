// hbm_probe.cuh — sm_90a health-probe kernels (HBM stream verify + copy).
//
// This is the GPU work that replaces the reference's node-level text check
// `simpleHealthCheck` (internal/pkg/plugin/plugin.go:161-206) and the external
// exporter's per-GPU verdict consumed by `PopulatePerGPUDHealth`
// (internal/pkg/exporter/health.go:86-106): instead of inferring "healthy" from
// two kfd property lines, every heartbeat streams the whole probe buffer
// through the SMs, verifies each 32-bit word against a closed-form pattern and
// writes the re-keyed pattern to the twin buffer.
//
// Pattern (integer, bit-exact, oracle: oracle/probe_oracle.c + oracle/probe.py):
//     word(i, seed) = (uint32(i) * 2654435761u) ^ seed         i = word index
// One probe pass over n_vec 16-byte vectors:
//     for every word w = src[i]:  checksum += w  (mod 2^64)
//                                 mismatches += (w != word(i, seed))
//                                 dst[i] = w ^ delta            (delta = seed ^ next_seed)
// so a clean src leaves dst == pattern(next_seed) and the buffers ping-pong.
// Algorithmic traffic: 16 B read + 16 B written per vector (2*S per launch).
//
// No tensor cores: there is no contraction, the kernel is HBM-bound; what
// matters is coalesced 16/32-byte accesses, enough bytes in flight per SM
// (~25 KB to cover HBM latency at 3.35 TB/s / 132 SMs) and a grid that is a
// multiple of the SM count.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace b2dp {

constexpr uint32_t kPatternMul = 2654435761u;

// Dynamic shared memory of one hbm_probe_tma CTA: the tile ring plus its full/done mbarriers.
constexpr size_t tma_smem_bytes(int tile_vec, int stages) { return (size_t)stages * tile_vec * 16 + 2 * stages * 8; }

// ---- the product's kernel shapes, chosen with tools/probe_sweep on an H100 SXM (80 GB HBM3, 700 W) ----------------
constexpr int kTmaCW = 4;           // verifier warps
constexpr int kTmaTileVec = 1024;   // 16 KiB tiles
constexpr int kTmaStages = 3;
constexpr int kTmaCtasPerSm = 2;    // 2 x 3 x 16 KiB = 96 KiB staged per SM
constexpr size_t kTmaSmem = tma_smem_bytes(kTmaTileVec, kTmaStages);
constexpr int kRegThreads = 512, kRegUnroll = 2, kRegCtasPerSm = 2;

// Dynamic shared memory of one hbm_probe_queue CTA: the tile ring, its full/done/empty mbarriers and the tile of each slot.
constexpr size_t queue_smem_bytes(int tile_vec, int stages) { return (size_t)stages * tile_vec * 16 + 4 * stages * 8; }
// The health probe's kernel (hbm_probe_queue); hbm_probe_tma above stays the P2P and memtest shape.
constexpr int kQueueCW = 4;           // verifier warps (plus a loader and a storer warp)
constexpr int kQueueTileVec = 512;    // 8 KiB tiles
constexpr int kQueueStages = 6;
constexpr int kQueueCtasPerSm = 2;    // 2 x 6 x 8 KiB = 96 KiB staged per SM, as hbm_probe_tma
constexpr size_t kQueueSmem = queue_smem_bytes(kQueueTileVec, kQueueStages);

// Device-resident control block (one per GPU, zero-initialised once).
struct ProbeCtl {
    unsigned long long checksum;      // running sum over this launch
    unsigned long long mismatches;
    unsigned long long first_bad;     // min word index with a mismatch (~0 = none)
    unsigned long long t_start_ns;    // min %globaltimer over CTAs
    unsigned int       done;          // CTA completion ticket
    unsigned int       next_tile;     // hbm_probe_queue's tile queue (0 between launches)
};

// Result block; lives in pinned, device-mapped host memory so the last CTA
// publishes it without a separate D2H copy.
struct ProbeOut {
    unsigned long long checksum;
    unsigned long long mismatches;
    unsigned long long first_bad;
    unsigned long long t_start_ns;
    unsigned long long t_end_ns;
    unsigned long long seq;           // launch sequence number echoed back
};

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// ---- streaming 128-bit / 256-bit global accesses -------------------------
__device__ __forceinline__ uint4 ldg_na(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_na(uint4* p, const uint4& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// L2 cache-policy variants: the probe streams every byte exactly once, so both directions
// can be marked evict-first to keep the 50 MB L2 from retaining dead lines.
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
// 32 contiguous bytes per thread as two 128-bit accesses (sm_90 has no 256-bit LDG/STG); the L2
// eviction priority comes from a createpolicy operand (`pol`, see policy_evict_first above).
struct alignas(32) u32x8 { uint32_t v[8]; };
__device__ __forceinline__ u32x8 ldg2x128_hint(const u32x8* p, uint64_t pol) {
    u32x8 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]) : "l"(p), "l"(pol));
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4+16], %5;"
                 : "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7]) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ void stg2x128_hint(u32x8* p, const u32x8& r, uint64_t pol) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;"
                 :: "l"(p), "r"(r.v[0]), "r"(r.v[1]), "r"(r.v[2]), "r"(r.v[3]), "l"(pol) : "memory");
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0+16], {%1,%2,%3,%4}, %5;"
                 :: "l"(p), "r"(r.v[4]), "r"(r.v[5]), "r"(r.v[6]), "r"(r.v[7]), "l"(pol) : "memory");
}

// ---- per-thread accumulator -----------------------------------------------
struct Acc {
    unsigned long long sum = 0;
    unsigned int bad = 0;
    unsigned long long first_bad = ~0ull;
};

// Verify the 4 words of vector `vec_idx`, accumulate, and re-key in place.
__device__ __forceinline__ void check4(uint4& v, unsigned long long vec_idx, uint32_t seed,
                                       uint32_t delta, Acc& a) {
    const uint32_t m0 = (uint32_t)(vec_idx * 4ull) * kPatternMul;
    const uint32_t e0 = m0 ^ seed;
    const uint32_t e1 = (m0 + kPatternMul) ^ seed;
    const uint32_t e2 = (m0 + 2u * kPatternMul) ^ seed;
    const uint32_t e3 = (m0 + 3u * kPatternMul) ^ seed;
    a.sum += ((unsigned long long)v.x + v.y) + ((unsigned long long)v.z + v.w);
    const unsigned int nb = (v.x != e0) + (v.y != e1) + (v.z != e2) + (v.w != e3);
    if (nb) {  // cold path
        a.bad += nb;
        unsigned long long w = vec_idx * 4ull + ((v.x != e0) ? 0 : (v.y != e1) ? 1 : (v.z != e2) ? 2 : 3);
        if (w < a.first_bad) a.first_bad = w;
    }
    v.x ^= delta; v.y ^= delta; v.z ^= delta; v.w ^= delta;
}

// Block-reduce the accumulators, add them to ctl, and let the last CTA publish.
template <int THREADS>
__device__ __forceinline__ void finish(Acc a, ProbeCtl* ctl, ProbeOut* out,
                                       unsigned long long seq, unsigned long long t0) {
    __shared__ unsigned long long s_sum[THREADS / 32];
    __shared__ unsigned long long s_bad[THREADS / 32];
    __shared__ unsigned long long s_first[THREADS / 32];
    unsigned long long sum = a.sum, bad = a.bad, fb = a.first_bad;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
        unsigned long long f2 = __shfl_xor_sync(0xffffffffu, fb, o);
        fb = f2 < fb ? f2 : fb;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { s_sum[warp] = sum; s_bad[warp] = bad; s_first[warp] = fb; }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 1; w < THREADS / 32; ++w) {
            sum += s_sum[w]; bad += s_bad[w];
            fb = s_first[w] < fb ? s_first[w] : fb;
        }
        atomicAdd(&ctl->checksum, sum);
        if (bad) { atomicAdd(&ctl->mismatches, bad); atomicMin(&ctl->first_bad, fb); }
        atomicMin(&ctl->t_start_ns, t0);
        __threadfence();
        const unsigned int ticket = atomicAdd(&ctl->done, 1u);
        if (ticket == gridDim.x - 1) {
            __threadfence();
            // read through atomics so we observe every CTA's contribution
            const unsigned long long cs = atomicAdd(&ctl->checksum, 0ull);
            const unsigned long long mm = atomicAdd(&ctl->mismatches, 0ull);
            const unsigned long long fbad = atomicMin(&ctl->first_bad, ~0ull);
            const unsigned long long ts = atomicMin(&ctl->t_start_ns, ~0ull);
            // reset for the next launch on this stream
            ctl->checksum = 0; ctl->mismatches = 0; ctl->first_bad = ~0ull;
            ctl->t_start_ns = ~0ull; ctl->done = 0;
            __threadfence();
            out->checksum = cs; out->mismatches = mm; out->first_bad = fbad;
            out->t_start_ns = ts; out->t_end_ns = globaltimer_ns();
            __threadfence_system();
            *((volatile unsigned long long*)&out->seq) = seq;
        }
    }
}

// ===========================================================================
// Variant R128: register path. LDG.128 x UNROLL in flight per thread, verify,
// re-key, STG.128. Persistent grid-stride over "chunks" of THREADS*UNROLL vectors
// so that each warp instruction touches 512 contiguous bytes.
// ===========================================================================
template <int THREADS, int UNROLL>
__global__ void __launch_bounds__(THREADS)
hbm_probe_r128(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned long long n_vec,
               uint32_t seed, uint32_t delta, ProbeCtl* ctl, ProbeOut* out, unsigned long long seq) {
    const unsigned long long t0 = globaltimer_ns();
    Acc a;
    const unsigned long long chunk = (unsigned long long)THREADS * UNROLL;
    const unsigned long long n_full = n_vec / chunk;
    for (unsigned long long c = blockIdx.x; c < n_full; c += gridDim.x) {
        const unsigned long long base = c * chunk + threadIdx.x;
        uint4 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) v[u] = ldg_na(src + base + (unsigned long long)u * THREADS);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            check4(v[u], base + (unsigned long long)u * THREADS, seed, delta, a);
            stg_na(dst + base + (unsigned long long)u * THREADS, v[u]);
        }
    }
    // ragged tail (n_vec not a multiple of the chunk): plain grid-stride
    for (unsigned long long i = n_full * chunk + (unsigned long long)blockIdx.x * THREADS + threadIdx.x;
         i < n_vec; i += (unsigned long long)gridDim.x * THREADS) {
        uint4 v = ldg_na(src + i);
        check4(v, i, seed, delta, a);
        stg_na(dst + i, v);
    }
    finish<THREADS>(a, ctl, out, seq, t0);
}

// ===========================================================================
// Variant R256: same, with 32 bytes per thread per access (two LDG/STG.128) and L2 evict-first.
// Requires n_vec even for the main loop; odd tail handled with 128-bit ops.
// ===========================================================================
template <int THREADS, int UNROLL>
__global__ void __launch_bounds__(THREADS)
hbm_probe_r256(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned long long n_vec,
               uint32_t seed, uint32_t delta, ProbeCtl* ctl, ProbeOut* out, unsigned long long seq) {
    const unsigned long long t0 = globaltimer_ns();
    Acc a;
    const unsigned long long n_pair = n_vec / 2;
    const unsigned long long chunk = (unsigned long long)THREADS * UNROLL;
    const unsigned long long n_full = n_pair / chunk;
    const u32x8* s8 = reinterpret_cast<const u32x8*>(src);
    u32x8* d8 = reinterpret_cast<u32x8*>(dst);
    const uint64_t pol = policy_evict_first();
    for (unsigned long long c = blockIdx.x; c < n_full; c += gridDim.x) {
        const unsigned long long base = c * chunk + threadIdx.x;
        u32x8 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) v[u] = ldg2x128_hint(s8 + base + (unsigned long long)u * THREADS, pol);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const unsigned long long p = base + (unsigned long long)u * THREADS;
            uint4 lo = make_uint4(v[u].v[0], v[u].v[1], v[u].v[2], v[u].v[3]);
            uint4 hi = make_uint4(v[u].v[4], v[u].v[5], v[u].v[6], v[u].v[7]);
            check4(lo, 2 * p, seed, delta, a);
            check4(hi, 2 * p + 1, seed, delta, a);
            u32x8 o; o.v[0] = lo.x; o.v[1] = lo.y; o.v[2] = lo.z; o.v[3] = lo.w;
            o.v[4] = hi.x; o.v[5] = hi.y; o.v[6] = hi.z; o.v[7] = hi.w;
            stg2x128_hint(d8 + p, o, pol);
        }
    }
    for (unsigned long long i = n_full * chunk * 2 + (unsigned long long)blockIdx.x * THREADS + threadIdx.x;
         i < n_vec; i += (unsigned long long)gridDim.x * THREADS) {
        uint4 v = ldg_na(src + i);
        check4(v, i, seed, delta, a);
        stg_na(dst + i, v);
    }
    finish<THREADS>(a, ctl, out, seq, t0);
}

// ===========================================================================
// Variant TMA: shared-memory staged. One elected thread drives the bulk-copy
// engine: cp.async.bulk global->smem (mbarrier complete_tx) into a ring of
// STAGES tiles; all threads verify + re-key the tile in place (LDS.128/STS.128,
// conflict-free: consecutive lanes touch consecutive 16-B slots), fence to the
// async proxy, and the elected thread issues cp.async.bulk smem->global.
// The data never occupies registers across a memory round trip, so bytes in
// flight per SM = (STAGES-1) * TILE_BYTES * CTAs/SM regardless of occupancy.
// ===========================================================================
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}"
        :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// HINT template parameter of hbm_probe_tma (tools/probe_sweep only; the product uses 0 = no hints: an evict_last
// policy on the loads lets the rate of consecutive passes drift up with what the L2 retains, so it no longer measures HBM):
//   bit 0 loads evict_first, bit 1 stores evict_first, bit 2 stores evict_last, bit 3 loads evict_last
__device__ __forceinline__ void bulk_g2s_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar,
                                              uint64_t pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 :: "r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
__device__ __forceinline__ void bulk_s2g_hint(void* gdst, const void* smem_src, uint32_t bytes, uint64_t pol) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
                 :: "l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes), "l"(pol) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 :: "l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_all() {
    asm volatile("cp.async.bulk.wait_group %0;" :: "n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}

// Warp-specialised: warp 0 lane 0 = bulk-copy driver, warps 1..CW = verifiers.
//   full[s]  : armed by the driver with expect_tx, completed by the copy engine
//   done[s]  : every verifier thread arrives after re-keying its share of slot s
// Driver, tile k: wait done[slot k] -> bulk store slot k -> wait until the store of
// tile k-1 has finished READING smem -> bulk load tile k-1+STAGES into that slot.
// TILE_VEC: vectors (16 B) per tile. Dynamic smem = STAGES*TILE_VEC*16 + 2*STAGES*8.
template <int CW, int TILE_VEC, int STAGES, int HINT = 0>
__global__ void __launch_bounds__((CW + 1) * 32)
hbm_probe_tma(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned long long n_vec,
              uint32_t seed, uint32_t delta, ProbeCtl* ctl, ProbeOut* out, unsigned long long seq) {
    constexpr int THREADS = (CW + 1) * 32;
    constexpr int CT = CW * 32;  // verifier threads
    static_assert(TILE_VEC % CT == 0, "tile must be a multiple of the verifier width");
    static_assert(STAGES >= 3, "need >=3 stages");
    constexpr int PER_THREAD = TILE_VEC / CT;
    constexpr uint32_t TILE_BYTES = TILE_VEC * 16u;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint4* tiles = reinterpret_cast<uint4*>(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)STAGES * TILE_BYTES);
    uint64_t* done = full + STAGES;

    const unsigned long long t0 = globaltimer_ns();
    const unsigned long long n_tiles = n_vec / TILE_VEC;  // full tiles; tail handled below
    const unsigned long long my_tiles =
        n_tiles > blockIdx.x ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (threadIdx.x == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&done[s], CT); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async_smem();
    }
    __syncthreads();

    Acc a;
    if (threadIdx.x < 32) {
        if (threadIdx.x == 0) {
            const uint64_t pol_ld = (HINT & 8) ? policy_evict_last() : (HINT & 1) ? policy_evict_first() : 0ull;
            const uint64_t pol_st = (HINT & 4) ? policy_evict_last() : (HINT & 2) ? policy_evict_first() : 0ull;
            for (int k = 0; k < STAGES && (unsigned long long)k < my_tiles; ++k) {
                const unsigned long long t = blockIdx.x + (unsigned long long)k * gridDim.x;
                mbar_expect_tx(&full[k], TILE_BYTES);
                if (HINT & 9) bulk_g2s_hint(tiles + (size_t)k * TILE_VEC, src + t * TILE_VEC, TILE_BYTES, &full[k], pol_ld);
                else bulk_g2s(tiles + (size_t)k * TILE_VEC, src + t * TILE_VEC, TILE_BYTES, &full[k]);
            }
            for (unsigned long long k = 0; k < my_tiles; ++k) {
                const int slot = (int)(k % STAGES);
                const uint32_t parity = (uint32_t)((k / STAGES) & 1);
                const unsigned long long t = blockIdx.x + k * gridDim.x;
                mbar_wait(&done[slot], parity);
                if (HINT & 6) bulk_s2g_hint(dst + t * TILE_VEC, tiles + (size_t)slot * TILE_VEC, TILE_BYTES, pol_st);
                else bulk_s2g(dst + t * TILE_VEC, tiles + (size_t)slot * TILE_VEC, TILE_BYTES);
                bulk_commit();
                if (k >= 1) {
                    const unsigned long long kn = k - 1 + STAGES;
                    if (kn < my_tiles) {
                        bulk_wait_read<1>();  // store of tile k-1 no longer reads its slot
                        const int sn = (int)(kn % STAGES);
                        const unsigned long long tn = blockIdx.x + kn * gridDim.x;
                        mbar_expect_tx(&full[sn], TILE_BYTES);
                        if (HINT & 9) bulk_g2s_hint(tiles + (size_t)sn * TILE_VEC, src + tn * TILE_VEC, TILE_BYTES, &full[sn], pol_ld);
                        else bulk_g2s(tiles + (size_t)sn * TILE_VEC, src + tn * TILE_VEC, TILE_BYTES, &full[sn]);
                    }
                }
            }
            bulk_wait_all<0>();
        }
    } else {
        const int ct = threadIdx.x - 32;
        for (unsigned long long k = 0; k < my_tiles; ++k) {
            const int slot = (int)(k % STAGES);
            const uint32_t parity = (uint32_t)((k / STAGES) & 1);
            const unsigned long long t = blockIdx.x + k * gridDim.x;
            mbar_wait(&full[slot], parity);
            uint4* tile = tiles + (size_t)slot * TILE_VEC;
            uint4 v[PER_THREAD];
#pragma unroll
            for (int u = 0; u < PER_THREAD; ++u) v[u] = tile[ct + u * CT];
#pragma unroll
            for (int u = 0; u < PER_THREAD; ++u) {
                check4(v[u], t * TILE_VEC + ct + u * CT, seed, delta, a);
                tile[ct + u * CT] = v[u];
            }
            fence_proxy_async_smem();
            mbar_arrive(&done[slot]);
        }
    }

    // ragged tail: vectors past the last full tile, register path
    for (unsigned long long i = n_tiles * TILE_VEC + (unsigned long long)blockIdx.x * THREADS + threadIdx.x;
         i < n_vec; i += (unsigned long long)gridDim.x * THREADS) {
        uint4 v = ldg_na(src + i);
        check4(v, i, seed, delta, a);
        stg_na(dst + i, v);
    }
    finish<THREADS>(a, ctl, out, seq, t0);
}

// ===========================================================================
// Variant QUEUE (the health probe's kernel): a TMA ring like hbm_probe_tma's, with two changes
// that tools/probe_sweep --gap measured (profiles/README.md):
//  * CTAs take tiles from a grid-wide queue (ctl->next_tile) instead of tile t -> CTA t mod grid.
//    With a fixed split the CTAs of a full grid finish up to a third of a pass apart, and HBM idles
//    while the slowest drain; from a queue, a CTA that streams faster simply takes more tiles.
//  * Loads and stores are issued by different warps, so a refill never waits behind a store.
// Roles:
//   warp 0 lane 0 = loader : wait empty[s] -> claim a tile -> tile_of[s] = t -> bulk load into s
//                            (no tile left: tile_of[s] = kNoTile, plain arrive on full[s], stop)
//   warp 1 lane 0 = storer : wait full[s] -> wait done[s] -> bulk store s -> wait until it has read
//                            s -> arrive empty[s]
//   warps 2..CW+1 = verifiers: wait full[s] -> check4 + re-key their share in place -> arrive done[s]
// The mbarrier arrive that publishes full[s] releases tile_of[s]; every reader waits on full[s].
// Every CTA makes exactly one claim past the last tile, so n_tiles + gridDim.x claims are made per
// launch and the CTA that gets the last one resets the queue for the next launch on the stream
// (n_tiles + gridDim.x must stay below 2^32: 32 TiB of 8 KiB tiles).
// The ragged tail (n_vec mod TILE_VEC vectors) is a static grid-stride register loop, as in hbm_probe_tma.
// Dynamic smem = STAGES*TILE_VEC*16 + 4*STAGES*8.
// ===========================================================================
template <int CW, int TILE_VEC, int STAGES>
__global__ void __launch_bounds__((CW + 2) * 32)
hbm_probe_queue(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned long long n_vec,
                uint32_t seed, uint32_t delta, ProbeCtl* ctl, ProbeOut* out, unsigned long long seq) {
    constexpr int THREADS = (CW + 2) * 32;
    constexpr int CT = CW * 32;  // verifier threads
    static_assert(TILE_VEC % CT == 0, "tile must be a multiple of the verifier width");
    static_assert(STAGES >= 2, "need >=2 stages");
    constexpr int PER_THREAD = TILE_VEC / CT;
    constexpr uint32_t TILE_BYTES = TILE_VEC * 16u;
    constexpr unsigned long long kNoTile = ~0ull;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint4* tiles = reinterpret_cast<uint4*>(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)STAGES * TILE_BYTES);
    uint64_t* done = full + STAGES;
    uint64_t* empty = done + STAGES;
    unsigned long long* tile_of = reinterpret_cast<unsigned long long*>(empty + STAGES);

    const unsigned long long t0 = globaltimer_ns();
    const unsigned long long n_tiles = n_vec / TILE_VEC;

    if (threadIdx.x == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&done[s], CT); mbar_init(&empty[s], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async_smem();
    }
    __syncthreads();

    Acc a;
    if (threadIdx.x == 0) {
        unsigned long long t = atomicAdd(&ctl->next_tile, 1u);
        for (unsigned long long k = 0;; ++k) {
            const int slot = (int)(k % STAGES);
            if (k >= STAGES) mbar_wait(&empty[slot], (uint32_t)((k / STAGES - 1) & 1));
            if (t >= n_tiles) {
                tile_of[slot] = kNoTile;
                mbar_arrive(&full[slot]);
                if (t == n_tiles + gridDim.x - 1) atomicExch(&ctl->next_tile, 0u);  // the launch's last claim
                break;
            }
            tile_of[slot] = t;
            mbar_expect_tx(&full[slot], TILE_BYTES);
            bulk_g2s(tiles + (size_t)slot * TILE_VEC, src + t * TILE_VEC, TILE_BYTES, &full[slot]);
            t = atomicAdd(&ctl->next_tile, 1u);  // the next claim travels while the ring is full
        }
    } else if (threadIdx.x == 32) {
        for (unsigned long long k = 0;; ++k) {
            const int slot = (int)(k % STAGES);
            const uint32_t parity = (uint32_t)((k / STAGES) & 1);
            mbar_wait(&full[slot], parity);
            const unsigned long long t = tile_of[slot];
            if (t == kNoTile) break;
            mbar_wait(&done[slot], parity);
            bulk_s2g(dst + t * TILE_VEC, tiles + (size_t)slot * TILE_VEC, TILE_BYTES);
            bulk_commit();
            bulk_wait_read<0>();  // the store no longer reads the slot: hand it back to the loader
            mbar_arrive(&empty[slot]);
        }
        bulk_wait_all<0>();
    } else if (threadIdx.x >= 64) {
        const int ct = threadIdx.x - 64;
        for (unsigned long long k = 0;; ++k) {
            const int slot = (int)(k % STAGES);
            mbar_wait(&full[slot], (uint32_t)((k / STAGES) & 1));
            const unsigned long long t = tile_of[slot];
            if (t == kNoTile) break;
            uint4* tile = tiles + (size_t)slot * TILE_VEC;
            uint4 v[PER_THREAD];
#pragma unroll
            for (int u = 0; u < PER_THREAD; ++u) v[u] = tile[ct + u * CT];
#pragma unroll
            for (int u = 0; u < PER_THREAD; ++u) {
                check4(v[u], t * TILE_VEC + ct + u * CT, seed, delta, a);
                tile[ct + u * CT] = v[u];
            }
            fence_proxy_async_smem();
            mbar_arrive(&done[slot]);
        }
    }

    for (unsigned long long i = n_tiles * TILE_VEC + (unsigned long long)blockIdx.x * THREADS + threadIdx.x;
         i < n_vec; i += (unsigned long long)gridDim.x * THREADS) {
        uint4 v = ldg_na(src + i);
        check4(v, i, seed, delta, a);
        stg_na(dst + i, v);
    }
    finish<THREADS>(a, ctl, out, seq, t0);
}

// ===========================================================================
// Fill: dst[i] = word(i, seed). Write-only, S bytes.
// ===========================================================================
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
hbm_fill(uint4* __restrict__ dst, unsigned long long n_vec, uint32_t seed) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * THREADS + threadIdx.x; i < n_vec;
         i += (unsigned long long)gridDim.x * THREADS) {
        const uint32_t m0 = (uint32_t)(i * 4ull) * kPatternMul;
        uint4 v = make_uint4(m0 ^ seed, (m0 + kPatternMul) ^ seed, (m0 + 2u * kPatternMul) ^ seed,
                             (m0 + 3u * kPatternMul) ^ seed);
        stg_na(dst + i, v);
    }
}

// Fault injection for tests: word[idx] ^= mask.
__global__ void hbm_poke(uint32_t* buf, unsigned long long idx, uint32_t mask) { buf[idx] ^= mask; }

}  // namespace b2dp
