// hbm_memtest.cuh -- sm_90a kernel of the on-demand memory test (b2dp_memtest): an in-place march over free HBM.
//
// The health probe streams its own ring (2 x 1 GiB); the memory test covers whatever else is free at the time it
// runs.  It uses the TMA pipeline of hbm_probe_tma (bulk copy global -> smem, verify and rewrite in smem, bulk copy
// smem -> global) with one difference: the tile goes back to the SAME address it came from, so no second buffer is
// needed and every byte of the tested span is read and written in place.
//
// Memory is a list of segments (separate allocations).  Every segment holds `tiles_per_seg` tiles except the last,
// which may hold fewer; tile t belongs to segment t / tiles_per_seg and its base address comes from the segment
// table.  Word i is the global word index over the concatenated segments and segment g is keyed with its own seed:
//     word(i) = (uint32(i) * K) ^ seed_g,    seed_g = memtest_segment_seed(seed, g)     (memtest_math.hpp)
// so two virtual ranges that alias one physical page read each other's values and mismatch, and so do aliases
// 2^32 words (16 GiB) apart, across which the index wraps but the seed does not.
//
// The march (MATS++ shape; fixed):  E0 w(P)   E1 r(P) w(~P)   E2 r(~P) w(P)   E3 r(P)
// where ~P is the pattern under seed ~seed_g (= P ^ 0xFFFFFFFF).  Every bit is written and read back as 0 and as 1
// and makes both transitions, so a stuck-at or transition fault of any bit is detected deterministically.  Tile
// order across thousands of CTAs is not an address order, so nothing is claimed about coupling faults.
//
// One launch per element; MODE selects what a tile sees:
//   MARCH_WRITE       generate the pattern in smem (no load), store      (checksum / mismatches stay 0)
//   MARCH_READ_WRITE  load, check4 against seed_g ^ inv, XOR delta, store back
//   MARCH_READ        load, check4, no store
// Results go through the probe's Acc / finish<> into a ProbeCtl / ProbeOut of the element's own.
#pragma once
#include "hbm_probe.cuh"
#include "memtest_math.hpp"

namespace b2dp {

enum MarchMode { MARCH_WRITE = 0, MARCH_READ_WRITE = 1, MARCH_READ = 2 };

// The segment table, passed by value as a __grid_constant__ parameter (no copy, no extra allocation to free).
struct MarchSegs {
    uint4* base[kMemtestMaxSegments];
    uint32_t seed[kMemtestMaxSegments];
};

// Warp 0 lane 0 drives the bulk copies, warps 1..CW verify (the roles and barriers of hbm_probe_tma).  full[s] is
// completed by the copy engine (or, in WRITE mode, by the driver's plain arrive once the slot's previous store has
// finished reading it); done[s] by every verifier thread.
template <int CW, int TILE_VEC, int STAGES, int MODE>
__global__ void __launch_bounds__((CW + 1) * 32)
hbm_march_tma(const __grid_constant__ MarchSegs segs, unsigned int tiles_per_seg, unsigned long long n_tiles,
              uint32_t inv, uint32_t delta, ProbeCtl* ctl, ProbeOut* out, unsigned long long seq) {
    constexpr int THREADS = (CW + 1) * 32;
    constexpr int CT = CW * 32;
    static_assert(TILE_VEC % CT == 0, "tile must be a multiple of the verifier width");
    static_assert(STAGES >= 3, "need >=3 stages");
    constexpr int PER_THREAD = TILE_VEC / CT;
    constexpr uint32_t TILE_BYTES = TILE_VEC * 16u;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint4* tiles = reinterpret_cast<uint4*>(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)STAGES * TILE_BYTES);
    uint64_t* done = full + STAGES;

    const unsigned long long t0 = globaltimer_ns();
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
            // n_tiles < 2^32 (the host bounds it), so the segment lookup is a 32-bit division
            auto tile_addr = [&](unsigned long long t) {
                const unsigned int g = (unsigned int)t / tiles_per_seg;
                return segs.base[g] + (size_t)((unsigned int)t - g * tiles_per_seg) * TILE_VEC;
            };
            auto fill = [&](int s, unsigned long long t) {
                if (MODE == MARCH_WRITE) {
                    mbar_arrive(&full[s]);  // nothing to load: the slot is free
                } else {
                    mbar_expect_tx(&full[s], TILE_BYTES);
                    bulk_g2s(tiles + (size_t)s * TILE_VEC, tile_addr(t), TILE_BYTES, &full[s]);
                }
            };
            for (int k = 0; k < STAGES && (unsigned long long)k < my_tiles; ++k)
                fill(k, blockIdx.x + (unsigned long long)k * gridDim.x);
            for (unsigned long long k = 0; k < my_tiles; ++k) {
                const int slot = (int)(k % STAGES);
                const uint32_t parity = (uint32_t)((k / STAGES) & 1);
                const unsigned long long t = blockIdx.x + k * gridDim.x;
                mbar_wait(&done[slot], parity);
                if (MODE == MARCH_READ) {  // no store: the slot is free as soon as its verifiers are done
                    const unsigned long long kn = k + STAGES;
                    if (kn < my_tiles) fill(slot, blockIdx.x + kn * gridDim.x);
                } else {
                    bulk_s2g(tile_addr(t), tiles + (size_t)slot * TILE_VEC, TILE_BYTES);
                    bulk_commit();
                    if (k >= 1) {
                        const unsigned long long kn = k - 1 + STAGES;
                        if (kn < my_tiles) {
                            bulk_wait_read<1>();  // store of tile k-1 no longer reads its slot
                            fill((int)(kn % STAGES), blockIdx.x + kn * gridDim.x);
                        }
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
            const uint32_t seed = segs.seed[(unsigned int)t / tiles_per_seg] ^ inv;
            mbar_wait(&full[slot], parity);
            uint4* tile = tiles + (size_t)slot * TILE_VEC;
            if (MODE == MARCH_WRITE) {
#pragma unroll
                for (int u = 0; u < PER_THREAD; ++u) {
                    const uint32_t m0 = (uint32_t)((t * TILE_VEC + ct + u * CT) * 4ull) * kPatternMul;
                    tile[ct + u * CT] = make_uint4(m0 ^ seed, (m0 + kPatternMul) ^ seed, (m0 + 2u * kPatternMul) ^ seed,
                                                   (m0 + 3u * kPatternMul) ^ seed);
                }
            } else {
                uint4 v[PER_THREAD];
#pragma unroll
                for (int u = 0; u < PER_THREAD; ++u) v[u] = tile[ct + u * CT];
#pragma unroll
                for (int u = 0; u < PER_THREAD; ++u) {
                    check4(v[u], t * TILE_VEC + ct + u * CT, seed, delta, a);
                    if (MODE == MARCH_READ_WRITE) tile[ct + u * CT] = v[u];
                }
            }
            fence_proxy_async_smem();
            mbar_arrive(&done[slot]);
        }
    }
    finish<THREADS>(a, ctl, out, seq, t0);
}

}  // namespace b2dp
