// l2_selftest.cuh -- sm_90a self-test kernel of the on-demand L2 self-test (b2dp_l2_test).
//
// A cooperative grid (every CTA resident) marches an L2-resident span with ownership that rotates across CTAs, or
// drives the L2's atomic and reduction units on a hot block every CTA shares (l2_test_math.hpp):
//     format    accesses (inline PTX inside the repetition loop)                 SASS
//     L2_WORD   ld/st.global.cg.v4.u32, March C-                                 LDG.E.128.STRONG.GPU / STG.E.128.STRONG.GPU
//     L2_BYTE   st.global.cg.u8 / .u16, ld.global.cg.v4.u32                      STG.E.U8 / STG.E.U16 .STRONG.GPU, LDG.E.128
//     L2_ATOM   atom add / inc / dec / exch / cas.b32 / cas.b64, red and / or /  ATOMG.E.*, REDG.E.*, ATOMG/REDG .ADD.F32x4
//               xor / min / max, red.add.u64 / f32 / f64 / noftz.f16x2 /
//               noftz.bf16x2, red / atom .v4.f32.add
//
// The round / tile / repetition structure is the other self-tests': a round runs each of the kCtTiles tiles kCtReps
// times; CTA 0 alone reads %globaltimer and publishes its decision to stop at the grid barrier that ends a round, so
// every CTA runs the same rounds (at least one).  One comparison is one (tile, repetition).
//
// L2_WORD / L2_BYTE: every element ends at a grid barrier, after which the slice a CTA wrote belongs to CTA c - 1.  A
// comparison is a mismatch for a CTA if any value it read differs from P or ~P (direct compare; it catches a stuck
// bit 31, which cancels in the fold), or if a thread's fold differs from K x the host's check.
// L2_ATOM: after the atomic phase each CTA stores the sum and xor of l2_mix over its returns (plain stores), then a
// grid barrier; the checker, CTA (comparison index % G), compares every hot word with the host's final value for its
// count of contributors and the combined folds with the host's, rewrites the initial values of the next comparison,
// and a grid barrier ends the comparison.  Only the checker counts a mismatch, so a faulty L2 unit names every SM over
// a run and an SM's own fault names that SM only.
//
// The grid barrier is l2_grid_sync: every wait gives up past the deadline plus kL2GraceNs, and so does every CAS
// retry; a CTA that gave up stops and reports rounds = 0, which the verdict counts as an incomplete record.  Every
// decision to stop is CTA-uniform before the next barrier: the grid barrier broadcasts its own through shared memory,
// and the CAS give-ups are combined with __syncthreads_and.
//
// Fault hook: in the first comparison the first CTA on %smid == fault_sm to claim the scratch's claim word XORs
// fault_mask into one word: word table[3] of the slice it wrote in element table[4] (WORD / BYTE; read wrong by the
// next owner), or the first hot word (ATOM; read wrong by the checker).  Every CTA then passes one more grid barrier.
//
// DUMP (the test harness only; its area starts at scratch word hdr[kL2HdrDump]):
//   WORD / BYTE: round 0, repetition 0 of tile T: every thread's fold and direct-compare error count at
//                [T][cta][2][kCtThreads], then the window image after the march at [kCtTiles * G * 256 + T * span words].
//   ATOM:        round 0, repetition 0 of tile T: the checker writes the hot block it found, then the 12 combined
//                folds and the 12 expected ones, at [T][kL2AtomHotWords + 24].
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "hbm_probe.cuh"  // globaltimer_ns
#include "l2_test_math.hpp"

namespace b2dp {

__device__ __forceinline__ uint4 l2_ld128(const uint32_t* p) {
    uint4 v;
    asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ void l2_st128(uint32_t* p, uint4 v) {
    asm volatile("st.global.cg.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}
__device__ __forceinline__ void l2_st8(uint8_t* p, uint32_t v) {
    asm volatile("st.global.cg.u8 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void l2_st16(uint8_t* p, uint32_t v) {
    asm volatile("st.global.cg.u16 [%0], %1;" ::"l"(p), "h"((unsigned short)v) : "memory");
}
__device__ __forceinline__ uint32_t l2_ld32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void l2_st32(uint32_t* p, uint32_t v) {
    asm volatile("st.global.cg.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t l2_ld_relaxed(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// The grid barrier: thread 0 of every CTA arrives on a counter; the last one resets it and bumps the generation the
// others poll.  false if this CTA gave up waiting at t_bound.
__device__ __forceinline__ bool l2_grid_sync(uint32_t* hdr, unsigned long long t_bound, int* s_ok) {
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t g0 = l2_ld_relaxed(hdr + kL2HdrGen);
        int ok = 1;
        __threadfence();
        if (atomicAdd(hdr + kL2HdrCount, 1u) == gridDim.x - 1) {
            atomicExch(hdr + kL2HdrCount, 0u);
            __threadfence();
            atomicExch(hdr + kL2HdrGen, g0 + 1u);
        } else {
            while (l2_ld_relaxed(hdr + kL2HdrGen) == g0) {
                if (globaltimer_ns() > t_bound) { ok = 0; break; }
                __nanosleep(64);
            }
        }
        __threadfence();
        *s_ok = ok;
    }
    __syncthreads();
    return *s_ok != 0;
}

// A thread's fold (weight 2j + 1 for the j-th value of a block, block key XORed out) and its direct-compare errors.
struct L2Acc {
    uint32_t h = 0u, err = 0u;
    __device__ __forceinline__ void take(uint32_t wt, uint32_t v, uint32_t bk, uint32_t want) {
        h += wt * (v ^ bk);
        err += v != want;
    }
};

enum L2Mode { L2_W, L2_RW, L2_R };

// One 16-byte vector of a WORD / BYTE element: read (expect P ^ xr) then write (P ^ xw) with the format's widths.
// pl: the thread's four in-block pattern words; RE: the element's index among the reading elements.
template <int FMT, int MODE, int RE>
__device__ __forceinline__ void l2_vec(uint32_t* vp, const uint32_t (&pl)[4], uint32_t bk, uint32_t xr, uint32_t xw,
                                       L2Acc& a, uint4 v) {
    if constexpr (MODE != L2_W) {
        const uint32_t got[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) a.take(2u * (4u * RE + i) + 1u, got[i], bk, pl[i] ^ bk ^ xr);
    }
    if constexpr (MODE != L2_R) {
        const uint32_t w[4] = {pl[0] ^ bk ^ xw, pl[1] ^ bk ^ xw, pl[2] ^ bk ^ xw, pl[3] ^ bk ^ xw};
        uint8_t* b = reinterpret_cast<uint8_t*>(vp);
        if constexpr (FMT == L2_WORD) {
            l2_st128(vp, make_uint4(w[0], w[1], w[2], w[3]));
        } else if constexpr (RE == 0 && MODE == L2_RW) {  // BYTE element 1: two u16 per word
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                l2_st16(b + 4 * i, w[i]);
                l2_st16(b + 4 * i + 2, w[i] >> 16);
            }
        } else {                                           // BYTE elements 0 and 2: four u8 per word, order 3, 0, 2, 1
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                l2_st8(b + 4 * i + 3, w[i] >> 24);
                l2_st8(b + 4 * i + 0, w[i]);
                l2_st8(b + 4 * i + 2, w[i] >> 16);
                l2_st8(b + 4 * i + 1, w[i] >> 8);
            }
        }
    }
}

// One element over the K blocks of `slice` in window `win`: batches of 4 vectors, all loads first.
template <int FMT, int MODE, bool UP, int RE>
__device__ __forceinline__ void l2_element(uint32_t* win, uint32_t slice, uint32_t K, uint32_t blockmul,
                                           const uint32_t (&pl)[4], uint32_t xr, uint32_t xw, L2Acc& a) {
    const int t = threadIdx.x;
#pragma unroll 1
    for (uint32_t b0 = 0; b0 < K; b0 += 4) {
        uint4 v[4];
        uint32_t* vp[4];
        uint32_t bk[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t b = UP ? b0 + i : K - 1 - (b0 + i);
            const uint32_t blk = slice * K + (b0 + i < K ? b : 0u);
            vp[i] = win + (size_t)blk * kL2BlockWords + 4 * t;
            bk[i] = (blk + 1u) * blockmul;
            if (MODE != L2_W && b0 + i < K) v[i] = l2_ld128(vp[i]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (b0 + i < K) l2_vec<FMT, MODE, RE>(vp[i], pl, bk[i], xr, xw, a, v[i]);
    }
}

// ---- L2_ATOM ops, one inline PTX statement each ----
#define B2DP_LA_RET(NAME, PTX)                                                                          \
    __device__ __forceinline__ uint32_t NAME(uint32_t* p, uint32_t b) {                                 \
        uint32_t d;                                                                                     \
        asm volatile(PTX " %0, [%1], %2;" : "=r"(d) : "l"(p), "r"(b) : "memory");                       \
        return d;                                                                                       \
    }
B2DP_LA_RET(la_add, "atom.global.add.u32")
B2DP_LA_RET(la_inc, "atom.global.inc.u32")
B2DP_LA_RET(la_dec, "atom.global.dec.u32")
B2DP_LA_RET(la_exch, "atom.global.exch.b32")
#undef B2DP_LA_RET
#define B2DP_LA_RED(NAME, PTX)                                                                          \
    __device__ __forceinline__ void NAME(uint32_t* p, uint32_t b) {                                     \
        asm volatile(PTX " [%0], %1;" ::"l"(p), "r"(b) : "memory");                                     \
    }
B2DP_LA_RED(la_and, "red.global.and.b32")
B2DP_LA_RED(la_or, "red.global.or.b32")
B2DP_LA_RED(la_xor, "red.global.xor.b32")
B2DP_LA_RED(la_min_s, "red.global.min.s32")
B2DP_LA_RED(la_max_s, "red.global.max.s32")
B2DP_LA_RED(la_min_u, "red.global.min.u32")
B2DP_LA_RED(la_max_u, "red.global.max.u32")
B2DP_LA_RED(la_f32, "red.global.add.f32")
B2DP_LA_RED(la_f16x2, "red.global.add.noftz.f16x2")
B2DP_LA_RED(la_bf16x2, "red.global.add.noftz.bf16x2")
#undef B2DP_LA_RED
__device__ __forceinline__ uint32_t la_cas(uint32_t* p, uint32_t cmp, uint32_t v) {
    uint32_t d;
    asm volatile("atom.global.cas.b32 %0, [%1], %2, %3;" : "=r"(d) : "l"(p), "r"(cmp), "r"(v) : "memory");
    return d;
}
__device__ __forceinline__ unsigned long long la_cas64(uint32_t* p, unsigned long long cmp, unsigned long long v) {
    unsigned long long d;
    asm volatile("atom.global.cas.b64 %0, [%1], %2, %3;" : "=l"(d) : "l"(p), "l"(cmp), "l"(v) : "memory");
    return d;
}
__device__ __forceinline__ void la_add64(uint32_t* p, unsigned long long b) {
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(b) : "memory");
}
__device__ __forceinline__ void la_f64(uint32_t* p, unsigned long long b) {
    asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(__longlong_as_double((long long)b)) : "memory");
}
__device__ __forceinline__ void la_v4red(uint32_t* p, const uint32_t* b) {
    asm volatile("red.global.v4.f32.add [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(__uint_as_float(b[0])),
                 "f"(__uint_as_float(b[1])), "f"(__uint_as_float(b[2])), "f"(__uint_as_float(b[3])) : "memory");
}
__device__ __forceinline__ uint32_t la_v4atom(uint32_t* p, const uint32_t* b) {
    float d0, d1, d2, d3;
    asm volatile("atom.global.v4.f32.add {%0, %1, %2, %3}, [%4], {%5, %6, %7, %8};"
                 : "=f"(d0), "=f"(d1), "=f"(d2), "=f"(d3)
                 : "l"(p), "f"(__uint_as_float(b[0])), "f"(__uint_as_float(b[1])), "f"(__uint_as_float(b[2])),
                   "f"(__uint_as_float(b[3]))
                 : "memory");
    return __float_as_uint(d0) ^ __float_as_uint(d1) ^ __float_as_uint(d2) ^ __float_as_uint(d3);
}

// table: kCtTiles tables of l2_table_bytes(FMT) bytes; checks: [kCtTiles][kCtThreads]; rec: one per CTA; scratch: the
// header, fold slots and data of l2_test_math.hpp (header words zero but K and the DUMP offset).  Block: kCtThreads
// threads, launched cooperatively on every resident CTA.  Same signature as tc_selftest.
template <int FMT, bool DUMP>
__global__ void __launch_bounds__(kCtThreads)
l2_selftest(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks, unsigned long long duration_ns,
            int fault_sm, uint32_t fault_mask, CtRecord* rec, unsigned long long seq, uint32_t* scratch) {
    __shared__ int s_ok;
    __shared__ uint32_t s_red[4][2 * kL2AtomRet + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t G = gridDim.x, c = blockIdx.x;
    uint32_t smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned long long t0 = globaltimer_ns();
    const unsigned long long t_end = t0 + duration_ns, t_bound = t_end + kL2GraceNs;
    uint32_t* hdr = scratch;
    uint32_t* data = scratch + kL2DataOff;
    const uint32_t K = hdr[kL2HdrBlocks];
    uint32_t* dump = DUMP ? scratch + hdr[kL2HdrDump] : nullptr;
    const uint32_t* tab = reinterpret_cast<const uint32_t*>(table);
    const size_t span_words = (size_t)K * G * kL2BlockWords;
    unsigned long long rounds = 0, comparisons = 0, mismatches = 0;
    int bad_tile = -1, bad_rep = -1;
    bool ok = true;
    auto claim = [&]() -> bool {  // thread 0: the first CTA on fault_sm to get here
        return (int)smid == fault_sm && atomicCAS(hdr + kL2HdrClaim, 0u, 1u) == 0u;
    };

    if constexpr (FMT == L2_ATOM) {
        const uint32_t g = 4u * c + (uint32_t)warp, row = g % kL2AtomRows, q = g / kL2AtomRows;
        auto hot = [&](int s, uint32_t r, uint32_t l) { return data + ((size_t)s * kL2AtomRows + r) * 32 + l; };
        // the initial values of tile 0, then every CTA starts
        if (c == 0)
            for (int i = tid; i < kL2AtomHotWords; i += kCtThreads) {
                int rr, ll;
                l2_st32(data + i, __ldg(tab + kL2AtomFinalOff + l2_atom_word(i, rr, ll) * (kL2AtomMaxN + 1)));
            }
        ok = l2_grid_sync(hdr, t_bound, &s_ok);
        int stop = 0;
        while (ok && !stop) {
            for (int tile = 0; tile < kCtTiles && ok; ++tile) {
                const uint32_t* tt = tab + (size_t)tile * kL2AtomTableWords;
                uint32_t x[kL2AtomSlots];
#pragma unroll
                for (int s = 0; s < kL2AtomSlots; ++s) x[s] = __ldg(tt + kL2AtomOpOff + s * kL2AtomMaxN + q);
                const uint32_t init_cas = __ldg(tt + kL2AtomFinalOff + LA_CAS32 * (kL2AtomMaxN + 1));
                const unsigned long long init_cas64 =
                    (unsigned long long)__ldg(tt + kL2AtomFinalOff + (LA_CAS64 + 1) * (kL2AtomMaxN + 1)) << 32 |
                    __ldg(tt + kL2AtomFinalOff + LA_CAS64 * (kL2AtomMaxN + 1));
                for (int rep = 0; rep < kCtReps && ok; ++rep) {
                    const bool first = (rounds | (unsigned)tile | (unsigned)rep) == 0;
                    uint32_t sm[kL2AtomRet], xr[kL2AtomRet], r;
                    auto take = [&](int k, uint32_t m) { sm[k] = m; xr[k] = m; };
                    take(0, l2_mix(la_add(hot(LA_ADD, row, lane), x[LA_ADD]), lane));
                    take(1, l2_mix(la_inc(hot(LA_INC, row, lane), x[LA_INC]), lane));
                    take(2, l2_mix(la_dec(hot(LA_DEC, row, lane), x[LA_DEC]), lane));
                    take(3, l2_mix(la_exch(hot(LA_EXCH, row, lane), x[LA_EXCH]), lane));
                    la_and(hot(LA_AND, row, lane), x[LA_AND]);
                    la_or(hot(LA_OR, row, lane), x[LA_OR]);
                    la_xor(hot(LA_XOR, row, lane), x[LA_XOR]);
                    la_min_s(hot(LA_MIN_S, row, lane), x[LA_MIN_S]);
                    la_max_s(hot(LA_MAX_S, row, lane), x[LA_MAX_S]);
                    la_min_u(hot(LA_MIN_U, row, lane), x[LA_MIN_U]);
                    la_max_u(hot(LA_MAX_U, row, lane), x[LA_MAX_U]);
                    // the 64-bit ops take words (slot, row, lane) and (slot + 1, row, lane) as one 8-byte word: their
                    // slots are laid out as 64-bit words of row-major [row][lane] over two slot planes
                    la_add64(hot(LA_ADD64, 0, 0) + 2 * (row * 32 + lane),
                             (unsigned long long)x[LA_ADD64 + 1] << 32 | x[LA_ADD64]);
                    la_f32(hot(LA_F32, row, lane), x[LA_F32]);
                    la_f64(hot(LA_F64, 0, 0) + 2 * (row * 32 + lane),
                           (unsigned long long)x[LA_F64 + 1] << 32 | x[LA_F64]);
                    la_f16x2(hot(LA_F16X2, row, lane), x[LA_F16X2]);
                    la_bf16x2(hot(LA_BF16X2, row, lane), x[LA_BF16X2]);
                    la_v4red(hot(LA_V4RED, 0, 0) + 4 * (row * 32 + lane), x + LA_V4RED);
                    const uint32_t v4ret = la_v4atom(hot(LA_V4ATOM, 0, 0) + 4 * (row * 32 + lane), x + LA_V4ATOM);
                    {   // increment-by-one CAS loops, bounded like every wait
                        uint32_t* p = hot(LA_CAS32, row, lane);
                        uint32_t want = init_cas;
                        for (;;) {
                            r = la_cas(p, want, want + 1u);
                            if (r == want) break;
                            want = r;
                            if (globaltimer_ns() > t_bound) { ok = false; break; }
                        }
                        take(4, l2_mix(r, lane));
                        uint32_t* p64 = hot(LA_CAS64, 0, 0) + 2 * (row * 32 + lane);
                        unsigned long long w64 = init_cas64, r64;
                        for (;;) {
                            r64 = la_cas64(p64, w64, w64 + 1ull);
                            if (r64 == w64) break;
                            w64 = r64;
                            if (globaltimer_ns() > t_bound) { ok = false; break; }
                        }
                        take(5, l2_mix64(r64, lane));
                    }
                    // A CAS that never matched gives up in its own thread only.  The CTA stops as a whole here, before
                    // any block or grid barrier, so that no barrier is reached under divergent control flow; the
                    // record then reports rounds = 0, and the other CTAs give up at their next grid barrier.
                    ok = __syncthreads_and(ok) != 0;
                    if (!ok) break;
                    // the CTA's folds: sum and xor over its 128 threads, stored plainly in its slot
#pragma unroll
                    for (int k = 0; k < kL2AtomRet; ++k)
#pragma unroll
                        for (int o = 16; o; o >>= 1) {
                            sm[k] += __shfl_xor_sync(0xffffffffu, sm[k], o);
                            xr[k] ^= __shfl_xor_sync(0xffffffffu, xr[k], o);
                        }
                    if (lane == 0) {
#pragma unroll
                        for (int k = 0; k < kL2AtomRet; ++k) { s_red[warp][k] = sm[k]; s_red[warp][kL2AtomRet + k] = xr[k]; }
                        s_red[warp][2 * kL2AtomRet] = v4ret;  // kept live: the v4 atom's returns are not checked
                    }
                    __syncthreads();
                    if (tid < 2 * kL2AtomRet) {
                        const uint32_t a = s_red[0][tid], b = s_red[1][tid], d = s_red[2][tid], e = s_red[3][tid];
                        l2_st32(scratch + kL2HdrWords + c * kL2FoldWords + tid,
                                tid < kL2AtomRet ? a + b + d + e : a ^ b ^ d ^ e);
                    }
                    if (!l2_grid_sync(hdr, t_bound, &s_ok)) ok = false;
                    if (!ok) break;
                    if (first) {
                        if (tid == 0 && claim()) l2_st32(data, l2_ld32(data) ^ fault_mask);
                        if (!l2_grid_sync(hdr, t_bound, &s_ok)) { ok = false; break; }
                    }
                    int bad = 0;
                    const uint32_t checker = (uint32_t)(comparisons % G);
                    if (c == checker) {
                        const int next_tile = rep + 1 < kCtReps ? tile : (tile + 1) % kCtTiles;
                        const uint32_t* nt = tab + (size_t)next_tile * kL2AtomTableWords;
                        uint32_t err = 0, esum = 0, exor = 0;
                        uint32_t* dd = (DUMP && rounds == 0 && rep == 0)
                                           ? dump + (size_t)tile * (kL2AtomHotWords + 4 * kL2AtomRet) : nullptr;
                        for (int i = tid; i < kL2AtomHotWords; i += kCtThreads) {
                            int rr, ll;
                            const int ws = l2_atom_word(i, rr, ll);
                            const uint32_t v = l2_ld32(data + i);
                            if (dd) dd[i] = v;
                            if (ws == LA_EXCH) {
                                const uint32_t m = l2_mix(v, (uint32_t)ll);
                                esum += m;
                                exor ^= m;
                            } else {
                                err += v != __ldg(tt + kL2AtomFinalOff + ws * (kL2AtomMaxN + 1) + l2_atom_n((int)G, rr));
                            }
                            l2_st32(data + i, __ldg(nt + kL2AtomFinalOff + ws * (kL2AtomMaxN + 1)));
                        }
                        // the combined folds against the host's, per return op
                        uint32_t fs[kL2AtomRet] = {}, fx[kL2AtomRet] = {};
                        for (uint32_t cc = tid; cc < G; cc += kCtThreads)
#pragma unroll
                            for (int k = 0; k < kL2AtomRet; ++k) {
                                fs[k] += l2_ld32(scratch + kL2HdrWords + cc * kL2FoldWords + k);
                                fx[k] ^= l2_ld32(scratch + kL2HdrWords + cc * kL2FoldWords + kL2AtomRet + k);
                            }
                        fs[3] += esum;
                        fx[3] ^= exor;
#pragma unroll
                        for (int k = 0; k < kL2AtomRet; ++k)
#pragma unroll
                            for (int o = 16; o; o >>= 1) {
                                fs[k] += __shfl_xor_sync(0xffffffffu, fs[k], o);
                                fx[k] ^= __shfl_xor_sync(0xffffffffu, fx[k], o);
                            }
#pragma unroll
                        for (int o = 16; o; o >>= 1) err += __shfl_xor_sync(0xffffffffu, err, o);
                        __syncthreads();
                        if (lane == 0) {
#pragma unroll
                            for (int k = 0; k < kL2AtomRet; ++k) { s_red[warp][k] = fs[k]; s_red[warp][kL2AtomRet + k] = fx[k]; }
                            s_red[warp][2 * kL2AtomRet] = err;
                        }
                        __syncthreads();
                        if (tid < kL2AtomRet) {
                            uint32_t gs = 0, gx = 0, es = 0, ex = 0;
                            for (int w = 0; w < 4; ++w) { gs += s_red[w][tid]; gx ^= s_red[w][kL2AtomRet + tid]; }
                            for (int rr = 0; rr < kL2AtomRows; ++rr) {
                                const int n = l2_atom_n((int)G, rr);
                                es += __ldg(tt + kL2AtomSumOff + tid * (kL2AtomMaxN + 1) + n);
                                ex ^= __ldg(tt + kL2AtomXorOff + tid * (kL2AtomMaxN + 1) + n);
                            }
                            if (dd) {
                                dd[kL2AtomHotWords + tid] = gs;
                                dd[kL2AtomHotWords + kL2AtomRet + tid] = gx;
                                dd[kL2AtomHotWords + 2 * kL2AtomRet + tid] = es;
                                dd[kL2AtomHotWords + 3 * kL2AtomRet + tid] = ex;
                            }
                            s_red[0][tid] = (gs != es) | ((gx != ex) << 1);
                        }
                        __syncthreads();
                        uint32_t any = s_red[0][2 * kL2AtomRet] | s_red[1][2 * kL2AtomRet] | s_red[2][2 * kL2AtomRet] |
                                       s_red[3][2 * kL2AtomRet];
                        for (int k = 0; k < kL2AtomRet; ++k) any |= s_red[0][k];
                        bad = any != 0;
                    }
                    // the last comparison of a round: CTA 0 decides whether it was the last round
                    const bool round_end = tile == kCtTiles - 1 && rep == kCtReps - 1;
                    if (round_end && c == 0 && tid == 0) l2_st32(hdr + kL2HdrStop, globaltimer_ns() >= t_end ? 1u : 0u);
                    if (!l2_grid_sync(hdr, t_bound, &s_ok)) { ok = false; break; }
                    if (round_end) stop = (int)l2_ld32(hdr + kL2HdrStop);
                    ++comparisons;
                    if (bad && mismatches++ == 0) { bad_tile = tile; bad_rep = rep; }
                }
            }
            if (ok) ++rounds;
        }
    } else {
        const int t = tid;
        int stop = 0;
        while (ok && !stop) {
            uint32_t* win = data + (size_t)(rounds % kL2Windows) * span_words;
            for (int tile = 0; tile < kCtTiles && ok; ++tile) {
                const uint32_t* tt = tab + tile * kL2TableWords;
                const uint32_t kind = __ldg(tt), key = __ldg(tt + 1), blockmul = __ldg(tt + 2);
                const uint32_t hook_word = __ldg(tt + 3), hook_elem = __ldg(tt + 4);
                uint32_t pl[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) pl[i] = sh_pattern(kind, key, (uint32_t)(4 * t + i));
                const uint32_t want = __ldg(checks + tile * kCtThreads + t) * K;
                for (int rep = 0; rep < kCtReps && ok; ++rep) {
                    const bool first = (rounds | (unsigned)tile | (unsigned)rep) == 0;
                    L2Acc a;
                    // after every element: a grid barrier, and in the first comparison the hook and one more barrier
                    auto sep = [&](uint32_t e) {
                        if (!ok) return;
                        if (!l2_grid_sync(hdr, t_bound, &s_ok)) { ok = false; return; }
                        if (first && e == hook_elem) {
                            if (tid == 0 && claim()) {
                                uint32_t* p = win + (size_t)((c + e) % G) * K * kL2BlockWords + hook_word % (K * kL2BlockWords);
                                l2_st32(p, l2_ld32(p) ^ fault_mask);
                            }
                            if (!l2_grid_sync(hdr, t_bound, &s_ok)) ok = false;
                        }
                    };
                    const uint32_t s0 = c % G, s1 = (c + 1) % G, s2 = (c + 2) % G, s3 = (c + 3) % G;
                    if constexpr (FMT == L2_WORD) {
                        const uint32_t s4 = (c + 4) % G, s5 = (c + 5) % G;
                        l2_element<FMT, L2_W, true, 0>(win, s0, K, blockmul, pl, 0u, 0u, a);
                        sep(0);
                        if (ok) l2_element<FMT, L2_RW, true, 0>(win, s1, K, blockmul, pl, 0u, ~0u, a);
                        sep(1);
                        if (ok) l2_element<FMT, L2_RW, true, 1>(win, s2, K, blockmul, pl, ~0u, 0u, a);
                        sep(2);
                        if (ok) l2_element<FMT, L2_RW, false, 2>(win, s3, K, blockmul, pl, 0u, ~0u, a);
                        sep(3);
                        if (ok) l2_element<FMT, L2_RW, false, 3>(win, s4, K, blockmul, pl, ~0u, 0u, a);
                        sep(4);
                        if (ok) l2_element<FMT, L2_R, true, 4>(win, s5, K, blockmul, pl, 0u, 0u, a);
                    } else {
                        l2_element<FMT, L2_W, true, 1>(win, s0, K, blockmul, pl, 0u, 0u, a);
                        sep(0);
                        if (ok) l2_element<FMT, L2_RW, true, 0>(win, s1, K, blockmul, pl, 0u, ~0u, a);
                        sep(1);
                        if (ok) l2_element<FMT, L2_RW, false, 1>(win, s2, K, blockmul, pl, ~0u, 0u, a);
                        sep(2);
                        if (ok) l2_element<FMT, L2_R, true, 2>(win, s3, K, blockmul, pl, 0u, 0u, a);
                    }
                    if (!ok) break;
                    if (DUMP && rounds == 0 && rep == 0) {
                        uint32_t* d = dump + ((size_t)tile * G + c) * 2 * kCtThreads;
                        d[t] = a.h;
                        d[kCtThreads + t] = a.err;
                        // the last element's slice, as the window holds it now
                        const uint32_t sl = (c + kL2Elements[FMT] - 1) % G, n = K * kL2BlockWords;
                        uint32_t* img = dump + (size_t)kCtTiles * G * 2 * kCtThreads + (size_t)tile * span_words +
                                        (size_t)sl * n;
                        const uint32_t* src = win + (size_t)sl * n;
#pragma unroll 1
                        for (uint32_t w = t; w < n; w += kCtThreads) img[w] = l2_ld32(src + w);
                    }
                    const int bad = __syncthreads_or(a.err != 0 || a.h != want);
                    const bool round_end = tile == kCtTiles - 1 && rep == kCtReps - 1;
                    if (round_end && c == 0 && tid == 0) l2_st32(hdr + kL2HdrStop, globaltimer_ns() >= t_end ? 1u : 0u);
                    // ends the comparison: the next one's first element writes slices this one's last element read
                    if (!l2_grid_sync(hdr, t_bound, &s_ok)) { ok = false; break; }
                    if (round_end) stop = (int)l2_ld32(hdr + kL2HdrStop);
                    ++comparisons;
                    if (bad && mismatches++ == 0) { bad_tile = tile; bad_rep = rep; }
                }
            }
            if (ok) ++rounds;
        }
    }
    if (tid == 0) {
        volatile CtRecord* r = rec + blockIdx.x;
        r->smid = smid;
        r->nsmid = nsmid;
        r->rounds = ok ? rounds : 0ull;  // a CTA that gave up waiting reports an incomplete record
        r->comparisons = comparisons;
        r->mismatches = mismatches;
        r->first_bad_tile = bad_tile;
        r->first_bad_rep = bad_rep;
        __threadfence_system();
        r->seq = seq;
    }
}

}  // namespace b2dp
