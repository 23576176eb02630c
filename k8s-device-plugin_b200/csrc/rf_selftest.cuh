// rf_selftest.cuh -- sm_90a self-test kernel of the on-demand register-file self-test (b2dp_regfile_test).
//
// Two CTAs of 128 threads per SM (__launch_bounds__(128, 2): up to 255 registers per thread, allocated as 256, so the
// two CTAs take the SM's whole 64 K-register file).  Every thread holds kRfHeld values in general registers and marches
// them with the marches of rf_test_math.hpp:
//     format    writes of the held registers                                  SASS
//     RF_ALU    March C-: in-place LOP3 (r ^= m) after a first ld.shared.v4     LOP3.LUT Rd == Ra, LDS.128
//     RF_LOAD   ld.shared.v4 / ld.shared.v2 of P and ~P into quads and pairs     LDS.128, LDS.64
//     RF_HOLD   ld.shared.v4, then an in-place LOP3, each held kRfHoldNs         NANOSLEEP
//
// The round / tile / repetition structure is the other self-tests': a round runs each of the kCtTiles tiles kCtReps
// times, and a CTA repeats rounds until its %globaltimer deadline (at least one round).  A tile is a data background
// (its table: kind, key).  One comparison is one (tile, repetition): one march over the held registers.  It is a
// mismatch if, for any thread,
//   (a) a held value read differs from P or ~P, which the kernel computes from the tile's generator, or
//   (b) the thread's fold of every held value it read, in read order, differs from the host's check (rf_reads).
// (a) is what catches a stuck bit: March C- reads it wrong twice, and at bit 31 two such errors cancel in the fold.
//
// Keeping the march in registers.  ptxas keeps a value in a register only if it cannot do better, so:
//   - the held values enter through shared-memory loads (the image, refilled with P at every tile), which ptxas cannot
//     recompute; a value derived from a key would be rematerialised after each barrier instead of held;
//   - after every barrier each thread re-loads the generator and the transition mask m (= ~0) with ld.volatile.shared,
//     so no element's expected values or transitions can be hoisted above its barrier or shared with another element;
//   - before every barrier each thread stores (volatile) a word that depends on every compare, the fold and every
//     transitioned value of the element, so none of them can sink below it;
//   - a transition is the only reader of the value it replaces (RfAcc::take_flipped), so ptxas writes it in place.
// tests/test_regfile_test_cpu.py checks the result in the SASS, leaving out the hook's cold code: no local memory,
// kRfHeld registers held across every barrier (last written by the element's load or transition, first touched after
// it by a read), every transition ending the value it replaces, and how many are in place (DESIGN 4.10).
//
// Fault hook: in the first comparison (round 0, tile 0, repetition 0), after element table[3] of tile 0, thread
// table[4] of a CTA whose %smid == fault_sm XORs fault_mask into held register table[2] (the product: register
// kRfHookReg of thread 0 after element 0).  The register index is a compile-time-unrolled, predicated select behind a
// branch no clean run takes: an indexed register array would be placed in local memory.
//
// DUMP (the test harness only): round 0, repetition 0 of every tile writes every thread's held registers after the
// march, then its fold and the OR of its direct-compare differences, to dump + (blockIdx.x * kCtTiles + tile) *
// kRfDumpWords (register j of thread t at word j * kCtThreads + t).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "hbm_probe.cuh"  // globaltimer_ns
#include "rf_test_math.hpp"

namespace b2dp {

__device__ __forceinline__ uint32_t rf_ldv(uint32_t a) {
    uint32_t v;
    asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void rf_stv(uint32_t a, uint32_t v) {
    asm volatile("st.volatile.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void rf_ld128(uint32_t a, uint32_t& x, uint32_t& y, uint32_t& z, uint32_t& w) {
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "r"(a) : "memory");
}
__device__ __forceinline__ void rf_ld64(uint32_t a, uint32_t& x, uint32_t& y) {
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(x), "=r"(y) : "r"(a) : "memory");
}
__device__ __forceinline__ void rf_st128(uint32_t a, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ void rf_st64(uint32_t a, uint32_t x, uint32_t y) {
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory");
}

// Shared memory: [0, kRfParamWords) the generator (mul, even, odd, one), the mask, an opaque 0, the deadline and the
// tallies (mismatches, first bad tile and repetition), then one pin word and one check value per thread,
// then the image: quad q (registers 4q .. 4q + 3) of thread t at byte 16 (q * kCtThreads + t), pair p (registers 2p,
// 2p + 1) in the half p & 1 of quad p / 2.
constexpr uint32_t kRfMaskByte = 16;
constexpr uint32_t kRfZeroByte = 20;
constexpr uint32_t kRfDeadlineByte = 24;
constexpr uint32_t kRfTallyByte = 32;
constexpr uint32_t kRfPinByte = 4u * kRfParamWords;
constexpr uint32_t kRfCheckByte = kRfPinByte + 4u * kCtThreads;
constexpr uint32_t kRfImageByte = kRfCheckByte + 4u * kCtThreads;
static_assert(kRfImageByte % 16 == 0, "the image holds 16-byte quads");

__device__ __forceinline__ uint32_t rf_quad(uint32_t base, int t, int q) {
    return base + kRfImageByte + 16u * (uint32_t)(q * kCtThreads + t);
}

// The generator of this thread, loaded afresh after a barrier: P(t, j) = (tm + j * mul) ^ (j odd ? odd : even) ^
// rotl(rl, j), tm = t * kRfHeld * mul, rl = rotl(one, t).
struct RfGen {
    uint32_t tm, mul, even, odd, rl;
    __device__ __forceinline__ uint32_t want(int j, bool inv) const {  // j, inv: constants once unrolled
        const uint32_t p = (tm + (uint32_t)j * mul) ^ ((j & 1) ? odd : even) ^ __funnelshift_l(rl, rl, (uint32_t)j);
        return inv ? ~p : p;
    }
};
__device__ __forceinline__ RfGen rf_gen(uint32_t base, int t) {
    RfGen g;
    g.mul = rf_ldv(base);
    g.even = rf_ldv(base + 4);
    g.odd = rf_ldv(base + 8);
    const uint32_t one = rf_ldv(base + 12);
    g.tm = (uint32_t)t * (uint32_t)kRfHeld * g.mul;
    g.rl = __funnelshift_l(one, one, (uint32_t)t);
    return g;
}

// A thread's fold (read i enters with weight 2i + 1), the OR of its direct-compare differences, and the sum of the
// values its transitions wrote (the pin word's share of them; a sum, because ptxas would rewrite an XOR of u = v ^ m
// as one of v and m, and keep v alive past its transition).
struct RfAcc {
    uint32_t h = 0u, err = 0u, x = 0u;
    __device__ __forceinline__ void take(uint32_t i, uint32_t v, uint32_t want) {  // i: a constant once unrolled
        h += (2u * i + 1u) * v;
        err |= v ^ want;
    }
    // The same read, taken from u = v ^ m, what the in-place transition of v wrote: with m = ~0, v = ~u = -1 - u, so
    // (2i + 1) v = -(2i + 1)(u + 1) and u ^ ~want = v ^ want.  The fold and the error bits are those of v, and a wrong
    // mask changes both.  The transition is then the only reader of v, so ptxas has no reason to keep v alive and
    // write u to another register.
    __device__ __forceinline__ void take_flipped(uint32_t i, uint32_t u, uint32_t want) {
        h -= (2u * i + 1u) * (u + 1u);
        err |= u ^ ~want;
    }
    __device__ __forceinline__ uint32_t pin() const { return h ^ err ^ x; }
};

// One element's reads and in-place transitions over every held register (j ascending, or descending when DOWN): the
// element reads register j as read i0 + k, against P (~P when INV); FLIP XORs the mask into it in place first, and
// the read is taken from the transitioned value (RfAcc::take_flipped).
template <bool DOWN, bool INV, bool FLIP>
__device__ __forceinline__ void rf_alu_element(uint32_t (&r)[kRfHeld], const RfGen& g, uint32_t m, uint32_t i0,
                                               RfAcc& a) {
#pragma unroll
    for (int k = 0; k < kRfHeld; ++k) {
        const int j = DOWN ? kRfHeld - 1 - k : k;
        if (FLIP) {
            r[j] ^= m;
            a.take_flipped(i0 + (uint32_t)k, r[j], g.want(j, INV));
            a.x += r[j];
        } else {
            a.take(i0 + (uint32_t)k, r[j], g.want(j, INV));
        }
    }
}

// Every held register loaded from the image as quads.
__device__ __forceinline__ void rf_load_quads(uint32_t (&r)[kRfHeld], uint32_t base, int t) {
#pragma unroll
    for (int q = 0; q < kRfHeld / 4; ++q) rf_ld128(rf_quad(base, t, q), r[4 * q], r[4 * q + 1], r[4 * q + 2], r[4 * q + 3]);
}

// One RF_LOAD element, quad by quad (WIDTH 4) or pair by pair (WIDTH 2): when READ, compare the registers with P (~P
// when INV) as reads i0 + j; load them from the image, which holds the complement of what they held; then store into
// the image what they held, for the next element's load.  The image is the thread's own, so no barrier separates the
// load from the store.  Each load's address carries (fold ^ err) & z, z an opaque 0: ptxas would otherwise issue the
// loads ahead of the compares and hold old and new values at once.
template <int WIDTH, bool READ, bool INV>
__device__ __forceinline__ void rf_load_element(uint32_t (&r)[kRfHeld], uint32_t base, int t, const RfGen& g,
                                                uint32_t i0, RfAcc& a) {
    const uint32_t z = rf_ldv(base + kRfZeroByte);
#pragma unroll
    for (int q = 0; q < kRfHeld / WIDTH; ++q) {
        uint32_t w[WIDTH];
#pragma unroll
        for (int i = 0; i < WIDTH; ++i) {
            const int j = WIDTH * q + i;
            w[i] = g.want(j, INV);
            if (READ) a.take(i0 + (uint32_t)j, r[j], w[i]);
        }
        if constexpr (WIDTH == 4) {
            const uint32_t addr = rf_quad(base, t, q) + ((a.h ^ a.err) & z);
            rf_ld128(addr, r[4 * q], r[4 * q + 1], r[4 * q + 2], r[4 * q + 3]);
            rf_st128(addr, w[0], w[1], w[2], w[3]);
        } else {
            const uint32_t addr = rf_quad(base, t, q / 2) + 8u * (uint32_t)(q & 1) + ((a.h ^ a.err) & z);
            rf_ld64(addr, r[2 * q], r[2 * q + 1]);
            rf_st64(addr, w[0], w[1]);
        }
    }
}

__device__ __forceinline__ uint32_t rf_ldg_volatile(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// The fault hook: XOR fault_mask into held register tt[2] of thread tt[4] without indexing the array.  The table is
// read here, with volatile loads, so that no select can be computed ahead of the branch and held in registers.
__device__ __forceinline__ void rf_hook(uint32_t (&r)[kRfHeld], const uint32_t* tt, int tid, uint32_t fault_mask) {
    const uint32_t reg = rf_ldg_volatile(tt + 2);
    const uint32_t fm = (uint32_t)tid == rf_ldg_volatile(tt + 4) ? fault_mask : 0u;
#pragma unroll
    for (int j = 0; j < kRfHeld; ++j) r[j] ^= reg == (uint32_t)j ? fm : 0u;
}

// RF_HOLD: every thread of the CTA sleeps for kRfHoldNs, by its own %globaltimer.
__device__ __forceinline__ void rf_hold() {
    const unsigned long long t1 = globaltimer_ns() + kRfHoldNs;
    while (globaltimer_ns() < t1) __nanosleep(kRfSleepNs);
}

// table: kCtTiles tables of kRfTableWords words; checks: [kCtTiles][kCtThreads] (DUMP: may be null); rec: one per CTA.
// Block: kCtThreads threads, kRfSmemBytes of dynamic shared memory.  Same signature as tc_selftest.
template <int FMT, bool DUMP>
__global__ void __launch_bounds__(kCtThreads, 2)
rf_selftest(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks, unsigned long long duration_ns,
            int fault_sm, uint32_t fault_mask, CtRecord* rec, unsigned long long seq, uint32_t* dump) {
    extern __shared__ __align__(16) uint32_t rf_smem[];
    const int tid = threadIdx.x;
    uint32_t smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const uint32_t base = (uint32_t)__cvta_generic_to_shared(rf_smem);
    // The deadline and the tallies live in shared memory (thread 0's), so that the registers are the march's.
    if (tid == 0) {
        const unsigned long long t_end = globaltimer_ns() + duration_ns;
        rf_stv(base + kRfDeadlineByte, (uint32_t)t_end);
        rf_stv(base + kRfDeadlineByte + 4, (uint32_t)(t_end >> 32));
        rf_stv(base + kRfTallyByte, 0u);
        rf_stv(base + kRfTallyByte + 4, ~0u);
        rf_stv(base + kRfTallyByte + 8, ~0u);
    }
    const bool compare = !DUMP || checks != nullptr;
    const uint32_t* tab = reinterpret_cast<const uint32_t*>(table);
    const bool hook_here = (int)smid == fault_sm;
    uint32_t rounds = 0;
    uint32_t r[kRfHeld];
    for (;;) {
        for (int tile = 0; tile < kCtTiles; ++tile) {
            const uint32_t* tt = tab + tile * kRfTableWords;
            const uint32_t hook_elem = __ldg(tt + 3);
            {   // the generator and the mask for this tile, and the image of P
                __syncthreads();  // every thread is done with the last tile's generator
                if (tid == 0) {
                    const RfGenParams p = rf_gen_params(__ldg(tt), __ldg(tt + 1));
                    rf_stv(base, p.mul);
                    rf_stv(base + 4, p.even);
                    rf_stv(base + 8, p.odd);
                    rf_stv(base + 12, p.one);
                    rf_stv(base + kRfMaskByte, ~0u);
                    rf_stv(base + kRfZeroByte, 0u);
                }
                __syncthreads();
                rf_stv(base + kRfCheckByte + 4u * (uint32_t)tid, compare ? __ldg(checks + tile * kCtThreads + tid) : 0u);
                const RfGen g = rf_gen(base, tid);
#pragma unroll 4
                for (int q = 0; q < kRfHeld / 4; ++q)
                    rf_st128(rf_quad(base, tid, q), g.want(4 * q, false), g.want(4 * q + 1, false),
                             g.want(4 * q + 2, false), g.want(4 * q + 3, false));
            }
            for (int rep = 0; rep < kCtReps; ++rep) {
                const bool first = (rounds | (unsigned)tile | (unsigned)rep) == 0;
                RfAcc a;
                // after every element: its pin word, a barrier, and in the first comparison the fault hook
                auto sep = [&](uint32_t e) {
                    rf_stv(base + kRfPinByte + 4u * (uint32_t)tid, a.pin());
                    __syncthreads();
                    if (first && e == hook_elem && hook_here) rf_hook(r, tt, tid, fault_mask);
                };
                if constexpr (FMT == RF_ALU) {
                    rf_load_quads(r, base, tid);
                    sep(0);
                    {
                        const RfGen g = rf_gen(base, tid);
                        rf_alu_element<false, false, true>(r, g, rf_ldv(base + kRfMaskByte), 0, a);
                    }
                    sep(1);
                    {
                        const RfGen g = rf_gen(base, tid);
                        rf_alu_element<false, true, true>(r, g, rf_ldv(base + kRfMaskByte), kRfHeld, a);
                    }
                    sep(2);
                    {
                        const RfGen g = rf_gen(base, tid);
                        rf_alu_element<true, false, true>(r, g, rf_ldv(base + kRfMaskByte), 2 * kRfHeld, a);
                    }
                    sep(3);
                    {
                        const RfGen g = rf_gen(base, tid);
                        rf_alu_element<true, true, true>(r, g, rf_ldv(base + kRfMaskByte), 3 * kRfHeld, a);
                    }
                    sep(4);
                    {
                        const RfGen g = rf_gen(base, tid);
                        rf_alu_element<false, false, false>(r, g, 0u, 4 * kRfHeld, a);
                    }
                    sep(5);
                } else if constexpr (FMT == RF_LOAD) {
                    rf_load_element<4, false, true>(r, base, tid, rf_gen(base, tid), 0, a);
                    sep(0);
                    rf_load_element<4, true, false>(r, base, tid, rf_gen(base, tid), 0, a);
                    sep(1);
                    rf_load_element<2, true, true>(r, base, tid, rf_gen(base, tid), kRfHeld, a);
                    sep(2);
                    rf_load_element<2, true, false>(r, base, tid, rf_gen(base, tid), 2 * kRfHeld, a);
                    sep(3);
                    {
                        const RfGen g = rf_gen(base, tid);
                        rf_alu_element<false, true, false>(r, g, 0u, 3 * kRfHeld, a);
                    }
                    sep(4);
                } else {
                    rf_load_quads(r, base, tid);
                    sep(0);
                    rf_hold();
                    {
                        const RfGen g = rf_gen(base, tid);
                        rf_alu_element<false, false, true>(r, g, rf_ldv(base + kRfMaskByte), 0, a);
                    }
                    sep(1);
                    rf_hold();
                    {
                        const RfGen g = rf_gen(base, tid);
                        rf_alu_element<false, true, false>(r, g, 0u, kRfHeld, a);
                    }
                    sep(2);
                }
                if (DUMP && rounds == 0 && rep == 0) {
                    uint32_t* d = dump + ((size_t)blockIdx.x * kCtTiles + tile) * kRfDumpWords;
#pragma unroll
                    for (int j = 0; j < kRfHeld; ++j) d[j * kCtThreads + tid] = r[j];
                    d[kRfImageWords + tid] = a.h;
                    d[kRfImageWords + kCtThreads + tid] = a.err;
                }
                // the check is loaded here, not ahead of the repetitions, where it (or its address) would take
                // registers throughout
                const bool wrong = compare && (a.err != 0 || a.h != rf_ldv(base + kRfCheckByte + 4u * (uint32_t)tid));
                const int bad = __syncthreads_or(wrong);
                if (bad && tid == 0) {  // the mismatch count, and the first mismatch's tile and repetition
                    const uint32_t n = rf_ldv(base + kRfTallyByte);
                    rf_stv(base + kRfTallyByte, n + 1u);
                    if (n == 0) {
                        rf_stv(base + kRfTallyByte + 4, (uint32_t)tile);
                        rf_stv(base + kRfTallyByte + 8, (uint32_t)rep);
                    }
                }
            }
        }
        ++rounds;
        const unsigned long long t_end =
            rf_ldv(base + kRfDeadlineByte) | (unsigned long long)rf_ldv(base + kRfDeadlineByte + 4) << 32;
        if (__syncthreads_or(tid == 0 && globaltimer_ns() >= t_end)) break;
    }
    if (tid == 0) {
        volatile CtRecord* rc = rec + blockIdx.x;
        rc->smid = smid;
        rc->nsmid = nsmid;
        rc->rounds = rounds;
        rc->comparisons = (unsigned long long)rounds * kCtTiles * kCtReps;
        rc->mismatches = rf_ldv(base + kRfTallyByte);
        rc->first_bad_tile = (int)rf_ldv(base + kRfTallyByte + 4);
        rc->first_bad_rep = (int)rf_ldv(base + kRfTallyByte + 8);
        __threadfence_system();
        rc->seq = seq;
    }
}

}  // namespace b2dp
