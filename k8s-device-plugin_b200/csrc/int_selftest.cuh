// int_selftest.cuh -- sm_90a self-test kernel of the on-demand integer and warp-exchange self-test (b2dp_int_test).
//
// Four warps per CTA run the SM's integer pipes and its lane-exchange network on operands the host generated, and
// compare against results the host computed exactly (int_test_math.hpp).  Every op under test is inline PTX and runs
// on every operand set of its format (20 / 12 / 12 sets per thread):
//     format  PTX under test, per set                                                       result words per set
//     MAD     mad.lo.u32, mul.hi.u32, mul.hi.s32, mad.wide.u32, mad.wide.s32,               14
//             add.cc + addc, sub.cc + subc (64-bit through the carry flag), dp4a s32.s32 / s32.u32 / u32.u32
//     BIT     lop3.b32 x 8 immediates, shf.l.wrap, shf.r.wrap, shr.s32, shl.b32, popc, clz (of b), bfind.u32, bfind.s32,
//             brev, prmt (selector from a register), min / max .s32 / .u32, sad.u32          23
//     WARP    shfl.sync.idx / .up / .down / .bfly (b and c from registers, d|p form), vote.sync.ballot,
//             redux.sync.add / min.s32 / max.s32 / min.u32 / max.u32 / and / or / xor, match.any, match.all (d|p)
//                                                                                            20
// The results are independent -- no result feeds another op under test, because a later op would hide an earlier wrong
// bit -- and every result word enters the thread's fold (it_fold: four multiply-and-rotate chains) as it is produced.  In
// MAD the fold's own IMAD and LOP3 are part of what the comparison verifies.
//
// The round / tile / repetition structure is tc_selftest's and fp_selftest's: a round runs each of the kCtTiles tiles
// kCtReps times, and a CTA repeats rounds until its %globaltimer deadline (at least one round).  Per tile every thread
// loads its operands from an L2-resident table ([slot][thread] words) into registers, and its comparison value; each
// repetition feeds the ops operands the compiler must treat as changed (sf_perturb's device: v ^ (rep & zero)), so no
// op leaves the repetition loop.  Every thread then compares its fold with the host's; the CTA counts the repetition as
// one mismatch if any thread disagrees, and publishes one CtRecord.  WARP uses the full member mask only: all 32 lanes
// of every warp are converged at every op.
//
// Test hooks: as tc_selftest -- in round 0, thread 0 of a CTA whose %smid == fault_sm XORs fault_mask into its first
// result word of tile 0, repetition 0, before the fold.  DUMP (instantiated only by tests/native/int_test_kernels.cu)
// makes CTA 0 write every result word of repetition 0 of every tile of round 0 to dump[tile][thread][kItWords[FMT]].
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "hbm_probe.cuh"  // globaltimer_ns
#include "int_test_math.hpp"

namespace b2dp {

#define B2DP_IT_OP2(NAME, PTX)                                                 \
    __device__ __forceinline__ uint32_t NAME(uint32_t a, uint32_t b) {         \
        uint32_t d;                                                            \
        asm volatile(PTX " %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));           \
        return d;                                                              \
    }
#define B2DP_IT_OP3(NAME, PTX)                                                 \
    __device__ __forceinline__ uint32_t NAME(uint32_t a, uint32_t b, uint32_t c) { \
        uint32_t d;                                                            \
        asm volatile(PTX " %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); \
        return d;                                                              \
    }
#define B2DP_IT_OP1(NAME, PTX)                                                 \
    __device__ __forceinline__ uint32_t NAME(uint32_t a) {                     \
        uint32_t d;                                                            \
        asm volatile(PTX " %0, %1;" : "=r"(d) : "r"(a));                       \
        return d;                                                              \
    }
B2DP_IT_OP3(it_mad_lo, "mad.lo.u32")
B2DP_IT_OP2(it_mul_hi_u, "mul.hi.u32")
B2DP_IT_OP2(it_mul_hi_s, "mul.hi.s32")
B2DP_IT_OP3(it_dp4a_ss, "dp4a.s32.s32")
B2DP_IT_OP3(it_dp4a_su, "dp4a.s32.u32")
B2DP_IT_OP3(it_dp4a_uu, "dp4a.u32.u32")
B2DP_IT_OP3(it_shf_l, "shf.l.wrap.b32")
B2DP_IT_OP3(it_shf_r, "shf.r.wrap.b32")
B2DP_IT_OP2(it_shr_s, "shr.s32")
B2DP_IT_OP2(it_shl_b, "shl.b32")
B2DP_IT_OP1(it_popc_b, "popc.b32")
B2DP_IT_OP1(it_clz_b, "clz.b32")
B2DP_IT_OP1(it_bfind_ub, "bfind.u32")
B2DP_IT_OP1(it_bfind_sb, "bfind.s32")
B2DP_IT_OP1(it_brev_b, "brev.b32")
B2DP_IT_OP3(it_prmt_b, "prmt.b32")
B2DP_IT_OP2(it_min_sb, "min.s32")
B2DP_IT_OP2(it_max_sb, "max.s32")
B2DP_IT_OP2(it_min_ub, "min.u32")
B2DP_IT_OP2(it_max_ub, "max.u32")
B2DP_IT_OP3(it_sad_ub, "sad.u32")
#undef B2DP_IT_OP1
#undef B2DP_IT_OP2
#undef B2DP_IT_OP3

template <bool SIGNED>
__device__ __forceinline__ void it_mad_wide(uint32_t a, uint32_t b, uint32_t ylo, uint32_t yhi, uint32_t& lo,
                                            uint32_t& hi) {
    if (SIGNED)
        asm volatile("{ .reg .b64 y, d; mov.b64 y, {%4, %5}; mad.wide.s32 d, %2, %3, y; mov.b64 {%0, %1}, d; }"
                     : "=r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(ylo), "r"(yhi));
    else
        asm volatile("{ .reg .b64 y, d; mov.b64 y, {%4, %5}; mad.wide.u32 d, %2, %3, y; mov.b64 {%0, %1}, d; }"
                     : "=r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(ylo), "r"(yhi));
}
// (b:a) + (d:c) and (b:a) - (d:c) through the carry flag; one asm statement each, so nothing comes between the pair
__device__ __forceinline__ void it_add64(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t& lo, uint32_t& hi) {
    asm volatile("add.cc.u32 %0, %2, %4; addc.u32 %1, %3, %5;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(c), "r"(d));
}
__device__ __forceinline__ void it_sub64(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t& lo, uint32_t& hi) {
    asm volatile("sub.cc.u32 %0, %2, %4; subc.u32 %1, %3, %5;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(c), "r"(d));
}
template <uint32_t IMM>
__device__ __forceinline__ uint32_t it_lop3_b(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm volatile("lop3.b32 %0, %1, %2, %3, %4;" : "=r"(d) : "r"(a), "r"(b), "r"(c), "n"(IMM));
    return d;
}

#define B2DP_IT_SHFL(NAME, MODE)                                                                        \
    __device__ __forceinline__ void NAME(uint32_t v, uint32_t b, uint32_t c, uint32_t& d, uint32_t& p) { \
        asm volatile("{ .reg .pred q; shfl.sync." MODE ".b32 %0|q, %2, %3, %4, 0xffffffff; selp.u32 %1, 1, 0, q; }" \
                     : "=r"(d), "=r"(p) : "r"(v), "r"(b), "r"(c));                                       \
    }
B2DP_IT_SHFL(it_shfl_idx, "idx")
B2DP_IT_SHFL(it_shfl_up, "up")
B2DP_IT_SHFL(it_shfl_down, "down")
B2DP_IT_SHFL(it_shfl_bfly, "bfly")
#undef B2DP_IT_SHFL
__device__ __forceinline__ uint32_t it_ballot(uint32_t q) {
    uint32_t d;
    asm volatile("{ .reg .pred q; setp.ne.u32 q, %1, 0; vote.sync.ballot.b32 %0, q, 0xffffffff; }" : "=r"(d) : "r"(q));
    return d;
}
#define B2DP_IT_REDUX(NAME, OP)                                                          \
    __device__ __forceinline__ uint32_t NAME(uint32_t r) {                               \
        uint32_t d;                                                                      \
        asm volatile("redux.sync." OP " %0, %1, 0xffffffff;" : "=r"(d) : "r"(r));         \
        return d;                                                                        \
    }
B2DP_IT_REDUX(it_redux_add, "add.u32")
B2DP_IT_REDUX(it_redux_min_s, "min.s32")
B2DP_IT_REDUX(it_redux_max_s, "max.s32")
B2DP_IT_REDUX(it_redux_min_u, "min.u32")
B2DP_IT_REDUX(it_redux_max_u, "max.u32")
B2DP_IT_REDUX(it_redux_and, "and.b32")
B2DP_IT_REDUX(it_redux_or, "or.b32")
B2DP_IT_REDUX(it_redux_xor, "xor.b32")
#undef B2DP_IT_REDUX
__device__ __forceinline__ uint32_t it_match_any(uint32_t m) {
    uint32_t d;
    asm volatile("match.any.sync.b32 %0, %1, 0xffffffff;" : "=r"(d) : "r"(m));
    return d;
}
__device__ __forceinline__ void it_match_all(uint32_t m, uint32_t& d, uint32_t& p) {
    asm volatile("{ .reg .pred q; match.all.sync.b32 %0|q, %2, 0xffffffff; selp.u32 %1, 1, 0, q; }"
                 : "=r"(d), "=r"(p) : "r"(m));
}

// The thread's fold in progress (it_fold) and where its result words go.
template <bool DUMP>
struct ItSink {
    uint32_t h[4];
    uint32_t inj;
    uint32_t* dump;
    // result word J: the fault hook on word 0, the dump, and chain J % 4
    template <int J>
    __device__ __forceinline__ void emit(uint32_t w) {
        if (J == 0) w ^= inj;
        if (DUMP && dump) dump[J] = w;
        const uint32_t x = (h[J & 3] ^ w) * kItMul;
        h[J & 3] = __funnelshift_l(x, x, kItFoldRot);
    }
    __device__ __forceinline__ uint32_t value() const {
        return h[0] ^ __funnelshift_l(h[1], h[1], 8) ^ __funnelshift_l(h[2], h[2], 16) ^ __funnelshift_l(h[3], h[3], 24);
    }
};

// Set S of format FMT on this repetition's operand words o[0 .. kItSetSlots[FMT]), in int_test_math.hpp's word order.
template <int FMT, int S, bool DUMP>
__device__ __forceinline__ void it_set(const uint32_t* o, ItSink<DUMP>& k) {
    constexpr int J = S * kItSetWords[FMT];
    if constexpr (FMT == IT_MAD) {
        const uint32_t a = o[0], b = o[1], c = o[2], d = o[3];
        uint32_t lo, hi;
        k.template emit<J + IM_MAD_LO>(it_mad_lo(a, b, c));
        k.template emit<J + IM_MULHI_U>(it_mul_hi_u(a, b));
        k.template emit<J + IM_MULHI_S>(it_mul_hi_s(a, b));
        it_mad_wide<false>(a, b, c, d, lo, hi);
        k.template emit<J + IM_WIDE_U_LO>(lo);
        k.template emit<J + IM_WIDE_U_HI>(hi);
        it_mad_wide<true>(a, b, c, d, lo, hi);
        k.template emit<J + IM_WIDE_S_LO>(lo);
        k.template emit<J + IM_WIDE_S_HI>(hi);
        it_add64(a, b, c, d, lo, hi);
        k.template emit<J + IM_ADD_LO>(lo);
        k.template emit<J + IM_ADD_HI>(hi);
        it_sub64(a, b, c, d, lo, hi);
        k.template emit<J + IM_SUB_LO>(lo);
        k.template emit<J + IM_SUB_HI>(hi);
        k.template emit<J + IM_DP4A_SS>(it_dp4a_ss(a, b, c));
        k.template emit<J + IM_DP4A_SU>(it_dp4a_su(a, b, c));
        k.template emit<J + IM_DP4A_UU>(it_dp4a_uu(a, b, c));
    } else if constexpr (FMT == IT_BIT) {
        const uint32_t a = o[0], b = o[1], c = o[2];
        k.template emit<J + IB_LOP3 + 0>(it_lop3_b<kItLop3Imm[0]>(a, b, c));
        k.template emit<J + IB_LOP3 + 1>(it_lop3_b<kItLop3Imm[1]>(a, b, c));
        k.template emit<J + IB_LOP3 + 2>(it_lop3_b<kItLop3Imm[2]>(a, b, c));
        k.template emit<J + IB_LOP3 + 3>(it_lop3_b<kItLop3Imm[3]>(a, b, c));
        k.template emit<J + IB_LOP3 + 4>(it_lop3_b<kItLop3Imm[4]>(a, b, c));
        k.template emit<J + IB_LOP3 + 5>(it_lop3_b<kItLop3Imm[5]>(a, b, c));
        k.template emit<J + IB_LOP3 + 6>(it_lop3_b<kItLop3Imm[6]>(a, b, c));
        k.template emit<J + IB_LOP3 + 7>(it_lop3_b<kItLop3Imm[7]>(a, b, c));
        k.template emit<J + IB_SHF_L>(it_shf_l(a, b, c));
        k.template emit<J + IB_SHF_R>(it_shf_r(a, b, c));
        k.template emit<J + IB_SHR_S>(it_shr_s(a, c));
        k.template emit<J + IB_SHL>(it_shl_b(a, c));
        k.template emit<J + IB_POPC>(it_popc_b(a));
        k.template emit<J + IB_CLZ>(it_clz_b(b));
        k.template emit<J + IB_BFIND_U>(it_bfind_ub(a));
        k.template emit<J + IB_BFIND_S>(it_bfind_sb(a));
        k.template emit<J + IB_BREV>(it_brev_b(a));
        k.template emit<J + IB_PRMT>(it_prmt_b(a, b, c));
        k.template emit<J + IB_MIN_S>(it_min_sb(a, b));
        k.template emit<J + IB_MAX_S>(it_max_sb(a, b));
        k.template emit<J + IB_MIN_U>(it_min_ub(a, b));
        k.template emit<J + IB_MAX_U>(it_max_ub(a, b));
        k.template emit<J + IB_SAD>(it_sad_ub(a, b, c));
    } else {
        const uint32_t v = o[0], b = o[1], c = o[2];
        uint32_t d, p;
        it_shfl_idx(v, b, c, d, p);
        k.template emit<J + IW_IDX>(d);
        k.template emit<J + IW_IDX_P>(p);
        it_shfl_up(v, b, c & 0x1f00u, d, p);
        k.template emit<J + IW_UP>(d);
        k.template emit<J + IW_UP_P>(p);
        it_shfl_down(v, b, c, d, p);
        k.template emit<J + IW_DOWN>(d);
        k.template emit<J + IW_DOWN_P>(p);
        it_shfl_bfly(v, b, c, d, p);
        k.template emit<J + IW_BFLY>(d);
        k.template emit<J + IW_BFLY_P>(p);
        k.template emit<J + IW_BALLOT>(it_ballot(o[3]));
        k.template emit<J + IW_ADD>(it_redux_add(o[4]));
        k.template emit<J + IW_MIN_S>(it_redux_min_s(o[4]));
        k.template emit<J + IW_MAX_S>(it_redux_max_s(o[4]));
        k.template emit<J + IW_MIN_U>(it_redux_min_u(o[4]));
        k.template emit<J + IW_MAX_U>(it_redux_max_u(o[4]));
        k.template emit<J + IW_AND>(it_redux_and(o[4]));
        k.template emit<J + IW_OR>(it_redux_or(o[4]));
        k.template emit<J + IW_XOR>(it_redux_xor(o[4]));
        k.template emit<J + IW_MATCH_ANY>(it_match_any(o[5]));
        it_match_all(o[6], d, p);
        k.template emit<J + IW_MATCH_ALL>(d);
        k.template emit<J + IW_MATCH_ALL_P>(p);
    }
}

template <int FMT, bool DUMP, int S = 0>
__device__ __forceinline__ void it_sets(const uint32_t* w, ItSink<DUMP>& k) {
    if constexpr (S < kItSets[FMT]) {
        constexpr int OFF = S * kItSetSlots[FMT];
        it_set<FMT, S, DUMP>(w + OFF, k);
        it_sets<FMT, DUMP, S + 1>(w, k);
    }
}

// table: kCtTiles tables of it_table_bytes(FMT) bytes; checks: [kCtTiles][kCtThreads]; rec: one per CTA.
// Block: kCtThreads threads, no dynamic shared memory.  Same signature as tc_selftest.
template <int FMT, bool DUMP>
__global__ void __launch_bounds__(kCtThreads)
int_selftest(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks, unsigned long long duration_ns,
             int fault_sm, uint32_t fault_mask, CtRecord* rec, unsigned long long seq, uint32_t* dump) {
    constexpr int SLOTS = kItSlots[FMT];
    constexpr int W = kItWords[FMT];
    const int tid = threadIdx.x;
    uint32_t smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned long long t_end = globaltimer_ns() + duration_ns;
    const uint32_t inj0 = (tid == 0 && (int)smid == fault_sm) ? fault_mask : 0u;
    // 0 at run time, but not provably so at compile time: an empty asm statement leaves no trace in the PTX, and ptxas
    // then hoists the ops of loop-invariant operands out of the repetition loop
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
                it_sets<FMT, DUMP>(w, k);
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
