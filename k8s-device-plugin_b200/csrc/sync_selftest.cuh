// sync_selftest.cuh -- sm_90a self-test kernel of the on-demand synchronization self-test (b2dp_sync_test).
//
// Four warps per CTA run the SM's synchronization hardware on a table the host generated and compare against results
// the host computed from the PTX ISA (sync_test_math.hpp):
//     SY_ATOM  atom.shared add / inc / dec / exch / cas / and / or / xor / min / max (.u32, .s32), red.shared add / xor,
//              atom.shared add .f32 / .noftz.f16x2 / .noftz.bf16x2, and add.u64 / exch.b64 / cas.b64 / min.s64 /
//              max.u64 / and.b64 / add.f64, each on a per-lane plane, a same-bank plane and one hot word; one cas per
//              thread on a private word (hit or miss)
//     SY_BAR   bar.arrive / bar.sync on ids 1..15 at 64, 96 and 128 threads, bar.red.popc / .and / .or with and without
//              a thread count, one mbarrier through two phases (arrive with counts, arrive.noComplete, arrive_drop,
//              arrive.expect_tx, complete_tx, test_wait, try_wait.parity)
//     SY_WARP  shfl.sync idx / up / down / bfly, vote.sync ballot / any / all / uni, redux.sync, match.any / match.all,
//              elect.sync, activemask and a __syncwarp exchange, inside diverged groups of three nested partitions
//
// The skeleton is int_selftest's: rounds of kCtTiles tiles x kCtReps repetitions until the %globaltimer deadline (at least
// one round), the fold (ItSink / it_fold), the __syncthreads_or verdict, the CtRecord, the fault hook (thread 0 of the CTA
// whose %smid == fault_sm XORs fault_mask into its first result word of the first comparison, before the fold) and DUMP
// (CTA 0 writes every result word of repetition 0 of every tile of round 0).
//
// Nothing here can hang the SM:
//   - every named-barrier id, thread count and participant set comes from sy_bar_step(tile, step), which every thread
//     evaluates alike; each count is a multiple of 32 and equals the threads that reach it; a __syncthreads separates
//     two uses of one id, except the back-to-back bar.red of one participant set (each of which blocks them all); every thread runs every step (the give-up below changes no control flow);
//   - every mbarrier wait and every CAS loop is bounded by %globaltimer at the deadline plus kL2GraceNs; a thread that
//     gives up only sets a flag, which the CTA makes uniform at the repetition's __syncthreads_or and then publishes an
//     incomplete record (the verdict counts it as a timeout);
//   - arrive.noComplete runs while the other warps are held on a named barrier, so it never completes the phase;
//   - every member mask is a group of sy_color's partition, which any table word yields, and only its lanes enter it;
//   - every shared address is inside this CTA's static arrays by construction.
#pragma once
#include <cstdint>
#include <type_traits>
#include <cuda_runtime.h>

#include "hbm_probe.cuh"      // globaltimer_ns
#include "int_selftest.cuh"   // ItSink
#include "sync_test_math.hpp"

namespace b2dp {

// The fold of a format whose word index is known only at run time: it keeps ItSink's chains and hook.
template <bool DUMP>
struct SySink : ItSink<DUMP> {
    __device__ __forceinline__ void emit_at(int j, uint32_t w) {
        if (j == 0) w ^= this->inj;
        if (DUMP && this->dump) this->dump[j] = w;
        const uint32_t x = (this->h[j & 3] ^ w) * kItMul;
        this->h[j & 3] = __funnelshift_l(x, x, kItFoldRot);
    }
};

// ---- the shared-memory atomics -------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t sy_saddr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int O>
__device__ __forceinline__ uint32_t sy_atom32(uint32_t a, uint32_t x) {
    uint32_t d = 0;
    if constexpr (O == A_ADD) asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_INC) asm volatile("atom.shared.inc.u32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_DEC) asm volatile("atom.shared.dec.u32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_EXCH) asm volatile("atom.shared.exch.b32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_AND) asm volatile("atom.shared.and.b32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_OR) asm volatile("atom.shared.or.b32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_XOR) asm volatile("atom.shared.xor.b32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_MINU) asm volatile("atom.shared.min.u32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_MAXU) asm volatile("atom.shared.max.u32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_MINS) asm volatile("atom.shared.min.s32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_MAXS) asm volatile("atom.shared.max.s32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_RADD) asm volatile("red.shared.add.u32 [%0], %1;" :: "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_RXOR) asm volatile("red.shared.xor.b32 [%0], %1;" :: "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_F32) asm volatile("atom.shared.add.f32 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_F16)
        asm volatile("atom.shared.add.noftz.f16x2 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    else if constexpr (O == A_BF16)
        asm volatile("atom.shared.add.noftz.bf16x2 %0, [%1], %2;" : "=r"(d) : "r"(a), "r"(x) : "memory");
    return d;
}
template <int O>
__device__ __forceinline__ uint64_t sy_atom64(uint32_t a, uint64_t x) {
    uint64_t d = 0;
    if constexpr (O == B_ADD) asm volatile("atom.shared.add.u64 %0, [%1], %2;" : "=l"(d) : "r"(a), "l"(x) : "memory");
    else if constexpr (O == B_EXCH) asm volatile("atom.shared.exch.b64 %0, [%1], %2;" : "=l"(d) : "r"(a), "l"(x) : "memory");
    else if constexpr (O == B_MINS) asm volatile("atom.shared.min.s64 %0, [%1], %2;" : "=l"(d) : "r"(a), "l"(x) : "memory");
    else if constexpr (O == B_MAXU) asm volatile("atom.shared.max.u64 %0, [%1], %2;" : "=l"(d) : "r"(a), "l"(x) : "memory");
    else if constexpr (O == B_AND) asm volatile("atom.shared.and.b64 %0, [%1], %2;" : "=l"(d) : "r"(a), "l"(x) : "memory");
    else if constexpr (O == B_F64) asm volatile("atom.shared.add.f64 %0, [%1], %2;" : "=l"(d) : "r"(a), "l"(x) : "memory");
    return d;
}
__device__ __forceinline__ uint32_t sy_cas32(uint32_t a, uint32_t c, uint32_t x) {
    uint32_t d;
    asm volatile("atom.shared.cas.b32 %0, [%1], %2, %3;" : "=r"(d) : "r"(a), "r"(c), "r"(x) : "memory");
    return d;
}
__device__ __forceinline__ uint64_t sy_cas64(uint32_t a, uint64_t c, uint64_t x) {
    uint64_t d;
    asm volatile("atom.shared.cas.b64 %0, [%1], %2, %3;" : "=l"(d) : "r"(a), "l"(c), "l"(x) : "memory");
    return d;
}
__device__ __forceinline__ uint32_t sy_ld32(uint32_t a) {
    uint32_t d;
    asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(d) : "r"(a) : "memory");
    return d;
}
__device__ __forceinline__ uint64_t sy_ld64(uint32_t a) {
    uint64_t d;
    asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(d) : "r"(a) : "memory");
    return d;
}

struct SyAtomSmem {
    uint32_t lane32[kSyA32][32];
    uint32_t bank32[32][32];          // word (lane, op): lane * 32 + op, so a warp's 32 lanes hit one bank
    uint32_t hot32[kSyA32];
    uint32_t casonce[kCtThreads];
    uint64_t lane64[kSyA64][32];
    uint64_t bank64[32][16];          // 16 64-bit words per 128-byte row: one bank pair
    uint64_t hot64[kSyA64];
    uint32_t mix[kSyRets][kCtThreads];  // each thread's l2_mix of each return
    uint32_t part[2][8][32];          // the hot plane's per-lane partial sum and xor
};

template <int O, bool DUMP>
__device__ __forceinline__ void sy_atom32_op(SyAtomSmem& sm, const uint32_t* w, int lane, uint32_t* ret,
                                             unsigned long long t_bound, bool& gave_up) {
    const uint32_t x = w[2 * O];
    const uint32_t a[3] = {sy_saddr(&sm.lane32[O][lane]), sy_saddr(&sm.bank32[lane][O]), sy_saddr(&sm.hot32[O])};
#pragma unroll
    for (int p = 0; p < kSyPlanes; ++p) {
        if constexpr (O == A_CAS) {  // the store f(x) = x * kSyCasMul + operand, retried until it lands
            uint32_t old = sy_ld32(a[p]);
            for (;;) {
                const uint32_t got = sy_cas32(a[p], old, old * kSyCasMul + x);
                if (got == old) break;
                old = got;
                if (globaltimer_ns() > t_bound) { gave_up = true; break; }
            }
            ret[p] = old;
        } else {
            ret[p] = sy_atom32<O>(a[p], x);
        }
    }
}
template <int O>
__device__ __forceinline__ void sy_atom64_op(SyAtomSmem& sm, const uint32_t* w, int lane, uint64_t* ret,
                                             unsigned long long t_bound, bool& gave_up) {
    const int s = kSyA64Slot0 + 4 * O;
    const uint64_t x = (uint64_t)w[s + 1] << 32 | w[s];
    const uint32_t a[3] = {sy_saddr(&sm.lane64[O][lane]), sy_saddr(&sm.bank64[lane][O]), sy_saddr(&sm.hot64[O])};
#pragma unroll
    for (int p = 0; p < kSyPlanes; ++p) {
        if constexpr (O == B_CAS) {
            uint64_t old = sy_ld64(a[p]);
            for (;;) {
                const uint64_t got = sy_cas64(a[p], old, old * kSyCasMul64 + x);
                if (got == old) break;
                old = got;
                if (globaltimer_ns() > t_bound) { gave_up = true; break; }
            }
            ret[p] = old;
        } else {
            ret[p] = sy_atom64<O>(a[p], x);
        }
    }
}

template <bool DUMP>
__device__ __forceinline__ void sy_atom_rep(SyAtomSmem& sm, const uint32_t* w, int tid, SySink<DUMP>& k,
                                            unsigned long long t_bound, bool& gave_up) {
    const int lane = tid % 32, warp = tid / 32;
    // the owners store the initial values (plain stores), then one barrier
#pragma unroll
    for (int o = 0; o < kSyA32; ++o) {
        if (warp == 0) sm.lane32[o][lane] = w[2 * o + 1];
        if (warp == 1) sm.bank32[lane][o] = w[2 * o + 1];
        if (tid == 64) sm.hot32[o] = w[2 * o + 1];
    }
#pragma unroll
    for (int o = 0; o < kSyA64; ++o) {
        const int s = kSyA64Slot0 + 4 * o;
        const uint64_t v = (uint64_t)w[s + 3] << 32 | w[s + 2];
        if (warp == 0) sm.lane64[o][lane] = v;
        if (warp == 1) sm.bank64[lane][o] = v;
        if (tid == 64) sm.hot64[o] = v;
    }
    sm.casonce[tid] = w[kSyCasOnceSlot];
    __syncthreads();
    uint32_t r32[5][3], scratch[3];
    uint64_t r64[3][3], s64[3];
    sy_atom32_op<A_ADD, DUMP>(sm, w, lane, r32[0], t_bound, gave_up);
    sy_atom32_op<A_INC, DUMP>(sm, w, lane, r32[1], t_bound, gave_up);
    sy_atom32_op<A_DEC, DUMP>(sm, w, lane, r32[2], t_bound, gave_up);
    sy_atom32_op<A_EXCH, DUMP>(sm, w, lane, r32[3], t_bound, gave_up);
    sy_atom32_op<A_CAS, DUMP>(sm, w, lane, r32[4], t_bound, gave_up);
    sy_atom32_op<A_AND, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_OR, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_XOR, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_MINU, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_MAXU, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_MINS, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_MAXS, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_RADD, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_RXOR, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_F32, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_F16, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom32_op<A_BF16, DUMP>(sm, w, lane, scratch, t_bound, gave_up);
    sy_atom64_op<B_ADD>(sm, w, lane, r64[0], t_bound, gave_up);
    sy_atom64_op<B_EXCH>(sm, w, lane, r64[1], t_bound, gave_up);
    sy_atom64_op<B_CAS>(sm, w, lane, r64[2], t_bound, gave_up);
    sy_atom64_op<B_MINS>(sm, w, lane, s64, t_bound, gave_up);
    sy_atom64_op<B_MAXU>(sm, w, lane, s64, t_bound, gave_up);
    sy_atom64_op<B_AND>(sm, w, lane, s64, t_bound, gave_up);
    sy_atom64_op<B_F64>(sm, w, lane, s64, t_bound, gave_up);
    const uint32_t co = sy_cas32(sy_saddr(&sm.casonce[tid]), w[kSyCasOnceSlot + 1], w[kSyCasOnceSlot + 2]);
    // the returns, mixed and published with plain stores
#pragma unroll
    for (int p = 0; p < kSyPlanes; ++p) {
        const uint32_t key = p == 2 ? kSyHotKey : (uint32_t)lane;
#pragma unroll
        for (int r = 0; r < 5; ++r) sm.mix[r * kSyPlanes + p][tid] = l2_mix(r32[r][p], key);
#pragma unroll
        for (int r = 0; r < 3; ++r) sm.mix[(5 + r) * kSyPlanes + p][tid] = l2_mix64(r64[r][p], key);
    }
    __syncthreads();
    // finals: every op's word on each plane (exch excepted: it enters its return fold)
#pragma unroll
    for (int o = 0; o < kSyA32; ++o) {
        if (o == A_EXCH) continue;
        const int j = (o < A_EXCH ? o : o - 1) * kSyPlanes;
        k.emit_at(j + 0, sm.lane32[o][lane]);
        k.emit_at(j + 1, sm.bank32[lane][o]);
        k.emit_at(j + 2, sm.hot32[o]);
    }
#pragma unroll
    for (int o = 0; o < kSyA64; ++o) {
        if (o == B_EXCH) continue;
        const int j = kSyAtomFin32 + (o < B_EXCH ? o : o - 1) * kSyPlanes * 2;
        const uint64_t v[3] = {sm.lane64[o][lane], sm.bank64[lane][o], sm.hot64[o]};
#pragma unroll
        for (int p = 0; p < kSyPlanes; ++p) {
            k.emit_at(j + 2 * p, (uint32_t)v[p]);
            k.emit_at(j + 2 * p + 1, (uint32_t)(v[p] >> 32));
        }
    }
    k.emit_at(kSyAtomFin32 + kSyAtomFin64, co);
    k.emit_at(kSyAtomFin32 + kSyAtomFin64 + 1, sm.casonce[tid]);
    // return folds: the lane planes sum over the 4 warps at this lane; the hot word over all 128 threads, in two steps
    uint32_t fs[kSyRets], fx[kSyRets];
#pragma unroll
    for (int i = 0; i < kSyRets; ++i) {
        uint32_t s = 0, x = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) { const uint32_t m = sm.mix[i][q * 32 + lane]; s += m; x ^= m; }
        fs[i] = s; fx[i] = x;
    }
    if (warp == 0) {
#pragma unroll
        for (int r = 0; r < 8; ++r) { sm.part[0][r][lane] = fs[r * kSyPlanes + 2]; sm.part[1][r][lane] = fx[r * kSyPlanes + 2]; }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        uint32_t s = 0, x = 0;
        for (int l = 0; l < 32; ++l) { s += sm.part[0][r][l]; x ^= sm.part[1][r][l]; }
        fs[r * kSyPlanes + 2] = s; fx[r * kSyPlanes + 2] = x;
    }
    // exch: the final joins its returns
    const uint32_t ex[3] = {sm.lane32[A_EXCH][lane], sm.bank32[lane][A_EXCH], sm.hot32[A_EXCH]};
    const uint64_t ex64[3] = {sm.lane64[B_EXCH][lane], sm.bank64[lane][B_EXCH], sm.hot64[B_EXCH]};
#pragma unroll
    for (int p = 0; p < kSyPlanes; ++p) {
        const uint32_t key = p == 2 ? kSyHotKey : (uint32_t)lane;
        const uint32_t m = l2_mix(ex[p], key), m64 = l2_mix64(ex64[p], key);
        fs[3 * kSyPlanes + p] += m; fx[3 * kSyPlanes + p] ^= m;
        fs[6 * kSyPlanes + p] += m64; fx[6 * kSyPlanes + p] ^= m64;
    }
    const int j0 = kSyAtomFin32 + kSyAtomFin64 + 2;
#pragma unroll
    for (int i = 0; i < kSyRets; ++i) { k.emit_at(j0 + 2 * i, fs[i]); k.emit_at(j0 + 2 * i + 1, fx[i]); }
}

// Table word of slot s for this thread, read from the L1-resident table (SY_BAR and SY_WARP index their slots at run
// time, which a register array would turn into local memory); w points at this thread's word of slot 0.
__device__ __forceinline__ uint32_t sy_tw(const uint32_t* w, int s) { return __ldg(w + s * kCtThreads); }

// ---- the barrier unit and the mbarrier -----------------------------------------------------------------------------
__device__ __forceinline__ void sy_bar_arrive(int id, int n) {
    asm volatile("bar.arrive %0, %1;" :: "r"(id), "r"(n) : "memory");
}
__device__ __forceinline__ void sy_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ uint32_t sy_bar_popc(int id, uint32_t q) {
    uint32_t d;
    asm volatile("{ .reg .pred p; setp.ne.u32 p, %2, 0; bar.red.popc.u32 %0, %1, p; }" : "=r"(d) : "r"(id), "r"(q) : "memory");
    return d;
}
__device__ __forceinline__ uint32_t sy_bar_popc_n(int id, int n, uint32_t q) {
    uint32_t d;
    asm volatile("{ .reg .pred p; setp.ne.u32 p, %3, 0; bar.red.popc.u32 %0, %1, %2, p; }"
                 : "=r"(d) : "r"(id), "r"(n), "r"(q) : "memory");
    return d;
}
#define B2DP_SY_BAR_PRED(NAME, OP, ARGS, ...)                                                                  \
    __device__ __forceinline__ uint32_t NAME(__VA_ARGS__) {                                                  \
        uint32_t d;                                                                                          \
        asm volatile("{ .reg .pred p, r; setp.ne.u32 p, %1, 0; bar.red." OP ".pred r, " ARGS ", p; selp.u32 %0, 1, 0, r; }" \
                     : "=r"(d) : "r"(q), "r"(id), "r"(n) : "memory");                                       \
        return d;                                                                                            \
    }
B2DP_SY_BAR_PRED(sy_bar_and, "and", "%2", uint32_t q, int id, int n)
B2DP_SY_BAR_PRED(sy_bar_or, "or", "%2", uint32_t q, int id, int n)
B2DP_SY_BAR_PRED(sy_bar_and_n, "and", "%2, %3", uint32_t q, int id, int n)
B2DP_SY_BAR_PRED(sy_bar_or_n, "or", "%2, %3", uint32_t q, int id, int n)
#undef B2DP_SY_BAR_PRED

__device__ __forceinline__ uint32_t sy_test_wait(uint32_t mb, uint64_t state) {
    uint32_t d;
    asm volatile("{ .reg .pred p; mbarrier.test_wait.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(d) : "r"(mb), "l"(state) : "memory");
    return d;
}
__device__ __forceinline__ uint32_t sy_test_parity(uint32_t mb, uint32_t parity) {
    uint32_t d;
    asm volatile("{ .reg .pred p; mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(d) : "r"(mb), "r"(parity) : "memory");
    return d;
}
// try_wait.parity until the phase of that parity completes, or the bound passes (then *gave_up)
__device__ __forceinline__ void sy_wait_parity(uint32_t mb, uint32_t parity, unsigned long long t_bound, bool& gave_up) {
    for (;;) {
        uint32_t done;
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(mb), "r"(parity) : "memory");
        if (done) return;
        if (globaltimer_ns() > t_bound) { gave_up = true; return; }
    }
}

struct SyBarSmem {
    uint32_t val[kSyNamed][kCtThreads];
    unsigned long long mbar;
};

template <bool DUMP>
__device__ __forceinline__ void sy_bar_rep(SyBarSmem& sm, const uint32_t* w, int tile, uint32_t key, int tid,
                                           SySink<DUMP>& k, unsigned long long t_bound, bool& gave_up) {
    const int lane = tid % 32, warp = tid / 32;
    // named barriers: three groups (64, 96, 128 threads) of ids 1..15, a __syncthreads between groups
#pragma unroll 1
    for (int g = 0; g < 3; ++g) {
#pragma unroll 1
        for (int i = 0; i < 15; ++i) {
            const int s = g * 15 + i;
            int id, n;
            uint32_t pm, cm;
            sy_bar_step(tile, s, id, n, pm, cm);
            uint32_t word = 0;
            if (pm >> warp & 1) {
                sm.val[s][tid] = sy_tw(w, s) ^ key;
                sy_bar_arrive(id, n);
            } else if (cm >> warp & 1) {
                sy_bar_sync(id, n);
                word = sm.val[s][sy_bar_source(pm, cm, warp) * 32 + lane] ^ key;
            }
            k.emit_at(s, word);
        }
        __syncthreads();
    }
    // bar.red: id 1 over the CTA without a count; ids 2 / 3 over warps {0, 1} / {2, 3} with a count of 64.  The three
    // reductions on one id run back to back without a __syncthreads between them: each is a blocking barrier of the
    // same participant set, so every participant leaves one before any enters the next (the one exception to the
    // __syncthreads-between-uses rule)
    k.emit_at(kSyNamed + 0, sy_bar_popc(1, sy_tw(w, kSyNamed + 0) & 1));
    k.emit_at(kSyNamed + 1, sy_bar_and(sy_tw(w, kSyNamed + 1) & 1, 1, 0));
    k.emit_at(kSyNamed + 2, sy_bar_or(sy_tw(w, kSyNamed + 2) & 1, 1, 0));
    const int pid = 2 + warp / 2;
    k.emit_at(kSyNamed + 3, sy_bar_popc_n(pid, 64, sy_tw(w, kSyNamed + 3) & 1));
    k.emit_at(kSyNamed + 4, sy_bar_and_n(sy_tw(w, kSyNamed + 4) & 1, pid, 64));
    k.emit_at(kSyNamed + 5, sy_bar_or_n(sy_tw(w, kSyNamed + 5) & 1, pid, 64));
    // the mbarrier
    const int j = kSyNamed + kSyRed;
    const uint32_t mb = sy_saddr(&sm.mbar);
    const uint32_t a0 = sy_mbar_a0(tile), a1 = sy_mbar_a1(tile);
    if (tid == 0) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(mb), "r"(a0 + a1 + 2) : "memory");
    __syncthreads();
    // phase 0: warp 0 arrives without completing while warps 1..3 wait on named barrier 1, which it opens after its test
    uint32_t w0 = 0;
    if (warp == 0) {
        if (lane == 0) {
            uint64_t st;
            asm volatile("mbarrier.arrive.noComplete.shared::cta.b64 %0, [%1], %2;" : "=l"(st) : "r"(mb), "r"(a0) : "memory");
            w0 = sy_test_wait(mb, st);
        }
        __syncwarp();
        sy_bar_arrive(1, 128);
    } else {
        sy_bar_sync(1, 128);
        if (lane == 0) {
            uint64_t st;
            if (warp == 1)
                asm volatile("mbarrier.arrive.shared::cta.b64 %0, [%1], %2;" : "=l"(st) : "r"(mb), "r"(a1) : "memory");
            else if (warp == 2)
                asm volatile("mbarrier.arrive_drop.shared::cta.b64 %0, [%1];" : "=l"(st) : "r"(mb) : "memory");
            else
                asm volatile("mbarrier.arrive.shared::cta.b64 %0, [%1];" : "=l"(st) : "r"(mb) : "memory");
        }
    }
    k.emit_at(j + 0, w0);
    sy_wait_parity(mb, 0, t_bound, gave_up);
    k.emit_at(j + 1, sy_test_parity(mb, 0));
    k.emit_at(j + 2, sy_test_parity(mb, 1));
    __syncthreads();
    // phase 1: every arrival first, expect_tx among them; then the complete_tx of warps 2 and 3 completes it
    if (lane == 0) {
        uint64_t st;
        if (warp == 0)
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 %0, [%1], %2;"
                         : "=l"(st) : "r"(mb), "r"(sy_tw(w, kSyBarSlots - 1)) : "memory");
        else if (warp == 1)
            asm volatile("mbarrier.arrive.shared::cta.b64 %0, [%1], %2;" : "=l"(st) : "r"(mb), "r"(a0 + a1 - 1) : "memory");
        else if (warp == 3)
            asm volatile("mbarrier.arrive.shared::cta.b64 %0, [%1];" : "=l"(st) : "r"(mb) : "memory");
    }
    __syncthreads();
    k.emit_at(j + 3, sy_test_parity(mb, 1));
    __syncthreads();
    if (warp >= 2)
        asm volatile("mbarrier.complete_tx.shared::cta.b64 [%0], %1;" :: "r"(mb), "r"(sy_tw(w, kSyBarSlots - 1)) : "memory");
    sy_wait_parity(mb, 1, t_bound, gave_up);
    k.emit_at(j + 4, sy_test_parity(mb, 1));
    k.emit_at(j + 5, sy_test_parity(mb, 0));
    __syncthreads();
    if (tid == 0) asm volatile("mbarrier.inval.shared::cta.b64 [%0];" :: "r"(mb) : "memory");
}

// ---- collectives in diverged warps ---------------------------------------------------------------------------------
struct SyWarpSmem {
    uint32_t elect[4][32];
    uint32_t xchg[4][32];
};

template <bool DUMP>
__device__ __forceinline__ void sy_group_ops(SyWarpSmem& sm, const uint32_t* x, uint32_t m, int lane, int warp, int J,
                                             SySink<DUMP>& k) {
    uint32_t b[4], d, p;
    sy_shfl_b(m, lane, b);
    const uint32_t v = sy_tw(x, 3), q = sy_tw(x, 4) & 1, r = sy_tw(x, 5), mv = sy_tw(x, 6), m2 = sy_tw(x, 7);
    asm volatile("{ .reg .pred q; shfl.sync.idx.b32 %0|q, %2, %3, 0x1f, %4; selp.u32 %1, 1, 0, q; }"
                 : "=r"(d), "=r"(p) : "r"(v), "r"(b[0]), "r"(m));
    k.emit_at(J + SW_IDX, d); k.emit_at(J + SW_IDX_P, p);
    asm volatile("{ .reg .pred q; shfl.sync.up.b32 %0|q, %2, %3, 0, %4; selp.u32 %1, 1, 0, q; }"
                 : "=r"(d), "=r"(p) : "r"(v), "r"(b[1]), "r"(m));
    k.emit_at(J + SW_UP, d); k.emit_at(J + SW_UP_P, p);
    asm volatile("{ .reg .pred q; shfl.sync.down.b32 %0|q, %2, %3, 0x1f, %4; selp.u32 %1, 1, 0, q; }"
                 : "=r"(d), "=r"(p) : "r"(v), "r"(b[2]), "r"(m));
    k.emit_at(J + SW_DOWN, d); k.emit_at(J + SW_DOWN_P, p);
    asm volatile("{ .reg .pred q; shfl.sync.bfly.b32 %0|q, %2, %3, 0x1f, %4; selp.u32 %1, 1, 0, q; }"
                 : "=r"(d), "=r"(p) : "r"(v), "r"(b[3]), "r"(m));
    k.emit_at(J + SW_BFLY, d); k.emit_at(J + SW_BFLY_P, p);
    asm volatile("{ .reg .pred q; setp.ne.u32 q, %1, 0; vote.sync.ballot.b32 %0, q, %2; }" : "=r"(d) : "r"(q), "r"(m));
    k.emit_at(J + SW_BALLOT, d);
    asm volatile("{ .reg .pred q, o; setp.ne.u32 q, %1, 0; vote.sync.any.pred o, q, %2; selp.u32 %0, 1, 0, o; }"
                 : "=r"(d) : "r"(q), "r"(m));
    k.emit_at(J + SW_ANY, d);
    asm volatile("{ .reg .pred q, o; setp.ne.u32 q, %1, 0; vote.sync.all.pred o, q, %2; selp.u32 %0, 1, 0, o; }"
                 : "=r"(d) : "r"(q), "r"(m));
    k.emit_at(J + SW_ALL, d);
    asm volatile("{ .reg .pred q, o; setp.ne.u32 q, %1, 0; vote.sync.uni.pred o, q, %2; selp.u32 %0, 1, 0, o; }"
                 : "=r"(d) : "r"(q), "r"(m));
    k.emit_at(J + SW_UNI, d);
    asm volatile("redux.sync.add.u32 %0, %1, %2;" : "=r"(d) : "r"(r), "r"(m));
    k.emit_at(J + SW_ADD, d);
    asm volatile("redux.sync.min.s32 %0, %1, %2;" : "=r"(d) : "r"(r), "r"(m));
    k.emit_at(J + SW_MIN_S, d);
    asm volatile("redux.sync.max.u32 %0, %1, %2;" : "=r"(d) : "r"(r), "r"(m));
    k.emit_at(J + SW_MAX_U, d);
    asm volatile("redux.sync.and.b32 %0, %1, %2;" : "=r"(d) : "r"(r), "r"(m));
    k.emit_at(J + SW_AND, d);
    asm volatile("redux.sync.or.b32 %0, %1, %2;" : "=r"(d) : "r"(r), "r"(m));
    k.emit_at(J + SW_OR, d);
    asm volatile("redux.sync.xor.b32 %0, %1, %2;" : "=r"(d) : "r"(r), "r"(m));
    k.emit_at(J + SW_XOR, d);
    asm volatile("match.any.sync.b32 %0, %1, %2;" : "=r"(d) : "r"(mv), "r"(m));
    k.emit_at(J + SW_MATCH_ANY, d);
    asm volatile("{ .reg .pred q; match.all.sync.b32 %0|q, %2, %3; selp.u32 %1, 1, 0, q; }"
                 : "=r"(d), "=r"(p) : "r"(m2), "r"(m));
    k.emit_at(J + SW_MATCH_ALL, d); k.emit_at(J + SW_MATCH_ALL_P, p);
    // elect.sync: the elected lane is a member, exactly one member holds the predicate, every member names that lane
    uint32_t el, ep;
    asm volatile("{ .reg .pred q; elect.sync %0|q, %2; selp.u32 %1, 1, 0, q; }" : "=r"(el), "=r"(ep) : "r"(m));
    k.emit_at(J + SW_ELECT_IN, (m >> (el & 31)) & 1 & (el < 32));
    sm.elect[warp][lane] = ep | el << 1;
    __syncwarp(m);
    uint32_t ones = 0, agree = 1;
    for (int l = 0; l < 32; ++l) {
        if (!(m >> l & 1)) continue;
        const uint32_t e = sm.elect[warp][l];
        ones += e & 1;
        agree &= (e >> 1) == el && ((e & 1) == (uint32_t)(l == (int)el));
    }
    __syncwarp(m);
    k.emit_at(J + SW_ELECT_ONE, (uint32_t)(ones == 1) & agree);
    uint32_t am;
    asm volatile("activemask.b32 %0;" : "=r"(am));
    k.emit_at(J + SW_ACTIVE, (am >> lane & 1) & (uint32_t)((am & ~m) == 0));
    // __syncwarp(m) orders a store to shared memory before the group's loads
    const int n = __popc(m), rk = __popc(m & ((1u << lane) - 1u));
    sm.xchg[warp][lane] = v ^ kSyXchg;
    __syncwarp(m);
    d = sm.xchg[warp][sy_nth(m, (rk + n - 1) % n)];
    __syncwarp(m);
    k.emit_at(J + SW_XCHG, d);
}

template <bool DUMP>
__device__ __forceinline__ void sy_warp_rep(SyWarpSmem& sm, const uint32_t* w, const uint32_t* w0, int tid,
                                            SySink<DUMP>& k) {
    const int lane = tid % 32, warp = tid / 32;
#pragma unroll 1
    for (int s = 0; s < kSyWarpSets; ++s) {
        const uint32_t* x = w + s * kSyWarpSetSlots * kCtThreads;
        // the level words: lane 0's, one address per warp
        const uint32_t wl[3] = {sy_tw(w0, s * kSyWarpSetSlots), sy_tw(w0, s * kSyWarpSetSlots + 1),
                                sy_tw(w0, s * kSyWarpSetSlots + 2)};
        const uint32_t m1 = sy_group(wl, 1, lane), m2 = sy_group(wl, 2, lane), m3 = sy_group(wl, 3, lane);
        const int J = s * kSyLevels * kSyLevelWords;
        // lanes enter their group's body one group at a time: at the loop index that equals the group's lowest lane
#pragma unroll 1
        for (int l1 = 0; l1 < 32; ++l1) {
            if (__ffs(m1) - 1 != l1) continue;
            sy_group_ops(sm, x, m1, lane, warp, J, k);
#pragma unroll 1
            for (int l2 = 0; l2 < 32; ++l2) {
                if (__ffs(m2) - 1 != l2) continue;
                sy_group_ops(sm, x, m2, lane, warp, J + kSyLevelWords, k);
#pragma unroll 1
                for (int l3 = 0; l3 < 32; ++l3) {
                    if (__ffs(m3) - 1 != l3) continue;
                    sy_group_ops(sm, x, m3, lane, warp, J + 2 * kSyLevelWords, k);
                }
            }
        }
    }
    __syncwarp();
}

// table: kCtTiles tables of sy_table_bytes(FMT) bytes; checks: [kCtTiles][kCtThreads]; rec: one per CTA.
// Block: kCtThreads threads, static shared memory only.  Same signature as int_selftest.
template <int FMT, bool DUMP>
__global__ void __launch_bounds__(kCtThreads)
sync_selftest(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks, unsigned long long duration_ns,
              int fault_sm, uint32_t fault_mask, CtRecord* rec, unsigned long long seq, uint32_t* dump) {
    constexpr int SLOTS = kSySlots[FMT];
    constexpr int W = kSyWords[FMT];
    using Smem = typename std::conditional<FMT == SY_ATOM, SyAtomSmem,
                                           typename std::conditional<FMT == SY_BAR, SyBarSmem, SyWarpSmem>::type>::type;
    __shared__ __align__(16) Smem sm;
    const int tid = threadIdx.x;
    uint32_t smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned long long t_end = globaltimer_ns() + duration_ns, t_bound = t_end + kL2GraceNs;
    const uint32_t inj0 = (tid == 0 && (int)smid == fault_sm) ? fault_mask : 0u;
    const uint32_t zero = smid < nsmid ? 0u : ~0u;  // int_selftest: no op leaves the repetition loop
    constexpr int RS = FMT == SY_ATOM ? SLOTS : 1;  // SY_ATOM keeps its operands in registers; the others read the table
    uint32_t v[RS], w[RS];
    unsigned long long rounds = 0, comparisons = 0, mismatches = 0;
    int bad_tile = -1, bad_rep = -1;
    bool stop = false;
    while (!stop) {
        for (int tile = 0; tile < kCtTiles && !stop; ++tile) {
            const uint32_t* tt = reinterpret_cast<const uint32_t*>(table) + (size_t)tile * SLOTS * kCtThreads;
            if constexpr (FMT == SY_ATOM) {
#pragma unroll
                for (int s = 0; s < SLOTS; ++s) v[s] = __ldg(tt + s * kCtThreads + tid);
            }
            const uint32_t want = __ldg(checks + tile * kCtThreads + tid);
            for (int rep = 0; rep < kCtReps; ++rep) {
#pragma unroll
                for (int s = 0; s < RS; ++s) w[s] = v[s] ^ ((uint32_t)rep & zero);
                SySink<DUMP> k;
                constexpr uint32_t i0 = kItFoldInit[0], i1 = kItFoldInit[1], i2 = kItFoldInit[2], i3 = kItFoldInit[3];
                k.h[0] = i0; k.h[1] = i1; k.h[2] = i2; k.h[3] = i3;
                k.inj = (rounds | (unsigned)tile | (unsigned)rep) == 0 ? inj0 : 0u;
                k.dump = (DUMP && blockIdx.x == 0 && rounds == 0 && rep == 0)
                             ? dump + ((size_t)tile * kCtThreads + tid) * W : nullptr;
                bool gave_up = false;
                if constexpr (FMT == SY_ATOM) {
                    sy_atom_rep(sm, w, tid, k, t_bound, gave_up);
                } else if constexpr (FMT == SY_BAR) {
                    const uint32_t key = (uint32_t)((rounds * kCtTiles + tile) * kCtReps + rep + 1) * kSyKeyMul;
                    sy_bar_rep(sm, tt + tid, tile, key, tid, k, t_bound, gave_up);
                } else {
                    sy_warp_rep(sm, tt + tid, tt + (tid & ~31), tid, k);
                }
                // one barrier: the verdict, and (bit 1) a give-up anywhere in the CTA
                const int flags = __syncthreads_or((k.value() != want ? 1 : 0) | (gave_up ? 2 : 0));
                if (flags & 2) { stop = true; break; }
                ++comparisons;
                if ((flags & 1) && mismatches++ == 0) { bad_tile = tile; bad_rep = rep; }
            }
        }
        if (stop) break;  // an incomplete round: the record's comparisons no longer match its rounds
        ++rounds;
        if (__syncthreads_or(tid == 0 && globaltimer_ns() >= t_end)) break;
    }
    if (tid == 0) {
        volatile CtRecord* r = rec + blockIdx.x;
        r->smid = smid;
        r->nsmid = nsmid;
        r->rounds = rounds;
        r->comparisons = comparisons + (stop ? 1 : 0);
        r->mismatches = mismatches;
        r->first_bad_tile = bad_tile;
        r->first_bad_rep = bad_rep;
        __threadfence_system();
        r->seq = seq;
    }
}

}  // namespace b2dp
