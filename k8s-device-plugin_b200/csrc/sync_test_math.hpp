// sync_test_math.hpp -- host-side reference of the on-demand synchronization self-test (b2dp_sync_test,
// sync_selftest.cuh): the SM's shared-memory atomic unit, its barrier unit and mbarriers, and warp collectives under
// partial member masks.
//
// Pure C++ (no CUDA, apart from the schedule and partition functions the kernel shares), so the CPU tests compile it as
// it is (tests/native/sync_test_math_test.cpp) and compare it with tests/sync_test_oracle.py:
//   - sy_operands:      seed, format, tile -> the table ([slot][thread] words), crafted classes included
//   - sy_results:       every thread's reference result words, in the kernel's word order
//   - sy_build_tile:    the table a launch reads verbatim and the check values (it_fold of each thread's words)
// Every expected value follows from the PTX ISA alone; nothing comes from the device under test.
//
// SY_ATOM.  Every op runs on three planes: the per-lane plane (word `lane`, one contribution from each of the 4 warps),
// the same-bank plane (word lane * 32 + op: the 32 lanes of a warp hit 32 words of one bank, 4 contributions each) and
// one hot word that all 128 threads hit.  Final values are order-free; the returns of add / inc / dec / cas (uniform
// operands, so the returns are {f^i(init) : i < n}) and of exch ({returns} + {final} = {init} + {operands}) enter the
// sum and the xor of l2_mix(value, key) over a word's contributors, which the CTA forms with plain shared loads and
// stores behind a barrier.
// SY_BAR.  Named barriers 1..15 at 64, 96 and 128 threads (producers bar.arrive, consumers bar.sync and read what the
// producers wrote, keyed by round, tile and repetition), bar.red.popc / .and / .or with and without a thread count, and
// one mbarrier through two phases (arrive with counts, noComplete, arrive_drop, expect_tx and complete_tx).  Who takes
// part in which barrier is a function of the tile and the step (sy_bar_step), never of table data.
// SY_WARP.  A warp-uniform word per level (sy_color) partitions the 32 lanes; three nested levels refine it.  Every group
// runs shfl.sync (idx / up / down / bfly), vote.sync, redux.sync, match.sync, elect.sync, activemask and a __syncwarp
// exchange with its own member mask; sources are always inside the mask by construction.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "int_test_math.hpp"  // it_fold, ct_mix, ct_hash, CtRecord, kCtThreads, kCtTiles, kCtReps
#include "l2_test_math.hpp"   // l2_mix, l2_mix64, l2_inc, l2_dec, float bit helpers and bounds, kL2GraceNs

namespace b2dp {

enum SyFormat { SY_ATOM = 0, SY_BAR = 1, SY_WARP = 2 };
constexpr int kSyFormats = 3;
static_assert(kSyFormats == kCtFormats, "the verdict and the result struct are shared with the tensor-core test");

// ---- SY_ATOM layout -----------------------------------------------------------------------------------------------
enum SyA32 { A_ADD, A_INC, A_DEC, A_EXCH, A_CAS, A_AND, A_OR, A_XOR, A_MINU, A_MAXU, A_MINS, A_MAXS, A_RADD, A_RXOR,
             A_F32, A_F16, A_BF16, kSyA32 };
enum SyA64 { B_ADD, B_EXCH, B_CAS, B_MINS, B_MAXU, B_AND, B_F64, kSyA64 };
constexpr int kSyPlanes = 3;                        // per-lane, same-bank, hot
constexpr int kSyA64Slot0 = 2 * kSyA32;             // 32-bit op o: slots 2o (operand), 2o + 1 (init)
constexpr int kSyCasOnceSlot = kSyA64Slot0 + 4 * kSyA64;  // 64-bit op o: operand lo, hi, init lo, hi
constexpr int kSyAtomSlots = kSyCasOnceSlot + 3;    // cas-once: init, compare, new
constexpr int kSyRet32[5] = {A_ADD, A_INC, A_DEC, A_EXCH, A_CAS};
constexpr int kSyRet64[3] = {B_ADD, B_EXCH, B_CAS};
constexpr int kSyRets = (5 + 3) * kSyPlanes;        // return folds: sum and xor of each
constexpr int kSyAtomFin32 = (kSyA32 - 1) * kSyPlanes;       // exch has no order-free final of its own
constexpr int kSyAtomFin64 = (kSyA64 - 1) * kSyPlanes * 2;
constexpr int kSyAtomWords = kSyAtomFin32 + kSyAtomFin64 + 2 + 2 * kSyRets;
constexpr uint32_t kSyCasMul = 0x01000193u;         // the CAS loops store f(x) = x * kSyCasMul + operand
constexpr uint64_t kSyCasMul64 = 0x100000001B3ull;
constexpr uint32_t kSyHotKey = 32;                  // the hot word's l2_mix key (the lane planes use the lane)

// ---- SY_BAR layout ------------------------------------------------------------------------------------------------
constexpr int kSyNamed = 45;                        // ids 1..15 at 64, then 96, then 128 threads
constexpr int kSyRed = 6;                           // popc / and / or over 128 threads on id 1, over 64 on ids 2 and 3
constexpr int kSyMbarWords = 6;
constexpr int kSyBarSlots = kSyNamed + kSyRed + 1;  // the last slot: complete_tx bytes (warps 2, 3), expect_tx (thread 0)
constexpr int kSyBarWords = kSyNamed + 3 * 2 + kSyMbarWords;
constexpr uint32_t kSyKeyMul = 0x9E3779B9u;         // a consumer's word is read ^ (comparison index * kSyKeyMul)

// Named-barrier step s (0..44) of tile `tile`: id, thread count, producer and consumer warp masks.  Participants are k
// consecutive warps (mod 4) from a start that moves with the tile; the first np of them produce.
B2DP_L2_HD inline void sy_bar_step(int tile, int s, int& id, int& count, uint32_t& pmask, uint32_t& cmask) {
    const int g = s / 15, k = g + 2;
    id = s % 15 + 1;
    count = 32 * k;
    const int start = (tile + id + g) % 4, np = 1 + (tile + 2 * id + g) % (k - 1);
    pmask = cmask = 0;
    for (int i = 0; i < k; ++i) (i < np ? pmask : cmask) |= 1u << ((start + i) % 4);
}
// the producer warp a consumer warp reads from: its index among the consumers, modulo the producer count
B2DP_L2_HD inline int sy_bar_source(uint32_t pmask, uint32_t cmask, int warp) {
    int ci = 0, np = 0;
    for (int w = 0; w < warp; ++w) ci += cmask >> w & 1;
    for (int w = 0; w < 4; ++w) np += pmask >> w & 1;
    int want = ci % np;
    for (int w = 0; w < 4; ++w)
        if (pmask >> w & 1 && want-- == 0) return w;
    return -1;
}
// mbarrier arrival counts of tile `tile`: phase 0 expects a0 (noComplete, warp 0) + a1 (warp 1) + 1 (arrive_drop, warp 2)
// + 1 (warp 3); phase 1 expects one fewer: 1 (expect_tx, warp 0) + a0 + a1 - 1 (warp 1) + 1 (warp 3).
B2DP_L2_HD inline int sy_mbar_a0(int tile) { return 1 + tile % 3; }
B2DP_L2_HD inline int sy_mbar_a1(int tile) { return 1 + tile % 4; }

// ---- SY_WARP layout -----------------------------------------------------------------------------------------------
constexpr int kSyWarpSets = 4;
constexpr int kSyLevels = 3;
constexpr int kSyWarpSetSlots = 8;                  // W1, W2, W3 (warp-uniform: lane 0's), V, Q, R, M, M2
constexpr int kSyLevelWords = 25;
constexpr int kSyWarpWords = kSyWarpSets * kSyLevels * kSyLevelWords;
constexpr uint32_t kSyXchg = 0x5A5A5A5Au;           // what a lane publishes for the __syncwarp exchange: V ^ this
enum SyLevelWord {
    SW_IDX = 0, SW_IDX_P, SW_UP, SW_UP_P, SW_DOWN, SW_DOWN_P, SW_BFLY, SW_BFLY_P,
    SW_BALLOT, SW_ANY, SW_ALL, SW_UNI,
    SW_ADD, SW_MIN_S, SW_MAX_U, SW_AND, SW_OR, SW_XOR,
    SW_MATCH_ANY, SW_MATCH_ALL, SW_MATCH_ALL_P,
    SW_ELECT_IN, SW_ELECT_ONE, SW_ACTIVE, SW_XCHG,
};
// A level's colour of a lane: a group of k lanes (after an odd-stride rotation of the lane order) and its complement,
// each split by fm's bits of the rotated position.  Every word gives a valid partition.
B2DP_L2_HD inline uint32_t sy_color(uint32_t w, int lane) {
    const uint32_t k = (w & 31u) + 1u, odd = ((w >> 8) & 15u) * 2u + 1u, off = (w >> 16) & 31u, fm = (w >> 24) & 31u;
    const uint32_t p = ((uint32_t)lane * odd + off) & 31u;
    return (p < k ? 0u : 64u) | (p & fm);
}
// member mask of `lane`'s group at level `level` (1..3): lanes whose colours agree on every level up to it
B2DP_L2_HD inline uint32_t sy_group(const uint32_t* wl, int level, int lane) {
    uint32_t m = 0;
    for (int l = 0; l < 32; ++l) {
        bool same = true;
        for (int v = 0; v < level; ++v) same = same && sy_color(wl[v], l) == sy_color(wl[v], lane);
        m |= (uint32_t)same << l;
    }
    return m;
}
B2DP_L2_HD inline int sy_nth(uint32_t m, int i) {  // lane of member i (0-based) of mask m
    for (int k = 0; k < i; ++k) m &= m - 1;
    for (int l = 0; l < 32; ++l)
        if (m >> l & 1) return l;
    return -1;
}
B2DP_L2_HD inline int sy_popc(uint32_t m) {
    int n = 0;
    for (int l = 0; l < 32; ++l) n += m >> l & 1;
    return n;
}
// the per-lane b operands of the four shuffles (c = 0 for up, 0x1f otherwise); every source they name is a member
B2DP_L2_HD inline void sy_shfl_b(uint32_t m, int lane, uint32_t b[4]) {
    const int n = sy_popc(m), r = sy_popc(m & ((1u << lane) - 1u));
    b[0] = (uint32_t)sy_nth(m, (r + 1) % n);
    b[1] = r > 0 ? (uint32_t)(lane - sy_nth(m, r - 1)) : (uint32_t)(lane + 1);
    b[2] = r < n - 1 ? (uint32_t)(sy_nth(m, r + 1) - lane) : (uint32_t)(32 - lane);
    b[3] = (uint32_t)(lane ^ ((r ^ 1) < n ? sy_nth(m, r ^ 1) : lane));
}

constexpr int kSySlots[kSyFormats] = {kSyAtomSlots, kSyBarSlots, kSyWarpSets * kSyWarpSetSlots};
constexpr int kSyWords[kSyFormats] = {kSyAtomWords, kSyBarWords, kSyWarpWords};

inline uint32_t sy_table_bytes(int fmt) { return (uint32_t)(kSySlots[fmt] * kCtThreads * 4); }
// Rate units of one comparison (one repetition of one tile by one CTA): SY_ATOM atomic ops, SY_BAR barrier and mbarrier
// thread-instructions, SY_WARP result words.
inline double sy_ops_per_tile(int fmt) {
    if (fmt == SY_ATOM) return (double)kCtThreads * ((kSyA32 + kSyA64) * kSyPlanes + 1);
    if (fmt == SY_BAR) {
        const double named = 15.0 * (64 + 96 + 128), red = 3.0 * 128 * 2;
        const double mbar = 2 + 4 + 3 + 64 + 1 + kCtThreads * 7.0;  // init, inval, arrivals, complete_tx, waits and tests
        return named + red + mbar;
    }
    return (double)kCtThreads * kSyWarpWords;
}

// tflops[] of the result struct is 2 x this x comparisons / ms / 1e9 (the shared driver's rule): G atomic ops/s for
// SY_ATOM, G barrier ops/s for SY_BAR, T result words/s for SY_WARP.
inline double sy_rate_half_units(int fmt) { return (fmt == SY_WARP ? 0.5 : 500.0) * sy_ops_per_tile(fmt); }

// ---- generator ------------------------------------------------------------------------------------------------------
inline uint32_t sy_stream_key(uint32_t seed, int fmt, int tile) {
    return ct_mix(seed ^ (uint32_t)(fmt * 16 + tile + 1) * 0x165667B1u);
}
inline uint32_t sy_rand(uint32_t seed, int fmt, int tile, int t, int slot) {
    return ct_hash(sy_stream_key(seed, fmt, tile), (uint32_t)(t * 256 + slot));
}
inline int sy_small(uint32_t r, int max) { return (int)(r % (uint32_t)(2 * max + 1)) - max; }  // in [-max, max]

inline void sy_operands(uint32_t seed, int fmt, int tile, uint32_t* tab) {
    const int S = kSySlots[fmt];
    auto R = [&](int t, int s) { return sy_rand(seed, fmt, tile, t, s); };
    auto U = [&](int s) { return sy_rand(seed, fmt, tile, 1000, s); };  // a CTA-uniform draw
    for (int t = 0; t < kCtThreads; ++t) {
        const int lane = t % 32, warp = t / 32;
        auto at = [&](int s) -> uint32_t& { return tab[s * kCtThreads + t]; };
        struct Slots {  // slots s0, s0 + 1, ... of thread t
            uint32_t* p;
            uint32_t& operator[](int k) const { return p[k * kCtThreads]; }
        };
        auto from = [&](int s0) { return Slots{&at(s0)}; };
        for (int s = 0; s < S; ++s) at(s) = R(t, s);
        if (fmt == SY_ATOM) {
            // the owner of a word holds its initial value: warp 0 the per-lane plane, warp 1 the bank plane, thread 64
            // the hot word; every other thread's init slot is 0
            const bool owner = warp < 2 || t == 64;
            const int k = (lane + tile) % 4;  // distance to the wrap bound: crossed within the 4 contributions
            for (int o = 0; o < kSyA32; ++o) {
                uint32_t& op = at(2 * o);
                uint32_t& in = at(2 * o + 1);
                switch (o) {
                    case A_ADD: case A_CAS: op = U(2 * o); break;
                    case A_INC: op = 2u + U(2 * o) % 15u; in = op - (uint32_t)k; break;
                    case A_DEC: op = 2u + U(2 * o) % 15u; in = (uint32_t)k; break;
                    case A_MINU: case A_MAXU:
                        if (t % 3 == 0) op |= 0x80000000u; else op &= 0x7FFFFFFFu;
                        break;
                    case A_MINS: case A_MAXS:  // both signs among every word's contributors
                        op = warp & 1 ? op | 0x80000000u : op & 0x7FFFFFFFu;
                        in ^= (uint32_t)(lane & 1) << 31;
                        break;
                    case A_F32: op = l2_f32_bits(sy_small(op, kL2F32Max)); in = l2_f32_bits(sy_small(in, 1000)); break;
                    case A_F16:
                        op = l2_f16_bits(sy_small(op, kL2F16Max)) | l2_f16_bits(sy_small(op >> 16, kL2F16Max)) << 16;
                        in = l2_f16_bits(sy_small(in, 64)) | l2_f16_bits(sy_small(in >> 16, 64)) << 16;
                        break;
                    case A_BF16:
                        op = l2_bf16_bits(sy_small(op, kL2Bf16Max)) | l2_bf16_bits(sy_small(op >> 16, kL2Bf16Max)) << 16;
                        in = l2_bf16_bits(sy_small(in, 64)) | l2_bf16_bits(sy_small(in >> 16, 64)) << 16;
                        break;
                    default: break;
                }
                if (!owner) in = 0;
            }
            for (int o = 0; o < kSyA64; ++o) {
                const Slots x = from(kSyA64Slot0 + 4 * o);
                const int s0 = kSyA64Slot0 + 4 * o;
                if (o == B_ADD || o == B_CAS) { x[0] = U(s0); x[1] = U(s0 + 1); }
                if (o == B_ADD) { x[0] |= 0xF0000000u; x[2] |= 0xF0000000u; }  // every addition carries into the high half
                if (o == B_MINS) x[1] = warp & 1 ? x[1] | 0x80000000u : x[1] & 0x7FFFFFFFu;
                if (o == B_F64) {
                    const uint64_t a = l2_f64_bits((double)((int64_t)(((uint64_t)x[1] << 32 | x[0]) % (2 * kL2F64Max + 1)) -
                                                            kL2F64Max));
                    const uint64_t b = l2_f64_bits((double)(int32_t)x[2]);
                    x[0] = (uint32_t)a; x[1] = (uint32_t)(a >> 32); x[2] = (uint32_t)b; x[3] = (uint32_t)(b >> 32);
                }
                if (!owner) x[2] = x[3] = 0;
            }
            const Slots c = from(kSyCasOnceSlot);
            if ((t + tile) & 1) c[1] = c[0];  // a hit in half the threads, a miss in the others
        } else if (fmt == SY_BAR) {
            for (int i = 0; i < kSyRed; ++i) {
                uint32_t& q = at(kSyNamed + i);
                const int cls = (tile + i) % 4;  // all zero, all one, one thread different, random
                const int odd = (tile * 5 + i * 3) % (i < 3 ? 128 : 64);
                const int me = i < 3 ? t : t % 64;
                if (cls == 0) q = me == odd;
                else if (cls == 1) q = me != odd;
                else if (cls == 2) q = (tile & 1) ? 0u : 1u;
                else q &= 1;
            }
            uint32_t& tx = at(kSyBarSlots - 1);
            tx = 1u + tx % 63u;
        } else {
            for (int s = 0; s < kSyWarpSets; ++s) {
                const Slots x = from(s * kSyWarpSetSlots);
                const int L = (tile * 4 + warp) % 32;
                // the level words are lane 0's; the other lanes hold the same value
                uint32_t w[3] = {R(warp * 32, s * 8), R(warp * 32, s * 8 + 1), R(warp * 32, s * 8 + 2)};
                if (s == 0) {  // contiguous groups of L + 1 and 31 - L lanes, then single lanes
                    w[0] = (uint32_t)L;
                    w[1] = 31u << 24;
                } else if (s == 1) {  // complementary non-contiguous halves
                    w[0] = (w[0] & 0x000F1F00u) | 15u | 0x100u;
                }
                x[0] = w[0]; x[1] = w[1]; x[2] = w[2];
                x[4] &= 1;                                         // Q
                if (s == 2) x[5] |= 0x80000000u;                   // R: signed and unsigned extremes apart
                x[6] &= 3;                                         // M: groups of equal values
                if (s & 1) x[7] = R(warp * 32, s * 8 + 7);         // M2 uniform: match.all true
            }
        }
    }
}

// ---- reference ----------------------------------------------------------------------------------------------------
inline uint32_t sy_a32(int o, uint32_t old, uint32_t x) {  // the value op o stores
    switch (o) {
        case A_ADD: case A_RADD: return old + x;
        case A_INC: return l2_inc(old, x);
        case A_DEC: return l2_dec(old, x);
        case A_EXCH: return x;
        case A_CAS: return old * kSyCasMul + x;
        case A_AND: return old & x;
        case A_OR: return old | x;
        case A_XOR: case A_RXOR: return old ^ x;
        case A_MINU: return old < x ? old : x;
        case A_MAXU: return old > x ? old : x;
        case A_MINS: return (int32_t)old < (int32_t)x ? old : x;
        case A_MAXS: return (int32_t)old > (int32_t)x ? old : x;
        case A_F32: return l2_f32_bits((double)l2_bits_f32(old) + l2_bits_f32(x));
        case A_F16:
            return l2_f16_bits(l2_f16_int(old & 0xFFFF) + l2_f16_int(x & 0xFFFF)) |
                   l2_f16_bits(l2_f16_int(old >> 16) + l2_f16_int(x >> 16)) << 16;
        default:
            return l2_bf16_bits(l2_bf16_int(old & 0xFFFF) + l2_bf16_int(x & 0xFFFF)) |
                   l2_bf16_bits(l2_bf16_int(old >> 16) + l2_bf16_int(x >> 16)) << 16;
    }
}
inline uint64_t sy_a64(int o, uint64_t old, uint64_t x) {
    switch (o) {
        case B_ADD: return old + x;
        case B_EXCH: return x;
        case B_CAS: return old * kSyCasMul64 + x;
        case B_MINS: return (int64_t)old < (int64_t)x ? old : x;
        case B_MAXU: return old > x ? old : x;
        case B_AND: return old & x;
        default: return l2_f64_bits(l2_bits_f64(old) + l2_bits_f64(x));
    }
}
// the contributors of plane p's word at `lane`, and its owner (who holds the initial value)
inline int sy_contributors(int p, int lane, int* ts) {
    if (p == 2) { for (int t = 0; t < kCtThreads; ++t) ts[t] = t; return kCtThreads; }
    for (int w = 0; w < 4; ++w) ts[w] = w * 32 + lane;
    return 4;
}
inline int sy_owner(int p, int lane) { return p == 0 ? lane : p == 1 ? 32 + lane : 64; }

inline void sy_results_bar(int tile, const uint32_t* tab, uint32_t* words);
inline void sy_results(int fmt, int tile, const uint32_t* tab, uint32_t* words) {
    const int W = kSyWords[fmt];
    auto op = [&](int t, int s) { return tab[s * kCtThreads + t]; };
    if (fmt == SY_BAR) return sy_results_bar(tile, tab, words);
    if (fmt == SY_ATOM) {
        for (int t = 0; t < kCtThreads; ++t) {
            const int lane = t % 32;
            uint32_t* o = words + (size_t)t * W;
            int j = 0, ts[kCtThreads];
            for (int a = 0; a < kSyA32; ++a) {
                if (a == A_EXCH) continue;
                for (int p = 0; p < kSyPlanes; ++p) {
                    const int n = sy_contributors(p, lane, ts);
                    uint32_t v = op(sy_owner(p, lane), 2 * a + 1);
                    for (int i = 0; i < n; ++i) v = sy_a32(a, v, op(ts[i], 2 * a));
                    o[j++] = v;
                }
            }
            for (int a = 0; a < kSyA64; ++a) {
                if (a == B_EXCH) continue;
                const int s = kSyA64Slot0 + 4 * a;
                for (int p = 0; p < kSyPlanes; ++p) {
                    const int n = sy_contributors(p, lane, ts), ow = sy_owner(p, lane);
                    uint64_t v = (uint64_t)op(ow, s + 3) << 32 | op(ow, s + 2);
                    for (int i = 0; i < n; ++i) v = sy_a64(a, v, (uint64_t)op(ts[i], s + 1) << 32 | op(ts[i], s));
                    o[j++] = (uint32_t)v;
                    o[j++] = (uint32_t)(v >> 32);
                }
            }
            const uint32_t ci = op(t, kSyCasOnceSlot), cc = op(t, kSyCasOnceSlot + 1), cn = op(t, kSyCasOnceSlot + 2);
            o[j++] = ci;
            o[j++] = ci == cc ? cn : ci;
            // return folds: {f^i(init) : i < n} for add / inc / dec / cas; {init} + {operands} for exch
            for (int r = 0; r < 8; ++r) {
                for (int p = 0; p < kSyPlanes; ++p) {
                    const int n = sy_contributors(p, lane, ts), ow = sy_owner(p, lane);
                    const uint32_t key = p == 2 ? kSyHotKey : (uint32_t)lane;
                    uint32_t sum = 0, x = 0;
                    auto add = [&](uint32_t m) { sum += m; x ^= m; };
                    if (r < 5) {
                        const int a = kSyRet32[r];
                        uint32_t v = op(ow, 2 * a + 1);
                        if (a == A_EXCH) {
                            add(l2_mix(v, key));
                            for (int i = 0; i < n; ++i) add(l2_mix(op(ts[i], 2 * a), key));
                        } else {
                            for (int i = 0; i < n; ++i) { add(l2_mix(v, key)); v = sy_a32(a, v, op(ts[0], 2 * a)); }
                        }
                    } else {
                        const int a = kSyRet64[r - 5], s = kSyA64Slot0 + 4 * a;
                        uint64_t v = (uint64_t)op(ow, s + 3) << 32 | op(ow, s + 2);
                        auto opnd = [&](int tt) { return (uint64_t)op(tt, s + 1) << 32 | op(tt, s); };
                        if (a == B_EXCH) {
                            add(l2_mix64(v, key));
                            for (int i = 0; i < n; ++i) add(l2_mix64(opnd(ts[i]), key));
                        } else {
                            for (int i = 0; i < n; ++i) { add(l2_mix64(v, key)); v = sy_a64(a, v, opnd(ts[0])); }
                        }
                    }
                    o[j++] = sum;
                    o[j++] = x;
                }
            }
        }
    } else {
        for (int w = 0; w < 4; ++w) {
            for (int s = 0; s < kSyWarpSets; ++s) {
                const int b = s * kSyWarpSetSlots;
                const uint32_t wl[3] = {op(w * 32, b), op(w * 32, b + 1), op(w * 32, b + 2)};
                for (int lv = 1; lv <= kSyLevels; ++lv) {
                    for (int lane = 0; lane < 32; ++lane) {
                        const int t = w * 32 + lane;
                        const uint32_t m = sy_group(wl, lv, lane);
                        uint32_t* o = words + (size_t)t * W + (s * kSyLevels + lv - 1) * kSyLevelWords;
                        auto V = [&](int l) { return op(w * 32 + l, b + 3); };
                        uint32_t bb[4];
                        sy_shfl_b(m, lane, bb);
                        for (int mode = 0; mode < 4; ++mode) {  // idx, up (c = 0), down, bfly (c = 0x1f)
                            const int bv = (int)(bb[mode] & 31);
                            int j;
                            bool pv;
                            if (mode == 0) { j = bv; pv = true; }
                            else if (mode == 1) { j = lane - bv; pv = j >= 0; }
                            else if (mode == 2) { j = lane + bv; pv = j <= 31; }
                            else { j = lane ^ bv; pv = true; }
                            if (!pv) j = lane;
                            o[2 * mode] = V(j);
                            o[2 * mode + 1] = pv;
                        }
                        uint32_t ballot = 0, add = 0, band = ~0u, bor = 0, bx = 0, mins = 0x7FFFFFFFu, maxu = 0, any = 0;
                        bool all = true, alleq = true;
                        const uint32_t m2 = op(t, b + 7);
                        for (int l = 0; l < 32; ++l) {
                            if (!(m >> l & 1)) continue;
                            const uint32_t q = op(w * 32 + l, b + 4) & 1, r = op(w * 32 + l, b + 5);
                            ballot |= q << l;
                            add += r; band &= r; bor |= r; bx ^= r;
                            if ((int32_t)r < (int32_t)mins) mins = r;
                            if (r > maxu) maxu = r;
                            if (op(w * 32 + l, b + 6) == op(t, b + 6)) any |= 1u << l;
                            alleq = alleq && op(w * 32 + l, b + 7) == m2;
                        }
                        all = (ballot == m);
                        o[SW_BALLOT] = ballot;
                        o[SW_ANY] = ballot != 0;
                        o[SW_ALL] = all;
                        o[SW_UNI] = ballot == 0 || all;
                        o[SW_ADD] = add; o[SW_MIN_S] = mins; o[SW_MAX_U] = maxu;
                        o[SW_AND] = band; o[SW_OR] = bor; o[SW_XOR] = bx;
                        o[SW_MATCH_ANY] = any;
                        o[SW_MATCH_ALL] = alleq ? m : 0u;
                        o[SW_MATCH_ALL_P] = alleq;
                        o[SW_ELECT_IN] = 1;
                        o[SW_ELECT_ONE] = 1;
                        o[SW_ACTIVE] = 1;
                        const int n = sy_popc(m), r = sy_popc(m & ((1u << lane) - 1u));
                        o[SW_XCHG] = V(sy_nth(m, (r + n - 1) % n)) ^ kSyXchg;
                    }
                }
            }
        }
    }
}

// SY_BAR's words of tile `tile` (its schedule depends on the tile).  A consumer's word is the producer's table value; a
// producer's or a bystander's word is 0.
inline void sy_results_bar(int tile, const uint32_t* tab, uint32_t* words) {
    const int W = kSyBarWords;
    auto op = [&](int t, int s) { return tab[s * kCtThreads + t]; };
    for (int t = 0; t < kCtThreads; ++t) {
        const int warp = t / 32, lane = t % 32;
        uint32_t* o = words + (size_t)t * W;
        for (int s = 0; s < kSyNamed; ++s) {
            int id, count;
            uint32_t pm, cm;
            sy_bar_step(tile, s, id, count, pm, cm);
            o[s] = cm >> warp & 1 ? op(sy_bar_source(pm, cm, warp) * 32 + lane, s) : 0u;
        }
        int j = kSyNamed;
        for (int mode = 0; mode < 2; ++mode) {  // id 1 over 128 threads; ids 2 / 3 over warps {0, 1} / {2, 3}
            const int lo = mode == 0 ? 0 : (t / 64) * 64, n = mode == 0 ? 128 : 64;
            uint32_t pc = 0, pa = 1, po = 0;
            for (int u = lo; u < lo + n; ++u) {
                pc += op(u, kSyNamed + 3 * mode) & 1;
                pa &= op(u, kSyNamed + 3 * mode + 1) & 1;
                po |= op(u, kSyNamed + 3 * mode + 2) & 1;
            }
            o[j++] = pc; o[j++] = pa; o[j++] = po;
        }
        // mbarrier: test_wait after noComplete (0), parity 0 / 1 after phase 0 (1, 0), parity 1 with tx pending (0),
        // parity 1 / 0 after phase 1 (1, 0)
        o[j++] = 0; o[j++] = 1; o[j++] = 0; o[j++] = 0; o[j++] = 1; o[j++] = 0;
    }
}

// table: sy_table_bytes(fmt) bytes, copied verbatim to the device; check: kCtThreads comparison values; words
// (optional): [thread][kSyWords[fmt]] reference results.
inline void sy_build_tile(uint32_t seed, int fmt, int tile, uint32_t* table, uint32_t* check,
                          std::vector<uint32_t>* words = nullptr) {
    std::vector<uint32_t> own;
    std::vector<uint32_t>& w = words ? *words : own;
    w.assign((size_t)kCtThreads * kSyWords[fmt], 0);
    sy_operands(seed, fmt, tile, table);
    sy_results(fmt, tile, table, w.data());
    for (int t = 0; t < kCtThreads; ++t) check[t] = it_fold(&w[(size_t)t * kSyWords[fmt]], kSyWords[fmt]);
    if (fmt == SY_BAR) {  // the expect_tx total thread 0 announces: the complete_tx bytes of warps 2 and 3
        uint32_t tx = 0;
        for (int t = 64; t < kCtThreads; ++t) tx += table[(kSyBarSlots - 1) * kCtThreads + t];
        table[(kSyBarSlots - 1) * kCtThreads] = tx;
    }
}

}  // namespace b2dp
