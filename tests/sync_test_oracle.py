"""An independent restatement of the synchronization self-test's reference (csrc/sync_test_math.hpp), from the PTX ISA.

The C++ reference computes order-free values in closed form (a final by folding the contributions in thread order, a
return set as {f^i(init)}).  This module instead *simulates* the shared-memory words: every contribution reads the
word, returns what it read and stores the op's result, in an order drawn at random, and the result words are formed
the way the kernel forms them (finals read back, returns mixed and summed / xored per word).  `results` replays each
tile in several orders and asserts that every word is the same in all of them.  Barrier words follow the producer /
consumer schedule and the mbarrier phase rules; warp words follow the ISA's definition of each collective over the
group's member mask.

`fault` names a hardware fault model; the words are then what a device with that fault would fold, so
`checks(..., fault=...)` are the check values such a device would match (test_sync_test_cpu.py, test_gpu_sync_test.py).
"""
import random

import int_test_oracle as it
from l2_test_oracle import bf16_bits, bf16_int, bits_f32, bits_f64, f16_bits, f16_int, f32_bits, f64_bits, l2_mix, \
    l2_mix64

M32, M64 = 0xFFFFFFFF, (1 << 64) - 1
THREADS, TILES = 128, 8
ATOM, BAR, WARP = 0, 1, 2
# SY_ATOM: 32-bit ops, 64-bit ops, planes (per-lane, same-bank, hot)
A_ADD, A_INC, A_DEC, A_EXCH, A_CAS, A_AND, A_OR, A_XOR, A_MINU, A_MAXU, A_MINS, A_MAXS, A_RADD, A_RXOR, A_F32, A_F16, \
    A_BF16 = range(17)
B_ADD, B_EXCH, B_CAS, B_MINS, B_MAXU, B_AND, B_F64 = range(7)
A64_SLOT0, CASONCE_SLOT = 34, 62
SLOTS = (65, 52, 32)
WORDS = (134, 57, 300)
CAS_MUL, CAS_MUL64 = 0x01000193, 0x100000001B3
HOT_KEY = 32
F32_MAX, F16_MAX, BF16_MAX, F64_MAX = 1000, 3, 1, 1 << 40
# SY_BAR
NAMED, RED = 45, 6
KEY_MUL = 0x9E3779B9
# SY_WARP
SETS, LEVELS, SET_SLOTS, LEVEL_WORDS = 4, 3, 8, 25
XCHG = 0x5A5A5A5A

FAULTS = {
    ATOM: ("dropped", "doubled", "post_value", "cas_stores_on_miss", "wrap_bound", "lost_carry", "signedness",
           "f16_halves"),
    BAR: ("early_release", "popc_off_by_one", "and_or_swapped", "parity_stuck", "tx_ignored"),
    WARP: ("shfl_whole_warp", "ballot_whole_warp", "redux_whole_warp", "elect_none", "elect_two", "syncwarp_unordered"),
}


def s32(x):
    return it.s32(x & M32)


def s64(x):
    return x - (1 << 64) if x >> 63 else x


# ---- generator: the table is [slot][thread] words --------------------------------------------------------------------
def stream_key(seed, fmt, tile):
    return it.mix(seed ^ ((fmt * 16 + tile + 1) * 0x165667B1 & M32))


def rnd(seed, fmt, tile, t, slot):
    return it.hash32(stream_key(seed, fmt, tile), (t * 256 + slot) & M32)


def small(r, mx):
    return r % (2 * mx + 1) - mx


def table(seed, fmt, tile):
    T = [[rnd(seed, fmt, tile, t, s) for t in range(THREADS)] for s in range(SLOTS[fmt])]
    U = lambda s: rnd(seed, fmt, tile, 1000, s)  # noqa: E731  a CTA-uniform draw
    for t in range(THREADS):
        lane, warp = t % 32, t // 32
        if fmt == ATOM:
            owner = warp < 2 or t == 64
            k = (lane + tile) % 4
            for o in range(17):
                op, inn = T[2 * o][t], T[2 * o + 1][t]
                if o in (A_ADD, A_CAS):
                    op = U(2 * o)
                elif o == A_INC:
                    op = 2 + U(2 * o) % 15
                    inn = (op - k) & M32
                elif o == A_DEC:
                    op = 2 + U(2 * o) % 15
                    inn = k
                elif o in (A_MINU, A_MAXU):
                    op = op | 0x80000000 if t % 3 == 0 else op & 0x7FFFFFFF
                elif o in (A_MINS, A_MAXS):
                    op = op | 0x80000000 if warp & 1 else op & 0x7FFFFFFF
                    inn ^= (lane & 1) << 31
                elif o == A_F32:
                    op, inn = f32_bits(small(op, F32_MAX)), f32_bits(small(inn, 1000))
                elif o == A_F16:
                    op = f16_bits(small(op, F16_MAX)) | f16_bits(small(op >> 16, F16_MAX)) << 16
                    inn = f16_bits(small(inn, 64)) | f16_bits(small(inn >> 16, 64)) << 16
                elif o == A_BF16:
                    op = bf16_bits(small(op, BF16_MAX)) | bf16_bits(small(op >> 16, BF16_MAX)) << 16
                    inn = bf16_bits(small(inn, 64)) | bf16_bits(small(inn >> 16, 64)) << 16
                T[2 * o][t], T[2 * o + 1][t] = op, inn if owner else 0
            for o in range(7):
                s0 = A64_SLOT0 + 4 * o
                x = [T[s0 + i][t] for i in range(4)]
                if o in (B_ADD, B_CAS):
                    x[0], x[1] = U(s0), U(s0 + 1)
                if o == B_ADD:
                    x[0] |= 0xF0000000
                    x[2] |= 0xF0000000
                if o == B_MINS:
                    x[1] = x[1] | 0x80000000 if warp & 1 else x[1] & 0x7FFFFFFF
                if o == B_F64:
                    a = f64_bits(float((x[1] << 32 | x[0]) % (2 * F64_MAX + 1) - F64_MAX))
                    b = f64_bits(float(s32(x[2])))
                    x = [a & M32, a >> 32, b & M32, b >> 32]
                if not owner:
                    x[2] = x[3] = 0
                for i in range(4):
                    T[s0 + i][t] = x[i]
            if (t + tile) & 1:
                T[CASONCE_SLOT + 1][t] = T[CASONCE_SLOT][t]
        elif fmt == BAR:
            for i in range(RED):
                cls, odd = (tile + i) % 4, (tile * 5 + i * 3) % (128 if i < 3 else 64)
                me = t if i < 3 else t % 64
                q = T[NAMED + i][t]
                T[NAMED + i][t] = [int(me == odd), int(me != odd), 0 if tile & 1 else 1, q & 1][cls]
            T[51][t] = 1 + T[51][t] % 63
        else:
            L = (tile * 4 + warp) % 32
            for s in range(SETS):
                b = s * SET_SLOTS
                w = [rnd(seed, fmt, tile, warp * 32, s * 8 + v) for v in range(3)]
                if s == 0:
                    w[0], w[1] = L, 31 << 24
                elif s == 1:
                    w[0] = (w[0] & 0x000F1F00) | 15 | 0x100
                T[b][t], T[b + 1][t], T[b + 2][t] = w
                T[b + 4][t] &= 1
                if s == 2:
                    T[b + 5][t] |= 0x80000000
                T[b + 6][t] &= 3
                if s & 1:
                    T[b + 7][t] = rnd(seed, fmt, tile, warp * 32, s * 8 + 7)
    if fmt == BAR:
        T[51][0] = sum(T[51][64:])  # thread 0's expect_tx: the complete_tx bytes of warps 2 and 3
    return T


# ---- SY_ATOM: the ops as the ISA states them (d = old; [a] = f(old, b)) ----------------------------------------------
def f16_add(a, b, fault=None):
    lo = f16_bits(f16_int(a & 0xFFFF) + f16_int(b & 0xFFFF)) & 0xFFFF
    hi = f16_bits(f16_int(a >> 16) + f16_int(b >> 16)) & 0xFFFF
    return lo << 16 | hi if fault == "f16_halves" else hi << 16 | lo


def bf16_add(a, b):
    return bf16_bits(bf16_int(a & 0xFFFF) + bf16_int(b & 0xFFFF)) | bf16_bits(bf16_int(a >> 16) + bf16_int(b >> 16)) << 16


def op32(o, old, b, fault=None):
    if o in (A_ADD, A_RADD):
        return (old + b) & M32
    if o == A_INC:  # atom.inc: (old >= b) ? 0 : old + 1
        return 0 if old >= b + (1 if fault == "wrap_bound" else 0) else old + 1
    if o == A_DEC:  # atom.dec: (old == 0 || old > b) ? b : old - 1
        return b if old == 0 or old > b else old - 1
    if o == A_EXCH:
        return b
    if o == A_CAS:
        return (old * CAS_MUL + b) & M32
    if o == A_AND:
        return old & b
    if o == A_OR:
        return old | b
    if o in (A_XOR, A_RXOR):
        return old ^ b
    if o == A_MINU:
        return min(old, b)
    if o == A_MAXU:
        return max(old, b)
    if o in (A_MINS, A_MAXS):
        key = (lambda v: v) if fault == "signedness" else s32
        pick = min if o == A_MINS else max
        return pick(old, b, key=key)
    if o == A_F32:
        return f32_bits(bits_f32(old) + bits_f32(b))
    if o == A_F16:
        return f16_add(old, b, fault)
    return bf16_add(old, b)


def op64(o, old, b, fault=None):
    if o == B_ADD:
        if fault == "lost_carry":
            return (((old >> 32) + (b >> 32)) & M32) << 32 | ((old + b) & M32)
        return (old + b) & M64
    if o == B_EXCH:
        return b
    if o == B_CAS:
        return (old * CAS_MUL64 + b) & M64
    if o == B_MINS:
        return min(old, b, key=s64)
    if o == B_MAXU:
        return max(old, b)
    if o == B_AND:
        return old & b
    return f64_bits(bits_f64(old) + bits_f64(b))


def _contributors(p, lane):
    return list(range(THREADS)) if p == 2 else [w * 32 + lane for w in range(4)]


def _owner(p, lane):
    return (lane, 32 + lane, 64)[p]


def _word(T, s, t, wide):
    return T[s + 1][t] << 32 | T[s][t] if wide else T[s][t]


def atom_words(T, rng, fault=None):
    """One replay of every contribution in a random order per word; returns [thread][word]."""
    fin, ret = {}, {}  # (wide, o, p, lane) -> final; (wide, o, p, t) -> returned value
    for wide, nops in ((False, 17), (True, 7)):
        for o in range(nops):
            s_op = A64_SLOT0 + 4 * o if wide else 2 * o
            s_in = s_op + 2 if wide else s_op + 1
            for p in range(3):
                for lane in (range(32) if p < 2 else (0,)):
                    ts = _contributors(p, lane)
                    rng.shuffle(ts)
                    v = _word(T, s_in, _owner(p, lane), wide)
                    for i, t in enumerate(ts):
                        b = _word(T, s_op, t, wide)
                        if fault == "dropped" and not wide and o == A_ADD and p == 2 and i == 0:
                            ret[wide, o, p, t] = v  # the unit answers but never stores
                            continue
                        new = op64(o, v, b, fault) if wide else op32(o, v, b, fault)
                        if fault == "doubled" and not wide and o == A_ADD and p == 2 and i == 0:
                            new = op32(o, new, b)
                        ret[wide, o, p, t] = new if fault == "post_value" and o in (A_ADD, A_INC, A_DEC) \
                            and not wide else v
                        v = new
                    fin[wide, o, p, lane] = v
    out = []
    for t in range(THREADS):
        lane = t % 32
        w = []
        for o in range(17):
            if o != A_EXCH:
                w += [fin[False, o, p, lane if p < 2 else 0] for p in range(3)]
        for o in range(7):
            if o != B_EXCH:
                for p in range(3):
                    v = fin[True, o, p, lane if p < 2 else 0]
                    w += [v & M32, v >> 32]
        ci, cc, cn = T[CASONCE_SLOT][t], T[CASONCE_SLOT + 1][t], T[CASONCE_SLOT + 2][t]
        w += [ci, cn if ci == cc or fault == "cas_stores_on_miss" else ci]
        for wide, o in [(False, x) for x in (A_ADD, A_INC, A_DEC, A_EXCH, A_CAS)] + \
                       [(True, x) for x in (B_ADD, B_EXCH, B_CAS)]:
            mixf = l2_mix64 if wide else l2_mix
            for p in range(3):
                key = HOT_KEY if p == 2 else lane
                vals = [ret[wide, o, p, u] for u in _contributors(p, lane)]
                if o == (B_EXCH if wide else A_EXCH):
                    vals.append(fin[wide, o, p, lane if p < 2 else 0])
                m = [mixf(v, key) for v in vals]
                x = 0
                for v in m:
                    x ^= v
                w += [sum(m) & M32, x]
        out.append(w)
    return out


# ---- SY_BAR ----------------------------------------------------------------------------------------------------------
def bar_step(tile, s):
    g, ident = s // 15, s % 15 + 1
    k = g + 2
    start, np_ = (tile + ident + g) % 4, 1 + (tile + 2 * ident + g) % (k - 1)
    part = [(start + i) % 4 for i in range(k)]
    return ident, 32 * k, part[:np_], part[np_:]


def bar_words(T, tile, fault=None):
    out = []
    for t in range(THREADS):
        warp, lane = t // 32, t % 32
        w = []
        for s in range(NAMED):
            _, _, prod, cons = bar_step(tile, s)
            if warp in cons:
                # the consumer's rank among the consumers picks a producer, both in warp order
                src = sorted(prod)[sorted(cons).index(warp) % len(prod)]
                v = T[s][src * 32 + lane]
                # released one repetition early: the producer has not stored yet, so the consumer reads the previous
                # comparison's value, keyed one step back (here as in comparison 1: key 1 instead of key 2)
                w.append(v ^ ((KEY_MUL ^ (2 * KEY_MUL)) & M32 if fault == "early_release" else 0))
            else:
                w.append(0)
        for mode in range(2):
            us = range(128) if mode == 0 else range(t // 64 * 64, t // 64 * 64 + 64)
            q = [[T[NAMED + 3 * mode + i][u] & 1 for u in us] for i in range(3)]
            popc, band, bor = sum(q[0]), int(all(q[1])), int(any(q[2]))
            if fault == "popc_off_by_one":
                popc += 1
            if fault == "and_or_swapped":
                band, bor = int(any(q[1])), int(all(q[2]))
            w += [popc, band, bor]
        # mbarrier: noComplete leaves the phase pending; each completed phase flips the parity once; pending tx holds
        # phase 1 open until the last complete_tx
        done0, done1 = (0, 0) if fault == "parity_stuck" else (1, 1)
        pending_tx = 0 if fault == "tx_ignored" else 1
        w += [0, done0, 1 - done0 if fault != "parity_stuck" else 0, 1 - pending_tx, done1,
              1 - done1 if fault != "parity_stuck" else 0]
        out.append(w)
    return out


# ---- SY_WARP ---------------------------------------------------------------------------------------------------------
def color(w, lane):
    k, odd, off, fm = (w & 31) + 1, ((w >> 8) & 15) * 2 + 1, (w >> 16) & 31, (w >> 24) & 31
    p = (lane * odd + off) & 31
    return (0 if p < k else 64) | (p & fm)


def group(wl, level, lane):
    c = tuple(color(wl[v], lane) for v in range(level))
    return [l for l in range(32) if tuple(color(wl[v], l) for v in range(level)) == c]


def warp_words(T, fault=None):
    out = [[0] * WORDS[WARP] for _ in range(THREADS)]
    for w in range(4):
        for s in range(SETS):
            b = s * SET_SLOTS
            wl = [T[b + v][w * 32] for v in range(3)]
            V = [T[b + 3][w * 32 + l] for l in range(32)]
            Q = [T[b + 4][w * 32 + l] & 1 for l in range(32)]
            R = [T[b + 5][w * 32 + l] for l in range(32)]
            Mv = [T[b + 6][w * 32 + l] for l in range(32)]
            M2 = [T[b + 7][w * 32 + l] for l in range(32)]
            prevV = [T[((s - 1) % SETS) * SET_SLOTS + 3][w * 32 + l] for l in range(32)]
            for lv in range(1, LEVELS + 1):
                for lane in range(32):
                    g = group(wl, lv, lane)
                    n, r = len(g), g.index(lane)
                    o = out[w * 32 + lane]
                    J = (s * LEVELS + lv - 1) * LEVEL_WORDS
                    # shuffles: the source is a member (idx: the next, up: the previous, down: the next, bfly: the
                    # rank ^ 1 partner); up / down with no such member name a lane out of range: p false, own value
                    gs = list(range(32)) if fault == "shfl_whole_warp" else g
                    rs = gs.index(lane)
                    src = [gs[(rs + 1) % len(gs)], gs[rs - 1] if rs > 0 else None,
                           gs[rs + 1] if rs < len(gs) - 1 else None, gs[rs ^ 1] if (rs ^ 1) < len(gs) else lane]
                    if src[2] is None and lane == 0:
                        src[2] = 0  # b = 32 - lane is 32, whose low five bits name lane 0 itself: in range
                    if src[1] is None and lane == 31:
                        src[1] = 31  # b = lane + 1 = 32 names lane 31 itself
                    for mode in range(4):
                        j = src[mode]
                        o[J + 2 * mode] = V[j] if j is not None else V[lane]
                        o[J + 2 * mode + 1] = int(j is not None)
                    vg = list(range(32)) if fault == "ballot_whole_warp" else g
                    ballot = sum(Q[l] << l for l in vg)
                    mem = sum(1 << l for l in g)
                    o[J + 8] = ballot
                    o[J + 9] = int(any(Q[l] for l in g))
                    o[J + 10] = int(all(Q[l] for l in g))
                    o[J + 11] = int(len({Q[l] for l in g}) == 1)
                    rg = list(range(32)) if fault == "redux_whole_warp" else g
                    rv = [R[l] for l in rg]
                    a = o_ = 0
                    an = M32
                    for v in rv:
                        a ^= v
                        o_ |= v
                        an &= v
                    o[J + 12] = sum(rv) & M32
                    o[J + 13] = min(rv, key=s32)
                    o[J + 14] = max(rv)
                    o[J + 15], o[J + 16], o[J + 17] = an, o_, a
                    o[J + 18] = sum(1 << l for l in g if Mv[l] == Mv[lane])
                    alleq = len({M2[l] for l in g}) == 1
                    o[J + 19], o[J + 20] = (mem if alleq else 0), int(alleq)
                    # elect.sync: one member elected, every member names it; which member is not checked
                    o[J + 21] = 1
                    o[J + 22] = 0 if fault == "elect_none" or (fault == "elect_two" and n > 1) else 1
                    o[J + 23] = 1  # activemask: own lane set, nothing outside the group
                    prev = g[(r + n - 1) % n]
                    stale = fault == "syncwarp_unordered" and lv == 1 and n > 1
                    o[J + 24] = (prevV[prev] if stale else V[prev]) ^ XCHG
    return out


# ---- the tile --------------------------------------------------------------------------------------------------------
def fold(words):
    h = list(it.FOLD_INIT)
    for i, w in enumerate(words):
        h[i & 3] = it.rotl(((h[i & 3] ^ w) * it.FOLD_MUL) & M32, it.FOLD_ROT)
    return h[0] ^ it.rotl(h[1], 8) ^ it.rotl(h[2], 16) ^ it.rotl(h[3], 24)


def results(T, fmt, tile, fault=None, orders=3, seed=0):
    """Every thread's result words; SY_ATOM is replayed in `orders` random orders, which must all agree."""
    if fmt == ATOM:
        rng = random.Random(seed * 7919 + tile)
        first = atom_words(T, rng, fault)
        for _ in range(orders - 1):
            assert atom_words(T, rng, fault) == first, "an SY_ATOM word depends on the order of the atomics"
        return first
    if fmt == BAR:
        return bar_words(T, tile, fault)
    return warp_words(T, fault)


def checks(seed, fmt, tile, fault=None, orders=1):
    T = table(seed, fmt, tile)
    return [fold(w) for w in results(T, fmt, tile, fault, orders, seed)]
