"""Independent restatement of the integer and warp-exchange self-test's host arithmetic (csrc/int_test_math.hpp) in
plain Python integers, written from the PTX ISA's text: the operand generator with its crafted classes, every op under
test, the result-word order and the fold.  It shares no code with the C++; tests/test_int_test_cpu.py holds the two
against each other, and tests/test_gpu_int_test.py holds the kernel's DUMP against this file.

Every op takes and returns unsigned 32-bit Python ints.  Optional `fault` arguments select a fault model
(tests/test_int_test_cpu.py): the default is the correct op."""
from functools import lru_cache

M32 = 0xFFFFFFFF
M64 = 0xFFFFFFFFFFFFFFFF
THREADS, TILES, REPS = 128, 8, 16
MAD, BIT, WARP = 0, 1, 2
SETS = (20, 12, 12)
SET_SLOTS = (4, 3, 7)
SET_WORDS = (14, 23, 20)
SLOTS = tuple(a * b for a, b in zip(SETS, SET_SLOTS))
WORDS = tuple(a * b for a, b in zip(SETS, SET_WORDS))
LOP3_IMM = (0x80, 0xFE, 0x96, 0xE8, 0xCA, 0x3C, 0x01, 0x69)
MAD_WORDS = ("mad_lo", "mulhi_u", "mulhi_s", "wide_u_lo", "wide_u_hi", "wide_s_lo", "wide_s_hi", "add_lo", "add_hi",
             "sub_lo", "sub_hi", "dp4a_ss", "dp4a_su", "dp4a_uu")
BIT_WORDS = tuple("lop3_%02x" % i for i in LOP3_IMM) + (
    "shf_l", "shf_r", "shr_s", "shl", "popc", "clz", "bfind_u", "bfind_s", "brev", "prmt", "min_s", "max_s", "min_u",
    "max_u", "sad")
WARP_WORDS = ("idx", "idx_p", "up", "up_p", "down", "down_p", "bfly", "bfly_p", "ballot", "add", "min_s", "max_s",
              "min_u", "max_u", "and", "or", "xor", "match_any", "match_all", "match_all_p")
WORD_NAMES = (MAD_WORDS, BIT_WORDS, WARP_WORDS)
FOLD_MUL = 2654435761
FOLD_ROT = 13
FOLD_INIT = (0x9E3779B1, 0x85EBCA77, 0xC2B2AE3D, 0x27D4EB2F)
DISTINCT_MUL = 0x9E3779B1


def s32(x):
    return x - (1 << 32) if x & 0x80000000 else x


def rotl(x, n):
    n &= 31
    return ((x << n) | (x >> (32 - n))) & M32


# ---- generator (compute_test_math.hpp's hash) ----
def mix(x):
    x ^= x >> 16
    x = x * 0x7FEB352D & M32
    x ^= x >> 15
    x = x * 0x846CA68B & M32
    x ^= x >> 16
    return x


def hash32(key, i):
    return mix((key + mix(i)) & M32)


def stream_key(seed, fmt, tile):
    return mix(seed ^ ((fmt * 16 + tile + 1) * 0xC2B2AE3D & M32))


def operand(seed, fmt, tile, t, slot):
    return hash32(stream_key(seed, fmt, tile), t * 128 + slot)


def warp_base(seed, tile, w, slot):
    return hash32(stream_key(seed, WARP, tile), 0x10000 + w * 128 + slot)


def shfl_c(width):
    return (32 - width) << 8 | 0x1F


def warp_lane(tile, w):
    """The lane a warp's one-lane classes single out: every lane over a round's 8 tiles x 4 warps."""
    return (tile * 4 + w) % 32


def thread_operands(seed, fmt, tile, t):
    """[set][k] operand words of thread t."""
    ss = SET_SLOTS[fmt]
    o = [[operand(seed, fmt, tile, t, s * ss + k) for k in range(ss)] for s in range(SETS[fmt])]
    i, w = t % 32, t // 32
    j = w * 8 + tile
    if fmt == MAD:
        o[0][0] = o[0][1] = M32
        o[1][0] = o[1][1] = 0x80000000
        o[2][1] = 0
        o[3][1] = 1
        o[4][1] = M32
        o[5][0], o[5][1] = 1 << i, 1 << j
        o[6][0], o[6][1], o[6][2] = 0x55555555, 0xAAAAAAAA, 0x2AAAAAAA
        o[7][0] |= 1
        o[7][1] |= 1
        o[7][2] = -(o[7][0] * o[7][1]) & M32
        o[8][0] |= 0x80000000
        o[8][1] |= 0x80000000
        y = (t - o[8][0] * o[8][1]) & M64
        o[8][2], o[8][3] = y & M32, y >> 32
        k = (t + tile) % 32 + 1
        o[9][0], o[9][2] = (1 << k) - 1, 1
        o[10][0], o[10][2] = M32, 1
        o[11][0], o[11][2] = 0, 1
        lane = (t + tile) % 4
        o[12][0] = o[12][1] = 0x80 << 8 * lane
        o[12][2] |= 0xFFFFC000
        o[13][0], o[13][1], o[13][2] = 0x80808080, 0x80FF80FF, M32
        o[14][0], o[14][1] = 0x80 << 8 * lane, 0xFF << 8 * lane
        o[15][0] = o[15][1] = 0xFF << 8 * lane
        o[15][2] |= 0xFFFFFF00
    elif fmt == BIT:
        o[0] = [rotl(0xF0F0F0F0, i), rotl(0xCCCCCCCC, i), rotl(0xAAAAAAAA, i)]
        o[1] = [1 << i, 1 << j, j]
        o[2] = [~(1 << i) & M32, ~(1 << j) & M32, 32 + j]
        if tile % 2 == 0:
            o[3][2] &= 63
        o[4][0], o[4][1] = 0, M32
        o[5][0] = o[5][1] = M32
        sel = o[6][2] & 0xFFFF0000
        for p in range(4):
            sel |= ((t + 5 * p + tile) & 15) << 4 * p
        o[6][2] = sel
        o[7] = [0x80000000, 0x7FFFFFFF, M32]
        o[8][1] = o[8][0]
        o[9][0] &= 0x7FFFFFFF
        o[9][1] |= 0x80000000
        o[10][0], o[10][1] = M32, 0
    else:
        V, B, C, Q, R, MA, M2 = range(7)
        L = warp_lane(tile, w)
        mask = L % 31 + 1
        for s in range(SETS[WARP]):
            o[s][V] = (warp_base(seed, tile, w, s * 7 + V) ^ i) * DISTINCT_MUL & M32
            o[s][C] = shfl_c(32)
            o[s][Q] &= 1
            o[s][MA] &= 3
            if s % 2 == 0:
                o[s][M2] = warp_base(seed, tile, w, s * 7 + M2)
        o[0][B] = i
        o[1][B] = 31 - i
        o[2][B] = (i + mask) & 31
        o[3][B] = L
        o[4][B] &= 31
        o[5][B] |= 32
        o[5][C] = shfl_c(16)
        o[6][B] = 31 - L
        o[7][B], o[7][C] = L, shfl_c(16)
        o[8][B], o[8][C] = L, shfl_c(8)
        o[9][V], o[9][B] = (M32 if tile & 1 else 0), mask
        o[10][V], o[10][B], o[10][C] = (0xAAAAAAAA if i & 1 else 0x55555555), mask, shfl_c(16)
        o[11][V], o[11][B], o[11][C] = 1 << i, mask, shfl_c(8)
        o[0][Q] = 0
        o[1][Q] |= 1
        o[2][Q] = int(i == L)
        o[3][Q] = int(i != L)
        o[0][R] = 0x80000000 if i == L else 0x40000000 | o[0][R] >> 2
        o[1][R] = 0x7FFFFFFF if i == L else 0x80000000 | o[1][R] >> 2
        o[2][R] |= 0xF0000000
        bit = 1 << (3 * L + 1) % 32
        flip = bit if i == L else 0
        o[3][R] = (warp_base(seed, tile, w, 3 * 7 + R) | bit) ^ flip
        o[4][R] = (warp_base(seed, tile, w, 4 * 7 + R) & ~bit & M32) ^ flip
        o[0][MA] = warp_base(seed, tile, w, 0 * 7 + MA)
        o[1][MA] = (warp_base(seed, tile, w, 1 * 7 + MA) ^ i) * DISTINCT_MUL & M32
        o[2][MA] = (warp_base(seed, tile, w, 2 * 7 + MA) + i % 16) & M32
        o[3][MA] = (warp_base(seed, tile, w, 3 * 7 + MA) + i % 8) & M32
        o[4][MA] = (warp_base(seed, tile, w, 4 * 7 + MA) + i % 2) & M32
        o[1][M2] = warp_base(seed, tile, w, 1 * 7 + M2) ^ ((1 << L) if i == L else 0)
    return o


@lru_cache(maxsize=None)
def tile_operands(seed, fmt, tile):
    """[thread][set][k]"""
    return [thread_operands(seed, fmt, tile, t) for t in range(THREADS)]


def table(seed, fmt, tile):
    """The [slot][thread] table the device reads, flattened."""
    ops = tile_operands(seed, fmt, tile)
    ss = SET_SLOTS[fmt]
    return [ops[t][slot // ss][slot % ss] for slot in range(SLOTS[fmt]) for t in range(THREADS)]


# ---- the ops, from the PTX ISA.  `fault` = None is the correct op. ----
def mul_u64(a, b, fault=None):
    """a * b, unsigned, as the sum of 32 x 32 partial-product bits; ('column', c) drops every partial-product bit of
    weight 2^c."""
    if fault and fault[0] == "column":
        c = fault[1]
        dropped = sum(1 for x in range(32) if 0 <= c - x < 32 and a >> x & 1 and b >> (c - x) & 1)
        return a * b - (dropped << c)
    return a * b


def mul_s64(a, b, fault=None):
    if fault and fault[0] == "column":  # Baugh-Wooley on the unsigned array: signed = unsigned - (a<0 ? b<<32) - ...
        p = mul_u64(a, b, fault)
        if a & 0x80000000:
            p -= b << 32
        if b & 0x80000000:
            p -= a << 32
        return p & M64
    return s32(a) * s32(b) & M64


def add64(x, y, fault=None):
    """x + y mod 2^64; ('carry', k): the carry out of bit k - 1 into bit k is lost."""
    if fault and fault[0] == "carry":
        k = fault[1]
        lo = (x & ((1 << k) - 1)) + (y & ((1 << k) - 1))
        return ((lo & ((1 << k) - 1)) | ((x >> k) + (y >> k) << k)) & M64
    return (x + y) & M64


def dp4a(a, b, c, sa, sb, fault=None):
    if fault and fault[0] == "dp4a_sign" and fault[1] == (sa, sb):
        lane_fault = fault[2]
    else:
        lane_fault = None
    s = 0
    for i in range(4):
        xa, xb = a >> 8 * i & 0xFF, b >> 8 * i & 0xFF
        sa_i = (not sa) if lane_fault == i else sa
        if sa_i and xa & 0x80:
            xa -= 256
        if sb and xb & 0x80:
            xb -= 256
        s += xa * xb
    if fault and fault[0] == "dp4a_sat":
        if sa or sb:
            return max(-(1 << 31), min((1 << 31) - 1, s32(c) + s)) & M32
        return min(M32, max(0, c + s))
    return (c + s) & M32


def mad_words(o, fault=None):
    a, b, c, d = o
    x, y = b << 32 | a, d << 32 | c
    colf = fault if fault and fault[0] == "column" else None
    carf = fault if fault and fault[0] == "carry" else None
    pu, ps = mul_u64(a, b, colf), mul_s64(a, b, colf)
    mulhi_s = ps >> 32 & M32
    if fault and fault[0] == "mulhi_unsigned":
        mulhi_s = a * b >> 32
    wu, ws = (pu + y) & M64, (ps + y) & M64
    add, sub = add64(x, y, carf), add64(x, (-y) & M64, None)
    if carf:  # the borrow chain is the carry chain of x + ~y + 1
        sub = add64(add64(x, ~y & M64, carf), 1, carf)
    return [(pu + c) & M32, pu >> 32 & M32, mulhi_s, wu & M32, wu >> 32, ws & M32, ws >> 32, add & M32, add >> 32,
            sub & M32, sub >> 32, dp4a(a, b, c, True, True, fault), dp4a(a, b, c, True, False, fault),
            dp4a(a, b, c, False, False, fault)]


def lop3(a, b, c, imm):
    d = 0
    for bit in range(32):
        idx = (a >> bit & 1) << 2 | (b >> bit & 1) << 1 | (c >> bit & 1)
        d |= (imm >> idx & 1) << bit
    return d


def shift_amount(c, fault):
    if fault and fault[0] == "shift_stage":
        return c & ~(1 << fault[1]) & M32
    return c


def shf_l_wrap(lo, hi, c):
    n = c & 31
    return ((hi << 32 | lo) << n >> 32) & M32


def shf_r_wrap(lo, hi, c):
    n = c & 31
    return ((hi << 32 | lo) >> n) & M32


def shr_s32(a, c):
    return (s32(a) >> min(c, 32)) & M32


def shl(a, c):
    return (a << min(c, 32)) & M32


def popc(a):
    return bin(a).count("1")


def clz(a):
    return 32 - a.bit_length()


def bfind_u(a):
    return a.bit_length() - 1 if a else M32


def bfind_s(a):
    return bfind_u(~a & M32 if a & 0x80000000 else a)


def brev(a):
    return int("{:032b}".format(a)[::-1], 2)


def prmt(a, b, c, fault=None):
    src = (a | b << 32).to_bytes(8, "little")
    d = 0
    for i in range(4):
        sel = c >> 4 * i & 0xF
        if fault and fault[0] == "prmt_route" and sel == fault[1]:
            sel ^= 1
        byte = src[sel & 7]
        if sel & 8:
            byte = 0xFF if byte & 0x80 else 0
        d |= byte << 8 * i
    return d


def bit_words(o, fault=None):
    a, b, c = o
    f = fault[0] if fault else None
    out = []
    for imm in LOP3_IMM:
        out.append(lop3(a, b, c, imm ^ (1 << fault[1]) if f == "lop3_minterm" else imm))
    n = shift_amount(c, fault)
    out += [shf_l_wrap(a, b, n), shf_r_wrap(a, b, n), shr_s32(a, n), shl(a, n)]
    pc = popc(a)
    if f == "popc_off" and a >> fault[1] & 1:
        pc += 1
    cz = clz(b)
    if f == "clz0" and b == 0:
        cz = 31
    br = brev(a)
    if f == "brev_bytes":
        br = int.from_bytes(a.to_bytes(4, "little"), "big")
    out += [pc, cz, bfind_u(a), bfind_s(a), br, prmt(a, b, c, fault)]
    sa, sb = s32(a), s32(b)
    mins, maxs = (a if sa < sb else b), (a if sa > sb else b)
    minu, maxu = min(a, b), max(a, b)
    if f == "cmp_swapped":
        mins, maxs, minu, maxu = minu, maxu, mins, maxs
    out += [mins, maxs, minu, maxu, (c + abs(a - b)) & M32]
    return out


def shfl(mode, v, b, c, fault=None):
    """One warp: lists of 32.  Returns (d, p)."""
    f = fault[0] if fault else None
    d, p = [], []
    for lane in range(32):
        bval, cval, segmask = b[lane] & 31, c[lane] & 31, c[lane] >> 8 & 31
        if f == "segment_ignored" and segmask == 0x10:
            segmask = 0
        max_lane = (lane & segmask) | (cval & ~segmask & 31)
        min_lane = lane & segmask
        if mode == "up":
            j = lane - bval
            pv = j >= max_lane
        elif mode == "down":
            j = lane + bval
            pv = j <= max_lane
        elif mode == "bfly":
            j = lane ^ bval
            pv = j <= max_lane
        else:
            j = min_lane | (bval & ~segmask & 31)
            pv = j <= max_lane
        if not pv:
            j = lane
        if f == "lane_swap" and j == fault[1] and j != lane:
            j = fault[2]
        x = v[j]
        if f == "bit_dropped" and j == fault[1] and j != lane:
            x &= ~(1 << fault[2]) & M32
        d.append(x)
        p.append(1 if f == "pred_true" else int(pv))
    return d, p


def warp_words(ops, fault=None):
    """ops: [lane][k] of one set of one warp.  Returns [lane][word]."""
    f = fault[0] if fault else None
    col = lambda k: [ops[l][k] for l in range(32)]
    v, b, c, q, r, m, m2 = (col(k) for k in range(7))
    out = [[] for _ in range(32)]
    for mode in ("idx", "up", "down", "bfly"):
        cc = [x & 0x1F00 for x in c] if mode == "up" else c
        d, p = shfl(mode, v, b, cc, fault)
        for l in range(32):
            out[l] += [d[l], p[l]]
    ballot = sum(1 << l for l in range(32) if q[l] and not (f == "ballot_miss" and l == fault[1]))
    rr = [x for l, x in enumerate(r) if not (f == "redux_skip" and l == fault[1])]
    band, bor, bxor = M32, 0, 0
    for x in rr:
        band, bor, bxor = band & x, bor | x, bxor ^ x
    red = [sum(rr) & M32, min(rr, key=s32), max(rr, key=s32), min(rr), max(rr), band, bor, bxor]
    allsame = all(x == m2[0] for x in m2)
    for l in range(32):
        any_ = sum(1 << k for k in range(32) if m[k] == m[l] and not (f == "match_miss" and k == fault[1] and k != l))
        out[l] += [ballot] + red + [any_, M32 if allsame else 0, int(allsame)]
    return out


@lru_cache(maxsize=None)
def tile_words(seed, fmt, tile, fault=None):
    """[thread][word] result words of a tile under an optional fault model."""
    ops = tile_operands(seed, fmt, tile)
    if fmt == WARP:
        res = [[] for _ in range(THREADS)]
        for s in range(SETS[WARP]):
            for w in range(THREADS // 32):
                ww = warp_words([ops[w * 32 + l][s] for l in range(32)], fault)
                for l in range(32):
                    res[w * 32 + l] += ww[l]
        return res
    fn = mad_words if fmt == MAD else bit_words
    return [[x for s in range(SETS[fmt]) for x in fn(ops[t][s], fault)] for t in range(THREADS)]


def fold(words):
    h = list(FOLD_INIT)
    for i, w in enumerate(words):
        h[i & 3] = rotl(((h[i & 3] ^ w) * FOLD_MUL) & M32, FOLD_ROT)
    return h[0] ^ rotl(h[1], 8) ^ rotl(h[2], 16) ^ rotl(h[3], 24)


def old_fold(words):
    """The other self-tests' fold, sum (2j + 1) w_j: kept to show what it misses."""
    return sum((2 * j + 1) * w for j, w in enumerate(words)) & M32


def tile_checks(seed, fmt, tile, fault=None):
    return [fold(w) for w in tile_words(seed, fmt, tile, fault)]
