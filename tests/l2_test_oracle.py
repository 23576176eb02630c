"""Python restatement of the L2 self-test's host arithmetic (csrc/l2_test_math.hpp) and a model of what its kernel
(csrc/l2_selftest.cuh) leaves behind, written from the march and op definitions rather than from the C++.

- WORD / BYTE: tile(seed, fmt, t) gives the tile table and every thread's check; window(table, span) the image a clean
  march leaves (P everywhere); reads(fmt, kd, ky, t) the values a thread reads from one block, block key removed.
- ATOM: operand(), init(), finals(seed, t) (every slot's value after n = 0 .. MAX_N contributions, in contribution
  order q = 0, 1, ...) and atom_expected(seed, t, G) -- the hot block and the combined return folds after one
  comparison on a grid of G CTAs.  The ops commute, so applying them in any order gives the same finals.
The data backgrounds are the shared-memory test's (tests/smem_test_oracle.py).
"""
import struct

import numpy as np

import smem_test_oracle as so

TILES, THREADS, REPS = so.TILES, so.THREADS, so.REPS
WORD, BYTE, ATOM = 0, 1, 2
BLOCK_WORDS = 4 * THREADS
BLOCK_MUL = 0x9E3779B9
HOOK_WORD, HOOK_ELEMENT = 37, 0
TABLE_WORDS = 8
M32 = 0xFFFFFFFF

# ATOM slots (l2_test_math.hpp L2AtomSlot)
ADD, INC, DEC, EXCH, CAS32, CAS64 = 0, 1, 2, 3, 4, 5
AND, OR, XOR, MIN_S, MAX_S, MIN_U, MAX_U = 7, 8, 9, 10, 11, 12, 13
ADD64, F32, F64, F16X2, BF16X2, V4RED, V4ATOM = 14, 16, 17, 19, 20, 21, 25
SLOTS, ROWS, MAX_N = 29, 32, 512
ATOM_HOT_WORDS = SLOTS * ROWS * 32
RET_SLOTS = (ADD, INC, DEC, EXCH, CAS32, CAS64)
ATOM_RET = len(RET_SLOTS)
F32_MAX, F16_MAX, BF16_MAX, F64_MAX = 1000, 3, 1, 1 << 40
WRAP_MAX = 16                      # inc / dec bounds 2 .. 16: every word wraps once it takes 17 contributions


# ---- WORD / BYTE ------------------------------------------------------------------------------------------------------
def l2_pattern(kd, ky, blockmul, w):
    w = np.asarray(w, dtype=np.uint64)
    bk = (((w // BLOCK_WORDS) + 1) * np.uint64(blockmul)) & np.uint64(M32)
    return so.pattern(kd, ky, w % BLOCK_WORDS) ^ bk.astype(np.uint32)


def reads(fmt, kd, ky, t):
    base = so.pattern(kd, ky, np.arange(4 * t, 4 * t + 4))
    invs = (0, M32, 0, M32, 0) if fmt == WORD else (0, M32, 0)
    return np.concatenate([base ^ np.uint32(i) for i in invs])


def tile(seed, fmt, t):
    kd = so.kind(t)
    table = np.zeros(TABLE_WORDS, np.uint32)
    table[:5] = [kd, so.key(seed, 3 + fmt, t), BLOCK_MUL if kd == 4 else 0, HOOK_WORD, HOOK_ELEMENT]
    checks = np.array([so.fold(reads(fmt, kd, int(table[1]), th)) for th in range(THREADS)], np.uint32)
    return table, checks


def window(table, span_words):
    return l2_pattern(int(table[0]), int(table[1]), int(table[2]), np.arange(span_words))


# ---- ATOM -------------------------------------------------------------------------------------------------------------
def fmix(h):
    h &= M32
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M32
    h ^= h >> 16
    return h


def l2_mix(v, lane):
    return fmix(v ^ (((lane + 1) * 0x9E3779B9) & M32))


def l2_mix64(v, lane):
    return l2_mix((v & M32) ^ l2_mix(v >> 32, lane + 32), lane)


def rand(seed, t, a, b):
    return l2_mix(seed ^ l2_mix((t * 0x632BE5AB + a * 0x85157AF5 + b) & M32, 77), 91)


def f32_bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def bits_f32(u):
    return struct.unpack("<f", struct.pack("<I", u))[0]


def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def bits_f64(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


def f16_bits(i):
    return int(np.array(i, np.float16).view(np.uint16))


def f16_int(b):
    return int(np.array(b & 0xFFFF, np.uint16).view(np.float16))


def bf16_bits(i):
    return f32_bits(float(i)) >> 16


def bf16_int(b):
    return int(bits_f32((b & 0xFFFF) << 16))


def operand(seed, t, s, q):
    r, b = rand(seed, t, 100 + s, q), rand(seed, t, 200 + s, 0)
    if s == ADD:
        return 1
    if s in (INC, DEC):
        return 2 + b % (WRAP_MAX - 1)
    if s in (EXCH, XOR):
        return r | 1
    if s in (CAS32, CAS64, CAS64 + 1):
        return 0
    if s == AND:
        return ~(1 << (q & 31)) & M32
    if s == OR:
        return 1 << (q & 31)
    if s == ADD64:
        return r
    if s == ADD64 + 1:
        return r & 0xFF
    if s in (F64, F64 + 1):
        v = ((rand(seed, t, 100 + F64, q) << 9) % (2 * F64_MAX + 1)) - F64_MAX
        u = f64_bits(float(v))
        return u & M32 if s == F64 else u >> 32
    if s == F16X2:
        lo, hi = r % (2 * F16_MAX + 1) - F16_MAX, (r >> 8) % (2 * F16_MAX + 1) - F16_MAX
        return f16_bits(lo) | f16_bits(hi) << 16
    if s == BF16X2:
        if q & 1:
            return 0
        lo, hi = (BF16_MAX if r & 1 else -BF16_MAX), (BF16_MAX if r & 2 else -BF16_MAX)
        return bf16_bits(lo) | bf16_bits(hi) << 16
    if s == F32 or s >= V4RED:
        return f32_bits(float(r % (2 * F32_MAX + 1) - F32_MAX))
    return r


def init(seed, t, s):
    r = rand(seed, t, 300 + s, 0)
    if s in (INC, DEC):
        return r % (operand(seed, t, s, 0) + 1)
    if s == CAS64:
        return 0xFFFFFF00 + (r & 0x7F)
    if s in (F64, F64 + 1):
        u = f64_bits(float(rand(seed, t, 300 + F64, 0) % 2001 - 1000))
        return u & M32 if s == F64 else u >> 32
    if s == F16X2:
        return f16_bits(r % 7 - 3) | f16_bits((r >> 8) % 7 - 3) << 16
    if s == BF16X2:
        return 0
    if s == F32 or s >= V4RED:
        return f32_bits(float(r % 2001 - 1000))
    return r


def _s32(x):
    return x - (1 << 32) if x & 0x80000000 else x


def finals(seed, t):
    """F[s][n]: slot s after contributions q = 0 .. n-1 (EXCH: 0, it has no order-free final)."""
    X = [[operand(seed, t, s, q) for q in range(MAX_N)] for s in range(SLOTS)]
    v = [init(seed, t, s) for s in range(SLOTS)]
    F = np.zeros((SLOTS, MAX_N + 1), np.uint32)
    for n in range(MAX_N + 1):
        F[:, n] = v
        if n == MAX_N:
            break
        q = n
        v[ADD] = (v[ADD] + 1) & M32
        v[INC] = 0 if v[INC] >= X[INC][q] else v[INC] + 1
        v[DEC] = X[DEC][q] if v[DEC] == 0 or v[DEC] > X[DEC][q] else v[DEC] - 1
        v[EXCH] = 0
        v[CAS32] = (v[CAS32] + 1) & M32
        c = ((v[CAS64 + 1] << 32 | v[CAS64]) + 1) & ((1 << 64) - 1)
        v[CAS64], v[CAS64 + 1] = c & M32, c >> 32
        v[AND] &= X[AND][q]
        v[OR] |= X[OR][q]
        v[XOR] ^= X[XOR][q]
        v[MIN_S] = min(v[MIN_S], X[MIN_S][q], key=_s32)
        v[MAX_S] = max(v[MAX_S], X[MAX_S][q], key=_s32)
        v[MIN_U] = min(v[MIN_U], X[MIN_U][q])
        v[MAX_U] = max(v[MAX_U], X[MAX_U][q])
        a = ((v[ADD64 + 1] << 32 | v[ADD64]) + (X[ADD64 + 1][q] << 32 | X[ADD64][q])) & ((1 << 64) - 1)
        v[ADD64], v[ADD64 + 1] = a & M32, a >> 32
        v[F32] = f32_bits(bits_f32(v[F32]) + bits_f32(X[F32][q]))
        d = f64_bits(bits_f64(v[F64 + 1] << 32 | v[F64]) + bits_f64(X[F64 + 1][q] << 32 | X[F64][q]))
        v[F64], v[F64 + 1] = d & M32, d >> 32
        v[F16X2] = f16_bits(f16_int(v[F16X2]) + f16_int(X[F16X2][q])) | \
            f16_bits(f16_int(v[F16X2] >> 16) + f16_int(X[F16X2][q] >> 16)) << 16
        v[BF16X2] = bf16_bits(bf16_int(v[BF16X2]) + bf16_int(X[BF16X2][q])) | \
            bf16_bits(bf16_int(v[BF16X2] >> 16) + bf16_int(X[BF16X2][q] >> 16)) << 16
        for i in range(8):
            v[V4RED + i] = f32_bits(bits_f32(v[V4RED + i]) + bits_f32(X[V4RED + i][q]))
    return F, X


def word_slot(i):
    """Hot word i -> (slot it follows, row, lane)."""
    s = i // (ROWS * 32)
    base, span = s, 1
    for b, n in ((CAS64, 2), (ADD64, 2), (F64, 2), (V4RED, 4), (V4ATOM, 4)):
        if b <= s < b + n:
            base, span = b, n
    j = i - base * ROWS * 32
    return base + j % span, (j // span) // 32, (j // span) % 32


def n_of(G, row):
    warps = 4 * G
    return (warps - 1 - row) // ROWS + 1 if row < warps else 0


def return_fold(F, X, k, n):
    """Sum and xor over the 32 lanes of l2_mix of the multiset return op k's n contributions leave (exch: + final)."""
    s = RET_SLOTS[k]
    sm = x = 0
    for lane in range(32):
        ms = []
        if s == EXCH:
            ms = [l2_mix(int(X[EXCH][q]), lane) for q in range(n)]
        elif s == CAS64:
            ms = [l2_mix64(int(F[CAS64 + 1, i]) << 32 | int(F[CAS64, i]), lane) for i in range(n)]
        else:
            ms = [l2_mix(int(F[s, i]), lane) for i in range(n)]
        for m in ms:
            sm = (sm + m) & M32
            x ^= m
    return sm, x


def atom_expected(seed, t, G):
    """The hot block after one comparison of tile t on G CTAs (exch words: the initial value, though the device may
    hold any operand there), and the 12 expected combined folds: the grid's sums, then its xors."""
    F, X = finals(seed, t)
    hot = np.zeros(ATOM_HOT_WORDS, np.uint32)
    for i in range(ATOM_HOT_WORDS):
        s, row, _ = word_slot(i)
        hot[i] = F[s, n_of(G, row)]
    e0 = init(seed, t, EXCH)
    for i in range(ATOM_HOT_WORDS):
        if word_slot(i)[0] == EXCH:
            hot[i] = e0
    sums, xors = [0] * ATOM_RET, [0] * ATOM_RET
    folds = {}
    for k in range(ATOM_RET):
        for row in range(ROWS):
            n = n_of(G, row)
            if (k, n) not in folds:
                s, x = return_fold(F, X, k, n)
                if RET_SLOTS[k] == EXCH:           # {returns} + {final} = {init} + {operands}
                    for lane in range(32):
                        m = l2_mix(e0, lane)
                        s, x = (s + m) & M32, x ^ m
                folds[k, n] = (s, x)
            s, x = folds[k, n]
            sums[k] = (sums[k] + s) & M32
            xors[k] ^= x
    return hot, np.array(sums + xors, np.uint32)
