"""An independent restatement of the SFU self-test's host arithmetic (csrc/sfu_test_math.hpp), in numpy and Python:
the operand generator with its crafted classes, the guard (error bounds and specials), the fold and the majority.

The device's results cannot be computed here either -- NVIDIA publishes no bit-level model of MUFU -- so what this
module predicts is: the operand tables bit for bit, and whether a given result passes the guard.  Everything is
vectorised over threads (and over words for the majority), so a test can sweep many seeds."""
import math

import numpy as np

TILES, THREADS, REPS = 8, 128, 16
N = 16                                    # operand words per op per thread
F32, ROOT, F16 = 0, 1, 2
FORMATS = (F32, ROOT, F16)
NAMES = {F32: "f32", ROOT: "root", F16: "f16"}
SLOTS = {F32: 64, ROOT: 112, F16: 32}
WORDS = {F32: 80, ROOT: 112, F16: 32}
RESULTS = {F32: 5 * N, ROOT: 5 * N, F16: 4 * N}     # MUFU results per thread and repetition
T32, T64, T16 = 0, 1, 2
EX2, LG2, SIN, COS, TANH, RCP, RSQ, SQRT = range(8)
FN_NAMES = ["ex2", "lg2", "sin", "cos", "tanh", "rcp", "rsqrt", "sqrt"]
M32 = (1 << 32) - 1

TAIL = ["sub_in", "+0", "-0", "+inf", "-inf", "nan"]
# name, format, type, ftz, first slot, first word, functions, op-specific crafted classes, random (sign, elo, ehi)
OPS = [
    ("ex2", F32, T32, True, 0, 0, [EX2], ["exact", "edge_hi", "edge_lo", "overflow", "underflow"], (-1, -20, 6)),
    ("lg2", F32, T32, True, 16, 16, [LG2], ["exact", "edge_lo", "edge_hi", "near_one", "negative"], (0, -126, 127)),
    ("sincos", F32, T32, True, 32, 32, [SIN, COS], ["edge", "large", "huge", "small"], (-1, -20, 2)),
    ("tanh", F32, T32, False, 48, 64, [TANH], ["saturate", "small"], (-1, -20, 3)),
    ("rcp", ROOT, T32, True, 0, 0, [RCP], ["exact", "edge_lo", "edge_hi", "underflow"], (-1, -125, 124)),
    ("rsqrt", ROOT, T32, True, 16, 16, [RSQ], ["exact", "edge_lo", "edge_hi", "negative"], (0, -126, 127)),
    ("sqrt", ROOT, T32, True, 32, 32, [SQRT], ["exact", "edge_lo", "edge_hi", "negative"], (0, -126, 127)),
    ("rcp64", ROOT, T64, True, 48, 48, [RCP], ["exact", "edge_lo", "edge_hi", "underflow"], (-1, -1021, 1020)),
    ("rsqrt64", ROOT, T64, True, 80, 80, [RSQ], ["exact", "edge_lo", "edge_hi", "negative"], (0, -1022, 1023)),
    ("ex2h", F16, T16, False, 0, 0, [EX2], ["exact", "edge_hi", "edge_lo", "overflow", "subnormal", "underflow"],
     (-1, -10, 3)),
    ("tanhh", F16, T16, False, 16, 16, [TANH], ["saturate", "small"], (-1, -10, 2)),
]
OP_INDEX = {o[0]: i for i, o in enumerate(OPS)}
BIN = {T32: (32, 23, 127), T64: (64, 52, 1023), T16: (16, 10, 15)}   # width, stored mantissa bits, bias


def classes(op):
    return OPS[op][7] + TAIL


def values(op):
    return 2 * N if OPS[op][2] == T16 else N


# ---- hashing (compute_test_math.hpp's ct_mix family), vectorised ---------------------------------------------------
def mix(x):
    x = np.asarray(x, dtype=np.uint64) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7FEB352D)) & np.uint64(M32)
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846CA68B)) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    return x


def chash(key, i):
    return mix((np.uint64(key) + mix(i)) & np.uint64(M32))


def uniform(h, lo, hi):
    return lo + ((np.asarray(h, dtype=np.uint64) * np.uint64(hi - lo + 1)) >> np.uint64(32)).astype(np.int64)


def stream_key(seed, op, tile):
    return int(mix((seed ^ ((((tile * 16 + op) + 1) * 0x27D4EB2F) & M32)) & M32))


# ---- bits ---------------------------------------------------------------------------------------------------------------
def make(t, s, e, m):
    """sign * 1.m * 2^e (normal), on arrays"""
    W, M, B = BIN[t]
    s = np.asarray(s, dtype=np.uint64)
    e = (np.asarray(e, dtype=np.int64) + B).astype(np.uint64)
    m = np.asarray(m, dtype=np.uint64)
    return (s & np.uint64(1)) << np.uint64(W - 1) | e << np.uint64(M) | (m & np.uint64((1 << M) - 1))


def bits_of(t, x):
    """The bits of a Python number the type holds exactly."""
    if t == T64:
        return int(np.float64(x).view(np.uint64))
    if t == T32:
        return int(np.float32(x).view(np.uint32))
    return int(np.float16(x).view(np.uint16))


def value(t, bits):
    """float64 values of an array of bits."""
    b = np.asarray(bits, dtype=np.uint64)
    if t == T64:
        return b.view(np.float64).copy()
    if t == T32:
        return b.astype(np.uint32).view(np.float32).astype(np.float64)
    return b.astype(np.uint16).view(np.float16).astype(np.float64)


def is_subnormal(t, bits):
    W, M, _ = BIN[t]
    b = np.asarray(bits, dtype=np.uint64)
    return ((b >> np.uint64(M)) & np.uint64((1 << (W - 1 - M)) - 1) == 0) & (b & np.uint64((1 << M) - 1) != 0)


def min_normal(t):
    return 2.0 ** (1 - BIN[t][2])


def max_finite(t):
    _, M, B = BIN[t]
    return (2.0 - 2.0 ** -M) * 2.0 ** B


# ---- the generator --------------------------------------------------------------------------------------------------------
def operands(seed, op, tile):
    """[THREADS][values(op)] operand bits of op for one tile."""
    name, _, T, _, _, _, _, head, (rsign, elo, ehi) = OPS[op]
    W, M, B = BIN[T]
    nv = values(op)
    key = stream_key(seed, op, tile)
    t = np.arange(THREADS, dtype=np.int64)[:, None]
    v = np.arange(nv, dtype=np.int64)[None, :]
    d = [chash(key, ((t * 64 + v) * 4 + j).astype(np.uint64)) for j in range(4)]
    d0, d1, d2, d3 = d
    m = (d2 << np.uint64(32)) | d0
    rs = d3 >> np.uint64(31)
    c = (v - t) % nv
    out = make(T, rs if rsign < 0 else np.full_like(rs, rsign), uniform(d1, elo, ehi), m)
    EMAX, EMIN = B, 1 - B

    def put(cls, val):
        nonlocal out
        out = np.where(c == cls, np.broadcast_to(np.asarray(val, dtype=np.uint64), out.shape), out)

    def ints(k):
        return np.vectorize(lambda q: bits_of(T, int(q)), otypes=[np.uint64])(k)

    nh = len(head)
    sign_bit = np.uint64(1 << (W - 1))
    inf = np.uint64(((2 * B + 1) << M))
    put(nh + 0, (rs << np.uint64(W - 1)) | (m & np.uint64((1 << M) - 1)) | np.uint64(1))
    put(nh + 1, 0)
    put(nh + 2, sign_bit)
    put(nh + 3, inf)
    put(nh + 4, inf | sign_bit)
    put(nh + 5, inf | np.uint64(1 << (M - 1)))
    low6, low8 = d0 & np.uint64(63), d0 & np.uint64(255)
    if name == "ex2":
        put(0, ints(uniform(d1, -125, 127)))
        put(1, np.uint64(0x42FFFFFF) - low6)
        put(2, np.uint64(0xC2FBFD00) - low6)
        put(3, ints(128 + (d0 % np.uint64(64)).astype(np.int64)))
        put(4, ints(-(130 + (d0 % np.uint64(100)).astype(np.int64))))
    elif name == "lg2":
        put(0, make(T, 0, uniform(d1, EMIN, EMAX), 0))
        put(1, make(T, 0, EMIN, m))
        put(2, make(T, 0, EMAX, m))
        put(3, make(T, 0, 0, d0 & np.uint64(0xFF)))
        put(4, make(T, 1, uniform(d1, EMIN, EMAX), m))
    elif name == "sincos":
        put(0, (rs << np.uint64(31)) | (np.uint64(0x41490FDA) - low8))
        put(1, make(T, rs, uniform(d1, 4, 20), m))
        put(2, make(T, rs, uniform(d1, 60, EMAX), m))
        put(3, make(T, rs, uniform(d1, EMIN, -60), m))
    elif name in ("tanh", "tanhh"):
        h16 = T == T16
        put(0, make(T, rs, uniform(d1, 3 if h16 else 4, 15 if h16 else 20), m))
        put(1, make(T, rs, uniform(d1, EMIN, -5 if h16 else -20), m))
    elif name in ("rcp", "rcp64", "rsqrt", "sqrt", "rsqrt64"):
        rcp = name.startswith("rcp")
        s = rs if rcp else np.zeros_like(rs)
        put(0, make(T, s, 2 * uniform(d1, -(EMAX // 2), EMAX // 2), 0))
        put(1, make(T, s, EMIN, m))
        put(2, make(T, s, EMAX - 2, m & np.uint64(((1 << M) - 1) >> 1)) if rcp else make(T, s, EMAX, m))
        put(3, make(T, s, EMAX, m) if rcp else make(T, 1, uniform(d1, EMIN, EMAX), m))
    else:  # ex2h
        low3 = d0 & np.uint64(7)
        put(0, ints(uniform(d1, -14, 15)))
        put(1, np.uint64(0x4BFF) - low3)
        put(2, np.uint64(0xCAFF) - low3)
        put(3, np.uint64(0x4C00) + (d0 & np.uint64(0x1FF)))
        put(4, ints(-(15 + (d0 % np.uint64(9)).astype(np.int64))))
        put(5, ints(-(25 + (d0 % np.uint64(40)).astype(np.int64))))
    return out


def thread_words(seed, fmt, tile):
    """[THREADS][SLOTS[fmt]] operand words, as the kernel's registers hold them."""
    w = np.zeros((THREADS, SLOTS[fmt]), dtype=np.uint64)
    for op, o in enumerate(OPS):
        if o[1] != fmt:
            continue
        x, T, s0 = operands(seed, op, tile), o[2], o[4]
        if T == T32:
            w[:, s0:s0 + N] = x
        elif T == T64:
            w[:, s0:s0 + 2 * N:2] = x & np.uint64(M32)
            w[:, s0 + 1:s0 + 2 * N:2] = x >> np.uint64(32)
        else:
            w[:, s0:s0 + N] = x[:, 0::2] | (x[:, 1::2] << np.uint64(16))
    return w.astype(np.uint32)


def table(seed, fmt, tile):
    """The operand table of one tile: [slot][thread] words."""
    return np.ascontiguousarray(thread_words(seed, fmt, tile).T)


def tables(seed, fmt):
    return np.stack([table(seed, fmt, t) for t in range(TILES)])


# ---- results: operand / result pairs per function ----------------------------------------------------------------------
def pairs(fmt, ops, words):
    """Yield (op, fn, x bits, r bits) for every result of one or more threads: ops [..., SLOTS] and words [..., WORDS]
    (uint32 arrays)."""
    ops = np.asarray(ops, dtype=np.uint64)
    words = np.asarray(words, dtype=np.uint64)
    for op, (_, f, T, _, s0, w0, fns, _, _) in enumerate(OPS):
        if f != fmt:
            continue
        if T == T32:
            x = ops[..., s0:s0 + N]
            for k, fn in enumerate(fns):
                yield op, fn, x, words[..., w0 + k * N:w0 + (k + 1) * N]
        elif T == T64:
            x = ops[..., s0:s0 + 2 * N:2] | (ops[..., s0 + 1:s0 + 2 * N:2] << np.uint64(32))
            r = words[..., w0:w0 + 2 * N:2] | (words[..., w0 + 1:w0 + 2 * N:2] << np.uint64(32))
            yield op, fns[0], x, r
        else:
            def halves(a, base):
                h = a[..., base:base + N]
                return np.stack([h & np.uint64(0xFFFF), h >> np.uint64(16)], axis=-1).reshape(h.shape[:-1] + (2 * N,))
            yield op, fns[0], halves(ops, s0), halves(words, w0)


# ---- the guard ---------------------------------------------------------------------------------------------------------------
def bound(fn, t):
    if t == T16:
        return 2.0 ** -7
    if t == T64:
        return 2.0 ** -16
    if fn in (SIN, COS):
        return 2.0 ** -16
    if fn == TANH:
        return 2.0 ** -8
    return 2.0 ** -18


ABSOLUTE = (LG2, SIN, COS)


def abs_bound(fn, t, e):
    """lg2: 2^-18 up to |e| = 16, 2^-22 |e| beyond (2^-18 is half an f32 ulp of a result in [64, 128)); sin, cos: 2^-16"""
    B = bound(fn, t)
    return B * np.maximum(1.0, np.abs(e) / 16) if fn == LG2 else B
TRIG_GUARDED = 4 * math.pi


def exact(fn, x):
    with np.errstate(all="ignore"):
        return {EX2: np.exp2, LG2: np.log2, SIN: np.sin, COS: np.cos, TANH: np.tanh,
                RCP: lambda v: 1.0 / v, RSQ: lambda v: 1.0 / np.sqrt(v), SQRT: np.sqrt}[fn](x)


def guard(fn, t, ftz, xb, rb):
    """(pass, error) arrays for results rb of fn on operands xb (bits).  The rule, restated from the design:
    exact NaN -> NaN; exact +-inf -> that infinity; +-0 or +-inf input with an exact zero -> that signed zero;
    lg2 / sin / cos: |r - e| <= bound (sin, cos only for |x| <= 4 pi); the others: |r - e| <= bound |e|, where a bound
    reaching past the largest finite value admits the infinity and one reaching below the smallest normal checks only
    the class (+-0 for .ftz forms, +-0 or a same-signed subnormal otherwise)."""
    x = value(t, xb)
    if ftz:
        x = np.where(is_subnormal(t, xb), np.copysign(0.0, x), x)
    e, r = exact(fn, x), value(t, rb)
    B = bound(fn, t)
    ok = np.zeros(np.shape(e), dtype=bool)
    err = np.zeros(np.shape(e))
    done = np.zeros(np.shape(e), dtype=bool)

    def settle(mask, val):
        nonlocal ok, done
        m = mask & ~done
        ok = np.where(m, val, ok)
        done |= m

    with np.errstate(all="ignore"):
        settle(np.isnan(e), np.isnan(r))
        settle(np.isnan(r), False)
        settle(np.isinf(e), r == e)
        settle((e == 0) & ((x == 0) | np.isinf(x)), (r == 0) & (np.signbit(r) == np.signbit(e)))
        if fn in ABSOLUTE:
            if fn in (SIN, COS):
                settle(np.abs(x) > TRIG_GUARDED, True)
            settle(np.isinf(r), False)
            d = np.abs(r - e)
            err = np.where(done, 0.0, d)
            settle(np.ones_like(done), d <= abs_bound(fn, t, e))
            return ok, err
        ae, ar = np.abs(e), np.abs(r)
        mn = min_normal(t)
        settle((ae * (1 - B) < mn) & (ar < mn), (r == 0) | ((not ftz) & (np.signbit(r) == np.signbit(e))))
        settle(np.signbit(r) != np.signbit(e), False)
        settle(np.isinf(r), ae * (1 + B) > max_finite(t))
        if ftz:
            settle(ar < mn, False)
        d = np.abs(ar - ae) / ae
        err = np.where(done, 0.0, d)
        settle(np.ones_like(done), d <= B)
    return ok, err


def guard_words(fmt, ops, words):
    """Failures of the guard over [..., SLOTS] operands and [..., WORDS] results, and the worst error per (op, fn)."""
    bad, worst = 0, {}
    for op, fn, x, r in pairs(fmt, ops, words):
        ok, err = guard(fn, OPS[op][2], OPS[op][3], x, r)
        bad += int((~ok).sum())
        k = (OPS[op][0], FN_NAMES[fn])
        worst[k] = max(worst.get(k, 0.0), float(np.where(ok, err, 0).max()))
    return bad, worst


# ---- fold and majority -------------------------------------------------------------------------------------------------------
def fold(words):
    """sum_j (2j + 1) w_j mod 2^32 over the last axis."""
    w = np.asarray(words, dtype=np.uint64)
    weights = 2 * np.arange(w.shape[-1], dtype=np.uint64) + 1
    return ((w * weights).sum(axis=-1) & np.uint64(M32)).astype(np.uint32)


def majority(dumps):
    """dumps [cta][...]: (value, has) where has marks words held by strictly more than half of the CTAs."""
    d = np.asarray(dumps)
    med = np.sort(d, axis=0)[d.shape[0] // 2]
    cnt = (d == med[None]).sum(axis=0)
    return med, 2 * cnt > d.shape[0]
