"""Oracle for the on-demand FP32 / FP64 self-test (pure Python integers; test infrastructure only).

The specification of the arithmetic the CUDA kernel (k8s-device-plugin_b200/csrc/fp_selftest.cuh) and its host side
(csrc/fp_test_math.hpp) must reproduce bit for bit.  Every floating-point value is handled as sign, integer significand
and exponent, and every FMA result is the exact value x * a + b rounded once to nearest-even in binary32 / binary64,
subnormals and signed zeros included.  No floating-point arithmetic (and no C fma) is involved.

    mix, hash       : as tests/compute_test_oracle.py; key = mix(seed ^ uint32((((fmt * 16 + tile) * 4 + op) + 1) * 0x85EBCA77))
    draw(t, s, j)   : hash(key, (t * 64 + s) * 4 + j);  r64 = draw(j=0) << 32 | draw(j=1)
    random value    : sign = r64 >> 63, mantissa = r64 & (2^M - 1), exponent uniform(draw(j=2)) in the slot's range
    FMA thread      : x_0..7 (x_0 odd significand, x_1 even and not a power of two, x_2 exponent -8), (a_k, b_k) k < 16,
                      b's exponent = a's +- spread; crafted class c at k = (2c + t) % 16 (see fp_test_math.hpp)
    results         : r_j = RN(x_i * a_k + b_k), j = 8k + i; FP64 results are two words (low, high)
    DMMA            : integers in [-max, max]; warp tile % 4: A_s row 0 and B_s (k != n) all -max; set c of warp w sums
                      A_s B_{(s + c) % 4} over s; result * 2^(ea + eb), +0 for 0; fragments per the PTX ISA m16n8k16 .f64
    check value     : sum_j (2j + 1) * word_j  mod 2^32 over the thread's words
"""
import numpy as np

THREADS, TILES, REPS = 128, 8, 16
FP32, FP64, DMMA = 0, 1, 2
FORMATS = (FP32, FP64, DMMA)
NAMES = {FP32: "fp32", FP64: "fp64", DMMA: "dmma"}
NX, NAB = 8, 16
RESULTS = NX * NAB
WORDS = {FP32: RESULTS, FP64: 2 * RESULTS, DMMA: 32}
SLOTS = {FP32: NX + 2 * NAB, FP64: NX + 2 * NAB, DMMA: 48}
M32 = 0xFFFFFFFF

# width, stored mantissa bits M, bias, EMIN, x exponent range, a exponent range, b spread
BIN = {FP32: (32, 23, 127, -126, 16, 40, 28), FP64: (64, 52, 1023, -1022, 16, 300, 60)}
CANCEL_BITS = {FP32: 20, FP64: 40}
SUBNORMAL_X_EXP = -8
CLASSES = ("tie_away", "tie_toward", "cancel", "subnormal", "zero_pos", "zero_neg", "sticky", "subnormal_operand")
CLASS_X = (0, 1, 0, 2, 1, 3, 0, 3)

DMMA_STEPS, DMMA_SETS, DMMA_K = 4, 4, 64
DMMA_MAX = 11863283
DMMA_SCALE_EXP = 480


def mix(x: int) -> int:
    x &= M32
    x ^= x >> 16
    x = (x * 0x7FEB352D) & M32
    x ^= x >> 15
    x = (x * 0x846CA68B) & M32
    x ^= x >> 16
    return x


def hash_(key: int, i: int) -> int:
    return mix((key + mix(i)) & M32)


def uniform(h: int, lo: int, hi: int) -> int:
    return lo + ((h * (hi - lo + 1)) >> 32)


def stream_key(seed: int, fmt: int, tile: int, op: int) -> int:
    return mix(seed ^ (((((fmt * 16 + tile) * 4 + op) + 1) * 0x85EBCA77) & M32))


# ---- binary formats on integers -----------------------------------------------------------------------------------------
def make(fmt, sign, e, mant):
    W, M, BIAS = BIN[fmt][:3]
    return sign << (W - 1) | (e + BIAS) << M | (mant & ((1 << M) - 1))


class NaNResult(ValueError):
    """An operation whose IEEE 754 result is NaN (or a NaN operand): its payload is unspecified, so no test uses one."""


def decode(fmt, bits):
    """(sign, N, E): the value is (-1)^sign * N * 2^E with N a non-negative integer; N is None for an infinity."""
    W, M, BIAS, EMIN = BIN[fmt][:4]
    sign = bits >> (W - 1) & 1
    be = bits >> M & ((1 << (W - M - 1)) - 1)
    mant = bits & ((1 << M) - 1)
    if be == 0:
        return sign, mant, EMIN - M
    if be == (1 << (W - M - 1)) - 1:
        if mant:
            raise NaNResult("NaN operand 0x%x" % bits)
        return sign, None, 0
    return sign, mant | 1 << M, be - BIAS - M


def inf(fmt, sign):
    W, M = BIN[fmt][:2]
    return sign << (W - 1) | ((1 << (W - M - 1)) - 1) << M


def exponent(fmt, bits):
    W, M, BIAS = BIN[fmt][:3]
    return (bits >> M & ((1 << (W - M - 1)) - 1)) - BIAS


# Rounding rules: IEEE 754's round to nearest, ties to even ("rne"), and wrong ones for the fault models of
# tests/fp_test_faults.py: ties away from zero, ties toward zero, truncation, and "no_sticky", which sees only the round
# bit (a set round bit is taken for a tie).
def round_shift(N, sh, mode="rne"):
    """(N >> sh rounded by `mode`, tie, rounded_up) for sh >= 1."""
    mant, rem, half = N >> sh, N & ((1 << sh) - 1), 1 << (sh - 1)
    tie = rem == half
    if mode == "rne":
        up = rem > half or (tie and mant & 1 == 1)
    elif mode == "ties_away":
        up = rem >= half
    elif mode == "ties_toward_zero":
        up = rem > half
    elif mode == "truncate":
        up = False
    elif mode == "no_sticky":
        up = rem & half != 0 and mant & 1 == 1
    else:
        raise ValueError(mode)
    return mant + up, tie, up


def round_rne(fmt, sign, N, E, ties_away=False, mode="rne"):
    """Bits of (-1)^sign N 2^E (N > 0) rounded to nearest-even, and how: (bits, tie, rounded_up).  A value whose
    rounded magnitude exceeds the largest finite one is an infinity (a truncating rule gives the largest finite value).
    ties_away, or another `mode` of round_shift, rounds by a wrong rule instead (for tests that need one)."""
    W, M, BIAS, EMIN = BIN[fmt][:4]
    mode = "ties_away" if ties_away else mode
    lead = E + N.bit_length() - 1
    q = max(lead - M, EMIN - M)           # exponent of the result's last significand bit
    tie = up = False
    if E >= q:
        mant = N << (E - q)
    else:
        mant, tie, up = round_shift(N, q - E, mode)
    if mant == 1 << (M + 1):
        mant >>= 1
        q += 1
    if q + M > BIAS:                       # beyond the largest finite binade
        if mode == "truncate":
            return inf(fmt, sign) - 1, tie, up
        return inf(fmt, sign), tie, up
    if mant < 1 << M:                      # subnormal (q == EMIN - M)
        return sign << (W - 1) | mant, tie, up
    return sign << (W - 1) | (q + M + BIAS) << M | (mant - (1 << M)), tie, up


def _infinite(fmt, sp, np_, sb, nb, factor_zero):
    """x * a + b when x, a or b is infinite (np_ None: the product is), or NaNResult."""
    if np_ is None and factor_zero:
        raise NaNResult("0 * inf")
    if np_ is None and nb is None and sp != sb:
        raise NaNResult("inf - inf")
    return inf(fmt, sp if np_ is None else sb)


def fma(fmt, x, a, b, detail=False, ties_away=False, mode="rne"):
    """RN(x * a + b) on bits, exactly as IEEE 754 defines it (round_rne's wrong rules on request)."""
    sx, nx, ex = decode(fmt, x)
    sa, na, ea = decode(fmt, a)
    sb, nb, eb = decode(fmt, b)
    sp = sx ^ sa
    if nx is None or na is None or nb is None:
        np_ = None if nx is None or na is None else nx * na
        r = (_infinite(fmt, sp, np_, sb, nb, nx == 0 or na == 0), False, False)
        return r if detail else r[0]
    np_, ep = nx * na, ex + ea
    e = min(ep, eb)
    v = (-1) ** sp * (np_ << (ep - e)) + (-1) ** sb * (nb << (eb - e))
    W = BIN[fmt][0]
    if v == 0:
        zero_sign = (sp & sb) if (np_ == 0 and nb == 0) else 0
        r = (zero_sign << (W - 1), False, False)
    else:
        r = round_rne(fmt, 1 if v < 0 else 0, abs(v), e, ties_away, mode)
    return r if detail else r[0]


def mul(fmt, x, a):
    """RN(x * a)."""
    sx, nx, ex = decode(fmt, x)
    sa, na, ea = decode(fmt, a)
    if nx is None or na is None:
        return _infinite(fmt, sx ^ sa, None, 0, 0, nx == 0 or na == 0)
    if nx * na == 0:
        return (sx ^ sa) << (BIN[fmt][0] - 1)
    return round_rne(fmt, sx ^ sa, nx * na, ex + ea)[0]


# ---- FMA operands -------------------------------------------------------------------------------------------------------
def fma_thread(seed, fmt, tile, t):
    """(x[8], a[16], b[16]) as bits."""
    W, M, BIAS, EMIN, XE, AE, BS = BIN[fmt]
    key = stream_key(seed, fmt, tile, 0)
    mm = (1 << M) - 1

    def draw(s, j):
        return hash_(key, (t * 64 + s) * 4 + j)

    def r64(s):
        return draw(s, 0) << 32 | draw(s, 1)

    x = []
    for i in range(NX):
        r = r64(i)
        mant, e = r & mm, uniform(draw(i, 2), -XE, XE)
        if i == 0:
            mant |= 1
        if i == 1:
            mant = (mant & ~1) | 2
        if i == 2:
            e = SUBNORMAL_X_EXP
        x.append(make(fmt, r >> 63, e, mant))
    a, b = [], []
    for k in range(NAB):
        ra, rb = r64(NX + k), r64(NX + NAB + k)
        ea = uniform(draw(NX + k, 2), -AE, AE)
        eb = ea + uniform(draw(NX + NAB + k, 2), -BS, BS)
        a.append(make(fmt, ra >> 63, ea, ra & mm))
        b.append(make(fmt, rb >> 63, eb, rb & mm))
    sbit = 1 << (W - 1)
    for c in range(len(CLASSES)):
        k = (2 * c + t) % NAB
        xv = x[CLASS_X[c]]
        sa, sb = a[k] >> (W - 1) & 1, b[k] >> (W - 1) & 1
        j = exponent(fmt, a[k])
        pow2 = make(fmt, sa, j, 0)
        q = exponent(fmt, xv) + j
        sp = (xv >> (W - 1) & 1) ^ sa
        name = CLASSES[c]
        if name in ("tie_away", "tie_toward"):
            a[k], b[k] = pow2, make(fmt, sp, q - M - 1, 0)
        elif name == "cancel":
            a[k] |= 1
            b[k] = mul(fmt, xv, a[k]) ^ sbit
        elif name == "subnormal":
            a[k] = make(fmt, sa, EMIN + 3, a[k])
            b[k] = make(fmt, sp, EMIN - 1, b[k] & ((1 << (M - 5)) - 1))
        elif name == "zero_pos":
            a[k] = pow2
            b[k] = mul(fmt, xv, pow2) ^ sbit
        elif name == "zero_neg":
            a[k], b[k] = ((xv >> (W - 1) & 1) ^ 1) << (W - 1), sbit
        elif name == "sticky":
            a[k], b[k] = pow2, make(fmt, sb, q + M + 1, b[k] & ~1)
        else:  # subnormal_operand: a subnormal with its top stored bit set, b normal in [2^EMIN, 2^(EMIN + 4))
            a[k] = make(fmt, sa, EMIN - 1, a[k] | 1 << (M - 1))
            b[k] = make(fmt, sb, uniform(draw(NX + NAB + k, 3), EMIN, EMIN + 3), b[k])
    return x, a, b


def wrong_fma(fmt, x, a, b, rule):
    """What a unit that breaks IEEE 754 in one way would return: 'ties_away' rounds ties away from zero, 'ftz' flushes
    subnormal results to zero, 'unfused' rounds the product before the add."""
    W, M = BIN[fmt][:2]
    if rule == "ties_away":
        return fma(fmt, x, a, b, ties_away=True)
    if rule == "unfused":
        return fma(fmt, mul(fmt, x, a), make(fmt, 0, 0, 0), b)
    r = fma(fmt, x, a, b)
    return r & (1 << (W - 1)) if r & ((1 << (W - 1)) - 1) < 1 << M else r


def fma_words(fmt, x, a, b, rule=None):
    out = []
    for k in range(NAB):
        for i in range(NX):
            r = fma(fmt, x[i], a[k], b[k]) if rule is None else wrong_fma(fmt, x[i], a[k], b[k], rule)
            out += [r] if fmt == FP32 else [r & M32, r >> 32]
    return out


def classify(fmt, x, a, b):
    """The crafted classes fma(x, a, b) belongs to, judged from the exact value."""
    W, M, BIAS, EMIN = BIN[fmt][:4]
    r, tie, up = fma(fmt, x, a, b, detail=True)
    sx, nx, ex = decode(fmt, x)
    sa, na, ea = decode(fmt, a)
    sb, nb, eb = decode(fmt, b)
    p = nx * na
    out = set()
    if tie:
        out.add("tie_away" if up else "tie_toward")
    mag = r & ((1 << (W - 1)) - 1)
    if p and r == 0:
        out.add("zero_pos")
    if r == 1 << (W - 1):
        out.add("zero_neg")
    if 0 < mag < 1 << M:
        out.add("subnormal")
    e = min(ex + ea, eb)
    v = abs((-1) ** (sx ^ sa) * (p << (ex + ea - e)) + (-1) ** sb * (nb << (eb - e)))
    big = max(p << (ex + ea - e), nb << (eb - e))
    if v and big >= v << CANCEL_BITS[fmt]:
        out.add("cancel")
    # b dominates: x * a lies wholly below b's last significand bit, and still moves the rounded result off b
    if p and (nb << (eb - e)) >= (p << (ex + ea - e)) << M and r != b:
        out.add("sticky")
    # a multiplicand is subnormal, and reading it as a signed zero would change the result
    for v, other, first in ((x, a, True), (a, x, False)):
        if v & ((1 << (W - 1)) - 1) and exponent(fmt, v) == EMIN - 1:
            z = v & (1 << (W - 1))
            if fma(fmt, *((z, other) if first else (other, z)), b) != r:
                out.add("subnormal_operand")
    return out


# ---- DMMA -----------------------------------------------------------------------------------------------------------------
def dmma_scale_exp(seed, tile, op):
    return uniform(hash_(stream_key(seed, DMMA, tile, 2), op), -DMMA_SCALE_EXP, DMMA_SCALE_EXP)


def dmma_matrix(seed, tile, op, w, s):
    """A_s (16 x 16, M x K) for op 0, B_s (16 x 8, K x N) for op 1, as int64."""
    rows, cols = (16, 16) if op == 0 else (16, 8)
    key = stream_key(seed, DMMA, tile, op)
    v = np.empty((rows, cols), dtype=np.int64)
    for r in range(rows):
        for c in range(cols):
            if w == tile % 4 and (r == 0 if op == 0 else r != c):
                v[r, c] = -DMMA_MAX
            else:
                h = hash_(key, ((w * DMMA_STEPS + s) * 16 + r) * cols + c)
                v[r, c] = -DMMA_MAX + ((h * (2 * DMMA_MAX + 1)) >> 32)
    return v


def dmma_exact(seed, tile, w):
    """[set] 16 x 8 exact int64 results of warp w, and the step products [set][step] (for the K-chain model)."""
    A = [dmma_matrix(seed, tile, 0, w, s) for s in range(DMMA_STEPS)]
    B = [dmma_matrix(seed, tile, 1, w, s) for s in range(DMMA_STEPS)]
    steps = [[A[s] @ B[(s + c) % DMMA_STEPS] for s in range(DMMA_STEPS)] for c in range(DMMA_SETS)]
    return [sum(st) for st in steps], steps, A, B


def a_frag(l, i):
    return l // 4 + 8 * (i % 2), l % 4 + 4 * (i // 2)


def b_frag(l, i):
    return l % 4 + 4 * i, l // 4


def d_frag(l, i):
    return l // 4 + 8 * (i // 2), 2 * (l % 4) + i % 2


def f64_bits(n: int, e: int) -> int:
    """Bits of the binary64 value n * 2^e (exact by construction; +0 for 0)."""
    if n == 0:
        return 0
    return round_rne(FP64, 1 if n < 0 else 0, abs(n), e)[0]


# ---- tiles ----------------------------------------------------------------------------------------------------------------
def fold(words) -> int:
    return sum((2 * j + 1) * w for j, w in enumerate(words)) & M32


def tile(seed, fmt, t):
    """(table [slot][thread] as Python ints (bits), words [thread][W], checks [thread], operands per thread)."""
    table = [[0] * THREADS for _ in range(SLOTS[fmt])]
    words, ops = [], []
    if fmt != DMMA:
        for th in range(THREADS):
            x, a, b = fma_thread(seed, fmt, t, th)
            for s, v in enumerate(x + a + b):
                table[s][th] = v
            ops.append((x, a, b))
            words.append(fma_words(fmt, x, a, b))
    else:
        ea, eb = dmma_scale_exp(seed, t, 0), dmma_scale_exp(seed, t, 1)
        for w in range(4):
            D, _, A, B = dmma_exact(seed, t, w)
            for l in range(32):
                th = w * 32 + l
                for s in range(DMMA_STEPS):
                    for i in range(8):
                        table[s * 8 + i][th] = f64_bits(int(A[s][a_frag(l, i)]), ea)
                    for i in range(4):
                        table[32 + s * 4 + i][th] = f64_bits(int(B[s][b_frag(l, i)]), eb)
                ws = []
                for c in range(DMMA_SETS):
                    for i in range(4):
                        r = f64_bits(int(D[c][d_frag(l, i)]), ea + eb)
                        ws += [r & M32, r >> 32]
                words.append(ws)
    return table, words, [fold(w) for w in words], ops
