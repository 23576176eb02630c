"""Independent restatement of the half-precision and conversion self-test's host arithmetic (csrc/half_test_math.hpp),
written from the PTX ISA's text and IEEE 754: the operand generator with its crafted classes, every op under test, the
result-word order and the fold.  Values are exact `fractions.Fraction`s and every result is rounded once, by searching
the representable neighbours of the exact value; no float type of the host is used.  It shares no arithmetic with the
C++; tests/test_half_test_cpu.py holds the two against each other, and tests/test_gpu_half_test.py holds the kernel's
DUMP against this file.

`fault` arguments select a fault model of a unit (tests/test_half_test_cpu.py); the default is the correct unit."""
from fractions import Fraction
from functools import lru_cache

import int_test_oracle as it

M32 = 0xFFFFFFFF
THREADS, TILES, REPS = 128, 8, 16
F16, BF16, CVT = 0, 1, 2
SETS = (12, 12, 9)
CRAFTED = (6, 6, 8)
SET_SLOTS = (6, 6, 13)
SET_WORDS = (12, 9, 58)
SLOTS = tuple(a * b for a, b in zip(SETS, SET_SLOTS))
WORDS = tuple(a * b for a, b in zip(SETS, SET_WORDS))
F16_WORDS = ("fma", "fma_relu", "fma_sat", "fma_ftz", "add", "sub", "mul", "min", "max", "min_nan", "max_nan",
             "min_xorsign")
BF16_WORDS = ("fma", "fma_relu", "add", "sub", "mul", "min", "max", "min_nan", "max_nan")
MODES = ("rn", "rz", "rm", "rp")
CVT_WORDS = (("f16x2_rn", "f16x2_rz", "f16x2_relu", "f16x2_satf", "bf16x2_rn", "bf16x2_rz", "bf16x2_relu",
              "bf16x2_satf", "e4m3_f32", "e5m2_f32", "e4m3_f16", "e5m2_f16", "f16_e4m3", "f16_e5m2", "tf32", "f16_rm",
              "f16_rp", "bf16_rm", "bf16_rp")
             + tuple("s32_" + m for m in MODES) + tuple("u32_" + m for m in MODES)
             + tuple("s64_%s_%s" % (m, h) for m in MODES for h in ("lo", "hi"))
             + tuple("i2f_s32_" + m for m in MODES) + tuple("i2f_u64_" + m for m in MODES)
             + tuple("i2f_s64_%s_%s" % (m, h) for m in MODES for h in ("lo", "hi"))
             + tuple("f32_f64_" + m for m in MODES) + ("frnd_f32", "frnd_f64_lo", "frnd_f64_hi"))
WORD_NAMES = (F16_WORDS, BF16_WORDS, CVT_WORDS)
X, Y, P, Q, F, H, E4, E5, I, DLO, DHI, LLO, LHI = range(13)

# formats: (exponent bits, fraction bits, has infinity)
FMT_F16, FMT_BF16, FMT_F32, FMT_F64 = (5, 10, True), (8, 7, True), (8, 23, True), (11, 52, True)
FMT_TF32, FMT_E4M3, FMT_E5M2 = (8, 10, True), (4, 3, False), (5, 2, True)
CANON = 0x7FFF
NAN, INF = "nan", "inf"


# ---- exact values --------------------------------------------------------------------------------------------------
def decode(bits, fmt):
    """(sign, value): value is a Fraction (magnitude), INF or NAN."""
    eb, mb, has_inf = fmt
    sign = bits >> (eb + mb) & 1
    e = bits >> mb & ((1 << eb) - 1)
    m = bits & ((1 << mb) - 1)
    if e == (1 << eb) - 1:
        if has_inf:
            return sign, INF if m == 0 else NAN
        if m == (1 << mb) - 1:
            return sign, NAN
    bias = (1 << (eb - 1)) - 1
    if e == 0:
        return sign, Fraction(m, 1) * Fraction(2) ** (1 - bias - mb)
    return sign, Fraction((1 << mb) + m) * Fraction(2) ** (e - bias - mb)


def max_finite(fmt):
    eb, mb, has_inf = fmt
    top = (1 << eb) - 1
    return ((top - 1) << mb | ((1 << mb) - 1)) if has_inf else (top << mb | ((1 << mb) - 2))


def log2_floor(v):
    """The e with 2^e <= v < 2^(e + 1), for a positive Fraction."""
    e = v.numerator.bit_length() - v.denominator.bit_length()
    if Fraction(2) ** e > v:
        e -= 1
    if Fraction(2) ** (e + 1) <= v:
        e += 1
    return e


def encode_exact(v, fmt):
    """Bits of the non-negative representable value v (assumed representable, below the overflow bound)."""
    eb, mb, _ = fmt
    bias = (1 << (eb - 1)) - 1
    if v == 0:
        return 0
    e = log2_floor(v)
    if v < Fraction(2) ** (1 - bias):                    # subnormal
        n = v / Fraction(2) ** (1 - bias - mb)
        assert n.denominator == 1
        return int(n)
    n = v / Fraction(2) ** (e - mb)
    assert n.denominator == 1 and (1 << mb) <= n < (2 << mb), (v, fmt)
    return (e + bias) << mb | (int(n) - (1 << mb))


def round_value(sign, v, fmt, mode, satfinite=False):
    """The bits of (-1)^sign * v (v >= 0 a Fraction) rounded once to fmt.  mode: 'rn' (ties to even), 'rz', 'rm',
    'rp'.  The quantum is that of the exponent v has with an unbounded exponent range above and the least exponent
    below; a result above the largest finite value is infinity (rn, and rm / rp away from zero) or that value."""
    eb, mb, has_inf = fmt
    sbit = sign << (eb + mb)
    if v == 0:
        return sbit
    bias = (1 << (eb - 1)) - 1
    e = max(log2_floor(v), 1 - bias)
    quantum = Fraction(2) ** (e - mb)
    lo = (v / quantum).numerator // (v / quantum).denominator
    rest = v / quantum - lo
    away = {"rn": rest > Fraction(1, 2) or (rest == Fraction(1, 2) and lo % 2 == 1),
            "rz": False, "rm": rest > 0 and sign == 1, "rp": rest > 0 and sign == 0}[mode]
    r = (lo + (1 if away else 0)) * quantum
    if r == 0:
        return sbit
    _, top = decode(max_finite(fmt), fmt)
    if r > top:
        toward_max = satfinite or mode == "rz" or (mode == "rm" and sign == 0) or (mode == "rp" and sign == 1)
        return sbit | (max_finite(fmt) if toward_max or not has_inf else ((1 << eb) - 1) << mb)
    return sbit | encode_exact(r, fmt)


def signed(sign, v):
    return -v if sign else v


# ---- the 16-bit arithmetic -------------------------------------------------------------------------------------------
def fma_lane(a, b, c, fmt, mod=None, fault=None):
    """fma.rn{.relu,.sat,.ftz} of one lane."""
    sbit = 1 << (fmt[0] + fmt[1])
    one = ((1 << (fmt[0] - 1)) - 1) << fmt[1]

    def flush(h):
        return h & sbit if (h >> fmt[1]) & ((1 << fmt[0]) - 1) == 0 else h
    if mod == "ftz" and fault != "ftz_ignored":
        a, b, c = flush(a), flush(b), flush(c)
    if mod is None and fault == "ftz_everywhere":
        a, b, c = flush(a), flush(b), flush(c)
    (sa, va), (sb, vb), (sc, vc) = decode(a, fmt), decode(b, fmt), decode(c, fmt)
    nan = False
    if NAN in (va, vb, vc):
        nan = True
    elif INF in (va, vb):
        ps = sa ^ sb
        if va == 0 or vb == 0 or (vc == INF and sc != ps):
            nan = True
        else:
            r = sbit * ps | (((1 << fmt[0]) - 1) << fmt[1])
    elif vc == INF:
        r = c
    else:
        exact = signed(sa ^ sb, va * vb) + signed(sc, vc)
        if exact == 0:
            zsign = 1 if (va * vb == 0 and vc == 0 and (sa ^ sb) and sc) else 0
            r = zsign * sbit
        elif fault == "double_round":           # through an FP32 FMA first: two roundings
            f32 = round_value(1 if exact < 0 else 0, abs(exact), FMT_F32, "rn")
            s2, v2 = decode(f32, FMT_F32)
            r = sbit * s2 | (((1 << fmt[0]) - 1) << fmt[1]) if v2 == INF else round_value(s2, v2, fmt, "rn")
        else:
            r = round_value(1 if exact < 0 else 0, abs(exact), fmt, "rz" if fault == "rz" else "rn")
            if fault == "sticky_lost":          # the bits below the guard bit dropped before rounding
                q = abs(exact)
                e = max(log2_floor(q), 2 - (1 << (fmt[0] - 1)))
                g =Fraction(2) ** (e - fmt[1] - 1)
                t = (q / g).numerator // (q / g).denominator * g
                r = round_value(1 if exact < 0 else 0, t, fmt, "rn")
    if mod == "relu" and fault != "relu_ignored":
        return CANON if nan else (0 if r & sbit else r)
    if mod == "sat" and fault != "sat_ignored":
        if nan or r & sbit:
            return 0
        return one if r > one else r
    if mod == "ftz":
        return flush(r)
    return CANON if nan else r


def lanes(fn, *words):
    return fn(*[w & 0xFFFF for w in words]) | fn(*[w >> 16 for w in words]) << 16


def key(h, fmt):
    sbit = 1 << (fmt[0] + fmt[1])
    return -(h & (sbit - 1)) - 1 if h & sbit else h


def minmax_lane(a, b, fmt, is_max, nan_mode):
    na, nb = decode(a, fmt)[1] == NAN, decode(b, fmt)[1] == NAN
    if na and nb:
        return CANON
    if na or nb:
        return CANON if nan_mode else (b if na else a)
    return (a if key(a, fmt) > key(b, fmt) else b) if is_max else (a if key(a, fmt) < key(b, fmt) else b)


def xorsign_lane(a, b, fmt):
    sbit = 1 << (fmt[0] + fmt[1])
    return min(a & (sbit - 1), b & (sbit - 1)) | ((a ^ b) & sbit)


def half_words(fmt, s, fault=None):
    """Result words of one set (slots a, b, c, x, y, z) of F16 or BF16."""
    a, b, c, x, y, z = s
    ft = FMT_F16 if fmt == F16 else FMT_BF16
    one = ((1 << (ft[0] - 1)) - 1) << ft[1]
    neg0 = 1 << (ft[0] + ft[1])
    fl = None if fault in ("lane_swap",) else fault
    out = {
        "fma": lanes(lambda p, q, r: fma_lane(p, q, r, ft, None, fl), a, b, c),
        "fma_relu": lanes(lambda p, q, r: fma_lane(p, q, r, ft, "relu", fl), x, y, z),
        "fma_sat": lanes(lambda p, q, r: fma_lane(p, q, r, ft, "sat", fl), x, y, z),
        "fma_ftz": lanes(lambda p, q, r: fma_lane(p, q, r, ft, "ftz", fl), a, b, c),
        "add": lanes(lambda p, q: fma_lane(p, one, q, ft, None, fl), a, b),
        "sub": lanes(lambda p, q: fma_lane(p, one, q ^ neg0, ft, None, fl), a, b),
        "mul": lanes(lambda p, q: fma_lane(p, q, neg0, ft, None, fl), a, b),
        "min": lanes(lambda p, q: minmax_lane(p, q, ft, False, False), x, y),
        "max": lanes(lambda p, q: minmax_lane(p, q, ft, True, False), x, y),
        "min_nan": lanes(lambda p, q: minmax_lane(p, q, ft, False, True), x, y),
        "max_nan": lanes(lambda p, q: minmax_lane(p, q, ft, True, True), x, y),
        "min_xorsign": lanes(lambda p, q: xorsign_lane(p, q, ft), a, b),
    }
    words = [out[n] for n in WORD_NAMES[fmt]]
    if fault == "lane_swap":
        words[0] = (words[0] >> 16 | words[0] << 16) & M32
    return words


# ---- conversions -------------------------------------------------------------------------------------------------------
def cvt_float(bits, src, dst, mode, satfinite=False, relu=False, fault=None):
    sign, v = decode(bits, src)
    if v == NAN:
        return 0x7F if not dst[2] else CANON
    if v == INF:
        sat = satfinite and fault != "satfinite_ignored"
        r = sign << (dst[0] + dst[1]) | (max_finite(dst) if sat or not dst[2] else ((1 << dst[0]) - 1) << dst[1])
    else:
        r = round_value(sign, v, dst, "rz" if fault == "rz" else mode, satfinite and fault != "satfinite_ignored")
    if relu and fault != "relu_ignored" and r >> (dst[0] + dst[1]):
        r = 0
    return r


def round_to_int(sign, v, mode):
    fl = v.numerator // v.denominator
    rest = v - fl
    up = {"rn": rest > Fraction(1, 2) or (rest == Fraction(1, 2) and fl % 2 == 1), "rz": False,
          "rm": rest > 0 and sign == 1, "rp": rest > 0 and sign == 0}[mode]
    return fl + (1 if up else 0)


def f2i(bits, src, mode, width, is_signed, fault=None):
    sign, v = decode(bits, src)
    if v == NAN:
        return 0 if fault != "nan_not_zero" else (1 << (width - 1) if is_signed else 0)
    lo, hi = (-(1 << (width - 1)), (1 << (width - 1)) - 1) if is_signed else (0, (1 << width) - 1)
    n = (1 << 200) if v == INF else round_to_int(sign, v, "rz" if fault == "f2i_trunc" else mode)
    n = -n if sign else n
    if fault != "f2i_wraps":
        n = max(lo, min(hi, n))
    return n & ((1 << width) - 1)


def i2f(value, width, is_signed, dst, mode, fault=None):
    value &= (1 << width) - 1
    if is_signed and value >> (width - 1):
        value -= 1 << width
    return round_value(1 if value < 0 else 0, Fraction(abs(value)), dst, "rn" if fault == "i2f_rn" else mode)


def frnd(bits, fmt, mode, fault=None):
    sign, v = decode(bits, fmt)
    n = round_to_int(sign, v, "rz" if fault == "frnd_trunc" else mode)
    return round_value(sign, Fraction(n), fmt, "rn")


def cvt_words(s, fault=None):
    x, y, p, q, f, h, e4, e5, i, dlo, dhi, llo, lhi = s
    d, L = dhi << 32 | dlo, lhi << 32 | llo

    def pk(hi, lo):
        return hi << 16 | lo
    fl = fault

    def c(bits, dst, mode, sat=False, relu=False):
        return cvt_float(bits, FMT_F32, dst, mode, sat, relu, fl)
    out = [pk(c(x, FMT_F16, "rn"), c(y, FMT_F16, "rn")), pk(c(x, FMT_F16, "rz"), c(y, FMT_F16, "rz")),
           pk(c(p, FMT_F16, "rn", relu=True), c(q, FMT_F16, "rn", relu=True)),
           pk(c(p, FMT_F16, "rn", sat=True), c(q, FMT_F16, "rn", sat=True)),
           pk(c(x, FMT_BF16, "rn"), c(y, FMT_BF16, "rn")), pk(c(x, FMT_BF16, "rz"), c(y, FMT_BF16, "rz")),
           pk(c(p, FMT_BF16, "rn", relu=True), c(q, FMT_BF16, "rn", relu=True)),
           pk(c(p, FMT_BF16, "rn", sat=True), c(q, FMT_BF16, "rn", sat=True))]
    e4f = (c(p, FMT_E4M3, "rn", sat=True), c(q, FMT_E4M3, "rn", sat=True))
    e5f = (c(x, FMT_E5M2, "rn", sat=True), c(y, FMT_E5M2, "rn", sat=True))
    e4h = tuple(cvt_float(w, FMT_F16, FMT_E4M3, "rn", True, False, fl) for w in (h >> 16, h & 0xFFFF))
    e5h = tuple(cvt_float(w, FMT_F16, FMT_E5M2, "rn", True, False, fl) for w in (h >> 16, h & 0xFFFF))
    for hi, lo in (e4f, e5f, e4h, e5h):
        out.append(lo << 8 | hi if fault == "fp8_order" else hi << 8 | lo)

    def widen(b, src):
        sign, v = decode(b, src)
        return sign << 15 | 0x7C00 if v == INF else round_value(sign, v, FMT_F16, "rn")
    out.append(pk(widen(e4 >> 8 & 0xFF, FMT_E4M3), widen(e4 & 0xFF, FMT_E4M3)))
    out.append(pk(widen(e5 >> 8 & 0xFF, FMT_E5M2), widen(e5 & 0xFF, FMT_E5M2)))
    t = c(x, FMT_TF32, "rn")
    out.append((t >> 18 & 1) << 31 | (t & 0x3FFFF) << 13)
    out += [c(x, FMT_F16, "rm"), c(x, FMT_F16, "rp"), c(x, FMT_BF16, "rm"), c(x, FMT_BF16, "rp")]
    out += [f2i(f, FMT_F32, m, 32, True, fl) for m in MODES]
    out += [f2i(f, FMT_F32, m, 32, False, fl) for m in MODES]
    for m in MODES:
        r = f2i(d, FMT_F64, m, 64, True, fl)
        out += [r & M32, r >> 32]
    out += [i2f(i, 32, True, FMT_F32, m, fl) for m in MODES]
    out += [i2f(L, 64, False, FMT_F32, m, fl) for m in MODES]
    for m in MODES:
        r = i2f(L, 64, True, FMT_F64, m, fl)
        out += [r & M32, r >> 32]
    out += [cvt_float(d, FMT_F64, FMT_F32, m, fault=fl) for m in MODES]
    out.append(frnd(x, FMT_F32, "rn", fl))
    r = frnd(d, FMT_F64, "rm", fl)
    out += [r & M32, r >> 32]
    return out


# ---- generator (compute_test_math.hpp's hash) -----------------------------------------------------------------------
def stream_key(seed, fmt, tile):
    return it.mix(seed ^ ((fmt * 16 + tile + 1) * 0x27D4EB2F & M32))


def h32(seed, fmt, tile, t, slot, k):
    return it.hash32(stream_key(seed, fmt, tile), ((t * 256 + slot) * 4 + k) & M32)


def rand_f16(h):
    return (h & 0x83FF) | ((h >> 10) % 29 + 1) << 10


def rand_bf16(h):
    return (h & 0x807F) | ((h >> 7) % 41 + 107) << 7


def rand_f32(h, h2, lo, span):
    return (h & 0x807FFFFF) | (lo + h2 % span) << 23


def rand_e4m3(h):
    return h & 0xFE if h & 0x7F == 0x7F else h & 0xFF


def rand_e5m2(h):
    return (h & 0xFF) - 4 if h & 0x7F > 0x7C else h & 0xFF


# the crafted classes (the same constants as half_test_math.hpp, with what each is for)
ABC_F16 = [(0x1000, 0x3C00, 0x3C00), (0x1000, 0x3C00, 0x3C01), (0x3C01, 0x3C01, 0xBC02), (0x0E55, 0x2E66, 0x8001),
           (0x0155, 0x4A00, 0x0003), (0x7800, 0x4000, 0x3C00), (0xF800, 0x4000, 0x3C00), (0x8000, 0x4500, 0x8000),
           (0x0000, 0xC500, 0x0000), (0x1001, 0x3C01, 0x3C00), (0x3C01, 0x4200, 0x8001), (0x0400, 0x3800, 0x0000)]
XYZ_F16 = [(0x4000, 0x4200, 0x3800), (0xC000, 0x4200, 0x3C00), (0x8000, 0x3C00, 0x8000), (0x7E01, 0x4000, 0x3C00),
           (0xFE10, 0x7D00, 0x0000), (0x7C00, 0x4000, 0xBC00), (0x7C00, 0x3C00, 0xFC00), (0x0000, 0x8000, 0x0000),
           (0x3800, 0x3A00, 0x3000), (0x3C00, 0x3C00, 0x0000), (0xFC00, 0x4000, 0x3C00), (0x4500, 0xC500, 0x4E40)]
ABC_BF16 = [(0x3B80, 0x3F80, 0x3F80), (0x3B80, 0x3F80, 0x3F81), (0x3F81, 0x3F81, 0xBF82), (0x1CD5, 0x21B3, 0x8001),
            (0x0055, 0x4140, 0x0003), (0x7F00, 0x4000, 0x3F80), (0xFF00, 0x4040, 0x3F80), (0x8000, 0x40A0, 0x8000),
            (0x0000, 0xC0A0, 0x0000), (0x3B81, 0x3F81, 0x3F80), (0x3F81, 0x4040, 0xAB80), (0x0080, 0x3F00, 0x0000)]
XYZ_BF16 = [(0x4000, 0x4040, 0x3F00), (0xC000, 0x4040, 0x3F80), (0x8000, 0x3F80, 0x8000), (0x7FC1, 0x4000, 0x3F80),
            (0xFFC2, 0x7F81, 0x0000), (0x7F80, 0x4000, 0xBF80), (0x7F80, 0x3F80, 0xFF80), (0x0000, 0x8000, 0x0000),
            (0x3F00, 0x3F40, 0x3E00), (0x3F80, 0x3F80, 0x0000), (0xFF80, 0x4000, 0x3F80), (0x40A0, 0xC0A0, 0x41C8)]
HALF_CLASSES = ("tie_down", "tie_up", "cancel", "subnormal_result", "subnormal_multiplicand", "overflow_pos",
                "overflow_neg", "neg_zero", "pos_zero", "sticky", "double_round", "ftz_result")
CVT_XY = [0x3F801000, 0x3F803000, 0x3F808000, 0x3F818000, 0x477FF000, 0xC7800000, 0x35A12345, 0x33000000, 0x33000001,
          0xBF800001, 0x47700000, 0x47600000, 0x37000000, 0x36FFFFFF, 0xC0200000, 0x3FC00000]
CVT_PQ = [0x7F800000, 0xFF800000, 0x7FC00001, 0x43E00000, 0x43F00000, 0x43E80000, 0x3B000000, 0x3A800000, 0x3A800001,
          0x3A7FFFFF, 0xBFC00000, 0x80000000, 0x477FF000, 0x7F7FFFFF, 0xC3E80000, 0x3E2AAAAB]
CVT_H = [0x7C00, 0xFC00, 0x5F00, 0x5F80, 0x5F40, 0x7B00, 0x7B80, 0x1800, 0x1400, 0x1401, 0x13FF, 0x0100, 0x0080,
         0x0081, 0xBE00, 0x8000]
CVT_E4 = [0x01, 0x81, 0x7E, 0xFE, 0x08, 0x07, 0x00, 0x80, 0x38, 0x3F, 0x77, 0xC5, 0x02, 0x40, 0x0F, 0x70]
CVT_E5 = [0x01, 0x81, 0x7B, 0xFB, 0x7C, 0xFC, 0x04, 0x03, 0x00, 0x80, 0x3C, 0x3F, 0x02, 0xC1, 0x5A, 0x43]
CVT_F = [0x4F000000, 0xCF000000, 0x4F800000, 0xBF000000, 0x3F000000, 0x3FC00000, 0x40200000, 0x7FC00000]
CVT_I = [0x01000001, 0xFEFFFFFD, 0x80000000, 0x7FFFFFFF, 0x01000003, 0x00000000, 0xFFFFFFFF, 0x00FFFFFF]
CVT_D = [0x43E0000000000000, 0xC3E0000000000000, 0x47F0000000000001, 0xC7F0000000000001, 0x3738000000000001,
         0x3FF0000010000000, 0xC004000000000000, 0x8000000000000001]
CVT_L = [0x0020000000000001, 0x8000010000000001, 0xFFFFFFFFFFFFFFFF, 0x8000000000000000, 0x7FFFFFFFFFFFFFFF,
         0x0000000001000001, 0xFFDFFFFFFFFFFFFF, 0x0020000000000003]


def thread_operands(seed, fmt, tile, t):
    """[set][k] operand words of thread t."""
    ss = SET_SLOTS[fmt]
    sets = []
    for s in range(SETS[fmt]):
        crafted = s < CRAFTED[fmt]

        def hh(k, i):
            return h32(seed, fmt, tile, t, s * ss + k, i)
        if fmt != CVT:
            abc, xyz = (ABC_F16, XYZ_F16) if fmt == F16 else (ABC_BF16, XYZ_BF16)
            rnd = rand_f16 if fmt == F16 else rand_bf16
            row = []
            for k in range(6):
                w = 0
                for L in range(2):
                    c = (2 * s + L + t) % 12
                    lane = (abc[c][k] if k < 3 else xyz[c][k - 3]) if crafted else rnd(hh(k, L))
                    w |= lane << 16 * L
                row.append(w)
            sets.append(row)
            continue
        l0, l1, c = (2 * s + t) % 16, (2 * s + 1 + t) % 16, (s + t) % 8
        if crafted:
            sets.append([CVT_XY[l0], CVT_XY[l1], CVT_PQ[l0], CVT_PQ[l1], CVT_F[c], CVT_H[l0] << 16 | CVT_H[l1],
                         CVT_E4[l0] << 8 | CVT_E4[l1], CVT_E5[l0] << 8 | CVT_E5[l1], CVT_I[c], CVT_D[c] & M32,
                         CVT_D[c] >> 32, CVT_L[c] & M32, CVT_L[c] >> 32])
        else:
            dh = hh(DHI, 0)
            sets.append([rand_f32(hh(X, 0), hh(X, 1), 97, 61), rand_f32(hh(Y, 0), hh(Y, 1), 97, 61),
                         rand_f32(hh(P, 0), hh(P, 1), 110, 30), rand_f32(hh(Q, 0), hh(Q, 1), 110, 30),
                         rand_f32(hh(F, 0), hh(F, 1), 123, 36), rand_f16(hh(H, 0)) << 16 | rand_f16(hh(H, 1)),
                         rand_e4m3(hh(E4, 0)) << 8 | rand_e4m3(hh(E4, 1)),
                         rand_e5m2(hh(E5, 0)) << 8 | rand_e5m2(hh(E5, 1)), hh(I, 0), hh(DLO, 0),
                         (dh & 0x800FFFFF) | (1023 - 160 + hh(DHI, 1) % 321) << 20, hh(LLO, 0),
                         hh(LHI, 0) >> (hh(LHI, 1) % 32)])
    return sets


@lru_cache(maxsize=None)
def tile_operands(seed, fmt, tile):
    return tuple(tuple(tuple(s) for s in thread_operands(seed, fmt, tile, t)) for t in range(THREADS))


def table(seed, fmt, tile):
    """The table a launch reads: [slot][thread] words, flattened."""
    ops = tile_operands(seed, fmt, tile)
    ss = SET_SLOTS[fmt]
    return [ops[t][slot // ss][slot % ss] for slot in range(SLOTS[fmt]) for t in range(THREADS)]


def thread_words(fmt, sets, fault=None):
    out = []
    for s in sets:
        out += cvt_words(s, fault) if fmt == CVT else half_words(fmt, s, fault)
    return out


@lru_cache(maxsize=None)
def _tile_words(seed, fmt, tile, fault):
    return tuple(tuple(thread_words(fmt, s, fault)) for s in tile_operands(seed, fmt, tile))


def tile_words(seed, fmt, tile, fault=None):
    return [list(w) for w in _tile_words(seed, fmt, tile, fault)]


def fold(words):
    return it.fold(words)


def tile_checks(seed, fmt, tile, fault=None):
    return [fold(w) for w in _tile_words(seed, fmt, tile, fault)]
