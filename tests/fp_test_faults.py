"""Fault models of the FP32 / FP64 self-test: FMA units that break IEEE 754 in one way, on top of the exact oracle
(tests/fp_test_oracle.py).  Each rule returns what such a unit computes for fma(x, a, b); a rule the self-test covers
changes the check value of at least one thread in every tile.  tests/test_fp_test_edges_cpu.py writes the table of
DESIGN.md §4.7 from these counts, and tests/test_gpu_fp_test_edges.py runs the kernel on checks built with each rule.

    ties_away, ties_toward_zero   a tie rounds away from / toward zero instead of to even
    truncate                      every inexact result rounds toward zero
    no_sticky                     only the round bit is seen: a set round bit is taken for a tie
    ftz                           a subnormal result is flushed to a zero of its sign
    daz_add                       a subnormal b is read as a zero of its sign
    daz_mul                       a subnormal x or a is read as a zero of its sign
    unfused                       RN(RN(x * a) + b)
    zero_sign                     an exact zero result takes the other sign (+0 <-> -0)
    subnormal_double_round        a result below 2^EMIN is rounded to M + 1 bits first, then to the subnormal grid
"""
import fp_test_oracle as ft

RULES = ("ties_away", "ties_toward_zero", "truncate", "no_sticky", "ftz", "daz_add", "daz_mul", "unfused", "zero_sign",
         "subnormal_double_round")
# every tile of the product's tables must catch these; subnormal_double_round has no crafted class and is only counted
REQUIRED = RULES[:-1]
ROUNDING = ("ties_away", "ties_toward_zero", "truncate", "no_sticky")


def is_subnormal(fmt, v):
    W, M = ft.BIN[fmt][:2]
    return 0 < v & ((1 << (W - 1)) - 1) < 1 << M


def flush(fmt, v):
    """v, or a zero of its sign if v is subnormal."""
    return v & (1 << (ft.BIN[fmt][0] - 1)) if is_subnormal(fmt, v) else v


def exact(fmt, x, a, b):
    """The exact x * a + b as (sign, N, E), N >= 0, or None if an operand is infinite."""
    sx, nx, ex = ft.decode(fmt, x)
    sa, na, ea = ft.decode(fmt, a)
    sb, nb, eb = ft.decode(fmt, b)
    if nx is None or na is None or nb is None:
        return None
    sp, p, ep = sx ^ sa, nx * na, ex + ea
    e = min(ep, eb)
    v = (-1) ** sp * (p << (ep - e)) + (-1) ** sb * (nb << (eb - e))
    return (1 if v < 0 else 0), abs(v), e


def wrong_fma(fmt, x, a, b, rule, rn=None):
    """What a unit with fault `rule` returns for fma(x, a, b).  rn: the correct result, if the caller has it.  Where the
    wrong unit's result is NaN (an unfused unit's inf - inf), the canonical quiet NaN stands for it: any NaN differs
    from the correct result, which never is one."""
    rn = ft.fma(fmt, x, a, b) if rn is None else rn
    try:
        return _wrong(fmt, x, a, b, rule, rn)
    except ft.NaNResult:
        return ft.inf(fmt, 0) | 1 << (ft.BIN[fmt][1] - 1)


def _wrong(fmt, x, a, b, rule, rn):
    if rule in ROUNDING:
        return ft.fma(fmt, x, a, b, mode=rule)
    if rule == "ftz":
        return flush(fmt, rn)
    if rule == "daz_add":
        return ft.fma(fmt, x, a, flush(fmt, b)) if is_subnormal(fmt, b) else rn
    if rule == "daz_mul":
        if not (is_subnormal(fmt, x) or is_subnormal(fmt, a)):
            return rn
        return ft.fma(fmt, flush(fmt, x), flush(fmt, a), b)
    if rule == "unfused":
        return ft.fma(fmt, ft.mul(fmt, x, a), ft.make(fmt, 0, 0, 0), b)
    ex = exact(fmt, x, a, b)
    if rule == "zero_sign":
        return rn ^ 1 << (ft.BIN[fmt][0] - 1) if ex is not None and ex[1] == 0 else rn
    if rule == "subnormal_double_round":
        W, M, BIAS, EMIN = ft.BIN[fmt][:4]
        if ex is None or ex[1] == 0:
            return rn
        s, N, E = ex
        lead = E + N.bit_length() - 1
        if lead >= EMIN or E >= lead - M:     # normal, or already M + 1 bits: one rounding either way
            return rn
        n1, _, _ = ft.round_shift(N, lead - M - E)
        return ft.round_rne(fmt, s, n1, lead - M)[0]
    raise ValueError(rule)


def words(fmt, x, a, b, rule=None):
    """The thread's result words (as fp_test_oracle.fma_words) from a unit with fault `rule` (None: IEEE 754)."""
    out = []
    for k in range(ft.NAB):
        for i in range(ft.NX):
            r = ft.fma(fmt, x[i], a[k], b[k])
            if rule is not None:
                r = wrong_fma(fmt, x[i], a[k], b[k], rule, r)
            out += [r] if fmt == ft.FP32 else [r & ft.M32, r >> 32]
    return out


def wrong_checks(fmt, ops, rules):
    """{rule: [check value of each thread]} for one tile's operands ops[thread] = (x, a, b)."""
    out = {r: [] for r in rules}
    for x, a, b in ops:
        rn = [ft.fma(fmt, x[i], a[k], b[k]) for k in range(ft.NAB) for i in range(ft.NX)]
        for rule in rules:
            ws = []
            for j, r in enumerate(rn):
                k, i = divmod(j, ft.NX)
                w = wrong_fma(fmt, x[i], a[k], b[k], rule, r)
                ws += [w] if fmt == ft.FP32 else [w & ft.M32, w >> 32]
            out[rule].append(ft.fold(ws))
    return out
