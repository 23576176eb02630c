"""Inputs for testing the FP32 / FP64 self-test (fp_selftest.cuh) beyond what its generator makes.
tests/test_fp_test_edges_cpu.py checks what each one reaches; tests/test_gpu_fp_test_edges.py runs them.

- Crafted FMA tables (one table of TILES tiles per format), written from the documented layout: slot s of thread t of
  a tile is table[s][t], slots x_0..7, a_0..15, b_0..15.  Thread t holds eight crafted triples (x_i, a_i, b_i) and
  their mirrors (x_i, -a_i, -b_i) in pair 8 + i (but for exact_zero's, see fma_tiles); every one of the 128
  combinations x_i * a_k + b_k is compared, so the
  other 120 combinations reach infinities, overflow and underflow too.  The families (FAMILIES):
  - subnormal x, subnormal a or both, with x * a normal, subnormal, or below half the smallest subnormal (a nonzero
    value that underflows keeps its sign: -0), and x * a at exactly and just above that half;
  - results at 2^EMIN: the largest subnormal rounding up to the smallest normal, ties on the subnormal grid both ways;
  - the top of the range: the largest finite value, MAX + ulp/2 (rounds to infinity), MAX + ulp/2 - tiny (rounds to
    MAX), and x * a beyond the range with b bringing the exact sum back (finite only if the unit is fused);
  - b = +-inf;
  - a carry through the whole product width into a new binade, and ties decided by the product's last bit.
  No combination may give NaN, whose payload IEEE 754 leaves open: fma_table refuses such a table.
- Crafted DMMA tiles, written through the oracle's fragment maps: every product +max^2 (the 2^53 bound) at three
  scale corners, a late +-1 addend at every K position of every step, Walsh rows that cancel to exactly 0, and a tile
  of -0 products.
- Edge seeds: the first seed, ascending from 0, with a DMMA tile at each scale corner (found by a numpy scan).
"""
import functools
import random

import numpy as np

import fp_test_oracle as ft

# ---- encoding -----------------------------------------------------------------------------------------------------------


def val(fmt, n, e):
    """Bits of n * 2^e, which must be representable exactly (n may be negative; 0 gives +0)."""
    if n == 0:
        return 0
    r = ft.round_rne(fmt, 1 if n < 0 else 0, abs(n), e)[0]
    _, N, E = ft.decode(fmt, r)
    m = min(E, e)
    assert N is not None and N << (E - m) == abs(n) << (e - m), ("not exact", n, e)
    return r


def neg(fmt, v):
    return v ^ 1 << (ft.BIN[fmt][0] - 1)


def emax(fmt):
    return ft.BIN[fmt][2]


def max_finite(fmt, sign=0):
    return ft.inf(fmt, sign) - 1


# ---- FMA families -------------------------------------------------------------------------------------------------------
# Each family draws one triple (x, a, b) from a random.Random.


def _sig(fmt, rng, odd=False):
    """A random M + 1-bit significand in [2^M, 2^(M + 1)), odd on request."""
    M = ft.BIN[fmt][1]
    s = 1 << M | rng.getrandbits(M)
    if odd:
        s |= 1
    return s


def _sub(fmt, rng, top=False):
    """A random subnormal magnitude as (N, E): N in [1, 2^M), top: its top stored bit set."""
    M, EMIN = ft.BIN[fmt][1], ft.BIN[fmt][3]
    n = rng.getrandbits(M) or 1
    if top:
        n |= 1 << (M - 1)
    return n, EMIN - M


def _sgn(rng):
    return -1 if rng.getrandbits(1) else 1


def sub_x_normal_product(fmt, rng):
    """x subnormal, |a| in [2^(M + 2), 2^(M + 10)): x * a normal; b a random value of about its size, or a zero."""
    M, EMIN = ft.BIN[fmt][1], ft.BIN[fmt][3]
    n, e = _sub(fmt, rng, top=True)
    x = val(fmt, _sgn(rng) * n, e)
    a = val(fmt, _sgn(rng) * _sig(fmt, rng), 2 + rng.randrange(8))
    b = val(fmt, _sgn(rng) * _sig(fmt, rng), EMIN + rng.randrange(2 * M + 4) - M) if rng.getrandbits(1) else 0
    return x, a, b


def sub_a_subnormal_product(fmt, rng):
    """a subnormal, |x| in [1/2, 1): x * a is subnormal and needs rounding; b a zero of either sign."""
    M = ft.BIN[fmt][1]
    n, e = _sub(fmt, rng)
    a = val(fmt, _sgn(rng) * n, e)
    x = val(fmt, _sgn(rng) * _sig(fmt, rng, odd=True), -M - 1)
    return x, a, neg(fmt, 0) if rng.getrandbits(1) else 0


def sub_x_underflow(fmt, rng):
    """x subnormal, |a| < 2^-(M + 2): x * a is below half the smallest subnormal.  b is a zero of the other sign, so
    the result is the product's sign: a negative product gives -0."""
    M = ft.BIN[fmt][1]
    n, e = _sub(fmt, rng)
    sx, sa = _sgn(rng), _sgn(rng)
    x = val(fmt, sx * n, e)
    a = val(fmt, sa * _sig(fmt, rng), -2 * M - 3 - rng.randrange(20))
    return x, a, 0 if sx * sa < 0 else neg(fmt, 0)


def sub_both(fmt, rng):
    """x and a subnormal: x * a is far below the smallest subnormal; b the smallest subnormal or a zero."""
    nx, e = _sub(fmt, rng)
    na, _ = _sub(fmt, rng)
    x, a = val(fmt, _sgn(rng) * nx, e), val(fmt, _sgn(rng) * na, e)
    b = rng.choice([0, neg(fmt, 0), 1, neg(fmt, 1)])
    return x, a, b


def half_smallest_subnormal(fmt, rng):
    """x * a = exactly half the smallest subnormal (a tie: rounds to 0, the even neighbour), or just above it (rounds
    to the smallest subnormal).  x is subnormal (2^(EMIN - 1)); b is a zero."""
    M, EMIN = ft.BIN[fmt][1], ft.BIN[fmt][3]
    x = val(fmt, _sgn(rng), EMIN - 1)
    above = rng.getrandbits(1)
    a = val(fmt, _sgn(rng) * ((1 << M) + above), -2 * M)   # 2^-M, or 2^-M (1 + 2^-M)
    return x, a, rng.choice([0, neg(fmt, 0)])


def subnormal_rounds_to_normal(fmt, rng):
    """x = the largest subnormal, a = 1 + 2^-M: x * a = 2^EMIN (1 - 2^-2M), which rounds up to the smallest normal."""
    M, EMIN = ft.BIN[fmt][1], ft.BIN[fmt][3]
    x = val(fmt, _sgn(rng) * ((1 << M) - 1), EMIN - M)
    a = val(fmt, _sgn(rng) * ((1 << M) + 1), -M)
    return x, a, rng.choice([0, neg(fmt, 0)])


def subnormal_tie(fmt, rng):
    """b subnormal, x * a = half a subnormal ulp with b's sign: a tie on the subnormal grid, to even (up for an odd b,
    stays for an even one)."""
    M, EMIN = ft.BIN[fmt][1], ft.BIN[fmt][3]
    nb = rng.getrandbits(M) or 2
    sb = _sgn(rng)
    b = val(fmt, sb * nb, EMIN - M)
    ex = EMIN // 2
    sx = _sgn(rng)
    x = val(fmt, sx, ex)
    a = val(fmt, sx * sb, EMIN - M - 1 - ex)
    return x, a, b


def largest_finite(fmt, rng):
    """A result of exactly MAX: MAX / 2 * 2, or MAX + something below half its ulp."""
    M = ft.BIN[fmt][1]
    s = _sgn(rng)
    if rng.getrandbits(1):
        return val(fmt, s * ((1 << (M + 1)) - 1), emax(fmt) - M - 1), val(fmt, 1, 1), 0
    x = val(fmt, _sgn(rng) * _sig(fmt, rng), -M)
    a = val(fmt, _sgn(rng) * _sig(fmt, rng), emax(fmt) - 3 * M)      # |x * a| < 2^(EMAX - 2M + 2) << ulp(MAX) / 2
    return x, a, max_finite(fmt, 0 if s > 0 else 1)


def max_plus_half_ulp(fmt, rng):
    """b = MAX, x * a = ulp(MAX) / 2 with b's sign: a tie whose even neighbour is 2^(EMAX + 1): infinity."""
    M = ft.BIN[fmt][1]
    s = _sgn(rng)
    k = rng.randrange(-20, 20)
    return val(fmt, s, k), val(fmt, 1, emax(fmt) - M - 1 - k), max_finite(fmt, 0 if s > 0 else 1)


def max_plus_just_below_half_ulp(fmt, rng):
    """b = MAX, x * a = ulp(MAX) / 2 (1 - 2^-(M + 1)) with b's sign: rounds to MAX."""
    M = ft.BIN[fmt][1]
    s = _sgn(rng)
    k = rng.randrange(-20, 20)
    x = val(fmt, s * ((1 << (M + 1)) - 1), k - M)
    return x, val(fmt, 1, emax(fmt) - M - 2 - k), max_finite(fmt, 0 if s > 0 else 1)


def product_overflows_sum_does_not(fmt, rng):
    """|x| in [1, 1.25) 2^EMAX, |a| in [2, 2.5): x * a lies in [2, 3.125) 2^EMAX, beyond MAX; b has the other sign and
    |b| in [1.5, 2) 2^EMAX, so the exact sum is in (0, 1.625) 2^EMAX: finite.  A unit that rounds the product first
    returns infinity."""
    M = ft.BIN[fmt][1]
    s = _sgn(rng)
    x = val(fmt, s * (1 << M | rng.getrandbits(M - 2)), emax(fmt) - M)
    a = val(fmt, 1 << M | rng.getrandbits(M - 2), 1 - M)
    b = val(fmt, -s * (3 << (M - 1) | rng.getrandbits(M - 1)), emax(fmt) - M)
    return x, a, b


def infinite_b(fmt, rng):
    """b = +-inf, x and a random finite values: the result is b."""
    M = ft.BIN[fmt][1]
    x = val(fmt, _sgn(rng) * _sig(fmt, rng), rng.randrange(-20, 20) - M)
    a = val(fmt, _sgn(rng) * _sig(fmt, rng), rng.randrange(-20, 20) - M)
    return x, a, ft.inf(fmt, rng.getrandbits(1))


def carry_into_new_binade(fmt, rng):
    """x = a = 2 - 2^-M (all-ones significands): x * a = (2^(M+1) - 1)^2 units, and b = 2^(M+2) - 2 units makes the exact
    sum 2^(2M+2) - 1, all ones over the whole product width: rounding carries into the next binade."""
    M = ft.BIN[fmt][1]
    k = rng.randrange(-20, 20)
    s = _sgn(rng)
    ones = (1 << (M + 1)) - 1
    x = val(fmt, s * ones, k - M)
    a = val(fmt, _sgn(rng) * ones, -M)
    sp = s * (1 if ft.decode(fmt, a)[0] == 0 else -1)
    return x, a, val(fmt, sp * ((1 << (M + 2)) - 2), k - 2 * M)


def product_last_bit_tie(fmt, rng):
    """x, a with odd significands and a 2M + 2-bit product P; b cancels P's low M + 2 bits down to exactly half an ulp,
    plus d in {-1, 0, +1} units of P's last bit (2M + 1 bits below its leading one): d = 0 is a tie to even, d = +-1
    is decided by that last bit alone.  |b| <= 2^M + 1 units fits M + 1 bits."""
    M = ft.BIN[fmt][1]
    while True:
        nx, na = _sig(fmt, rng, odd=True), _sig(fmt, rng, odd=True)
        P = nx * na
        if P.bit_length() == 2 * M + 2:
            break
    nb = (1 << M) - (P & ((1 << (M + 1)) - 1)) + rng.choice([-1, 0, 1])
    k = rng.randrange(-20, 20)
    s = _sgn(rng)
    return val(fmt, s * nx, k - M), val(fmt, na, -M), val(fmt, s * nb, k - 2 * M)


def exact_zero(fmt, rng):
    """a = +-2^j (subnormal when j < EMIN), x * a in [2^EMIN, 2^(EMIN + 41)), b = -(x * a) exactly: +0 (and the
    mirror's too)."""
    M, EMIN = ft.BIN[fmt][1], ft.BIN[fmt][3]
    nx, ex = _sig(fmt, rng), rng.randrange(-20, 20)
    t = EMIN + rng.randrange(40)
    sx, sa = _sgn(rng), _sgn(rng)
    return val(fmt, sx * nx, ex - M), val(fmt, sa, t - ex), val(fmt, -sx * sa * nx, t - M)


FAMILIES = (sub_x_normal_product, sub_a_subnormal_product, sub_x_underflow, sub_both, half_smallest_subnormal,
            subnormal_rounds_to_normal, subnormal_tie, largest_finite, max_plus_half_ulp, max_plus_just_below_half_ulp,
            product_overflows_sum_does_not, infinite_b, carry_into_new_binade, product_last_bit_tie, exact_zero)


def family_of(tile, thread, i):
    """The family of triple i of a thread: every tile holds every family, in several threads and slots."""
    return (tile + thread * ft.NX + i) % len(FAMILIES)


@functools.lru_cache(maxsize=None)
def fma_tiles(fmt):
    """[tile] -> [thread] -> (x[8], a[16], b[16]) as bits."""
    tiles = []
    for t in range(ft.TILES):
        rng = random.Random(0xF7E0 + 16 * fmt + t)
        ops = []
        for th in range(ft.THREADS):
            x, a, b = [], [0] * ft.NAB, [0] * ft.NAB
            for i in range(ft.NX):
                fam = FAMILIES[family_of(t, th, i)]
                xi, ai, bi = fam(fmt, rng)
                x.append(xi)
                a[i], b[i] = ai, bi
                # the exact zero's mirror keeps b (x * -a + b = 2b): a thread holds one exact zero, not two, because
                # the sign-bit flips of two results change the fold by (2j + 1 + 2j' + 1) 2^31, a multiple of 2^32
                a[ft.NX + i], b[ft.NX + i] = neg(fmt, ai), bi if fam is exact_zero else neg(fmt, bi)
            ops.append((x, a, b))
        tiles.append(ops)
    return tiles


def fma_table(fmt, tiles):
    """(tables [tile][slot][thread], words [tile][thread][word], checks [tile][thread]) of tiles[tile][thread] =
    (x, a, b).  Refuses (NaNResult) a table in which any of a thread's 128 combinations would be NaN."""
    dt = np.uint32 if fmt == ft.FP32 else np.uint64
    tables = np.zeros((ft.TILES, ft.SLOTS[fmt], ft.THREADS), dtype=dt)
    words = np.zeros((ft.TILES, ft.THREADS, ft.WORDS[fmt]), dtype=np.uint32)
    checks = np.zeros((ft.TILES, ft.THREADS), dtype=np.uint32)
    for t, ops in enumerate(tiles):
        for th, (x, a, b) in enumerate(ops):
            for s, v in enumerate(list(x) + list(a) + list(b)):
                tables[t, s, th] = v
            try:
                w = ft.fma_words(fmt, x, a, b)
            except ft.NaNResult as e:
                raise ft.NaNResult("tile %d thread %d: %s" % (t, th, e)) from None
            words[t, th] = w
            checks[t, th] = ft.fold(w)
    return tables, words, checks


# ---- DMMA tiles ---------------------------------------------------------------------------------------------------------
# A tile is (A[w][s] 16 x 16, B[w][s] 16 x 8 integer matrices, ea, eb); set c of warp w sums A_s B_{(s + c) % 4}.
MAX = ft.DMMA_MAX


def dmma_results(A, B):
    """[w][c] 16 x 8 exact results (Python ints in an object array)."""
    return [[sum(A[w][s].astype(object) @ B[w][(s + c) % ft.DMMA_STEPS].astype(object) for s in range(ft.DMMA_STEPS))
             for c in range(ft.DMMA_SETS)] for w in range(4)]


def dmma_table(tiles, neg_zero_a=()):
    """(tables [tile][slot][thread], words, checks) of DMMA tiles (A, B, ea, eb), through the oracle's fragment maps.
    Tiles listed in neg_zero_a hold -0 where A is 0."""
    tables = np.zeros((ft.TILES, ft.SLOTS[ft.DMMA], ft.THREADS), dtype=np.uint64)
    words = np.zeros((ft.TILES, ft.THREADS, ft.WORDS[ft.DMMA]), dtype=np.uint32)
    for t, (A, B, ea, eb) in enumerate(tiles):
        D = dmma_results(A, B)
        for w in range(4):
            for l in range(32):
                th = w * 32 + l
                for s in range(ft.DMMA_STEPS):
                    for i in range(8):
                        v = int(A[w][s][ft.a_frag(l, i)])
                        tables[t, s * 8 + i, th] = ft.f64_bits(v, ea) | (1 << 63 if v == 0 and t in neg_zero_a else 0)
                    for i in range(4):
                        tables[t, 32 + s * 4 + i, th] = ft.f64_bits(int(B[w][s][ft.b_frag(l, i)]), eb)
                for c in range(ft.DMMA_SETS):
                    for i in range(4):
                        d = int(D[w][c][ft.d_frag(l, i)])
                        assert abs(d) < 1 << 53, d
                        r = ft.f64_bits(d, ea + eb)
                        words[t, th, 8 * c + 2 * i:8 * c + 2 * i + 2] = (r & ft.M32, r >> 32)
    checks = np.array([[ft.fold(words[t, th].tolist()) for th in range(ft.THREADS)] for t in range(ft.TILES)],
                      dtype=np.uint32)
    return tables, words, checks


def generator_dmma_tile(seed, tile):
    """The generator's tile as integer matrices (to check dmma_table against fp_test_oracle.tile, and to corrupt)."""
    A = [[ft.dmma_matrix(seed, tile, 0, w, s) for s in range(ft.DMMA_STEPS)] for w in range(4)]
    B = [[ft.dmma_matrix(seed, tile, 1, w, s) for s in range(ft.DMMA_STEPS)] for w in range(4)]
    return A, B, ft.dmma_scale_exp(seed, tile, 0), ft.dmma_scale_exp(seed, tile, 1)


def bound_tile(ea=0, eb=0):
    """Every product +max^2 (warps 0, 2: max * max; warps 1, 3: -max * -max): every result is 64 max^2 =
    2^53 - 308,303,296, and every partial sum climbs straight to it."""
    A = [[np.full((16, 16), MAX if w % 2 == 0 else -MAX, np.int64) for _ in range(4)] for w in range(4)]
    B = [[np.full((16, 8), MAX if w % 2 == 0 else -MAX, np.int64) for _ in range(4)] for w in range(4)]
    return A, B, ea, eb


def late_entries(w, n):
    """B column n of warp w: its (step, k) entries that hold sigma_n = +1 (n < 4) or -1 (n >= 4) instead of max."""
    return [((w + m) % 4, m) for m in range(4 * (n % 4), 4 * (n % 4) + 4)]


def late_tile():
    """A_w[m][m] = 1 in warp w (step w, k = m), B as late_entries, every other element max.  Result (c, m, n) with
    n % 4 = m // 4 and c = m % 4 holds the single product 1 * sigma_n: it is 60 max^2 + sigma_n (3 max + 1), above
    2^52.9 where one ulp is 1, and that +-1 product at (step w, k = m) decides its last unit.  Over the four warps the
    +-1 sits at every k of every step, with both signs."""
    A = [[np.full((16, 16), MAX, np.int64) for _ in range(4)] for _ in range(4)]
    B = [[np.full((16, 8), MAX, np.int64) for _ in range(4)] for _ in range(4)]
    for w in range(4):
        for m in range(16):
            A[w][w][m, m] = 1
        for n in range(8):
            for s, k in late_entries(w, n):
                B[w][s][k, n] = 1 if n < 4 else -1
    return A, B, 0, 0


def late_cases():
    """(w, c, m, n, sigma) of every result that holds a +-1 product."""
    return [(w, m % 4, m, n, 1 if n < 4 else -1) for w in range(4) for m in range(16) for n in range(8)
            if n % 4 == m // 4]


def walsh(K=ft.DMMA_K):
    H = np.ones((1, 1), np.int64)
    while len(H) < K:
        H = np.block([[H, H], [H, -H]])
    return H


def walsh_tile(ea=0, eb=0):
    """Row m of warp w's A (over the 64 k of the four steps) is max * Walsh row (16 w + m) % 64; column n of B is
    -max * Walsh row r_n, with r_n = (16 w + n) for n < 4 and that row XOR 32 for n >= 4.  Every result is 0 or
    +-64 max^2; the Walsh row 32 products climb to 32 max^2 after two steps and cancel to exactly 0."""
    H = walsh()
    A, B = [], []
    for w in range(4):
        a = np.stack([MAX * H[(16 * w + m) % 64] for m in range(16)])                # 16 x 64
        b = np.stack([-MAX * H[((16 * w + n % 4) ^ (32 if n >= 4 else 0)) % 64] for n in range(8)], axis=1)  # 64 x 8
        A.append([a[:, 16 * s:16 * s + 16].copy() for s in range(4)])
        B.append([b[16 * s:16 * s + 16, :].copy() for s in range(4)])
    return A, B, ea, eb


def neg_zero_tile():
    """A all zero (written as -0 by dmma_table), B positive: every product is -0; the accumulators start at +0, so
    every result is +0."""
    A = [[np.zeros((16, 16), np.int64) for _ in range(4)] for _ in range(4)]
    B = [[np.full((16, 8), 1 + (w * 4 + s) * 1000, np.int64) for s in range(4)] for w in range(4)]
    return A, B, 0, 0


NEG_ZERO_TILE = 7
LATE_TILE = 3


def dmma_crafted():
    """[(name, tile)] * TILES: one table of crafted DMMA tiles."""
    E = ft.DMMA_SCALE_EXP
    return [
        ("bound", bound_tile()),
        ("bound scaled up", bound_tile(E, E)),
        ("bound scaled down", bound_tile(-E, -E)),
        ("late +-1", late_tile()),
        ("walsh", walsh_tile()),
        ("walsh scaled", walsh_tile(E, -E)),
        ("bound mixed scale", bound_tile(E, -E)),
        ("all -0 products", neg_zero_tile()),
    ]


def dmma_crafted_table():
    return dmma_table([t for _, t in dmma_crafted()], neg_zero_a=(NEG_ZERO_TILE,))


# ---- edge seeds ---------------------------------------------------------------------------------------------------------
CORNERS = ((480, 480), (-480, -480), (480, -480))
SCAN_LIMIT = 1 << 22


def _mix(x):
    x = x ^ (x >> np.uint32(16))
    x = x * np.uint32(0x7FEB352D)
    x = x ^ (x >> np.uint32(15))
    x = x * np.uint32(0x846CA68B)
    return x ^ (x >> np.uint32(16))


def scale_exps(seeds, tile):
    """(ea, eb) of DMMA tile `tile` for every seed of a uint32 array: fp_test_oracle.dmma_scale_exp, vectorised."""
    key = _mix(seeds ^ np.uint32(((((ft.DMMA * 16 + tile) * 4 + 2) + 1) * 0x85EBCA77) & ft.M32))
    out = []
    for op in (0, 1):
        h = _mix(key + _mix(np.uint32(op))).astype(np.uint64)
        span = 2 * ft.DMMA_SCALE_EXP + 1
        out.append(-ft.DMMA_SCALE_EXP + ((h * np.uint64(span)) >> np.uint64(32)).astype(np.int64))
    return out


@functools.lru_cache(maxsize=None)
def corner_seed(ea, eb):
    """(seed, tile): the first seed with a DMMA tile scaled by exactly (2^ea, 2^eb)."""
    chunk = 1 << 18
    with np.errstate(over="ignore"):
        for lo in range(0, SCAN_LIMIT, chunk):
            seeds = np.arange(lo, lo + chunk, dtype=np.uint32)
            best = None
            for t in range(ft.TILES):
                a, b = scale_exps(seeds, t)
                hit = np.nonzero((a == ea) & (b == eb))[0]
                if len(hit) and (best is None or hit[0] < best[0]):
                    best = (int(hit[0]), t)
            if best is not None:
                return lo + best[0], best[1]
    raise AssertionError("no seed below %d reaches (%d, %d)" % (SCAN_LIMIT, ea, eb))


def edge_seeds():
    return sorted({corner_seed(*c)[0] for c in CORNERS})


SWEEP_SEEDS = 256


def sweep_seeds():
    """SWEEP_SEEDS seeds: the edge seeds, then 0, 1, 2, ... ."""
    edges = edge_seeds()
    return edges + [s for s in range(SWEEP_SEEDS) if s not in edges][:SWEEP_SEEDS - len(edges)]
