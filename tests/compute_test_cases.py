"""Inputs for testing the tensor-core self-test (tc_selftest.cuh) beyond the generator's fixed seeds.
tests/test_compute_test_tables_cpu.py checks what each one reaches; tests/test_gpu_compute_test_tables.py runs them.

- Edge seeds, found by a deterministic scan from seed 0: the first seed whose BF16 scale exponents reach each corner
  (a, b) = (+-30, +-30), and per format the first seed with a result element that cancels to exactly 0.
- Crafted tiles the generator cannot make (one table of TILES tiles per format):
  - every element at the bound: A and B filled with lo (or hi), so D = K * lo^2 (or K * lo * hi) everywhere;
  - a late small addend: A row i and B row i hold lo everywhere except at one k*, where A = +-1 and B = +-1, so
    D[i][i] = (K - 1) lo^2 +- 1.  k* is the first and the last k of every K step (every k for FP8), both signs;
  - exact zeros by cancellation: A and B rows are +-hi times Walsh (Hadamard) rows, so D[m][n] = -K hi^2 when the two
    rows are the same Walsh row and exactly 0 otherwise, with mixed-sign sums that climb as far as (K / 2) hi^2.
- Corruption plans, each of which must be counted by the kernel: a wrong check value in every thread and tile, a wrong
  operand element in every warp and in the first and last K step, a one-unit change of a late-addend result, and two
  wrong tiles in one table."""
import functools

import numpy as np

import compute_test_oracle as ct
import compute_test_tables as tb

SCAN_LIMIT = 1 << 13                # the scan gives up here; every edge below is reached far earlier
CORNERS = ((30, 30), (-30, -30), (-30, 30), (30, -30))


# ---- edge seeds -----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def corner_seed(ea: int, eb: int):
    """(seed, tile): the first seed with a BF16 tile scaled by exactly (2^ea, 2^eb)."""
    for seed in range(SCAN_LIMIT):
        for t in range(ct.TILES):
            if (ct.scale_exp(seed, ct.BF16, t, 0), ct.scale_exp(seed, ct.BF16, t, 1)) == (ea, eb):
                return seed, t
    raise AssertionError("no seed below %d reaches (%d, %d)" % (SCAN_LIMIT, ea, eb))


@functools.lru_cache(maxsize=None)
def zero_seed(fmt: int):
    """(seed, tile, m, n): the first seed whose generated tiles hold a result element that is exactly 0."""
    for seed in range(SCAN_LIMIT):
        for t in range(ct.TILES):
            s = ct.operand(seed, fmt, t, 0) @ ct.operand(seed, fmt, t, 1).T
            hit = np.argwhere(s == 0)
            if len(hit):
                return seed, t, int(hit[0][0]), int(hit[0][1])
    raise AssertionError("no seed below %d has an exact zero in %s" % (SCAN_LIMIT, ct.NAMES[fmt]))


def edge_seeds(fmt: int):
    """The scanned seeds that matter for format fmt (sorted, distinct)."""
    seeds = {zero_seed(fmt)[0]}
    if fmt == ct.BF16:
        seeds |= {corner_seed(*c)[0] for c in CORNERS}
    return sorted(seeds)


SWEEP_SEEDS = 256


def sweep_seeds(fmt: int):
    """SWEEP_SEEDS seeds: the edge seeds, then 0, 1, 2, ... ."""
    edges = edge_seeds(fmt)
    return edges + [s for s in range(SWEEP_SEEDS) if s not in edges][:SWEEP_SEEDS - len(edges)]


# ---- crafted tiles --------------------------------------------------------------------------------------------------
def bound_tile(fmt: int, a: int, b: int, ea: int = 0, eb: int = 0):
    """A filled with a, B with b: every element is K * a * b, and every partial sum climbs straight to it."""
    return np.full((ct.M, ct.K[fmt]), a, np.int64), np.full((ct.N, ct.K[fmt]), b, np.int64), ea, eb


def late_ks(fmt: int):
    """The k of the late small addend: the first and the last k of every K step (one step for FP8: every k)."""
    sk = tb.STEP_K[fmt]
    if tb.STEPS[fmt] == 1:
        return list(range(ct.K[fmt]))
    return [k for s in range(tb.STEPS[fmt]) for k in (s * sk, s * sk + sk - 1)]


def late_cases(fmt: int):
    """Case i (A row i, B row i): (k*, sign of B at k*)."""
    return [(k, sign) for k in late_ks(fmt) for sign in (1, -1)]


def late_tile(fmt: int, a_unit: int = 1, ea: int = 0, eb: int = 0):
    """A row i and B row i are lo except at case i's k*, where A = a_unit and B = the case's sign: D[i][i] = (K - 1) lo^2
    + a_unit * sign.  Rows past the cases hold lo."""
    A, B, _, _ = bound_tile(fmt, ct.LO[fmt], ct.LO[fmt])
    for i, (k, sign) in enumerate(late_cases(fmt)):
        A[i, k], B[i, k] = a_unit, sign
    return A, B, ea, eb


def walsh(K: int) -> np.ndarray:
    """Sylvester's Hadamard matrix: H[i][k] = (-1)^popcount(i & k)."""
    H = np.ones((1, 1), np.int64)
    while len(H) < K:
        H = np.block([[H, H], [H, -H]])
    return H


def walsh_rows(fmt: int):
    """The Walsh row of each A row (m mod K) and each B row (n for n < 64, then from K / 2 on), so that the pairs whose
    product is Walsh row K / 2 -- + for the first half of K, - for the second -- are among them."""
    K = ct.K[fmt]
    return np.arange(ct.M) % K, np.array([n if n < 64 else n - 64 + K // 2 for n in range(ct.N)]) % K


def walsh_tile(fmt: int, ea: int = 0, eb: int = 0):
    H = walsh(ct.K[fmt])
    p, q = walsh_rows(fmt)
    return ct.HI[fmt] * H[p], -ct.HI[fmt] * H[q], ea, eb


def crafted_tiles(fmt: int):
    """[(name, (A, B, ea, eb))] * TILES: one table of crafted tiles.  The scale exponents apply to BF16 only."""
    lo, hi = ct.LO[fmt], ct.HI[fmt]

    def sc(ea, eb):
        return (ea, eb) if fmt == ct.BF16 else (0, 0)
    return [
        ("bound lo*lo", bound_tile(fmt, lo, lo)),
        ("bound lo*lo scaled", bound_tile(fmt, lo, lo, *sc(30, 30))),
        ("bound lo*lo scaled down", bound_tile(fmt, lo, lo, *sc(-30, -30))),
        ("bound lo*hi", bound_tile(fmt, lo, hi, *sc(30, -30))),
        ("late +1", late_tile(fmt, 1)),
        ("late -1 scaled", late_tile(fmt, -1, *sc(-30, 30))),
        ("walsh", walsh_tile(fmt)),
        ("walsh scaled", walsh_tile(fmt, *sc(30, 30))),
    ]


LATE_TILE = 4                       # crafted_tiles' "late +1": unscaled, so one unit of D is one ulp near 2^24 (BF16)


# ---- corruption plans -----------------------------------------------------------------------------------------------
def check_flips():
    """(tile, thread, mask) for every thread t: bit t mod 32 of thread t's check value of tile t mod 8."""
    return [(t % ct.TILES, t, 1 << (t % 32)) for t in range(ct.THREADS)]


OPERAND_SEED = 0xC0FFEE17           # the generator tables the operand corruptions start from


def operand_plan(fmt: int):
    """(tile, op, row, k): one operand element to change.  A rows 0, 17, 34 and 63 lie in the four warps' result rows;
    B rows 0 and 127 are result columns 0 and 127; k is in the first or the last K step."""
    K, sk = ct.K[fmt], tb.STEP_K[fmt]
    return [(0, 0, 0, 0), (3, 0, 17, K - 1), (7, 0, 34, sk - 1), (0, 0, 63, K - sk),
            (3, 1, 0, K - 1), (7, 1, 127, 0)]


TWO_TILE_PLAN = [(2, 0, 5, 1), (6, 1, 100, -2)]      # (tile, op, row, k); k < 0 counts from the end of K


def generator_tiles(fmt: int, seed: int = OPERAND_SEED):
    return [ct.tile(seed, fmt, t)[:4] for t in range(ct.TILES)]


def with_element(tiles, tile: int, op: int, row: int, k: int, value: int):
    """A copy of tiles in which operand op of tile `tile` holds value at (row, k)."""
    out = [(A.copy(), B.copy(), ea, eb) for A, B, ea, eb in tiles]
    out[tile][op][row, k] = value
    return out


def nudged(fmt: int, v: int) -> int:
    """Another value in [lo, hi]: v + 1, or v - 1 at hi."""
    return v + 1 if v < ct.HI[fmt] else v - 1


def corrupt_operands(fmt: int, tiles, plan):
    """tiles with every (tile, op, row, k) of plan nudged to a neighbouring value in range."""
    for tile, op, row, k in plan:
        k %= ct.K[fmt]
        tiles = with_element(tiles, tile, op, row, k, nudged(fmt, int(tiles[tile][op][row, k])))
    return tiles


def one_unit_cases(fmt: int):
    """Late-addend cases (row i) whose B partner at k* is set to 0 in the one-unit corruption: k* = the last k of the
    last K step, both signs."""
    cases = late_cases(fmt)
    return [i for i, (k, _) in enumerate(cases) if k == ct.K[fmt] - 1]


def one_unit_corruption(fmt: int, tiles, case: int):
    k, _ = late_cases(fmt)[case]
    return with_element(tiles, LATE_TILE, 1, case, k, 0)
