"""The FP32 / FP64 self-test kernel (fp_selftest.cuh) on a real H100, on inputs its generator's fixed seeds never
reach.  Inputs are in tests/fp_test_edges.py and the fault models in tests/fp_test_faults.py; the CPU checks of what
they reach are in tests/test_fp_test_edges_cpu.py.  Everything goes in through the tables and check values the kernel
reads (tests/native/libfp_test_kernels_test.so), so the path under test is the product's own.

- No false alarm: 256 seeds per format through the product's table builder, one round on every CTA of a full grid,
  the DMMA scale-corner seeds included.
- Crafted FMA and DMMA tables: DUMP (CTA 0) equals the oracle bit for bit, and the product instantiation reports no
  mismatch on any CTA of a full grid.
- Check values built by each wrong-unit rule are counted in every tile, on the product's tables and the crafted ones.
- A DMMA operand one unit off, in every warp x {A, B} x step, and a late +-1 addend set to 0 (one ulp), are counted in
  every repetition of every round by every CTA."""
import numpy as np
import pytest

import fp_test_edges as fe
import fp_test_faults as ff
import fp_test_oracle as ft
from test_gpu_fp_test import H, launch_tables, oracle_tiles  # noqa: F401  (H is a fixture)

pytestmark = pytest.mark.gpu

FMA_FMTS = (ft.FP32, ft.FP64)
FMA_IDS = [ft.NAMES[f] for f in FMA_FMTS]
FMT_IDS = [ft.NAMES[f] for f in ft.FORMATS]
RULE_SEED = 0x1EEE


def _rec(r):
    return dict(smid=r.smid, seq=r.seq, rounds=r.rounds, comparisons=r.comparisons, mismatches=r.mismatches,
                first_bad_tile=r.first_bad_tile, first_bad_rep=r.first_bad_rep)


def _clean(r):
    return (r.seq == 7 and r.rounds >= 1 and r.comparisons == r.rounds * ft.TILES * ft.REPS and r.mismatches == 0
            and (r.first_bad_tile, r.first_bad_rep) == (-1, -1))


# ---- no false alarm -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ft.FORMATS, ids=FMT_IDS)
def test_seed_sweep_raises_no_false_alarm(H, fmt):  # noqa: F811
    grid = H.sms * H.occupancy(fmt)
    bad = []
    for seed in fe.sweep_seeds():
        recs, _ = H.run(fmt, seed, 0)
        assert len(recs) == grid
        wrong = [_rec(r) for r in recs if not _clean(r)]
        if wrong:
            bad.append((seed, len(wrong), wrong[0]))
    assert not bad, bad[:8]


@pytest.mark.parametrize("seed", fe.edge_seeds())
def test_dmma_dump_matches_the_oracle_at_the_corner_seeds(H, seed):  # noqa: F811
    got, rec = H.dump(ft.DMMA, seed)
    want = np.array([oracle_tiles(seed, ft.DMMA)[t][1] for t in range(ft.TILES)], dtype=np.uint32)
    assert np.array_equal(got, want), np.argwhere(got != want)[:4].tolist()
    assert (rec.seq, rec.rounds, rec.comparisons, rec.mismatches) == (7, 1, ft.TILES * ft.REPS, 0)


# ---- crafted tables -----------------------------------------------------------------------------------------------------
def crafted(fmt):
    """(tables, words, checks, names per tile)."""
    if fmt == ft.DMMA:
        return (*fe.dmma_crafted_table(), [n for n, _ in fe.dmma_crafted()])
    return (*fe.fma_table(fmt, fe.fma_tiles(fmt)), ["crafted FMA tile %d" % t for t in range(ft.TILES)])


def _describe(fmt, got, want, names):
    out = []
    for t in range(ft.TILES):
        if not np.array_equal(got[t], want[t]):
            idx = np.argwhere(got[t] != want[t])
            th, j = idx[0]
            out.append("%s: %d words differ; first thread %d word %d got 0x%08x want 0x%08x"
                       % (names[t], len(idx), th, j, got[t][th, j], want[t][th, j]))
    return out


@pytest.mark.parametrize("fmt", ft.FORMATS, ids=FMT_IDS)
def test_crafted_tables_match_the_oracle_bit_for_bit(H, fmt):  # noqa: F811
    tables, words, checks, names = crafted(fmt)
    rc, (rec,), got = H.run_tables_rc(fmt, tables, checks, dump=True)
    assert rc == 0
    got = got.reshape(ft.TILES, ft.THREADS, ft.WORDS[fmt])
    bad = _describe(fmt, got, words, names)
    if bad and fmt != ft.DMMA:       # name the first differing operands (H100 against IEEE 754)
        t, th, j = np.argwhere(got != words)[0]
        j = j if fmt == ft.FP32 else j // 2
        x, a, b = fe.fma_tiles(fmt)[t][th]
        bad.append("first: fma(0x%x, 0x%x, 0x%x)" % (x[j % ft.NX], a[j // ft.NX], b[j // ft.NX]))
    assert not bad, "\n".join(bad)
    assert (rec.seq, rec.rounds, rec.comparisons, rec.mismatches) == (7, 1, ft.TILES * ft.REPS, 0), _rec(rec)
    grid = H.sms * H.occupancy(fmt)
    recs = H.run_tables(fmt, tables, checks, grid=grid)
    wrong = [_rec(r) for r in recs if not _clean(r)]
    assert len(recs) == grid and not wrong, wrong[:4]


# ---- wrong units --------------------------------------------------------------------------------------------------------
def _rule_checks(fmt, ops_per_tile, rule):
    return np.array([ff.wrong_checks(fmt, ops, [rule])[rule] for ops in ops_per_tile], dtype=np.uint32)


@pytest.mark.parametrize("rule", ff.REQUIRED)
@pytest.mark.parametrize("fmt", FMA_FMTS, ids=FMA_IDS)
def test_checks_of_every_wrong_unit_are_counted_in_every_tile(H, fmt, rule):  # noqa: F811
    """One CTA, one round: checks built by the rule mismatch in all 8 tiles x 16 repetitions, on the product's tables
    and on the crafted ones."""
    sources = [("generator", *launch_tables(RULE_SEED, fmt), [t[3] for t in oracle_tiles(RULE_SEED, fmt)])]
    tables, _, checks, _ = crafted(fmt)
    sources.append(("crafted", tables, checks, fe.fma_tiles(fmt)))
    for name, tables, checks, ops in sources:
        wrong = _rule_checks(fmt, ops, rule)
        assert all((wrong[t] != checks[t]).any() for t in range(ft.TILES)), name
        (r,) = H.run_tables(fmt, tables, wrong)
        assert (r.rounds, r.mismatches, r.first_bad_tile, r.first_bad_rep) == (1, ft.TILES * ft.REPS, 0, 0), \
            (name, _rec(r))


# ---- wrong DMMA operands ------------------------------------------------------------------------------------------------
RUN_MS = 5


def _every_cta_counts(H, tables, checks, tile):  # noqa: F811
    grid = H.sms * H.occupancy(ft.DMMA)
    recs = H.run_tables(ft.DMMA, tables, checks, grid=grid, duration_ms=RUN_MS)
    assert len(recs) == grid
    wrong = [_rec(r) for r in recs
             if not (r.seq == 7 and r.rounds >= 2 and r.comparisons == r.rounds * ft.TILES * ft.REPS
                     and r.mismatches == r.rounds * ft.REPS and (r.first_bad_tile, r.first_bad_rep) == (tile, 0))]
    assert not wrong, (len(wrong), wrong[:4])


OPERAND_SEED = 0x0BAD
DMMA_FLIPS = [(w, op, s) for w in range(4) for op in (0, 1) for s in range(ft.DMMA_STEPS)]


@pytest.mark.parametrize("w,op,s", DMMA_FLIPS, ids=["w%d-%s-s%d" % (w, "AB"[op], s) for w, op, s in DMMA_FLIPS])
def test_a_dmma_operand_one_unit_off_is_counted_by_every_cta(H, w, op, s):  # noqa: F811
    """Warp w's A_s or B_s: one element (row and column vary with the case) one unit off, in tile (w + s) % 8."""
    tiles = [fe.generator_dmma_tile(OPERAND_SEED, t) for t in range(ft.TILES)]
    _, _, checks = fe.dmma_table(tiles)
    tile = (w + 2 * s + op) % ft.TILES
    A, B, ea, eb = tiles[tile]
    M = [[m.copy() for m in mw] for mw in (A if op == 0 else B)]
    r, c = (5 * w + s) % 16, (3 * s + w + op) % (16 if op == 0 else 8)
    v = int(M[w][s][r, c])
    M[w][s][r, c] = v + 1 if v < ft.DMMA_MAX else v - 1
    tiles[tile] = (M, B, ea, eb) if op == 0 else (A, M, ea, eb)
    tables, _, wrong_checks = fe.dmma_table(tiles)
    assert (wrong_checks[tile] != checks[tile]).any()
    _every_cta_counts(H, tables, checks, tile)


@pytest.mark.parametrize("case", [0, 1], ids=["+1", "-1"])
def test_a_late_addend_set_to_zero_is_counted_by_every_cta(H, case):  # noqa: F811
    """The late tile's +-1 product of one result (warp 3, set c, row 15 at step 3, k = 15: the last k of the last
    step) with its B partner set to 0: that result moves by one ulp."""
    w, c, m, n, sigma = [cs for cs in fe.late_cases() if cs[0] == 3 and cs[2] == 15][case]
    assert sigma == (1, -1)[case]
    named = fe.dmma_crafted()
    tiles = [t for _, t in named]
    _, _, checks = fe.dmma_crafted_table()
    A, B, ea, eb = tiles[fe.LATE_TILE]
    B2 = [[b.copy() for b in bw] for bw in B]
    B2[w][(w + c) % 4][m, n] = 0
    tiles[fe.LATE_TILE] = (A, B2, ea, eb)
    tables, _, wrong = fe.dmma_table(tiles, neg_zero_a=(fe.NEG_ZERO_TILE,))
    assert (wrong[fe.LATE_TILE] != checks[fe.LATE_TILE]).any()
    _every_cta_counts(H, tables, checks, fe.LATE_TILE)
