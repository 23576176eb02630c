"""The FP32 / FP64 self-test's inputs beyond its generator (tests/fp_test_edges.py) and its fault models
(tests/fp_test_faults.py), on the CPU:
- the oracle's infinities, overflow and wrong rounding rules on spot values;
- the fault-model table of DESIGN.md §4.7: every wrong-unit rule but subnormal double rounding changes the check value
  of every thread of every tile the product builds, and of at least one thread of every crafted tile;
- every crafted FMA family reaches the edge it names, the host's std::fma equals the oracle on all 128 combinations of
  every crafted thread, and a table with a NaN result is refused;
- every crafted DMMA tile reaches what it names, the fragment writer equals the generator's tables, and the host equals
  the oracle at the scanned scale-corner seeds.  No GPU needed."""
import subprocess

import numpy as np
import pytest

import fp_test_edges as fe
import fp_test_faults as ff
import fp_test_oracle as ft
import test_fp_test_cpu
from test_fp_test_cpu import drv  # noqa: F401  (fixture: the host arithmetic's CPU driver)

FMA_FMTS = (ft.FP32, ft.FP64)
FMA_IDS = [ft.NAMES[f] for f in FMA_FMTS]
FAULT_SEEDS = (0, 0xC0FFEE17)       # the seeds the DUMP tests compare on the GPU


# ---- the oracle at the edges --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMA_FMTS, ids=FMA_IDS)
def test_oracle_infinities_and_overflow(fmt):
    W, M, BIAS = ft.BIN[fmt][:3]
    one, two = ft.make(fmt, 0, 0, 0), ft.make(fmt, 0, 1, 0)
    mx, pinf, ninf = fe.max_finite(fmt), ft.inf(fmt, 0), ft.inf(fmt, 1)
    assert ft.decode(fmt, pinf) == (0, None, 0) and ft.decode(fmt, ninf) == (1, None, 0)
    with pytest.raises(ft.NaNResult):
        ft.decode(fmt, pinf | 1)
    assert ft.fma(fmt, mx, one, 0) == mx
    assert ft.fma(fmt, mx, two, 0) == pinf and ft.fma(fmt, mx, two | 1 << (W - 1), 0) == ninf
    half_ulp = ft.make(fmt, 0, BIAS - M - 1, 0)
    assert ft.fma(fmt, half_ulp, one, mx) == pinf                       # MAX + ulp/2: a tie, to even = infinity
    assert ft.fma(fmt, half_ulp, one, mx, mode="truncate") == mx
    below = ft.make(fmt, 0, BIAS - M - 2, (1 << M) - 1)                # ulp/2 (1 - 2^-(M+1))
    assert ft.fma(fmt, below, one, mx) == mx
    assert ft.fma(fmt, one, one, ninf) == ninf and ft.fma(fmt, mx, two, ninf) == ninf
    assert ft.mul(fmt, mx, two) == pinf
    for x, a, b in ((pinf, 0, one), (pinf, one, ninf)):     # inf * 0, inf - inf
        with pytest.raises(ft.NaNResult):
            ft.fma(fmt, x, a, b)


def test_oracle_rounding_rules_on_a_tie_and_a_sticky_case():
    f = ft.FP32
    # 1 + 2^-23 (odd) + 2^-24: a tie
    one_odd, half_ulp, one = ft.make(f, 0, 0, 1), ft.make(f, 0, -24, 0), ft.make(f, 0, 0, 0)
    assert ft.fma(f, one_odd, one, half_ulp) == ft.make(f, 0, 0, 2)
    assert ft.fma(f, one_odd, one, half_ulp, mode="ties_toward_zero") == one_odd
    assert ft.fma(f, one_odd, one, half_ulp, mode="truncate") == one_odd
    even = ft.make(f, 0, 0, 2)
    assert ft.fma(f, even, one, half_ulp, mode="ties_away") == ft.make(f, 0, 0, 3)
    # 1 + 2^-22 (even) + 2^-24 + 2^-30: above the tie; a unit without the sticky bit takes it for a tie and stays
    above = ft.make(f, 0, -24, 1 << 17)
    assert ft.fma(f, even, one, above) == ft.make(f, 0, 0, 3)
    assert ft.fma(f, even, one, above, mode="no_sticky") == even


# ---- fault models -------------------------------------------------------------------------------------------------------
def fault_counts(fmt, seed):
    """{rule: [threads whose check value differs, per tile]} on the product's tables."""
    out = {r: [] for r in ff.RULES}
    for t in range(ft.TILES):
        _, _, checks, ops = ft.tile(seed, fmt, t)
        wrong = ff.wrong_checks(fmt, ops, ff.RULES)
        for r in ff.RULES:
            out[r].append(sum(int(w != c) for w, c in zip(wrong[r], checks)))
    return out


@pytest.mark.parametrize("fmt", FMA_FMTS, ids=FMA_IDS)
@pytest.mark.parametrize("seed", FAULT_SEEDS)
def test_fault_model_table(fmt, seed):
    """Every thread of every tile holds a result each required rule gets wrong (daz_mul: the subnormal-operand class),
    so each changes all 128 check values of every tile.  Subnormal double rounding has no crafted class: its counts are
    recorded, not required."""
    counts = fault_counts(fmt, seed)
    for r in ff.RULES:
        print("%s seed 0x%x %-24s threads changed per tile: %s" % (ft.NAMES[fmt], seed, r, counts[r]))
    for r in ff.REQUIRED:
        assert counts[r] == [ft.THREADS] * ft.TILES, (r, counts[r])
    assert all(0 <= c <= ft.THREADS for c in counts["subnormal_double_round"])


@pytest.mark.parametrize("fmt", FMA_FMTS, ids=FMA_IDS)
def test_two_sign_flips_cancel_in_the_fold_and_the_tables_hold_an_odd_number_of_exact_zeros(fmt):
    """The fold sum (2j + 1) w_j mod 2^32 catches any single flipped bit, but flipping bit 31 of two words changes it
    by (2j + 1 + 2j' + 1) 2^31 = 0 mod 2^32.  So a unit that gives every exact zero the wrong sign is caught only in a
    thread with an odd number of exact-zero results: every thread of the product's tables holds nine (the -0 class's
    pair gives eight, the +0 class one)."""
    _, words, checks, ops = ft.tile(0xC0FFEE17, fmt, 2)
    w = list(words[5])
    top = 0 if fmt == ft.FP32 else 1            # the word holding the sign bit of result 0
    for j2 in (1, 2, 50):
        y = list(w)
        y[top] ^= 1 << 31
        y[2 * j2 + top if fmt == ft.FP64 else j2] ^= 1 << 31
        assert ft.fold(y) == checks[5]
    for seed in FAULT_SEEDS:
        for t in range(ft.TILES):
            for x, a, b in ft.tile(seed, fmt, t)[3]:
                zeros = sum(ff.exact(fmt, x[i], a[k], b[k])[1] == 0 for k in range(ft.NAB) for i in range(ft.NX))
                assert zeros == 9, (seed, t, zeros)


@pytest.mark.parametrize("fmt", FMA_FMTS, ids=FMA_IDS)
def test_every_required_rule_changes_a_check_in_every_crafted_tile(fmt):
    tiles = fe.fma_tiles(fmt)
    _, _, checks = fe.fma_table(fmt, tiles)
    for t, ops in enumerate(tiles):
        wrong = ff.wrong_checks(fmt, ops, ff.REQUIRED)
        for r in ff.REQUIRED:
            assert any(int(w) != int(c) for w, c in zip(wrong[r], checks[t])), (t, r)


@pytest.mark.parametrize("fmt", FMA_FMTS, ids=FMA_IDS)
def test_subnormal_double_round_on_a_spot_value(fmt):
    """b = k units of the subnormal grid (k = 2^(M-1) + 1, odd), x * a = 3/8 unit: one rounding gives k; rounding to
    M + 1 bits first gives k + 1/2, a tie, which then goes to the even k + 1.  A normal result is rounded once."""
    M, EMIN = ft.BIN[fmt][1], ft.BIN[fmt][3]
    k = (1 << (M - 1)) + 1
    x, a, b = fe.val(fmt, 3, EMIN - M - 3 + 40), fe.val(fmt, 1, -40), fe.val(fmt, k, EMIN - M)
    assert ft.fma(fmt, x, a, b) == k
    assert ff.wrong_fma(fmt, x, a, b, "subnormal_double_round") == k + 1
    n = ft.make(fmt, 0, 0, 5)
    assert ff.wrong_fma(fmt, n, n, n, "subnormal_double_round") == ft.fma(fmt, n, n, n)


# ---- crafted FMA tables -------------------------------------------------------------------------------------------------
def _family_triples(fmt):
    """{family name: [(x, a, b)]} over every tile and thread (the crafted triples, not their mirrors)."""
    out = {f.__name__: [] for f in fe.FAMILIES}
    for t, ops in enumerate(fe.fma_tiles(fmt)):
        for th, (x, a, b) in enumerate(ops):
            for i in range(ft.NX):
                out[fe.FAMILIES[fe.family_of(t, th, i)].__name__].append((x[i], a[i], b[i]))
    return out


def _mag(fmt, v):
    return v & ((1 << (ft.BIN[fmt][0] - 1)) - 1)


@pytest.mark.parametrize("fmt", FMA_FMTS, ids=FMA_IDS)
def test_crafted_fma_families_reach_their_edges(fmt):
    W, M, BIAS, EMIN = ft.BIN[fmt][:4]
    sub, sign = ff.is_subnormal, 1 << (W - 1)
    normal_min, mx, pinf = ft.make(fmt, 0, EMIN, 0), fe.max_finite(fmt), ft.inf(fmt, 0)
    fams = _family_triples(fmt)
    for t in range(ft.TILES):      # every tile holds every family
        assert {fe.family_of(t, th, i) for th in range(ft.THREADS) for i in range(ft.NX)} == set(range(len(fe.FAMILIES)))
    seen = {}
    for name, triples in fams.items():
        assert len(triples) >= 400, name
        for x, a, b in triples:
            r, tie, up = ft.fma(fmt, x, a, b, detail=True)
            ex = ff.exact(fmt, x, a, b)
            s, N, E = ex if ex is not None else (None, None, None)
            key = name
            if name == "sub_x_normal_product":
                assert sub(fmt, x) and not sub(fmt, ft.mul(fmt, x, a)) and _mag(fmt, ft.mul(fmt, x, a)) >= normal_min
            elif name == "sub_a_subnormal_product":
                assert sub(fmt, a) and sub(fmt, r) and N.bit_length() + E - 1 < EMIN
            elif name == "sub_x_underflow":
                assert sub(fmt, x) and N > 0 and r == s << (W - 1)         # a nonzero value underflows to its signed zero
                seen[key, "-0"] = seen.get((key, "-0"), 0) + (r == sign)
            elif name == "sub_both":
                assert sub(fmt, x) and sub(fmt, a)
            elif name == "half_smallest_subnormal":
                assert sub(fmt, x) and _mag(fmt, r) in (0, 1)
                seen[key, _mag(fmt, r)] = 1
                if _mag(fmt, r) == 0:
                    assert tie and not up
            elif name == "subnormal_rounds_to_normal":
                assert sub(fmt, x) and _mag(fmt, r) == normal_min and up and N.bit_length() + E - 1 < EMIN
            elif name == "subnormal_tie":
                assert sub(fmt, b) and tie and (sub(fmt, r) or _mag(fmt, r) == normal_min)
                seen[key, up] = 1
            elif name == "largest_finite":
                assert _mag(fmt, r) == mx
            elif name == "max_plus_half_ulp":
                assert _mag(fmt, r) == pinf and tie and up
            elif name == "max_plus_just_below_half_ulp":
                assert _mag(fmt, r) == mx and not up
            elif name == "product_overflows_sum_does_not":
                assert _mag(fmt, ft.mul(fmt, x, a)) == pinf and 0 < _mag(fmt, r) < pinf
                assert _mag(fmt, ff.wrong_fma(fmt, x, a, b, "unfused")) == pinf
            elif name == "infinite_b":
                assert _mag(fmt, b) == pinf and r == b
            elif name == "carry_into_new_binade":
                assert up and _mag(fmt, r) & ((1 << M) - 1) == 0 and N == (1 << (2 * M + 2)) - 1
            elif name == "product_last_bit_tie":
                _, nx, ex_ = ft.decode(fmt, x)
                _, na, ea_ = ft.decode(fmt, a)
                assert (nx * na).bit_length() == 2 * M + 2 and nx * na & 1
                n = N << (E - ex_ - ea_) if E >= ex_ + ea_ else N >> (ex_ + ea_ - E)   # in units of the product's last bit
                assert n.bit_length() == 2 * M + 2 and n & ((1 << (M + 1)) - 1) in ((1 << M) - 1, 1 << M, (1 << M) + 1)
                seen[key, (n & ((1 << (M + 1)) - 1)) - (1 << M)] = 1
            elif name == "exact_zero":
                assert N == 0 and r == 0
            else:
                raise AssertionError(name)
    assert seen["sub_x_underflow", "-0"] > 0
    assert all((k, v) in seen for k, vs in (("half_smallest_subnormal", (0, 1)), ("subnormal_tie", (False, True)),
                                            ("product_last_bit_tie", (-1, 0, 1))) for v in vs), seen


@pytest.mark.parametrize("fmt", FMA_FMTS, ids=FMA_IDS)
def test_crafted_fma_tables_follow_the_layout_and_give_no_nan(fmt):
    tiles = fe.fma_tiles(fmt)
    tables, words, checks = fe.fma_table(fmt, tiles)
    W = ft.BIN[fmt][0]
    for t in (0, ft.TILES - 1):
        for th in (0, 77, ft.THREADS - 1):
            x, a, b = tiles[t][th]
            assert tables[t, :, th].tolist() == list(x) + list(a) + list(b)
            assert a[ft.NX:] == [v ^ 1 << (W - 1) for v in a[:ft.NX]]
            assert b[ft.NX:] == [v if fe.FAMILIES[fe.family_of(t, th, i)] is fe.exact_zero else v ^ 1 << (W - 1)
                                 for i, v in enumerate(b[:ft.NX])]
            assert words[t, th].tolist() == ft.fma_words(fmt, x, a, b) and checks[t, th] == ft.fold(words[t, th].tolist())
    # the other combinations of the crafted values reach both infinities and signed zeros too
    res = words.reshape(ft.TILES, ft.THREADS, ft.RESULTS, -1)
    res = res[..., 0].astype(np.uint64) | (res[..., 1].astype(np.uint64) << np.uint64(32) if fmt == ft.FP64 else 0)
    assert {ft.inf(fmt, 0), ft.inf(fmt, 1), 0, 1 << (W - 1)} <= set(np.unique(res).tolist())
    bad = [[tuple(list(v) for v in op) for op in ops] for ops in tiles]
    x, a, b = bad[5][9]
    x[3], a[4], b[4] = ft.inf(fmt, 0), ft.make(fmt, 0, 0, 0), ft.inf(fmt, 1)     # inf * 1 + -inf
    with pytest.raises(ft.NaNResult, match="tile 5 thread 9"):
        fe.fma_table(fmt, bad)


@pytest.mark.parametrize("fmt", FMA_FMTS, ids=FMA_IDS)
def test_host_fma_equals_the_oracle_on_every_crafted_combination(drv, fmt):  # noqa: F811
    """std::fmaf / std::fma (ft_fma, the product's host reference) on all 128 combinations of every crafted thread."""
    tiles = fe.fma_tiles(fmt)
    _, words, _ = fe.fma_table(fmt, tiles)
    lines, want = [], []
    for t, ops in enumerate(tiles):
        for th, (x, a, b) in enumerate(ops):
            for k in range(ft.NAB):
                for i in range(ft.NX):
                    lines.append("fma %d %d %d %d" % (fmt, x[i], a[k], b[k]))
                    j = k * ft.NX + i
                    w = words[t, th]
                    want.append(int(w[j]) if fmt == ft.FP32 else int(w[2 * j]) | int(w[2 * j + 1]) << 32)
    r = subprocess.run(drv.p.args, input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    got = [int(v) for v in r.stdout.split()]
    assert len(got) == len(want)
    bad = [(lines[i], hex(g), hex(w)) for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, (len(bad), bad[:5])


# ---- crafted DMMA tiles -------------------------------------------------------------------------------------------------
def test_dmma_fragment_writer_equals_the_generator_tables():
    tiles = [fe.generator_dmma_tile(0x0BAD, t) for t in range(ft.TILES)]
    tables, words, checks = fe.dmma_table(tiles)
    for t in range(ft.TILES):
        table, w, c, _ = ft.tile(0x0BAD, ft.DMMA, t)
        assert np.array_equal(tables[t], np.array(table, dtype=np.uint64))
        assert np.array_equal(words[t], np.array(w, dtype=np.uint32)) and checks[t].tolist() == c


def _results(tile):
    A, B, _, _ = tile
    return fe.dmma_results(A, B)


def test_dmma_bound_tiles_sit_at_the_2_to_53_bound():
    bound = ft.DMMA_K * ft.DMMA_MAX ** 2
    assert bound == 9007198946437696 == (1 << 53) - 308303296
    named = dict(fe.dmma_crafted())
    scales = set()
    for name in ("bound", "bound scaled up", "bound scaled down", "bound mixed scale"):
        A, B, ea, eb = named[name]
        scales.add((ea, eb))
        for w in range(4):
            for c in range(ft.DMMA_SETS):
                assert (_results(named[name])[w][c] == bound).all()
            assert all((A[w][s] * B[w][s][0, 0] == ft.DMMA_MAX ** 2).all() for s in range(4))
    assert {(0, 0), (480, 480), (-480, -480), (480, -480)} <= scales
    _, words, _ = fe.dmma_crafted_table()
    hi = words[1, :, 1::2].astype(np.uint64) << np.uint64(32) | words[1, :, 0::2].astype(np.uint64)
    assert (hi.view(np.float64) == np.ldexp(float(bound), 960)).all()


def test_dmma_late_addend_reaches_every_k_of_every_step_with_both_signs():
    tile = fe.late_tile()
    D = _results(tile)
    cases = fe.late_cases()
    placed = set()
    for w, c, m, n, sigma in cases:
        want = 60 * ft.DMMA_MAX ** 2 + sigma * (3 * ft.DMMA_MAX + 1)
        assert D[w][c][m, n] == want and want > 2 ** 52.9 and want < 1 << 53, (w, c, m, n)
        placed.add((w, m, sigma))              # the +-1 product: step w, k = m
        # without the +-1 product the result moves by exactly one unit, which is one ulp at this size
        A, B, _, _ = tile
        B2 = [[b.copy() for b in bw] for bw in B]
        B2[w][(w + c) % 4][m, n] = 0
        assert fe.dmma_results(A, B2)[w][c][m, n] == want - sigma
    assert placed == {(s, k, sg) for s in range(4) for k in range(16) for sg in (1, -1)}


def test_dmma_walsh_tiles_cancel_to_exact_zero_after_climbing():
    A, B, _, _ = fe.walsh_tile()
    top = 0
    zeros = 0
    for w in range(4):
        for c in range(ft.DMMA_SETS):
            parts = [A[w][s].astype(object) @ B[w][(s + c) % 4].astype(object) for s in range(4)]
            D = sum(parts)
            assert set(np.abs(D).ravel().tolist()) <= {0, 64 * ft.DMMA_MAX ** 2}
            prefix = np.abs(np.cumsum(np.stack(parts), axis=0))
            z = D == 0
            zeros += int(z.sum())
            top = max(top, int(prefix[:, z].max()))
    assert zeros > 0 and top == 32 * ft.DMMA_MAX ** 2


def test_dmma_neg_zero_tile():
    tables, words, _ = fe.dmma_crafted_table()
    t = fe.NEG_ZERO_TILE
    assert fe.dmma_crafted()[t][0] == "all -0 products"
    assert (tables[t, :32] == np.uint64(1 << 63)).all() and (tables[t, 32:] < np.uint64(1 << 63)).all()
    assert (tables[t, 32:] != 0).all() and (words[t] == 0).all()        # every result +0


def test_corner_seeds_are_the_first_and_the_host_is_held_to_the_oracle_there():
    """The scan's seeds are the first to reach each corner, and test_fp_test_cpu holds the host's tables equal to the
    oracle's at each of them (in every format)."""
    rng = np.random.default_rng(5)
    sample = rng.integers(0, 1 << 32, 300, dtype=np.uint64).astype(np.uint32)
    with np.errstate(over="ignore"):
        for t in (0, 7):
            ea, eb = fe.scale_exps(sample, t)
            assert [(int(a), int(b)) for a, b in zip(ea, eb)] == \
                [(ft.dmma_scale_exp(int(s), t, 0), ft.dmma_scale_exp(int(s), t, 1)) for s in sample]
    for c in fe.CORNERS:
        seed, tile = fe.corner_seed(*c)
        assert (ft.dmma_scale_exp(seed, tile, 0), ft.dmma_scale_exp(seed, tile, 1)) == c
        with np.errstate(over="ignore"):
            below = np.arange(seed, dtype=np.uint32)
            assert not any(((lambda e: (e[0] == c[0]) & (e[1] == c[1]))(fe.scale_exps(below, t))).any()
                           for t in range(ft.TILES))
    print("DMMA scale-corner seeds:", {c: fe.corner_seed(*c) for c in fe.CORNERS})
    assert set(fe.edge_seeds()) <= set(test_fp_test_cpu.SEEDS)
    sweep = fe.sweep_seeds()
    assert len(sweep) == len(set(sweep)) == fe.SWEEP_SEEDS and set(fe.edge_seeds()) <= set(sweep)
