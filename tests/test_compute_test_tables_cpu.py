"""CPU side of the table-driven tests of the tensor-core self-test (tests/test_gpu_compute_test_tables.py):

- the oracle's shared-memory image, written from the layout's description, equals ct_build_tile's byte for byte;
- the oracle refuses operands the exactness argument does not cover;
- the scanned edge seeds reach what they were picked for, read from the numbers;
- the crafted tiles stay under every bound, and the late addend moves a BF16 result by one ulp at >= 2^23.9;
- every planned corruption changes some thread's check value, and together they reach every thread, tile and warp
  and the first and last K step of each format.  No GPU needed."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import compute_test_cases as cc
import compute_test_oracle as ct
import compute_test_tables as tb
from test_compute_test_cpu import BOUND, CSRC, ROOT, MathDriver

FMT_IDS = [ct.NAMES[f] for f in ct.FORMATS]


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    """tests/native/compute_test_image_test.cpp, compiled with g++ against csrc/compute_test_math.hpp."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("ct_image") / "compute_test_image_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                        os.path.join(ROOT, "tests", "native", "compute_test_image_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = MathDriver(exe)
    yield d
    d.close()


def _sums(A, B):
    """M x N x K: every prefix sum of every result element."""
    return np.cumsum(A[:, None, :].astype(np.int64) * B[None, :, :], axis=2)


# ---- the image --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", [0, 0xC0FFEE17, 0xFFFFFFFF, cc.corner_seed(30, -30)[0]])
def test_oracle_image_equals_the_products_image(drv, seed, fmt):
    for t in range(ct.TILES):
        A, B, ea, eb, _, _ = ct.tile(seed, fmt, t)
        want = tb.image(fmt, A, B, ea, eb)
        assert want.size == tb.SMEM[fmt]
        got = np.array(drv.ask("image", seed, fmt, t), dtype=np.int64)
        assert np.array_equal(got, want), (t, np.argwhere(got != want)[:4].ravel())


def test_oracle_refuses_operands_out_of_range():
    for fmt in ct.FORMATS:
        A, B, _, _ = cc.bound_tile(fmt, ct.LO[fmt], ct.HI[fmt])
        tb.image(fmt, A, B)
        for op, v in ((0, ct.LO[fmt] - 1), (1, ct.HI[fmt] + 1)):
            bad = [A.copy(), B.copy()]
            bad[op][5, 3] = v
            for fn in (tb.image, tb.reference):
                with pytest.raises(ValueError):
                    fn(fmt, *bad)
        with pytest.raises(ValueError):
            tb.image(fmt, A[:, :-1], B)
        with pytest.raises(ValueError):
            tb.tables(fmt, [(A, B, 0, 0)] * (ct.TILES - 1))
    A, B, _, _ = cc.bound_tile(ct.BF16, 1, 1)
    tb.image(ct.BF16, A, B, -30, 30)
    for ea, eb in ((31, 0), (0, -31)):
        with pytest.raises(ValueError):
            tb.image(ct.BF16, A, B, ea, eb)
    with pytest.raises(ValueError):
        tb.image(ct.INT8, A, B[:, :ct.K[ct.INT8]], 1, 0)


# ---- edge seeds -------------------------------------------------------------------------------------------------------
def test_corner_seeds_reach_the_bf16_scale_extremes():
    for ea, eb in cc.CORNERS:
        seed, t = cc.corner_seed(ea, eb)
        assert (ct.scale_exp(seed, ct.BF16, t, 0), ct.scale_exp(seed, ct.BF16, t, 1)) == (ea, eb)
        d = ct.tile(seed, ct.BF16, t)[4].view(np.float32).astype(np.float64)
        s = ct.operand(seed, ct.BF16, t, 0) @ ct.operand(seed, ct.BF16, t, 1).T
        assert np.array_equal(d, np.ldexp(s.astype(np.float64), ea + eb))
        # row 0 is the extreme row: its results reach the top of the range at this scale
        assert np.abs(d[0]).max() >= 2.0 ** (23.9 + ea + eb)
        for s0 in range(seed):                                # and it is the first seed that does
            assert all((ct.scale_exp(s0, ct.BF16, u, 0), ct.scale_exp(s0, ct.BF16, u, 1)) != (ea, eb)
                       for u in range(ct.TILES))


@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_zero_seed_has_an_exact_zero_from_mixed_signs(fmt):
    seed, t, m, n = cc.zero_seed(fmt)
    A, B, _, _, d, _ = ct.tile(seed, fmt, t)
    terms = A[m].astype(np.int64) * B[n]
    assert terms.sum() == 0 and terms.max() > 0 and terms.min() < 0
    assert d[m, n] == 0                                        # +0, not -0
    for s0 in range(seed):
        assert all(np.all(ct.operand(s0, fmt, u, 0) @ ct.operand(s0, fmt, u, 1).T != 0) for u in range(ct.TILES))


def test_sweep_seeds_hold_the_edge_seeds():
    for fmt in ct.FORMATS:
        seeds = cc.sweep_seeds(fmt)
        assert len(seeds) == len(set(seeds)) == cc.SWEEP_SEEDS
        assert set(cc.edge_seeds(fmt)) <= set(seeds)
    assert {cc.corner_seed(*c)[0] for c in cc.CORNERS} <= set(cc.sweep_seeds(ct.BF16))


# ---- crafted tiles ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_crafted_tiles_stay_under_the_bounds(fmt):
    tiles = cc.crafted_tiles(fmt)
    assert len(tiles) == ct.TILES
    for name, (A, B, ea, eb) in tiles:
        partial = _sums(A, B)
        assert np.abs(partial).max() < BOUND[fmt] or (fmt == ct.INT8 and np.abs(partial).max() <= 1 << 22), name
        if fmt != ct.INT8:                                     # the FP32 result is the exact sum
            f = tb.reference(fmt, A, B, ea, eb).view(np.float32).astype(np.float64)
            assert np.array_equal(f, np.ldexp(partial[:, :, -1].astype(np.float64), ea + eb)), name


@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_bound_tiles_sit_at_the_bound(fmt):
    K, lo = ct.K[fmt], ct.LO[fmt]
    tiles = dict(cc.crafted_tiles(fmt))
    A, B, ea, eb = tiles["bound lo*lo"]
    assert (ea, eb) == (0, 0) and np.all(A @ B.T == K * lo * lo)
    assert K * lo * lo == {ct.BF16: 16646400, ct.FP8: 7200, ct.INT8: 1 << 22}[fmt]
    if fmt == ct.BF16:
        assert (tiles["bound lo*lo scaled"][2:], tiles["bound lo*lo scaled down"][2:]) == ((30, 30), (-30, -30))
        d = tb.reference(fmt, *tiles["bound lo*lo scaled"]).view(np.float32)
        assert np.all(d == np.float32(16646400.0 * 2.0 ** 60))


@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_late_addend_sits_in_every_k_step(fmt):
    K, lo, sk = ct.K[fmt], ct.LO[fmt], tb.STEP_K[fmt]
    ks = cc.late_ks(fmt)
    # first and last k of every step; every k for FP8's single step
    assert {(k // sk, k % sk) for k in ks} >= {(s, 0) for s in range(tb.STEPS[fmt])} | \
        {(s, sk - 1) for s in range(tb.STEPS[fmt])}
    if fmt == ct.FP8:
        assert ks == list(range(K))
    cases = cc.late_cases(fmt)
    assert len(cases) <= ct.M and {sign for _, sign in cases} == {1, -1}
    for name, (A, B, ea, eb) in cc.crafted_tiles(fmt):
        if not name.startswith("late"):
            continue
        a_unit = int(A[0, cases[0][0]])
        s = A @ B.T
        for i, (k, sign) in enumerate(cases):
            assert s[i, i] == (K - 1) * lo * lo + a_unit * sign, (name, i)
        if fmt == ct.BF16:
            assert abs((K - 1) * lo * lo) >= 2.0 ** 23.9
            d = tb.reference(fmt, A, B, ea, eb).view(np.float32)
            base = np.float32(np.ldexp(float((K - 1) * lo * lo), ea + eb))
            for i, (k, sign) in enumerate(cases):
                # the small addend is exactly one ulp of a result just below 2^24 (times the scale)
                assert d[i, i] != base and abs(float(d[i, i]) - float(base)) == float(np.spacing(base)), (name, i)


@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_walsh_tile_cancels_to_exact_zeros_after_climbing(fmt):
    K, hi = ct.K[fmt], ct.HI[fmt]
    A, B, ea, eb = dict(cc.crafted_tiles(fmt))["walsh"]
    partial = _sums(A, B)
    s = partial[:, :, -1]
    p, q = cc.walsh_rows(fmt)
    same = p[:, None] == q[None, :]
    assert np.all(s[same] == -K * hi * hi) and np.all(s[~same] == 0)
    assert same.any() and (~same).any()
    zero_peak = np.abs(partial[~same]).max(axis=-1)
    assert zero_peak.max() == (K // 2) * hi * hi                     # climbs to (K / 2) hi^2 and comes back
    d = tb.reference(fmt, A, B, ea, eb)
    assert np.all(d[~same] == 0)                                        # +0


# ---- corruption plans -------------------------------------------------------------------------------------------------
def _changed_threads(fmt, clean, bad):
    """{tile: threads whose check value differs} between two lists of TILES (A, B, ea, eb)."""
    out = {}
    for t in range(ct.TILES):
        c0 = ct.fold(ct.fragments(tb.reference(fmt, *clean[t])))
        c1 = ct.fold(ct.fragments(tb.reference(fmt, *bad[t])))
        if not np.array_equal(c0, c1):
            out[t] = set(np.flatnonzero(c0 != c1).tolist())
    return out


@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_every_corruption_changes_a_check_value_and_together_they_cover_everything(fmt):
    flips = cc.check_flips()
    assert {t for _, t, _ in flips} == set(range(ct.THREADS)) and {tile for tile, _, _ in flips} == set(range(ct.TILES))
    assert all(mask and mask & (mask - 1) == 0 for _, _, mask in flips)
    covered = {(tile, t) for tile, t, _ in flips}

    clean = cc.generator_tiles(fmt)
    warps, steps = set(), set()
    for plan in cc.operand_plan(fmt):
        tile, op, row, k = plan
        bad = cc.corrupt_operands(fmt, clean, [plan])
        changed = _changed_threads(fmt, clean, bad)
        assert list(changed) == [tile], (plan, changed)
        warps |= {t // 32 for t in changed[tile]}
        steps.add(k // tb.STEP_K[fmt])
        covered |= {(tile, t) for t in changed[tile]}
        if op == 0:                                   # a wrong A row is seen by the warp that owns that result row
            assert {t // 32 for t in changed[tile]} == {row // 16}
    assert warps == {0, 1, 2, 3}
    assert {0, tb.STEPS[fmt] - 1} <= steps
    assert {row for _, op, row, _ in cc.operand_plan(fmt) if op == 1} == {0, ct.N - 1}
    assert {tile for tile, *_ in cc.operand_plan(fmt)} == {0, 3, 7}

    bad = cc.corrupt_operands(fmt, clean, cc.TWO_TILE_PLAN)
    assert sorted(_changed_threads(fmt, clean, bad)) == sorted(t for t, *_ in cc.TWO_TILE_PLAN)

    crafted = [t for _, t in cc.crafted_tiles(fmt)]
    for case in cc.one_unit_cases(fmt):
        bad = cc.one_unit_corruption(fmt, crafted, case)
        changed = _changed_threads(fmt, crafted, bad)
        assert list(changed) == [cc.LATE_TILE] and changed[cc.LATE_TILE], case
    assert {t for _, t in covered} == set(range(ct.THREADS)) and {tile for tile, _ in covered} == set(range(ct.TILES))


@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_one_unit_corruption_moves_a_result_by_one_unit_near_the_top(fmt):
    K, lo = ct.K[fmt], ct.LO[fmt]
    crafted = [t for _, t in cc.crafted_tiles(fmt)]
    cases = cc.one_unit_cases(fmt)
    assert {cc.late_cases(fmt)[i] for i in cases} == {(K - 1, 1), (K - 1, -1)}   # the last k of the last step
    A, B, ea, eb = crafted[cc.LATE_TILE]
    assert (ea, eb) == (0, 0)
    for case in cases:
        A1, B1, _, _ = cc.one_unit_corruption(fmt, crafted, case)[cc.LATE_TILE]
        s0, s1 = A @ B.T, A1 @ B1.T
        diff = np.argwhere(s0 != s1)
        assert (abs(s0[case, case] - s1[case, case]), s1[case, case]) == (1, (K - 1) * lo * lo)
        assert [case, case] in diff.tolist()
        if fmt == ct.BF16:
            d0, d1 = tb.reference(fmt, A, B).view(np.float32), tb.reference(fmt, A1, B1).view(np.float32)
            assert float(d1[case, case]) >= 2.0 ** 23.9
            assert abs(int(d0.view(np.uint32)[case, case]) - int(d1.view(np.uint32)[case, case])) == 1  # one ulp
