"""CPU side of the on-demand FP32 / FP64 self-test (b2dp_fp_test): the host arithmetic in csrc/fp_test_math.hpp against
the exact restatement in tests/fp_test_oracle.py; the crafted operand classes; the single-bit guarantee of the fold;
the injection experiment behind the kernel's independent FMAs; the bounds; the backends without the test; the daemon's
flag; and the SASS the kernels assemble to.  No GPU needed."""
import os
import re
import shutil
import signal
import subprocess
import time

import numpy as np
import pytest

import fake_sysfs
import fp_test_oracle as ft
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
# 87917, 71720 and 67507: the first seeds with a DMMA tile scaled by (2^480, 2^480), (2^-480, 2^-480) and
# (2^480, 2^-480) (fp_test_edges.corner_seed)
SEEDS = [0, 1, 0xC0FFEE17, 0xFFFFFFFF, 87917, 71720, 67507]
FMT_IDS = [ft.NAMES[f] for f in ft.FORMATS]


class MathDriver:
    """tests/native/fp_test_math_test.cpp, compiled with g++ against csrc/fp_test_math.hpp."""

    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(self, *words):
        self.p.stdin.write(" ".join(str(w) for w in words) + "\n")
        self.p.stdin.flush()
        return self.p.stdout.readline().split()

    def close(self):
        self.p.stdin.close()
        self.p.wait(timeout=10)


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("ft") / "fp_test_math_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                        os.path.join(ROOT, "tests", "native", "fp_test_math_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = MathDriver(exe)
    yield d
    d.close()


# ---- the host against the oracle --------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ft.FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", SEEDS)
def test_host_tables_results_and_checks_match_the_oracle(drv, seed, fmt):
    """Every operand, every result word of every thread and every check value of every tile, bit for bit."""
    for t in range(ft.TILES):
        got = [int(x) for x in drv.ask("tile", seed, fmt, t)]
        table, words, checks, _ = ft.tile(seed, fmt, t)
        want = [v for row in table for v in row] + [w for ws in words for w in ws] + checks
        assert len(got) == len(want) and got == want, (t, next(i for i, (a, b) in enumerate(zip(got, want)) if a != b))


def test_host_cost_is_milliseconds(drv):
    ms = min(float(drv.ask("time", s)[0]) for s in (1, 2, 3))
    print("host tables of one b2dp_fp_test call: %.2f ms" % ms)
    assert ms < 200


# ---- crafted classes ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [ft.FP32, ft.FP64], ids=FMT_IDS[:2])
@pytest.mark.parametrize("seed", [0, 0xC0FFEE17])
def test_every_tile_has_every_crafted_class_in_every_thread(seed, fmt):
    """The oracle classifies each crafted result from its exact value: every thread of every tile holds every class."""
    for t in range(ft.TILES):
        for th in range(ft.THREADS):
            x, a, b = ft.fma_thread(seed, fmt, t, th)
            for c, name in enumerate(ft.CLASSES):
                k = (2 * c + th) % ft.NAB
                got = ft.classify(fmt, x[ft.CLASS_X[c]], a[k], b[k])
                assert name in got, (t, th, name, got)


def test_crafted_classes_are_what_they_claim():
    """Spot values: a tie both ways, +0 and -0 bits, a subnormal, a 24-bit cancellation."""
    f = ft.FP32
    one, half_ulp = ft.make(f, 0, 0, 1), ft.make(f, 0, -24, 0)       # 1 + 2^-23 (odd) and 2^-24
    assert ft.fma(f, one, ft.make(f, 0, 0, 0), half_ulp) == ft.make(f, 0, 0, 2)      # tie -> even, away
    two = ft.make(f, 0, 0, 2)                                                         # 1 + 2^-22 (even)
    assert ft.fma(f, two, ft.make(f, 0, 0, 0), half_ulp) == two                       # tie -> even, toward
    assert ft.fma(f, one, ft.make(f, 1, 0, 0), one) == 0                              # x a = -b: +0
    assert ft.fma(f, one, 1 << 31, 1 << 31) == 1 << 31                                # -0 + -0: -0
    assert ft.fma(f, ft.make(f, 0, -100, 0), ft.make(f, 0, -40, 0), 0) == 1 << 9      # 2^-140: subnormal
    assert ft.fma(f, 0x3F800001, 0x3F800001, ft.mul(f, 0x3F800001, 0x3F800001) ^ (1 << 31)) == ft.make(f, 0, -46, 0)


# ---- the fold -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ft.FORMATS, ids=FMT_IDS)
def test_every_single_bit_flip_of_every_result_changes_the_check(fmt):
    """Exhaustive for one thread of one tile: every result word, every bit (an FP64 result is two words)."""
    _, words, checks, _ = ft.tile(0xC0FFEE17, fmt, 3)
    w = np.array(words[77], dtype=np.uint64)
    base = checks[77]
    assert ft.fold(words[77]) == base
    weights = 2 * np.arange(len(w), dtype=np.uint64) + 1
    for j in range(len(w)):
        for b in range(32):
            y = w.copy()
            y[j] ^= np.uint64(1 << b)
            assert int((y * weights).sum() & np.uint64(ft.M32)) != base, (j, b)


def test_fold_matches_the_host(drv):
    rng = np.random.default_rng(7)
    for n in (32, 128, 256):
        for _ in range(5):
            w = rng.integers(0, 1 << 32, n, dtype=np.uint64).tolist()
            assert int(drv.ask("fold", n, *w)[0]) == ft.fold(w)


# ---- why every FMA result is compared: the injection experiment -----------------------------------------------------------
def _chain_lost(a_lo, a_hi, steps=1024, pairs=16, stride=7, seed=1):
    """A dependent chain x <- fma(x, a_i, b_i) in binary32, one bit flipped after one step: for each bit, how many of the
    injected steps leave the final x unchanged.  (The chain is a numerical model of a design the kernel does not use:
    each step is rounded through float64, which equals an FMA but for rare double roundings.)"""
    rng = np.random.default_rng(seed)
    a = (rng.uniform(a_lo, a_hi, pairs) * rng.choice([-1, 1], pairs)).astype(np.float32)
    b = rng.uniform(-1, 1, pairs).astype(np.float32)
    where = np.arange(0, steps, stride)
    n = len(where) * 32
    x = np.full(n + 1, 0.3, dtype=np.float32)                     # column n: the fault-free chain
    step = np.repeat(where, 32)
    bit = np.tile(np.arange(32, dtype=np.uint32), len(where))
    for i in range(steps):
        x = (x.astype(np.float64) * a[i % pairs] + b[i % pairs]).astype(np.float32)
        hit = np.nonzero(step == i)[0]
        if len(hit):
            v = x.view(np.uint32)
            v[hit] ^= np.uint32(1) << bit[hit]
    final = x.view(np.uint32)
    lost = (final[:n] == final[n]).reshape(len(where), 32).sum(axis=0)
    return lost, len(where)


def test_a_dependent_fma_chain_loses_most_single_bit_errors():
    with np.errstate(over="ignore", invalid="ignore"):
        lost, total = _chain_lost(0.5, 1.0)
        lost2, _ = _chain_lost(0.9, 1.1)
    assert total == 147
    # |a| in [0.5, 1): the chain contracts, and most flips at every bit position are forgotten (the top exponent bit,
    # which sends x out of range, least often)
    assert (np.delete(lost, 30) >= 0.9 * total).all() and lost[30] > 0, lost.tolist()
    # |a| near 1: the low mantissa bits are still lost in many cases
    assert lost2[0] >= total // 2 and (lost2[:4] > 0).all(), lost2.tolist()
    print("chain |a| in [0.5,1): lost per bit", lost.tolist())
    print("chain |a| in [0.9,1.1): lost per bit", lost2.tolist())


def dmma_chain_survivors(seed=0x5EED, tile=1):
    """The DMMA K chain (d <- d + A_s B_s over 4 steps, binary64) with one bit flipped in an intermediate accumulator
    after step 0, 1 or 2: per (step, bit), how many of the 4 sets x 4 warps x 128 elements still end different."""
    ea, eb = ft.dmma_scale_exp(seed, tile, 0), ft.dmma_scale_exp(seed, tile, 1)
    out = np.zeros((3, 64), dtype=np.int64)
    total = 0
    for w in range(4):
        _, steps, _, _ = ft.dmma_exact(seed, tile, w)
        for c in range(ft.DMMA_SETS):
            parts = [np.ldexp(p.astype(np.float64), ea + eb) for p in steps[c]]   # exact: |p| < 2^53
            ref = parts[0] + parts[1] + parts[2] + parts[3]
            total += ref.size
            for s in range(3):
                d = parts[0].copy()
                for q in range(1, s + 1):
                    d = d + parts[q]
                for b in range(64):
                    e = (d.view(np.uint64) ^ np.uint64(1 << b)).view(np.float64)
                    for q in range(s + 1, 4):
                        e = e + parts[q]
                    out[s, b] += int((e.view(np.uint64) != ref.view(np.uint64)).sum())
    return out, total


def test_dmma_k_chain_keeps_high_intermediate_flips_and_rounds_away_some_low_ones():
    """The DMMA chain keeps every flip of bits 16-63 of an intermediate accumulator: its partial sums are exact
    integers, so such a change carries into the final value.  A flip of one of the lowest mantissa bits of a small
    intermediate adds a fraction below the integer grid, which a later, larger sum can round away.  DESIGN.md §4.7
    records this table."""
    with np.errstate(over="ignore", invalid="ignore"):
        surv, total = dmma_chain_survivors()
    assert total == 4 * 4 * 128
    for s in range(3):
        print("DMMA K chain, flip after step %d: survivors of %d at bits 0-15: %s" % (s, total, surv[s, :16].tolist()))
    assert (surv[:, 16:] == total).all(), surv
    assert (surv[:, 0] < total).all() and (np.diff(surv[:, :16], axis=1) >= -1).all(), surv[:, :16]


# ---- bounds ---------------------------------------------------------------------------------------------------------------
def test_bounds_mirror_the_static_asserts(drv):
    nx, nab, k, mx, se, w32, w64, wd, sx = (int(v) for v in drv.ask("bounds"))
    assert (nx, nab, k, mx, se) == (ft.NX, ft.NAB, ft.DMMA_K, ft.DMMA_MAX, ft.DMMA_SCALE_EXP)
    assert (w32, w64, wd, sx) == (ft.WORDS[ft.FP32], ft.WORDS[ft.FP64], ft.WORDS[ft.DMMA], ft.SUBNORMAL_X_EXP)
    assert k * mx * mx < 1 << 53 and (k - 8) * mx * mx > 1 << 52
    assert 2 * se + 53 < 1024 and -2 * se > -1022
    for fmt in (ft.FP32, ft.FP64):
        W, M, BIAS, EMIN, XE, AE, BS = ft.BIN[fmt]
        assert XE + AE + M + 2 < BIAS and AE + BS < BIAS and -(XE + AE + M + 1) > EMIN
    for seed in (0, 0xFFFFFFFF):      # the extreme rows of the DMMA operands take sums above 2^52, all below 2^53
        for t in (0, 3):
            D, steps, _, _ = ft.dmma_exact(seed, t, t % 4)
            for c in range(ft.DMMA_SETS):
                assert np.abs(D[c][0]).min() > 1 << 52 and np.abs(D[c]).max() < 1 << 53
                prefix = np.cumsum(np.stack(steps[c]), axis=0)
                assert np.abs(prefix).max() < 1 << 53


# ---- ABI, backends, daemon, SASS ----------------------------------------------------------------------------------------
def test_backends_without_an_fp_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    assert (N.FT_FP32, N.FT_FP64, N.FT_DMMA) == (0, 1, 2)
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.fp_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:      # cuda:probe=off (NVML only)
        with pytest.raises(N.B2dpError) as ei:
            ctx.fp_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "in-process only" in str(ei.value)


def test_daemon_fp_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-fp_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "fp test at start not run: not supported by this backend" in err, err[-2000:]
    assert "Failed to start plugin gpu: Register:" in err


def test_sass_has_the_planned_instructions_per_repetition():
    """The harness's product instantiations: 128 FFMA (none .FTZ), 128 DFMA and 16 DMMA.16x8x16, each inside the
    repetition loop (between its head and the backward branch), so nothing was hoisted or merged."""
    lib = os.path.join(ROOT, "tests", "native", "libfp_test_kernels_test.so")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib) or not os.path.exists(tool):
        pytest.skip("needs the built harness and cuobjdump")
    sass = subprocess.run([tool, "-sass", lib], capture_output=True, text=True).stdout
    funcs = {}
    for part in re.split(r"\n\s+Function : ", sass)[1:]:
        funcs[part.split("\n")[0].strip()] = part
    want = {0: ("FFMA", 128), 1: ("DFMA", 128), 2: ("DMMA.16x8x16", 16)}
    for fmt, (op, n) in want.items():
        (body,) = [b for name, b in funcs.items() if "fp_selftestILi%dELb0E" % fmt in name]
        ins = re.findall(r"/\*([0-9a-f]{4})\*/\s+([^;]*);", body)
        at = [int(a, 16) for a, i in ins if re.search(r"\b%s\b" % re.escape(op), i)]
        assert len(at) == n, (op, len(at))
        assert not any(".FTZ" in i for _, i in ins if "FFMA" in i)
        # the innermost loop holding them branches back to an address at or before the first
        back = [(int(a, 16), int(m.group(1), 16)) for a, i in ins for m in [re.search(r"BRA (?:`\()?0x([0-9a-f]+)", i)] if m]
        assert any(tgt <= min(at) and src > max(at) for src, tgt in back), (op, back)
