"""CPU side of the on-demand tensor-core self-test (b2dp_compute_test): the host arithmetic in
csrc/compute_test_math.hpp -- generator, encodings, exact GEMM, per-thread comparison values, verdict -- against
tests/compute_test_oracle.py; the exactness bounds; the single-bit guarantee of the comparison; the ABI structs against
gcc; the backends without the test; the daemon's flag.  No GPU needed."""
import ctypes
import os
import random
import shutil
import signal
import subprocess
import time

import numpy as np
import pytest

import compute_test_oracle as ct
import fake_sysfs
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
SEEDS = [0, 1, 0xC0FFEE17, 0xFFFFFFFF]
FMT_IDS = [ct.NAMES[f] for f in ct.FORMATS]


class MathDriver:
    """tests/native/compute_test_math_test.cpp, compiled with g++ against csrc/compute_test_math.hpp."""

    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(self, *words):
        self.p.stdin.write(" ".join(str(w) for w in words) + "\n")
        self.p.stdin.flush()
        return self.p.stdout.readline().split()

    def ints(self, *words):
        return np.array([int(x) for x in self.ask(*words)], dtype=np.int64)

    def close(self):
        self.p.stdin.close()
        self.p.wait(timeout=10)


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("ct") / "compute_test_math_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                        os.path.join(ROOT, "tests", "native", "compute_test_math_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = MathDriver(exe)
    yield d
    d.close()


# ---- generator and encodings ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", SEEDS)
def test_operands_match_oracle(drv, seed, fmt):
    for tile in (0, 3, ct.TILES - 1):
        for op in (0, 1):
            got = drv.ints("operand", seed, fmt, tile, op)
            want = ct.operand(seed, fmt, tile, op)
            assert got[0] == ct.scale_exp(seed, fmt, tile, op), (tile, op)
            assert np.array_equal(got[1:], want.ravel()), (tile, op)
            assert want.min() >= ct.LO[fmt] and want.max() <= ct.HI[fmt]


def test_generator_covers_the_ranges():
    """Random operands reach both ends of every range, and the BF16 scale exponents reach +-30."""
    for fmt in ct.FORMATS:
        vals = np.unique(np.concatenate([ct.operand(s, fmt, t, 1)[8:].ravel() for s in (0, 1) for t in range(ct.TILES)]))
        assert vals[0] == ct.LO[fmt] and vals[-1] == ct.HI[fmt] and len(vals) == ct.HI[fmt] - ct.LO[fmt] + 1
    exps = {ct.scale_exp(s, ct.BF16, t, op) for s in range(200) for t in range(ct.TILES) for op in (0, 1)}
    assert exps == set(range(-ct.SCALE_EXP, ct.SCALE_EXP + 1))
    assert {ct.scale_exp(s, f, 0, 0) for s in range(20) for f in (ct.FP8, ct.INT8)} == {0}


@pytest.mark.parametrize("fmt,e", [(ct.BF16, -30), (ct.BF16, 0), (ct.BF16, 30), (ct.FP8, 0), (ct.INT8, 0)])
def test_encodings_match_oracle_and_are_exact(drv, fmt, e):
    v = np.arange(ct.LO[fmt], ct.HI[fmt] + 1)
    got = drv.ints("encode", fmt, e)
    want = ct.encode(fmt, v, e)
    assert np.array_equal(got, want)
    if fmt == ct.BF16:
        back = (want.astype(np.uint32) << np.uint32(16)).view(np.float32).astype(np.float64)
        assert np.array_equal(back, np.ldexp(v.astype(np.float64), e))
    elif fmt == ct.FP8:
        assert [ct.decode_e4m3(int(b)) for b in want] == [float(x) for x in v]
        assert ct.encode(fmt, np.array([0, 1, 15, -15]))[[1, 2, 3]].tolist() == [0x38, 0x57, 0xD7]
    else:
        assert np.array_equal(want.astype(np.uint8).view(np.int8), v)


# ---- the exact GEMM and the comparison values -------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", SEEDS)
def test_reference_tiles_and_check_values_match_oracle(drv, seed, fmt):
    n = ct.M * ct.N
    for t in range(ct.TILES):
        got = drv.ints("tile", seed, fmt, t)
        _, _, _, _, d, checks = ct.tile(seed, fmt, t)
        assert np.array_equal(got[:n], d.ravel()), t
        assert np.array_equal(got[n:], checks), t


@pytest.mark.parametrize("ea,eb", [(30, 30), (-30, -30), (30, -30), (-30, 29)])
def test_scaled_bf16_reference_at_the_exponent_extremes(drv, ea, eb):
    for seed in (0, 0xFFFFFFFF):
        A, B = ct.operand(seed, ct.BF16, 1, 0), ct.operand(seed, ct.BF16, 1, 1)
        want = ct.reference(ct.BF16, A, B, ea, eb)
        assert np.array_equal(drv.ints("scaled", seed, ct.BF16, 1, ea, eb), want.ravel())
        exact = (A @ B.T).astype(np.float64) * 2.0 ** (ea + eb)
        assert np.array_equal(want.view(np.float32).astype(np.float64), exact)


BOUND = {ct.BF16: 1 << 24, ct.FP8: 1 << 13, ct.INT8: 1 << 31}


@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_partial_sums_stay_below_the_bound_and_results_survive_float32(fmt):
    worst = ct.K[fmt] * max(-ct.LO[fmt], ct.HI[fmt]) ** 2
    assert worst < BOUND[fmt] or (fmt == ct.INT8 and worst == 1 << 22)
    for seed in (0, 0xFFFFFFFF):
        for t in (0, ct.TILES - 1):
            A, B = ct.operand(seed, fmt, t, 0), ct.operand(seed, fmt, t, 1)
            partial = np.cumsum(A[:, None, :] * B[None, :, :], axis=2)      # M x N x K, every prefix of every element
            assert np.abs(partial).max() < BOUND[fmt]
            s = partial[:, :, -1]
            # the extreme rows take row 0 of the result to at least (K - 2) / K of the worst case
            assert np.abs(s[0, :8]).min() >= (ct.K[fmt] - 2) * ct.LO[fmt] ** 2
            if fmt != ct.INT8:
                ea, eb = ct.scale_exp(seed, fmt, t, 0), ct.scale_exp(seed, fmt, t, 1)
                f = ct.reference(fmt, A, B, ea, eb).view(np.float32)
                assert np.array_equal(f.astype(np.float64), np.ldexp(s.astype(np.float64), ea + eb))


def test_fragment_map_is_a_permutation():
    rows, cols = ct.frag_index()
    assert sorted(zip(rows.ravel().tolist(), cols.ravel().tolist())) == [(m, n) for m in range(ct.M) for n in range(ct.N)]


def test_every_single_bit_flip_changes_the_check_value():
    """Exhaustive for one tile: every thread, every one of its 64 elements, every bit 0..31."""
    x = ct.fragments(ct.tile(0xC0FFEE17, ct.BF16, 0)[4])              # THREADS x ACC
    base = ct.fold(x)
    for j in range(ct.ACC):
        for b in range(32):
            y = x.copy()
            y[:, j] ^= np.uint32(1 << b)
            assert np.all(ct.fold(y) != base), (j, b)


def test_fold_matches_oracle(drv):
    rng = np.random.default_rng(5)
    for _ in range(20):
        x = rng.integers(0, 1 << 32, ct.ACC, dtype=np.uint64).astype(np.uint32)
        assert int(drv.ask("fold", *x.tolist())[0]) == int(ct.fold(x))
    assert int(drv.ask("fold", *([0xFFFFFFFF] * ct.ACC))[0]) == int(ct.fold(np.full(ct.ACC, 0xFFFFFFFF, np.uint32)))


# ---- verdict ----------------------------------------------------------------------------------------------------------
FULL = ct.TILES * ct.REPS


def _rec(f, rounds=2, comparisons=None, mismatches=0, seq=None):
    return (f + 1 if seq is None else seq, rounds, rounds * FULL if comparisons is None else comparisons, mismatches)


def _ask_verdict(drv, ok, records):
    words = [int(ok)] + [len(records[f]) for f in ct.FORMATS]
    for f in ct.FORMATS:
        for r in records[f]:
            words += list(r)
    return drv.ask("verdict", *words)[0] == "1"


VERDICT_TABLE = [
    ("clean", True, {}, True),
    ("launch_failed", False, {}, False),
    ("mismatch_bf16", True, {0: [_rec(0, mismatches=1)]}, False),
    ("mismatch_int8", True, {2: [_rec(2, mismatches=3)]}, False),
    ("record_missing", True, {1: [_rec(1, seq=0)]}, False),
    ("stale_seq", True, {0: [_rec(0, seq=2)]}, False),
    ("no_round", True, {2: [_rec(2, rounds=0, comparisons=0)]}, False),
    ("short_round", True, {1: [_rec(1, rounds=3, comparisons=3 * FULL - 1)]}, False),
    ("extra_comparison", True, {0: [_rec(0, rounds=1, comparisons=FULL + 1)]}, False),
    ("one_round_only", True, {0: [_rec(0, rounds=1)]}, True),
    ("no_ctas", True, {1: None}, False),
]


@pytest.mark.parametrize("name,ok,override,want", VERDICT_TABLE, ids=[v[0] for v in VERDICT_TABLE])
def test_verdict_matches_oracle(drv, name, ok, override, want):
    records = {f: [_rec(f), _rec(f, rounds=5)] for f in ct.FORMATS}
    for f, recs in override.items():
        records[f] = [] if recs is None else records[f] + recs
    assert ct.healthy(ok, records, {f: f + 1 for f in ct.FORMATS}) is want
    assert _ask_verdict(drv, ok, records) is want


def test_verdict_random_table(drv):
    rng = random.Random(11)
    for _ in range(200):
        records = {}
        for f in ct.FORMATS:
            records[f] = []
            for _ in range(rng.choice([0, 1, 3])):
                rounds = rng.choice([0, 1, 4])
                records[f].append((rng.choice([f + 1, f + 1, f + 1, 0]), rounds,
                                   rounds * FULL + rng.choice([0, 0, 0, -1, 1]), rng.choice([0, 0, 0, 1])))
        ok = rng.random() > .1
        want = ct.healthy(ok, records, {f: f + 1 for f in ct.FORMATS})
        assert _ask_verdict(drv, ok, records) is want


# ---- ABI, backends, daemon --------------------------------------------------------------------------------------------
def test_struct_layouts_match_the_c_header(pkg, tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    N = pkg._native
    pairs = [("b2dp_compute_test_opts", N.ComputeTestOpts), ("b2dp_compute_test_result", N.ComputeTestResult)]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200dp.h"', 'int main(void) {']
    for cname, ctyp in pairs:
        src.append('printf("%s %%zu", sizeof(%s));' % (cname, cname))
        for fname, _ in ctyp._fields_:
            src.append('printf(" %s=%%zu", offsetof(%s, %s));' % (fname, cname, fname))
        src.append('printf("\\n");')
    src += ['printf("%u %u %u %u %u\\n", B2DP_RES_COMPUTE, B2DP_CT_EVEN_IF_BUSY, B2DP_CT_SKIPPED_BUSY, '
            'B2DP_CT_PARTIAL_COVERAGE, B2DP_CT_INT8);', 'return 0; }']
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = str(tmp_path / "layout")
    r = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([exe], capture_output=True, text=True).stdout.splitlines()
    for line, (cname, ctyp) in zip(out, pairs):
        parts = line.split()
        assert parts[0] == cname and int(parts[1]) == ctypes.sizeof(ctyp)
        for tok, (fname, _) in zip(parts[2:], ctyp._fields_):
            k, v = tok.split("=")
            assert k == fname and int(v) == getattr(ctyp, fname).offset, (cname, fname)
    assert [int(x) for x in out[2].split()] == [N.RES_COMPUTE, N.CT_EVEN_IF_BUSY, N.CT_SKIPPED_BUSY,
                                                 N.CT_PARTIAL_COVERAGE, N.CT_INT8] == [0x400, 1, 1, 2, 2]
    assert ctypes.sizeof(N.ComputeTestOpts) == 24 and ctypes.sizeof(N.ComputeTestResult) == 128


def test_backends_without_a_compute_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.compute_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:      # cuda:probe=off (NVML only)
        with pytest.raises(N.B2dpError) as ei:
            ctx.compute_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "in-process only" in str(ei.value)


def test_daemon_compute_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    """-compute_test_at_start=1 parses; on a backend without the test the daemon logs that and carries on."""
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-compute_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "compute test at start not run: not supported by this backend" in err, err[-2000:]
    assert "Failed to start plugin gpu: Register:" in err          # and the daemon went on to serve
