"""CPU side of the on-demand half-precision and conversion self-test (b2dp_half_test): the host arithmetic in
csrc/half_test_math.hpp against the independent restatement in tests/half_test_oracle.py -- the operand tables, the
crafted classes, fault models of the 16-bit pipes and the converters, and the double-rounded reference it must not be --
then the backends without the test, the daemon's flag, the header and the SASS the kernels assemble to.  No GPU
needed."""
import os
import re
import shutil
import signal
import subprocess
import time
from fractions import Fraction

import pytest

import fake_sysfs
import half_test_oracle as hp
from test_int_test_cpu import MathDriver
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
SEEDS = [0, 1, 0xC0FFEE17, 0xFFFFFFFF]
FORMATS = (hp.F16, hp.BF16, hp.CVT)
FMT_IDS = ["f16", "bf16", "cvt"]


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("hp") / "half_test_math_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                        os.path.join(ROOT, "tests", "native", "half_test_math_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = MathDriver(exe)
    yield d
    d.close()


# ---- the tables ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", SEEDS)
def test_host_tables_words_and_checks_match_the_oracle(drv, seed, fmt):
    nt, nw = hp.SLOTS[fmt] * hp.THREADS, hp.WORDS[fmt] * hp.THREADS
    for tile in range(hp.TILES):
        v = [int(x) for x in drv.ask("tile", seed, fmt, tile)]
        assert len(v) == nt + nw + hp.THREADS
        assert v[:nt] == hp.table(seed, fmt, tile), (tile, "table")
        want = [x for t in hp.tile_words(seed, fmt, tile) for x in t]
        diff = [i for i in range(nw) if v[nt + i] != want[i]]
        assert not diff, (tile, len(diff), diff[0] // hp.WORDS[fmt],
                          hp.WORD_NAMES[fmt][diff[0] % hp.WORDS[fmt] % hp.SET_WORDS[fmt]])
        assert v[nt + nw:] == hp.tile_checks(seed, fmt, tile), (tile, "checks")


def test_layout(drv):
    v = drv.ask("bounds")
    for f in FORMATS:
        sets, ss, sw, slots, words, tbytes, ops = (int(x) for x in v[7 * f:7 * f + 7])
        assert (sets, ss, sw, slots, words) == (hp.SETS[f], hp.SET_SLOTS[f], hp.SET_WORDS[f], hp.SLOTS[f], hp.WORDS[f])
        assert tbytes == slots * hp.THREADS * 4 and ops == hp.THREADS * words
        assert len(hp.WORD_NAMES[f]) == sw


# ---- the crafted classes, recognised from the table -----------------------------------------------------------------
def _value(bits, fmt):
    s, v = hp.decode(bits, fmt)
    return v if isinstance(v, str) else (-v if s else v)


def _half_classes(fmt):
    """Predicates over one lane (a, b, c) or (x, y, z) that recognise each crafted class from its operands."""
    ft = hp.FMT_F16 if fmt == hp.F16 else hp.FMT_BF16
    sub = lambda h: (h >> ft[1]) & ((1 << ft[0]) - 1) == 0 and h & ((1 << ft[1]) - 1)    # noqa: E731
    val = lambda h: _value(h, ft)                                                          # noqa: E731

    def exact(a, b, c):    # None when an operand is infinite or NaN
        v = [val(a), val(b), val(c)]
        return None if any(isinstance(x, str) for x in v) else v[0] * v[1] + v[2]

    def rounds_to(a, b, c):
        return hp.decode(hp.fma_lane(a, b, c, ft), ft)

    def tie(a, b, c, up):
        q = exact(a, b, c)
        if not q:
            return False
        r = hp.round_value(0, abs(q), ft, "rz")
        _, lo = hp.decode(r, ft)
        _, hi = hp.decode(r + 1, ft)
        return not isinstance(hi, str) and abs(q) == (lo + hi) / 2 and (r & 1) == up

    def double_round(a, b, c):
        return hp.fma_lane(a, b, c, ft) != hp.fma_lane(a, b, c, ft, fault="double_round")

    def sticky(a, b, c):
        return hp.fma_lane(a, b, c, ft) != hp.fma_lane(a, b, c, ft, fault="sticky_lost")
    abc = {
        "tie_down": lambda a, b, c: tie(a, b, c, 0), "tie_up": lambda a, b, c: tie(a, b, c, 1),
        "cancel": lambda a, b, c: val(c) != 0 and 0 < abs(exact(a, b, c)) < abs(val(c)) / 256,
        "subnormal_result": lambda a, b, c: sub(hp.fma_lane(a, b, c, ft)) and not sub(a),
        "subnormal_multiplicand": lambda a, b, c: sub(a) and hp.fma_lane(a, b, c, ft, "ftz") !=
        hp.fma_lane(a, b, c, ft),
        "overflow_pos": lambda a, b, c: rounds_to(a, b, c) == (0, hp.INF),
        "overflow_neg": lambda a, b, c: rounds_to(a, b, c) == (1, hp.INF),
        "neg_zero": lambda a, b, c: hp.fma_lane(a, b, c, ft) == 1 << (ft[0] + ft[1]),
        "pos_zero": lambda a, b, c: hp.fma_lane(a, b, c, ft) == 0 and (a | c) == 0 and b >> (ft[0] + ft[1]),
        "sticky": sticky, "double_round": double_round,
        "ftz_result": lambda a, b, c: not sub(a) and sub(hp.fma_lane(a, b, c, ft)) and
        hp.fma_lane(a, b, c, ft, "ftz") == 0,
    }
    one = val(((1 << (ft[0] - 1)) - 1) << ft[1])
    xyz = {
        "above_one": lambda x, y, z: isinstance(exact(x, y, z), Fraction) and exact(x, y, z) > one,
        "negative": lambda x, y, z: isinstance(exact(x, y, z), Fraction) and exact(x, y, z) < 0,
        "neg_zero_relu": lambda x, y, z: hp.fma_lane(x, y, z, ft) == 1 << (ft[0] + ft[1]),
        "one_nan": lambda x, y, z: (val(x) == hp.NAN) != (val(y) == hp.NAN),
        "two_nans": lambda x, y, z: val(x) == val(y) == hp.NAN,
        "inf": lambda x, y, z: val(x) == hp.INF and val(y) != hp.NAN and val(z) != hp.INF,
        "inf_minus_inf": lambda x, y, z: val(x) == hp.INF and val(z) == hp.INF and (x ^ z) >> (ft[0] + ft[1]),
        "signed_zeros": lambda x, y, z: {x, y} == {0, 1 << (ft[0] + ft[1])},
        "inside": lambda x, y, z: isinstance(exact(x, y, z), Fraction) and 0 < exact(x, y, z) < one,
        "exactly_one": lambda x, y, z: isinstance(exact(x, y, z), Fraction) and exact(x, y, z) == one,
    }
    return abc, xyz


@pytest.mark.parametrize("fmt", (hp.F16, hp.BF16), ids=FMT_IDS[:2])
@pytest.mark.parametrize("seed", [0, 0xC0FFEE17])
def test_every_half_class_is_in_every_thread_of_every_tile(seed, fmt):
    abc, xyz = _half_classes(fmt)
    if fmt == hp.BF16:
        del xyz["above_one"], xyz["inside"], xyz["exactly_one"]      # no .sat on bf16: the classes still run .relu
    for tile in range(hp.TILES):
        for t, sets in enumerate(hp.tile_operands(seed, fmt, tile)):
            lanes = [[(w >> sh) & 0xFFFF for w in s] for s in sets[:hp.CRAFTED[fmt]] for sh in (0, 16)]
            for name, pred in abc.items():
                assert any(pred(*ln[:3]) for ln in lanes), (tile, t, name)
            for name, pred in xyz.items():
                assert any(pred(*ln[3:]) for ln in lanes), (tile, t, name)
            for s in sets[:hp.CRAFTED[fmt]]:                            # the two lanes of every word differ
                assert all((w & 0xFFFF) != (w >> 16) for w in s[:3]) or s[0] != s[1]
            assert len(sets) - hp.CRAFTED[fmt] == 6, "random sets"


def test_every_cvt_class_is_in_every_thread_of_every_tile():
    F32, F64 = hp.FMT_F32, hp.FMT_F64
    for seed in (0, 0xC0FFEE17):
        for tile in range(hp.TILES):
            for t, sets in enumerate(hp.tile_operands(seed, hp.CVT, tile)):
                c = sets[:hp.CRAFTED[hp.CVT]]
                xy = {w for s in c for w in s[:2]}
                pq = {w for s in c for w in s[2:4]}
                hh = {w >> sh & 0xFFFF for s in c for sh in (0, 16) for w in (s[hp.H],)}
                assert set(hp.CVT_XY) <= xy and set(hp.CVT_PQ) <= pq and set(hp.CVT_H) <= hh
                assert {s[hp.F] for s in c} == set(hp.CVT_F) and {s[hp.I] for s in c} == set(hp.CVT_I)
                assert {s[hp.DHI] << 32 | s[hp.DLO] for s in c} == set(hp.CVT_D)
                assert {s[hp.LHI] << 32 | s[hp.LLO] for s in c} == set(hp.CVT_L)
                for s in c:                                              # the two lanes of every pair differ
                    assert s[hp.X] != s[hp.Y] and s[hp.P] != s[hp.Q] and s[hp.H] >> 16 != s[hp.H] & 0xFFFF
    # and the lists hold what the classes are for
    v = lambda b: _value(b, F32)                                             # noqa: E731
    for fmt in (hp.FMT_F16, hp.FMT_BF16):                                    # ties in both directions, every target
        for mode in ("rn",):
            ties = [x for x in hp.CVT_XY if hp.cvt_float(x, F32, fmt, mode) != hp.cvt_float(x, F32, fmt, "rz") and
                    hp.cvt_float(x, F32, fmt, "rp") == hp.cvt_float(x, F32, fmt, "rn")]
            assert ties
    assert {hp.cvt_float(x, F32, hp.FMT_F16, "rn") for x in (0x477FF000, 0xC7800000)} == {0x7C00, 0xFC00}
    assert hp.cvt_float(0x477FF000, F32, hp.FMT_F16, "rz") == 0x7BFF
    assert hp.cvt_float(0x43F00000, F32, hp.FMT_E4M3, "rn", True) == 0x7E                 # 480 -> 448
    assert hp.cvt_float(0x47700000, F32, hp.FMT_E5M2, "rn", True) == 0x7B                 # 61440 -> 57344
    assert [hp.cvt_float(x, F32, hp.FMT_E4M3, "rn", True) for x in (0x7F800000, 0xFF800000, 0x7FC00001)] == \
        [0x7E, 0xFE, 0x7F]
    assert [hp.cvt_float(x, F32, hp.FMT_E4M3, "rn", True) for x in (0x3A800000, 0x3A800001, 0x3A7FFFFF)] == [0, 1, 0]
    assert [hp.cvt_float(x, F32, hp.FMT_E5M2, "rn", True) for x in (0x37000000, 0x36FFFFFF)] == [0, 0]
    assert hp.cvt_float(0x0081, hp.FMT_F16, hp.FMT_E5M2, "rn", True) == 1
    s32 = {f: [hp.f2i(f, F32, m, 32, True) for m in hp.MODES] for f in hp.CVT_F}
    u32 = {f: [hp.f2i(f, F32, m, 32, False) for m in hp.MODES] for f in hp.CVT_F}
    assert s32[0x4F000000] == [0x7FFFFFFF] * 4 and u32[0x4F800000] == [M32] * 4 and s32[0x7FC00000] == [0] * 4
    assert u32[0xBF000000] == [0] * 4 and s32[0x40200000] == [2, 2, 2, 3] and s32[0x3FC00000] == [2, 1, 1, 2]
    assert s32[0xBF000000] == [0, 0, M32, 0] and s32[0x3F000000] == [0, 0, 0, 1]
    s64 = {d: [hp.f2i(d, F64, m, 64, True) for m in hp.MODES] for d in hp.CVT_D}
    assert s64[0x43E0000000000000] == [(1 << 63) - 1] * 4 and s64[0xC3E0000000000000] == [1 << 63] * 4
    i2f = {i: [hp.i2f(i, 32, True, F32, m) for m in hp.MODES] for i in hp.CVT_I}
    assert v(i2f[0x01000001][0]) == 1 << 24 and v(i2f[0x01000001][3]) == (1 << 24) + 2     # just above 2^24
    d53 = [hp.i2f(0x0020000000000001, 64, True, F64, m) for m in hp.MODES]
    assert _value(d53[0], F64) == 1 << 53 and _value(d53[3], F64) == (1 << 53) + 2          # just above 2^53
    u = [hp.i2f(0x8000010000000001, 64, False, F32, m) for m in hp.MODES]
    assert v(u[1]) < v(u[3])                                                                 # above 2^63, inexact
    big = [hp.cvt_float(0x47F0000000000001, F64, F32, m) for m in hp.MODES]
    assert big == [0x7F800000, 0x7F7FFFFF, 0x7F7FFFFF, 0x7F800000]                           # rn, rz, rm, rp
    assert [hp.cvt_float(0xC7F0000000000001, F64, F32, m) for m in hp.MODES] == \
        [0xFF800000, 0xFF7FFFFF, 0xFF800000, 0xFF7FFFFF]
    assert 0 < hp.cvt_float(0x3738000000000001, F64, F32, "rn") < 0x00800000                # an f32 subnormal
    assert [hp.frnd(x, F32, "rn") for x in (0xC0200000, 0x3FC00000, 0xBF000000, 0x4B000001)] == \
        [0xC0000000, 0x40000000, 0x80000000, 0x4B000001]                                     # halfway and integral
    assert hp.frnd(0x8000000000000001, F64, "rm") == 0xBFF0000000000000


M32 = hp.M32


# ---- fault models -----------------------------------------------------------------------------------------------------
# (format, model): each is one wrong unit behaviour; every tile's checks must change.
FAULTS = [(hp.F16, "lane_swap"), (hp.F16, "rz"), (hp.F16, "sticky_lost"), (hp.F16, "ftz_everywhere"),
          (hp.F16, "sat_ignored"), (hp.F16, "relu_ignored"), (hp.F16, "ftz_ignored"), (hp.F16, "double_round"),
          (hp.BF16, "lane_swap"), (hp.BF16, "rz"), (hp.BF16, "sticky_lost"), (hp.BF16, "ftz_everywhere"),
          (hp.BF16, "relu_ignored"), (hp.BF16, "double_round"),
          (hp.CVT, "rz"), (hp.CVT, "satfinite_ignored"), (hp.CVT, "relu_ignored"), (hp.CVT, "fp8_order"),
          (hp.CVT, "f2i_wraps"), (hp.CVT, "nan_not_zero"), (hp.CVT, "f2i_trunc"), (hp.CVT, "i2f_rn"),
          (hp.CVT, "frnd_trunc")]


@pytest.mark.parametrize("fmt,fault", FAULTS, ids=["%s-%s" % (FMT_IDS[f], m) for f, m in FAULTS])
def test_fault_model_is_caught_in_every_tile(fmt, fault):
    for seed in (1, 0xC0FFEE17):
        for tile in range(hp.TILES):
            good, bad = hp.tile_checks(seed, fmt, tile), hp.tile_checks(seed, fmt, tile, fault)
            n = sum(g != b for g, b in zip(good, bad))
            assert n > 0, (seed, tile, "no thread catches the model: a gap in the classes")
            if fault in ("double_round", "sticky_lost", "lane_swap", "fp8_order", "nan_not_zero", "f2i_wraps"):
                assert n == hp.THREADS, (seed, tile, n)       # a crafted class in every thread


def test_the_double_rounded_reference_disagrees_with_the_oracle():
    """(half)fmaf(a, b, c) rounds twice; the trap class makes it differ from the one correctly rounded result."""
    for fmt, ft in ((hp.F16, hp.FMT_F16), (hp.BF16, hp.FMT_BF16)):
        a, b, c = (hp.ABC_F16 if fmt == hp.F16 else hp.ABC_BF16)[hp.HALF_CLASSES.index("double_round")]
        good, bad = hp.fma_lane(a, b, c, ft), hp.fma_lane(a, b, c, ft, fault="double_round")
        assert good != bad and good + 1 == bad, (hex(good), hex(bad))
        assert hp.tile_words(0, fmt, 0) != hp.tile_words(0, fmt, 0, "double_round")


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_one_wrong_word_at_any_position_changes_the_check(drv, fmt):
    words = hp.tile_words(5, fmt, 2)[77]
    base = hp.fold(words)
    assert int(drv.ask("fold", len(words), *words)[0]) == base
    for j in range(len(words)):
        for mask in (1, 1 << 15, 1 << 16, 1 << 31, M32):
            bad = list(words)
            bad[j] ^= mask
            assert hp.fold(bad) != base, (j, hex(mask))


# ---- ABI, backends, daemon, CLI ------------------------------------------------------------------------------------
def test_header_and_bindings(pkg):
    N = pkg._native
    assert (N.HP_F16, N.HP_BF16, N.HP_CVT) == (0, 1, 2)
    assert N.SIGNATURES["b2dp_half_test"] == N.SIGNATURES["b2dp_compute_test"]
    hdr = open(os.path.join(ROOT, "include", "b200dp.h")).read()
    for name, v in (("B2DP_HP_F16", 0), ("B2DP_HP_BF16", 1), ("B2DP_HP_CVT", 2)):
        assert re.search(r"#define %s %s\b" % (name, v), hdr), name
    assert re.search(r"B2DP_API int b2dp_half_test\(b2dp_ctx \*ctx, int device, const b2dp_compute_test_opts \*opts,\s+"
                     r"b2dp_compute_test_result \*out, int cap, int \*n\);", hdr)
    assert "#define B2DP_ABI_VERSION 3" in hdr
    cli = open(os.path.join(ROOT, "tools", "b200dp_cli.cpp")).read()
    assert "half_test [duration_ms]" in cli and "tresults_f16=%.2f" in cli and "tresults_cvt=%.2f" in cli


def test_backends_without_a_half_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.half_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:      # cuda:probe=off (NVML only)
        with pytest.raises(N.B2dpError) as ei:
            ctx.half_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "in-process only" in str(ei.value)
        assert "half-precision self-test" in str(ei.value)


def test_mig_backend_has_no_half_test(pkg, monkeypatch, stub, tmp_path):  # noqa: F811
    N = pkg._native
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 3) as ctx:
        with pytest.raises(N.B2dpError) as ei:
            ctx.half_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "in-process only" in str(ei.value)


def test_daemon_half_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-half_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "half test at start not run: not supported by this backend" in err, err[-2000:]
    assert "Failed to start plugin gpu: Register:" in err


# ---- SASS ----------------------------------------------------------------------------------------------------------------
# Opcode family -> count inside the repetition loop per operand set.  What each PTX form became (DESIGN.md §4.14):
# add.rn.f16x2 / .bf16x2 -> HADD2; sub.rn -> HFMA2.MMA a, 1, 1, -b; fma.rn.f16x2 -> HFMA2.MMA, .relu -> HFMA2.MMA.RELU,
# .sat -> HFMA2.SAT, .ftz -> HFMA2.FTZ; cvt.{rn,rz}.f32.s32 -> I2FP, cvt.{rm,rp}.f32.s32 -> I2F.
PER_SET = {
    hp.F16: {"HFMA2": 5, "HADD2": 1, "HMUL2": 1, "HMNMX2": 5},
    hp.BF16: {"HFMA2": 3, "HADD2": 1, "HMUL2": 1, "HMNMX2": 4},
    hp.CVT: {"F2FP": 15, "F2F": 8, "F2I": 12, "I2F": 10, "I2FP": 2, "FRND": 2},
}
FAMILIES = ("HFMA2", "HADD2", "HMUL2", "HMNMX2", "F2FP", "F2F", "F2I", "I2F", "I2FP", "FRND")


@pytest.mark.parametrize("dump", [0, 1], ids=["product", "dump"])
@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_sass_has_the_planned_ops_per_repetition(fmt, dump):
    """Inside the repetition loop -- found by its own back-edge, the first backward branch after the compare's
    BAR.RED.OR -- exactly the planned count of every opcode family under test, none of them anywhere else, and no
    local memory or spill."""
    lib = os.path.join(ROOT, "tests", "native", "libhalf_test_kernels_test.so")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib) or not os.path.exists(tool):
        pytest.skip("needs the built harness and cuobjdump")
    sass = subprocess.run([tool, "-sass", lib], capture_output=True, text=True).stdout
    (body,) = [p for p in re.split(r"\n\s+Function : ", sass)[1:]
               if "half_selftestILi%dELb%dE" % (fmt, dump) in p.split("\n")[0]]
    ins = [(int(a, 16), re.sub(r"^@!?U?P\w+\s+", "", i.strip()))
           for a, i in re.findall(r"/\*([0-9a-f]{4,5})\*/\s+([^;]*);", body)]
    bar = min(a for a, i in ins if "BAR.RED.OR" in i)
    back = [(a, int(m.group(1), 16)) for a, i in ins for m in [re.search(r"BRA\S* (?:\S+, )?(?:`\()?0x([0-9a-f]+)", i)]
            if m and int(m.group(1), 16) < a and a > bar]
    src, tgt = min(back)
    inside, whole = {}, {}
    for a, i in ins:
        fam = i.split()[0].split(".")[0]
        whole[fam] = whole.get(fam, 0) + 1
        if tgt <= a <= src:
            inside[fam] = inside.get(fam, 0) + 1
    for fam in FAMILIES:
        n = PER_SET[fmt].get(fam, 0) * hp.SETS[fmt]
        assert inside.get(fam, 0) == n and whole.get(fam, 0) == n, (fam, inside.get(fam, 0), whole.get(fam, 0), n)
    assert not any(op.startswith(("STL", "LDL")) for op in whole), "local memory"
    usage = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True).stdout
    m = re.search(r"half_selftestILi%dELb%dE[^\n]*\n\s*REG:(\d+)[^\n]*?LOCAL:(\d+)" % (fmt, dump), usage)
    assert m, usage[-500:]
    assert int(m.group(2)) == 0 and int(m.group(1)) <= 255, m.groups()
