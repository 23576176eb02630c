"""CPU side of the on-demand integer and warp-exchange self-test (b2dp_int_test): the host arithmetic in
csrc/int_test_math.hpp against the independent restatement in tests/int_test_oracle.py -- the operand tables, the
crafted classes, fault models of the integer pipes and the lane-exchange network, and the fold -- then the backends
without the test, the daemon's flag, the header and the SASS the kernels assemble to.  No GPU needed."""
import os
import re
import shutil
import signal
import subprocess
import time

import pytest

import fake_sysfs
import int_test_oracle as it
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
SEEDS = [0, 1, 0xC0FFEE17, 0xFFFFFFFF]
FORMATS = (it.MAD, it.BIT, it.WARP)
FMT_IDS = ["mad", "bit", "warp"]
M32 = it.M32


class MathDriver:
    """tests/native/int_test_math_test.cpp, compiled with g++ against csrc/int_test_math.hpp."""

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
    exe = str(tmp_path_factory.mktemp("it") / "int_test_math_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                        os.path.join(ROOT, "tests", "native", "int_test_math_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = MathDriver(exe)
    yield d
    d.close()


# ---- the tables ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", SEEDS)
def test_host_tables_words_and_checks_match_the_oracle(drv, seed, fmt):
    nt, nw = it.SLOTS[fmt] * it.THREADS, it.WORDS[fmt] * it.THREADS
    for tile in range(it.TILES):
        v = [int(x) for x in drv.ask("tile", seed, fmt, tile)]
        assert len(v) == nt + nw + it.THREADS
        assert v[:nt] == it.table(seed, fmt, tile), (tile, "table")
        want = [x for t in it.tile_words(seed, fmt, tile) for x in t]
        diff = [i for i in range(nw) if v[nt + i] != want[i]]
        assert not diff, (tile, len(diff), diff[0] // it.WORDS[fmt],
                          it.WORD_NAMES[fmt][diff[0] % it.WORDS[fmt] % it.SET_WORDS[fmt]])
        assert v[nt + nw:] == it.tile_checks(seed, fmt, tile), (tile, "checks")


def test_layout(drv):
    v = drv.ask("bounds")
    for f in FORMATS:
        sets, ss, sw, slots, words, tbytes, ops = (int(x) for x in v[7 * f:7 * f + 7])
        assert (sets, ss, sw, slots, words) == (it.SETS[f], it.SET_SLOTS[f], it.SET_WORDS[f], it.SLOTS[f], it.WORDS[f])
        assert tbytes == slots * it.THREADS * 4 and ops == it.THREADS * words
        assert len(it.WORD_NAMES[f]) == sw


# ---- the crafted classes, recognised from the table ---------------------------------------------------------------------------
def _has(sets, pred):
    return any(pred(*s) for s in sets)


@pytest.mark.parametrize("seed", [0, 0xC0FFEE17])
def test_every_mad_class_is_in_every_thread_of_every_tile(seed):
    pairs = set()
    runs = set()
    for tile in range(it.TILES):
        for t, sets in enumerate(it.tile_operands(seed, it.MAD, tile)):
            assert _has(sets, lambda a, b, c, d: a == b == M32), "0xFFFFFFFF squared"
            assert _has(sets, lambda a, b, c, d: a == b == 0x80000000)
            for m in (0, 1, M32):
                assert _has(sets, lambda a, b, c, d: b == m and a not in (0, 1, M32, 0x80000000)), "x %x" % m
            one = [(a, b) for a, b, c, d in sets[5:6]]
            assert all(a & (a - 1) == 0 and b & (b - 1) == 0 and a and b for a, b in one)
            pairs.add((one[0][0].bit_length() - 1, one[0][1].bit_length() - 1))
            assert _has(sets, lambda a, b, c, d: (a, b) == (0x55555555, 0xAAAAAAAA))
            # an addend whose low word carries into mad.wide's high word, and one that wraps all 64 bits
            assert _has(sets, lambda a, b, c, d: (a * b & M32) + c == 1 << 32)
            assert _has(sets, lambda a, b, c, d: a * b + (d << 32 | c) >= 1 << 64 and (a * b + (d << 32 | c)) & it.M64 < 128)
            # carry pairs: a carry that runs k bits and stops, through all 32 bits, a borrow through all 32, none
            run = [a for a, b, c, d in sets[9:10] if c == 1 and a & (a + 1) == 0 and a]
            assert run
            runs.add(run[0].bit_length())
            assert _has(sets, lambda a, b, c, d: a == M32 and c == 1)
            assert _has(sets, lambda a, b, c, d: a == 0 and c == 1)
            assert _has(sets, lambda a, b, c, d: a + c < 1 << 32 and (a, c) == (0x55555555, 0x2AAAAAAA))
            # dp4a extremes in one byte lane alone and in all four, with an accumulator that wraps
            lane = [a.bit_length() // 8 for a, b, c, d in sets if a == b and a in [0x80 << 8 * k for k in range(4)]
                    and c >= 0xFFFFC000]
            assert lane, "(-128)(-128) alone, wrapping"
            assert _has(sets, lambda a, b, c, d: a in [0x80 << 8 * k for k in range(4)] and b == a // 0x80 * 0xFF)
            assert _has(sets, lambda a, b, c, d: a == b and a in [0xFF << 8 * k for k in range(4)] and c >= 0xFFFFFF00)
            assert _has(sets, lambda a, b, c, d: (a, b, c) == (0x80808080, 0x80FF80FF, M32))
            assert sum(1 for s in sets[16:] if all(x not in (0, M32) for x in s)) == 4, "random sets"
    assert pairs == {(i, j) for i in range(32) for j in range(32)}, "every partial-product column pair over a round"
    assert runs == set(range(1, 33))


@pytest.mark.parametrize("seed", [0, 0xC0FFEE17])
def test_every_bit_class_is_in_every_thread_of_every_tile(seed):
    amounts, sel = set(), [set() for _ in range(4)]
    for tile in range(it.TILES):
        for t, sets in enumerate(it.tile_operands(seed, it.BIT, tile)):
            a, b, c = sets[0]                               # lop3: all 8 input combinations at every bit position
            assert {(a >> k & 1, b >> k & 1, c >> k & 1) for k in range(32)} == {(x, y, z) for x in (0, 1) for y in (0, 1)
                                                                               for z in (0, 1)}
            assert all({(a >> (k + d) % 32 & 1, b >> (k + d) % 32 & 1, c >> (k + d) % 32 & 1) for d in range(8)}
                       .__len__() == 8 for k in range(32))
            one = [(x, z) for x, y, z in sets if x and x & (x - 1) == 0 and z < 32 and y and y & (y - 1) == 0]
            zero = [(x, z) for x, y, z in sets if (x ^ M32) and (x ^ M32) & ((x ^ M32) - 1) == 0 and 32 <= z < 64]
            assert one and zero, "walking one with an amount 0..31, walking zero with an amount 32..63"
            amounts.add((one[0][0].bit_length() - 1, one[0][1]))
            assert _has(sets, lambda x, y, z: x not in (0, M32) and x & (x - 1) and (z < 64 if tile % 2 == 0 else True))
            for v in (0, M32):                               # popc / bfind / brev of 0 and ~0; clz (of b) likewise
                assert _has(sets, lambda x, y, z: x == v) and _has(sets, lambda x, y, z: y == v)
            assert _has(sets, lambda x, y, z: y and y & (y - 1) == 0) and _has(sets, lambda x, y, z: (y ^ M32) and
                                                                             (y ^ M32) & ((y ^ M32) - 1) == 0)
            for p in range(4):
                sel[p].add(sets[6][2] >> 4 * p & 15)
            assert _has(sets, lambda x, y, z: (x, y) == (0x80000000, 0x7FFFFFFF))       # INT_MIN, INT_MAX
            assert _has(sets, lambda x, y, z: (x, y) == (0, M32))                       # 0, -1
            assert _has(sets, lambda x, y, z: x == y and x not in (0, M32))             # equal operands
            assert _has(sets, lambda x, y, z: x < y and it.s32(x) > it.s32(y) and x not in (0,))  # order differs
            assert _has(sets, lambda x, y, z: z + abs(x - y) > M32)                      # sad wraps
    assert amounts == {(i, j) for i in range(32) for j in range(32)}, "every bit at every amount over a round"
    assert all(s == set(range(16)) for s in sel), "every selector value in every position"
    big = {it.tile_operands(seed, it.BIT, tile)[t][3][2] >> 6 != 0 for tile in (1, 3) for t in range(it.THREADS)}
    assert True in big, "amounts beyond 6 bits"


@pytest.mark.parametrize("seed", [0, 0xC0FFEE17])
def test_every_warp_class_is_in_every_warp_of_every_tile(seed):
    V, B, C, Q, R, MA, M2 = range(7)
    lanes, masks, bits, deltas = set(), set(), set(), {32: set(), 16: set(), 8: set()}
    for tile in range(it.TILES):
        ops = it.tile_operands(seed, it.WARP, tile)
        for w in range(4):
            L = it.warp_lane(tile, w)
            lanes.add(L)
            col = lambda s, k: [ops[w * 32 + l][s][k] for l in range(32)]   # noqa: E731
            width = lambda s: 32 - (col(s, C)[0] >> 8 & 31)                   # noqa: E731
            distinct = [s for s in range(it.SETS[it.WARP]) if len(set(col(s, V))) == 32]
            assert len(distinct) >= 9, "distinct-value-per-lane backgrounds"
            bg = [col(s, V) for s in range(it.SETS[it.WARP])]
            assert any(len(set(v)) == 1 and v[0] in (0, M32) for v in bg), "solid"
            assert any(v == [0xAAAAAAAA if l & 1 else 0x55555555 for l in range(32)] for v in bg), "checkerboard"
            assert any(v == [1 << l for l in range(32)] for v in bg), "walking one per lane"
            srcs = [col(s, B) for s in distinct]
            assert list(range(32)) in srcs and list(range(31, -1, -1)) in srcs, "identity, reverse"
            assert any(v != list(range(32)) and sorted(v) == list(range(32)) and len({(v[l] - l) % 32 for l in range(32)})
                       == 1 for v in srcs), "rotation"
            assert [L] * 32 in srcs, "broadcast"
            assert any(len(set(v)) < 32 and len(set(v)) > 1 and max(v) < 32 for v in srcs), "random non-permutation"
            assert any(min(v) >= 32 for v in srcs), "sources >= 32"
            for s in range(it.SETS[it.WARP]):
                b = col(s, B)
                assert len(set(col(s, C))) == 1 and col(s, C)[0] & 0x1F == 0x1F and width(s) in (32, 16, 8)
                if len(set(b)) == 1 and b[0] < 32 and s in distinct:
                    deltas[width(s)].add(b[0])
                if len(set(b)) == 1 and 1 <= b[0] < 32 and s not in distinct:
                    masks.add(b[0])
            q = [sum((x != 0) << l for l, x in enumerate(col(s, Q))) for s in range(it.SETS[it.WARP])]
            assert 0 in q and M32 in q and 1 << L in q and M32 ^ 1 << L in q, "ballot classes"
            assert any(x not in (0, M32, 1 << L, M32 ^ 1 << L) for x in q), "random ballot"
            r = [col(s, R) for s in range(it.SETS[it.WARP])]
            assert any(min(range(32), key=lambda l: it.s32(v[l])) == L and v[L] == 0x80000000 and max(v) == v[L]
                       for v in r), "min.s32 / max.u32 extreme in lane L"
            assert any(max(range(32), key=lambda l: it.s32(v[l])) == L and v[L] == 0x7FFFFFFF and min(v) == v[L]
                       for v in r), "max.s32 / min.u32 extreme in lane L"
            assert any(sum(v) > M32 for v in r), "add wraps"
            one_bit = [v for v in r if len(set(v)) == 2 and sorted(map(v.count, set(v))) == [1, 31]]
            assert len(one_bit) == 2
            for v in one_bit:
                (odd,) = [x for x in set(v) if v.count(x) == 1]
                (base,) = [x for x in set(v) if v.count(x) == 31]
                assert v[L] == odd and bin(odd ^ base).count("1") == 1
                bits.add((odd ^ base).bit_length() - 1)
            groups = [sorted(col(s, MA).count(x) for x in set(col(s, MA))) for s in range(it.SETS[it.WARP])]
            for g in ([32], [1] * 32, [2] * 16, [4] * 8, [16] * 2):
                assert g in groups, ("match.any groups", g)
            m2 = [col(s, M2) for s in range(it.SETS[it.WARP])]
            assert any(len(set(v)) == 1 for v in m2), "match.all equal"
            assert any(len(set(v)) == 2 and v.count(v[L]) == 1 for v in m2), "match.all with one lane different"
    assert lanes == set(range(32)) and bits == set(range(32))
    assert masks == set(range(1, 32)), "every bfly lane mask"
    assert all(d == set(range(32)) for d in deltas.values()), "every delta at widths 32, 16 and 8"


# ---- fault models ---------------------------------------------------------------------------------------------------------
# (format, model, every): `every` = every thread of every tile catches it at both seeds; otherwise every tile still
# catches it, in the threads whose operands reach the fault.
FAULTS = [(it.MAD, ("column", c), c != 62) for c in (0, 5, 31, 32, 40, 62)] + \
         [(it.MAD, ("carry", k), k != 63) for k in (1, 16, 32, 33, 63)] + \
         [(it.MAD, ("mulhi_unsigned",), True), (it.MAD, ("dp4a_sign", (True, True), 0), True),
          (it.MAD, ("dp4a_sign", (True, False), 3), True), (it.MAD, ("dp4a_sign", (False, False), 2), True),
          (it.MAD, ("dp4a_sat",), True)] + \
         [(it.BIT, ("lop3_minterm", m), True) for m in range(8)] + \
         [(it.BIT, ("shift_stage", s), s != 5) for s in range(6)] + \
         [(it.BIT, ("popc_off", b), True) for b in (0, 17, 31)] + \
         [(it.BIT, ("clz0",), True), (it.BIT, ("brev_bytes",), True)] + \
         [(it.BIT, ("prmt_route", v), v == 15) for v in (0, 7, 8, 15)] + [(it.BIT, ("cmp_swapped",), True)] + \
         [(it.WARP, ("lane_swap", 3, 20), False), (it.WARP, ("bit_dropped", 9, 13), False),
          (it.WARP, ("segment_ignored",), False), (it.WARP, ("pred_true",), True), (it.WARP, ("ballot_miss", 5), True),
          (it.WARP, ("redux_skip", 13), True), (it.WARP, ("match_miss", 7), False)]


@pytest.mark.parametrize("fmt,fault,every", FAULTS, ids=["-".join(str(x) for x in f[1]).replace(" ", "") for f in FAULTS])
def test_fault_model_is_caught_in_every_tile(fmt, fault, every):
    for seed in (1, 0xC0FFEE17):
        for tile in range(it.TILES):
            good, bad = it.tile_checks(seed, fmt, tile), it.tile_checks(seed, fmt, tile, fault)
            n = sum(g != b for g, b in zip(good, bad))
            assert n > 0, (seed, tile, "no thread catches the model: a gap in the classes")
            if every:
                assert n == it.THREADS, (seed, tile, n)


# ---- the fold -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_one_wrong_word_at_any_position_changes_the_check(drv, fmt):
    words = it.tile_words(5, fmt, 2)[77]
    base = it.fold(words)
    assert int(drv.ask("fold", len(words), *words)[0]) == base
    for j in range(len(words)):
        for mask in [1 << b for b in (0, 1, 7, 15, 16, 30, 31)] + [M32, 0x80000001, 0x00010000, words[j] or 1]:
            bad = list(words)
            bad[j] ^= mask
            assert it.fold(bad) != base, (j, hex(mask))
    bad = list(words)
    bad[3] ^= 0x1234
    assert int(drv.ask("fold", len(bad), *bad)[0]) == it.fold(bad)


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_two_words_wrong_in_bit_31_are_caught_where_the_weighted_sum_is_blind(fmt):
    words = it.tile_words(5, fmt, 0)[0]
    n = len(words)
    pairs = [(0, 1), (0, 4), (3, 7), (2, n - 2), (n - 5, n - 1), (8, 12)]     # same chain and different chains
    for i, j in pairs:
        bad = list(words)
        bad[i] ^= 1 << 31
        bad[j] ^= 1 << 31
        assert it.old_fold(bad) == it.old_fold(words), "the odd-weighted sum cancels two bit-31 errors"
        assert it.fold(bad) != it.fold(words), (i, j)
    for i in range(0, n - 4, 9):                                                # every chain, neighbours in a chain
        bad = list(words)
        bad[i] ^= 1 << 31
        bad[i + 4] ^= 1 << 31
        assert it.fold(bad) != it.fold(words), i


# ---- ABI, backends, daemon, CLI --------------------------------------------------------------------------------------------
def test_header_and_bindings(pkg):
    N = pkg._native
    assert (N.IT_MAD, N.IT_BIT, N.IT_WARP) == (0, 1, 2)
    assert N.SIGNATURES["b2dp_int_test"] == N.SIGNATURES["b2dp_compute_test"]
    hdr = open(os.path.join(ROOT, "include", "b200dp.h")).read()
    for name, v in (("B2DP_IT_MAD", 0), ("B2DP_IT_BIT", 1), ("B2DP_IT_WARP", 2)):
        assert re.search(r"#define %s %s\b" % (name, v), hdr), name
    assert re.search(r"B2DP_API int b2dp_int_test\(b2dp_ctx \*ctx, int device, const b2dp_compute_test_opts \*opts,\s+"
                     r"b2dp_compute_test_result \*out, int cap, int \*n\);", hdr)
    assert "#define B2DP_ABI_VERSION 3" in hdr
    cli = open(os.path.join(ROOT, "tools", "b200dp_cli.cpp")).read()
    assert "int_test [duration_ms]" in cli and "tresults_mad=%.2f" in cli and "tresults_warp=%.2f" in cli


def test_backends_without_an_int_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.int_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:      # cuda:probe=off (NVML only)
        with pytest.raises(N.B2dpError) as ei:
            ctx.int_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "in-process only" in str(ei.value)
        assert "integer self-test" in str(ei.value)


def test_daemon_int_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-int_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "int test at start not run: not supported by this backend" in err, err[-2000:]
    assert "Failed to start plugin gpu: Register:" in err


# ---- SASS -----------------------------------------------------------------------------------------------------------------
# Opcode -> count inside the repetition loop, per format: 20 / 12 / 12 operand sets, every op once per set.
SETS_MAD, SETS_BIT, SETS_WARP = it.SETS
SASS_EXACT = {
    it.MAD: {"IMAD.HI.U32": SETS_MAD, "IMAD.HI": SETS_MAD, "IMAD.WIDE.U32": SETS_MAD, "IMAD.WIDE": SETS_MAD,
             "IDP.4A.S8.S8": SETS_MAD, "IDP.4A.S8.U8": SETS_MAD, "IDP.4A.U8.U8": SETS_MAD},
    it.BIT: {"SHF.R.W.U32": SETS_BIT, "SHF.R.S32.HI": SETS_BIT, "SHF.L.U32": SETS_BIT, "POPC": SETS_BIT,
             "FLO.U32": 2 * SETS_BIT, "FLO": SETS_BIT, "BREV": SETS_BIT, "PRMT": SETS_BIT, "VIMNMX": 2 * SETS_BIT,
             "VIMNMX.U32": 2 * SETS_BIT, "VABSDIFF.U32": SETS_BIT},
    it.WARP: {"SHFL.IDX": SETS_WARP, "SHFL.UP": SETS_WARP, "SHFL.DOWN": SETS_WARP, "SHFL.BFLY": SETS_WARP,
              "VOTE.ANY": SETS_WARP, "REDUX.SUM": SETS_WARP, "REDUX.MIN.S32": SETS_WARP, "REDUX.MAX.S32": SETS_WARP,
              "REDUX.MIN": SETS_WARP, "REDUX.MAX": SETS_WARP, "REDUX": SETS_WARP, "REDUX.OR": SETS_WARP,
              "REDUX.XOR": SETS_WARP, "MATCH.ANY": SETS_WARP, "MATCH.ALL": SETS_WARP},
}
ROT = 3                                   # the fold's rotations are SHF.L.W.U32.HI too: one per word and three to combine


@pytest.mark.parametrize("dump", [0, 1], ids=["product", "dump"])
@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_sass_has_the_planned_ops_per_repetition(fmt, dump, lib=None):
    """Inside the repetition loop -- found by its own back-edge, the first backward branch after the compare's
    BAR.RED.OR -- exactly the planned count of every opcode under test, no
    local memory and no spill.  The tile and round loops also enclose the ops, so "some loop around them" would still
    hold if ptxas hoisted an op out of the repetition loop and repeated only the fold."""
    lib = lib or os.path.join(ROOT, "tests", "native", "libint_test_kernels_test.so")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib) or not os.path.exists(tool):
        pytest.skip("needs the built harness and cuobjdump")
    sass = subprocess.run([tool, "-sass", lib], capture_output=True, text=True).stdout
    (body,) = [p for p in re.split(r"\n\s+Function : ", sass)[1:]
               if "int_selftestILi%dELb%dE" % (fmt, dump) in p.split("\n")[0]]
    ins = [(int(a, 16), re.sub(r"^@!?U?P\w+\s+", "", i.strip()))
           for a, i in re.findall(r"/\*([0-9a-f]{4,5})\*/\s+([^;]*);", body)]
    bar = min(a for a, i in ins if "BAR.RED.OR" in i)
    back = [(a, int(m.group(1), 16)) for a, i in ins for m in [re.search(r"BRA\S* (?:\S+, )?(?:`\()?0x([0-9a-f]+)", i)]
            if m and int(m.group(1), 16) < a and a > bar]
    src, tgt = min(back)
    inside, whole = {}, {}
    for a, i in ins:
        op = i.split()[0]
        whole[op] = whole.get(op, 0) + 1
        if tgt <= a <= src:
            inside[op] = inside.get(op, 0) + 1
    for op, n in SASS_EXACT[fmt].items():
        assert inside.get(op, 0) == n, (op, inside.get(op, 0), n)
        # nowhere else either, where nothing else in the kernel needs the opcode (addressing multiplies and shifts;
        # the divergent-warp fallback ptxas emits behind BRA.DIV repeats the warp ops once, cold)
        if op.startswith(("IDP", "POPC", "FLO", "BREV", "VIMNMX", "VABSDIFF")):
            assert whole[op] == n, (op, "also outside the repetition loop", whole[op])
    assert inside.get("SHF.L.W.U32.HI", 0) == it.WORDS[fmt] + ROT + (SETS_BIT if fmt == it.BIT else 0)
    if fmt == it.MAD:
        # mad.lo next to the fold's own multiplies; add.cc / sub.cc and the two mad.wide addends as IADD3 with a carry
        # out, each consumed by one IMAD.X or IADD3.X (ptxas picks either); + 2 for the 64-bit tallies
        assert inside.get("IMAD", 0) >= it.WORDS[fmt] + SETS_MAD
        carry_out = [i for a, i in ins if tgt <= a <= src and re.match(r"IADD3 R\d+, P\d", i)]
        assert len(carry_out) == 4 * SETS_MAD + 2, len(carry_out)
        assert inside.get("IMAD.X", 0) + inside.get("IADD3.X", 0) == 4 * SETS_MAD + 2
    if fmt == it.WARP:                      # the source lane / delta / mask and the c operand come from registers
        shfl = [i for a, i in ins if tgt <= a <= src and i.startswith("SHFL.")]
        assert shfl and all(re.match(r"SHFL\.\w+ P\d, R\d+, R\d+, R\d+, R\d+$", i.strip()) for i in shfl), shfl[:4]
    if fmt == it.BIT:
        luts = {}
        for a, i in ins:
            m = re.search(r"LOP3\.LUT .*, (0x[0-9a-f]+), !?PT", i)
            if m and tgt <= a <= src:
                luts[int(m.group(1), 16)] = luts.get(int(m.group(1), 16), 0) + 1
        for imm in it.LOP3_IMM:
            assert luts.get(imm, 0) >= SETS_BIT, (hex(imm), luts)
    assert not any(op.startswith(("STL", "LDL")) for op in whole), "local memory"
    usage = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True).stdout
    m = re.search(r"int_selftestILi%dELb%dE[^\n]*\n\s*REG:(\d+)[^\n]*?LOCAL:(\d+)" % (fmt, dump), usage)
    assert m, usage[-500:]
    assert int(m.group(2)) == 0 and int(m.group(1)) <= (255 if fmt == it.WARP and not dump else 128), m.groups()
