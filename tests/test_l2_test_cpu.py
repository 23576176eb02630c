"""CPU side of the on-demand L2 self-test (b2dp_l2_test): the host arithmetic in csrc/l2_test_math.hpp against the
independent restatement in tests/l2_test_oracle.py, faulty-L2 models of the marches and the atomic units, the
backends without the test, the daemon's flag, the header and the SASS the kernels assemble to.  No GPU needed."""
import os
import re
import shutil
import signal
import subprocess
import time

import numpy as np
import pytest

import fake_sysfs
import l2_test_oracle as lo
import smem_test_oracle as so
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
SEEDS = [0, 1, 0xC0FFEE17, 0xFFFFFFFF]
M32 = lo.M32


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("l2") / "l2_test_math_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                        os.path.join(ROOT, "tests", "native", "l2_test_math_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(*words):
        p.stdin.write(" ".join(str(w) for w in words) + "\n")
        p.stdin.flush()
        return [int(x) for x in p.stdout.readline().split()]
    yield ask
    p.stdin.close()
    p.wait(timeout=10)


# ---- the tables -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", SEEDS)
def test_march_tables_and_checks_match_the_oracle(drv, seed):
    for fmt in (lo.WORD, lo.BYTE):
        for t in range(lo.TILES):
            got = drv("tile", seed, fmt, t)
            table, checks = lo.tile(seed, fmt, t)
            assert got[:lo.TABLE_WORDS] == table.tolist() and got[lo.TABLE_WORDS:] == checks.tolist(), (fmt, t)


@pytest.mark.parametrize("seed", SEEDS)
def test_atom_tables_match_the_oracle(drv, seed):
    for t in (0, 3, 7):
        got = np.array(drv("tile", seed, lo.ATOM, t), np.uint32)
        F, X = lo.finals(seed, t)
        assert np.array_equal(got[:lo.SLOTS * lo.MAX_N].reshape(lo.SLOTS, lo.MAX_N), np.array(X, np.uint32))
        off = lo.SLOTS * lo.MAX_N
        assert np.array_equal(got[off:off + lo.SLOTS * (lo.MAX_N + 1)].reshape(lo.SLOTS, lo.MAX_N + 1), F)
        off += lo.SLOTS * (lo.MAX_N + 1)
        e0 = lo.init(seed, t, lo.EXCH)
        for k in range(lo.ATOM_RET):
            for n in (0, 1, 2, 33, 264, 511, 512):
                s, x = lo.return_fold(F, X, k, n)
                if lo.RET_SLOTS[k] == lo.EXCH:
                    for lane in range(32):
                        m = lo.l2_mix(e0, lane)
                        s, x = (s + m) & M32, x ^ m
                n1 = lo.MAX_N + 1
                assert (got[off + k * n1 + n], got[off + lo.ATOM_RET * n1 + k * n1 + n]) == (s, x), (k, n)
        assert (got[off + 2 * lo.ATOM_RET * (lo.MAX_N + 1):] == 0).all()


def test_layout_and_contributor_counts(drv):
    b = drv("bounds")
    assert b[:6] == [lo.BLOCK_WORDS, 4, lo.SLOTS, lo.ROWS, lo.MAX_N, lo.ATOM_HOT_WORDS]
    assert b[7:] == [lo.TABLE_WORDS, 64 + 16 * 4096, 4096]
    for G in (1, 7, 132, 264, 1056, 2112, 4096):
        n = drv("n", G)
        assert n == [lo.n_of(G, r) for r in range(lo.ROWS)] and sum(n) == 4 * G and max(n) <= lo.MAX_N


def test_float_operands_keep_every_partial_sum_exact():
    """Every prefix and every subset bound: |init| + sum of |operands| within the format's exact-integer range."""
    for seed in SEEDS[:2]:
        for t in range(lo.TILES):
            F, X = lo.finals(seed, t)
            f16 = [lo.f16_int(x) for x in X[lo.F16X2]] + [lo.f16_int(x >> 16) for x in X[lo.F16X2]]
            assert 3 + sum(abs(v) for v in f16[:lo.MAX_N]) <= 2048 and 3 + sum(abs(v) for v in f16[lo.MAX_N:]) <= 2048
            bf = [lo.bf16_int(x) for x in X[lo.BF16X2]]
            assert sum(abs(v) for v in bf) <= 256
            assert 1000 + sum(abs(lo.bits_f32(x)) for x in X[lo.F32]) < 2 ** 24


# ---- fault models: the marches ------------------------------------------------------------------------------------------
def _march_word(fmt, p, prev, fault=None):
    """One word of one thread through one march (every element's reads and writes of that word), with a fault model
    on what a write stores: fault(kind, old, new, element) -> stored.  prev: what the word held before (the previous
    comparison's P).  Returns (reads, wrong reads)."""
    mem, reads, wrong = prev, [], 0
    if fmt == lo.WORD:
        plan = [(None, p), (p, ~p & M32), (~p & M32, p), (p, ~p & M32), (~p & M32, p), (p, None)]
    else:
        plan = [(None, p), (p, ~p & M32), (~p & M32, p), (p, None)]
    for e, (want, new) in enumerate(plan):
        if want is not None:
            reads.append(mem)
            wrong += mem != want
        if new is not None:
            mem = fault(mem, new, e) if fault else new
    return reads, wrong


def _stuck(bit, v):
    return lambda old, new, e: (new & ~(1 << bit) & M32) | (v << bit)


def _no_rise(bit):
    return lambda old, new, e: new & ~(1 << bit) & M32 if not (old >> bit) & 1 and (new >> bit) & 1 else new


def _no_fall(bit):
    return lambda old, new, e: new | (1 << bit) if (old >> bit) & 1 and not (new >> bit) & 1 else new


@pytest.mark.parametrize("fmt", [lo.WORD, lo.BYTE], ids=["word", "byte"])
def test_stuck_at_and_transition_faults_in_every_bit_are_caught_in_every_tile(fmt):
    seed = 0xC0FFEE17
    for t in range(lo.TILES):
        table, _ = lo.tile(seed, fmt, t)
        p = int(lo.window(table, lo.BLOCK_WORDS)[41])
        for bit in range(32):
            for model in (_stuck(bit, 0), _stuck(bit, 1), _no_rise(bit), _no_fall(bit)):
                assert _march_word(fmt, p, p, model)[1] > 0, (t, bit)


def test_the_fold_alone_misses_bit_31_stuck_under_the_solid_tile():
    """Two wrong reads of 2^31 enter the fold with odd weights: 2^31 x (odd + odd) = 0 mod 2^32.  The direct compare
    sees them."""
    reads, wrong = _march_word(lo.WORD, 0, 0, _stuck(31, 0))
    good, _ = _march_word(lo.WORD, 0, 0)
    assert wrong == 2
    w = [2 * j + 1 for j in range(len(reads))]
    assert sum(a * b for a, b in zip(w, reads)) % 2 ** 32 == sum(a * b for a, b in zip(w, good)) % 2 ** 32


def test_a_write_lost_between_owners_is_caught():
    """Every write of the march but the first is read by the next owner with the other polarity; the first is caught
    where the word held something else (the first repetition of each tile)."""
    for t in range(lo.TILES):
        table, _ = lo.tile(0x1234, lo.WORD, t)
        p = int(lo.window(table, lo.BLOCK_WORDS)[100])
        for lost in range(1, 5):
            assert _march_word(lo.WORD, p, p, lambda old, new, e, L=lost: old if e == L else new)[1] > 0, (t, lost)
        prev_table, _ = lo.tile(0x1234, lo.WORD, (t - 1) % lo.TILES)
        prev = int(lo.window(prev_table, lo.BLOCK_WORDS)[100])
        assert (_march_word(lo.WORD, p, prev, lambda old, new, e: old if e == 0 else new)[1] > 0) == (p != prev)


def test_a_write_to_the_wrong_block_is_caught_in_the_keyed_tiles():
    for t in range(lo.TILES):
        table, _ = lo.tile(7, lo.WORD, t)
        win = lo.window(table, 4 * lo.BLOCK_WORDS)
        # word 5 of block 0 lands on word 5 of block 2: the owner of block 2 reads block 0's value there
        caught = win[5] != win[2 * lo.BLOCK_WORDS + 5]
        assert caught == (so.kind(t) == 4), t


def _byte_march(p, spill=None, drop=None):
    """BYTE's three writes of one word at byte granularity: bytes (3, 0, 2, 1), two halves, bytes again.  spill: a
    byte store also writes the next byte of the word; drop: the store of this byte index (or half 0 / 1 as 10 / 11)
    does not happen.  Returns the wrong reads."""
    mem = bytearray(int(~p & M32).to_bytes(4, "little"))
    wrong = 0

    def st8(v, b):
        if drop == b:
            return
        mem[b] = (v >> (8 * b)) & 0xFF
        if spill and b < 3:
            mem[b + 1] = (v >> (8 * b)) & 0xFF

    def st16(v, h):
        if drop == 10 + h:
            return
        mem[2 * h:2 * h + 2] = ((v >> (16 * h)) & 0xFFFF).to_bytes(2, "little")

    def rd(want):
        nonlocal wrong
        wrong += int.from_bytes(mem, "little") != want
    for b in (3, 0, 2, 1):
        st8(p, b)
    rd(p)
    for h in (0, 1):
        st16(~p & M32, h)
    rd(~p & M32)
    for b in (3, 0, 2, 1):
        st8(p, b)
    rd(p)
    return wrong


def test_byte_spill_and_dropped_byte_enables_are_caught_where_the_bytes_differ():
    seed = 0xC0FFEE17
    for t in range(lo.TILES):
        table, _ = lo.tile(seed, lo.BYTE, t)
        p = int(lo.window(table, lo.BLOCK_WORDS)[201])
        assert _byte_march(p) == 0
        for drop in (0, 1, 2, 3, 10, 11):       # P and ~P differ in every bit: a dropped store always shows
            assert _byte_march(p, drop=drop) > 0, (t, drop)
        bs = p.to_bytes(4, "little")
        spill_seen = _byte_march(p, spill=True) > 0
        # a spill writes byte b's value into byte b + 1: invisible only if the word's bytes are all equal
        assert spill_seen == (len(set(bs)) > 1 or len(set((~p & M32).to_bytes(4, "little"))) > 1), t


# ---- fault models: the atomic units -----------------------------------------------------------------------------------
def _apply(s, v, x):
    if s == lo.ADD:
        return (v + x) & M32
    if s == lo.INC:
        return 0 if v >= x else v + 1
    if s == lo.DEC:
        return x if v == 0 or v > x else v - 1
    if s == lo.AND:
        return v & x
    if s == lo.OR:
        return v | x
    if s == lo.XOR:
        return v ^ x
    if s in (lo.MIN_U, lo.MAX_U):
        return min(v, x) if s == lo.MIN_U else max(v, x)
    if s in (lo.MIN_S, lo.MAX_S):
        return (min if s == lo.MIN_S else max)(v, x, key=lo._s32)
    if s == lo.F32:
        return lo.f32_bits(lo.bits_f32(v) + lo.bits_f32(x))
    if s == lo.F16X2:
        return lo.f16_bits(lo.f16_int(v) + lo.f16_int(x)) | lo.f16_bits(lo.f16_int(v >> 16) + lo.f16_int(x >> 16)) << 16
    if s == lo.BF16X2:
        return lo.bf16_bits(lo.bf16_int(v) + lo.bf16_int(x)) | \
            lo.bf16_bits(lo.bf16_int(v >> 16) + lo.bf16_int(x >> 16)) << 16
    raise ValueError(s)


def _word(seed, t, s, n, fault=None, q_bad=None):
    """Final value and return fold (lane 0; add / inc / dec only) of one word of slot s after n contributions, with a
    fault: "drop" / "double" contribution q_bad, "wrong" (the unit stores a wrong result for it), "wrap" (inc / dec
    wrap at bound + 1 throughout), "ret" (contribution q_bad returns a wrong value)."""
    v = lo.init(seed, t, s)
    rets = []
    for q in range(n):
        x = lo.operand(seed, t, s, q)
        if fault == "wrap" and s in (lo.INC, lo.DEC):
            x += 1
        times = 1
        if q == q_bad and fault == "drop":
            continue
        if q == q_bad and fault == "double":
            times = 2
        for _ in range(times):
            rets.append(v)
            v = _apply(s, v, x)
        if q == q_bad and fault == "wrong":       # a result one off: in the low half of the packed halves
            if s == lo.F16X2:
                v = _apply(s, v, lo.f16_bits(1))
            elif s == lo.BF16X2:
                v = _apply(s, v, lo.bf16_bits(1))
            else:
                v ^= 1 << 20 if s == lo.F32 else 1 << 3
    if fault == "ret" and q_bad is not None and rets:
        rets[q_bad] ^= 1
    fold = sum(lo.l2_mix(r, 0) for r in rets) & M32 if s in (lo.ADD, lo.INC, lo.DEC) else 0
    return v, fold


ALWAYS = [lo.ADD, lo.INC, lo.DEC, lo.XOR, lo.F32, lo.F16X2, lo.BF16X2]
WHERE_VISIBLE = [lo.AND, lo.OR, lo.MIN_S, lo.MAX_S, lo.MIN_U, lo.MAX_U]


@pytest.mark.parametrize("fault", ["drop", "double", "wrong"])
def test_a_dropped_doubled_or_wrong_atomic_is_caught_in_every_tile(fault):
    seed, n = 0xC0FFEE17, 264
    for t in range(lo.TILES):
        for s in ALWAYS:
            for q in (0, 1, 100, n - 1):
                if s == lo.BF16X2 and q & 1 and fault != "wrong":
                    continue                         # its odd-rank operands are zero: dropping or doubling one is a no-op
                good, gret = _word(seed, t, s, n)
                bad, bret = _word(seed, t, s, n, fault, q)
                assert (good, gret) != (bad, bret), (t, s, q, fault)


def test_and_or_min_max_faults_are_seen_only_where_the_final_value_can_show_them():
    seed, n = 0xC0FFEE17, 40
    seen = {s: 0 for s in WHERE_VISIBLE}
    for t in range(lo.TILES):
        for s in WHERE_VISIBLE:
            for q in range(n):
                seen[s] += _word(seed, t, s, n) != _word(seed, t, s, n, "drop", q)
    assert all(seen.values()), seen                            # each is caught somewhere ...
    assert all(v < lo.TILES * n for v in seen.values()), seen   # ... and not everywhere: stated in DESIGN 4.12


# contributions per word: the fewest with which every word still crosses its bound (grids of 136 CTAs), and an H100's
# (4 x 132 = 528 L2_ATOM CTAs: 66 per word)
WRAP_N = [lo.WRAP_MAX + 1, 4 * 528 // lo.ROWS]


@pytest.mark.parametrize("n", WRAP_N)
def test_every_inc_dec_word_crosses_its_bound(n):
    for seed in SEEDS:
        for t in range(lo.TILES):
            for s in (lo.INC, lo.DEC):
                v, b = lo.init(seed, t, s), lo.operand(seed, t, s, 0)
                assert 2 <= b <= lo.WRAP_MAX and v <= b
                steps = b - v + 1 if s == lo.INC else v + 1      # contributions until the word wraps
                assert steps <= n, (seed, t, s, v, b)


@pytest.mark.parametrize("n", WRAP_N)
def test_inc_dec_wrapping_at_the_wrong_bound_is_caught_in_every_tile(n):
    for seed in SEEDS:
        for t in range(lo.TILES):
            for s in (lo.INC, lo.DEC):
                assert _word(seed, t, s, n) != _word(seed, t, s, n, "wrap", 0), (seed, t, s)


def test_one_wrong_returned_value_changes_the_return_fold():
    for t in range(lo.TILES):
        for s in (lo.ADD, lo.INC, lo.DEC):
            for q in (0, 77, 263):
                assert _word(9, t, s, 264)[1] != _word(9, t, s, 264, "ret", q)[1], (t, s, q)


def test_a_float_reduction_that_flushes_or_rounds_is_caught():
    """A unit that flushes its result to zero is caught wherever the exact sum is not zero; one that rounds it to bf16's
    8 significand bits wherever the exact sum needs more.  Neither can be seen otherwise."""
    flushed = rounded = 0
    for t in range(lo.TILES):
        F, _ = lo.finals(5, t)
        for s in (lo.F32, lo.V4RED, lo.V4RED + 3, lo.V4ATOM):
            exact = lo.bits_f32(int(F[s, 264]))
            flushed += exact != 0
            rounded += lo.bits_f32(lo.f32_bits(exact) & 0xFFFF0000) != exact
    assert flushed == 4 * lo.TILES and rounded >= 2 * lo.TILES, (flushed, rounded)


# ---- ABI, backends, daemon, CLI ---------------------------------------------------------------------------------------
def test_header_and_bindings(pkg):
    N = pkg._native
    assert (N.L2_WORD, N.L2_BYTE, N.L2_ATOM) == (0, 1, 2)
    assert N.SIGNATURES["b2dp_l2_test"] == N.SIGNATURES["b2dp_compute_test"]
    hdr = open(os.path.join(ROOT, "include", "b200dp.h")).read()
    for name, v in (("B2DP_L2_WORD", 0), ("B2DP_L2_BYTE", 1), ("B2DP_L2_ATOM", 2)):
        assert re.search(r"#define %s %s\b" % (name, v), hdr), name
    assert re.search(r"B2DP_API int b2dp_l2_test\(b2dp_ctx \*ctx, int device, const b2dp_compute_test_opts \*opts,\s+"
                     r"b2dp_compute_test_result \*out, int cap, int \*n\);", hdr)
    assert "#define B2DP_ABI_VERSION 3" in hdr
    cli = open(os.path.join(ROOT, "tools", "b200dp_cli.cpp")).read()
    assert "l2_test [duration_ms]" in cli and "tbs_word=%.2f" in cli and "gops_atom=%.2f" in cli


def test_backends_without_an_l2_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.l2_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:
        with pytest.raises(N.B2dpError) as ei:
            ctx.l2_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "in-process only" in str(ei.value)
        assert "L2 self-test" in str(ei.value)


def test_daemon_l2_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-l2_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "L2 test at start not run: not supported by this backend" in err, err[-2000:]
    assert "-l2_test_at_start=0|1|2" in open(os.path.join(ROOT, "USAGE.md")).read().replace("\\|", "|")


# ---- SASS -------------------------------------------------------------------------------------------------------------
SASS_AT_LEAST = {
    lo.WORD: {"LDG.E.128.STRONG.GPU": 4, "STG.E.128.STRONG.GPU": 4},
    lo.BYTE: {"LDG.E.128.STRONG.GPU": 4, "STG.E.U8.STRONG.GPU": 16, "STG.E.U16.STRONG.GPU": 8},
    lo.ATOM: {"ATOMG.E.ADD.STRONG.GPU": 1, "ATOMG.E.INC.STRONG.GPU": 1, "ATOMG.E.DEC.STRONG.GPU": 1,
              "ATOMG.E.EXCH.STRONG.GPU": 1, "ATOMG.E.CAS.STRONG.GPU": 1, "ATOMG.E.CAS.64.STRONG.GPU": 1,
              "REDG.E.AND.STRONG.GPU": 1, "REDG.E.OR.STRONG.GPU": 1, "REDG.E.XOR.STRONG.GPU": 1,
              "REDG.E.MIN.S32.STRONG.GPU": 1, "REDG.E.MAX.S32.STRONG.GPU": 1, "REDG.E.MIN.STRONG.GPU": 1,
              "REDG.E.MAX.STRONG.GPU": 1, "REDG.E.ADD.64.STRONG.GPU": 1, "REDG.E.ADD.F32.FTZ.RN.STRONG.GPU": 1,
              "REDG.E.ADD.F64.RN.STRONG.GPU": 1, "REDG.E.ADD.F16x2.RN.STRONG.GPU": 1,
              "REDG.E.ADD.BF16x2.RN.STRONG.GPU": 1, "REDG.E.ADD.F32x4.FTZ.RN.STRONG.GPU": 1,
              "ATOMG.E.ADD.F32x4.FTZ.RN.STRONG.GPU": 1},
}
# ops whose count is exact: each appears once per thread per repetition and nowhere else in the kernel
SASS_EXACT = {lo.ATOM: ["ATOMG.E.INC.STRONG.GPU", "ATOMG.E.DEC.STRONG.GPU", "ATOMG.E.CAS.64.STRONG.GPU",
                        "REDG.E.AND.STRONG.GPU", "REDG.E.OR.STRONG.GPU", "REDG.E.XOR.STRONG.GPU",
                        "REDG.E.MIN.S32.STRONG.GPU", "REDG.E.MAX.S32.STRONG.GPU", "REDG.E.MIN.STRONG.GPU",
                        "REDG.E.MAX.STRONG.GPU", "REDG.E.ADD.F32.FTZ.RN.STRONG.GPU",
                        "REDG.E.ADD.64.STRONG.GPU", "REDG.E.ADD.F64.RN.STRONG.GPU", "REDG.E.ADD.F16x2.RN.STRONG.GPU",
                        "REDG.E.ADD.BF16x2.RN.STRONG.GPU", "REDG.E.ADD.F32x4.FTZ.RN.STRONG.GPU",
                        "ATOMG.E.ADD.F32x4.FTZ.RN.STRONG.GPU"]}
# The kernel's own atomics share opcodes with three ops under test, so those are counted exactly with them: every
# inlined grid barrier (one NANOSLEEP each, in its wait) is one ATOMG.E.ADD (arrive) and two ATOMG.E.EXCH (reset,
# release), and every fault-hook claim site is one ATOMG.E.CAS -- one per separator of WORD / BYTE (elements - 1),
# one in ATOM.  ATOM then adds exactly one atom.add, one atom.exch and one cas.b32 under test.
CLAIM_SITES = {lo.WORD: 5, lo.BYTE: 3, lo.ATOM: 1}


@pytest.mark.parametrize("dump", [0, 1], ids=["product", "dump"])
@pytest.mark.parametrize("fmt", [lo.WORD, lo.BYTE, lo.ATOM], ids=["word", "byte", "atom"])
def test_sass_has_the_planned_accesses_and_no_warp_aggregation(fmt, dump):
    lib = os.path.join(ROOT, "tests", "native", "libl2_test_kernels_test.so")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib) or not os.path.exists(tool):
        pytest.skip("needs the built harness and cuobjdump")
    sass = subprocess.run([tool, "-sass", lib], capture_output=True, text=True).stdout
    (body,) = [p for p in re.split(r"\n\s+Function : ", sass)[1:] if "l2_selftestILi%dELb%dE" % (fmt, dump) in
               p.split("\n")[0]]
    ops = [re.sub(r"^@!?U?P\w+\s+", "", i.strip()).split()[0] for i in re.findall(r"/\*[0-9a-f]{4,5}\*/\s+([^;]*);", body)]
    count = {}
    for op in ops:
        count[op] = count.get(op, 0) + 1
    for op, n in SASS_AT_LEAST[fmt].items():
        assert count.get(op, 0) >= n, (op, count.get(op, 0))
    for op in SASS_EXACT.get(fmt, []):
        assert count[op] == 1, (op, count[op])
    barriers, under_test = count.get("NANOSLEEP", 0), int(fmt == lo.ATOM)
    assert barriers >= (4 if fmt == lo.ATOM else 6), barriers
    assert count.get("ATOMG.E.ADD.STRONG.GPU", 0) == barriers + under_test, (count.get("ATOMG.E.ADD.STRONG.GPU"), barriers)
    assert count.get("ATOMG.E.EXCH.STRONG.GPU", 0) == 2 * barriers + under_test, count.get("ATOMG.E.EXCH.STRONG.GPU")
    assert count.get("ATOMG.E.CAS.STRONG.GPU", 0) == CLAIM_SITES[fmt] + under_test, count.get("ATOMG.E.CAS.STRONG.GPU")
    assert not any(op.startswith(("STL", "LDL")) for op in count), "local memory"
    # no warp-aggregated atomic: nvcc turns a uniform-address atom.add into VOTE.ANY + a SHFL.UP scan + one ATOMG
    assert "SHFL.UP" not in count, "warp-aggregation shape"
    usage = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True).stdout
    m = re.search(r"l2_selftestILi%dELb%dE[^\n]*\n\s*REG:(\d+)[^\n]*?LOCAL:(\d+)" % (fmt, dump), usage)
    assert m and int(m.group(2)) == 0, usage[-500:]
