"""CPU tests of the on-demand shared-memory self-test (b2dp_smem_test): the host arithmetic against the oracle, the
marches' coverage, the faulty-SRAM model against the direct compare and the fold, the ABI constants, the backends and
daemon without the test, and the SASS of the product kernels."""
import ctypes as C
import os
import re
import shutil
import signal
import subprocess
import time

import numpy as np
import pytest

import fake_sysfs
import smem_test_oracle as so
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
SEEDS = [0, 1, 0xC0FFEE17, 0xFFFFFFFF]
FMT_IDS = [so.NAMES[f] for f in so.FORMATS]
# a word in every bank (word j is in bank j), and the first and last words
BANK_WORDS = list(range(32)) + [so.WORDS - 1]


class MathDriver:
    """tests/native/smem_test_math_test.cpp, compiled with g++ against csrc/smem_test_math.hpp."""

    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(self, *words):
        self.p.stdin.write(" ".join(str(w) for w in words) + "\n")
        self.p.stdin.flush()
        return [int(x) for x in self.p.stdout.readline().split()]

    def close(self):
        self.p.stdin.close()
        self.p.wait(timeout=10)


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("sh") / "smem_test_math_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                        os.path.join(ROOT, "tests", "native", "smem_test_math_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = MathDriver(exe)
    yield d
    d.close()


def _one(r, key, rank=0):
    return r[key][rank] if isinstance(r[key], list) else r[key]


def _tile(seed, fmt, t):
    return so.kind(t), so.key(seed, fmt, t)


# ---- the host arithmetic against the oracle ---------------------------------------------------------------------
def test_layout(drv):
    assert drv.ask("layout") == [so.BYTES, so.WORDS, so.WPT, so.VECS, so.VPT, so.VTAIL, so.PPT, so.TABLE_WORDS,
                                 so.HOOK_WORD, so.HOOK_ELEMENT, so.DUMP_WORDS] + [so.ELEMENTS[f] for f in so.FORMATS]
    assert (so.WORDS, so.WPT, so.VECS, so.VPT, so.VTAIL) == (58112, 454, 14528, 113, 64)
    assert [drv.ask("rank_key", r)[0] for r in (0, 1)] == [so.rank_key(0), so.rank_key(1)]


@pytest.mark.parametrize("seed", SEEDS)
def test_patterns_match_the_oracle(drv, seed):
    for t in range(so.TILES):
        kd, ky = _tile(seed, 0, t)
        for w0 in (0, 28000, so.WORDS - 1000):
            assert drv.ask("pattern", kd, ky, w0, 1000) == so.pattern(kd, ky, np.arange(w0, w0 + 1000)).tolist()


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", SEEDS)
def test_host_tables_and_checks_match_the_oracle(drv, seed, fmt):
    """Every tile's table, and every thread's check value: the fold of the oracle's clean march."""
    tabs = so.tables(seed, fmt)
    for t in range(so.TILES):
        got = drv.ask("tile", seed, fmt, t)
        assert got[:so.TABLE_WORDS] == tabs[t].tolist()
        if so.kind(t) == 4 or seed == SEEDS[0]:        # tiles 0..3 do not depend on the seed
            r = so.march(fmt, *_tile(seed, fmt, t))
            assert got[so.TABLE_WORDS:] == _one(r, "fold").tolist(), (seed, fmt, t)
            for rank in range(2 if fmt == so.DSMEM else 1):
                assert not _one(r, "err", rank).any()
                assert np.array_equal(_one(r, "fold", rank), _one(r, "fold"))   # both ranks fold the same sequence
                img = so.pattern(*_tile(seed, fmt, t), np.arange(so.WORDS))
                rk = so.rank_key(rank) if fmt == so.DSMEM else 0
                assert np.array_equal(_one(r, "image", rank), img ^ np.uint32(rk))


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_read_order_matches_the_oracle(drv, fmt):
    kd, ky = 4, 0x9E3779B9
    r = so.march(fmt, kd, ky, keep_reads=True)
    n = {so.WORD: [5 * so.WPT] * 2, so.BYTE: [4 * 114 + 16 * 114 + 2 * so.PPT, 4 * 113 + 16 * 113 + 2 * so.PPT],
         so.DSMEM: [3 * so.WPT] * 2}[fmt]
    for t in (0, 1, 31, 63, 64, 127):
        want = r["reads"][0][t]
        assert len(want) == n[t >= 64]
        assert drv.ask("reads", fmt, kd, ky, t) == want, (fmt, t)
        assert so.fold(want) == int(_one(r, "fold")[t])
        if fmt == so.DSMEM:
            assert r["reads"][1][t] == want


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_every_element_touches_every_byte_exactly_once(fmt):
    """Words, bytes, the 16-byte vectors with their 64-vector tail, the 8-byte pairs; for SH_DSMEM, both arrays."""
    r = so.march(fmt, 1, 0)
    assert len(r["touched"]) == so.ELEMENTS[fmt]
    for e, tc in enumerate(r["touched"]):
        for rank, counts in enumerate(tc):
            assert (counts == 1).all(), (fmt, e, rank, np.flatnonzero(counts != 1)[:4])


# ---- the faulty-SRAM model ------------------------------------------------------------------------------------------
def _bytes_of(words):
    return np.array([4 * w + b for w in words for b in range(4)])


def _mask(words, value=0xFF):
    m = np.zeros(so.BYTES, np.uint8)
    m[_bytes_of(words)] = value
    return m


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_stuck_at_every_bit_is_caught_by_the_direct_compare_in_every_tile(fmt):
    """Every bit of a word in every bank and of the first and last words, stuck at 0 (those words) and at 1 (a
    second word in every bank): every stuck bit is read wrong somewhere in every tile.  The faults sit in different
    cells, so the error-bit map attributes each one."""
    stuck0 = BANK_WORDS
    stuck1 = [32 * 100 + j for j in range(32)]
    mask = _mask(stuck0) | _mask(stuck1)
    value = _mask(stuck1)
    for t in range(so.TILES):
        r = so.march(fmt, *_tile(7, fmt, t), mem=so.Stuck(mask, value))
        em = _one(r, "errmap")
        assert (em[_bytes_of(stuck0 + stuck1)] == 0xFF).all(), (fmt, t)
        assert _one(r, "err").sum() > 0


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_transition_faults_are_caught_in_every_tile(fmt):
    up = BANK_WORDS
    down = [32 * 200 + j for j in range(32)]
    for t in range(so.TILES):
        for init in (0x00, 0xFF):
            mem = so.Transition(_mask(up), _mask(down), init=np.full(so.BYTES, init, np.uint8))
            r = so.march(fmt, *_tile(7, fmt, t), mem=mem)
            assert (_one(r, "errmap")[_bytes_of(up + down)] == 0xFF).all(), (fmt, t, init)


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_two_addresses_on_one_cell_are_caught_in_the_distinct_value_tiles(fmt):
    pairs = [(0, so.WORDS - 1), (5, 4096 + 5), (100, 101), (so.HOOK_WORD, 3 * so.THREADS + 1)]
    caught = {}
    for t in range(so.TILES):
        r = so.march(fmt, *_tile(11, fmt, t), mem=so.Alias(pairs))
        em = _one(r, "errmap")
        caught[t] = [bool(em[_bytes_of([a, b])].any()) for a, b in pairs]
        if t >= 4:
            assert all(caught[t]), (fmt, t, caught[t])
    print(so.NAMES[fmt], "aliased pairs caught per tile:", caught)


def _write_key(a):
    """SH_BYTE element 0's write order of byte a: step k, then byte order 3, 0, 2, 1 (all threads at once)."""
    return (a // 4 // so.THREADS, (3, 0, 2, 1).index(a % 4))


@pytest.mark.parametrize("d", [1, -1])
def test_a_byte_write_that_also_writes_its_neighbour(d):
    """The spill survives when the neighbour was written before the faulty byte, and is then visible when the two
    bytes of P differ: the model says exactly where it must be caught, and the direct compare catches it there."""
    must_seen = 0
    for f in [4 * 1000 + b for b in range(4)] + [4 * 130 + b for b in range(4)] + [4 * (so.WORDS - 1) - 4 + 3]:
        if not 0 <= f + d < so.BYTES:
            continue
        for t in range(so.TILES):
            kd, ky = _tile(5, so.BYTE, t)
            p = so.pattern(kd, ky, np.arange(so.WORDS)).view(np.uint8)
            must = _write_key(f + d) < _write_key(f) and p[f] != p[f + d]
            r = so.march(so.BYTE, kd, ky, mem=so.ByteSpill(f, d))
            assert bool(r["err"].any()) == must, (f, d, t)
            must_seen += must
    assert must_seen >= 8


@pytest.mark.parametrize("width", [2, 16], ids=["u16", "v4"])
def test_a_wide_write_that_drops_a_lane_is_caught_in_every_tile(width):
    for f in (0, 4 * 777 + 2, 4 * (so.WORDS - 1) + 3, 16 * (so.VPT * so.THREADS) + 9):
        for t in range(so.TILES):
            r = so.march(so.BYTE, *_tile(9, so.BYTE, t), mem=so.LaneDrop(f, width))
            assert r["err"].any() and r["errmap"][f], (width, f, t)


@pytest.mark.parametrize("lost", [True, False], ids=["lost", "misrouted"])
@pytest.mark.parametrize("order", [(0, 1), (1, 0)])
def test_a_dsmem_write_lost_or_delivered_to_the_writer_is_caught_in_every_tile(lost, order):
    for w in (0, 4660, so.WORDS - 1):
        for t in range(so.TILES):
            r = so.march(so.DSMEM, *_tile(13, so.DSMEM, t), peer=so.RemoteFault(w, lost), order=order)
            assert r["err"][0].any() or r["err"][1].any(), (w, t, lost, order)


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_the_fault_hook_is_read_back_after_every_element_but_the_last(fmt):
    for e in range(so.ELEMENTS[fmt]):
        for w in (0, so.HOOK_WORD, so.WORDS - 1):
            r = so.march(fmt, *_tile(3, fmt, 4), hook=(0, e, w, 0x80000000))
            seen = r["err"][0].any() or r["err"][1].any() if fmt == so.DSMEM else r["err"].any()
            assert seen == (e < so.ELEMENTS[fmt] - 1), (fmt, e, w)


def test_the_fold_alone_misses_a_stuck_bit_31_and_the_direct_compare_does_not():
    """March C- reads a bit stuck at 0 under a 0 background wrong in its two r(~P) elements: at bit 31 the two errors
    are 2^31 (w1 + w2) with w1 + w2 even, 0 mod 2^32."""
    w = 1000
    t = w % so.THREADS
    r = so.march(so.WORD, 0, 0, mem=so.Stuck(_bit31(w), np.zeros(so.BYTES, np.uint8)))
    clean = so.march(so.WORD, 0, 0)
    assert r["err"][t] == 2
    assert r["fold"][t] == clean["fold"][t]


def _bit31(w):
    m = np.zeros(so.BYTES, np.uint8)
    m[4 * w + 3] = 0x80
    return m


def test_the_fold_catches_every_single_bit_error():
    r = so.march(so.BYTE, 4, 0x12345678, keep_reads=True)
    for t in (0, 127):
        v = np.array(r["reads"][0][t], dtype=np.uint64)
        j = np.arange(v.size, dtype=np.uint64)
        base = so.fold(v)
        for b in range(32):
            flipped = v ^ np.uint64(1 << b)
            delta = ((2 * j + 1) * ((flipped - v) & np.uint64(so.M32))) & np.uint64(so.M32)
            assert ((np.uint64(base) + delta) & np.uint64(so.M32) != np.uint64(base)).all(), (t, b)


# ---- ABI, backends, daemon, SASS ------------------------------------------------------------------------------------
def test_constants_and_struct_layouts(pkg):
    N = pkg._native
    assert (N.SH_WORD, N.SH_BYTE, N.SH_DSMEM) == (0, 1, 2)
    assert (N.CT_ECC_CORRECTED, N.CT_ECC, N.CT_NO_ECC) == (0x10, 0x20, 0x40)
    assert C.sizeof(N.ComputeTestOpts) == 24 and C.sizeof(N.ComputeTestResult) == 128
    hdr = open(os.path.join(ROOT, "include", "b200dp.h")).read()
    for name, v in (("B2DP_SH_WORD", 0), ("B2DP_SH_BYTE", 1), ("B2DP_SH_DSMEM", 2), ("B2DP_CT_ECC_CORRECTED", "0x10u"),
                    ("B2DP_CT_ECC", "0x20u"), ("B2DP_CT_NO_ECC", "0x40u")):
        assert re.search(r"#define %s %s\b" % (name, v), hdr), name
    assert "b2dp_smem_test" in hdr


def test_backends_without_a_smem_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.smem_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:      # cuda:probe=off (NVML only)
        with pytest.raises(N.B2dpError) as ei:
            ctx.smem_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "in-process only" in str(ei.value)
        assert "shared-memory self-test" in str(ei.value)


def test_daemon_smem_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-smem_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "smem test at start not run: not supported by this backend" in err, err[-2000:]
    assert "Failed to start plugin gpu: Register:" in err


SASS = {0: ["LDS", "STS"],
        1: ["STS.U8", "STS.U16", "LDS.128", "LDS.U8", "STS.128", "LDS.64"],
        2: ["ST.E", "LD.E", "UCGABAR_ARV", "UCGABAR_WAIT"]}


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_sass_has_the_planned_accesses_inside_the_repetition_loop(fmt):
    """The product instantiation: every required access inside the repetition loop, found by its own back-edge (the
    innermost backward branch around the repetition's BAR.RED.OR compare), and no local memory (no spills).  ptxas
    puts the divergent paths of the cluster barrier out of line after the last EXIT; their jumps back are not loops."""
    lib = os.path.join(ROOT, "tests", "native", "libsmem_test_kernels_test.so")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib) or not os.path.exists(tool):
        pytest.skip("needs the built harness and cuobjdump")
    name = "smem_selftestILi%dELb0E" % fmt
    sass = subprocess.run([tool, "-sass", lib], capture_output=True, text=True).stdout
    (body,) = [p for p in re.split(r"\n\s+Function : ", sass)[1:] if name in p.split("\n")[0]]
    ins = [(int(a, 16), i.strip()) for a, i in re.findall(r"/\*([0-9a-f]{4,})\*/\s+([^;]*);", body)]
    ops = [(a, re.sub(r"^@!?U?P\w+\s+", "", i).split()[0]) for a, i in ins]
    bar = min(a for a, o in ops if o.startswith("BAR.RED.OR"))
    end = max(a for a, o in ops if o == "EXIT")
    back = [(a, int(m.group(1), 16)) for a, i in ins for m in [re.search(r"BRA (?:`\()?0x([0-9a-f]+)", i)]
            if m and int(m.group(1), 16) <= bar < a < end]
    src, tgt = min(back, key=lambda st: st[0] - st[1])
    for want in SASS[fmt]:
        inside = [a for a, o in ops if (o == want or o.startswith(want + ".")) and tgt <= a < src]
        assert inside, (fmt, want, "repetition loop 0x%x..0x%x" % (tgt, src))
    if fmt == so.BYTE:   # the u16 stores stay u16: no wider store merges the halves of a word
        assert sum(o == "STS.U16" for a, o in ops if tgt <= a < src) >= 16
    res = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True).stdout
    lines = res.splitlines()
    for k, ln in enumerate(lines):
        if "smem_selftestILi" in ln:
            assert re.search(r"\bLOCAL:0\b", lines[k + 1]), (ln, lines[k + 1])
