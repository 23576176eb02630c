"""The L1 self-test's host side, without a GPU.

- l1_test_math.hpp (through tests/native/l1_test_math_test.cpp) equals tests/l1_test_oracle.py, restated from the
  kernel's stated layout, the programming guide's address modes and the PTX ISA's tld4, at four seeds: tables, every
  result word, every check, L1_DATA's raw reads and block orders, the texel image and the constant bank.
- In every read pass every span vector, texel and window word is read exactly once and lies in range; L1_DATA's reader
  is never the writer.
- Hand-written address-mode cases pin wrap, mirror, clamp and border at m = -2..2 for the first, a middle and the last
  texel.
- Every fault model of the oracle changes the checks of exactly the tiles where it says the fault is visible, and a
  one-bit error in any result word changes the check.
- The SASS of the built harness: inside the loops (found by their back-edges) the planned opcode families; no spills;
  the 32 KiB constant bank in bank 3.
- The interfaces: the header, the binding, B2DP_E_UNSUPPORTED on backends without the test, the daemon flag."""
import os
import re
import shutil
import signal
import subprocess
import time

import numpy as np
import pytest

import fake_sysfs
import l1_test_oracle as lo
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
THREADS, TILES = 128, 8
DATA, TEX, CONST = 0, 1, 2
SEEDS = [1, 2, 0xC0FFEE, 0xFFFFFFFF]


class Drv:
    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
        b = [float(x) for x in self.ask("bounds").split()]
        self.words = [int(b[3 * f]) for f in range(3)]
        self.bytes1 = [b[3 * f + 2] for f in range(3)]
        self.default_k1 = int(b[9])

    def ask(self, q):
        self.p.stdin.write(q + "\n")
        self.p.stdin.flush()
        return self.p.stdout.readline()

    def arr(self, q):
        return np.array(self.ask(q).split(), dtype=np.uint64)

    def tile(self, seed, fmt, tile):
        v = self.arr("tile %d %d %d" % (seed, fmt, tile))
        nw = self.words[fmt] * THREADS
        return v[:4], v[4:4 + nw].reshape(THREADS, -1), v[4 + nw:]


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("l1") / "l1_test_math_test")
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                    os.path.join(HERE, "native", "l1_test_math_test.cpp"), "-o", exe], check=True)
    d = Drv(exe)
    yield d
    d.p.stdin.close()
    d.p.wait()


def test_layout(drv):
    assert drv.words == [12, 64 * 32, 2048 + 64 + 64 + 64]
    assert drv.bytes1 == [4 * 2048, 128 * 64 * 8 * 16, 128 * 2240 * 4]
    assert drv.default_k1 == 64                  # 128 KiB per SM in 2 KiB blocks


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("fmt", [DATA, TEX, CONST])
def test_oracle_equals_cpp(drv, seed, fmt):
    for tile in range(TILES):
        tab, words, checks = drv.tile(seed, fmt, tile)
        assert [int(x) for x in tab] == lo.table(seed, fmt, tile), tile
        assert (lo.results(seed, fmt, tile) == words).all(), tile
        c = lo.checks(seed, fmt, tile)
        if fmt == DATA:   # the host's check is the even fold; the odd one is -144 - it
            assert all(o == (-144 - e) & lo.M32 for e, o in c)
            c = [e for e, _ in c]
        assert [int(x) for x in checks] == c, tile
    if fmt == DATA:
        for K, cta in ((1, 0), (5, 2), (12, 7)):
            assert (drv.arr("span %d %d %d %d" % (seed, 4, K, cta)).reshape(THREADS, -1) ==
                    lo.data_reads(seed, 4, K, cta)).all()
    elif fmt == TEX:
        assert (drv.arr("image %d" % seed) == lo.texels(seed).ravel()).all()
    else:
        assert (drv.arr("bank %d" % seed) == lo.bank(seed)).all()


@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 7, 12, 64, 257])
def test_data_every_vector_once_per_pass_never_by_its_writer(drv, K):
    got = [int(x) for x in drv.ask("order %d" % K).split()]
    for p in range(3):
        assert sorted(got[p * K:(p + 1) * K]) == list(range(K))
        assert got[p * K:(p + 1) * K] == lo.order(p, K)
        readers = [lo.writer(t, p) for t in range(THREADS)]
        assert sorted(readers) == list(range(THREADS)) and all(lo.writer(t, p) != t for t in range(THREADS))


@pytest.mark.parametrize("tile", range(TILES))
def test_tex_and_const_read_every_texel_and_window_word_once_per_pass(tile):
    A, B, D, _ = lo.table(9, TEX, tile)
    seen = sorted((A * (THREADS * j + t) + B) & (lo.TEXELS - 1) for t in range(THREADS) for j in range(lo.STEPS))
    assert seen == list(range(lo.TEXELS))
    offs = {((t + j + D) % 5 - 2, (t // 5 + 2 * j + 3 * D) % 5 - 2) for t in range(THREADS) for j in range(lo.STEPS)}
    assert offs == {(a, b) for a in range(-2, 3) for b in range(-2, 3)}
    win, rot, _, _ = lo.table(9, CONST, tile)
    assert win == tile % 4 and 0 <= rot < lo.WIN
    for w in range(4):
        uni = [(k + 512 * w + rot) % lo.WIN for k in range(lo.WIN)]
        div = [(64 * l + k + 512 * w + rot) % lo.WIN for l in range(32) for k in range(64)]
        v2 = [(2 * (32 * l + k) + 512 * w + 2 * rot) % lo.WIN + e for l in range(32) for k in range(32) for e in (0, 1)]
        v4 = [(4 * (16 * l + k) + 512 * w + 4 * rot) % lo.WIN + e for l in range(32) for k in range(16) for e in range(4)]
        for form in (uni, div, v2, v4):
            assert sorted(form) == list(range(lo.WIN))
        for k in range(64):   # a divergent load touches 32 distinct 128-byte lines
            assert len({((64 * l + k + 512 * w + rot) % lo.WIN) // 32 for l in range(32)}) == 32


# (mode, x, N) -> texel at m = -2, -1, 0, 1, 2 (None: the border colour)
ADDR_CASES = {
    (lo.WRAP, 0, 64): [0, 0, 0, 0, 0], (lo.WRAP, 31, 64): [31] * 5, (lo.WRAP, 63, 64): [63] * 5,
    (lo.MIRROR, 0, 64): [0, 63, 0, 63, 0], (lo.MIRROR, 31, 64): [31, 32, 31, 32, 31],
    (lo.MIRROR, 63, 64): [63, 0, 63, 0, 63], (lo.MIRROR, 64, 128): [64, 63, 64, 63, 64],
    (lo.CLAMP, 0, 64): [0, 0, 0, 63, 63], (lo.CLAMP, 31, 64): [0, 0, 31, 63, 63], (lo.CLAMP, 63, 64): [0, 0, 63, 63, 63],
    (lo.CLAMP, 127, 128): [0, 0, 127, 127, 127],
    (lo.BORDER, 0, 64): [None, None, 0, None, None], (lo.BORDER, 31, 64): [None, None, 31, None, None],
    (lo.BORDER, 63, 64): [None, None, 63, None, None], (lo.BORDER, 0, 128): [None, None, 0, None, None],
}


@pytest.mark.parametrize("case", sorted(ADDR_CASES, key=str))
def test_address_modes_by_hand(case):
    mode, x, n = case
    assert [lo.tex_addr(mode, x, m, n) for m in range(-2, 3)] == ADDR_CASES[case]


def test_tex_results_follow_the_modes_and_tld4_order():
    img = lo.texels(3)
    W = lo.results(3, TEX, 2).reshape(THREADS, lo.STEPS, 8, 4)
    A, B, D, _ = lo.table(3, TEX, 2)
    for t in (0, 77):
        for j in (0, 1, 2, 3, 63):
            i = (A * (THREADS * j + t) + B) & (lo.TEXELS - 1)
            x, y = i % 64, i // 64
            assert (W[t, j, 0] == img[y, x]).all() and (W[t, j, 7] == img[y, x]).all()
            c = j % 4
            x1, y1 = min(x + 1, 63), min(y + 1, 127)
            assert list(W[t, j, 6]) == [img[y1, x, c], img[y1, x1, c], img[y, x1, c], img[y, x, c]]
    assert (img[:64] ^ img[64:] != 0).all()        # the two halves: P and ~P of different keyed words


_CLEAN = {}


def _checks(fmt, tile, fault=None):
    if fault is None:
        if (fmt, tile) not in _CLEAN:
            _CLEAN[(fmt, tile)] = lo.checks(5, fmt, tile)
        return _CLEAN[(fmt, tile)]
    return lo.checks(5, fmt, tile, fault=fault)


@pytest.mark.parametrize("fmt,fault", [(f, m) for f in (DATA, TEX, CONST) for m in lo.FAULTS[f]], ids=str)
def test_fault_model_is_caught_where_visible(fmt, fault):
    changed = {tile for tile in range(TILES) if _checks(fmt, tile) != _checks(fmt, tile, fault)}
    assert changed == lo.VISIBLE[fmt][fault], (fault, sorted(changed))


@pytest.mark.parametrize("fmt", [DATA, TEX, CONST])
def test_one_bit_error_in_any_word_changes_the_check(fmt):
    W = lo.results(9, fmt, 3)
    rng = np.random.default_rng(fmt)
    n = W.shape[1]
    for t in (0, 31, 64, 127):
        base = lo.sum_fold(W[t]) if fmt == DATA else lo.it_fold_rows(W[t:t + 1])[0]
        for j in sorted(set(list(range(0, n, max(1, n // 24))) + [n - 1])):
            for b in (0, 31, int(rng.integers(32))):
                w = W[t].copy()
                w[j] ^= np.uint64(1 << b)
                got = lo.sum_fold(w) if fmt == DATA else lo.it_fold_rows(w[None, :])[0]
                assert got != base, (t, j, b)


def test_table_ranges_are_refused(drv):
    assert drv.ask("ok 0 4 0 0 37").strip() == "1" and drv.ask("ok 0 5 0 0 37").strip() == "0"
    assert drv.ask("ok 0 4 0 0 512").strip() == "0"
    assert drv.ask("ok 1 8191 0 4 0").strip() == "1" and drv.ask("ok 1 8190 0 4 0").strip() == "0"
    assert drv.ask("ok 1 1 8192 0 0").strip() == "0" and drv.ask("ok 1 1 0 5 0").strip() == "0"
    assert drv.ask("ok 2 3 2047 0 0").strip() == "1" and drv.ask("ok 2 4 0 0 0").strip() == "0"
    assert drv.ask("ok 2 0 2048 0 0").strip() == "0" and drv.ask("ok 3 0 0 0 0").strip() == "0"


# ---- SASS and ptxas -----------------------------------------------------------------------------------------------------
LIB = os.path.join(HERE, "native", "libl1_test_kernels_test.so")


def _loops(lib):
    """Per function: the opcodes (with their operands) inside every loop, found by its backward branch."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib) or not os.path.exists(tool):
        pytest.skip("harness not built or no cuobjdump")
    fns, fn = {}, None
    for line in subprocess.run([tool, "-sass", lib], capture_output=True, text=True).stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            fns[fn] = []
            continue
        m = re.search(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]+)([^;]*);", line)
        if m and fn:
            fns[fn].append((int(m.group(1), 16), m.group(2), m.group(3)))
    out = {}
    for f, ins in fns.items():
        inside = []
        for addr, op, args in ins:
            t = re.search(r"0x([0-9a-f]+)", args)
            if op == "BRA" and t and int(t.group(1), 16) < addr:
                lo_, hi = int(t.group(1), 16), addr
                inside += [(o, a) for ad, o, a in ins if lo_ <= ad <= hi]
        out[f] = inside
    return out


@pytest.mark.parametrize("dump", [0, 1])
def test_sass_opcode_families_in_the_loops(dump):
    s = _loops(LIB)
    k = {f: s["_ZN4b2dp11l1_selftestILi%dELb%dEEEvPKhPKjyijPNS_8CtRecordEyPj" % (f, dump)] for f in range(3)}
    ops = {f: {o for o, _ in k[f]} for f in range(3)}
    assert "LDG.E.128" in ops[DATA] and "STG.E.128" in ops[DATA], ops[DATA]
    assert not {o for o in ops[DATA] if o.startswith("LDG") and ("STRONG" in o or "CONSTANT" in o) and ".128" in o}
    for op in ("TLD.LZ", "TEX.LL", "TLD4.R", "TLD4.G", "TLD4.B", "TLD4.A", "LDG.E.128.CONSTANT"):
        assert op in ops[TEX], (op, ops[TEX])
    bank3 = {o for o, a in k[CONST] if o.startswith("LDC") and "c[0x3]" in a}
    assert {"LDC", "LDC.64"} <= bank3, bank3      # the 128-bit loads assemble to pairs of LDC.64


def test_ptxas_no_spills_and_the_constant_bank(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    cubin = str(tmp_path / "k.cubin")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
                        "-I", CSRC, os.path.join(HERE, "native", "l1_test_kernels.cu"), "-o", cubin],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    fn, spills = None, {}
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            fn = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn and "l1_selftest" in fn:
            spills[fn] = int(m.group(1)) + int(m.group(2))
    assert len(spills) == 6 and not any(spills.values()), spills
    elf = subprocess.run([tool, "-elf", cubin], capture_output=True, text=True).stdout
    m = re.search(r"\.nv\.constant3\s*\n?", elf)
    assert m, "no constant bank 3"
    sym = [ln for ln in elf.splitlines() if ln.rstrip().endswith(" b2dp_l1_bank")]
    assert sym and "0x8000" in sym[0], sym                     # cmem[3]: 32,768 bytes


# ---- interfaces ---------------------------------------------------------------------------------------------------------
def test_header_and_binding(pkg):
    N = pkg._native
    assert N.SIGNATURES["b2dp_l1_test"] == N.SIGNATURES["b2dp_compute_test"]
    assert (N.L1_DATA, N.L1_TEX, N.L1_CONST) == (0, 1, 2)
    hdr = open(os.path.join(ROOT, "include", "b200dp.h")).read()
    for name, v in (("B2DP_L1_DATA", 0), ("B2DP_L1_TEX", 1), ("B2DP_L1_CONST", 2)):
        assert re.search(r"#define %s %s\b" % (name, v), hdr), name
    assert re.search(r"B2DP_API int b2dp_l1_test\(b2dp_ctx \*ctx, int device, const b2dp_compute_test_opts \*opts,"
                     r"\s+b2dp_compute_test_result \*out, int cap, int \*n\);", hdr)
    assert "#define B2DP_ABI_VERSION 3" in hdr and "exporter/health.go:42-82" in hdr
    assert len(re.findall(r"^B2DP_API ", hdr, re.M)) == 63
    cli = open(os.path.join(ROOT, "tools", "b200dp_cli.cpp")).read()
    assert "l1_test [duration_ms]" in cli and "tbs_data=%.2f" in cli and "tbs_const=%.2f" in cli


def test_backends_without_an_l1_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.l1_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:      # cuda:probe=off (NVML only)
        with pytest.raises(N.B2dpError) as ei:
            ctx.l1_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "L1 self-test" in str(ei.value)


def test_daemon_l1_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-l1_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "L1 test at start not run: not supported by this backend" in err, err[-2000:]
