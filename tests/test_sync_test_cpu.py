"""The synchronization self-test's host side, without a GPU.

- sync_test_math.hpp (through tests/native/sync_test_math_test.cpp): the layout, the crafted classes in every tile, the
  named-barrier schedule's coverage and legality, the warp partitions, and that a one-bit error in any result word of
  any thread changes that thread's check value.
- tests/sync_test_oracle.py, restated from the PTX ISA, equals the C++ at four seeds (tables, every result word, every
  check); it replays the atomics in random orders and asserts that no word depends on the order.
- Every fault model of the oracle changes the check values of every tile.
- The SASS of the built harness: the planned opcode families, the 16 barriers ptxas reports for SY_BAR.
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
import sync_test_oracle as so
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
THREADS, TILES = 128, 8
ATOM, BAR, WARP = 0, 1, 2


class Drv:
    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
        b = [float(x) for x in self.ask("bounds").split()]
        self.slots = [int(b[4 * f]) for f in range(3)]
        self.words = [int(b[4 * f + 1]) for f in range(3)]

    def ask(self, q):
        self.p.stdin.write(q + "\n")
        self.p.stdin.flush()
        return self.p.stdout.readline()

    def tile(self, seed, fmt, tile):
        v = np.array([int(x) for x in self.ask("tile %d %d %d" % (seed, fmt, tile)).split()], dtype=np.uint64)
        v = v.astype(np.uint32)
        ns, nw = self.slots[fmt] * THREADS, self.words[fmt] * THREADS
        return v[:ns].reshape(-1, THREADS), v[ns:ns + nw].reshape(THREADS, -1), v[ns + nw:]

    def fold(self, words):
        return int(self.ask("fold %d %s" % (len(words), " ".join(str(int(w)) for w in words))))


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("sy") / "sync_test_math_test")
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                    os.path.join(HERE, "native", "sync_test_math_test.cpp"), "-o", exe], check=True)
    d = Drv(exe)
    yield d
    d.p.stdin.close()
    d.p.wait()


def test_layout(drv):
    assert drv.slots == [65, 52, 32]
    assert drv.words == [134, 57, 300]


@pytest.mark.parametrize("seed", [1, 2, 0xC0FFEE, 0xFFFFFFFF])
@pytest.mark.parametrize("fmt", [ATOM, BAR, WARP])
def test_checks_are_folds_and_deterministic(drv, seed, fmt):
    for tile in (0, 5):
        tab, words, checks = drv.tile(seed, fmt, tile)
        tab2, words2, checks2 = drv.tile(seed, fmt, tile)
        assert (tab == tab2).all() and (words == words2).all() and (checks == checks2).all()
        for t in (0, 63, 127):
            assert drv.fold(words[t]) == checks[t]


@pytest.mark.parametrize("fmt", [ATOM, BAR, WARP])
def test_one_bit_error_in_any_word_changes_the_check(drv, fmt):
    _, words, checks = drv.tile(9, fmt, 3)
    rng = np.random.default_rng(fmt)
    for t in (0, 31, 64, 127):
        for j in list(range(0, drv.words[fmt], max(1, drv.words[fmt] // 16))) + [drv.words[fmt] - 1]:
            w = words[t].copy()
            w[j] ^= np.uint32(1 << int(rng.integers(32)))
            assert drv.fold(w) != checks[t], (t, j)


@pytest.mark.parametrize("seed", [1, 2, 0xC0FFEE, 0xFFFFFFFF])
@pytest.mark.parametrize("fmt", [ATOM, BAR, WARP])
def test_oracle_equals_cpp(drv, seed, fmt):
    for tile in range(TILES):
        tab, words, checks = drv.tile(seed, fmt, tile)
        T = so.table(seed, fmt, tile)
        assert (np.array(T, dtype=np.uint64).astype(np.uint32) == tab).all(), tile
        W = so.results(T, fmt, tile, orders=3, seed=seed)
        assert (np.array(W, dtype=np.uint64).astype(np.uint32) == words).all(), tile
        assert [so.fold(w) for w in W] == [int(c) for c in checks], tile


@pytest.mark.parametrize("fmt,fault", [(f, m) for f in (ATOM, BAR, WARP) for m in so.FAULTS[f]])
def test_fault_model_is_caught_in_every_tile(fmt, fault):
    for tile in range(TILES):
        clean = so.checks(5, fmt, tile)
        bad = so.checks(5, fmt, tile, fault=fault)
        assert clean != bad, (fault, tile)


def test_atom_crafted_classes(drv):
    """Inc / dec cross their bound within each lane word's 4 contributions; the hot word wraps many times; cas-once
    hits and misses; signed min / max see both signs; every 64-bit add carries into the high half."""
    for tile in range(TILES):
        tab, words, _ = drv.tile(5, ATOM, tile)
        inc_b, dec_b = tab[2 * 1][0], tab[2 * 2][0]
        assert (tab[2 * 1] == inc_b).all() and (tab[2 * 2] == dec_b).all()
        for lane in range(32):
            assert inc_b - tab[2 * 1 + 1][lane] <= 3 and tab[2 * 2 + 1][lane] <= 3
        casonce = tab[65 - 3], tab[65 - 2]
        hits = casonce[0] == casonce[1]
        assert hits.any() and (~hits).any()
        for o in (10, 11):  # min.s32 / max.s32 operands: both signs among each lane's 4 contributors
            signs = tab[2 * o].reshape(4, 32) >> 31
            assert (signs.min(axis=0) == 0).all() and (signs.max(axis=0) == 1).all()
        assert (tab[34] >= 0xF0000000).all()


def test_bar_schedule_is_legal_and_covers_every_id_count_and_producer(drv):
    """Reimplements sy_bar_step from its comment: k consecutive warps, the first np produce."""
    seen = set()
    for tile in range(TILES):
        for s in range(45):
            g, ident = s // 15, s % 15 + 1
            k = g + 2
            start, np_ = (tile + ident + g) % 4, 1 + (tile + 2 * ident + g) % (k - 1)
            part = [(start + i) % 4 for i in range(k)]
            assert len(set(part)) == k and 1 <= np_ < k
            for w in part[:np_]:
                seen.add((ident, 32 * k, w))
    assert seen == {(i, n, w) for i in range(1, 16) for n in (64, 96, 128) for w in range(4)}


def test_bar_reductions_hold_all_zero_all_one_and_one_different(drv):
    classes = set()
    for tile in range(TILES):
        tab, words, _ = drv.tile(3, BAR, tile)
        for i in range(3):
            q = tab[45 + i] & 1
            classes.add("zero" if q.sum() == 0 else "one" if q.sum() == 128 else
                        "single" if q.sum() in (1, 127) else "mixed")
        tx = tab[51]
        assert tx[0] == tx[64:].sum() and (tx[64:] >= 1).all()
    assert {"zero", "one", "single"} <= classes


def _color(w, lane):
    k, odd, off, fm = (w & 31) + 1, ((w >> 8) & 15) * 2 + 1, (w >> 16) & 31, (w >> 24) & 31
    p = (lane * odd + off) & 31
    return (0 if p < k else 64) | (p & fm)


def test_warp_partitions_cover_every_group_size_and_shape(drv):
    sizes, noncontig, depth3 = set(), False, False
    for tile in range(TILES):
        tab, _, _ = drv.tile(11, WARP, tile)
        for w in range(4):
            for s in range(4):
                wl = [int(tab[s * 8 + v][w * 32]) for v in range(3)]
                assert all((tab[s * 8 + v][w * 32:(w + 1) * 32] == wl[v]).all() for v in range(3))
                for lv in range(1, 4):
                    groups = {}
                    for lane in range(32):
                        groups.setdefault(tuple(_color(wl[v], lane) for v in range(lv)), []).append(lane)
                    for g in groups.values():
                        sizes.add(len(g))
                        noncontig = noncontig or g[-1] - g[0] + 1 != len(g)
                    depth3 = depth3 or (lv == 3 and 1 < len(groups) < 32)
    assert sizes == set(range(1, 33)) and noncontig and depth3


# ---- SASS ---------------------------------------------------------------------------------------------------------------
def _sass(lib):
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib) or not os.path.exists(tool):
        pytest.skip("harness not built or no cuobjdump")
    out, fn = {}, None
    for line in subprocess.run([tool, "-sass", lib], capture_output=True, text=True).stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            out[fn] = {}
            continue
        m = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]+)", line)
        if m and fn:
            out[fn][m.group(1)] = out[fn].get(m.group(1), 0) + 1
    return out


LIB = os.path.join(HERE, "native", "libsync_test_kernels_test.so")


@pytest.mark.parametrize("dump", [0, 1])
def test_sass_opcode_families(dump):
    s = _sass(LIB)
    k = {f: s["_ZN4b2dp13sync_selftestILi%dELb%dEEEvPKhPKjyijPNS_8CtRecordEyPj" % (f, dump)] for f in range(3)}
    a = k[ATOM]
    for op in ("ATOMS.INC", "ATOMS.DEC", "ATOMS.EXCH", "ATOMS.EXCH.64", "ATOMS.MIN", "ATOMS.MAX", "ATOMS.MIN.S32",
               "ATOMS.MAX.S32", "ATOMS.OR", "ATOMS.AND", "ATOMS.CAS.64"):
        assert a.get(op) == 3, (op, a)
    assert a.get("ATOMS.XOR") == 6 and a.get("ATOMS.ADD") == 7 and a.get("ATOMS.CAS") == 4
    assert a.get("ATOMS.CAST.SPIN") == 9 and a.get("ATOMS.CAST.SPIN.64") == 15
    b = k[BAR]
    assert b.get("BAR.ARV") == 2 and b.get("BAR.SYNC.DEFER_BLOCKING") == 8
    assert b.get("BAR.RED.POPC.DEFER_BLOCKING") == 2 and b.get("BAR.RED.AND.DEFER_BLOCKING") == 2
    assert b.get("BAR.RED.OR.DEFER_BLOCKING") == 4
    assert b.get("SYNCS.ARRIVE.TRANS64.OPTOUT.A1T0") == 1 and b.get("SYNCS.ARRIVE.TRANS64.TMASK.ART0") == 1
    assert b.get("SYNCS.ARRIVE.TRANS64.RED.A0TX") == 1
    assert b.get("SYNCS.PHASECHK.TRANS64") == 6 and b.get("SYNCS.PHASECHK.TRANS64.TRYWAIT") == 2
    w = k[WARP]
    # ptxas emits the group body twice (the outer levels' copy and the innermost level's): every collective of a level
    # appears twice, and nothing else runs them
    for op in ("SHFL.IDX", "SHFL.UP", "SHFL.DOWN", "SHFL.BFLY", "ELECT", "MATCH.ALL", "VOTE.ALL", "VOTE.EQ",
               "REDUX.SUM", "REDUX.XOR", "REDUX.MIN.S32", "REDUX.MAX"):
        assert w.get(op) == 2, (op, w)
    for op in ("VOTE.ANY", "MATCH.ANY", "REDUX.OR"):  # the software mask loops add some of their own
        assert w.get(op, 0) >= 2, (op, w)


def test_ptxas_barrier_counts(tmp_path):
    """ptxas reports 16 named barriers for SY_BAR (ids 0-15) and 1 for the other formats."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
                        "-I", CSRC, os.path.join(HERE, "native", "sync_test_kernels.cu"), "-o",
                        str(tmp_path / "k.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    found = {}
    fn = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            fn = m.group(1)
        m = re.search(r"used (\d+) barriers", line)
        if m and fn and "sync_selftest" in fn:
            found[fn] = int(m.group(1))
    assert len(found) == 6, found
    assert all(n == (16 if "ILi1E" in f else 1) for f, n in found.items()), found


# ---- interfaces ---------------------------------------------------------------------------------------------------------
def test_header_and_binding(pkg):
    N = pkg._native
    assert N.SIGNATURES["b2dp_sync_test"] == N.SIGNATURES["b2dp_compute_test"]
    assert (N.SY_ATOM, N.SY_BAR, N.SY_WARP) == (0, 1, 2)
    hdr = open(os.path.join(ROOT, "include", "b200dp.h")).read()
    for name, v in (("B2DP_SY_ATOM", 0), ("B2DP_SY_BAR", 1), ("B2DP_SY_WARP", 2)):
        assert re.search(r"#define %s %s\b" % (name, v), hdr), name
    assert re.search(r"B2DP_API int b2dp_sync_test\(b2dp_ctx \*ctx, int device, const b2dp_compute_test_opts \*opts,"
                     r"\s+b2dp_compute_test_result \*out, int cap, int \*n\);", hdr)
    assert "#define B2DP_ABI_VERSION 3" in hdr
    cli = open(os.path.join(ROOT, "tools", "b200dp_cli.cpp")).read()
    assert "sync_test [duration_ms]" in cli and "gops_atom=%.2f" in cli


def test_backends_without_a_sync_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.sync_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:      # cuda:probe=off (NVML only)
        with pytest.raises(N.B2dpError) as ei:
            ctx.sync_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "synchronization self-test" in str(ei.value)


def test_daemon_sync_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-sync_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "sync test at start not run: not supported by this backend" in err, err[-2000:]
