"""CPU side of the on-demand memory test (b2dp_memtest): the host arithmetic in csrc/memtest_math.hpp -- sizing,
segment seeds, the range closed form, the verdict -- against tests/memtest_oracle.py; the march oracle against the
closed forms; the ABI structs against gcc; the backends without a memory test; the daemon's flag.  No GPU needed."""
import ctypes
import os
import random
import shutil
import signal
import subprocess
import time

import numpy as np
import pytest

import fake_sysfs
import memtest_oracle as mt
from oracle import probe as oprobe
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
MiB, GiB = 1 << 20, 1 << 30
U64 = (1 << 64) - 1


class MathDriver:
    """tests/native/memtest_math_test.cpp, compiled with g++ against csrc/memtest_math.hpp."""

    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(self, *words):
        self.p.stdin.write(" ".join(str(w) for w in words) + "\n")
        self.p.stdin.flush()
        return self.p.stdout.readline().strip()

    def plan(self, free, total, reserve, mx):
        out = self.ask("plan", free, total, reserve, mx)
        return [] if out == "-" else [int(x) for x in out.split()]

    def close(self):
        self.p.stdin.close()
        self.p.wait(timeout=10)


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("mt") / "memtest_math_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC, os.path.join(ROOT, "tests", "native", "memtest_math_test.cpp"),
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = MathDriver(exe)
    yield d
    d.close()


H100 = 85520809984           # an H100 80GB HBM3's cudaMemGetInfo total


@pytest.mark.parametrize("free,total,reserve,mx", [
    (H100 - 600 * MiB, H100, 0, 0),                       # an idle card: everything above 10 %
    (H100 - 600 * MiB, H100, 0, 2 * GiB + 6 * MiB),       # the GPU test's size: 1 GiB, 1 GiB, 6 MiB
    (H100 - 600 * MiB, H100, 0, 5 * MiB),                 # max below one chunk and not a multiple of 2 MiB
    (H100 - 600 * MiB, H100, 0, 1 * MiB),                 # max below the 2 MiB granule: nothing
    (H100 // 20, H100, 0, 0),                             # free below the default reserve: nothing
    (8 * GiB, H100, 8 * GiB, 0),                          # free == reserve: nothing
    (8 * GiB + 3 * MiB, H100, 8 * GiB, 0),                # 3 MiB above the reserve: one 2 MiB segment
    (40 * GiB + 123456789, H100, 1, 0),                   # a reserve of one byte
    (300 * GiB, 400 * GiB, 1, 0),                         # more than 256 chunks: capped
    (0, 0, 0, 0),
])
def test_plan_matches_oracle_and_its_rules(drv, free, total, reserve, mx):
    got = drv.plan(free, total, reserve, mx)
    assert got == mt.plan(free, total, reserve, mx)
    budget = max(0, free - (reserve or total // 10))
    if mx:
        budget = min(budget, mx)
    assert sum(got) <= budget
    assert all(s % (2 * MiB) == 0 and 0 < s <= GiB for s in got)
    assert all(s == GiB for s in got[:-1]) and len(got) <= 256
    assert sum(got) == min(budget, 256 * GiB) // (2 * MiB) * (2 * MiB)


def test_plan_random_table(drv):
    rng = random.Random(7)
    for _ in range(300):
        total = rng.choice([H100, 141 * GiB, 24 * GiB, rng.randrange(1, 1 << 40)])
        free = rng.randrange(0, total + 1)
        reserve = rng.choice([0, 1, rng.randrange(0, total + 1)])
        mx = rng.choice([0, rng.randrange(0, 16 * GiB), rng.randrange(0, 1 << 41)])
        assert drv.plan(free, total, reserve, mx) == mt.plan(free, total, reserve, mx), (free, total, reserve, mx)


def test_segment_seed(drv):
    for seed in (0, 1, 0x5EED0000, 0xFFFFFFFF, 0x12345678):
        for g in (0, 1, 2, 79, 255):
            assert int(drv.ask("seed", seed, g)) == mt.segment_seed(seed, g)
    assert mt.segment_seed(0xABCD, 0) == 0xABCD
    assert len({mt.segment_seed(7, g) for g in range(256)}) == 256


@pytest.mark.parametrize("base,n", [
    (0, 0), (0, 1), (0, 1000), (12345, 67890), (1 << 20, 1 << 22),
    ((1 << 32) - 1000, 3000),                  # across the 2^32-word wrap of the index
    ((1 << 32) - 1, 2), (1 << 32, 5000), (3 * (1 << 32) - 77, 1 << 16),
])
@pytest.mark.parametrize("seed", [0, 0x5EED0003, 0xFFFFFFFF])
def test_range_closed_form_matches_numpy(drv, base, n, seed):
    want = mt.range_checksum(base, n, seed)
    assert int(drv.ask("range", base, n, seed)) == want
    assert int(drv.ask("range", base, n, seed ^ 0xFFFFFFFF)) == mt.range_checksum(base, n, seed ^ 0xFFFFFFFF)
    # P and ~P sum to n * (2^32 - 1) word by word
    assert (want + mt.range_checksum(base, n, seed ^ 0xFFFFFFFF)) & U64 == (n * 0xFFFFFFFF) & U64


def test_range_closed_form_of_a_whole_period(drv):
    """2^32 words visit every 32-bit value once: the sum is 2^31 (2^32 - 1) for any seed and any start."""
    for base in (0, 12345, 1 << 32):
        assert int(drv.ask("range", base, 1 << 32, 0x77)) == (1 << 31) * 0xFFFFFFFF


def test_expected_checksum_over_segments(drv):
    segs = [GiB, GiB, 6 * MiB]
    seed = 0xC0FFEE11
    for inv in (0, 0xFFFFFFFF):
        got = int(drv.ask("expect", seed, inv, *segs))
        want, base = 0, 0
        for g, b in enumerate(segs):
            want += int(drv.ask("range", base, b // 4, mt.segment_seed(seed, g) ^ inv))
            base += b // 4
        assert got == want & U64
    small = [64 * 1024, 64 * 1024, 16 * 1024]
    for inv in (0, 0xFFFFFFFF):
        assert int(drv.ask("expect", seed, inv, *small)) == mt.expected_checksum([b // 4 for b in small], seed, inv)


@pytest.mark.parametrize("segments_words,faults", [
    ([4096 * 3, 4096 * 3, 4096], []),
    ([4096 * 3, 4096 * 3, 4096], [(0, 1), (4096 * 3 - 1, 0x80000000), (4096 * 7 - 1, 0xFFFFFFFF)]),
    ([4096], [(5, 0x10), (6, 0x10)]),
])
def test_march_oracle_is_consistent_with_the_closed_forms(drv, segments_words, faults):
    seed = 0x31415926
    res = mt.march(segments_words, seed, faults)
    assert len(res) == 4
    n = sum(segments_words)
    p = res[0][3]
    assert res[0][:3] == (0, 0, mt.NO_BAD)
    assert oprobe.checksum(p) == mt.expected_checksum(segments_words, seed)
    bad_words = sorted({w for w, m in faults if m})
    for k in (1, 2, 3):
        cs, mm, fb, buf = res[k]
        inv = 0xFFFFFFFF if k == 2 else 0
        assert mm == len(bad_words) and fb == (bad_words[0] if bad_words else mt.NO_BAD)
        if not faults:
            assert cs == mt.expected_checksum(segments_words, seed, inv)
            assert cs == int(drv.ask("expect", seed, inv, *[w * 4 for w in segments_words]))
    # E1 leaves ~P (plus faults), E2 leaves P, E3 does not write
    fmask = np.zeros(n, dtype=np.uint32)
    for w, m in faults:
        fmask[w] ^= np.uint32(m)
    assert np.array_equal(res[1][3], p ^ np.uint32(0xFFFFFFFF) ^ fmask)
    assert np.array_equal(res[2][3], p ^ fmask) and np.array_equal(res[3][3], res[2][3])


def test_march_oracle_catches_aliasing():
    """Two segments that are one physical range: whatever E0 left there, one of the two views mismatches."""
    n = 4096
    p0 = mt.march([n, n], 99)[0][3]
    for phys in (p0[:n], p0[n:]):                       # either write order
        seen = np.concatenate([phys, phys])
        assert np.count_nonzero(seen != p0) >= n - 2


VERDICT_TABLE = [
    # ok, mismatches, checksum-equal, ecc_unc, remap_failed, remap_pending, healthy
    (True, [0, 0, 0, 0], True, 0, False, False, True),
    (False, [0, 0, 0, 0], True, 0, False, False, False),
    (True, [0, 1, 1, 1], True, 0, False, False, False),
    (True, [0, 0, 0, 1], True, 0, False, False, False),
    (True, [0, 0, 0, 0], False, 0, False, False, False),
    (True, [0, 0, 0, 0], True, 1, False, False, False),
    (True, [0, 0, 0, 0], True, 0, True, False, False),
    (True, [0, 0, 0, 0], True, 0, False, True, False),
    (True, [5, 0, 0, 0], True, 0, False, False, True),     # element 0 only writes: its fields are not judged
]


@pytest.mark.parametrize("ok,mm,cs_ok,unc,rf,rp,want", VERDICT_TABLE)
def test_verdict_matches_oracle(drv, ok, mm, cs_ok, unc, rf, rp, want):
    exp = [0, 111, 222, 333]
    cs = list(exp) if cs_ok else [0, 111, 223, 333]
    cs[0] = 77                                            # E0's checksum is not compared either
    assert mt.memtest_healthy(ok, mm, cs, exp, unc, rf, rp) is want
    got = drv.ask("verdict", int(ok), *mm, *cs, *exp, unc, int(rf), int(rp))
    assert got == str(int(want))


def test_verdict_random_table(drv):
    rng = random.Random(3)
    for _ in range(200):
        ok, unc, rf, rp = rng.random() > .1, rng.choice([0, 0, 0, 1, 7]), rng.random() < .1, rng.random() < .1
        mm = [rng.choice([0, 0, 0, 1]) for _ in range(4)]
        exp = [rng.randrange(1 << 64) for _ in range(4)]
        cs = [e if rng.random() > .1 else rng.randrange(1 << 64) for e in exp]
        want = mt.memtest_healthy(ok, mm, cs, exp, unc, rf, rp)
        assert drv.ask("verdict", int(ok), *mm, *cs, *exp, unc, int(rf), int(rp)) == str(int(want))


def test_struct_layouts_match_the_c_header(pkg, tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    N = pkg._native
    pairs = [("b2dp_memtest_opts", N.MemtestOpts), ("b2dp_memtest_result", N.MemtestResult)]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200dp.h"', 'int main(void) {']
    for cname, ct in pairs:
        src.append('printf("%s %%zu", sizeof(%s));' % (cname, cname))
        for fname, _ in ct._fields_:
            src.append('printf(" %s=%%zu", offsetof(%s, %s));' % (fname, cname, fname))
        src.append('printf("\\n");')
    src += ['return 0; }']
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = str(tmp_path / "layout")
    r = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([exe], capture_output=True, text=True).stdout.splitlines()
    for line, (cname, ct) in zip(out, pairs):
        parts = line.split()
        assert parts[0] == cname and int(parts[1]) == ctypes.sizeof(ct)
        for tok, (fname, _) in zip(parts[2:], ct._fields_):
            k, v = tok.split("=")
            assert k == fname and int(v) == getattr(ct, fname).offset, (cname, fname)
    assert ctypes.sizeof(N.MemtestOpts) == 40 and ctypes.sizeof(N.MemtestResult) == 112


def test_backends_without_a_memory_test(pkg, kfd, tmp_path):
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.memtest(max_bytes=64 * MiB)
            assert ei.value.code == N.E_UNSUPPORTED


def test_daemon_memtest_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    """-memtest_at_start=1 parses; on a backend without a memory test the daemon logs that and carries on."""
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-memtest_at_start=1", "-memtest_max_bytes=67108864"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "memtest at start not run: not supported by this backend" in err, err[-2000:]
    assert "Failed to start plugin gpu: Register:" in err          # and the daemon went on to serve
