"""CPU side of the on-demand host-link self-test (b2dp_hostlink_test): the host arithmetic in csrc/hostlink_math.hpp --
the SM format's store-width schedule, the PCIe link capacity, the accepted buffer sizes, the seed schedule, the host's
check and the verdict -- against tests/hostlink_oracle.py; the ABI structs against gcc; the backends without the test;
the daemon's flag.  No GPU needed."""
import ctypes
import os
import re
import shutil
import signal
import subprocess
import time

import numpy as np
import pytest

import fake_sysfs
import hostlink_oracle as hl
from oracle import probe as oprobe
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
MiB, GiB = 1 << 20, 1 << 30


class MathDriver:
    """tests/native/hostlink_math_test.cpp, compiled with g++ against csrc/hostlink_math.hpp."""

    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(self, *words):
        self.p.stdin.write(" ".join(str(w) for w in words) + "\n")
        self.p.stdin.flush()
        return self.p.stdout.readline().strip()

    def close(self):
        self.p.stdin.close()
        self.p.wait(timeout=10)


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("hl") / "hostlink_math_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                        os.path.join(ROOT, "tests", "native", "hostlink_math_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = MathDriver(exe)
    yield d
    d.close()


def test_store_width_schedule(drv):
    vecs = list(range(0, 64)) + [(1 << 20) + 3 + k for k in range(10)] + [(1 << 40) + k for k in range(10)]
    for v in vecs:
        assert int(drv.ask("width", v)) == hl.store_width(v), v
    # every run of five consecutive vectors uses every width once, so every byte-enable shape crosses the link
    for start in (0, 1, 7, 12345):
        assert sorted(hl.store_width(v) for v in range(start, start + 5)) == [1, 2, 4, 8, 16]


def test_link_capacity_for_every_generation_and_width(drv):
    gens = list(range(-1, 8))
    widths = list(range(-1, 17)) + [32]
    for g in gens:
        for w in widths:
            got = float(drv.ask("link", g, w))
            want = hl.link_gbs(g, w)
            assert abs(got - want) <= 1e-12 * max(1.0, want), (g, w, got, want)
            if g not in (1, 2, 3, 4, 5) or w <= 0:
                assert got == 0.0
    assert round(hl.link_gbs(5, 16), 1) == 63.0
    assert round(hl.link_gbs(4, 16), 2) == 31.51 and hl.link_gbs(1, 1) == 0.25 and hl.link_gbs(2, 8) == 4.0


@pytest.mark.parametrize("requested", [0, 16, 32, 4096, 64 * MiB, 64 * MiB + 16, GiB - 16, GiB,
                                       1, 8, 15, 17, 64 * MiB + 8, GiB + 16, 2 * GiB, (1 << 63), (1 << 64) - 16])
def test_buffer_sizes_accepted_and_rejected(drv, requested):
    want = hl.buffer_bytes(requested)
    assert int(drv.ask("bytes", requested)) == want
    if requested == 0:
        assert want == 64 * MiB
    elif requested % 16 or requested > GiB:
        assert want == 0
    else:
        assert want == requested


def test_seed_schedule_is_the_probes(drv):
    for s in (0, 1, 0x5EED0000, 0xFFFFFFFF, 0x12345678):
        assert int(drv.ask("next", s)) == hl.next_seed(s) == oprobe.next_seed(s)


@pytest.mark.parametrize("n,faults", [
    (1, []), (4, [(0, 1)]), (1000, [(999, 0x80000000)]), (4096, [(17, 0x10), (3000, 0x3)]),
    (4096, [(5, 0xFFFFFFFF), (4, 0x1), (4095, 0x100)]),
])
def test_host_check_counts_and_first_bad(drv, n, faults):
    seed = 0xC0FFEE11
    buf = oprobe.pattern(n, seed)
    for w, m in faults:
        buf[w] ^= np.uint32(m)
    want = hl.check(buf, seed)
    got = drv.ask("check", n, seed, *[x for f in faults for x in f])
    assert tuple(int(x) for x in got.split()) == want
    assert want[0] == len(faults) and want[1] == (min(w for w, _ in faults) if faults else hl.NO_BAD)


VERDICT_TABLE = [
    # calls_ok, seq_ok, checksums_ok, rounds, mismatches, healthy
    (True, True, True, [3, 3, 9], [0, 0, 0], True),
    (False, True, True, [3, 3, 9], [0, 0, 0], False),
    (True, False, True, [3, 3, 9], [0, 0, 0], False),
    (True, True, False, [3, 3, 9], [0, 0, 0], False),
    (True, True, True, [0, 3, 9], [0, 0, 0], False),
    (True, True, True, [3, 3, 0], [0, 0, 0], False),
    (True, True, True, [1, 1, 1], [0, 1, 0], False),
    (True, True, True, [1, 1, 1], [2, 0, 0], False),
    (True, True, True, [1, 1, 1], [0, 0, 5], False),
]


@pytest.mark.parametrize("ok,seq_ok,cs_ok,rounds,mm,want", VERDICT_TABLE)
def test_verdict_matches_oracle(drv, ok, seq_ok, cs_ok, rounds, mm, want):
    assert hl.healthy(ok, seq_ok, cs_ok, rounds, mm) is want
    assert drv.ask("verdict", int(ok), int(seq_ok), int(cs_ok), *rounds, *mm) == str(int(want))


def test_oracle_sm_pass_counts_a_fault_once_and_the_host_sees_it():
    n, seed = 4096, 0x31415926
    nxt = hl.next_seed(seed)
    src = oprobe.pattern(n, seed)
    for word in (0, 2047, n - 1):
        cs, bad, first, dst = hl.sm_pass(src, seed, nxt, word, 0x40)
        assert (bad, first) == (1, word)
        assert cs != oprobe.expected_checksum(n, seed)
        assert hl.check(dst, nxt) == (1, word)
    cs, bad, first, dst = hl.sm_pass(src, seed, nxt)
    assert (cs, bad, first) == (oprobe.expected_checksum(n, seed), 0, hl.NO_BAD)
    assert np.array_equal(dst, oprobe.pattern(n, nxt))


# ---- ABI, backends, daemon, CLI ---------------------------------------------------------------------------------------
def test_struct_layouts_match_the_c_header(pkg, tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    N = pkg._native
    pairs = [("b2dp_hostlink_opts", N.HostlinkOpts), ("b2dp_hostlink_result", N.HostlinkResult)]
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
    r = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(c), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([exe], capture_output=True, text=True).stdout.splitlines()
    for line, (cname, ct) in zip(out, pairs):
        parts = line.split()
        assert parts[0] == cname and int(parts[1]) == ctypes.sizeof(ct)
        for tok, (fname, _) in zip(parts[2:], ct._fields_):
            k, v = tok.split("=")
            assert k == fname and int(v) == getattr(ct, fname).offset, (cname, fname)
    assert ctypes.sizeof(N.HostlinkOpts) == 40 and ctypes.sizeof(N.HostlinkResult) == 192


def test_header_and_bindings(pkg):
    N = pkg._native
    hdr = open(os.path.join(ROOT, "include", "b200dp.h")).read()
    consts = {"B2DP_HL_H2D": N.HL_H2D, "B2DP_HL_D2H": N.HL_D2H, "B2DP_HL_SM": N.HL_SM,
              "B2DP_HL_EVEN_IF_BUSY": N.HL_EVEN_IF_BUSY, "B2DP_HL_SKIPPED_BUSY": N.HL_SKIPPED_BUSY,
              "B2DP_HL_NUMA_UNBOUND": N.HL_NUMA_UNBOUND, "B2DP_HL_LINK_NARROW": N.HL_LINK_NARROW,
              "B2DP_HL_LINK_SLOW": N.HL_LINK_SLOW, "B2DP_HL_REPLAYS": N.HL_REPLAYS, "B2DP_HL_NO_NVML": N.HL_NO_NVML,
              "B2DP_RES_HOSTLINK": N.RES_HOSTLINK}
    for name, v in consts.items():
        m = re.search(r"#define %s (0x[0-9a-f]+|\d+)u?\b" % name, hdr)
        assert m and int(m.group(1), 0) == v, name
    assert N.RES_HOSTLINK == 0x800 and (N.HL_H2D, N.HL_D2H, N.HL_SM) == (0, 1, 2)
    assert re.search(r"B2DP_API int b2dp_hostlink_test\(b2dp_ctx \*ctx, int device, const b2dp_hostlink_opts \*opts, "
                     r"b2dp_hostlink_result \*out,\s+int cap, int \*n\);", hdr)
    assert "#define B2DP_ABI_VERSION 3" in hdr
    cli = open(os.path.join(ROOT, "tools", "b200dp_cli.cpp")).read()
    assert "hostlink_test [duration_ms]" in cli and "gbs_h2d=%.2f" in cli and "replays=%llu" in cli


def test_backends_without_a_hostlink_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.hostlink_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
            with pytest.raises(N.B2dpError) as ei:          # the backend is refused before the options are read
                ctx.hostlink_test(bytes=17)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:
        with pytest.raises(N.B2dpError) as ei:
            ctx.hostlink_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "in-process only" in str(ei.value)
        assert "host-link self-test" in str(ei.value)


def test_daemon_hostlink_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-hostlink_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "host-link test at start not run: not supported by this backend" in err, err[-2000:]
    assert "-hostlink_test_at_start=0|1|2" in open(os.path.join(ROOT, "USAGE.md")).read().replace("\\|", "|")
