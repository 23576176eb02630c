"""The on-demand diagnostics' entry points, without a GPU: what every caller sees before a test runs.

The ten SM self-tests, the memory test and the host-link self-test share one entry prologue in the library, and each
has a daemon flag, a CLI command and (for the SM tests) a Context method over it.  This pins, per test:
- the C ABI on backends without the test (kfd:, synthetic:) and on the NVML stub (cuda:probe=off, two GPUs): the
  return codes and the exact error texts, the device range, the E_NOSPC size report, a null result array;
- the Python methods: one signature, each with its docstring;
- the daemon: the exact "<test> at start not run" line of every -X_at_start flag, in the fixed order the tests run,
  and every flag it parses (literals and the SM self-test table) listed in USAGE.md;
- the CLI: exit status 1 and the exact error line of every test command on a backend without the test."""
import ctypes as C
import inspect
import os
import re
import signal
import subprocess
import time

import pytest

import fake_sysfs
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "tools", "b200dp_cli")
DAEMON = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")

# (entry point suffix, the name in the library's errors), in the header's order
SM_TESTS = [("compute_test", "compute self-test"), ("fp_test", "FP self-test"), ("sfu_test", "SFU self-test"),
            ("smem_test", "shared-memory self-test"), ("regfile_test", "register-file self-test"),
            ("int_test", "integer self-test"), ("l2_test", "L2 self-test"), ("half_test", "half-precision self-test"),
            ("sync_test", "synchronization self-test"), ("l1_test", "L1 self-test")]
ALL_TESTS = SM_TESTS + [("memtest", "memory test"), ("hostlink_test", "host-link self-test")]
IN_PROCESS_ONLY = "the %s runs in-process only (not with probe=helpers / probe=off / MIG)"
NO_CPU_FALLBACK = "the %s needs the cuda: backend (there is no CPU fallback)"


def _types(N, fn):
    """The opts and result structs of b2dp_<fn>."""
    return {"memtest": (N.MemtestOpts, N.MemtestResult),
            "hostlink_test": (N.HostlinkOpts, N.HostlinkResult)}.get(fn, (N.ComputeTestOpts, N.ComputeTestResult))


def _call(N, ctx, fn, device, cap, null_out=False):
    """b2dp_<fn>(ctx, device, &opts, out, cap, &n) through ctypes: (rc, n, b2dp_last_error)."""
    opts_t, res_t = _types(N, fn)
    opts = opts_t()
    out = None if null_out else (res_t * max(cap, 1))()
    n = C.c_int(-7)
    rc = getattr(N.lib, "b2dp_" + fn)(ctx._h, device, C.byref(opts), out, cap, C.byref(n))
    return rc, n.value, N.lib.b2dp_last_error(ctx._h).decode()


@pytest.mark.parametrize("fn,name", ALL_TESTS, ids=[t[0] for t in ALL_TESTS])
def test_backends_without_the_test(pkg, kfd, tmp_path, fn, name):
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            rc, _, err = _call(N, ctx, fn, -1, 8)
            assert (rc, err) == (N.E_UNSUPPORTED, NO_CPU_FALLBACK % name), uri
            with pytest.raises(N.B2dpError) as ei:
                getattr(ctx, fn)(duration_ms=10) if fn != "memtest" else ctx.memtest()
            assert (ei.value.code, ei.value.detail) == (N.E_UNSUPPORTED, NO_CPU_FALLBACK % name)


@pytest.mark.parametrize("fn,name", ALL_TESTS, ids=[t[0] for t in ALL_TESTS])
def test_entry_prologue_on_the_nvml_stub(pkg, monkeypatch, stub, tmp_path, fn, name):  # noqa: F811
    N = pkg._native
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:      # cuda:probe=off, two GPUs
        rc, _, err = _call(N, ctx, fn, 2, 8)
        assert (rc, err) == (N.E_INVAL, "device index out of range")
        rc, _, err = _call(N, ctx, fn, -2, 8)
        assert (rc, err) == (N.E_INVAL, "device index out of range")
        rc, n, _ = _call(N, ctx, fn, -1, 1)
        assert (rc, n) == (N.E_NOSPC, 2)
        rc, n, _ = _call(N, ctx, fn, 0, 0)
        assert (rc, n) == (N.E_NOSPC, 1)
        rc, _, _ = _call(N, ctx, fn, -1, 2, null_out=True)
        assert rc == N.E_INVAL
        for device, cap in ((-1, 2), (1, 1)):
            rc, _, err = _call(N, ctx, fn, device, cap)
            assert (rc, err) == (N.E_UNSUPPORTED, IN_PROCESS_ONLY % name)
        with pytest.raises(N.B2dpError) as ei:
            getattr(ctx, fn)()
        assert (ei.value.code, ei.value.detail) == (N.E_UNSUPPORTED, IN_PROCESS_ONLY % name)


def test_null_context_and_count(pkg):
    N = pkg._native
    for fn, _ in ALL_TESTS:
        opts_t, res_t = _types(N, fn)
        out, n = (res_t * 2)(), C.c_int(0)
        f = getattr(N.lib, "b2dp_" + fn)
        assert f(None, -1, C.byref(opts_t()), out, 2, C.byref(n)) == N.E_INVAL, fn
        assert f(None, -1, C.byref(opts_t()), out, 2, None) == N.E_INVAL, fn


def test_python_methods_share_one_signature(pkg):
    sigs = {fn: inspect.signature(getattr(pkg.Context, fn)) for fn, _ in SM_TESTS}
    assert len(set(map(str, sigs.values()))) == 1, sigs
    assert list(sigs["compute_test"].parameters) == ["self", "device", "duration_ms", "timeout_ms", "even_if_busy",
                                                     "fault_sm", "fault_mask"]
    assert [p.default for p in list(sigs["compute_test"].parameters.values())[1:]] == [-1, 0, 0, False, -1, 0]
    for fn, _ in SM_TESTS:
        doc = getattr(pkg.Context, fn).__doc__
        assert doc and ("b2dp_%s" % fn) in doc, fn


# the daemon's log prefix per flag, in the order main() runs them
DAEMON_ORDER = [("memtest", "memtest", "memory test"), ("compute_test", "compute test", "compute self-test"),
                ("fp_test", "fp test", "FP self-test"), ("sfu_test", "sfu test", "SFU self-test"),
                ("smem_test", "smem test", "shared-memory self-test"),
                ("regfile_test", "regfile test", "register-file self-test"),
                ("int_test", "int test", "integer self-test"), ("l2_test", "L2 test", "L2 self-test"),
                ("hostlink_test", "host-link test", "host-link self-test"),
                ("half_test", "half test", "half-precision self-test"),
                ("sync_test", "sync test", "synchronization self-test"), ("l1_test", "L1 test", "L1 self-test")]


def test_daemon_runs_every_flag_in_order(pkg, kfd, tmp_path, short_dir):
    if not os.path.exists(DAEMON):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    flags = ["-%s_at_start=1" % f for f, _, _ in reversed(DAEMON_ORDER)]     # the order of the flags does not matter
    proc = subprocess.Popen([DAEMON, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-compute_test_ms=50", *flags], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    got = [ln for ln in err.splitlines() if " at start not run: " in ln]
    want = ["%s at start not run: not supported by this backend (%s)" % (prefix, NO_CPU_FALLBACK % name)
            for _, prefix, name in DAEMON_ORDER]
    assert got == want, err[-3000:]


def test_every_daemon_flag_is_documented():
    """Every flag the daemon parses, whether a literal of parse_flags or a row of the SM self-test table, is listed in
    USAGE.md; all eleven -<x>_test_at_start flags are found (flag names may hold digits: -l1_..., -l2_...)."""
    d = open(os.path.join(ROOT, "k8s-device-plugin_b200", "csrc", "host", "plugind.cpp")).read()
    usage = open(os.path.join(ROOT, "USAGE.md")).read()
    flags = set(re.findall(r'name == "([a-z0-9_]+)"', d)) | set(re.findall(r'\{"([a-z0-9_]+_at_start)",', d))
    assert {f for f in flags if f.endswith("_test_at_start")} == {f + "_at_start" for f, _, _ in DAEMON_ORDER[1:]}
    for f in sorted(flags | {"labels", "reconcile", "patch", "version"}):
        assert ("-" + f) in usage, "USAGE.md does not list daemon flag -" + f


def test_daemon_rejects_an_unknown_test_flag(short_dir):
    if not os.path.exists(DAEMON):
        pytest.skip("b200dp_plugind not built")
    r = subprocess.run([DAEMON, "-plugin_dir", short_dir, "-tma_test_at_start=1"], stderr=subprocess.PIPE, text=True,
                       timeout=30)
    assert r.returncode == 2 and "flag provided but not defined: -tma_test_at_start" in r.stderr


@pytest.mark.skipif(not os.path.exists(CLI), reason="tools/b200dp_cli not built (run __graft_entry__.build())")
def test_cli_on_a_backend_without_the_tests(pkg, kfd, tmp_path):
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    strerror = N.lib.b2dp_strerror(N.E_UNSUPPORTED).decode()
    for fn, name in ALL_TESTS:
        for extra in ([], ["50"]):
            r = subprocess.run([CLI, "kfd:" + root, fn, *extra], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                               text=True, timeout=60)
            assert r.returncode == 1 and r.stdout == "", (fn, r)
            assert r.stderr == "b2dp_%s: %s [%d] %s\n" % (fn, strerror, N.E_UNSUPPORTED, NO_CPU_FALLBACK % name), fn
    r = subprocess.run([CLI, "kfd:" + root, "tma_test"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                       timeout=60)
    assert r.returncode == 2 and r.stderr == "unknown command tma_test\n"
