"""The heartbeat's SM check (cuda: sm_check=<ms>), without a GPU.

- The URI: sm_check= and its test hook sm_check_fault= are parsed strictly and refused with B2DP_E_INVAL and a text
  naming the key; on the NVML stub (cuda:probe=off, where no probe runs) a valid value opens and one log line at open
  says the SM checks are off and why.
- The ABI: B2DP_RES_SM_CHECK, and b2dp_probe_result.sm_check in place of the old reserved word (88 bytes unchanged).
- Python: ProbeResult.sm_check is the last field, 0 by default, so every other field keeps its position."""
import ctypes as C
import dataclasses
import os
import re
import shutil
import subprocess

import pytest

from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200dp.h")
SM_CHECK_TEXT = "sm_check= wants a whole number of ms in [0, 10000]"
FAULT_TEXT = "sm_check_fault= wants <smid>+<mask>, an SM id in [0, 255] and a 32-bit mask"
OFF_LINE = "SM checks are off (sm_check=5): probe=off runs no probe pass"


def _open_error(pkg, uri):
    with pytest.raises(pkg._native.B2dpError) as ei:
        pkg.Context(uri)
    return ei.value.code, ei.value.detail


@pytest.fixture
def logs(pkg):
    got = []
    pkg._native.set_log_callback(lambda level, msg: got.append((level, msg)))
    try:
        yield got
    finally:
        pkg._native.set_log_callback(None)


def test_sm_check_opens_on_the_nvml_stub_and_says_it_is_off(pkg, monkeypatch, stub, tmp_path, logs):  # noqa: F811
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0, ",sm_check=5,sm_check_fault=3+0x80000000") as ctx:
        assert len(ctx.enumerate()) == 2
    assert [(lv, m) for lv, m in logs if "SM check" in m] == [(1, OFF_LINE)], logs


def test_sm_check_zero_and_the_largest_value_open(pkg, monkeypatch, stub, tmp_path, logs):  # noqa: F811
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 1, 0, ",sm_check=0"):
        pass
    assert not [m for _, m in logs if "SM check" in m]                 # off: nothing to say
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 1, 0, ",sm_check=10000,sm_check_fault=255+4294967295"):
        pass
    assert [m for _, m in logs if "SM check" in m] == ["SM checks are off (sm_check=10000): probe=off runs no probe pass"]


@pytest.mark.parametrize("value", ["abc", "-1", "10001", "", "5ms", " 5", "+5", "0x10", "1e3", "99999999999999999999"])
def test_malformed_sm_check_is_refused(pkg, monkeypatch, stub, tmp_path, value):  # noqa: F811
    N = pkg._native
    with pytest.raises(N.B2dpError) as ei:
        open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 1, 0, ",sm_check=" + value)
    assert (ei.value.code, ei.value.detail) == (N.E_INVAL, SM_CHECK_TEXT)


@pytest.mark.parametrize("value", ["", "3", "3+", "+1", "abc+1", "3+xyz", "-1+1", "256+1", "3+0x100000000",
                                   "3+4294967296", "3+1+2", "3 +1", "0x3+1"])
def test_malformed_sm_check_fault_is_refused(pkg, monkeypatch, stub, tmp_path, value):  # noqa: F811
    N = pkg._native
    with pytest.raises(N.B2dpError) as ei:
        open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 1, 0, ",sm_check=5,sm_check_fault=" + value)
    assert (ei.value.code, ei.value.detail) == (N.E_INVAL, FAULT_TEXT)


def test_keys_are_checked_before_any_device_is_touched(pkg):
    """The parse comes first: a bad value is refused the same way on a host with no GPU and no NVML stub."""
    N = pkg._native
    assert _open_error(pkg, "cuda:sm_check=abc") == (N.E_INVAL, SM_CHECK_TEXT)
    assert _open_error(pkg, "cuda:sm_check_fault=1") == (N.E_INVAL, FAULT_TEXT)


def test_header_flag_and_field():
    hdr = open(HEADER).read()
    assert re.search(r"^#define B2DP_RES_SM_CHECK 0x1000u\b", hdr, re.M)
    body = re.search(r"typedef struct b2dp_probe_result \{(.*?)\} b2dp_probe_result;", hdr, re.S).group(1)
    fields = re.findall(r"^\s+\w+ (\w+);", body, re.M)
    assert fields[-1] == "sm_check" and "reserved" not in fields, fields


def test_sm_check_sits_at_the_old_reserved_offset(pkg, tmp_path):
    """offsetof(b2dp_probe_result, sm_check) == 84, the last 4 bytes of the 88 the struct has always had."""
    N = pkg._native
    assert N.ProbeResult.sm_check.offset == 84 and C.sizeof(N.ProbeResult) == 88
    assert N.RES_SM_CHECK == 0x1000
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200dp.h"\nint main(void) {\n'
                   'printf("%zu %zu %u\\n", offsetof(b2dp_probe_result, sm_check), sizeof(b2dp_probe_result), '
                   '(unsigned)B2DP_RES_SM_CHECK); return 0; }\n')
    exe = str(tmp_path / "off")
    r = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([exe], capture_output=True, text=True).stdout.split() == ["84", "88", "4096"]


def test_python_probe_result_keeps_its_field_order(pkg):
    from importlib import import_module
    ctx_mod = import_module(pkg.__name__ + ".context")
    names = [f.name for f in dataclasses.fields(ctx_mod.ProbeResult)]
    assert names == ["device", "healthy", "err", "seed", "checksum", "expected_checksum", "mismatches",
                     "first_bad_word", "bytes", "ms_event", "ms_device", "gbs", "flags", "gbs_ref", "frac",
                     "min_gbs_applied", "sm_check"]
    r = ctx_mod.ProbeResult(0, True, 0, 1, 2, 2, 0, 0, 8, 0.0, 1.0, 8.0)
    assert r.sm_check == 0 and r.flags == 0
