"""The heartbeat's SM check (cuda: sm_check=<ms>) on a real H100.

- Rotation: eleven passes run the ten SM self-tests in header order and then the first again, each Healthy on every SM;
  the HBM pass of each call still matches oracle/probe.py, the probe ring holds exactly what the passes wrote, and
  every slice hands its device memory back before the call returns.
- Fault through the heartbeat: with sm_check_fault= every suite's failure is reported Unhealthy (RES_COMPUTE) by the
  very call that ran it, while the HBM fields stay clean; a ListAndWatch heartbeat and the library's watch loop report
  it too.
- A GPU another process uses gets no slice and its rotation waits; prearm=1 does not arm while sm_check is on.

Every slice is short: 5 ms per format (the synchronization suite takes about 350 ms whatever the setting)."""
import queue
import re
import subprocess
import sys
import time

import numpy as np
import pytest

from oracle import probe as oprobe

pytestmark = pytest.mark.gpu

MiB = 1 << 20
NBYTES = 64 * MiB
URI = "cuda:devices=0,bytes=%d,calib=1,sm_check=5" % NBYTES
# DiagSuite::log_name of each SmTest, in the header's order (b2dp_probe_result.sm_check = index + 1)
LOG_NAMES = ["compute test", "FP test", "SFU test", "shared-memory test", "register-file test", "integer test",
             "L2 test", "half-precision test", "sync test", "L1 test"]
LINE = re.compile(r"^(\S+) SM check (.+?): (Healthy|Unhealthy \(latched\)), SMs (\d+)/(\d+), mismatches \S+ "
                  r"(\d+)/(\d+)/(\d+), ([\d.]+)/([\d.]+)/([\d.]+) ms, ([\d.]+) ms on the worker(.*)$")


def _gpu_busy():
    """True if NVML lists a compute process on GPU 0 besides this one (the rule the SM check applies).  None if NVML
    cannot tell."""
    try:
        import pynvml
        pynvml.nvmlInit()
        return len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0))) > 1
    except Exception:       # noqa: BLE001
        return None


@pytest.fixture
def logs(pkg):
    got = []
    pkg._native.set_log_callback(lambda level, msg: got.append((level, msg)))
    try:
        yield got
    finally:
        pkg._native.set_log_callback(None)


def _slices(logs):
    """(level, match) of every SM check line logged since `logs` was last cleared."""
    out = []
    for level, msg in logs:
        m = LINE.match(msg)
        if m:
            out.append((level, m))
    return out


@pytest.fixture(scope="module")
def fault_sm(pkg):
    """An SM id that runs CTAs: the first one the on-demand compute self-test attributes an injected fault to."""
    with pkg.Context("cuda:devices=0,bytes=%d,calib=1" % NBYTES) as ctx:
        for s in range(16):
            (r,) = ctx.compute_test(0, duration_ms=10, fault_sm=s, fault_mask=1)
            ctx.probe_reset(0)
            if r.bad_sms() == [s]:
                return s
    pytest.fail("no SM id in 0..15 ran a CTA of the compute self-test")


def test_rotation_runs_every_suite_in_order_and_leaves_the_pass_alone(pkg, logs):
    import torch
    torch.cuda.init()
    N = pkg._native
    if _gpu_busy():
        pytest.skip("another process uses the GPU: no SM check runs on it")
    n_words = NBYTES // 4
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    with pkg.Context(URI) as ctx:
        for _ in range(10):                                    # one rotation loads every suite's kernels: not counted
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert p.healthy and p.flags & N.RES_SM_CHECK, p
        seed = None
        walls = []
        for k in range(11):
            src = ctx.probe_peek(0, 0, n_words)
            del logs[:]
            free0, _ = torch.cuda.mem_get_info(0)
            (p,) = ctx.probe_health(min_gbs=1e-3)
            free1, _ = torch.cuda.mem_get_info(0)
            assert p.healthy and p.err == 0, p
            assert p.flags & N.RES_SM_CHECK and not p.flags & N.RES_COMPUTE, p
            assert p.sm_check == k % 10 + 1, (k, p.sm_check)
            if seed is not None:
                assert p.seed == seed
            cs, bad, _, _ = oprobe.probe_pass(src, p.seed, oprobe.next_seed(p.seed))
            assert (p.checksum, p.mismatches, bad) == (cs, 0, 0) and p.checksum == p.expected_checksum, p
            seed = oprobe.next_seed(p.seed)
            # the ring holds what the pass wrote and nothing a slice wrote
            assert np.array_equal(ctx.probe_peek(0, 0, n_words), oprobe.pattern(n_words, seed)), k
            assert abs(free1 - free0) < 2 * MiB, (k, free0, free1)
            got = _slices(logs)
            assert len(got) == 1, logs
            level, m = got[0]
            assert level == 0 and m.group(2) == LOG_NAMES[k % 10] and m.group(3) == "Healthy", m.group(0)
            assert (m.group(6), m.group(7), m.group(8), m.group(13)) == ("0", "0", "0", ""), m.group(0)
            assert int(m.group(5)) == sms
            if not _gpu_busy():
                assert int(m.group(4)) == sms, m.group(0)
            walls.append((m.group(2), [float(m.group(i)) for i in (9, 10, 11)], float(m.group(12))))
    for name, ms, wall in walls:
        print("%-20s kernel %s ms, %.1f ms on the worker" % (name, "/".join("%.1f" % x for x in ms), wall))


def test_every_suites_fault_reaches_the_same_call(pkg, fault_sm, logs):
    N = pkg._native
    if _gpu_busy():
        pytest.skip("another process uses the GPU: no SM check runs on it")
    with pkg.Context(URI + ",sm_check_fault=%d+1" % fault_sm) as ctx:
        for k in range(1, 11):
            del logs[:]
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.healthy and p.flags & N.RES_COMPUTE and p.flags & N.RES_SM_CHECK, (k, p)
            assert (p.sm_check, p.err, p.mismatches) == (k, 0, 0), p
            assert p.checksum == p.expected_checksum
            got = _slices(logs)
            assert len(got) == 1, logs
            level, m = got[0]
            assert level == 2 and m.group(2) == LOG_NAMES[k - 1] and m.group(3) == "Unhealthy (latched)", m.group(0)
            assert m.group(13) == "", m.group(0)                 # a wrong result, not a CUDA error or a timeout
            ctx.probe_reset(0)
        # the latch outlives the call that set it: the heartbeat that follows a faulted slice is Unhealthy
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.sm_check == 1 and p.flags & N.RES_COMPUTE and not p.healthy
        _, st = ctx.list_and_watch("gpu", N.LW_HEARTBEAT, min_gbs=1e-3)
        assert st.n_unhealthy == 1 and st.probe_bytes == 2 * NBYTES
        ctx.probe_reset(0)
    with pkg.Context(URI) as ctx:                               # and the same rotation without the hook is Healthy
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and p.sm_check == 1 and not p.flags & N.RES_COMPUTE, p


def _nvml_procs():
    import pynvml
    pynvml.nvmlInit()
    return len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0)))


def test_a_busy_gpu_gets_no_slice_and_its_rotation_waits(pkg):
    N = pkg._native
    helper = subprocess.Popen([sys.executable, "-c",
                               "import torch,time; torch.zeros(1, device='cuda:0'); print('ready', flush=True); time.sleep(60)"],
                              stdout=subprocess.PIPE, text=True)
    try:
        assert helper.stdout.readline().strip() == "ready"
        with pkg.Context(URI + ",sm_check_fault=0+1") as ctx:
            try:
                seen = _nvml_procs()
            except Exception as e:       # noqa: BLE001
                pytest.skip("NVML process accounting unavailable: %s" % e)
            if seen < 2:                                            # the child and this process
                pytest.skip("NVML does not list foreign compute processes in this container")
            for _ in range(3):
                (p,) = ctx.probe_health(min_gbs=1e-3)
                assert p.sm_check == 0 and not p.flags & (N.RES_SM_CHECK | N.RES_COMPUTE), p
                assert p.healthy and p.err == 0, p
            helper.kill()
            helper.wait()
            deadline = time.time() + 20
            while _nvml_procs() > 1 and time.time() < deadline:     # this process holds one context itself
                time.sleep(0.2)
            if _nvml_procs() > 1:
                pytest.skip("NVML still lists another compute process on GPU 0")
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert p.flags & N.RES_SM_CHECK and p.sm_check == 1, p     # the rotation starts where it stood
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def test_prearm_does_not_arm_with_sm_check(pkg):
    N = pkg._native
    with pkg.Context("cuda:devices=0,bytes=%d,calib=1,prearm=1" % NBYTES) as ctx:     # without sm_check: it arms
        armed = [ctx.probe_health(timed=False, min_gbs=1e-3)[0].flags & N.RES_PREARMED for _ in range(4)]
    if not any(armed):
        pytest.skip("prearm=1 does not arm on this driver (no cuStreamWaitValue32)")
    if _gpu_busy():
        pytest.skip("another process uses the GPU: no SM check runs on it")
    with pkg.Context(URI + ",prearm=1") as ctx:
        for k in range(5):
            (p,) = ctx.probe_health(timed=False, min_gbs=1e-3)
            assert p.healthy and p.flags & N.RES_SM_CHECK and p.sm_check == k + 1, p
            assert not p.flags & N.RES_PREARMED, p


def test_watch_loop_reports_a_faulted_slice_in_its_first_heartbeat(pkg, fault_sm):
    if _gpu_busy():
        pytest.skip("another process uses the GPU: no SM check runs on it")
    got = queue.Queue()
    with pkg.Context(URI + ",sm_check_fault=%d+1" % fault_sm) as ctx:
        w = ctx.watch(lambda rc, wire, st: got.put((rc, wire, st)), pulse_ms=200, min_gbs=1e-3)
        try:
            rc, wire, st = got.get(timeout=30)
            assert rc == 0 and st.probe_bytes == 0                      # stream start: no probe, all Healthy
            rc, wire, st = got.get(timeout=60)
            assert rc == 0 and st.probe_bytes == 2 * NBYTES and st.n_unhealthy == 1, st
            assert [d.health for d in pkg.v1beta1.ListAndWatchResponse.FromString(wire).devices] == ["Unhealthy"]
        finally:
            w.stop()
