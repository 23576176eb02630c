"""GPU tests of the on-demand shared-memory self-test (b2dp_smem_test, csrc/smem_selftest.cuh).

Through tests/native/libsmem_test_kernels_test.so (the kernel launched directly, one format at a time):
  - the DUMP instantiation's final array image, every thread's fold and direct-compare count equal
    tests/smem_test_oracle.py bit for bit, in every format, tile and CTA;
  - one CTA runs on every SM id for SH_WORD / SH_BYTE, and the two CTAs of every SH_DSMEM cluster report equal rounds;
  - a flip at a chosen word, after a chosen element, is counted in exactly the first comparison, by exactly the CTA on
    the chosen SM (SH_DSMEM: that CTA and its cluster peer), across banks, the first and last words and the v4 tail.
Through the ABI: a clean run, fault attribution, the latch and b2dp_probe_reset, the busy skip, the memory left
free, and the daemon's start-up test.
"""
import ctypes as C
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import smem_test_oracle as so

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "native", "libsmem_test_kernels_test.so")
MiB = 1 << 20
MS = 1000000
FMT_IDS = [so.NAMES[f] for f in so.FORMATS]
_P = C.POINTER


class CtRecord(C.Structure):
    _fields_ = [("smid", C.c_uint32), ("nsmid", C.c_uint32), ("rounds", C.c_uint64), ("comparisons", C.c_uint64),
                ("mismatches", C.c_uint64), ("first_bad_tile", C.c_int32), ("first_bad_rep", C.c_int32),
                ("seq", C.c_uint64)]


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.sh_open.restype = C.c_void_p
        L.sh_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.sh_close.argtypes = [C.c_void_p]
        L.sh_error.restype = C.c_char_p
        L.sh_error.argtypes = [C.c_void_p]
        for f in (L.sh_sms, L.sh_clusters):
            f.argtypes = [C.c_void_p]
        L.sh_grid.argtypes = [C.c_void_p, C.c_int]
        L.sh_occupancy.argtypes = [C.c_void_p, C.c_int, _P(C.c_int)]
        L.sh_dump.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32,
                              _P(C.c_uint32), _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float)]
        L.sh_run.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32,
                             _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float)]
        assert L.sh_record_bytes() == C.sizeof(CtRecord)
        assert L.sh_dump_words() == so.DUMP_WORDS
        self.L = L
        err = C.create_string_buffer(512)
        self.h = L.sh_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("sh_open: " + err.value.decode())
        self.sms = L.sh_sms(self.h)
        self.clusters = L.sh_clusters(self.h)

    def close(self):
        if self.h:
            self.L.sh_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == 1:
            raise RuntimeError("%s: %s" % (what, self.L.sh_error(self.h).decode()))
        assert rc == 0, "%s refused: code %d" % (what, rc)

    def grid(self, fmt):
        return self.L.sh_grid(self.h, fmt)

    def dump(self, fmt, seed, hook=(so.HOOK_WORD, so.HOOK_ELEMENT), fault_sm=-1, fault_mask=0):
        g = self.grid(fmt)
        out = np.zeros((g, so.TILES, so.DUMP_WORDS), dtype=np.uint32)
        recs = (CtRecord * g)()
        n, ms = C.c_int(), C.c_float()
        self._check(self.L.sh_dump(self.h, fmt, seed, hook[0], hook[1], fault_sm, fault_mask,
                                   out.ctypes.data_as(_P(C.c_uint32)), recs, g, C.byref(n), C.byref(ms)), "sh_dump")
        return out, list(recs[:n.value]), ms.value

    def run(self, fmt, seed, duration_ms, hook=(so.HOOK_WORD, so.HOOK_ELEMENT), fault_sm=-1, fault_mask=0):
        g = self.grid(fmt)
        recs = (CtRecord * g)()
        n, ms = C.c_int(), C.c_float()
        self._check(self.L.sh_run(self.h, fmt, seed, int(duration_ms * MS), hook[0], hook[1], fault_sm, fault_mask,
                                  recs, g, C.byref(n), C.byref(ms)), "sh_run")
        return list(recs[:n.value]), ms.value


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _gpu_busy():
    try:
        import pynvml
        pynvml.nvmlInit()
        return len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0))) > 1
    except Exception:       # noqa: BLE001
        return None


def _arrived(recs, seq=7):
    for r in recs:
        assert r.seq == seq and r.rounds >= 1 and r.comparisons == r.rounds * so.TILES * so.REPS, \
            (r.smid, r.seq, r.rounds, r.comparisons)
        assert r.smid < r.nsmid <= 256


def _check_clean(recs):
    _arrived(recs)
    for r in recs:
        assert r.mismatches == 0 and (r.first_bad_tile, r.first_bad_rep) == (-1, -1), (r.smid, r.mismatches)


# ---- the kernel against the oracle --------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_dump_equals_the_oracle(H, fmt):
    seed = 0xC0FFEE17
    d, recs, _ = H.dump(fmt, seed)
    _check_clean(recs)
    assert all(r.rounds == 1 for r in recs)
    for t in range(so.TILES):
        want = so.march(fmt, so.kind(t), so.key(seed, fmt, t))
        for cta in range(len(recs)):
            rank = cta % 2
            img = want["image"][rank] if fmt == so.DSMEM else want["image"]
            fold = want["fold"][rank] if fmt == so.DSMEM else want["fold"]
            got = d[cta, t]
            assert np.array_equal(got[:so.WORDS], img), (t, cta, np.argwhere(got[:so.WORDS] != img)[:4].ravel())
            assert np.array_equal(got[so.WORDS:so.WORDS + so.THREADS], fold), (t, cta)
            assert not got[so.WORDS + so.THREADS:].any(), (t, cta)


def test_every_sm_id_runs_exactly_one_cta(H):
    for fmt in (so.WORD, so.BYTE):
        recs, _ = H.run(fmt, 1, 0)
        _check_clean(recs)
        ids = [r.smid for r in recs]
        assert len(recs) == H.sms and sorted(ids) == sorted(set(ids)), (fmt, len(recs), H.sms)
        assert len(set(ids)) == H.sms


def test_dsmem_clusters_run_equal_rounds(H):
    occ = {f: C.c_int() for f in so.FORMATS}
    rcs = {f: H.L.sh_occupancy(H.h, f, C.byref(occ[f])) for f in so.FORMATS}
    print("smem test: %d SMs, cudaOccupancyMaxActiveClusters(SH_DSMEM) = %d clusters of two (%d CTAs); "
          "cudaOccupancyMaxActiveBlocksPerMultiprocessor rc/ctas: %s"
          % (H.sms, H.clusters, 2 * H.clusters, {so.NAMES[f]: (rcs[f], occ[f].value) for f in so.FORMATS}))
    assert H.clusters >= 1 and H.grid(so.DSMEM) == 2 * H.clusters <= H.sms
    for f in (so.WORD, so.BYTE):
        assert rcs[f] == 0 and occ[f].value == 1, (f, rcs[f], occ[f].value)
    recs, ms = H.run(so.DSMEM, 2, 200)
    _check_clean(recs)
    for i in range(0, len(recs), 2):
        a, b = recs[i], recs[i + 1]
        assert (a.rounds, a.comparisons) == (b.rounds, b.comparisons) and a.smid != b.smid, (i, a.rounds, b.rounds)
    assert len({r.smid for r in recs}) == len(recs)
    assert ms >= 190


FAULT_WORDS = [0, 31, 1000 + 17, so.HOOK_WORD, 4 * (so.VPT * so.THREADS) + 5, so.WORDS - 1]   # ... v4 tail, last word


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_flip_is_counted_in_exactly_its_comparison_by_exactly_its_cta(H, fmt):
    recs, _ = H.run(fmt, 3, 0)
    _check_clean(recs)
    smids = [r.smid for r in recs]
    targets = [0, len(recs) // 2 + 1, len(recs) - 1]
    n = 0
    for e in range(so.ELEMENTS[fmt] - 1):
        for w in FAULT_WORDS:
            for mask in (0x1, 0x80000000, 0x00010100):
                cta = targets[n % len(targets)]
                n += 1
                s = smids[cta]
                got, _ = H.run(fmt, 3, 0, hook=(w, e), fault_sm=s, fault_mask=mask)
                _arrived(got)
                # the CTA on s, and for SH_DSMEM its cluster peer, count exactly the first comparison
                hit = {i for i, r in enumerate(got) if r.smid == s}
                assert len(hit) == 1, (e, w, s)
                if fmt == so.DSMEM:
                    (i,) = hit
                    hit.add(i ^ 1)
                for i, r in enumerate(got):
                    want = (1, 0, 0) if i in hit else (0, -1, -1)
                    assert (r.mismatches, r.first_bad_tile, r.first_bad_rep) == want, (e, w, hex(mask), i, r.smid, s)


# ---- through the ABI ----------------------------------------------------------------------------------------------
def _open(pkg, nbytes=64 * MiB):
    return pkg.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


def test_smem_test_clean_and_memory_back(pkg, H):
    import torch
    torch.cuda.init()
    N = pkg._native
    with _open(pkg) as ctx:
        ctx.smem_test(0, duration_ms=10)                       # first launch loads the kernels: not counted below
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.smem_test(0, duration_ms=100)
        free1, _ = torch.cuda.mem_get_info(0)
        assert r.healthy and r.err == 0, r
        assert r.mismatches == [0, 0, 0] and r.bad_sm_mask == [0, 0, 0, 0], r
        assert not r.flags & N.CT_ECC, r
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (-1, -1, -1)
        assert r.sm_count == torch.cuda.get_device_properties(0).multi_processor_count
        assert all(ms >= 90 for ms in r.ms) and all(t > 0 for t in r.tflops), r
        if 2 * H.clusters == r.sm_count and not _gpu_busy():
            assert r.sms_covered == r.sm_count and not r.flags & N.CT_PARTIAL_COVERAGE, r
        elif 2 * H.clusters < r.sm_count:
            assert r.flags & N.CT_PARTIAL_COVERAGE and r.sms_covered <= 2 * H.clusters, r
        assert abs(free1 - free0) < 2 * MiB, (free0, free1)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE
    print("smem test 100 ms/format: flags 0x%x, SMs %d/%d, ms %s, TB/s word %.2f byte %.2f dsmem %.2f"
          % (r.flags, r.sms_covered, r.sm_count, ["%.1f" % x for x in r.ms], *r.tflops))


@pytest.mark.parametrize("where", ["first", "last"])
def test_smem_test_fault_is_attributed_and_latched_until_reset(pkg, H, where):
    N = pkg._native
    recs, _ = H.run(so.WORD, 1, 0)
    ids = sorted(r.smid for r in recs)
    s = ids[0] if where == "first" else ids[-1]
    with _open(pkg) as ctx:
        (r,) = ctx.smem_test(0, duration_ms=10, fault_sm=s, fault_mask=0x80000000)
        assert not r.healthy and r.err == 0, r
        assert s in r.bad_sms() and (r.first_bad_sm, r.first_bad_tile) == (s, 0), r
        assert r.first_bad_format == N.SH_WORD and r.mismatches[0] == 1 and r.mismatches[1] == 1, r
        assert r.mismatches[2] in (0, 2), r      # 2: the SM runs a DSMEM CTA, and its cluster peer counts it too
        assert len(r.bad_sms()) == (1 if r.mismatches[2] == 0 else 2), r.bad_sms()
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & N.RES_COMPUTE and not p.healthy and p.mismatches == 0
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE
        (r,) = ctx.smem_test(0, duration_ms=10)
        assert r.healthy and r.bad_sm_mask == [0, 0, 0, 0], r


def test_smem_test_skips_a_busy_gpu(pkg):
    N = pkg._native
    helper = subprocess.Popen([sys.executable, "-c",
                               "import torch,time; torch.zeros(1, device='cuda:0'); print('ready', flush=True); time.sleep(60)"],
                              stdout=subprocess.PIPE, text=True)
    try:
        assert helper.stdout.readline().strip() == "ready"
        try:
            import pynvml
            pynvml.nvmlInit()
            seen = len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0)))
        except Exception as e:       # noqa: BLE001
            pytest.skip("NVML process accounting unavailable: %s" % e)
        if seen < 1:
            pytest.skip("NVML does not list foreign compute processes in this container")
        with _open(pkg) as ctx:
            (r,) = ctx.smem_test(0, duration_ms=10, fault_sm=0, fault_mask=1)
            assert r.flags & N.CT_SKIPPED_BUSY and r.mismatches == [0, 0, 0] and r.ms == [0, 0, 0], r
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & N.RES_COMPUTE
            (r,) = ctx.smem_test(0, duration_ms=10, even_if_busy=True)
            assert not r.flags & N.CT_SKIPPED_BUSY and r.healthy and r.err == 0, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def test_daemon_smem_test_at_start_logs_a_clean_result(short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")

    def lines(level):
        proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", short_dir,
                                 "-start_retry_wait=0.05", "-smem_test_at_start=%d" % level, "-compute_test_ms=50"],
                                stderr=subprocess.PIPE, text=True)
        got = []
        try:
            t0 = time.time()
            while time.time() - t0 < 120:
                line = proc.stderr.readline()
                if not line:
                    break
                got.append(line)
                if "Failed to start plugin" in line:
                    break
        finally:
            proc.send_signal(signal.SIGINT)
            rest = proc.communicate(timeout=30)[1]
        log = "".join(got) + rest
        assert proc.returncode == 0, log[-3000:]
        assert log.index("smem test ") < log.index("Failed to start plugin"), log[-3000:]
        return [ln for ln in log.splitlines() if ln.startswith("smem test ")], log

    got, log = lines(1)
    assert len(got) == 1, log[-3000:]
    if "flags 0x1," in got[0]:
        got, log = lines(2)
        assert len(got) == 1, log[-3000:]
    assert ": Healthy, flags 0x" in got[0] and "mismatches 0/0/0, first bad SM -1" in got[0], log[-3000:]
