"""Context: one opened backend of libb200dp (`kfd:<sysroot>` parity mode or `cuda:` real H100s)."""
import ctypes as C
import threading
from dataclasses import dataclass
from typing import Dict, List, Optional

from . import _native as N


@dataclass
class ProbeResult:
    device: int
    healthy: bool
    err: int
    seed: int
    checksum: int
    expected_checksum: int
    mismatches: int
    first_bad_word: int
    bytes: int
    ms_event: float
    ms_device: float
    gbs: float
    flags: int = 0
    gbs_ref: float = 0.0           # the device's calibrated ceiling
    frac: float = 0.0              # gbs / gbs_ref
    min_gbs_applied: float = 0.0   # the floor the verdict used


@dataclass
class MemtestResult:
    device: int
    healthy: bool
    err: int
    flags: int
    seed: int
    n_segments: int
    bytes_tested: int
    free_before: int
    total_memory: int
    mismatches: List[int]          # per march element: E0 w(P), E1 r(P) w(~P), E2 r(~P) w(P), E3 r(P)
    first_bad_word: int
    ecc_corrected: int
    ecc_uncorrected: int
    ms: float
    gbs: float                     # 6 x bytes_tested / ms


@dataclass
class ComputeTestResult:
    device: int
    healthy: bool
    err: int
    flags: int
    seed: int
    sm_count: int
    nsmid: int
    sms_covered: int               # SM ids on which every format ran at least one CTA
    bad_sm_mask: List[int]         # 4 x 64 bits over %smid
    mismatches: List[int]          # per format: BF16, FP8, INT8 (fp_test: FP32, FP64, DMMA)
    first_bad_sm: int
    first_bad_format: int
    first_bad_tile: int
    ms: List[float]
    tflops: List[float]            # 2 M N K x result tiles compared / ms (TOPS for INT8; fp_test: 2 x FMAs / ms;
                                   # sfu_test: MUFU results / ms, in T results/s; smem_test, regfile_test: TB/s;
                                   # int_test, half_test: result words / ms, in T results/s; l2_test: TB/s, TB/s,
                                   # G ops/s; sync_test: G ops/s, G ops/s, T results/s; l1_test: TB/s)

    def bad_sms(self) -> List[int]:
        return [s for s in range(256) if (self.bad_sm_mask[s // 64] >> (s % 64)) & 1]


@dataclass
class HostlinkResult:
    device: int
    healthy: bool
    err: int
    flags: int
    seed: int
    sm_count: int
    sms_covered: int               # SM ids that ran a CTA of the SM format
    host_numa_node: int            # -1: the host buffers were not bound (HL_NUMA_UNBOUND)
    bad_sm_mask: List[int]         # 4 x 64 bits over %smid
    rounds: List[int]              # per format: H2D, D2H, SM
    mismatches: List[int]          # wrong words, device-side and host-side checks together
    first_bad_word: List[int]      # 2^64 - 1 if none
    replays: int                   # NVML PCIe replay counter delta
    ms: List[float]                # summed event time of the transfers
    gbs: List[float]               # bytes x rounds / ms (SM: read plus written)
    link_gen: int                  # sampled while a transfer was in flight (0: NVML gave none)
    link_width: int
    max_link_gen: int
    max_link_width: int
    link_gbs: float                # per-direction capacity of link_gen x link_width

    def bad_sms(self) -> List[int]:
        return [s for s in range(256) if (self.bad_sm_mask[s // 64] >> (s % 64)) & 1]


@dataclass
class CycleStats:
    n_devices: int
    n_unhealthy: int
    homogeneous: bool
    node_healthy: bool
    ms_total: float
    ms_enumerate: float
    ms_probe: float
    ms_encode: float
    probe_gbs_min: float
    probe_gbs_sum: float
    probe_bytes: int
    ms_link_check: float = 0.0
    n_link_faults: int = 0
    probe_ms_device_max: float = 0.0
    probe_frac_min: float = 0.0


class Context:
    def __init__(self, uri: str):
        self.uri = uri
        self._h = C.c_void_p()
        rc = N.lib.b2dp_open(uri.encode(), C.byref(self._h))
        if rc != N.OK:
            raise N.B2dpError(rc, N.lib.b2dp_last_error(None).decode())
        self._buf = (C.c_uint8 * (1 << 16))()
        self._buf_lock = threading.Lock()      # one response buffer, several gRPC handler threads
        self._opts_cache = {}

    def close(self):
        if self._h:
            N.lib.b2dp_close(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- enumerate -----------------------------------------------------------------------
    def enumerate_raw(self):
        rc, arr, n = N.grow_call(lambda cap: (N.Device * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_enumerate(self._h, a, cap, pn))
        N.check(rc, self._h)
        return arr, n

    def enumerate(self) -> Dict[str, dict]:
        """GetAMDGPUs()-shaped map (amdgpu.go:216), canonical order (sorted by id)."""
        arr, n = self.enumerate_raw()
        return {N.s(d.id): {"card": d.card, "renderD": d.render_d, "devID": N.s(d.dev_id),
                            "computePartitionType": N.s(d.compute_partition),
                            "memoryPartitionType": N.s(d.memory_partition), "numaNode": d.numa_node,
                            "nodeId": d.node_id} for d in arr[:n]}

    def partition_histogram(self) -> Dict[str, int]:
        rc, arr, n = N.grow_call(lambda cap: (N.KvCount * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_partition_histogram(self._h, a, cap, pn))
        N.check(rc, self._h)
        return {N.s(e.key): e.count for e in arr[:n]}

    def is_homogeneous(self) -> bool:
        v = C.c_int32()
        N.check(N.lib.b2dp_is_homogeneous(self._h, C.byref(v)), self._h)
        return bool(v.value)

    def partition_supported(self, which: int) -> bool:
        v = C.c_int32()
        N.check(N.lib.b2dp_partition_supported(self._h, which, C.byref(v)), self._h)
        return bool(v.value)

    def resource_list(self, strategy: str) -> List[str]:
        rc, arr, n = N.grow_call(lambda cap: (N.Id64 * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_resource_list(self._h, strategy.encode(), a, cap, pn))
        N.check(rc, self._h)
        return [N.s(arr[i].value) for i in range(n)]

    # ---- health --------------------------------------------------------------------------
    def node_health(self) -> bool:
        v = C.c_int32()
        N.check(N.lib.b2dp_node_health(self._h, C.byref(v)), self._h)
        return bool(v.value)

    def probe_health(self, timeout_ms=0, variant=N.PROBE_VARIANT_TMA, min_gbs=0.0, via_workers=False,
                     timed=True, grid_ctas=0) -> List[ProbeResult]:
        """One fan-out pass.  timed=True brackets each kernel with CUDA events (ms_event, what the roofline
        is measured with); timed=False is the kubelet-facing configuration (completion by the published
        result block alone, GB/s from the in-kernel timer)."""
        opts = N.ProbeOpts(timeout_ms, variant | (N.PROBE_VIA_WORKERS if via_workers else 0)
                           | (N.PROBE_EVENT_TIMING if timed else 0), min_gbs, grid_ctas)
        rc, arr, n = N.grow_call(lambda cap: (N.ProbeResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_probe_health(self._h, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ProbeResult(r.device, bool(r.healthy), r.err, r.seed, r.checksum, r.expected_checksum, r.mismatches,
                            r.first_bad_word, r.bytes, r.ms_event, r.ms_device, r.gbs, r.flags, r.gbs_ref, r.frac,
                            r.min_gbs_applied) for r in arr[:n]]

    def probe_inject_fault(self, device: int, word_index: int, mask: int):
        N.check(N.lib.b2dp_probe_inject_fault(self._h, device, word_index, mask), self._h)

    def probe_reset(self, device: int = -1):
        N.check(N.lib.b2dp_probe_reset(self._h, device), self._h)

    def probe_set_ref(self, device: int = -1, gbs_ref: float = 0.0):
        """Pin the bandwidth ceiling the fractional floor refers to (<= 0: back to the device's own calibration)."""
        N.check(N.lib.b2dp_probe_set_ref(self._h, device, gbs_ref), self._h)

    def probe_describe(self, device: int) -> dict:
        """Ring geometry, calibrated ceiling and runtime identity of `device` (b2dp_probe_describe); no pass runs."""
        info = N.ProbeInfo()
        N.check(N.lib.b2dp_probe_describe(self._h, device, C.byref(info)), self._h)
        return {"slot_bytes": info.slot_bytes, "total_memory": info.total_memory, "sm_count": info.sm_count,
                "slots": info.slots, "gbs_cal": info.gbs_cal, "gbs_ref": info.gbs_ref, "usable": bool(info.usable),
                "via_helper": bool(info.via_helper), "uuid": N.s(info.uuid), "name": N.s(info.name)}

    def probe_peek(self, device: int, word_index: int, n_words: int):
        import numpy as np
        out = np.empty(n_words, dtype=np.uint32)
        N.check(N.lib.b2dp_probe_peek(self._h, device, word_index, out.ctypes.data_as(C.POINTER(C.c_uint32)), n_words),
                self._h)
        return out

    def memtest(self, device: int = -1, max_bytes: int = 0, reserve_bytes: int = 0, timeout_ms: int = 0,
                even_if_busy: bool = False, fault_word: int = 0, fault_mask: int = 0) -> List[MemtestResult]:
        """On-demand march test of the free HBM of `device` (-1 = every GPU, b2dp_memtest).  max_bytes = 0 tests all
        free memory above the reserve (reserve_bytes = 0: 10 % of the device's memory).  A failure is latched: later
        probe results carry RES_MEMTEST and are Unhealthy until probe_reset().  fault_word / fault_mask is a test hook
        that flips bits of the tested span after the first element."""
        opts = N.MemtestOpts(max_bytes, reserve_bytes, timeout_ms, N.MT_EVEN_IF_BUSY if even_if_busy else 0, fault_word,
                             fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.MemtestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_memtest(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [MemtestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.n_segments, r.bytes_tested,
                              r.free_before, r.total_memory, list(r.mismatches), r.first_bad_word, r.ecc_corrected,
                              r.ecc_uncorrected, r.ms, r.gbs) for r in arr[:n]]

    def compute_test(self, device: int = -1, duration_ms: int = 0, timeout_ms: int = 0, even_if_busy: bool = False,
                     fault_sm: int = -1, fault_mask: int = 0) -> List[ComputeTestResult]:
        """On-demand tensor-core self-test of `device` (-1 = every GPU, b2dp_compute_test): BF16, FP8 and INT8 warpgroup
        GEMMs on every SM for duration_ms each (0 = 1000), every result compared bit for bit with the host's exact
        product.  A failure is latched: later probe results carry RES_COMPUTE and are Unhealthy until probe_reset().
        fault_sm / fault_mask is a test hook that flips bits of one accumulator on the SM with that %smid."""
        opts = N.ComputeTestOpts(duration_ms, timeout_ms, N.CT_EVEN_IF_BUSY if even_if_busy else 0, fault_sm, fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.ComputeTestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_compute_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ComputeTestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.nsmid, r.sms_covered,
                                  list(r.bad_sm_mask), list(r.mismatches), r.first_bad_sm, r.first_bad_format,
                                  r.first_bad_tile, list(r.ms), list(r.tflops)) for r in arr[:n]]

    def fp_test(self, device: int = -1, duration_ms: int = 0, timeout_ms: int = 0, even_if_busy: bool = False,
                fault_sm: int = -1, fault_mask: int = 0) -> List[ComputeTestResult]:
        """On-demand FP32 / FP64 self-test of `device` (-1 = every GPU, b2dp_fp_test): FFMA, DFMA and DMMA on every SM
        for duration_ms each (0 = 1000), every result compared bit for bit with the host's IEEE 754 result.  The
        per-format lists are indexed by FT_FP32, FT_FP64, FT_DMMA.  A failure is latched like compute_test()'s
        (RES_COMPUTE until probe_reset()); fault_sm / fault_mask flips bits of one result on the SM with that %smid."""
        opts = N.ComputeTestOpts(duration_ms, timeout_ms, N.CT_EVEN_IF_BUSY if even_if_busy else 0, fault_sm, fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.ComputeTestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_fp_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ComputeTestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.nsmid, r.sms_covered,
                                  list(r.bad_sm_mask), list(r.mismatches), r.first_bad_sm, r.first_bad_format,
                                  r.first_bad_tile, list(r.ms), list(r.tflops)) for r in arr[:n]]

    def sfu_test(self, device: int = -1, duration_ms: int = 0, timeout_ms: int = 0, even_if_busy: bool = False,
                 fault_sm: int = -1, fault_mask: int = 0) -> List[ComputeTestResult]:
        """On-demand SFU self-test of `device` (-1 = every GPU, b2dp_sfu_test): a reference launch of one CTA per SM
        whose result words' majority is bounded against the exact functions on the host, every dissenting SM named; then
        the MUFU ops on every SM for duration_ms per format (0 = 1000), compared with the majority.  The per-format
        lists are indexed by SF_F32, SF_ROOT, SF_F16; flags may carry CT_NO_CONSENSUS / CT_OUT_OF_BOUND.  A failure is
        latched like compute_test()'s (RES_COMPUTE until probe_reset()); fault_sm / fault_mask flips bits of one result
        on the SM with that %smid, in both launches."""
        opts = N.ComputeTestOpts(duration_ms, timeout_ms, N.CT_EVEN_IF_BUSY if even_if_busy else 0, fault_sm, fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.ComputeTestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_sfu_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ComputeTestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.nsmid, r.sms_covered,
                                  list(r.bad_sm_mask), list(r.mismatches), r.first_bad_sm, r.first_bad_format,
                                  r.first_bad_tile, list(r.ms), list(r.tflops)) for r in arr[:n]]

    def smem_test(self, device: int = -1, duration_ms: int = 0, timeout_ms: int = 0, even_if_busy: bool = False,
                  fault_sm: int = -1, fault_mask: int = 0) -> List[ComputeTestResult]:
        """On-demand shared-memory self-test of `device` (-1 = every GPU, b2dp_smem_test): one 227 KiB CTA per SM marches
        its whole array, and clusters of two march each other's, for duration_ms per format (0 = 1000).  The per-format
        lists are indexed by SH_WORD, SH_BYTE, SH_DSMEM; tflops holds TB/s; flags may carry CT_ECC_CORRECTED / CT_ECC /
        CT_NO_ECC.  A failure is latched like compute_test()'s (RES_COMPUTE until probe_reset()); fault_sm / fault_mask
        flips bits of one word of the array of the SM with that %smid, in the first comparison."""
        opts = N.ComputeTestOpts(duration_ms, timeout_ms, N.CT_EVEN_IF_BUSY if even_if_busy else 0, fault_sm, fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.ComputeTestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_smem_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ComputeTestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.nsmid, r.sms_covered,
                                  list(r.bad_sm_mask), list(r.mismatches), r.first_bad_sm, r.first_bad_format,
                                  r.first_bad_tile, list(r.ms), list(r.tflops)) for r in arr[:n]]

    def regfile_test(self, device: int = -1, duration_ms: int = 0, timeout_ms: int = 0, even_if_busy: bool = False,
                     fault_sm: int = -1, fault_mask: int = 0) -> List[ComputeTestResult]:
        """On-demand register-file self-test of `device` (-1 = every GPU, b2dp_regfile_test): two CTAs per SM hold 204
        values per thread in registers and march them, for duration_ms per format (0 = 1000).  The per-format lists
        are indexed by RF_ALU, RF_LOAD, RF_HOLD; tflops holds TB/s of register data; flags may carry CT_ECC_CORRECTED /
        CT_ECC / CT_NO_ECC.  A failure is latched like compute_test()'s (RES_COMPUTE until probe_reset()); fault_sm /
        fault_mask flips bits of one held register of one thread of the SM with that %smid, in the first comparison."""
        opts = N.ComputeTestOpts(duration_ms, timeout_ms, N.CT_EVEN_IF_BUSY if even_if_busy else 0, fault_sm, fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.ComputeTestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_regfile_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ComputeTestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.nsmid, r.sms_covered,
                                  list(r.bad_sm_mask), list(r.mismatches), r.first_bad_sm, r.first_bad_format,
                                  r.first_bad_tile, list(r.ms), list(r.tflops)) for r in arr[:n]]

    def int_test(self, device: int = -1, duration_ms: int = 0, timeout_ms: int = 0, even_if_busy: bool = False,
                 fault_sm: int = -1, fault_mask: int = 0) -> List[ComputeTestResult]:
        """On-demand integer and warp-exchange self-test of `device` (-1 = every GPU, b2dp_int_test): every SM's integer
        pipes (multiplier, adder and carries, logic, shifter, bit counts, byte permute, compare) and its shuffle / vote /
        redux / match network against results the host computed exactly, for duration_ms per format (0 = 1000).  The
        per-format lists are indexed by IT_MAD, IT_BIT, IT_WARP; tflops holds T result words/s.  A failure is latched
        like compute_test()'s (RES_COMPUTE until probe_reset()); fault_sm / fault_mask flips bits of one result word of
        one thread of the SM with that %smid, in the first comparison."""
        opts = N.ComputeTestOpts(duration_ms, timeout_ms, N.CT_EVEN_IF_BUSY if even_if_busy else 0, fault_sm, fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.ComputeTestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_int_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ComputeTestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.nsmid, r.sms_covered,
                                  list(r.bad_sm_mask), list(r.mismatches), r.first_bad_sm, r.first_bad_format,
                                  r.first_bad_tile, list(r.ms), list(r.tflops)) for r in arr[:n]]

    def l2_test(self, device: int = -1, duration_ms: int = 0, timeout_ms: int = 0, even_if_busy: bool = False,
                 fault_sm: int = -1, fault_mask: int = 0) -> List[ComputeTestResult]:
        """On-demand L2 self-test of `device` (-1 = every GPU, b2dp_l2_test): a March C- and a mixed-width march over
        an L2-resident span whose slices move between CTAs at every element, and the L2's atomic and reduction units,
        against values the host computed, for duration_ms per format (0 = 1000).  The per-format lists are indexed by
        L2_WORD, L2_BYTE, L2_ATOM; tflops holds TB/s, TB/s and G atomic ops/s.  A failure is latched like
        compute_test()'s (RES_COMPUTE until probe_reset()); fault_sm / fault_mask makes one CTA on the SM with that
        %smid flip bits of one word in the first comparison, which the CTA that reads the word next counts."""
        opts = N.ComputeTestOpts(duration_ms, timeout_ms, N.CT_EVEN_IF_BUSY if even_if_busy else 0, fault_sm, fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.ComputeTestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_l2_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ComputeTestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.nsmid, r.sms_covered,
                                  list(r.bad_sm_mask), list(r.mismatches), r.first_bad_sm, r.first_bad_format,
                                  r.first_bad_tile, list(r.ms), list(r.tflops)) for r in arr[:n]]

    def half_test(self, device: int = -1, duration_ms: int = 0, timeout_ms: int = 0, even_if_busy: bool = False,
                  fault_sm: int = -1, fault_mask: int = 0) -> List[ComputeTestResult]:
        """On-demand half-precision and conversion self-test of `device` (-1 = every GPU, b2dp_half_test): every SM's
        f16x2 and bf16x2 fma / add / sub / mul / min / max and its type converters (f32 to f16 / bf16 / fp8 / tf32, fp8
        to f16, float to and from integers, f64 to f32, round to integer) against results the host computed exactly,
        for duration_ms per format (0 = 1000).  The per-format lists are indexed by HP_F16, HP_BF16, HP_CVT; tflops
        holds T result words/s.  A failure is latched like compute_test()'s (RES_COMPUTE until probe_reset());
        fault_sm / fault_mask flips bits of one result word of one thread of the SM with that %smid, in the first
        comparison."""
        opts = N.ComputeTestOpts(duration_ms, timeout_ms, N.CT_EVEN_IF_BUSY if even_if_busy else 0, fault_sm, fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.ComputeTestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_half_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ComputeTestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.nsmid, r.sms_covered,
                                  list(r.bad_sm_mask), list(r.mismatches), r.first_bad_sm, r.first_bad_format,
                                  r.first_bad_tile, list(r.ms), list(r.tflops)) for r in arr[:n]]

    def sync_test(self, device: int = -1, duration_ms: int = 0, timeout_ms: int = 0, even_if_busy: bool = False,
                  fault_sm: int = -1, fault_mask: int = 0) -> List[ComputeTestResult]:
        """On-demand synchronization self-test of `device` (-1 = every GPU, b2dp_sync_test): every SM's shared-memory
        atomics, named barriers, bar.red, mbarriers and warp collectives under partial member masks, against results the
        host computed from the PTX ISA, for duration_ms per format (0 = 1000).  The per-format lists are indexed by
        SY_ATOM, SY_BAR, SY_WARP; tflops holds G atomic ops/s, G barrier ops/s and T result words/s.  A failure is
        latched like compute_test()'s (RES_COMPUTE until probe_reset()); fault_sm / fault_mask flips bits of one result
        word of one thread of the SM with that %smid, in the first comparison."""
        opts = N.ComputeTestOpts(duration_ms, timeout_ms, N.CT_EVEN_IF_BUSY if even_if_busy else 0, fault_sm, fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.ComputeTestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_sync_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ComputeTestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.nsmid, r.sms_covered,
                                  list(r.bad_sm_mask), list(r.mismatches), r.first_bad_sm, r.first_bad_format,
                                  r.first_bad_tile, list(r.ms), list(r.tflops)) for r in arr[:n]]

    def l1_test(self, device: int = -1, duration_ms: int = 0, timeout_ms: int = 0, even_if_busy: bool = False,
                fault_sm: int = -1, fault_mask: int = 0) -> List[ComputeTestResult]:
        """On-demand L1 self-test of `device` (-1 = every GPU, b2dp_l1_test): every SM's L1 data cache (each CTA's
        span written and read back), its texture and read-only data paths, and its constant cache, against data and
        results the host built, for duration_ms per format (0 = 1000).  The per-format lists are indexed by L1_DATA,
        L1_TEX, L1_CONST; tflops holds TB/s the loads deliver (L1_DATA: and its stores).  A failure is latched like
        compute_test()'s (RES_COMPUTE until probe_reset()); fault_sm / fault_mask flips bits of one word of the span
        (L1_DATA) or of one loaded value (L1_TEX, L1_CONST) on the SM with that %smid, in the first comparison."""
        opts = N.ComputeTestOpts(duration_ms, timeout_ms, N.CT_EVEN_IF_BUSY if even_if_busy else 0, fault_sm, fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.ComputeTestResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_l1_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [ComputeTestResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.nsmid, r.sms_covered,
                                  list(r.bad_sm_mask), list(r.mismatches), r.first_bad_sm, r.first_bad_format,
                                  r.first_bad_tile, list(r.ms), list(r.tflops)) for r in arr[:n]]

    def hostlink_test(self, device: int = -1, bytes: int = 0, duration_ms: int = 0, timeout_ms: int = 0,
                      even_if_busy: bool = False, fault_word: int = 0, fault_mask: int = 0) -> List[HostlinkResult]:
        """On-demand host-link self-test of `device` (-1 = every GPU, b2dp_hostlink_test): the probe's pattern moved
        between host buffers of `bytes` each (0 = 64 MiB) and the GPU by the copy engines (HL_H2D, HL_D2H) and by the
        SMs' own loads and stores (HL_SM), for duration_ms per format (0 = 1000), every word checked against the
        pattern on the side it arrived.  The PCIe link generation, width and replay count come from NVML, reported
        only.  A failure is latched: later probe results carry RES_HOSTLINK and are Unhealthy until probe_reset().
        fault_word / fault_mask is a test hook that flips bits of one word in the first round of every format."""
        opts = N.HostlinkOpts(bytes, duration_ms, timeout_ms, N.HL_EVEN_IF_BUSY if even_if_busy else 0, fault_word,
                              fault_mask, 0)
        rc, arr, n = N.grow_call(lambda cap: (N.HostlinkResult * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_hostlink_test(self._h, device, C.byref(opts), a, cap, pn))
        N.check(rc, self._h)
        return [HostlinkResult(r.device, bool(r.healthy), r.err, r.flags, r.seed, r.sm_count, r.sms_covered,
                               r.host_numa_node, list(r.bad_sm_mask), list(r.rounds), list(r.mismatches),
                               list(r.first_bad_word), r.replays, list(r.ms), list(r.gbs), r.link_gen, r.link_width,
                               r.max_link_gen, r.max_link_width, r.link_gbs) for r in arr[:n]]

    # ---- ListAndWatch --------------------------------------------------------------------
    def list_and_watch(self, resource: str = "gpu", flags: int = N.LW_INITIAL, external: Optional[Dict[str, bool]] = None,
                       timeout_ms=0, variant=N.PROBE_VARIANT_TMA, min_gbs=0.0, timed=False):
        """One ListAndWatch send: (serialized ListAndWatchResponse bytes, CycleStats)."""
        key = (flags, timeout_ms, variant, min_gbs, timed)
        opts = self._opts_cache.get(key) if external is None else None      # the heartbeat path re-uses its options block
        if opts is None:
            opts = N.CycleOpts()
            opts.flags = flags
            opts.probe = N.ProbeOpts(timeout_ms, variant | (N.PROBE_EVENT_TIMING if timed else 0), min_gbs, 0)
            if external is None:
                self._opts_cache[key] = opts
        keep = None
        if external is not None:
            opts.flags |= N.LW_EXTERNAL_SOURCE
            ids = (N.Id64 * max(1, len(external)))()
            hl = (C.c_int32 * max(1, len(external)))()
            for i, (k, v) in enumerate(external.items()):
                ids[i].value = k.encode()
                hl[i] = 1 if v else 0
            opts.src_ids, opts.src_health, opts.src_n = ids, hl, len(external)
            keep = (ids, hl)
        ln = C.c_size_t(0)
        st = N.CycleStats()
        with self._buf_lock:
            rc = N.lib.b2dp_list_and_watch(self._h, resource.encode(), C.byref(opts), self._buf, len(self._buf),
                                           C.byref(ln), C.byref(st))
            if rc == N.E_NOSPC:
                self._buf = (C.c_uint8 * (ln.value * 2))()
                rc = N.lib.b2dp_list_and_watch(self._h, resource.encode(), C.byref(opts), self._buf, len(self._buf),
                                               C.byref(ln), C.byref(st))
            N.check(rc, self._h)
            wire = C.string_at(self._buf, ln.value)
        del keep
        stats = CycleStats(st.n_devices, st.n_unhealthy, bool(st.homogeneous), bool(st.node_healthy), st.ms_total,
                           st.ms_enumerate, st.ms_probe, st.ms_encode, st.probe_gbs_min, st.probe_gbs_sum,
                           st.probe_bytes, st.ms_link_check, st.n_link_faults, st.probe_ms_device_max, st.probe_frac_min)
        return wire, stats

    def watch(self, callback, resource: str = "gpu", pulse_ms: int = 0, flags: int = 0, timeout_ms=0, min_gbs=0.0):
        """Start the library-owned ListAndWatch loop (b2dp_watch_start).  `callback(rc, wire, stats)`
        runs on the library's thread for the initial list and every heartbeat.  Returns a Watch."""
        return Watch(self, callback, resource, pulse_ms, flags, timeout_ms, min_gbs)

    # ---- Allocate ------------------------------------------------------------------------
    def device_specs(self, ids: List[str]):
        arr_in = N.str_array(ids)
        rc, arr, n = N.grow_call(lambda cap: (N.DevSpec * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_device_specs(self._h, arr_in, len(ids), a, cap, pn))
        N.check(rc, self._h)
        return [(N.s(x.host_path), N.s(x.container_path), N.s(x.permissions)) for x in arr[:n]]

    def allocate_response(self, ids: List[str]) -> bytes:
        arr_in = N.str_array(ids)
        buf = (C.c_uint8 * (256 + 256 * max(1, len(ids))))()
        ln = C.c_size_t(0)
        N.check(N.lib.b2dp_allocate_response(self._h, arr_in, len(ids), buf, len(buf), C.byref(ln)), self._h)
        return bytes(buf[:ln.value])

    # ---- Start / GetPreferredAllocation -----------------------------------------------------
    def start(self) -> int:
        """plugin.go:82-91 Start(); returns the allocator-init rc (0 ok) without raising."""
        return N.lib.b2dp_start(self._h)

    def pair_weights(self):
        """p2pWeights of the context's own allocator as {from: {to: weight}} (device.go:220-252); needs start()."""
        cap = 4096
        while True:
            arr = (N.PairWeight * cap)()
            n, rows = C.c_int(0), C.c_int(0)
            rc = N.lib.b2dp_pair_weights(self._h, arr, cap, C.byref(n), C.byref(rows))
            if rc == N.E_NOSPC:
                cap = n.value
                continue
            N.check(rc, self._h)
            break
        w = {}
        for e in arr[:n.value]:
            w.setdefault(e.node_from, {})[e.node_to] = e.weight
        return w

    def preferred_allocation_available(self) -> bool:
        v = C.c_int32()
        N.check(N.lib.b2dp_preferred_allocation_available(self._h, C.byref(v)), self._h)
        return bool(v.value)

    def preferred_allocation(self, available: List[str], must_include: List[str], size: int) -> List[str]:
        a, m = N.str_array(available), N.str_array(must_include)
        out = (N.Id64 * max(1, len(available), len(must_include)))()
        n = C.c_int(0)
        rc = N.lib.b2dp_preferred_allocation(self._h, a, len(available), m, len(must_include), size, out, len(out),
                                             C.byref(n))
        N.check(rc, self._h)
        return [N.s(out[i].value) for i in range(n.value)]

    # ---- P2P / export / labels -------------------------------------------------------------
    def p2p_matrix(self, bytes_per_pair: int = 0, iters: int = 0, bidir: bool = False):
        import numpy as np
        arr, n = self.enumerate_raw()
        gbs = np.zeros((n, n), dtype=np.float32)
        lt = np.zeros((n, n), dtype=np.int32)
        mm = np.zeros((n, n), dtype=np.uint64)
        opts = N.P2pOpts(bytes_per_pair, iters, 1 if bidir else 0)
        N.check(N.lib.b2dp_p2p_matrix(self._h, C.byref(opts), gbs.ctypes.data_as(C.POINTER(C.c_float)),
                                      lt.ctypes.data_as(C.POINTER(C.c_int32)),
                                      mm.ctypes.data_as(C.POINTER(C.c_uint64)), n), self._h)
        return gbs, lt, mm

    def export_kfd_tree(self, directory: str):
        N.check(N.lib.b2dp_export_kfd_tree(self._h, directory.encode()), self._h)

    def generate_labels(self, enabled: List[str]) -> Dict[str, str]:
        csv = ",".join(enabled).encode()
        rc, arr, n = N.grow_call(lambda cap: (N.Label * cap)(),
                                 lambda a, cap, pn: N.lib.b2dp_generate_labels(self._h, csv, a, cap, pn))
        N.check(rc, self._h)
        return {N.s(x.key): N.s(x.value) for x in arr[:n]}


class Watch:
    """Handle of a native ListAndWatch loop: beat() = one heartbeat tick, stop() ends the stream."""

    def __init__(self, ctx: Context, callback, resource, pulse_ms, flags, timeout_ms, min_gbs):
        opts = N.CycleOpts()
        opts.flags = flags
        opts.probe = N.ProbeOpts(timeout_ms, 0, min_gbs, 0)

        def tramp(_user, rc, buf, ln, st):
            s = st.contents
            stats = CycleStats(s.n_devices, s.n_unhealthy, bool(s.homogeneous), bool(s.node_healthy), s.ms_total,
                               s.ms_enumerate, s.ms_probe, s.ms_encode, s.probe_gbs_min, s.probe_gbs_sum, s.probe_bytes,
                               s.ms_link_check, s.n_link_faults, s.probe_ms_device_max, s.probe_frac_min)
            callback(rc, bytes(buf[:ln]) if ln else b"", stats)
        self._cb = N.WatchCb(tramp)          # keep the trampoline alive as long as the loop
        self._h = C.c_void_p()
        N.check(N.lib.b2dp_watch_start(ctx._h, resource.encode(), pulse_ms, C.byref(opts), self._cb, None,
                                       C.byref(self._h)), ctx._h)

    def beat(self):
        N.check(N.lib.b2dp_watch_beat(self._h))

    def stop(self):
        if self._h:
            N.lib.b2dp_watch_stop(self._h)
            self._h = C.c_void_p()
