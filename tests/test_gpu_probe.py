"""GPU parity tests (run with -m gpu on an H100): every result comes through the C ABI
(libb200dp.so, cuda: backend) and is compared bit-exactly with the oracle (oracle/probe.py for
the probe arithmetic; the reference-restating oracle on the exported kfd tree for enumerate /
pair weights / allocation / labels).  Nothing here reads /root/reference."""
import os

import numpy as np
import pytest

from oracle import allocator as oalloc
from oracle import amdgpu as oamd
from oracle import labeller as olab
from oracle import plugin as oplug
from oracle import probe as oprobe

pytestmark = pytest.mark.gpu

MiB = 1 << 20


@pytest.fixture(scope="module")
def P(pkg):
    return pkg


def _open(P, nbytes, extra=""):
    return P.Context("cuda:devices=0,bytes=%d%s" % (nbytes, extra))


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("nbytes", [4096, 16 * 1024 + 16, MiB + 48, 3 * MiB + 16 * 37, 64 * MiB])
def test_probe_pass_bit_exact(P, nbytes, variant):
    """Empty-ish, ragged (not a multiple of the 16 KiB tile / the CTA chunk) and larger buffers:
    buffer contents, checksum, mismatch count and the re-keyed output all equal the oracle."""
    n_words = nbytes // 4
    with _open(P, nbytes) as ctx:
        seed = oprobe.initial_seed(0)
        for step in range(3):
            before = ctx.probe_peek(0, 0, n_words)
            assert np.array_equal(before, oprobe.pattern(n_words, seed))
            (r,) = ctx.probe_health(variant=variant, min_gbs=1e-3)
            cs, bad, first, dst = oprobe.probe_pass(before, seed, oprobe.next_seed(seed))
            assert r.err == 0 and r.seed == seed and r.bytes == 2 * nbytes
            assert (r.checksum, r.mismatches, r.first_bad_word) == (cs, bad, first) == (cs, 0, oprobe.NO_BAD)
            assert r.expected_checksum == oprobe.expected_checksum(n_words, seed) == cs
            assert r.healthy
            assert np.array_equal(ctx.probe_peek(0, 0, n_words), dst)
            seed = oprobe.next_seed(seed)


@pytest.mark.parametrize("variant", [0, 1])
def test_fault_injection_flips_health(P, variant):
    nbytes = 8 * MiB + 16 * 5
    n_words = nbytes // 4
    with _open(P, nbytes) as ctx:
        seed = oprobe.initial_seed(0)
        (r,) = ctx.probe_health(variant=variant, min_gbs=1e-3)
        assert r.healthy
        seed = oprobe.next_seed(seed)
        # corrupt three words (first tile, middle, ragged tail) of the buffer the next pass reads
        bad_words = [5, n_words // 2 + 3, n_words - 1]
        for w in bad_words:
            ctx.probe_inject_fault(0, w, 0x00010000)
        src = ctx.probe_peek(0, 0, n_words)
        cs, bad, first, _ = oprobe.probe_pass(src, seed, oprobe.next_seed(seed))
        (r,) = ctx.probe_health(variant=variant, min_gbs=1e-3)
        assert (r.checksum, r.mismatches, r.first_bad_word) == (cs, 3, 5) == (cs, bad, first)
        assert r.checksum != r.expected_checksum and not r.healthy
        # the library re-fills after reporting: a transient fault is reported exactly once
        seed = oprobe.next_seed(seed)
        assert np.array_equal(ctx.probe_peek(0, 0, n_words), oprobe.pattern(n_words, seed))
        (r,) = ctx.probe_health(variant=variant, min_gbs=1e-3)
        assert r.healthy and r.mismatches == 0
        # ListAndWatch reflects the verdict
        ctx.probe_inject_fault(0, 12345, 1)
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, min_gbs=1e-3)
        msg = P.v1beta1.ListAndWatchResponse.FromString(wire)
        assert [d.health for d in msg.devices] == ["Unhealthy"] and st.n_unhealthy == 1
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, min_gbs=1e-3)
        assert [d.health for d in P.v1beta1.ListAndWatchResponse.FromString(wire).devices] == ["Healthy"]


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("nbytes", [MiB + 48, 3 * MiB + 16 * 37])
def test_grid_ctas_bit_exact(P, nbytes, variant):
    """`grid_ctas` from one CTA (every tile and the whole ragged tail on one CTA) to more CTAs than tiles: buffer
    contents and every result field equal the oracle, pass after pass on the same ring."""
    n_words = nbytes // 4
    with _open(P, nbytes) as ctx:
        seed = oprobe.initial_seed(0)
        for grid in (1, 2, 7, 131, 264, 1000):
            before = ctx.probe_peek(0, 0, n_words)
            assert np.array_equal(before, oprobe.pattern(n_words, seed)), grid
            (r,) = ctx.probe_health(variant=variant, min_gbs=1e-3, grid_ctas=grid)
            cs, bad, first, dst = oprobe.probe_pass(before, seed, oprobe.next_seed(seed))
            assert r.err == 0 and r.seed == seed and r.bytes == 2 * nbytes, grid
            assert (r.checksum, r.mismatches, r.first_bad_word) == (cs, bad, first) == (cs, 0, oprobe.NO_BAD), grid
            assert r.checksum == r.expected_checksum and r.healthy, grid
            assert np.array_equal(ctx.probe_peek(0, 0, n_words), dst), grid
            seed = oprobe.next_seed(seed)


@pytest.mark.parametrize("variant", [0, 1])
def test_dense_injected_faults_equal_oracle(P, variant):
    """48 corrupted words: all four lanes of one vector, both sides of several 16 KiB tile (chunk) boundaries, the
    ragged tail and the last word.  Every result field equals the oracle on the corrupted source; the fault is
    reported once and the next pass is clean."""
    nbytes = 8 * MiB + 16 * 5
    n_words = nbytes // 4
    tile = 4 * 1024                                   # words per TMA tile and per R128 chunk
    words = {4 * 777 + lane for lane in range(4)}
    for t in (1, 2, 263, 264, 511):
        words |= {t * tile - 1, t * tile}
    words |= {(n_words // tile) * tile, n_words - 17, n_words - 2, n_words - 1}
    rng = np.random.default_rng(48)
    while len(words) < 48:
        words.add(int(rng.integers(0, n_words)))
    words = sorted(words)
    masks = [int(m) for m in rng.integers(1, 1 << 32, len(words), dtype=np.uint64)]
    with _open(P, nbytes) as ctx:
        seed = oprobe.initial_seed(0)
        for w, m in zip(words, masks):
            ctx.probe_inject_fault(0, w, m)
        src = ctx.probe_peek(0, 0, n_words)
        cs, bad, first, _ = oprobe.probe_pass(src, seed, oprobe.next_seed(seed))
        (r,) = ctx.probe_health(variant=variant, min_gbs=1e-3)
        assert (r.checksum, r.mismatches, r.first_bad_word) == (cs, bad, first) == (cs, 48, words[0])
        assert r.seed == seed and not r.healthy
        seed = oprobe.next_seed(seed)
        assert np.array_equal(ctx.probe_peek(0, 0, n_words), oprobe.pattern(n_words, seed))
        (r,) = ctx.probe_health(variant=variant, min_gbs=1e-3)
        assert r.healthy and r.mismatches == 0 and r.first_bad_word == oprobe.NO_BAD


def _sum_preserving_pair(seed, n_words, bit, lo=0):
    """Two word indices >= lo whose pattern(seed) words have `bit` clear and set: flipping that bit in both keeps the
    sum of the buffer."""
    pat = oprobe.pattern(n_words - lo, seed, lo)
    b = (pat >> np.uint32(bit)) & np.uint32(1)
    i = lo + int(np.nonzero(b == 0)[0][0])
    j = lo + int(np.nonzero(b == 1)[0][-1])
    return i, j


@pytest.mark.parametrize("variant", [0, 1])
def test_checksum_preserving_pair_fails_the_device(P, variant):
    """Bit b flipped 0->1 in one word and 1->0 in another leaves the checksum equal to the closed form: only the
    mismatch count can fail the device, and it must."""
    nbytes = 4 * MiB + 16 * 3
    n_words = nbytes // 4
    with _open(P, nbytes) as ctx:
        seed = oprobe.initial_seed(0)
        i, j = _sum_preserving_pair(seed, n_words, 13, lo=1000)
        ctx.probe_inject_fault(0, i, 1 << 13)
        ctx.probe_inject_fault(0, j, 1 << 13)
        (r,) = ctx.probe_health(variant=variant, min_gbs=1e-3)
        assert r.checksum == r.expected_checksum == oprobe.expected_checksum(n_words, seed)
        assert (r.mismatches, r.first_bad_word, r.healthy) == (2, min(i, j), 0)
        # through the kubelet-facing heartbeat (the library re-filled the ring after reporting)
        seed = oprobe.next_seed(seed)
        i, j = _sum_preserving_pair(seed, n_words, 31)
        ctx.probe_inject_fault(0, i, 1 << 31)
        ctx.probe_inject_fault(0, j, 1 << 31)
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, variant=variant, min_gbs=1e-3)
        assert [d.health for d in P.v1beta1.ListAndWatchResponse.FromString(wire).devices] == ["Unhealthy"]
        assert st.n_unhealthy == 1
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, variant=variant, min_gbs=1e-3)
        assert [d.health for d in P.v1beta1.ListAndWatchResponse.FromString(wire).devices] == ["Healthy"]


def _driver_copy_gbs(nbytes):
    """Best of 10 CUDA-event-timed torch device-to-device copies of nbytes: GB/s read + written."""
    import torch
    a = torch.zeros(nbytes, dtype=torch.uint8, device="cuda:0")
    b = torch.empty_like(a)
    for _ in range(3):
        b.copy_(a)
    best = None
    for _ in range(10):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        b.copy_(a)
        e1.record()
        e1.synchronize()
        best = e0.elapsed_time(e1) if best is None else min(best, e0.elapsed_time(e1))
    del a, b
    torch.cuda.empty_cache()
    return 2.0 * nbytes / (best * 1e-3) / 1e9


def test_full_size_probe_and_bandwidth_floor(P):
    """BASELINE.json config 2 at full size (1 GiB src -> 1 GiB dst): checksum equals the oracle's
    closed form (size-independent property: sum of the pattern), and the stream is fast enough
    to be a meaningful health signal.  Too-slow streams flip the verdict (min_gbs)."""
    nbytes = 1 << 30
    with _open(P, nbytes) as ctx:
        seed = oprobe.initial_seed(0)
        best = 0.0
        for _ in range(4):
            (r,) = ctx.probe_health()
            assert r.err == 0 and r.mismatches == 0
            assert r.checksum == r.expected_checksum == oprobe.expected_checksum(nbytes // 4, seed)
            assert r.healthy
            best = max(best, r.gbs)
            seed = oprobe.next_seed(seed)
        # 2.8-2.9 TB/s on a healthy H100 SXM at 700 W.  The regression guard is relative to the box's measured copy peak
        # (MEASURED_PEAKS.json when present, else the driver's own D2D copy of the same size, measured here), and to the
        # ceiling calibrated at open
        try:
            import json
            peak = float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                     "MEASURED_PEAKS.json")))["hbm_gbs"])
        except Exception:
            peak = _driver_copy_gbs(nbytes)
        assert best > 0.9 * peak, (best, peak)
        assert r.gbs_ref > 0.9 * peak and 0.95 < r.frac < 1.05 and abs(r.min_gbs_applied - 0.8 * r.gbs_ref) < 1.0, r
        assert not (r.flags & (P._native.RES_NO_FLOOR | P._native.RES_SLOW))
        # spot-check the re-keyed buffer at both ends and in the middle
        for off in (0, nbytes // 8 - 17, nbytes // 4 - 4096):
            assert np.array_equal(ctx.probe_peek(0, off, 4096), oprobe.pattern(4096, seed, off))
        (r,) = ctx.probe_health(min_gbs=1e9)      # impossible floor => Unhealthy, data still verified
        assert not r.healthy and r.mismatches == 0 and r.checksum == r.expected_checksum


def test_worker_path_equals_direct_path(P):
    """B2DP_PROBE_VIA_WORKERS (per-GPU worker threads launch and wait) and the default low-latency
    path (caller enqueues, polls events) drive the same state machine: interleave them."""
    nbytes = 16 * MiB + 16
    with _open(P, nbytes) as ctx:
        seed = oprobe.initial_seed(0)
        for step in range(6):
            (r,) = ctx.probe_health(min_gbs=1e-3, via_workers=bool(step % 2), variant=step % 2)
            assert r.seed == seed and r.healthy and r.checksum == oprobe.expected_checksum(nbytes // 4, seed)
            seed = oprobe.next_seed(seed)
        ctx.probe_inject_fault(0, 99, 2)
        (r,) = ctx.probe_health(min_gbs=1e-3, via_workers=True)
        assert (r.mismatches, r.first_bad_word, r.healthy) == (1, 99, False)
        (r,) = ctx.probe_health(min_gbs=1e-3)
        assert r.healthy


def test_full_size_golden_checksums(P):
    """1 GiB passes against the committed golden checksums (tests/golden/probe_vectors.json)."""
    import json
    g = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "probe_vectors.json")))
    seeds = g["full_size"]["seeds"]
    with _open(P, g["full_size"]["n_words"] * 4) as ctx:
        for seed_s, want in seeds.items():
            (r,) = ctx.probe_health()
            assert r.seed == int(seed_s) and r.checksum == want == r.expected_checksum and r.mismatches == 0


def test_cuda_backend_equals_reference_algorithm_on_exported_tree(P, tmp_path):
    """The 'equivalent fixture' contract: export what the cuda backend sees as a kfd-shaped tree;
    the reference algorithm (oracle) on that tree must give the same device table, pair weights,
    allocation answers, ListAndWatch list and labels as the cuda backend itself."""
    root = str(tmp_path / "export")
    with P.Context("cuda:bytes=%d,p2p_bytes=%d" % (64 * MiB, 32 * MiB)) as ctx:
        devs = ctx.enumerate()
        assert len(devs) >= 1 and list(devs) == sorted(devs)
        ctx.export_kfd_tree(root)
        want = oamd.GetAMDGPUs(root)
        assert devs == want
        for k, v in devs.items():                       # id shapes are the reference's
            assert len(k) == 12 and k[4] == ":" and k.endswith(".0") and v["devID"] == k[:-2] + ":0"
        # Start(): pair weights from the measured P2P matrix == oracle on the exported link files
        assert ctx.start() == (0 if len(devs) > 1 else P._native.E_ALLOC_NO_WEIGHTS)
        ids = sorted(devs)
        opol = oalloc.BestEffortPolicy()
        oerr = opol.Init(oplug.getDevices(root), root + "/sys/class/kfd/kfd/topology/nodes")
        if len(devs) > 1:
            assert oerr is None
            for size in range(1, len(ids) + 1):
                assert ctx.preferred_allocation(ids, [], size) == opol.Allocate(list(ids), [], size)[0]
        else:
            assert oerr is not None and not ctx.preferred_allocation_available()
        # ListAndWatch initial list
        wire, st = ctx.list_and_watch("gpu", P._native.LW_INITIAL)
        homog, lw = oplug.list_and_watch_devices(want, "gpu")
        msg = P.v1beta1.ListAndWatchResponse.FromString(wire)
        assert [(d.ID, d.health, d.topology.nodes[0].ID) for d in msg.devices] == lw and msg.SerializeToString() == wire
        assert ctx.resource_list("single") == ["gpu"] == oplug.getResourceList("single", root)[0]
        # node health: the text check on the exported tree agrees with the driver-level check
        assert ctx.node_health() == oplug.simpleHealthCheck(root + "/sys/class/kfd/kfd") is True
        # labels from CUDA/NVML queries == reference generators on the exported tree
        gens = ["driver-version", "driver-src-version", "device-id", "product-name", "vram", "simd-count", "cu-count",
                "compute-memory-partition", "compute-partitioning-supported", "memory-partitioning-supported",
                "family", "firmware"]
        got = ctx.generate_labels(gens)
        # family / firmware: libdrm ioctls on the reference side (no file form); the export carries them as per-card
        # side files, which become the oracle's drm provider
        drm = {}
        for v in want.values():
            base = "%s/sys/class/drm/card%d/device/" % (root, v["card"])
            fw = dict(ln.split(" ", 1) for ln in open(base + "b2dp_firmware").read().splitlines()) \
                if os.path.exists(base + "b2dp_firmware") else {}
            fw = {k: "".join(ch if ch.isalnum() or ch in ".-_" else "_" for ch in ver.strip()) for k, ver in fw.items()}
            drm["card%d" % v["card"]] = {"family": open(base + "b2dp_family").read().strip(), "feat": {}, "fw": fw}
        assert got == olab.generateLabels({g: True for g in gens}, root, drm=drm)
        assert got["amd.com/gpu.cu-count"] == "132" and got["amd.com/gpu.product-name"].startswith("NVIDIA_H100")
        assert got["amd.com/gpu.family"] == "Hopper" and got["beta.amd.com/gpu.family.Hopper"] == str(len(devs))
        fw_keys = [k for k in got if k.startswith("beta.amd.com/gpu.firmware.")]
        assert any(k.startswith("beta.amd.com/gpu.firmware.vbios.fw.") for k in fw_keys), got
        assert all(len(k.split("/", 1)[1]) <= 63 for k in got)        # Kubernetes label-name limit
        # the kfd: reader on the exported tree gives the same 12-generator label set as the cuda: backend itself
        with P.Context("kfd:" + root) as kctx:
            assert kctx.generate_labels(gens) == got
        # Allocate: the NVIDIA device nodes exist on the box; the runtime-facing identifier is the GPU UUID (NVML's,
        # cross-checked), or the NVML index with id_strategy=index -- never the /dev/nvidia minor
        import pynvml
        pynvml.nvmlInit()

        def nv(bdf):
            h = pynvml.nvmlDeviceGetHandleByPciBusId(("0000" + bdf).encode())
            u = pynvml.nvmlDeviceGetUUID(h)
            return (u.decode() if isinstance(u, bytes) else u), pynvml.nvmlDeviceGetIndex(h), pynvml.nvmlDeviceGetMinorNumber(h)
        for i in ids:
            assert devs[i]["card"] == nv(i)[2]
        resp = P.v1beta1.ContainerAllocateResponse.FromString(ctx.allocate_response([ids[0], "unknown", ids[-1]]))
        assert dict(resp.envs) == {"NVIDIA_VISIBLE_DEVICES": ",".join(nv(i)[0] for i in (ids[0], ids[-1]))}
        assert nv(ids[0])[0].startswith("GPU-") and len(nv(ids[0])[0]) == 40
        assert [d.host_path for d in resp.devices][-1] == "/dev/nvidia%d" % devs[ids[-1]]["card"]
        with P.Context("cuda:devices=0,bytes=%d,cdi=nvidia.com/gpu" % MiB) as cctx:          # optional CDI names
            (cid,) = sorted(cctx.enumerate())
            cresp = P.v1beta1.ContainerAllocateResponse.FromString(cctx.allocate_response([cid, "unknown"]))
            assert [x.name for x in cresp.cdi_devices] == ["nvidia.com/gpu=" + nv(cid)[0]]
            assert cresp.SerializeToString() == cctx.allocate_response([cid, "unknown"])      # canonical field order
        with P.Context("cuda:bytes=%d,cdi=nvidia.com/gpu,id_strategy=index,calib=0" % MiB) as ictx:
            iresp = P.v1beta1.ContainerAllocateResponse.FromString(ictx.allocate_response(list(reversed(ids))))
            assert dict(iresp.envs) == {"NVIDIA_VISIBLE_DEVICES": ",".join(str(nv(i)[1]) for i in reversed(ids))}
            assert [x.name for x in iresp.cdi_devices] == ["nvidia.com/gpu=%d" % nv(i)[1] for i in reversed(ids)]
        assert dict(P.v1beta1.ContainerAllocateResponse.FromString(ctx.allocate_response(["unknown"])).envs) == \
            {"NVIDIA_VISIBLE_DEVICES": "void"}
        assert not resp.cdi_devices
        specs = ctx.device_specs(ids)
        assert [s[0] for s in specs[:3]] == ["/dev/nvidiactl", "/dev/nvidia-uvm", "/dev/nvidia-uvm-tools"]
        assert len(specs) == 3 + len(ids)
        for host, cont, perm in specs:
            assert host == cont and perm == "rw"
            if host == "/dev/nvidiactl" or host[len("/dev/nvidia"):].isdigit():
                assert os.path.exists(host), host


def test_p2p_matrix(P):
    with P.Context("cuda:bytes=%d,p2p_bytes=%d" % (256 * MiB, 256 * MiB)) as ctx:
        n = len(ctx.enumerate())
        gbs, lt, mm = ctx.p2p_matrix()
        assert gbs.shape == (n, n) and (mm == 0).all()
        for i in range(n):
            for j in range(n):
                if i == j:
                    assert lt[i, j] == 0
                else:
                    assert lt[i, j] == oprobe.classify_link(True, float(gbs[i, j])) == 11, (i, j, gbs[i, j])
        # probing afterwards still verifies clean (the matrix only wrote spare buffers)
        assert all(r.healthy for r in ctx.probe_health())
        # both directions at once (full-duplex stress) verifies too
        gb2, lt2, mm2 = ctx.p2p_matrix(bidir=True)
        assert (mm2 == 0).all() and (lt2 == lt).all()
        # extension label (no reference counterpart): interconnect class per GPU
        cls = "nvlink" if n > 1 else "none"
        assert ctx.generate_labels(["p2p-link"]) == {
            "amd.com/gpu.p2p-link": cls, "beta.amd.com/gpu.p2p-link": cls, "beta.amd.com/gpu.p2p-link." + cls: str(n)}
        assert P.labeller.removeOldNodeLabels(ctx.generate_labels(["p2p-link", "vram"])) == {}


def test_p2p_matrix_detects_a_corrupt_peer(P):
    """A P2P pass is a verify-only pass (delta 0) over the peer's current slot: a flipped word, and a checksum-
    preserving pair, in GPU j's slot show up as mism[i][j] for every reader i with peer access and nowhere else.  The
    matrix reads only the first p2p_bytes, so a fault past them is left for j's own next probe, which reports it once."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("the P2P matrix needs 2 or more GPUs; this node has %d" % torch.cuda.device_count())
    nbytes, p2p_bytes = 64 * MiB, 16 * MiB
    with P.Context("cuda:bytes=%d,p2p_bytes=%d" % (nbytes, p2p_bytes)) as ctx:
        n = len(ctx.enumerate())
        j = n - 1
        _, lt, mm = ctx.p2p_matrix()
        assert (mm == 0).all()
        readers = [i for i in range(n) if i != j and lt[i, j] != 0]     # link type 0 off the diagonal: no peer access
        assert readers, lt

        def expect(count):
            want = np.zeros((n, n), dtype=mm.dtype)
            want[readers, j] = count
            return want

        ctx.probe_inject_fault(j, 12345, 0x10)
        _, _, mm = ctx.p2p_matrix()
        assert (mm == expect(1)).all(), mm
        res = ctx.probe_health(min_gbs=1e-3)                            # the matrix left j's slot as it was
        assert [(r.mismatches, r.first_bad_word) for r in res if r.device == j] == [(1, 12345)]
        assert all(r.healthy for r in res if r.device != j)

        seed = oprobe.next_seed([r.seed for r in res if r.device == j][0])   # j's slot was re-filled for the next pass
        a, b = _sum_preserving_pair(seed, 1 << 16, 7)
        ctx.probe_inject_fault(j, a, 1 << 7)
        ctx.probe_inject_fault(j, b, 1 << 7)
        _, _, mm = ctx.p2p_matrix()
        assert (mm == expect(2)).all(), mm
        res = ctx.probe_health(min_gbs=1e-3)
        assert [(r.mismatches, r.checksum == r.expected_checksum) for r in res if r.device == j] == [(2, True)]

        past = p2p_bytes // 4 + 100
        ctx.probe_inject_fault(j, past, 0x1)
        _, _, mm = ctx.p2p_matrix()
        assert (mm == 0).all(), mm
        res = ctx.probe_health(min_gbs=1e-3)
        assert [(r.mismatches, r.first_bad_word) for r in res if r.device == j] == [(1, past)]
        assert all(r.healthy for r in ctx.probe_health(min_gbs=1e-3))


def test_multi_gpu_fanout_concurrent(P):
    """All GPUs probed in one call: per-device seeds differ, every device verifies, and the
    fan-out takes about one probe time, not N."""
    with P.Context("cuda:bytes=%d" % (1 << 30)) as ctx:
        n = len(ctx.enumerate())
        for _ in range(3):
            res = ctx.probe_health()
        assert len(res) == n and len({r.seed for r in res}) == n
        assert all(r.healthy and r.checksum == r.expected_checksum for r in res)
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT)
        assert st.n_devices == n and st.n_unhealthy == 0
        slowest = max(r.ms_event for r in res)
        assert st.ms_probe < 3.0 * slowest + 1.0, (st.ms_probe, slowest)
        # heartbeat + NVLink link check against the topology measured at Start()
        ctx.start()
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT | P._native.LW_LINK_CHECK)
        assert st.n_unhealthy == 0 and st.n_link_faults == 0
        assert (st.ms_link_check > 0) == (n > 1)
        assert all(r.healthy for r in ctx.probe_health())


def test_busy_policy_skip_and_shrink(P):
    """`busy=skip|shrink`: when another process owns the GPU the 2 GiB-traffic pass is skipped (last
    verdict stands) or shrunk to a verify-only prefix that leaves the seed/ping-pong state alone."""
    import subprocess
    import sys
    import time
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
        nbytes, shrink = 32 * MiB, 1 * MiB
        with _open(P, nbytes, ",busy=skip") as ctx:
            (r,) = ctx.probe_health(min_gbs=1e-3)
            assert r.flags & P._native.RES_SKIPPED_BUSY and r.healthy and r.bytes == 0 and r.err == 0
            wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, min_gbs=1e-3)
            assert st.n_unhealthy == 0
        with _open(P, nbytes, ",busy=shrink,shrink_bytes=%d" % shrink) as ctx:
            seed = oprobe.initial_seed(0)
            for _ in range(2):
                (r,) = ctx.probe_health(min_gbs=1e9)                 # the GB/s floor does not apply to a shrunk pass
                assert r.flags & P._native.RES_SHRUNK and r.healthy and r.bytes == 2 * shrink
                assert r.seed == seed and r.mismatches == 0
                assert r.checksum == r.expected_checksum == oprobe.expected_checksum(shrink // 4, seed)
            ctx.probe_inject_fault(0, 100, 1)
            (r,) = ctx.probe_health(min_gbs=1e-3)
            assert not r.healthy and r.mismatches == 1 and r.first_bad_word == 100
            (r,) = ctx.probe_health(min_gbs=1e-3)
            assert r.healthy and r.seed == seed                       # repaired in place, state untouched
            helper.kill()
            helper.wait()
            time.sleep(1.0)
            (r,) = ctx.probe_health(min_gbs=1e-3)                     # alone again: a full pass
            assert r.flags == 0 and r.bytes == 2 * nbytes and r.seed == seed and r.healthy
            assert r.checksum == oprobe.expected_checksum(nbytes // 4, seed)
    finally:
        if helper.poll() is None:
            helper.kill()


def test_scrub_ring_rotates_through_all_slots(P):
    """`slots=M`: pass k verifies slot k mod M and re-keys it into slot k+1 mod M.  Every pass stays
    bit-exact with the oracle, M*S bytes of HBM are held (and scrubbed once per M heartbeats), a fault
    poked into the current slot is caught by the next pass only, and M+1 passes later the ring has
    wrapped over the slot that once held the fault without any residue."""
    import torch
    nbytes, slots = 48 * MiB + 16 * 3, 5
    n_words = nbytes // 4
    free0, _ = torch.cuda.mem_get_info(0)
    with _open(P, nbytes, ",slots=%d" % slots) as ctx:
        free1, _ = torch.cuda.mem_get_info(0)
        assert free0 - free1 >= slots * (nbytes // MiB) * MiB
        seed = oprobe.initial_seed(0)
        for k in range(2 * slots + 3):
            if k == 2:
                ctx.probe_inject_fault(0, 12345, 0x10)
            before = ctx.probe_peek(0, 0, n_words)
            (r,) = ctx.probe_health(min_gbs=1e-3)
            cs, bad, first, dst = oprobe.probe_pass(before, seed, oprobe.next_seed(seed))
            assert (r.seed, r.checksum, r.mismatches, r.first_bad_word) == (seed, cs, bad, first)
            assert bad == (1 if k == 2 else 0) and r.healthy == (k != 2)
            seed = oprobe.next_seed(seed)
            if k != 2:                                                # after a fault the next slot is re-filled clean
                assert np.array_equal(ctx.probe_peek(0, 0, n_words), dst)
            else:
                assert np.array_equal(ctx.probe_peek(0, 0, n_words), oprobe.pattern(n_words, seed))
    for bad_uri in ("cuda:devices=0,slots=1", "cuda:devices=0,slots=99999", "cuda:devices=0+0", "cuda:devices=999"):
        with pytest.raises(P._native.B2dpError):
            P.Context(bad_uri)


def test_ecc_option_is_harmless(P):
    with _open(P, 16 * MiB, ",ecc=1") as ctx:
        (r,) = ctx.probe_health(min_gbs=1e-3)
        assert r.healthy and not (r.flags & P._native.RES_ECC)


def test_xid_option_latches_critical_events_and_ignores_application_xids(P):
    """`xid=1`: the NVML critical-Xid event set is drained once per pass.  No hardware fault can be
    provoked here, so synthetic events go through the same handler (word_index = UINT64_MAX): an
    application-level Xid (31 = MMU fault of a user context) changes nothing; a device-level one (79 =
    fallen off the bus) fails the device on every later pass although the HBM pass itself is clean,
    until probe_reset acknowledges it.  Without xid=1 the events are not looked at."""
    UINT64_MAX = (1 << 64) - 1
    with _open(P, 16 * MiB, ",xid=1") as ctx:
        (r,) = ctx.probe_health(min_gbs=1e-3)
        assert r.healthy and not (r.flags & P._native.RES_XID)     # live event set: nothing pending
        ctx.probe_inject_fault(0, UINT64_MAX, 31)
        (r,) = ctx.probe_health(min_gbs=1e-3)
        assert r.healthy and r.flags == 0
        ctx.probe_inject_fault(0, UINT64_MAX, 79)
        for _ in range(2):
            (r,) = ctx.probe_health(min_gbs=1e-3)
            assert not r.healthy and r.flags & P._native.RES_XID
            assert r.mismatches == 0 and r.checksum == r.expected_checksum and r.err == 0
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, min_gbs=1e-3)
        assert st.n_unhealthy == 1
        assert P.v1beta1.ListAndWatchResponse.FromString(wire).devices[0].health == "Unhealthy"
        ctx.probe_reset(0)
        (r,) = ctx.probe_health(min_gbs=1e-3)
        assert r.healthy and r.flags == 0
    with _open(P, 16 * MiB) as ctx:
        ctx.probe_inject_fault(0, UINT64_MAX, 79)
        (r,) = ctx.probe_health(min_gbs=1e-3)
        assert r.healthy and r.flags == 0


@pytest.mark.parametrize("via_workers", [False, True])
def test_deadline_expiry_reports_unhealthy_and_recovers(P, via_workers):
    """health.go:37 gives the exporter RPC a deadline; here a pass that misses `timeout_ms` is reported
    Unhealthy with B2DP_E_TIMEOUT without blocking the caller, the late pass is collected by the GPU's
    worker, and the next heartbeat carries on from the state that pass left (seed advanced once)."""
    import time
    import torch
    nbytes = 8 << 30                                   # ~2.7 ms per pass: a 1 ms deadline always expires
    free, _ = torch.cuda.mem_get_info(0)
    if free < 2 * nbytes + (2 << 30):
        pytest.skip("not enough free HBM")
    n_check = 1 << 20
    with _open(P, nbytes) as ctx:
        seed = oprobe.initial_seed(0)
        t0 = time.perf_counter()
        (r,) = ctx.probe_health(timeout_ms=1, via_workers=via_workers, min_gbs=1e-3)
        waited = time.perf_counter() - t0
        assert r.err == P._native.E_TIMEOUT and not r.healthy
        assert waited < 0.5                            # the call returned at the deadline, not at completion
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, timeout_ms=1, min_gbs=1e-3)
        assert st.n_unhealthy == 1                     # still in flight or timed out again: Unhealthy either way
        time.sleep(0.2)                                # the worker collects the late passes
        for _ in range(20):
            (r,) = ctx.probe_health(min_gbs=1e-3, via_workers=via_workers)
            if r.err == 0:
                break
            time.sleep(0.05)
        assert r.err == 0 and r.healthy and r.mismatches == 0 and r.checksum == r.expected_checksum
        # the timed-out passes did run to completion: the seed moved on once per completed pass
        steps = 0
        s = seed
        while s != r.seed and steps < 4:
            s = oprobe.next_seed(s)
            steps += 1
        assert 1 <= steps <= 2 and s == r.seed
        assert np.array_equal(ctx.probe_peek(0, 0, n_check), oprobe.pattern(n_check, oprobe.next_seed(r.seed)))


def test_word_index_wraps_past_16_gib(P):
    """Maximum sizes: a buffer larger than 2^32 words (16 GiB) makes the 32-bit word index of the
    pattern wrap.  Size-independent property: one full period of (uint32(i) * K) ^ seed visits every
    32-bit value once, so its sum is 2^31 * (2^32 - 1) for any seed; the remainder is a plain prefix."""
    import torch
    free, total = torch.cuda.mem_get_info(0)
    extra_words = 16 * MiB // 4
    n_words = (1 << 32) + extra_words
    nbytes = n_words * 4
    if free < 2 * nbytes + (4 << 30):
        pytest.skip("not enough free HBM for two %.1f GiB buffers" % (nbytes / 2 ** 30))
    period_sum = (1 << 31) * ((1 << 32) - 1)
    with _open(P, nbytes) as ctx:
        seed = oprobe.initial_seed(0)
        for _ in range(2):
            (r,) = ctx.probe_health()
            want = (period_sum + oprobe.expected_checksum(extra_words, seed)) & oprobe.NO_BAD
            assert r.mismatches == 0 and r.checksum == r.expected_checksum == want and r.healthy
            assert r.bytes == 2 * nbytes
            seed = oprobe.next_seed(seed)
        # the words just past the wrap repeat the start of the pattern
        assert np.array_equal(ctx.probe_peek(0, 1 << 32, 4096), oprobe.pattern(4096, seed))
        ctx.probe_inject_fault(0, (1 << 32) + 5, 0x80)
        (r,) = ctx.probe_health()
        assert (r.mismatches, r.first_bad_word, r.healthy) == (1, (1 << 32) + 5, False)


def test_native_watch_loop_on_cuda(P):
    """b2dp_watch_*: the library's own thread runs stream start + a 20 ms heartbeat ticker with the
    GPU probe in every tick; an injected fault shows up in exactly one response."""
    import queue
    got = queue.Queue()
    with _open(P, 64 * MiB) as ctx:
        w = ctx.watch(lambda rc, wire, st: got.put((rc, wire, st)), pulse_ms=20, min_gbs=1e-3)
        rc, wire, st = got.get(timeout=10)
        assert rc == 0 and st.probe_bytes == 0                      # stream start: no probe, all Healthy
        assert [d.health for d in P.v1beta1.ListAndWatchResponse.FromString(wire).devices] == ["Healthy"]
        healths = []
        for i in range(6):
            if i == 2:
                ctx.probe_inject_fault(0, 777, 0x10)
            rc, wire, st = got.get(timeout=10)
            assert rc == 0 and st.probe_bytes == 2 * 64 * MiB
            healths.append(P.v1beta1.ListAndWatchResponse.FromString(wire).devices[0].health)
        w.stop()
        assert healths.count("Unhealthy") == 1 and healths[0] == "Healthy" and healths[-1] == "Healthy", healths


def test_compiled_hosts_on_the_gpu(tmp_path):
    """The two compiled hosts over the C ABI, on real hardware: the C++ mirror of the reference's plugin
    package (include/b200dp_host.hpp; Start / ListAndWatch with the HBM pass in every heartbeat / Allocate /
    GetPreferredAllocation / labels) and tools/b200dp_cli's kubelet-facing cycle loop."""
    import json
    import shutil
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    libdir = os.path.join(root, "k8s-device-plugin_b200")
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path / "host_mirror_test")
    r = subprocess.run(["g++", "-std=c++17", "-O1", os.path.join(here, "native", "host_mirror_test.cpp"), "-o", exe,
                        "-L", libdir, "-lb200dp", "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, "--cuda", "cuda:bytes=%d,p2p_bytes=%d" % (256 * MiB, 64 * MiB)], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0 and "PASS" in r.stdout and ", 0 failed" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
    cli = os.path.join(root, "tools", "b200dp_cli")
    if os.path.exists(cli):
        r = subprocess.run([cli, "cuda:devices=0", "cycle", "50"], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-2000:]
        d = json.loads(r.stdout.strip().splitlines()[-1])
        assert d["n_devices"] == 1 and d["aggregate_gbs"] > 1750 and d["response_bytes"] > 0


def test_native_daemon_on_the_gpu(P):
    """b200dp_plugind on the cuda: backend with grpcio as the kubelet: registers, streams the initial list,
    and every SIGUSR1 heartbeat (HBM pass included) comes back Healthy."""
    import importlib
    dp = importlib.import_module("k8s-device-plugin_b200.daemon_probe")
    if not os.path.exists(dp.DAEMON):
        import __graft_entry__
        __graft_entry__.build()
    r = dp.heartbeat_latency_ms("cuda:devices=0,bytes=%d" % (256 * MiB), iters=30)
    assert r["n_devices"] == 1 and r["response_bytes"] > 0 and 0.05 < r["median_ms"] < 50.0


def test_xid_is_pushed_to_the_stream_at_once(P):
    """xid=1 with a running ListAndWatch loop and NO ticker: a device-level Xid makes every stream of the
    context run a heartbeat cycle immediately (the reference would only notice at its next pulse).  The
    synthetic event goes through the same latch + notification as one read from the NVML event set."""
    import queue
    UINT64_MAX = (1 << 64) - 1
    got = queue.Queue()
    with _open(P, 16 * MiB, ",xid=1") as ctx:
        w = ctx.watch(lambda rc, wire, st: got.put((rc, wire, st)), pulse_ms=0, min_gbs=1e-3)
        try:
            rc, wire, st = got.get(timeout=10)                       # initial list
            assert rc == 0 and P.v1beta1.ListAndWatchResponse.FromString(wire).devices[0].health == "Healthy"
            ctx.probe_inject_fault(0, UINT64_MAX, 31)                # application-level: nothing happens
            with pytest.raises(queue.Empty):
                got.get(timeout=0.5)
            ctx.probe_inject_fault(0, UINT64_MAX, 79)                # fallen off the bus
            rc, wire, st = got.get(timeout=5)                        # pushed without any beat()
            assert rc == 0 and st.n_unhealthy == 1
            assert P.v1beta1.ListAndWatchResponse.FromString(wire).devices[0].health == "Unhealthy"
        finally:
            w.stop()


def test_ring_shrinks_when_hbm_is_short_at_open(P):
    """A daemon restart under running pods finds HBM mostly taken.  Opening must not fail (that would take the
    node's GPUs away from the kubelet): the ring slots are halved until they fit, passes stay bit-exact on the
    smaller slots, carry B2DP_RES_SMALL_RING and no GB/s floor."""
    import subprocess
    import sys
    import torch
    free, total = torch.cuda.mem_get_info(0)
    want = 4 << 30                                                   # requested slot size; 2 slots = 8 GiB
    leave = 5 << 30                                                  # what the "pod" leaves free: < 8 GiB, > 2 x 2 GiB
    if free < leave + (8 << 30):
        pytest.skip("GPU already busy")
    helper = subprocess.Popen([sys.executable, "-c",
                               "import torch,time,sys; f,_=torch.cuda.mem_get_info(0); "
                               "x=torch.empty(f-%d, dtype=torch.uint8, device='cuda:0'); print('ready', flush=True); time.sleep(120)" % leave],
                              stdout=subprocess.PIPE, text=True)
    try:
        assert helper.stdout.readline().strip() == "ready"
        with _open(P, want) as ctx:
            seed = oprobe.initial_seed(0)
            for _ in range(3):
                (r,) = ctx.probe_health(min_gbs=1e9)                 # an impossible floor: must not apply
                slot = r.bytes // 2
                assert r.flags & P._native.RES_SMALL_RING and slot in (want // 2, want // 4) and r.err == 0
                assert r.healthy and r.mismatches == 0 and r.seed == seed
                assert r.checksum == r.expected_checksum == oprobe.expected_checksum(slot // 4, seed)
                seed = oprobe.next_seed(seed)
            n_check = 1 << 18
            assert np.array_equal(ctx.probe_peek(0, slot // 4 - n_check, n_check), oprobe.pattern(n_check, seed, slot // 4 - n_check))
            with pytest.raises(P._native.B2dpError):
                ctx.probe_peek(0, slot // 4 - 1, 2)                  # bounds follow the real slot size
            ctx.probe_inject_fault(0, slot // 4 - 1, 1)
            (r,) = ctx.probe_health(min_gbs=1e9)
            assert not r.healthy and r.mismatches == 1 and r.first_bad_word == slot // 4 - 1
    finally:
        helper.kill()
        helper.wait()


def test_one_unusable_gpu_does_not_take_the_node_down(P):
    """A GPU whose setup fails at open (simulated with the break= hook) stays in the device list and is sent
    Unhealthy on every heartbeat; the others keep being probed, allocated and linked.  Only a node with no usable
    GPU fails to open."""
    import torch
    n = torch.cuda.device_count()
    with pytest.raises(P._native.B2dpError) as ei:
        P.Context("cuda:devices=0,bytes=%d,break=0" % (16 * MiB))
    assert ei.value.code == P._native.E_CUDA
    if n < 2:
        pytest.skip("needs 2 GPUs for the partial-failure half")
    with P.Context("cuda:devices=0+1,bytes=%d,p2p_bytes=%d,break=1" % (64 * MiB, 16 * MiB)) as ctx:
        ids = sorted(ctx.enumerate())
        assert len(ids) == 2                                          # still listed
        res = ctx.probe_health(min_gbs=1e-3)
        assert [(r.healthy, r.err) for r in res] == [(True, 0), (False, P._native.E_CUDA)] and res[1].bytes == 0
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, min_gbs=1e-3)
        msg = P.v1beta1.ListAndWatchResponse.FromString(wire)
        assert [(d.ID, d.health) for d in msg.devices] == [(ids[0], "Healthy"), (ids[1], "Unhealthy")] and st.n_unhealthy == 1
        with pytest.raises(P._native.B2dpError):
            ctx.probe_peek(1, 0, 16)
        assert np.array_equal(ctx.probe_peek(0, 0, 16), oprobe.pattern(16, oprobe.next_seed(oprobe.next_seed(oprobe.initial_seed(0)))))
        gbs, lt, mm = ctx.p2p_matrix()
        assert lt[0][1] == 0 and lt[1][0] == 0                        # no link measured to or from the broken GPU
    # the FIRST GPU (lowest BDF) is the broken one: nothing may depend on device 0 being usable -- the checksum
    # reference is the host's closed form, not a kernel on gpus[0] (round-1 advisor finding)
    with P.Context("cuda:devices=0+1,bytes=%d,p2p_bytes=%d,break=0" % (64 * MiB, 16 * MiB)) as ctx:
        ids = sorted(ctx.enumerate())
        for _ in range(2):
            res = ctx.probe_health(min_gbs=1e-3)
            assert [(r.healthy, r.err) for r in res] == [(False, P._native.E_CUDA), (True, 0)] and res[0].bytes == 0
            assert res[1].checksum == res[1].expected_checksum == oprobe.expected_checksum(64 * MiB // 4, res[1].seed)
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, min_gbs=1e-3)
        msg = P.v1beta1.ListAndWatchResponse.FromString(wire)
        assert [(d.ID, d.health) for d in msg.devices] == [(ids[0], "Unhealthy"), (ids[1], "Healthy")]
        gbs, lt, mm = ctx.p2p_matrix()                                # does not fail: the matrix simply has no link to GPU 0
        assert lt[0][1] == 0 and lt[1][0] == 0 and (mm == 0).all()
        ctx.start()                                                   # allocator init degrades (no weights), never crashes
        assert ctx.generate_labels(["vram", "cu-count"])["amd.com/gpu.cu-count"] == "132"


def test_health_floor_is_80_percent_of_the_calibrated_ceiling(P):
    """BASELINE.json: "each per-GPU probe >= 80 % of HBM peak GB/s ... flipping the device Healthy/Unhealthy bit".
    The ceiling (gbs_ref) is calibrated when the context opens; the verdict flips exactly at min_frac = 0.8 of it:
    moving the ceiling so that the same stream sits at 0.81 keeps the device Healthy, at 0.79 it is Unhealthy (data
    still verified).  A pass that really is slow -- launched on a fraction of the SMs (grid_ctas, the stand-in for a
    part that lost bandwidth) -- flips on its own measured GB/s; ListAndWatch carries the verdict."""
    nbytes = 1 << 30
    with _open(P, nbytes) as ctx:
        rs = [ctx.probe_health(timed=False)[0] for _ in range(24)]
        assert all(r.healthy and r.gbs_ref > 0 and 0.95 < r.frac < 1.03 for r in rs), rs
        ref0 = rs[0].gbs_ref
        gbs = sorted(r.gbs for r in rs[4:])[10]                    # timed=False: gbs is on the verdict's in-kernel clock
        # pass-to-pass the in-kernel rate moves by about +-1.5 %, so a single pass parked 1 % from the line may land on
        # either side; what must hold is (a) EVERY verdict agrees with that pass's own measured fraction and floor, and
        # (b) over 9 passes the stream parked at 0.81 is Healthy and the one parked at 0.79 Unhealthy.  Each pass is
        # parked relative to the pass just before it: a power-capped card's rate drifts by more than that over the test
        last = gbs
        for frac, want in ((0.81, True), (0.79, False), (0.81, True), (0.79, False)):
            got = []
            for _ in range(9):
                ctx.probe_set_ref(0, last / frac)
                (r,) = ctx.probe_health(timed=False)
                last = r.gbs
                assert r.mismatches == 0 and r.checksum == r.expected_checksum and r.err == 0
                if abs(r.frac - 0.8) > 1e-4:
                    assert r.healthy == (r.frac >= 0.8) and bool(r.flags & P._native.RES_SLOW) == (r.frac < 0.8), r
                assert abs(r.min_gbs_applied - oprobe.health_floor(nbytes, r.gbs_ref)) < 1.0    # the oracle's floor rule
                if not got:     # the oracle's full verdict rule (it re-sums the 1 GiB pattern: once per setting is enough)
                    assert r.healthy == oprobe.probe_healthy(True, r.checksum, r.mismatches, nbytes // 4, r.seed,
                                                             r.frac * r.gbs_ref, r.min_gbs_applied) or abs(r.frac - 0.8) <= 1e-4
                got.append(r)
            fr = sorted(r.frac for r in got)
            assert abs(fr[4] - frac) < 0.008, (frac, fr)
            assert sum(r.healthy == want for r in got) >= 7, (frac, [(round(r.frac, 4), r.healthy) for r in got])
        ctx.probe_set_ref(0, last / 0.75)                         # well clear of the line for the single ListAndWatch check
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT)
        assert [d.health for d in P.v1beta1.ListAndWatchResponse.FromString(wire).devices] == ["Unhealthy"]
        assert 0.73 < st.probe_frac_min < 0.77 and st.probe_ms_device_max > 0
        ctx.probe_set_ref(0, 0.0)                                   # back to the calibration
        (r,) = ctx.probe_health(timed=False)
        assert r.healthy and abs(r.gbs_ref - ref0) < 1.0
        # a genuinely slow stream: the verdict follows the measured fraction on every grid
        verdicts = []
        for grid in (264, 198, 132, 99, 66, 33, 18):
            (r,) = ctx.probe_health(timed=False, grid_ctas=grid)
            assert r.mismatches == 0 and r.checksum == r.expected_checksum
            assert r.healthy == (r.frac >= 0.8), (grid, r)
            verdicts.append((grid, round(r.frac, 3), r.healthy))
        assert verdicts[0][2] and not verdicts[-1][2], verdicts     # full grid Healthy, 18 CTAs far below the floor
        # absolute override: min_gbs replaces the fractional floor for a call ...
        (r,) = ctx.probe_health(timed=False, grid_ctas=18, min_gbs=1.0)
        assert r.healthy and r.min_gbs_applied == 1.0
    # ... or for the context; min_frac moves the line; ref_gbs pins the ceiling
    with _open(P, nbytes, ",min_frac=0.5,ref_gbs=3600") as ctx:
        (r,) = ctx.probe_health(timed=False)
        assert r.gbs_ref == 3600.0 and r.healthy and abs(r.min_gbs_applied - 1800.0) < 1.0 and 0.7 < r.frac < 0.9
    with _open(P, nbytes, ",ref_gbs=4000") as ctx:
        (r,) = ctx.probe_health(timed=False)
        assert not r.healthy and r.flags & P._native.RES_SLOW       # ~2.85 of 4.0 TB/s = 0.71: below the line
    # slow_passes=3: a dip is flagged at once but only the third consecutive slow pass is a verdict; a fast pass resets it
    with _open(P, nbytes, ",slow_passes=3") as ctx:
        seen = [ctx.probe_health(timed=False, grid_ctas=18)[0] for _ in range(4)]
        assert all(r.flags & P._native.RES_SLOW for r in seen) and [r.healthy for r in seen] == [True, True, False, False]
        assert ctx.probe_health(timed=False)[0].healthy
        seen = [ctx.probe_health(timed=False, grid_ctas=18)[0] for _ in range(2)]
        assert [r.healthy for r in seen] == [True, True]
        ctx.probe_inject_fault(0, 5, 1)                             # integrity is never debounced
        assert not ctx.probe_health(timed=False)[0].healthy
    # a ring that fits the L2 carries no fractional floor (the pass does not measure HBM)
    with _open(P, 16 * MiB) as ctx:
        (r,) = ctx.probe_health(timed=False)
        assert r.healthy and r.flags & P._native.RES_NO_FLOOR and r.min_gbs_applied == 0.0 and r.gbs_ref > 0
        assert oprobe.health_floor(16 * MiB, r.gbs_ref) == 0.0 and oprobe.health_floor(16 * MiB, r.gbs_ref, abs_min_gbs=5.0) == 5.0
        (r,) = ctx.probe_health(timed=False, min_gbs=1e9)
        assert not r.healthy and not (r.flags & P._native.RES_NO_FLOOR)


def test_expected_checksum_is_the_host_closed_form(P):
    """The reference value of the verdict comes from the host (b2dp_expected_checksum), not from a kernel on the GPU
    under test: on ragged sizes it equals both the GPU's accumulated checksum and the oracle's numpy sum."""
    import ctypes as C
    for nbytes in (4096, MiB + 48, 3 * MiB + 16 * 37):
        with _open(P, nbytes) as ctx:
            (r,) = ctx.probe_health(min_gbs=1e-3)
            out = C.c_uint64(0)
            assert P._native.lib.b2dp_expected_checksum(nbytes // 4, r.seed, C.byref(out)) == 0
            assert r.expected_checksum == out.value == r.checksum == oprobe.expected_checksum(nbytes // 4, r.seed)


def test_helper_launcher_path_equals_direct_path(P):
    """`launchers=2,pin=1`: a second thread enqueues the other half of the GPUs while the caller enqueues its own.  Same
    state machine, same answers: seeds, checksums and verdicts equal those of a default context pass by pass, a fault
    on a helper-launched GPU is caught once, and the library's own ListAndWatch loop (which pre-arms the helper before
    each tick) streams Healthy."""
    import queue
    import torch
    n = torch.cuda.device_count()
    nbytes = 64 * MiB + 16 * 9
    with P.Context("cuda:bytes=%d,launchers=2,pin=1,spin_us=200" % nbytes) as a, P.Context("cuda:bytes=%d" % nbytes) as b:
        for step in range(5):
            ra, rb = a.probe_health(min_gbs=1e-3, timed=bool(step % 2)), b.probe_health(min_gbs=1e-3)
            assert [(r.seed, r.checksum, r.expected_checksum, r.mismatches, r.healthy) for r in ra] == \
                   [(r.seed, r.checksum, r.expected_checksum, r.mismatches, r.healthy) for r in rb]
            assert all(r.healthy for r in ra) and len(ra) == n
        a.probe_inject_fault(n - 1, 4321, 0x8)                   # the last GPU is the helper's when there are >= 2
        ra = a.probe_health(min_gbs=1e-3)
        assert [r.healthy for r in ra] == [True] * (n - 1) + [False] and ra[-1].first_bad_word == 4321
        assert all(r.healthy for r in a.probe_health(min_gbs=1e-3))
        got = queue.Queue()
        w = a.watch(lambda rc, wire, st: got.put((rc, wire, st)), pulse_ms=10, min_gbs=1e-3)
        try:
            for _ in range(6):
                rc, wire, st = got.get(timeout=10)
                assert rc == 0 and st.n_unhealthy == 0 and st.n_devices == n
        finally:
            w.stop()
    for bad in ("cuda:devices=0,launchers=3", "cuda:devices=0,spin_us=-1", "cuda:devices=0,min_frac=2", "cuda:devices=0,calib=99",
                "cuda:devices=0,id_strategy=minor"):
        with pytest.raises(P._native.B2dpError):
            P.Context(bad)


def test_probe_through_helper_processes(P):
    """probe=helpers: the parent never creates a CUDA context; one b200dp_probe_helper child per GPU (started with
    CUDA_VISIBLE_DEVICES=<its UUID>) runs the ordinary probe.  This is the path every MIG instance takes (CUDA shows a
    process a single compute instance); here it runs on whole GPUs so that it is verified on real hardware: passes are
    bit-exact with the oracle, the seed schedule is the enumeration index's, faults are caught once, the fractional
    floor applies, a killed helper is reported Unhealthy and restarted by the next heartbeat."""
    import signal
    import time
    import torch
    n = torch.cuda.device_count()
    nbytes = 192 * MiB + 16 * 11
    n_words = nbytes // 4
    with P.Context("cuda:bytes=%d,calib=0" % MiB) as direct:
        direct_table = direct.enumerate()
    with P.Context("cuda:probe=helpers,bytes=%d" % nbytes) as ctx:
        assert ctx.enumerate() == direct_table                       # same table as the in-process backend
        info = P._native.ProbeInfo()
        for i in range(n):
            assert P._native.lib.b2dp_probe_describe(ctx._h, i, info) == 0
            assert info.via_helper == 1 and info.usable == 1 and info.slot_bytes == nbytes and info.sm_count == 132
            assert info.uuid.decode().startswith("GPU-") and info.gbs_ref >= info.gbs_cal > 1000.0
        seeds = [oprobe.initial_seed(i) for i in range(n)]
        for step in range(3):
            before = ctx.probe_peek(n - 1, 0, n_words)
            assert np.array_equal(before, oprobe.pattern(n_words, seeds[n - 1]))
            res = ctx.probe_health(timed=False)
            assert [r.device for r in res] == list(range(n)) and [r.seed for r in res] == seeds
            for r in res:
                assert r.err == 0 and r.healthy and r.mismatches == 0 and r.bytes == 2 * nbytes
                assert r.checksum == r.expected_checksum == oprobe.expected_checksum(n_words, r.seed)
                assert r.frac > 0.8 and abs(r.min_gbs_applied - 0.8 * r.gbs_ref) < 1.0
            cs, bad, first, dst = oprobe.probe_pass(before, seeds[n - 1], oprobe.next_seed(seeds[n - 1]))
            assert np.array_equal(ctx.probe_peek(n - 1, 0, n_words), dst)
            seeds = [oprobe.next_seed(s) for s in seeds]
        ctx.probe_inject_fault(0, 31337, 0x40)
        res = ctx.probe_health(timed=False)
        assert (res[0].healthy, res[0].mismatches, res[0].first_bad_word) == (False, 1, 31337)
        assert all(r.healthy for r in res[1:])
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT)
        assert st.n_devices == n and st.n_unhealthy == 0            # reported once; the helper re-filled its ring
        ctx.probe_set_ref(0, 1e6)                                    # a ceiling no part reaches: below the 0.8 line
        res = ctx.probe_health(timed=False)
        assert res[0].flags & P._native.RES_SLOW and abs(res[0].min_gbs_applied - 0.8e6) < 1.0 and all(r.healthy for r in res[1:])
        # A slow pass is a verdict on the part only if nothing else was using the GPU.  This pytest process has held a
        # CUDA context on GPU 0 since the earlier in-process tests, so NVML lists two compute processes (it and the
        # helper): the pass is flagged CONTENDED and judged on integrity alone.  Without process accounting (some
        # containers) or with the helper alone on its GPU the verdict is Unhealthy.
        if res[0].flags & P._native.RES_CONTENDED:
            assert res[0].healthy and res[0].mismatches == 0 and res[0].checksum == res[0].expected_checksum
        else:
            assert not res[0].healthy
        ctx.probe_set_ref(0, 0.0)
        assert all(r.healthy for r in ctx.probe_health(timed=False))
        # Start(): no CUDA here, so the link classes are declared from NVML (NVLink on an HGX board), not measured
        if n > 1:
            assert ctx.start() == 0
            ids = sorted(ctx.enumerate())
            assert len(ctx.preferred_allocation(ids, [], 2)) == 2
            gbs, lt, mm = ctx.p2p_matrix()
            assert (gbs == 0).all() and all(lt[i, j] == 11 for i in range(n) for j in range(n) if i != j)
        # kill one helper: Unhealthy with E_CUDA on the next pass, restarted by the one after
        out = subprocess_pids_of_helpers()
        assert len(out) >= n
        os.kill(out[-1], signal.SIGKILL)
        time.sleep(0.2)
        res = ctx.probe_health(timed=False, min_gbs=1e-3)
        dead = [r for r in res if r.err != 0]
        assert len(dead) == 1 and dead[0].err == P._native.E_CUDA and not dead[0].healthy
        # the replacement (a fresh CUDA process: seconds) is started without stalling the heartbeats in between
        t_end = time.time() + 60
        while time.time() < t_end:
            t0 = time.perf_counter()
            res = ctx.probe_health(timed=False, min_gbs=1e-3)
            assert time.perf_counter() - t0 < 1.0
            if all(r.err == 0 for r in res):
                break
            time.sleep(0.2)
        assert all(r.err == 0 and r.healthy for r in res)
    time.sleep(0.3)
    assert subprocess_pids_of_helpers() == []                       # closing the context reaps every child
    # xid=1 works without CUDA in the parent: NVML delivers critical Xids for the physical GPU (synthetic events here)
    UINT64_MAX = (1 << 64) - 1
    with P.Context("cuda:probe=helpers,devices=0,bytes=%d,xid=1" % (16 * MiB)) as x:
        assert x.probe_health(min_gbs=1e-3)[0].healthy
        x.probe_inject_fault(0, UINT64_MAX, 31)                      # application-level: ignored
        assert x.probe_health(min_gbs=1e-3)[0].healthy
        x.probe_inject_fault(0, UINT64_MAX, 79)                      # fallen off the bus
        (r,) = x.probe_health(min_gbs=1e-3)
        assert not r.healthy and r.flags & P._native.RES_XID and r.mismatches == 0 and r.checksum == r.expected_checksum
        x.probe_reset(0)
        assert x.probe_health(min_gbs=1e-3)[0].healthy


def subprocess_pids_of_helpers():
    """pids of this process's b200dp_probe_helper children (by /proc, no pattern kill)."""
    me = os.getpid()
    pids = []
    for d in os.listdir("/proc"):
        if not d.isdigit():
            continue
        try:
            stat = open("/proc/%s/stat" % d).read()
            ppid = int(stat.rsplit(")", 1)[1].split()[1])
            if ppid == me and "b200dp_probe_h" in stat:
                pids.append(int(d))
        except OSError:
            pass
    return sorted(pids)


def test_probe_off_enumerates_real_gpus_through_nvml(P):
    """probe=off on real hardware: the same device table as the in-process backend, built from NVML alone (no CUDA
    context, no HBM ring -- the free memory of the GPUs does not move), labels from NVML equal to the in-process
    backend's CUDA/NVML answers, and the native daemon's labeller mode on top of it."""
    import json
    import subprocess
    import torch
    with P.Context("cuda:bytes=%d,calib=0" % MiB) as direct:
        table = direct.enumerate()
        gens = ["driver-version", "device-id", "product-name", "simd-count", "cu-count", "family", "firmware",
                "compute-memory-partition", "compute-partitioning-supported", "memory-partitioning-supported"]
        want = direct.generate_labels(gens)
        want_vram = direct.generate_labels(["vram"])
    free0 = [torch.cuda.mem_get_info(i)[0] for i in range(torch.cuda.device_count())]
    with P.Context("cuda:probe=off") as ctx:
        assert ctx.enumerate() == table
        assert [torch.cuda.mem_get_info(i)[0] for i in range(torch.cuda.device_count())] == free0      # nothing allocated
        assert ctx.generate_labels(gens) == want
        got_vram = ctx.generate_labels(["vram"])
        # NVML's total (the whole HBM) vs CUDA's totalGlobalMem (minus the driver's reservation) may round to
        # neighbouring GiB values; both are H100-sized (80 GB)
        assert set(got_vram) == set(k.replace(want_vram["amd.com/gpu.vram"], got_vram["amd.com/gpu.vram"]) for k in want_vram)
        assert 75 <= int(got_vram["amd.com/gpu.vram"][:-1]) <= 80
        d = ctx.probe_describe(0)
        assert d["uuid"].startswith("GPU-") and d["sm_count"] == 132 and not d["via_helper"]
        with pytest.raises(P._native.B2dpError) as ei:
            ctx.probe_health()
        assert ei.value.code == P._native.E_UNSUPPORTED
        ids = sorted(table)
        resp = P.v1beta1.ContainerAllocateResponse.FromString(ctx.allocate_response(ids[:1]))
        assert dict(resp.envs)["NVIDIA_VISIBLE_DEVICES"] == d["uuid"]
        assert [x.host_path for x in resp.devices][-1] == "/dev/nvidia%d" % table[ids[0]]["card"]
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "k8s-device-plugin_b200", "b200dp_plugind")
    r = subprocess.run([exe, "-labels=" + ",".join(gens), "-backend=cuda:"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert json.loads(r.stdout) == want


def test_prearmed_passes_equal_launched_passes(P):
    """prearm=1: while pass k runs, pass k+1 is enqueued behind a stream wait on a host-mapped doorbell and the next
    heartbeat only rings it.  Same state machine, same answers: seeds, checksums, buffers and verdicts equal those of a
    context that launches every pass; every steady-state pass carries B2DP_RES_PREARMED; whatever does not fit an armed
    pass (peek, poke, a timed or shrunk or differently shaped pass, a fault repair, reset, the P2P matrix, close) discards
    it without disturbing the sequence; a pass that misses its deadline with another armed behind it is still collected."""
    # Runs in its own process (tests/_prearm_scenario.py): while a pass is armed, device-synchronising calls of the SAME
    # process wait for the doorbell, and this pytest process holds a torch context -- prearm is for a process whose only
    # GPU user is the library.  A hang there is a clean failure here.
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, os.path.join(here, "_prearm_scenario.py")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PREARM_OK" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
