"""CPU tests of the on-demand register-file self-test (b2dp_regfile_test): the host arithmetic against the oracle, the
faulty-register models against the direct compare and the fold, the ABI constants, the backends and daemon without
the test, and the SASS of the product kernels (the march really held in registers)."""
import ctypes as C
import os
import re
import shutil
import signal
import subprocess
import time

import numpy as np
import pytest

import fake_sysfs
import rf_test_oracle as ro
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
LIB = os.path.join(ROOT, "tests", "native", "libregfile_test_kernels_test.so")
SEEDS = [0, 1, 0xC0FFEE17, 0xFFFFFFFF]
FMT_IDS = [ro.NAMES[f] for f in ro.FORMATS]
REGS = [0, ro.HELD // 2, ro.HELD - 1]          # the first, a middle and the last held register
MIN_HELD = 192                                  # 75 % of the 256 registers a thread is allocated
# Transitions ptxas writes in place (Rd == Ra), per element.  With CUDA 12.9 its register allocator writes up to 12 of an
# element's 204 transitions to a neighbouring register whose old value is dead, shifting a short chain of values by a
# register or two around the element's temporaries (DESIGN 4.10); the rest, 192-204, are in place.
MIN_IN_PLACE = 184                              # 90 % of kRfHeld


class MathDriver:
    """tests/native/rf_test_math_test.cpp, compiled with g++ against csrc/rf_test_math.hpp."""

    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(self, *words):
        self.p.stdin.write(" ".join(str(w) for w in words) + "\n")
        self.p.stdin.flush()
        return [int(x) for x in self.p.stdout.readline().split()]

    def close(self):
        self.p.stdin.close()
        self.p.wait(timeout=10)


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("rf") / "rf_test_math_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                        os.path.join(ROOT, "tests", "native", "rf_test_math_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = MathDriver(exe)
    yield d
    d.close()


def _tile(seed, fmt, t):
    return ro.kind(t), ro.key(seed, fmt, t)


# ---- the host arithmetic against the oracle ---------------------------------------------------------------------
def test_layout(drv):
    assert drv.ask("layout") == [ro.HELD, ro.TABLE_WORDS, ro.HOOK_REG, ro.HOOK_ELEMENT, ro.HOOK_THREAD,
                                 ro.PARAM_WORDS, ro.SMEM_BYTES, ro.DUMP_WORDS] + \
        [ro.ELEMENTS[f] for f in ro.FORMATS] + [ro.HOLD_NS]
    assert ro.HELD >= MIN_HELD and ro.HELD % 4 == 0
    # two CTAs per SM: 2 x (dynamic + the 1 KiB the runtime reserves) within the SM's 228 KiB
    assert 2 * (ro.SMEM_BYTES + 1024) <= 228 * 1024


@pytest.mark.parametrize("seed", SEEDS)
def test_patterns_and_the_kernel_generator_match_the_oracle(drv, seed):
    for t in range(ro.TILES):
        kd, ky = _tile(seed, 0, t)
        for th in (0, 1, 31, 64, 127):
            want = ro.pattern(kd, ky, th, np.arange(ro.HELD)).tolist()
            assert drv.ask("pattern", kd, ky, th) == want, (t, th)
            assert drv.ask("gen", kd, ky, th) == want, (t, th)


def test_distinct_value_tiles_give_every_register_of_the_cta_its_own_value():
    for t in range(4, ro.TILES):
        p = ro.pattern(*_tile(5, 0, t))
        assert np.unique(p).size == p.size, t


@pytest.mark.parametrize("fmt", ro.FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", SEEDS)
def test_host_tables_and_checks_match_the_oracle(drv, seed, fmt):
    """Every tile's table, and every thread's check value: the fold of the oracle's clean march."""
    tabs = ro.tables(seed, fmt)
    for t in range(ro.TILES):
        got = drv.ask("tile", seed, fmt, t)
        assert got[:ro.TABLE_WORDS] == tabs[t].tolist()
        r = ro.march(fmt, *_tile(seed, fmt, t))
        assert got[ro.TABLE_WORDS:] == r["fold"].tolist(), (seed, fmt, t)
        assert not r["err"].any()
        want_final = ro.pattern(*_tile(seed, fmt, t)) ^ np.uint32(0 if fmt == ro.ALU else ro.M32)
        assert np.array_equal(r["regs"], want_final)


@pytest.mark.parametrize("fmt", ro.FORMATS, ids=FMT_IDS)
def test_read_order_matches_the_oracle(drv, fmt):
    kd, ky = 4, 0x9E3779B9
    r = ro.march(fmt, kd, ky, keep_reads=True)
    for t in (0, 1, 31, 64, 127):
        want = r["reads"][t].tolist()
        assert len(want) == ro.READS[fmt] * ro.HELD
        assert drv.ask("reads", fmt, kd, ky, t) == want, (fmt, t)
        assert ro.fold(want) == int(r["fold"][t])


# ---- the faulty-register models -----------------------------------------------------------------------------------
def _cells(cells, value=ro.M32):
    m = np.zeros((ro.THREADS, ro.HELD), np.uint32)
    for t, j in cells:
        m[t, j] = value
    return m


@pytest.mark.parametrize("fmt", ro.FORMATS, ids=FMT_IDS)
def test_stuck_at_every_bit_is_caught_by_the_direct_compare_in_every_tile(fmt):
    """Every bit of the first, a middle and the last held register stuck at 0 (threads 0-2) and at 1 (threads 3-5):
    every stuck bit is read wrong somewhere in every tile, so each of those threads' error bits is all ones."""
    stuck0 = [(i, j) for i, j in enumerate(REGS)]
    stuck1 = [(3 + i, j) for i, j in enumerate(REGS)]
    mask = _cells(stuck0) | _cells(stuck1)
    for t in range(ro.TILES):
        kd, ky = _tile(7, fmt, t)
        r = ro.march(fmt, kd, ky, rf=ro.Stuck(mask, _cells(stuck1), init=ro.steady(fmt, kd, ky)))
        assert (r["err"][:6] == ro.M32).all(), (fmt, t, [hex(x) for x in r["err"][:6]])
        assert not r["err"][6:].any()


@pytest.mark.parametrize("fmt", ro.FORMATS, ids=FMT_IDS)
def test_transition_faults_are_caught_in_every_tile(fmt):
    """Every bit of those registers unable to rise (threads 0-2) or to fall (threads 3-5), from what the previous
    repetition left: every march writes each bit both ways and reads it after each."""
    up = [(i, j) for i, j in enumerate(REGS)]
    down = [(3 + i, j) for i, j in enumerate(REGS)]
    for t in range(ro.TILES):
        kd, ky = _tile(7, fmt, t)
        r = ro.march(fmt, kd, ky, rf=ro.Transition(_cells(up), _cells(down), init=ro.steady(fmt, kd, ky)))
        assert (r["err"][:6] == ro.M32).all(), (fmt, t, [hex(x) for x in r["err"][:6]])


@pytest.mark.parametrize("fmt", ro.FORMATS, ids=FMT_IDS)
def test_a_write_that_lands_in_another_register_is_caught_in_the_distinct_value_tiles(fmt):
    caught = {}
    for t in range(ro.TILES):
        kd, ky = _tile(11, fmt, t)
        caught[t] = []
        for th, j, j2 in ((0, 0, 1), (31, ro.HELD // 2, 7), (127, ro.HELD - 1, 0)):
            r = ro.march(fmt, kd, ky, rf=ro.Misroute(th, j, j2, init=ro.steady(fmt, kd, ky)))
            caught[t].append(bool(r["err"][th]))
        if t >= 4:
            assert all(caught[t]), (fmt, t, caught[t])
    print(ro.NAMES[fmt], "misrouted writes caught per tile:", caught)


@pytest.mark.parametrize("width", [4, 2], ids=["quad", "pair"])
def test_a_dropped_lane_of_a_wide_load_is_caught_in_every_tile(width):
    """RF_LOAD writes every register twice by quad and twice by pair loads, always with the complement of what it
    held: a lane the load drops keeps the old value, which the next read finds wrong."""
    for t in range(ro.TILES):
        kd, ky = _tile(9, ro.LOAD, t)
        for th, j in ((0, 0), (64, ro.HELD // 2 + 1), (127, ro.HELD - 1)):
            r = ro.march(ro.LOAD, kd, ky, rf=ro.LaneDrop(th, j, width, init=ro.steady(ro.LOAD, kd, ky)))
            assert r["err"][th] == ro.M32 and not np.delete(r["err"], th).any(), (width, t, th, j)


@pytest.mark.parametrize("n", [0, 1])
def test_a_value_that_flips_during_the_hold_is_caught_in_every_tile(n):
    for t in range(ro.TILES):
        kd, ky = _tile(13, ro.HOLD, t)
        for th, j in ((0, 0), (64, ro.HELD // 2), (127, ro.HELD - 1)):
            for mask in (1, 1 << 31, ro.M32):
                r = ro.march(ro.HOLD, kd, ky, rf=ro.HoldFlip(th, j, mask, n, init=ro.steady(ro.HOLD, kd, ky)))
                assert r["err"][th] == mask, (n, t, th, j, mask)


@pytest.mark.parametrize("fmt", ro.FORMATS, ids=FMT_IDS)
def test_the_fault_hook_is_read_back_after_every_element_but_the_last(fmt):
    for e in range(ro.ELEMENTS[fmt]):
        for th, j in ((0, 0), (127, ro.HELD - 1)):
            r = ro.march(fmt, *_tile(3, fmt, 4), hook=(e, th, j, 0x80000000))
            assert bool(r["err"][th]) == (e < ro.ELEMENTS[fmt] - 1), (fmt, e, th, j)


def test_the_fold_alone_misses_a_stuck_bit_31_and_the_direct_compare_does_not():
    """March C- reads a bit stuck at 0 under the solid tile wrong in its two r(~P) elements: at bit 31 the two errors
    add 2^31 (w1 + w2) with w1 + w2 even, 0 mod 2^32."""
    th, j = 5, 100
    r = ro.march(ro.ALU, 0, 0, rf=ro.Stuck(_cells([(th, j)], 1 << 31), np.zeros((ro.THREADS, ro.HELD), np.uint32)))
    clean = ro.march(ro.ALU, 0, 0)
    assert r["err"][th] == 1 << 31
    assert r["fold"][th] == clean["fold"][th]


# ---- ABI, backends, daemon ------------------------------------------------------------------------------------------
def test_constants_and_struct_layouts(pkg):
    N = pkg._native
    assert (N.RF_ALU, N.RF_LOAD, N.RF_HOLD) == (0, 1, 2)
    assert C.sizeof(N.ComputeTestOpts) == 24 and C.sizeof(N.ComputeTestResult) == 128
    hdr = open(os.path.join(ROOT, "include", "b200dp.h")).read()
    for name, v in (("B2DP_RF_ALU", 0), ("B2DP_RF_LOAD", 1), ("B2DP_RF_HOLD", 2)):
        assert re.search(r"#define %s %s\b" % (name, v), hdr), name
    assert "b2dp_regfile_test" in hdr and "b2dp_regfile_test" in N.SIGNATURES


def test_backends_without_a_regfile_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.regfile_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:      # cuda:probe=off (NVML only)
        with pytest.raises(N.B2dpError) as ei:
            ctx.regfile_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "in-process only" in str(ei.value)
        assert "register-file self-test" in str(ei.value)


def test_daemon_regfile_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-regfile_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "regfile test at start not run: not supported by this backend" in err, err[-2000:]
    assert "Failed to start plugin gpu: Register:" in err


# ---- the SASS: the march held in registers -------------------------------------------------------------------------
_NO_DST = ("ST", "STS", "STL", "STG", "BAR", "BRA", "EXIT", "RED", "ATOM", "NANOSLEEP", "MEMBAR", "WARPSYNC", "CALL",
           "RET", "BSSY", "BSYNC", "NOP", "ERRBAR", "CCTL", "DEPBAR", "YIELD", "ISETP")


def _regs(arg):
    """The general registers an operand names (R12, R12.reuse, [R12+0x4], -R3, R12.64 -> 12, 13); not UR / RZ."""
    out = []
    for m in re.finditer(r"(?<![A-Z])R(\d+)(\.64|\.128)?", arg):
        r = int(m.group(1))
        out += list(range(r, r + {".64": 2, ".128": 4}.get(m.group(2), 1)))
    return out


def _instructions(sass, name):
    (body,) = [p for p in re.split(r"\n\s+Function : ", sass)[1:] if name in p.split("\n")[0]]
    out = []
    for a, i in re.findall(r"/\*([0-9a-f]{4,})\*/\s+([^;]*);", body):
        i = i.strip()
        pred = re.match(r"^@!?U?P\w+\s+", i)
        i = i[pred.end():] if pred else i
        op, _, rest = i.partition(" ")
        args = [x.strip() for x in rest.split(",")] if rest else []
        base = op.split(".")[0]
        if base in _NO_DST or base.startswith("U") or not args or args[0].startswith("P"):
            dst, src = [], [r for x in args for r in _regs(x)]
        else:
            dst, src = _regs(args[0]), [r for x in args[1:] for r in _regs(x)]
            if base == "LDS" and dst:
                dst = list(range(dst[0], dst[0] + (4 if ".128" in op else 2 if ".64" in op else 1)))
        out.append(dict(a=int(a, 16), op=op, args=args, dst=dst, src=src, raw=i, pred=bool(pred)))
    return out


def _repetition_loop(ins):
    """The repetition loop, found by its own back-edge: the innermost backward branch around the repetition's
    BAR.RED.OR."""
    bar = min(x["a"] for x in ins if x["op"].startswith("BAR.RED.OR"))
    end = max(x["a"] for x in ins if x["op"] == "EXIT")
    back = []
    for x in ins:
        m = re.search(r"BRA (?:`\()?0x([0-9a-f]+)", x["raw"])
        if x["op"].startswith("BRA") and m and int(m.group(1), 16) <= bar < x["a"] < end:
            back.append((x["a"], int(m.group(1), 16)))
    src, tgt = min(back, key=lambda st: st[0] - st[1])
    return [x for x in ins if tgt <= x["a"] <= src]


def _without_hook(loop):
    """The loop without the fault hook's cold code.  After a barrier, a predicated forward BRA skips the hook, whose
    code reads its table with volatile global loads (LDG.E.STRONG.SYS) and XORs a select into every held register;
    those XORs are not the march's transitions and its reads are not the march's reads.  Returns the remaining
    instructions and the number of hook regions removed."""
    out, k, regions = [], 0, 0
    while k < len(loop):
        x = loop[k]
        out.append(x)
        nxt = loop[k + 1] if k + 1 < len(loop) else None
        m = nxt and re.search(r"BRA (?:`\()?0x([0-9a-f]+)", nxt["raw"])
        if x["op"].startswith("BAR.SYNC") and m and nxt["pred"] and int(m.group(1), 16) > nxt["a"]:
            tgt = int(m.group(1), 16)
            body = [y for y in loop[k + 2:] if y["a"] < tgt]
            if any(y["op"].startswith("LDG.E.STRONG.SYS") for y in body):
                regions += 1
                k += 2 + len(body)
                continue
        k += 1
    return out, regions


def _norm(arg):
    return arg.replace(".reuse", "")


def _is_xor(x):
    """A 2-input XOR: LOP3.LUT d, a, b, RZ, 0x3c."""
    return x["op"].startswith("LOP3") and len(x["args"]) >= 5 and x["args"][3] == "RZ" and x["args"][4] == "0x3c"


def _transitions(segment):
    """An element's transitions: the XORs with its mask, the operand most of the segment's XORs share (a uniform or
    general register loaded after the barrier).  Returns them and the mask operand."""
    xors = [x for x in segment if _is_xor(x)]
    if not xors:
        return [], None
    count = {}
    for x in xors:
        for arg in {_norm(x["args"][1]), _norm(x["args"][2])}:
            count[arg] = count.get(arg, 0) + 1
    mask = max(count, key=count.get)
    return [x for x in xors if mask in (_norm(x["args"][1]), _norm(x["args"][2]))], mask


def _in_place(x, mask):
    """The transition writes the register it reads: d == the operand that is not the mask."""
    a = _norm(x["args"][2]) if _norm(x["args"][1]) == mask else _norm(x["args"][1])
    return x["dst"] == _regs(a)


def _is_element_write(x):
    return x["op"].startswith("LDS") or _is_xor(x)


def _held_across(loop, b):
    """The registers holding march data across the barrier at loop[b]: last written before it by an element write
    (a shared-memory load, or a transition), and first touched after it by a read."""
    held = set()
    for reg in range(255):
        last = next((loop[k] for k in range(b - 1, -1, -1) if reg in loop[k]["dst"]), None)
        if last is None or not _is_element_write(last):
            continue
        first = next((x for x in loop[b + 1:] if reg in x["dst"] or reg in x["src"]), None)
        if first is None or reg not in first["src"]:
            continue
        held.add(reg)
    return held


def _first_touch(loop, b, reg):
    return next(k for k in range(b + 1, len(loop)) if reg in loop[k]["dst"] or reg in loop[k]["src"])


@pytest.fixture(scope="module")
def sass():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(LIB) or not os.path.exists(tool):
        pytest.skip("needs the built harness and cuobjdump")
    return (subprocess.run([tool, "-sass", LIB], capture_output=True, text=True).stdout,
            subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True).stdout)


SASS_REQUIRED = {ro.ALU: ["LDS.128"], ro.LOAD: ["LDS.128", "LDS.64"], ro.HOLD: ["LDS.128", "NANOSLEEP"]}
# the elements that transition their registers in place (an LOP3 with the mask) rather than load them
FLIPS = {ro.ALU: [1, 2, 3, 4], ro.LOAD: [], ro.HOLD: [1]}


@pytest.mark.parametrize("fmt", ro.FORMATS, ids=FMT_IDS)
def test_sass_holds_the_march_in_registers(sass, fmt):
    """The product instantiation, in the repetition loop without the fault hook's cold code: one barrier per element;
    at least MIN_HELD registers held across every element boundary, each last written before it by a shared-memory
    load or a transition and first touched after it by a read (a value recomputed after the barrier is not held: no
    rematerialisation); every transition an in-place LOP3 with the element's mask; RF_HOLD's held registers first read
    after the hold; no local memory; and each format's own accesses.  A register may serve as a temporary elsewhere in
    the loop."""
    text, res = sass
    name = "rf_selftestILi%dELb0E" % fmt
    ins = _instructions(text, name)
    assert not [x for x in ins if x["op"].split(".")[0] in ("STL", "LDL")], "local memory in " + name
    lines = res.splitlines()
    (k,) = [k for k, ln in enumerate(lines) if name in ln]
    assert re.search(r"\bLOCAL:0\b", lines[k + 1]), lines[k + 1]
    loop, hooks = _without_hook(_repetition_loop(ins))
    assert hooks >= ro.ELEMENTS[fmt] - 1, hooks           # after every element a read follows
    assert not [x for x in loop if x["op"].startswith("LDG.E.STRONG.SYS")], "hook code left in the loop"
    ops = [x["op"] for x in loop]
    for want in SASS_REQUIRED[fmt]:
        assert want in ops, (fmt, want)
    bars = [i for i, x in enumerate(loop) if x["op"].startswith("BAR.SYNC")]
    assert len(bars) == ro.ELEMENTS[fmt], [hex(loop[b]["a"]) for b in bars]
    held = [_held_across(loop, b) for b in bars[:-1]]      # the last barrier ends the march: nothing is read after it
    counts = [len(h) for h in held]
    union = set().union(*held)
    # element e runs between barriers e - 1 and e
    segments = [loop[(bars[e - 1] + 1 if e else 0):bars[e]] for e in range(ro.ELEMENTS[fmt])]
    flips, kept_alive = [], []
    for e in FLIPS[fmt]:
        trans, mask = _transitions(segments[e])
        flips.append((e, mask, len(trans), sum(_in_place(x, mask) for x in trans)))
        # a transition not in place must still end its source: the old value's next touch is a write
        for x in trans:
            if not _in_place(x, mask):
                src = [r for r in x["src"] if r not in _regs(mask)]
                k = loop.index(x)
                nxt = next((y for y in loop[k + 1:] if src[0] in y["dst"] or src[0] in y["src"]), None)
                if nxt is not None and src[0] in nxt["src"]:
                    kept_alive.append((x["raw"], nxt["raw"]))
    loads = {o: ops.count(o) for o in ("LDS.128", "LDS.64")}
    print("%s: held across each element boundary %s (N = %d, union %d registers R%d..R%d); transitions per element "
          "(element, mask, count, in place) %s; %s; %d hook regions left out"
          % (ro.NAMES[fmt], counts, min(counts), len(union), min(union), max(union), flips, loads, hooks))
    assert min(counts) >= MIN_HELD, counts
    assert max(counts) <= ro.HELD + 4, counts
    for e, mask, n, in_place in flips:
        assert n == ro.HELD and in_place >= MIN_IN_PLACE, (e, mask, n, in_place)
    assert not kept_alive, kept_alive[:4]
    if fmt == ro.LOAD:
        assert loads == {"LDS.128": 2 * ro.HELD // 4, "LDS.64": 2 * ro.HELD // 2}, loads
    if fmt == ro.HOLD:
        # each hold is a NANOSLEEP loop between two barriers; every register held across the first of them is first
        # read after the hold's last NANOSLEEP, so each value really sat in its register through the sleep
        for h, b in zip(held, bars[:-1]):
            nxt = bars[bars.index(b) + 1]
            sleeps = [k for k in range(b + 1, nxt) if ops[k] == "NANOSLEEP"]
            assert sleeps, hex(loop[b]["a"])
            early = [r for r in h if _first_touch(loop, b, r) < sleeps[-1]]
            assert not early, (hex(loop[b]["a"]), early[:8])
