"""CPU side of the on-demand SFU self-test (b2dp_sfu_test): the host arithmetic in csrc/sfu_test_math.hpp against the
restatement in tests/sfu_test_oracle.py -- the operand tables, the crafted classes, the specials table, the guard at
its edges, the consensus on synthetic dumps and the fold -- then the backends without the test, the daemon's flag, the
struct layouts and the SASS the kernels assemble to.  No GPU needed."""
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
import sfu_test_oracle as so
from test_mig_enumeration import _open as open_nvml_stub, stub  # noqa: F401  (stub is a fixture)
from test_oracle_golden import topo_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
SEEDS = [0, 1, 0xC0FFEE17, 0xFFFFFFFF]
FMT_IDS = [so.NAMES[f] for f in so.FORMATS]
OP_IDS = [o[0] for o in so.OPS]


class MathDriver:
    """tests/native/sfu_test_math_test.cpp, compiled with g++ against csrc/sfu_test_math.hpp."""

    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def ask(self, *words):
        self.p.stdin.write(" ".join(str(w) for w in words) + "\n")
        self.p.stdin.flush()
        return self.p.stdout.readline().split()

    def close(self):
        self.p.stdin.close()
        self.p.wait(timeout=10)


@pytest.fixture(scope="module")
def drv(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("sf") / "sfu_test_math_test")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I", CSRC,
                        os.path.join(ROOT, "tests", "native", "sfu_test_math_test.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    d = MathDriver(exe)
    yield d
    d.close()


# ---- the tables ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", SEEDS)
def test_host_tables_match_the_oracle(drv, seed, fmt):
    """Every operand word of every slot, thread and tile, bit for bit."""
    for t in range(so.TILES):
        got = np.array([int(x) for x in drv.ask("table", seed, fmt, t)], dtype=np.uint64)
        want = so.table(seed, fmt, t).astype(np.uint64).ravel()
        assert got.shape == want.shape and np.array_equal(got, want), (t, np.argwhere(got != want)[:4].ravel())


def test_layout_and_host_cost(drv):
    n, *rest = (int(v) for v in drv.ask("layout"))
    assert n == so.N
    assert rest == [so.SLOTS[f] for f in so.FORMATS] + [so.WORDS[f] for f in so.FORMATS] + \
        [so.RESULTS[f] for f in so.FORMATS]
    ms = min(float(drv.ask("time", s)[0]) for s in (1, 2, 3))
    print("host tables of one b2dp_sfu_test call: %.2f ms" % ms)
    assert ms < 200


def _in_class(op, name, x, b):
    """Does value x (bits b) belong to crafted class `name` of op?  Restated from the class's meaning, not from the
    generator."""
    T = so.OPS[op][2]
    W, M, B = so.BIN[T]
    EMIN, EMAX = 1 - B, B
    ax = np.abs(x)
    fin = np.isfinite(x)
    normal = fin & (ax >= so.min_normal(T))
    pow2 = normal & (np.frexp(ax)[0] == 0.5)
    pow4 = pow2 & (np.frexp(ax)[1] % 2 == 1)      # frexp(4^k) = (0.5, 2k + 1)
    integer = fin & (np.floor(x) == x)
    opn = so.OPS[op][0]
    common = {"sub_in": so.is_subnormal(T, b), "+0": b == 0, "-0": b == np.uint64(1 << (W - 1)),
              "+inf": x == np.inf, "-inf": x == -np.inf, "nan": np.isnan(x)}
    if name in common:
        return common[name]
    if opn == "ex2":
        return {"exact": integer & (x >= -125) & (x <= 127), "edge_hi": (x > 127.99) & (x < 128),
                "edge_lo": (x > -126) & (x < -125.99), "overflow": fin & (x >= 128), "underflow": x <= -130}[name]
    if opn == "lg2":
        return {"exact": pow2 & (x > 0), "edge_lo": (x >= 2.0 ** EMIN) & (x < 2.0 ** (EMIN + 1)),
                "edge_hi": fin & (x >= 2.0 ** EMAX), "near_one": (x >= 1) & (x < 1 + 2.0 ** -14),
                "negative": normal & (x < 0)}[name]
    if opn == "sincos":
        return {"edge": (ax > 12.56) & (ax <= so.TRIG_GUARDED), "large": (ax >= 16) & (ax < 2.0 ** 21),
                "huge": fin & (ax >= 2.0 ** 60), "small": normal & (ax < 2.0 ** -59)}[name]
    if opn in ("tanh", "tanhh"):
        h = T == so.T16
        return {"saturate": fin & (ax >= (8 if h else 16)), "small": normal & (ax < 2.0 ** (-4 if h else -19))}[name]
    if opn == "ex2h":
        return {"exact": integer & (x >= -14) & (x <= 15), "edge_hi": (x > 15.9) & (x < 16),
                "edge_lo": (x > -14) & (x < -13.9), "overflow": (x >= 16) & (x < 24),
                "subnormal": integer & (x >= -23) & (x <= -15), "underflow": integer & (x <= -25)}[name]
    rcp = opn.startswith("rcp")
    return {"exact": pow4 & ((x > 0) | rcp), "edge_lo": (ax >= 2.0 ** EMIN) & (ax < 2.0 ** (EMIN + 1)),
            "edge_hi": ((ax >= 2.0 ** (EMAX - 2)) & (ax < 1.5 * 2.0 ** (EMAX - 2))) if rcp else fin & (x >= 2.0 ** EMAX),
            "underflow": fin & (ax >= 2.0 ** EMAX), "negative": normal & (x < 0)}[name]


@pytest.mark.parametrize("seed", [0, 0xC0FFEE17])
def test_every_crafted_class_is_in_every_thread_of_every_tile(seed):
    for op in range(len(so.OPS)):
        T, nv = so.OPS[op][2], so.values(op)
        names = so.classes(op)
        assert len(names) <= nv - 4, "every op keeps at least four random operands"
        for tile in range(so.TILES):
            b = so.operands(seed, op, tile)
            x = so.value(T, b)
            for c, name in enumerate(names):
                t = np.arange(so.THREADS)
                v = (c + t) % nv
                got = _in_class(op, name, x[t, v], b[t, v])
                assert got.all(), (so.OPS[op][0], name, tile, int(np.argmin(got)))


# ---- the specials table, by hand ---------------------------------------------------------------------------------------
INF, NAN = float("inf"), float("nan")
SUB32, SUB64, SUB16 = 2.0 ** -140, 2.0 ** -1070, 2.0 ** -20
# (op, function, input, a result that passes, a result that must fail)
SPECIALS = [
    ("ex2", so.EX2, INF, INF, 3.4e38), ("ex2", so.EX2, -INF, 0.0, -0.0), ("ex2", so.EX2, NAN, NAN, 0.0),
    ("ex2", so.EX2, 0.0, 1.0, 0.0), ("ex2", so.EX2, -0.0, 1.0, NAN), ("ex2", so.EX2, SUB32, 1.0, 0.0),
    ("ex2", so.EX2, 200.0, INF, 3.4e38), ("ex2", so.EX2, -200.0, 0.0, 2.0 ** -126),
    ("ex2", so.EX2, -135.0, 0.0, 2.0 ** -135),                 # an .ftz unit never returns a subnormal
    ("lg2", so.LG2, 0.0, -INF, INF), ("lg2", so.LG2, -0.0, -INF, NAN), ("lg2", so.LG2, SUB32, -INF, -149.0),
    ("lg2", so.LG2, -1.0, NAN, 0.0), ("lg2", so.LG2, INF, INF, NAN), ("lg2", so.LG2, -INF, NAN, -INF),
    ("sincos", so.SIN, 0.0, 0.0, -0.0), ("sincos", so.SIN, -0.0, -0.0, 0.0), ("sincos", so.SIN, INF, NAN, 0.0),
    ("sincos", so.COS, 0.0, 1.0, NAN), ("sincos", so.COS, -INF, NAN, 1.0), ("sincos", so.SIN, SUB32, 0.0, -0.0),
    ("tanh", so.TANH, INF, 1.0, INF), ("tanh", so.TANH, -INF, -1.0, 1.0), ("tanh", so.TANH, -0.0, -0.0, 0.0),
    ("tanh", so.TANH, 20.0, 1.0, 0.99), ("tanh", so.TANH, -20.0, -1.0, 1.0), ("tanh", so.TANH, NAN, NAN, 1.0),
    ("tanh", so.TANH, -SUB32, -SUB32, SUB32),                  # tanh.approx.f32 has no .ftz: a subnormal stays
    ("rcp", so.RCP, 0.0, INF, -INF), ("rcp", so.RCP, -0.0, -INF, INF), ("rcp", so.RCP, INF, 0.0, -0.0),
    ("rcp", so.RCP, -INF, -0.0, 0.0), ("rcp", so.RCP, -SUB32, -INF, -0.0), ("rcp", so.RCP, 1.5 * 2.0 ** 127, 0.0,
                                                                            2.0 ** -126),
    ("rsqrt", so.RSQ, 0.0, INF, 0.0), ("rsqrt", so.RSQ, -0.0, -INF, INF), ("rsqrt", so.RSQ, INF, 0.0, -0.0),
    ("rsqrt", so.RSQ, -1.0, NAN, 1.0), ("rsqrt", so.RSQ, -INF, NAN, 0.0), ("rsqrt", so.RSQ, SUB32, INF, 2.0 ** 70),
    ("sqrt", so.SQRT, -0.0, -0.0, 0.0), ("sqrt", so.SQRT, -SUB32, -0.0, 0.0), ("sqrt", so.SQRT, INF, INF, NAN),
    ("sqrt", so.SQRT, -1.0, NAN, 1.0), ("sqrt", so.SQRT, SUB32, 0.0, 2.0 ** -70),
    ("rcp64", so.RCP, 0.0, INF, -INF), ("rcp64", so.RCP, -INF, -0.0, 0.0), ("rcp64", so.RCP, SUB64, INF, 1e300),
    ("rcp64", so.RCP, 2.0 ** 1023, 0.0, 2.0 ** -1023), ("rcp64", so.RCP, NAN, NAN, 0.0),
    ("rsqrt64", so.RSQ, -0.0, -INF, INF), ("rsqrt64", so.RSQ, -2.0, NAN, 0.0), ("rsqrt64", so.RSQ, INF, 0.0, -0.0),
    ("ex2h", so.EX2, 16.0, INF, 32768.0), ("ex2h", so.EX2, -INF, 0.0, -0.0), ("ex2h", so.EX2, NAN, NAN, 0.0),
    ("ex2h", so.EX2, -20.0, 2.0 ** -20, -(2.0 ** -20)), ("ex2h", so.EX2, -20.0, 0.0, 2.0 ** -14),
    ("ex2h", so.EX2, SUB16, 1.0, 0.0), ("ex2h", so.EX2, 0.0, 1.0, 1.02),
    ("tanhh", so.TANH, INF, 1.0, INF), ("tanhh", so.TANH, -0.0, -0.0, 0.0), ("tanhh", so.TANH, SUB16, SUB16, -SUB16),
    ("tanhh", so.TANH, 12.0, 1.0, 0.98),
]


@pytest.mark.parametrize("op,fn,x,good,bad", SPECIALS)
def test_specials_table(drv, op, fn, x, good, bad):
    o = so.OP_INDEX[op]
    T, ftz = so.OPS[o][2], so.OPS[o][3]
    xb = so.bits_of(T, x)
    for r, want in ((good, True), (bad, False)):
        rb = so.bits_of(T, r)
        ok, _ = so.guard(fn, T, ftz, np.array([xb], dtype=np.uint64), np.array([rb], dtype=np.uint64))
        assert bool(ok[0]) == want, ("oracle", op, x, r)
        assert drv.ask("guard", fn, T, int(ftz), xb, rb)[0] == str(int(want)), ("host", op, x, r)


# ---- the guard at its edges ----------------------------------------------------------------------------------------------
def _round(T, e, ftz):
    """The correctly rounded bits of exact values e in the type (flushed to a signed zero for .ftz forms)."""
    with np.errstate(all="ignore"):
        if T == so.T64:
            r = e.astype(np.float64)
        elif T == so.T32:
            r = e.astype(np.float32).astype(np.float64)
        else:
            r = e.astype(np.float16).astype(np.float64)
        if ftz:
            r = np.where(np.abs(r) < so.min_normal(T), np.copysign(0.0, r), r)
    return r


def _bits(T, r):
    if T == so.T64:
        return r.astype(np.float64).view(np.uint64)
    if T == so.T32:
        return r.astype(np.float32).view(np.uint32).astype(np.uint64)
    return r.astype(np.float16).view(np.uint16).astype(np.uint64)


def _past(T, fn, e):
    """Results just past the guard: the first value of the type beyond e +- bound (relative or absolute)."""
    B = so.bound(fn, T)
    dt = {so.T64: np.float64, so.T32: np.float32, so.T16: np.float16}[T]
    with np.errstate(all="ignore"):
        A = so.abs_bound(fn, T, e)
        far = e + np.where(e < 0, -1.5, 1.5) * A if fn in so.ABSOLUTE else e * (1 + 1.5 * B)
        r = far.astype(dt)
        for _ in range(4):
            d = np.abs(r.astype(np.float64) - e)
            inside = d <= (A if fn in so.ABSOLUTE else B * np.abs(e))
            r = np.where(inside, np.nextafter(r, (np.sign(far - e) * np.inf).astype(dt)), r)
    return r.astype(np.float64)


@pytest.mark.parametrize("op", range(len(so.OPS)), ids=OP_IDS)
def test_guard_accepts_the_correctly_rounded_value_and_rejects_one_just_past_it(drv, op):
    """For every operand of two tiles: the correctly rounded result passes; where the bound applies (a finite, normal
    exact result; sin and cos for |x| <= 4 pi) the first value past the bound fails.  The host's guard agrees with the
    oracle's on a sample."""
    name, _, T, ftz, _, _, fns, _, _ = so.OPS[op]
    checked = 0
    for tile in (0, 5):
        xb = so.operands(0x6A2D, op, tile).ravel()
        x = so.value(T, xb)
        xf = np.where(so.is_subnormal(T, xb), np.copysign(0.0, x), x) if ftz else x
        for fn in fns:
            e = so.exact(fn, xf)
            good = _bits(T, _round(T, e, ftz))
            ok, _ = so.guard(fn, T, ftz, xb, good)
            assert ok.all(), (name, so.FN_NAMES[fn], hex(int(xb[np.argmin(ok)])))
            ae = np.abs(e)
            B = so.bound(fn, T)
            applies = np.isfinite(e) & (ae >= so.min_normal(T) / (1 - B)) & (ae * (1 + 2 * B) < so.max_finite(T))
            if fn in so.ABSOLUTE:
                applies = np.isfinite(e) & np.isfinite(x)
                if fn in (so.SIN, so.COS):
                    applies &= np.abs(x) <= so.TRIG_GUARDED
            past = _past(T, fn, e)
            applies &= np.isfinite(past)
            bad, _ = so.guard(fn, T, ftz, xb, _bits(T, past))
            assert not bad[applies].any(), (name, so.FN_NAMES[fn], hex(int(xb[applies][np.argmax(bad[applies])])))
            checked += int(applies.sum())
            for i in range(0, len(xb), 23):
                assert drv.ask("guard", fn, T, int(ftz), int(xb[i]), int(good[i]))[0] == "1", (name, hex(int(xb[i])))
                if applies[i]:
                    assert drv.ask("guard", fn, T, int(ftz), int(xb[i]), int(_bits(T, past[i:i + 1])[0]))[0] == "0"
    assert checked > 1000


# ---- consensus on synthetic dumps --------------------------------------------------------------------------------------------
def rounded_words(fmt, seed):
    """[tile][thread][word]: the correctly rounded (flushed for .ftz) result of every operand of the seed's tables --
    a stand-in for a healthy SFU that passes the guard."""
    out = np.zeros((so.TILES, so.THREADS, so.WORDS[fmt]), dtype=np.uint64)
    for tile in range(so.TILES):
        ops = so.thread_words(seed, fmt, tile)
        for op, (_, f, T, ftz, s0, w0, fns, _, _) in enumerate(so.OPS):
            if f != fmt:
                continue
            for k, fn in enumerate(fns):
                x = so.operands(seed, op, tile)
                xf = so.value(T, x)
                if ftz:
                    xf = np.where(so.is_subnormal(T, x), np.copysign(0.0, xf), xf)
                r = _bits(T, _round(T, so.exact(fn, xf), ftz))
                if T == so.T32:
                    out[tile, :, w0 + k * so.N:w0 + (k + 1) * so.N] = r
                elif T == so.T64:
                    out[tile, :, w0:w0 + 2 * so.N:2] = r & np.uint64(so.M32)
                    out[tile, :, w0 + 1:w0 + 2 * so.N:2] = r >> np.uint64(32)
                else:
                    out[tile, :, w0:w0 + so.N] = r[:, 0::2] | (r[:, 1::2] << np.uint64(16))
        assert so.guard_words(fmt, ops, out[tile].astype(np.uint32))[0] == 0
    return out.astype(np.uint32)


REC = np.dtype([("smid", "<u4"), ("nsmid", "<u4"), ("rounds", "<u8"), ("comparisons", "<u8"), ("mismatches", "<u8"),
                ("first_bad_tile", "<i4"), ("first_bad_rep", "<i4"), ("seq", "<u8")])
SMIDS = [4, 9, 17, 30, 131]


class Consensus:
    def __init__(self, drv, tmp, fmt, seed=0x5A5A):
        self.drv, self.dir, self.fmt = drv, str(tmp), fmt
        self.words = rounded_words(fmt, seed)
        so.tables(seed, fmt).tofile(os.path.join(self.dir, "table.bin"))

    def run(self, dumps, smids=SMIDS, seqs=None):
        n = len(dumps)
        recs = np.zeros(n, dtype=REC)
        recs["smid"], recs["nsmid"], recs["rounds"] = smids[:n], 132, 1
        recs["comparisons"], recs["seq"] = so.TILES * so.REPS, 3 if seqs is None else seqs
        np.ascontiguousarray(dumps, dtype=np.uint32).tofile(os.path.join(self.dir, "dumps.bin"))
        recs.tofile(os.path.join(self.dir, "recs.bin"))
        v = [int(x) for x in self.drv.ask("consensus", self.fmt, n, 3, self.dir)]
        keys = ["arrived", "sm_ids", "no_consensus", "out_of_bound", "dissents", "flags", "clean", "first_bad_sm",
                "first_bad_tile"]
        out = dict(zip(keys, v))
        out["mask"] = v[9:13]
        out["check"] = np.fromfile(os.path.join(self.dir, "check.bin"), dtype=np.uint32).reshape(so.TILES, so.THREADS)
        return out

    def dumps(self, n=len(SMIDS)):
        return np.repeat(self.words[None], n, axis=0)


def _mask(*sms):
    m = [0, 0, 0, 0]
    for s in sms:
        m[s // 64] |= 1 << (s % 64)
    return m


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_consensus_unanimous_is_clean_and_checks_fold_the_words(drv, tmp_path, fmt):
    c = Consensus(drv, tmp_path, fmt)
    r = c.run(c.dumps())
    assert (r["arrived"], r["sm_ids"], r["no_consensus"], r["out_of_bound"], r["dissents"], r["flags"], r["clean"]) == \
        (5, 5, 0, 0, 0, 0, 1), r
    assert (r["first_bad_sm"], r["first_bad_tile"], r["mask"]) == (-1, -1, [0, 0, 0, 0])
    assert np.array_equal(r["check"], so.fold(c.words))


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_consensus_names_the_one_dissenting_sm_at_every_position(drv, tmp_path, fmt):
    """One CTA differs in one word: every word position with bit 0 and bit 31, and every thread and tile along the way."""
    c = Consensus(drv, tmp_path, fmt)
    W = so.WORDS[fmt]
    cases = [(j, (j * 37 + b) % so.THREADS, (j + b // 31) % so.TILES, b) for j in range(W) for b in (0, 31)]
    cases += [(t % W, t, t % so.TILES, 31 * (t % 2)) for t in range(so.THREADS)]
    seen = set()
    for k, (j, t, tile, b) in enumerate(cases):
        cta = k % len(SMIDS)
        d = c.dumps()
        d[cta, tile, t, j] ^= np.uint32(1 << b)
        r = c.run(d)
        assert (r["dissents"], r["no_consensus"], r["out_of_bound"], r["clean"]) == (1, 0, 0, 0), (j, t, tile, b, r)
        assert (r["first_bad_sm"], r["first_bad_tile"], r["mask"]) == (SMIDS[cta], tile, _mask(SMIDS[cta])), (j, t, b)
        assert np.array_equal(r["check"], so.fold(c.words))   # the majority, not the dissenter
        seen.add((j, b))
    assert len({t for _, t, _, _ in cases}) == so.THREADS and len({x for x, _, _, _ in cases}) == W


def test_consensus_names_two_bad_sms_and_counts_each_tile(drv, tmp_path):
    c = Consensus(drv, tmp_path, so.F32)
    d = c.dumps()
    d[3, 6, 100, 70] ^= np.uint32(4)      # SM 30, tile 6
    d[1, 2, 5, 1] ^= np.uint32(1)         # SM 9, tiles 2 and 4
    d[1, 4, 9, 9] ^= np.uint32(1 << 31)
    r = c.run(d)
    assert (r["dissents"], r["first_bad_sm"], r["first_bad_tile"], r["mask"]) == (3, 9, 2, _mask(9, 30)), r
    assert r["clean"] == 0 and r["flags"] == 0


def test_consensus_without_a_strict_majority(drv, tmp_path):
    c = Consensus(drv, tmp_path, so.ROOT)
    d = np.repeat(c.words[None], 4, axis=0)
    d[2:, 3, 64, 100] ^= np.uint32(1 << 12)     # an exact half split of one word
    r = c.run(d, smids=[1, 2, 3, 4])
    assert (r["no_consensus"], r["flags"] & 0x4, r["dissents"], r["clean"]) == (1, 0x4, 0, 0), r


@pytest.mark.parametrize("fmt,word,change", [(so.F32, 3, "double"), (so.F32, 40, "negate"), (so.ROOT, 49, "double"),
                                             (so.F16, 20, "double")])
def test_consensus_outside_the_guard(drv, tmp_path, fmt, word, change):
    """Every SM agrees on a wrong value: no dissent, but OUT_OF_BOUND."""
    c = Consensus(drv, tmp_path, fmt)
    d = c.dumps()
    th = [t for t in range(so.THREADS) if (word % so.N - t) % so.N >= 12][0]   # a random operand
    w = d[:, 0, th, word]
    if fmt == so.F16:
        w = w ^ np.uint32(0x0400 if change == "double" else 0x8000)          # the low half's exponent + 1
    else:
        w = w + np.uint32(1 << 23) if fmt == so.F32 and change == "double" else w ^ np.uint32(1 << 31) \
            if change == "negate" else w + np.uint32(1 << 20)                 # f32 x 2; sign; f64 high word: x 2
    d[:, 0, th, word] = w
    r = c.run(d)
    assert (r["dissents"], r["no_consensus"], r["flags"], r["clean"]) == (0, 0, 0x8, 0), r
    assert r["out_of_bound"] >= 1


def test_consensus_with_a_missing_record(drv, tmp_path):
    c = Consensus(drv, tmp_path, so.F16)
    r = c.run(c.dumps(), seqs=[3, 3, 0, 3, 3])
    assert (r["arrived"], r["sm_ids"], r["dissents"], r["clean"]) == (4, 4, 0, 0), r


# ---- the fold ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_every_single_bit_flip_of_every_result_word_changes_the_fold(drv, fmt):
    w = np.random.default_rng(fmt).integers(0, 1 << 32, so.WORDS[fmt], dtype=np.uint64)
    base = int(so.fold(w))
    assert int(drv.ask("fold", len(w), *w.tolist())[0]) == base
    flips = w[None, None, :] ^ np.zeros((len(w), 32, 1), dtype=np.uint64)
    j = np.arange(len(w))
    flips[j, :, j] ^= (np.uint64(1) << np.arange(32, dtype=np.uint64))[None, :]
    assert (so.fold(flips) != base).all()


# ---- ABI, backends, daemon, SASS --------------------------------------------------------------------------------------------
def test_constants_and_struct_layouts(pkg):
    N = pkg._native
    assert (N.SF_F32, N.SF_ROOT, N.SF_F16) == (0, 1, 2)
    assert (N.CT_SKIPPED_BUSY, N.CT_PARTIAL_COVERAGE, N.CT_NO_CONSENSUS, N.CT_OUT_OF_BOUND) == (1, 2, 4, 8)
    assert C.sizeof(N.ComputeTestOpts) == 24 and C.sizeof(N.ComputeTestResult) == 128
    assert N.ComputeTestResult.tflops.offset == 112 and N.ComputeTestResult.bad_sm_mask.offset == 32
    assert REC.itemsize == 48
    hdr = open(os.path.join(ROOT, "include", "b200dp.h")).read()
    for name, v in (("B2DP_SF_F32", 0), ("B2DP_SF_ROOT", 1), ("B2DP_SF_F16", 2), ("B2DP_CT_NO_CONSENSUS", "0x4u"),
                    ("B2DP_CT_OUT_OF_BOUND", "0x8u")):
        assert re.search(r"#define %s %s\b" % (name, v), hdr), name


def test_backends_without_an_sfu_test(pkg, kfd, tmp_path, monkeypatch, stub):  # noqa: F811
    N = pkg._native
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    for uri in ("kfd:" + root, "synthetic:2"):
        with pkg.Context(uri) as ctx:
            with pytest.raises(N.B2dpError) as ei:
                ctx.sfu_test(duration_ms=10)
            assert ei.value.code == N.E_UNSUPPORTED
    with open_nvml_stub(pkg, monkeypatch, stub, tmp_path, 2, 0) as ctx:      # cuda:probe=off (NVML only)
        with pytest.raises(N.B2dpError) as ei:
            ctx.sfu_test(duration_ms=10)
        assert ei.value.code == N.E_UNSUPPORTED and "in-process only" in str(ei.value)
        assert "SFU self-test" in str(ei.value)


def test_daemon_sfu_test_flag_on_a_backend_without_one(pkg, kfd, tmp_path, short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("b200dp_plugind not built")
    root = fake_sysfs.build(str(tmp_path / "r"), topo_dir(kfd, "mi210"))
    proc = subprocess.Popen([exe, "-backend=kfd:" + root, "-plugin_dir", short_dir, "-start_retry_wait=0.05",
                             "-sfu_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)
    proc.send_signal(signal.SIGINT)
    _, err = proc.communicate(timeout=10)
    assert proc.returncode == 0, err[-2000:]
    assert "sfu test at start not run: not supported by this backend" in err, err[-2000:]
    assert "Failed to start plugin gpu: Register:" in err


MUFU = {0: {"EX2": 16, "LG2": 16, "SIN": 16, "COS": 16, "TANH": 16},
        1: {"RCP": 16, "RSQ": 16, "SQRT": 16, "RCP64H": 16, "RSQ64H": 16},
        2: {"EX2.F16": 32, "TANH.F16": 32}}


@pytest.mark.parametrize("dump", [0, 1], ids=["product", "reference"])
def test_sass_has_the_planned_mufu_ops_per_repetition(dump):
    """Both instantiations of every format: inside the repetition loop, exactly the planned MUFU ops -- 16 per f32 /
    f64 op, 32 per f16x2 op -- and no other MUFU variant; sin and cos share one FMUL.RZ argument scaling per operand.
    The repetition loop is found by its own back-edge: the first backward branch after the first BAR.RED.OR (the
    repetition's __syncthreads_or compare).  The tile and round loops also enclose every MUFU, so "some backward branch
    around them" would still hold if ptxas hoisted the ops out of the repetition loop and repeated only the fold."""
    lib = os.path.join(ROOT, "tests", "native", "libsfu_test_kernels_test.so")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib) or not os.path.exists(tool):
        pytest.skip("needs the built harness and cuobjdump")
    sass = subprocess.run([tool, "-sass", lib], capture_output=True, text=True).stdout
    funcs = {}
    for part in re.split(r"\n\s+Function : ", sass)[1:]:
        funcs[part.split("\n")[0].strip()] = part
    for fmt, want in MUFU.items():
        (body,) = [b for name, b in funcs.items() if "sfu_selftestILi%dELb%dE" % (fmt, dump) in name]
        ins = [(int(a, 16), i) for a, i in re.findall(r"/\*([0-9a-f]{4})\*/\s+([^;]*);", body)]
        mufu = [(a, re.search(r"MUFU\.(\S+)", i).group(1)) for a, i in ins if "MUFU." in i]
        got = {}
        for _, op in mufu:
            got[op] = got.get(op, 0) + 1
        assert got == want, (fmt, got)
        fmul_rz = [a for a, i in ins if "FMUL.RZ" in i]
        assert len(fmul_rz) == (16 if fmt == 0 else 0)
        bar = min(a for a, i in ins if "BAR.RED.OR" in i)
        back = [(a, int(m.group(1), 16)) for a, i in ins for m in [re.search(r"BRA (?:`\()?0x([0-9a-f]+)", i)]
                if m and int(m.group(1), 16) < a and a > bar]
        src, tgt = min(back)
        outside = [hex(a) for a in [a for a, _ in mufu] + fmul_rz if not tgt <= a < src]
        assert not outside, (fmt, "repetition loop 0x%x..0x%x" % (tgt, src), outside[:8], len(outside))
        # no range-scaling code around the MUFU ops (what ex2 / lg2 without .ftz would add): no float compare at all
        assert not any(re.match(r"(@!?U?P\w+\s+)?(FSETP|FSEL)", i) for _, i in ins), fmt
