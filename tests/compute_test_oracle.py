"""Oracle for the on-demand tensor-core self-test (numpy; test infrastructure only).

The specification of the arithmetic the CUDA kernel (k8s-device-plugin_b200/csrc/tc_selftest.cuh) and its host side
(csrc/compute_test_math.hpp) must reproduce bit for bit:

    mix(x)          : x ^= x >> 16; x *= 0x7FEB352D; x ^= x >> 15; x *= 0x846CA68B; x ^= x >> 16      (uint32)
    stream key      : key = mix(seed ^ uint32((((fmt * 16 + tile) * 2 + op) + 1) * 0x9E3779B9))   op 0 = A, 1 = B
    hash(i)         : mix(key + mix(i))
    value           : lo + (hash(r * K + k) * (hi - lo + 1) >> 32), except A row 0 and B rows n < 8 at k != n: lo
    scale (BF16)    : a = -30 + (hash(0xFFFFFFFF) * 61 >> 32) per operand; FP8 and INT8: 0
    encodings       : bf16 = top 16 bits of the FP32 value v * 2^a; e4m3 = sign | (e + 7) << 3 | mantissa; s8
    result          : D[m][n] = sum_k A[m][k] B[n][k] (exact) * 2^(a + b) as FP32 bits (+0 for 0), or s32 bits
    fragment        : register j of thread t holds D[16 (t / 32) + (t % 32) / 4 + 8 ((j / 2) % 2)][8 (j / 4) + 2 (t % 4) + j % 2]
    check value     : sum_j (2j + 1) * x_j  mod 2^32 over the thread's 64 registers
    verdict         : launches ok; per format at least one record; every record arrived (seq), did >= 1 round, compared
                      rounds * TILES * REPS results and has no mismatch
"""
import numpy as np

M, N, THREADS, ACC = 64, 128, 128, 64
TILES, REPS = 8, 16
BF16, FP8, INT8 = 0, 1, 2
FORMATS = (BF16, FP8, INT8)
NAMES = {BF16: "bf16", FP8: "fp8", INT8: "int8"}
K = {BF16: 256, FP8: 32, INT8: 256}
LO = {BF16: -255, FP8: -15, INT8: -128}
HI = {BF16: 255, FP8: 15, INT8: 127}
SCALE_EXP = 30
M32 = 0xFFFFFFFF


def mix(x):
    x = np.asarray(x, dtype=np.uint64) & M32
    x = x ^ (x >> np.uint64(16))
    x = (x * np.uint64(0x7FEB352D)) & np.uint64(M32)
    x = x ^ (x >> np.uint64(15))
    x = (x * np.uint64(0x846CA68B)) & np.uint64(M32)
    x = x ^ (x >> np.uint64(16))
    return x


def stream_key(seed: int, fmt: int, tile: int, op: int) -> int:
    return int(mix(seed ^ (((((fmt * 16 + tile) * 2 + op) + 1) * 0x9E3779B9) & M32)))


def hash_(key: int, i):
    return mix((np.uint64(key) + mix(i)) & np.uint64(M32))


def uniform(h, lo: int, hi: int):
    return lo + ((np.asarray(h, dtype=np.uint64) * np.uint64(hi - lo + 1)) >> np.uint64(32)).astype(np.int64)


def scale_exp(seed: int, fmt: int, tile: int, op: int) -> int:
    if fmt != BF16:
        return 0
    return int(uniform(hash_(stream_key(seed, fmt, tile, op), M32), -SCALE_EXP, SCALE_EXP))


def operand(seed: int, fmt: int, tile: int, op: int) -> np.ndarray:
    """Integer operand values, rows x K (rows = 64 for A, 128 for B)."""
    rows, k = (N if op else M), K[fmt]
    key = stream_key(seed, fmt, tile, op)
    v = uniform(hash_(key, np.arange(rows * k, dtype=np.uint64)), LO[fmt], HI[fmt]).reshape(rows, k)
    if op == 0:
        v[0, :] = LO[fmt]
    else:
        for r in range(8):
            keep = v[r, r]
            v[r, :] = LO[fmt]
            v[r, r] = keep
    return v


def _e4m3(a: int) -> int:
    if a == 0:
        return 0
    s, a = (0x80, -a) if a < 0 else (0, a)
    e = a.bit_length() - 1
    return s | (e + 7) << 3 | ((a << 3) >> e) & 7


def encode(fmt: int, v: np.ndarray, e: int = 0) -> np.ndarray:
    """Operand bits: bf16 (uint16 values), e4m3 or s8 (uint8 values), as uint32."""
    v = np.asarray(v, dtype=np.int64)
    if fmt == BF16:
        f = np.ldexp(v.astype(np.float64), e).astype(np.float32)
        return (f.view(np.uint32) >> np.uint32(16)).astype(np.uint32)
    if fmt == INT8:
        return v.astype(np.int8).view(np.uint8).astype(np.uint32)
    table = {x: _e4m3(x) for x in range(LO[FP8], HI[FP8] + 1)}
    return np.vectorize(lambda x: table[int(x)], otypes=[np.uint32])(v)


def decode_e4m3(bits: int) -> float:
    s = -1.0 if bits & 0x80 else 1.0
    e, m = (bits >> 3) & 0xF, bits & 7
    return s * (m / 8.0) * 2.0 ** -6 if e == 0 else s * (1 + m / 8.0) * 2.0 ** (e - 7)


def reference(fmt: int, A: np.ndarray, B: np.ndarray, ea: int = 0, eb: int = 0) -> np.ndarray:
    """The exact M x N result as uint32 bits (FP32, or s32 for INT8)."""
    s = A.astype(np.int64) @ B.astype(np.int64).T
    if fmt == INT8:
        return s.astype(np.int32).view(np.uint32)
    return np.ldexp(s.astype(np.float64), ea + eb).astype(np.float32).view(np.uint32)


def frag_index():
    """(rows, cols), each THREADS x ACC: where register j of thread t sits in the M x N result."""
    t = np.arange(THREADS)[:, None]
    j = np.arange(ACC)[None, :]
    rows = 16 * (t // 32) + (t % 32) // 4 + 8 * ((j // 2) % 2)
    cols = 8 * (j // 4) + 2 * (t % 4) + j % 2
    return rows, cols


def fragments(d: np.ndarray) -> np.ndarray:
    rows, cols = frag_index()
    return d[rows, cols]


WEIGHTS = (2 * np.arange(ACC, dtype=np.uint64) + 1)


def fold(x: np.ndarray) -> np.ndarray:
    """sum_j (2j + 1) x_j mod 2^32 over the last axis (ACC registers)."""
    return ((np.asarray(x, dtype=np.uint64) * WEIGHTS).sum(axis=-1) & np.uint64(M32)).astype(np.uint32)


def tile(seed: int, fmt: int, t: int):
    """Everything about one tile: (A, B, ea, eb, D bits, per-thread check values)."""
    A, B = operand(seed, fmt, t, 0), operand(seed, fmt, t, 1)
    ea, eb = scale_exp(seed, fmt, t, 0), scale_exp(seed, fmt, t, 1)
    d = reference(fmt, A, B, ea, eb)
    return A, B, ea, eb, d, fold(fragments(d))


def record_complete(seq: int, rounds: int, comparisons: int, want_seq: int) -> bool:
    return seq == want_seq and rounds >= 1 and comparisons == rounds * TILES * REPS


def healthy(launch_ok: bool, records, seqs) -> bool:
    """records[f]: list of (seq, rounds, comparisons, mismatches) per CTA of format f; seqs[f]: its launch's seq."""
    if not launch_ok:
        return False
    for f in FORMATS:
        if not records[f]:
            return False
        for seq, rounds, comparisons, mismatches in records[f]:
            if not record_complete(seq, rounds, comparisons, seqs[f]) or mismatches:
                return False
    return True
