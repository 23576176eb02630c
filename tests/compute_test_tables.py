"""Oracle for the tensor-core self-test's input tables (numpy; test infrastructure only): the shared-memory image of a
tile and the per-thread check values, from integer operands a caller chooses.  tests/compute_test_oracle.py specifies the
generator and the arithmetic; this module adds what a launch on caller-built tables needs
(tests/native/compute_test_tables_kernels.cu, ck_run_tables):

    image : A then B, each K-major without swizzle in 8-row x 16-byte core matrices (128 contiguous bytes, row by row);
            per 32-byte K step s the operand's block of rows x 32 bytes starts at s * rows * 32, and in it the core
            matrix of rows 8g..8g+7 and K bytes 16c..16c+15 of the step starts at g * 256 + c * 128 (LBO = 128 along K,
            SBO = 256 per 8 rows); bf16 little-endian
    checks: the fold of each thread's fragment of the exact result (compute_test_oracle.fold / fragments / reference)

Operands outside [lo, hi], scale exponents outside [-30, 30] (0 for FP8 and INT8) and wrong shapes are refused: the
exactness argument covers nothing else."""
import numpy as np

import compute_test_oracle as ct

STEP_BYTES = 32                                                         # K bytes of one wgmma
ELEM_BYTES = {ct.BF16: 2, ct.FP8: 1, ct.INT8: 1}
SMEM = {f: (ct.M + ct.N) * ct.K[f] * ELEM_BYTES[f] for f in ct.FORMATS}  # bytes of one tile's image
STEP_K = {f: STEP_BYTES // ELEM_BYTES[f] for f in ct.FORMATS}           # k per wgmma: 16, 32, 32
STEPS = {f: ct.K[f] // STEP_K[f] for f in ct.FORMATS}                   # wgmmas per result tile: 16, 1, 8


def check_operands(fmt: int, A: np.ndarray, B: np.ndarray, ea: int = 0, eb: int = 0) -> None:
    if np.shape(A) != (ct.M, ct.K[fmt]) or np.shape(B) != (ct.N, ct.K[fmt]):
        raise ValueError("%s operands must be %dx%d and %dx%d, not %s and %s"
                         % (ct.NAMES[fmt], ct.M, ct.K[fmt], ct.N, ct.K[fmt], np.shape(A), np.shape(B)))
    for name, v in (("A", A), ("B", B)):
        if np.min(v) < ct.LO[fmt] or np.max(v) > ct.HI[fmt]:
            raise ValueError("%s operand %s leaves [%d, %d]: %d..%d"
                             % (ct.NAMES[fmt], name, ct.LO[fmt], ct.HI[fmt], np.min(v), np.max(v)))
    lim = ct.SCALE_EXP if fmt == ct.BF16 else 0
    if abs(ea) > lim or abs(eb) > lim:
        raise ValueError("%s scale exponents (%d, %d) leave [-%d, %d]" % (ct.NAMES[fmt], ea, eb, lim, lim))


def reference(fmt: int, A: np.ndarray, B: np.ndarray, ea: int = 0, eb: int = 0) -> np.ndarray:
    """compute_test_oracle.reference of operands that pass check_operands."""
    check_operands(fmt, A, B, ea, eb)
    return ct.reference(fmt, A, B, ea, eb)


def _operand_image(fmt: int, v: np.ndarray, e: int) -> np.ndarray:
    bits = ct.encode(fmt, v, e)
    b = bits.astype("<u2").view(np.uint8) if fmt == ct.BF16 else bits.astype(np.uint8)  # rows x K bytes, row-major
    rows, kb = b.shape
    # byte (8g + r, 32s + 16c + i) -> [s][g][c][r][i]
    return b.reshape(rows // 8, 8, kb // STEP_BYTES, 2, 16).transpose(2, 0, 3, 1, 4).ravel()


def image(fmt: int, A: np.ndarray, B: np.ndarray, ea: int = 0, eb: int = 0) -> np.ndarray:
    """The shared-memory image of one tile (uint8, SMEM[fmt] bytes) from integer operands A (M x K) and B (N x K)."""
    check_operands(fmt, A, B, ea, eb)
    return np.concatenate([_operand_image(fmt, A, ea), _operand_image(fmt, B, eb)])


def tables(fmt: int, tiles):
    """The kernel's inputs for TILES tiles, each (A, B, ea, eb): images (TILES x SMEM[fmt] uint8) and the per-thread
    check values (TILES x THREADS uint32)."""
    if len(tiles) != ct.TILES:
        raise ValueError("a table holds %d tiles, not %d" % (ct.TILES, len(tiles)))
    images = np.stack([image(fmt, *t) for t in tiles])
    checks = np.stack([ct.fold(ct.fragments(reference(fmt, *t))) for t in tiles])
    return images, checks
