"""ctypes binding of tests/native/libprobe_kernels_test.so (built by __graft_entry__.build()): direct launches of the
hbm_probe.cuh kernels on caller-owned device buffers (torch allocations), for tests/test_gpu_kernels.py.

The variant table is plain host data, so it can be read on a machine without a GPU."""
import ctypes as C
import os

from probe_cases import Variant

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "native", "libprobe_kernels_test.so")

# pk_run / pk_fill refusals (nothing launched) and failures
E_CUDA, E_VARIANT, E_SIZE, E_ALIGN, E_GRID, E_SEQ = 1, -1, -2, -3, -4, -5

U64 = C.c_uint64


class ProbeOut(C.Structure):
    _fields_ = [("checksum", U64), ("mismatches", U64), ("first_bad", U64), ("t_start_ns", U64), ("t_end_ns", U64),
                ("seq", U64)]


class ProbeCtl(C.Structure):
    _fields_ = [("checksum", U64), ("mismatches", U64), ("first_bad", U64), ("t_start_ns", U64), ("done", C.c_uint32),
                ("pad", C.c_uint32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError("%s is missing: run __graft_entry__.build() first" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.pk_num_variants.restype = C.c_int
        L.pk_variant.argtypes = [C.c_int, C.POINTER(C.c_char_p)] + [C.POINTER(C.c_int)] * 4
        L.pk_open.restype = C.c_void_p
        L.pk_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.pk_close.argtypes = [C.c_void_p]
        L.pk_error.restype = C.c_char_p
        L.pk_error.argtypes = [C.c_void_p]
        L.pk_sms.argtypes = [C.c_void_p]
        L.pk_run.argtypes = [C.c_void_p, C.c_int, U64, U64, U64, U64, U64, C.c_uint32, C.c_uint32, C.c_int, U64,
                             C.POINTER(ProbeOut)]
        L.pk_read_ctl.argtypes = [C.c_void_p, C.POINTER(ProbeCtl)]
        L.pk_fill.argtypes = [C.c_void_p, U64, U64, U64, C.c_uint32]
        L.pk_occupancy.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        _lib = L
    return _lib


def variants():
    """The harness's variant table, in its order (the index is what run() takes)."""
    L = lib()
    out = []
    for v in range(L.pk_num_variants()):
        name = C.c_char_p()
        vals = [C.c_int() for _ in range(4)]
        assert L.pk_variant(v, C.byref(name), *[C.byref(x) for x in vals]) == 0
        out.append(Variant(name.value.decode(), *[x.value for x in vals]))
    return out


def _span(t):
    """(device address, bytes) of a torch tensor."""
    return t.data_ptr(), t.numel() * t.element_size()


class Harness:
    def __init__(self, device=0):
        err = C.create_string_buffer(512)
        self.h = lib().pk_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("pk_open: " + err.value.decode())
        self.sms = lib().pk_sms(self.h)

    def close(self):
        if self.h:
            lib().pk_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == E_CUDA:
            raise RuntimeError("%s: %s" % (what, lib().pk_error(self.h).decode()))
        if rc != 0:
            raise RuntimeError("%s refused: code %d" % (what, rc))

    def run_rc(self, variant, src, dst, n_vec, seed, delta, grid, seq):
        """One launch over n_vec vectors of src (torch tensor) into dst -> (return code, ProbeOut)."""
        out = ProbeOut()
        (sp, sb), (dp, db) = _span(src), _span(dst)
        rc = lib().pk_run(self.h, variant, sp, sb, dp, db, n_vec, seed, delta, grid, seq, C.byref(out))
        return rc, out

    def run(self, variant, src, dst, n_vec, seed, delta, grid, seq):
        rc, out = self.run_rc(variant, src, dst, n_vec, seed, delta, grid, seq)
        self._check(rc, "pk_run")
        return out

    def read_ctl(self):
        c = ProbeCtl()
        self._check(lib().pk_read_ctl(self.h, C.byref(c)), "pk_read_ctl")
        return c

    def fill(self, dst, n_vec, seed):
        dp, db = _span(dst)
        self._check(lib().pk_fill(self.h, dp, db, n_vec, seed), "pk_fill")

    def occupancy(self, variant):
        n = C.c_int()
        self._check(lib().pk_occupancy(self.h, variant, C.byref(n)), "pk_occupancy")
        return n.value
