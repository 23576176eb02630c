"""ctypes binding of tests/native/libprobe_queue_test.so (built by __graft_entry__.build()): direct launches of
hbm_probe_queue, the health probe's kernel, on caller-owned device buffers (torch allocations), for
tests/test_gpu_probe_queue.py.

The kernel's shape is plain host data, so it can be read on a machine without a GPU."""
import ctypes as C
import os

from probe_cases import Variant
from probe_kernels import ProbeCtl, ProbeOut

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "native", "libprobe_queue_test.so")

# pq_run refusals (nothing launched) and failures
E_CUDA, E_SIZE, E_ALIGN, E_GRID, E_SEQ = 1, -2, -3, -4, -5

# hbm_probe_queue<kQueueCW=4, kQueueTileVec=512, kQueueStages=6>: 8 KiB tiles, a loader, a storer and 4 verifier warps
QUEUE = Variant("queue_4_512_6", 512, 6, 192, 2)

U64 = C.c_uint64

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError("%s is missing: run __graft_entry__.build() first" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.pq_variant.argtypes = [C.POINTER(C.c_char_p)] + [C.POINTER(C.c_int)] * 4
        L.pq_variant.restype = None
        L.pq_open.restype = C.c_void_p
        L.pq_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.pq_close.argtypes = [C.c_void_p]
        L.pq_error.restype = C.c_char_p
        L.pq_error.argtypes = [C.c_void_p]
        L.pq_sms.argtypes = [C.c_void_p]
        L.pq_run.argtypes = [C.c_void_p, U64, U64, U64, U64, U64, C.c_uint32, C.c_uint32, C.c_int, U64,
                             C.POINTER(ProbeOut)]
        L.pq_read_ctl.argtypes = [C.c_void_p, C.POINTER(ProbeCtl)]
        L.pq_occupancy.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
        _lib = L
    return _lib


def variant():
    """The kernel's shape as the harness reports it."""
    name = C.c_char_p()
    vals = [C.c_int() for _ in range(4)]
    lib().pq_variant(C.byref(name), *[C.byref(x) for x in vals])
    return Variant(name.value.decode(), *[x.value for x in vals])


def _span(t):
    """(device address, bytes) of a torch tensor."""
    return t.data_ptr(), t.numel() * t.element_size()


class Harness:
    def __init__(self, device=0):
        err = C.create_string_buffer(512)
        self.h = lib().pq_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("pq_open: " + err.value.decode())
        self.sms = lib().pq_sms(self.h)

    def close(self):
        if self.h:
            lib().pq_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == E_CUDA:
            raise RuntimeError("%s: %s" % (what, lib().pq_error(self.h).decode()))
        if rc != 0:
            raise RuntimeError("%s refused: code %d" % (what, rc))

    def run_rc(self, src, dst, n_vec, seed, delta, grid, seq):
        """One launch over n_vec vectors of src (torch tensor) into dst -> (return code, ProbeOut)."""
        out = ProbeOut()
        (sp, sb), (dp, db) = _span(src), _span(dst)
        rc = lib().pq_run(self.h, sp, sb, dp, db, n_vec, seed, delta, grid, seq, C.byref(out))
        return rc, out

    def run(self, src, dst, n_vec, seed, delta, grid, seq):
        rc, out = self.run_rc(src, dst, n_vec, seed, delta, grid, seq)
        self._check(rc, "pq_run")
        return out

    def read_ctl(self):
        c = ProbeCtl()
        self._check(lib().pq_read_ctl(self.h, C.byref(c)), "pq_read_ctl")
        return c

    def occupancy(self):
        n = C.c_int()
        self._check(lib().pq_occupancy(self.h, C.byref(n)), "pq_occupancy")
        return n.value
