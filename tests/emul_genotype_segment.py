"""TEST-ONLY stand-in for `whatshap_b200._lib.GenotypeSegment`: the same operations executed serially on the host by
tests/emul/libwhemul_gl_segment.so, with the kernels' per-cell code (whatshap_b200/csrc/gl_device.h: gl_transfer_cell and the
backward / forward cells) and the host packer and plans (gl_pack.cpp).  Lets the multi-GPU genotyping scheme of
`whatshap_b200.multigpu` be checked where there is no GPU; never part of the product."""
import ctypes as C
import os
import subprocess

import numpy as np

from whatshap_b200._abi import CProblem, raise_for

EMUL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
_F64P = C.POINTER(C.c_double)
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "gl_segment.mk"], check=True, capture_output=True)
        L = C.CDLL(os.path.join(EMUL_DIR, "libwhemul_gl_segment.so"))
        L.whemul_gl_segment_create.argtypes = [C.POINTER(CProblem), C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]
        L.whemul_gl_segment_transfer.argtypes = [C.c_void_p, _F64P, C.POINTER(C.c_uint32)]
        L.whemul_gl_segment_run.argtypes = [C.c_void_p, _F64P, _F64P, _F64P, C.c_uint64, C.POINTER(C.c_uint32), C.c_char_p, C.c_size_t]
        L.whemul_gl_segment_destroy.argtypes = [C.c_void_p]
        L.whemul_gl_segment_destroy.restype = None
        _lib = L
    return _lib


class Segment:
    """`budget_doubles`: what `run` may use for backward tables, checkpoints and projection buffers (gl_plan); a smaller budget
    than the segment's backward tables takes the memory-bounded mode, as WHMEC_GENOTYPE_ARENA_BUDGET does on the device."""

    def __init__(self, prob, continues, continued, budget_doubles: int = 1 << 62):
        self.prob, self.T, self.budget, self._h = prob, 4 ** prob.n_trios, budget_doubles, C.c_void_p()
        self.stats = {}
        cp, err = prob.as_c(), C.create_string_buffer(512)
        raise_for(lib().whemul_gl_segment_create(C.byref(cp), int(bool(continues)), int(bool(continued)), C.byref(self._h), err, len(err)),
                  err.value.decode())

    @staticmethod
    def _ptr(a):
        return None if a is None else a.ctypes.data_as(_F64P)

    def transfer(self):
        m, batches = np.zeros((self.T, self.T), np.float64), C.c_uint32(0)
        lib().whemul_gl_segment_transfer(self._h, self._ptr(m), C.byref(batches))
        self.stats = {"batches": int(batches.value)}
        return m

    def run(self, alpha=None, beta=None):
        out, err, segments = np.zeros((self.prob.n_ind, self.prob.n_cols, 3), np.float64), C.create_string_buffer(512), C.c_uint32(0)
        a = None if alpha is None else np.ascontiguousarray(alpha, np.float64)
        b = None if beta is None else np.ascontiguousarray(beta, np.float64)
        raise_for(lib().whemul_gl_segment_run(self._h, self._ptr(a), self._ptr(b), self._ptr(out), self.budget, C.byref(segments), err, len(err)),
                  err.value.decode())
        self.stats = {"segments": int(segments.value)}
        return out

    def close(self):
        if self._h:
            lib().whemul_gl_segment_destroy(self._h)
            self._h = C.c_void_p()
