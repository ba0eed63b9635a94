"""TEST-ONLY: the wide column sweep (T = 1024, whatshap_b200/csrc/wide_device.h) and its plan, computed on the host by
tests/emul/libwhemul_wide.so, so that five-trio tables can be checked without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np

from whatshap_b200._abi import CProblem, CSolution, FlatSolution, raise_for

EMUL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
PATHS = ("column", "batched", "fused", "wide")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "wide.mk"], check=True, capture_output=True)
        L = C.CDLL(os.path.join(EMUL_DIR, "libwhemul_wide.so"))
        u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
        L.whemul_wide_xform.argtypes = [u32p, C.c_uint64, C.c_uint32, C.c_int, u32p, C.POINTER(C.c_uint16), u32p, u32p]
        L.whemul_wide_xform.restype = None
        L.whemul_wide_solve.argtypes = [C.POINTER(CProblem), C.c_int, C.POINTER(CSolution), u32p, C.c_char_p, C.c_size_t]
        L.whemul_wide_plan.argtypes = [C.POINTER(CProblem), C.c_uint64, C.c_uint64, C.c_int, u64p, u32p, u32p, C.c_uint32, C.c_char_p, C.c_size_t]
        _lib = L
    return _lib


def _p(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


def xform(rows: np.ndarray, rc: int, first: bool = False):
    """(values, argmins) of the transition transform and of transition_min on rows [R, 1024] (uint32)."""
    rows = np.ascontiguousarray(rows, np.uint32)
    R = rows.shape[0]
    vals, args = np.zeros((R, 1024), np.uint32), np.zeros((R, 1024), np.uint16)
    rvals, rargs = np.zeros((R, 1024), np.uint32), np.zeros((R, 1024), np.uint32)
    lib().whemul_wide_xform(_p(rows, C.c_uint32), R, rc, int(first), _p(vals, C.c_uint32), _p(args, C.c_uint16), _p(rvals, C.c_uint32),
                            _p(rargs, C.c_uint32))
    return (vals, args), (rvals, rargs)


def solve(prob, transform: int = -1):
    """(FlatSolution, info) of the emulated wide sweep; info: nowrap, transformed columns, largest chunk split.  Raises as whmec_solve."""
    sol = FlatSolution(prob.n_cols, prob.n_reads, prob.n_ind)
    cp, cs, err = prob.as_c(), sol.as_c(), C.create_string_buffer(512)
    info = np.zeros(3, np.uint32)
    rc = lib().whemul_wide_solve(C.byref(cp), transform, C.byref(cs), _p(info, C.c_uint32), err, len(err))
    raise_for(rc, err.value.decode())
    sol.cost = cs.cost
    return sol, dict(nowrap=bool(info[0]), transformed=int(info[1]), max_chunk_bits=int(info[2]))


def plan(prob, free_bytes=1 << 40, hook=0, segment=0):
    """The column-kernel plan of `prob`: rc, msg, path, bounded, arena / ckpt / bp_words (words) and the column cuts."""
    cap = prob.n_cols + 2
    info, cuts, n_cuts = np.zeros(5, np.uint64), np.zeros(cap, np.uint32), C.c_uint32(0)
    cp, err = prob.as_c(), C.create_string_buffer(512)
    rc = lib().whemul_wide_plan(C.byref(cp), free_bytes, hook, segment, _p(info, C.c_uint64), _p(cuts, C.c_uint32), C.byref(n_cuts), cap,
                                err, len(err))
    return dict(rc=rc, msg=err.value.decode(), path=PATHS[int(info[0])], bounded=bool(info[1]), arena=int(info[2]), ckpt=int(info[3]),
                bp_words=int(info[4]), cuts=cuts[:n_cuts.value].astype(np.int64))
