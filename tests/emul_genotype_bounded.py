"""TEST-ONLY: whmec_genotype under a memory budget (gl_plan: groups of tables, and tables in memory-bounded mode) executed
serially on the host by tests/emul/libwhemul_gl_bounded.so, with the kernels' per-cell code (whatshap_b200/csrc/gl_device.h)
and host packer (gl_pack.cpp) — a stand-in for `whmec_genotype` where there is no GPU.  The resident path is emul_genotype."""
import ctypes as C
import os
import subprocess

import numpy as np

from whatshap_b200._abi import CProblem, raise_for

EMUL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "gl_bounded.mk"], check=True, capture_output=True)
        _lib = C.CDLL(os.path.join(EMUL_DIR, "libwhemul_gl_bounded.so"))
        _lib.whemul_genotype_bounded.argtypes = [C.POINTER(CProblem), C.POINTER(C.c_double), C.c_uint64, C.POINTER(C.c_uint32), C.c_char_p, C.c_size_t]
        _lib.whemul_genotype_bounded_plan.argtypes = [C.POINTER(CProblem), C.c_uint64, C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_uint32),
                                                      C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    return _lib


def genotype_bounded(prob, budget_doubles: int):
    """What whmec_genotype runs when `budget_doubles` doubles hold its backward tables, checkpoints and projection buffers: groups
    of tables as emul_genotype.genotype forms them, and a table that alone exceeds the budget in memory-bounded mode (segments
    of columns sharing one arena, swept backward again from checkpoints).  The second return value reports the most segments
    any table was cut into."""
    out = np.zeros((prob.n_ind, prob.n_cols, 3), np.float64)
    cp, err = prob.as_c(), C.create_string_buffer(512)
    segments = C.c_uint32(0)
    raise_for(lib().whemul_genotype_bounded(C.byref(cp), out.ctypes.data_as(C.POINTER(C.c_double)), budget_doubles, C.byref(segments), err, len(err)),
              err.value.decode())
    return out, {"segments": int(segments.value)}


def bounded_plan(prob, budget_doubles: int):
    """The cuts of the table with the most segments under `budget_doubles` (empty when no table is cut), its arena, checkpoint and
    projection-buffer doubles, and every column's backward-table doubles (0 for a table's last column)."""
    cp, err = prob.as_c(), C.create_string_buffer(512)
    cuts = np.zeros(prob.n_cols + 1, np.uint32)
    sizes = np.zeros(3, np.uint64)
    own = np.zeros(max(prob.n_cols, 1), np.uint64)
    n_cuts = C.c_uint32(0)
    raise_for(lib().whemul_genotype_bounded_plan(C.byref(cp), budget_doubles, cuts.ctypes.data_as(C.POINTER(C.c_uint32)), len(cuts), C.byref(n_cuts),
                                                 sizes.ctypes.data_as(C.POINTER(C.c_uint64)), own.ctypes.data_as(C.POINTER(C.c_uint64)), err, len(err)),
              err.value.decode())
    return {"cuts": cuts[:n_cuts.value].astype(np.int64), "arena": int(sizes[0]), "ckpt": int(sizes[1]), "pool": int(sizes[2]),
            "own": own[:prob.n_cols].astype(np.int64)}
