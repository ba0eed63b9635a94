"""TEST-ONLY: whmec_genotype_batch (groups of tables on one step list each, gl_batch.cpp) executed serially on the host by
tests/emul/libwhemul_gl_batch.so with the kernels' per-cell code (whatshap_b200/csrc/gl_device.h) and host packer: a stand-in for
`_lib.genotype_batch` where there is no GPU.  Steps of different tables run in a seeded random order within a launch, and the
the unread spare behind the backward store and a guard behind the work buffer hold NaN."""
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
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "gl_batch.mk"], check=True, capture_output=True)
        _lib = C.CDLL(os.path.join(EMUL_DIR, "libwhemul_gl_batch.so"))
        _lib.whemul_genotype_batch.argtypes = [C.POINTER(C.POINTER(CProblem)), C.POINTER(C.POINTER(C.c_double)), C.c_uint32, C.c_uint64, C.c_uint64,
                                               C.POINTER(C.c_int), C.c_char_p, C.c_size_t, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        _lib.whemul_genotype_batch.restype = C.c_int
        _lib.whemul_gl_batch_cost.argtypes = [C.POINTER(CProblem)]
        _lib.whemul_gl_batch_cost.restype = C.c_uint64
    return _lib


def genotype_batch(problems, budget_doubles: int = 0, seed: int = 0):
    """(results, info): per table its likelihoods or the exception `_lib.genotype` raises for it, and info = {"groups",
    "launches" (of the groups), "alone" (tables that fit no group: whmec_genotype's path under the same budget), "group_of"
    (per table its group, -1 for none)}.  budget_doubles = 0: no limit."""
    n = len(problems)
    outs = [np.zeros((p.n_ind, p.n_cols, 3), np.float64) for p in problems]
    cps = [p.as_c() for p in problems]
    pp = (C.POINTER(CProblem) * max(n, 1))(*[C.pointer(c) for c in cps])
    lp = (C.POINTER(C.c_double) * max(n, 1))(*[o.ctypes.data_as(C.POINTER(C.c_double)) for o in outs])
    status, group_of, info = (C.c_int * max(n, 1))(), (C.c_uint32 * max(n, 1))(), (C.c_uint32 * 3)()
    errlen = 512
    errs = C.create_string_buffer(errlen * max(n, 1))
    assert lib().whemul_genotype_batch(pp, lp, n, budget_doubles, seed, status, errs, errlen, group_of, info) == 0
    results = []
    for t in range(n):
        try:
            raise_for(int(status[t]), errs.raw[t * errlen:(t + 1) * errlen].split(b"\0", 1)[0].decode())
            results.append(outs[t])
        except Exception as e:  # noqa: BLE001 - in the table's place, as _lib.genotype_batch does
            results.append(e)
    groups = [int(group_of[t]) if group_of[t] != 0xFFFFFFFF else -1 for t in range(n)]
    return results, {"groups": int(info[0]), "launches": int(info[1]), "alone": int(info[2]), "group_of": groups}


def cost(prob) -> int:
    """Doubles `prob` takes in a group: backward tables, projection buffers and inputs (gl_batch_cost)."""
    cp = prob.as_c()
    return int(lib().whemul_gl_batch_cost(C.byref(cp)))
