"""TEST-ONLY: whmec_heuristic_batch (host plan heuristic_batch.cpp, sweep of whatshap_b200/csrc/heuristic_device.h) executed on
the host by tests/emul/libwhemul_heuristic_batch.so: a stand-in for `_lib.heuristic_batch` where there is no GPU.  Every phase
visits its rows in a seeded random order, the tables of a group run in a random order, and the work region starts as 0xFF bytes."""
import ctypes as C
import os
import subprocess

from whatshap_b200 import _lib as real
from whatshap_b200._abi import CHeuristicSolution, CProblem

EMUL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "heuristic_batch.mk"], check=True, capture_output=True)
        _lib = C.CDLL(os.path.join(EMUL_DIR, "libwhemul_heuristic_batch.so"))
        _lib.whemul_heuristic_batch.argtypes = [C.POINTER(C.POINTER(CProblem)), C.POINTER(C.POINTER(CHeuristicSolution)), C.POINTER(C.c_uint32),
                                                C.POINTER(C.c_int), C.c_uint32, C.c_uint64, C.c_uint64, C.POINTER(C.c_int), C.c_char_p,
                                                C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_uint32)]
        _lib.whemul_heuristic_batch.restype = C.c_int
    return _lib


def heuristic_batch(problems, row_limits=256, allow_mutations=True, budget: int = 0, seed: int = 0):
    """(results, info): per table its `HeuristicSolution` or the exception `_lib.heuristic` raises for it, and info = {"groups",
    "handed_back" (tables whose rows outgrew their buffers), "group_of" (per table its group, -1: run by whmec_heuristic)}.
    budget = 0: no limit."""
    keep, pp, sp, rl, am, status, errs, errlen, sols = real.heuristic_arguments(problems, row_limits, allow_mutations)
    n = len(sols)
    group_of, info = (C.c_int32 * max(n, 1))(), (C.c_uint32 * 2)()
    assert lib().whemul_heuristic_batch(pp, sp, rl, am, n, budget, seed, status, errs, errlen, group_of, info) == 0
    results = real.heuristic_results(keep, status, errs, errlen, sols)
    return results, {"groups": int(info[0]), "handed_back": int(info[1]), "group_of": [int(group_of[t]) for t in range(n)]}
