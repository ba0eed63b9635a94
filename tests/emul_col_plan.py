"""TEST-ONLY: the column-kernel plan (whatshap_b200/csrc/col_plan.cpp) computed on the host by tests/emul/libwhemul_col_plan.so for given
device figures and switches, so that path choice and memory-bounded segments can be checked without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np

from whatshap_b200._abi import CProblem

EMUL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
PATHS = ("column", "batched", "fused")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "col_plan.mk"], check=True, capture_output=True)
        L = C.CDLL(os.path.join(EMUL_DIR, "libwhemul_col_plan.so"))
        u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
        L.whemul_col_plan.argtypes = [C.POINTER(CProblem), C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_uint32,
                                      u64p, u32p, u32p, u32p, u32p, u64p, C.c_uint32, C.c_char_p, C.c_size_t]
        _lib = L
    return _lib


def col_plan(prob, free_bytes=1 << 40, hook=0, fused=True, sequential=False, segment=0, bounded_t1=False, sms=132, cluster=0):
    """The plan as a dict: rc and msg (WHMEC_OK = 0), path, bounded, over_hbm, arena / ckpt words, budget and fixed bytes,
    bp_words (resident), cluster, cuts (chain cuts of a two-pass plan, else column cuts), chain_begin and every column's bp_off."""
    cap = prob.n_cols + 1
    info = np.zeros(9, np.uint64)
    cuts, chain_begin, bp_off = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32), np.zeros(cap, np.uint64)
    n_cuts, n_cb = C.c_uint32(0), C.c_uint32(0)
    cp, err = prob.as_c(), C.create_string_buffer(512)
    u32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))  # noqa: E731
    u64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint64))  # noqa: E731
    rc = lib().whemul_col_plan(C.byref(cp), free_bytes, hook, int(fused), int(sequential), segment, int(bounded_t1), sms, cluster, u64(info),
                               u32(cuts), C.byref(n_cuts), u32(chain_begin), C.byref(n_cb), u64(bp_off), cap, err, len(err))
    keys = ("path", "bounded", "over_hbm", "arena", "ckpt", "budget", "fixed", "bp_words", "cluster")
    out = {k: int(v) for k, v in zip(keys, info)}
    out.update(rc=rc, msg=err.value.decode(), path=PATHS[out["path"]], bounded=bool(out["bounded"]), over_hbm=bool(out["over_hbm"]),
               cuts=cuts[:n_cuts.value].astype(np.int64), chain_begin=chain_begin[:n_cb.value].astype(np.int64),
               bp_off=bp_off[:prob.n_cols].astype(np.int64))
    return out
