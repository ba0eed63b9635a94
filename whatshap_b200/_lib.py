"""Loader and thin typed wrappers for libwhmec.so (the C ABI of include/whmec.h).

The CUDA library is the only compute path: if it is missing or cannot be loaded this module
raises at first use — there is no CPU fallback anywhere in this package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from functools import lru_cache
from typing import Optional, Tuple

import numpy as np

from ._abi import CHeuristicSolution, CProblem, CSolution, CStats, FlatProblem, FlatSolution, HeuristicSolution, raise_for

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("WHMEC_LIBRARY") or os.path.join(HERE, "libwhmec.so")  # WHMEC_LIBRARY: another build of the same library (A/B runs)

#: every symbol include/whmec.h declares (checked by tests/test_abi.py)
EXPORTS = (
    "whmec_abi_version",
    "whmec_build_info",
    "whmec_device_count",
    "whmec_plan_create",
    "whmec_plan_sweep",
    "whmec_plan_finish",
    "whmec_plan_stats",
    "whmec_plan_destroy",
    "whmec_solve",
    "whmec_segment_create",
    "whmec_segment_transfer",
    "whmec_segment_sweep",
    "whmec_segment_exits",
    "whmec_segment_finish",
    "whmec_selector_create",
    "whmec_selector_destroy",
    "whmec_selector_begin_slice",
    "whmec_selector_next",
    "whmec_selector_rescore",
    "whmec_selector_bridge",
    "whmec_read_sort_key",
    "whmec_genotype",
    "whmec_compute_genotypes",
    "whmec_heuristic",
)


def build(verbose: bool = False) -> str:
    """Compile libwhmec.so in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    res = subprocess.run(["make", "-C", os.path.join(HERE, "csrc")], capture_output=not verbose, text=True)
    if res.returncode != 0:
        raise RuntimeError("building libwhmec.so failed:\n" + (res.stdout or "") + (res.stderr or ""))
    return LIB_PATH


@lru_cache(maxsize=None)
def lib() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(whatshap_b200 has no CPU fallback)"
        )
    L = C.CDLL(LIB_PATH)
    L.whmec_abi_version.restype = C.c_int
    L.whmec_build_info.restype = C.c_char_p
    L.whmec_device_count.restype = C.c_int
    L.whmec_plan_create.argtypes = [C.POINTER(CProblem), C.c_int, C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]
    L.whmec_plan_sweep.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    L.whmec_plan_finish.argtypes = [C.c_void_p, C.POINTER(CSolution), C.c_char_p, C.c_size_t]
    L.whmec_plan_stats.argtypes = [C.c_void_p, C.POINTER(CStats)]
    L.whmec_plan_destroy.argtypes = [C.c_void_p]
    L.whmec_plan_destroy.restype = None
    L.whmec_solve.argtypes = [C.POINTER(CProblem), C.POINTER(CSolution), C.c_int, C.POINTER(CStats), C.c_char_p, C.c_size_t]
    L.whmec_genotype.argtypes = [C.POINTER(CProblem), C.POINTER(C.c_double), C.c_int, C.POINTER(CStats), C.c_char_p, C.c_size_t]
    L.whmec_genotype.restype = C.c_int
    L.whmec_compute_genotypes.argtypes = [C.POINTER(CProblem), C.POINTER(C.c_double), C.POINTER(C.c_int8), C.c_char_p, C.c_size_t]
    L.whmec_compute_genotypes.restype = C.c_int
    L.whmec_heuristic.argtypes = [C.POINTER(CProblem), C.c_uint32, C.c_int, C.POINTER(CHeuristicSolution), C.c_char_p, C.c_size_t]
    L.whmec_heuristic.restype = C.c_int
    L.whmec_read_sort_key.argtypes = [C.c_char_p, C.c_size_t, C.c_int32]
    L.whmec_read_sort_key.restype = C.c_uint64
    u32p = C.POINTER(C.c_uint32)
    i32p = C.POINTER(C.c_int32)
    u64p, u8p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint8)
    L.whmec_selector_create.argtypes = [C.c_uint32, C.c_uint32, u64p, i32p, u32p, i32p, C.c_uint32]
    L.whmec_selector_create.restype = C.c_void_p
    L.whmec_selector_destroy.argtypes = [C.c_void_p]
    L.whmec_selector_destroy.restype = None
    L.whmec_selector_begin_slice.argtypes = [C.c_void_p, u32p, i32p, C.c_uint32]
    L.whmec_selector_begin_slice.restype = None
    L.whmec_selector_next.argtypes = [C.c_void_p, u32p, u32p, u32p, u32p, u32p]
    L.whmec_selector_next.restype = C.c_int
    L.whmec_selector_rescore.argtypes = [C.c_void_p, u32p, C.c_uint32]
    L.whmec_selector_rescore.restype = None
    L.whmec_selector_bridge.argtypes = [C.c_void_p, u32p, i32p, C.c_uint32, u32p, C.c_uint32, u32p, u8p]
    L.whmec_selector_bridge.restype = C.c_uint32
    L.whmec_segment_create.argtypes = [C.POINTER(CProblem), C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]
    L.whmec_segment_transfer.argtypes = [C.c_void_p, u32p, C.c_char_p, C.c_size_t]
    L.whmec_segment_sweep.argtypes = [C.c_void_p, u32p, u32p, C.c_char_p, C.c_size_t]
    L.whmec_segment_exits.argtypes = [C.c_void_p, C.c_int, u32p, C.c_char_p, C.c_size_t]
    L.whmec_segment_finish.argtypes = [C.c_void_p, C.c_int, C.POINTER(CSolution), C.c_char_p, C.c_size_t]
    for name in ("whmec_plan_create", "whmec_plan_sweep", "whmec_plan_finish", "whmec_plan_stats", "whmec_solve",
                 "whmec_segment_create", "whmec_segment_transfer", "whmec_segment_sweep", "whmec_segment_exits",
                 "whmec_segment_finish"):
        getattr(L, name).restype = C.c_int
    return L


def device_count() -> int:
    return int(lib().whmec_device_count())


def solve(prob: FlatProblem, device: int = 0) -> Tuple[FlatSolution, dict]:
    """One-shot solve through `whmec_solve` (host buffers in, host buffers out)."""
    sol = FlatSolution(prob.n_cols, prob.n_reads, prob.n_ind)
    cp, cs, st = prob.as_c(), sol.as_c(), CStats()
    err = C.create_string_buffer(512)
    rc = lib().whmec_solve(C.byref(cp), C.byref(cs), device, C.byref(st), err, len(err))
    raise_for(rc, err.value.decode())
    sol.cost = int(cs.cost)
    return sol, st.as_dict()


def genotype(prob: FlatProblem, device: int = 0) -> Tuple[np.ndarray, dict]:
    """Genotype likelihoods [n_ind, n_cols, 3] by the forward-backward DP (`whmec_genotype`); `prob.gl` holds the priors."""
    out = np.zeros((prob.n_ind, prob.n_cols, 3), np.float64)
    cp, st = prob.as_c(), CStats()
    err = C.create_string_buffer(512)
    rc = lib().whmec_genotype(C.byref(cp), out.ctypes.data_as(C.POINTER(C.c_double)), device, C.byref(st), err, len(err))
    raise_for(rc, err.value.decode())
    return out, st.as_dict()


def heuristic(prob: FlatProblem, row_limit: int = 256, allow_mutations: bool = True) -> HeuristicSolution:
    """The row-limited heuristic PedMEC solver (`whmec_heuristic`, host code): `prob.read_ind` holds the reads' sample ids."""
    sol = HeuristicSolution(prob.n_cols, prob.n_reads, prob.n_ind)
    cp, cs = prob.as_c(), sol.as_c()
    err = C.create_string_buffer(512)
    rc = lib().whmec_heuristic(C.byref(cp), int(row_limit), int(bool(allow_mutations)), C.byref(cs), err, len(err))
    raise_for(rc, err.value.decode())
    sol.score, sol.n_samples = float(cs.score), int(cs.n_samples)
    return sol


def compute_genotypes(prob: FlatProblem) -> Tuple[np.ndarray, np.ndarray]:
    """Per-column genotype priors of the reads of `prob` (`whmec_compute_genotypes`, host only): (gl [n_cols, 3], gt [n_cols], -1 = none)."""
    gl = np.zeros((prob.n_cols, 3), np.float64)
    gt = np.zeros(prob.n_cols, np.int8)
    cp, err = prob.as_c(), C.create_string_buffer(512)
    rc = lib().whmec_compute_genotypes(C.byref(cp), gl.ctypes.data_as(C.POINTER(C.c_double)), gt.ctypes.data_as(C.POINTER(C.c_int8)), err, len(err))
    raise_for(rc, err.value.decode())
    return gl, gt


class Plan:
    """Device-resident problem: `sweep()` can be timed repeatedly with inputs already in HBM."""

    def __init__(self, prob: FlatProblem, device: int = 0):
        self.prob = prob
        self._h = C.c_void_p()
        cp = prob.as_c()
        err = C.create_string_buffer(512)
        rc = lib().whmec_plan_create(C.byref(cp), device, C.byref(self._h), err, len(err))
        raise_for(rc, err.value.decode())

    def sweep(self) -> None:
        err = C.create_string_buffer(512)
        raise_for(lib().whmec_plan_sweep(self._h, err, len(err)), err.value.decode())

    def finish(self) -> FlatSolution:
        sol = FlatSolution(self.prob.n_cols, self.prob.n_reads, self.prob.n_ind)
        cs = sol.as_c()
        err = C.create_string_buffer(512)
        raise_for(lib().whmec_plan_finish(self._h, C.byref(cs), err, len(err)), err.value.decode())
        sol.cost = int(cs.cost)
        return sol

    def stats(self) -> dict:
        st = CStats()
        lib().whmec_plan_stats(self._h, C.byref(st))
        return st.as_dict()

    def close(self) -> None:
        if self._h:
            lib().whmec_plan_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Segment:
    """A run of whole chains of a pedigree table on one GPU (`whmec_segment_*`, include/whmec.h):
    the unit `multigpu.solve_sharded` spreads over the ranks when T > 1."""

    def __init__(self, prob: FlatProblem, continues: bool, device: int = 0):
        self.prob = prob
        self.T = 4 ** prob.n_trios
        self._h = C.c_void_p()
        cp = prob.as_c()
        err = C.create_string_buffer(512)
        rc = lib().whmec_segment_create(C.byref(cp), device, int(bool(continues)), C.byref(self._h), err, len(err))
        raise_for(rc, err.value.decode())

    @staticmethod
    def _ptr(a):
        return a.ctypes.data_as(C.POINTER(C.c_uint32))

    def transfer(self):
        import numpy as np

        m = np.zeros((self.T, self.T), np.uint32)
        err = C.create_string_buffer(512)
        raise_for(lib().whmec_segment_transfer(self._h, self._ptr(m), err, len(err)), err.value.decode())
        return m

    def sweep(self, in_vec=None):
        import numpy as np

        out = np.zeros(self.T, np.uint32)
        vec = None if in_vec is None else np.ascontiguousarray(in_vec, np.uint32)
        err = C.create_string_buffer(512)
        rc = lib().whmec_segment_sweep(self._h, None if vec is None else self._ptr(vec), self._ptr(out), err, len(err))
        raise_for(rc, err.value.decode())
        return out

    def exits(self, is_last: bool):
        import numpy as np

        out = np.zeros(self.T, np.uint32)
        err = C.create_string_buffer(512)
        raise_for(lib().whmec_segment_exits(self._h, int(bool(is_last)), self._ptr(out), err, len(err)), err.value.decode())
        return out

    def finish(self, entry: int) -> FlatSolution:
        sol = FlatSolution(self.prob.n_cols, self.prob.n_reads, self.prob.n_ind)
        cs = sol.as_c()
        err = C.create_string_buffer(512)
        raise_for(lib().whmec_segment_finish(self._h, int(entry), C.byref(cs), err, len(err)), err.value.decode())
        sol.cost = int(cs.cost)
        return sol

    def stats(self) -> dict:
        st = CStats()
        lib().whmec_plan_stats(self._h, C.byref(st))
        return st.as_dict()

    def close(self) -> None:
        if self._h:
            lib().whmec_plan_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def read_sort_key(name: str, source_id: int) -> int:
    b = name.encode("utf-8")
    return int(lib().whmec_read_sort_key(b, len(b), source_id))
