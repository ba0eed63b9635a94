"""TEST INFRASTRUCTURE — loaders for the two CPU checkers.

Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference legs) may
import this module.  The product package (whatshap_b200/) never does.

  port()       oracle/liboracle.so        plain-C restatement (oracle/mec_oracle.c)
  reference()  oracle/_ref/libwhref.so    the unmodified reference C++, compiled in place
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from functools import lru_cache
from typing import List, Optional, Sequence

from whatshap_b200._abi import CProblem, CSolution, FlatProblem, FlatSolution, raise_for

HERE = os.path.dirname(os.path.abspath(__file__))
PORT_SO = os.path.join(HERE, "liboracle.so")
REF_SO = os.path.join(HERE, "_ref", "libwhref.so")


def build(quiet: bool = True) -> None:
    """Compile the checkers (oracle/Makefile).  The reference build is skipped where the WhatsHap
    sources ($WHATSHAP_REF) are absent: a prebuilt _ref/libwhref.so is used as is."""
    subprocess.run(["make", "-C", HERE], check=True, capture_output=quiet)


class _Checker:
    def __init__(self, path: str, prefix: str, has_time: bool):
        self.lib = C.CDLL(path)
        self.kind = "reference" if has_time else "port"
        self._solve = getattr(self.lib, prefix + "_solve")
        self._has_time = has_time
        if has_time:
            self._solve.argtypes = [C.POINTER(CProblem), C.POINTER(CSolution), C.POINTER(C.c_double), C.c_char_p, C.c_size_t]
            self._many = self.lib.whref_solve_many
            self._many.argtypes = [C.POINTER(C.POINTER(CProblem)), C.c_uint32, C.c_uint32, C.POINTER(C.c_double), C.c_char_p, C.c_size_t]
            self._many.restype = C.c_int
        else:
            self._solve.argtypes = [C.POINTER(CProblem), C.POINTER(CSolution), C.c_char_p, C.c_size_t]
        self._solve.restype = C.c_int
        self.last_seconds: Optional[float] = None
        # forward-backward genotyping DP (GenotypeDPTable): whref_genotype / whoracle_genotype
        self._genotype = getattr(self.lib, prefix + "_genotype", None)
        if self._genotype is not None:
            dp = C.POINTER(C.c_double)
            self._genotype.argtypes = ([C.POINTER(CProblem), dp, dp, C.c_char_p, C.c_size_t] if has_time
                                       else [C.POINTER(CProblem), dp, C.c_char_p, C.c_size_t])
            self._genotype.restype = C.c_int

    def solve(self, prob: FlatProblem) -> FlatSolution:
        sol = FlatSolution(prob.n_cols, prob.n_reads, prob.n_ind)
        cp, cs = prob.as_c(), sol.as_c()
        err = C.create_string_buffer(512)
        if self._has_time:
            secs = C.c_double(0.0)
            rc = self._solve(C.byref(cp), C.byref(cs), C.byref(secs), err, len(err))
            self.last_seconds = secs.value
        else:
            rc = self._solve(C.byref(cp), C.byref(cs), err, len(err))
        raise_for(rc, err.value.decode())
        sol.cost = int(cs.cost)
        return sol

    def heuristic(self, prob: FlatProblem, row_limit: int = 256, allow_mutations: bool = True):
        """The reference's PedMecHeuristic (compiled reference only): a HeuristicSolution."""
        from whatshap_b200._abi import CHeuristicSolution, HeuristicSolution

        fn = self.lib.whref_heuristic
        fn.argtypes = [C.POINTER(CProblem), C.c_uint32, C.c_int, C.POINTER(CHeuristicSolution), C.c_char_p, C.c_size_t]
        fn.restype = C.c_int
        sol = HeuristicSolution(prob.n_cols, prob.n_reads, prob.n_ind)
        cp, cs, err = prob.as_c(), sol.as_c(), C.create_string_buffer(512)
        raise_for(fn(C.byref(cp), int(row_limit), int(bool(allow_mutations)), C.byref(cs), err, len(err)), err.value.decode())
        sol.score, sol.n_samples = float(cs.score), int(cs.n_samples)
        return sol

    def genotype(self, prob: FlatProblem):
        """Genotype likelihoods [n_ind, n_cols, 3] of the reference's GenotypeDPTable (`prob.gl` = priors)."""
        import numpy as np

        out = np.zeros((prob.n_ind, prob.n_cols, 3), np.float64)
        cp, err = prob.as_c(), C.create_string_buffer(512)
        dp = out.ctypes.data_as(C.POINTER(C.c_double))
        if self._has_time:
            secs = C.c_double(0.0)
            rc = self._genotype(C.byref(cp), dp, C.byref(secs), err, len(err))
            self.last_seconds = secs.value
        else:
            rc = self._genotype(C.byref(cp), dp, err, len(err))
        raise_for(rc, err.value.decode())
        return out

    def solve_many_timed(self, probs: Sequence[FlatProblem], threads: int) -> float:
        """Wall seconds for solving all `probs` on `threads` host threads (reference only)."""
        assert self._has_time
        cps = [p.as_c() for p in probs]
        arr = (C.POINTER(CProblem) * len(cps))(*[C.pointer(c) for c in cps])
        err = C.create_string_buffer(512)
        wall = C.c_double(0.0)
        rc = self._many(arr, len(cps), threads, C.byref(wall), err, len(err))
        raise_for(rc, err.value.decode())
        return wall.value


@lru_cache(maxsize=None)
def port() -> _Checker:
    if not os.path.exists(PORT_SO):
        build()
    return _Checker(PORT_SO, "whoracle", has_time=False)


@lru_cache(maxsize=None)
def reference() -> Optional[_Checker]:
    if not os.path.exists(REF_SO):
        try:
            build()
        except Exception:
            return None
    if not os.path.exists(REF_SO):
        return None
    return _Checker(REF_SO, "whref", has_time=True)


def best() -> _Checker:
    """The strongest checker available: the compiled reference if present, else the C port."""
    return reference() or port()
