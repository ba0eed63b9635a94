"""Loader and thin typed wrappers for libwhmec.so (the C ABI of include/whmec.h).

The CUDA library is the only compute path: if it is missing or cannot be loaded this module
raises at first use — there is no CPU fallback anywhere in this package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from functools import lru_cache
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from ._abi import CHaplotagInput, CHaplotagOutput, CHaplotagphaseInput, CHaplotagphaseOutput, CHaplotagphaseStats, CHaplotagStats, CHeuristicSolution, CKmeraldParams, CLearnInput, CLearnOutput, CLearnStats, CMergeInput, CMergeOutput, CMergeStats, CProblem, CQueryQualities, CRealignInput, CRealignOutput, CRealignStats, CSolution, CStats, FlatProblem, FlatSolution, HeuristicSolution, raise_for

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
    "whmec_solve_batch",
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
    "whmec_genotype_batch",
    "whmec_genotype_segment_create",
    "whmec_genotype_segment_transfer",
    "whmec_genotype_segment_run",
    "whmec_genotype_segment_destroy",
    "whmec_compute_genotypes",
    "whmec_heuristic",
    "whmec_heuristic_batch",
    "whmec_realign",
    "whmec_realign_release",
    "whmec_edit_distance_batch",
    "whmec_realign_kmerald",
    "whmec_kmer_align_batch",
    "whmec_detect_alleles_cigar",
    "whmec_learn",
    "whmec_learn_release",
    "whmec_learn_write",
    "whmec_haplotag",
    "whmec_haplotagphase",
    "whmec_haplotagphase_release",
    "whmec_merge_reads",
    "whmec_merge_reads_release",
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
    L.whmec_solve_batch.argtypes = [C.POINTER(C.POINTER(CProblem)), C.POINTER(C.POINTER(CSolution)), C.c_uint32, C.c_int, C.POINTER(C.c_int),
                                    C.c_char_p, C.c_size_t, C.POINTER(CStats), C.POINTER(CStats)]
    L.whmec_solve_batch.restype = C.c_int
    L.whmec_genotype.argtypes = [C.POINTER(CProblem), C.POINTER(C.c_double), C.c_int, C.POINTER(CStats), C.c_char_p, C.c_size_t]
    L.whmec_genotype.restype = C.c_int
    L.whmec_genotype_batch.argtypes = [C.POINTER(C.POINTER(CProblem)), C.POINTER(C.POINTER(C.c_double)), C.c_uint32, C.c_int, C.POINTER(C.c_int),
                                       C.c_char_p, C.c_size_t, C.POINTER(CStats), C.POINTER(CStats)]
    L.whmec_genotype_batch.restype = C.c_int
    L.whmec_compute_genotypes.argtypes = [C.POINTER(CProblem), C.POINTER(C.c_double), C.POINTER(C.c_int8), C.c_char_p, C.c_size_t]
    L.whmec_compute_genotypes.restype = C.c_int
    L.whmec_heuristic.argtypes = [C.POINTER(CProblem), C.c_uint32, C.c_int, C.POINTER(CHeuristicSolution), C.c_char_p, C.c_size_t]
    L.whmec_heuristic.restype = C.c_int
    L.whmec_heuristic_batch.argtypes = [C.POINTER(C.POINTER(CProblem)), C.POINTER(C.POINTER(CHeuristicSolution)), C.POINTER(C.c_uint32),
                                        C.POINTER(C.c_int), C.c_uint32, C.c_int, C.POINTER(C.c_int), C.c_char_p, C.c_size_t, C.POINTER(CStats),
                                        C.POINTER(CStats)]
    L.whmec_heuristic_batch.restype = C.c_int
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
    f64p = C.POINTER(C.c_double)
    L.whmec_genotype_segment_create.argtypes = [C.POINTER(CProblem), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]
    L.whmec_genotype_segment_transfer.argtypes = [C.c_void_p, f64p, C.POINTER(CStats), C.c_char_p, C.c_size_t]
    L.whmec_genotype_segment_run.argtypes = [C.c_void_p, f64p, f64p, f64p, C.POINTER(CStats), C.c_char_p, C.c_size_t]
    L.whmec_genotype_segment_destroy.argtypes = [C.c_void_p]
    L.whmec_genotype_segment_destroy.restype = None
    realign_signatures(L)
    cigar_alleles_signatures(L)
    learn_signatures(L)
    haplotag_signatures(L)
    haplotagphase_signatures(L)
    merge_reads_signatures(L)
    for name in ("whmec_genotype_segment_create", "whmec_genotype_segment_transfer", "whmec_genotype_segment_run"):
        getattr(L, name).restype = C.c_int
    for name in ("whmec_plan_create", "whmec_plan_sweep", "whmec_plan_finish", "whmec_plan_stats", "whmec_solve",
                 "whmec_segment_create", "whmec_segment_transfer", "whmec_segment_sweep", "whmec_segment_exits",
                 "whmec_segment_finish"):
        getattr(L, name).restype = C.c_int
    return L


def cigar_alleles_signatures(L: C.CDLL) -> C.CDLL:
    """argtypes of whmec_detect_alleles_cigar and whmec_realign_release on `L` (this library or a test build that exports them)."""
    L.whmec_detect_alleles_cigar.argtypes = [C.POINTER(CRealignInput), C.POINTER(CQueryQualities), C.c_int, C.POINTER(CRealignOutput),
                                             C.POINTER(CRealignStats), C.c_char_p, C.c_size_t]
    L.whmec_detect_alleles_cigar.restype = C.c_int
    L.whmec_realign_release.argtypes = [C.POINTER(CRealignOutput)]
    L.whmec_realign_release.restype = None
    return L


def realign_signatures(L: C.CDLL) -> C.CDLL:
    """argtypes of whmec_realign, whmec_realign_release, whmec_edit_distance_batch, whmec_realign_kmerald and
    whmec_kmer_align_batch on `L` (this library or a test build that exports the same symbols; those it lacks are skipped)."""
    i64p = C.POINTER(C.c_int64)
    L.whmec_realign.argtypes = [C.POINTER(CRealignInput), C.c_int, C.POINTER(CRealignOutput), C.POINTER(CRealignStats), C.c_char_p, C.c_size_t]
    L.whmec_realign.restype = C.c_int
    L.whmec_realign_release.argtypes = [C.POINTER(CRealignOutput)]
    L.whmec_realign_release.restype = None
    L.whmec_edit_distance_batch.argtypes = [C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.POINTER(C.c_uint8),
                                            C.c_double, C.c_int32, C.c_int32, i64p, i64p, C.c_int, C.POINTER(CRealignStats), C.c_char_p, C.c_size_t]
    L.whmec_edit_distance_batch.restype = C.c_int
    if hasattr(L, "whmec_realign_kmerald"):
        L.whmec_realign_kmerald.argtypes = [C.POINTER(CRealignInput), C.POINTER(CKmeraldParams), C.c_int, C.POINTER(CRealignOutput),
                                            C.POINTER(CRealignStats), C.c_char_p, C.c_size_t]
        L.whmec_realign_kmerald.restype = C.c_int
        L.whmec_kmer_align_batch.argtypes = [C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.POINTER(C.c_uint8),
                                             C.POINTER(CKmeraldParams), C.POINTER(C.c_float), C.c_int, C.POINTER(CRealignStats), C.c_char_p,
                                             C.c_size_t]
        L.whmec_kmer_align_batch.restype = C.c_int
    return L


def learn_signatures(L: C.CDLL) -> C.CDLL:
    """argtypes of whmec_learn, whmec_learn_release and whmec_learn_write on `L` (this library or a test build)."""
    L.whmec_learn.argtypes = [C.POINTER(CLearnInput), C.c_int, C.POINTER(CLearnOutput), C.POINTER(CLearnStats), C.c_char_p, C.c_size_t]
    L.whmec_learn.restype = C.c_int
    L.whmec_learn_release.argtypes = [C.POINTER(CLearnOutput)]
    L.whmec_learn_release.restype = None
    L.whmec_learn_write.argtypes = [C.c_char_p, C.POINTER(CLearnOutput), C.c_int, C.c_char_p, C.c_size_t]
    L.whmec_learn_write.restype = C.c_int
    return L


def haplotag_signatures(L: C.CDLL) -> C.CDLL:
    """argtypes of whmec_haplotag on `L` (this library or a test build)."""
    L.whmec_haplotag.argtypes = [C.POINTER(CHaplotagInput), C.c_int, C.POINTER(CHaplotagOutput), C.POINTER(CHaplotagStats), C.c_char_p,
                                 C.c_size_t]
    L.whmec_haplotag.restype = C.c_int
    return L


def haplotagphase_signatures(L: C.CDLL) -> C.CDLL:
    """argtypes of whmec_haplotagphase and whmec_haplotagphase_release on `L` (this library or a test build)."""
    L.whmec_haplotagphase.argtypes = [C.POINTER(CHaplotagphaseInput), C.c_int, C.POINTER(CHaplotagphaseOutput), C.POINTER(CHaplotagphaseStats),
                                      C.c_char_p, C.c_size_t]
    L.whmec_haplotagphase.restype = C.c_int
    L.whmec_haplotagphase_release.argtypes = [C.POINTER(CHaplotagphaseOutput)]
    L.whmec_haplotagphase_release.restype = None
    return L


def merge_reads_signatures(L: C.CDLL) -> C.CDLL:
    """argtypes of whmec_merge_reads and whmec_merge_reads_release on `L` (this library or a test build)."""
    L.whmec_merge_reads.argtypes = [C.POINTER(CMergeInput), C.c_int, C.POINTER(CMergeOutput), C.POINTER(CMergeStats), C.c_char_p, C.c_size_t]
    L.whmec_merge_reads.restype = C.c_int
    L.whmec_merge_reads_release.argtypes = [C.POINTER(CMergeOutput)]
    L.whmec_merge_reads_release.restype = None
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


def solve_batch(problems: Sequence[FlatProblem], device: int = 0, with_stats: bool = False):
    """Several tables through one `whmec_solve_batch`: a list with, per table and in input order, its `FlatSolution` -- bit for
    bit what `solve` gives for it alone -- or the exception `solve` would have raised for it (the other tables are still solved).
    A failure of the call itself (no device, a CUDA error) raises.  `with_stats`: also returns (per-table stats, totals of the call)."""
    n = len(problems)
    sols = [FlatSolution(p.n_cols, p.n_reads, p.n_ind) for p in problems]
    cps, css = [p.as_c() for p in problems], [s.as_c() for s in sols]
    pp = (C.POINTER(CProblem) * max(n, 1))(*[C.pointer(c) for c in cps])
    sp = (C.POINTER(CSolution) * max(n, 1))(*[C.pointer(c) for c in css])
    status = (C.c_int * max(n, 1))()
    errlen = 512
    errs = C.create_string_buffer(errlen * max(n, 1))
    stats, total = (CStats * max(n, 1))(), CStats()
    rc = lib().whmec_solve_batch(pp, sp, n, device, status, errs, errlen, stats, C.byref(total))
    messages = [errs.raw[t * errlen:(t + 1) * errlen].split(b"\0", 1)[0].decode() for t in range(n)]
    if rc != 0:
        raise_for(rc, messages[0] if messages else "whmec_solve_batch: invalid arguments")
    out: List[Union[FlatSolution, Exception]] = []
    for t in range(n):
        try:
            raise_for(int(status[t]), messages[t])
            sols[t].cost = int(css[t].cost)
            out.append(sols[t])
        except Exception as e:  # noqa: BLE001 - handed to the caller in the table's place
            out.append(e)
    if with_stats:
        return out, ([stats[t].as_dict() for t in range(n)], total.as_dict())
    return out


def genotype(prob: FlatProblem, device: int = 0) -> Tuple[np.ndarray, dict]:
    """Genotype likelihoods [n_ind, n_cols, 3] by the forward-backward DP (`whmec_genotype`); `prob.gl` holds the priors."""
    out = np.zeros((prob.n_ind, prob.n_cols, 3), np.float64)
    cp, st = prob.as_c(), CStats()
    err = C.create_string_buffer(512)
    rc = lib().whmec_genotype(C.byref(cp), out.ctypes.data_as(C.POINTER(C.c_double)), device, C.byref(st), err, len(err))
    raise_for(rc, err.value.decode())
    return out, st.as_dict()


def genotype_batch(problems: Sequence[FlatProblem], device: int = 0, with_stats: bool = False):
    """Several tables through one `whmec_genotype_batch`: a list with, per table and in input order, its likelihoods
    [n_ind, n_cols, 3] -- what `genotype` gives for it alone -- or the exception `genotype` would have raised for it (the other
    tables are still genotyped).  A failure of the call itself (no device, a CUDA error) raises.  `with_stats`: also returns
    (per-table stats, totals of the call)."""
    n = len(problems)
    outs = [np.zeros((p.n_ind, p.n_cols, 3), np.float64) for p in problems]
    cps = [p.as_c() for p in problems]
    pp = (C.POINTER(CProblem) * max(n, 1))(*[C.pointer(c) for c in cps])
    lp = (C.POINTER(C.c_double) * max(n, 1))(*[o.ctypes.data_as(C.POINTER(C.c_double)) for o in outs])
    status = (C.c_int * max(n, 1))()
    errlen = 512
    errs = C.create_string_buffer(errlen * max(n, 1))
    stats, total = (CStats * max(n, 1))(), CStats()
    rc = lib().whmec_genotype_batch(pp, lp, n, device, status, errs, errlen, stats, C.byref(total))
    messages = [errs.raw[t * errlen:(t + 1) * errlen].split(b"\0", 1)[0].decode() for t in range(n)]
    if rc != 0:
        raise_for(rc, messages[0] if messages else "whmec_genotype_batch: invalid arguments")
    out: List[Union[np.ndarray, Exception]] = []
    for t in range(n):
        try:
            raise_for(int(status[t]), messages[t])
            out.append(outs[t])
        except Exception as e:  # noqa: BLE001 - handed to the caller in the table's place
            out.append(e)
    if with_stats:
        return out, ([stats[t].as_dict() for t in range(n)], total.as_dict())
    return out


def heuristic(prob: FlatProblem, row_limit: int = 256, allow_mutations: bool = True) -> HeuristicSolution:
    """The row-limited heuristic PedMEC solver (`whmec_heuristic`, host code): `prob.read_ind` holds the reads' sample ids."""
    sol = HeuristicSolution(prob.n_cols, prob.n_reads, prob.n_ind)
    cp, cs = prob.as_c(), sol.as_c()
    err = C.create_string_buffer(512)
    rc = lib().whmec_heuristic(C.byref(cp), int(row_limit), int(bool(allow_mutations)), C.byref(cs), err, len(err))
    raise_for(rc, err.value.decode())
    sol.score, sol.n_samples = float(cs.score), int(cs.n_samples)
    return sol


def heuristic_arguments(problems: Sequence[FlatProblem], row_limits, allow_mutations):
    """The ctypes arguments of `whmec_heuristic_batch` (and of its test emulation): (keep-alive objects, problems, solutions,
    row limits, allow_mutations, status, errs, errlen, result objects).  `row_limits` / `allow_mutations`: one per table or one
    for all."""
    n = len(problems)
    if isinstance(row_limits, (int, np.integer)):
        row_limits = [row_limits] * n
    if isinstance(allow_mutations, (bool, int, np.integer)):
        allow_mutations = [allow_mutations] * n
    row_limits, allow_mutations = list(row_limits), list(allow_mutations)
    if len(row_limits) != n or len(allow_mutations) != n:
        raise ValueError("row_limits and allow_mutations need one entry per table")
    sols = [HeuristicSolution(p.n_cols, p.n_reads, p.n_ind) for p in problems]
    cps, css = [p.as_c() for p in problems], [s.as_c() for s in sols]
    pp = (C.POINTER(CProblem) * max(n, 1))(*[C.pointer(c) for c in cps])
    sp = (C.POINTER(CHeuristicSolution) * max(n, 1))(*[C.pointer(c) for c in css])
    rl = (C.c_uint32 * max(n, 1))(*[int(r) for r in row_limits])
    am = (C.c_int * max(n, 1))(*[int(bool(a)) for a in allow_mutations])
    status = (C.c_int * max(n, 1))()
    errlen = 512
    errs = C.create_string_buffer(errlen * max(n, 1))
    return (cps, css), pp, sp, rl, am, status, errs, errlen, sols


def heuristic_results(keep, status, errs, errlen, sols) -> list:
    """Per table its `HeuristicSolution` or the exception `heuristic` raises for it (after `whmec_heuristic_batch`)."""
    css = keep[1]
    out: List[Union[HeuristicSolution, Exception]] = []
    for t, sol in enumerate(sols):
        try:
            raise_for(int(status[t]), errs.raw[t * errlen:(t + 1) * errlen].split(b"\0", 1)[0].decode())
            sol.score, sol.n_samples = float(css[t].score), int(css[t].n_samples)
            out.append(sol)
        except Exception as e:  # noqa: BLE001 - handed to the caller in the table's place
            out.append(e)
    return out


def heuristic_batch(problems: Sequence[FlatProblem], row_limits=256, allow_mutations=True, device: int = 0, with_stats: bool = False):
    """Several heuristic tables through one `whmec_heuristic_batch`: a list with, per table and in input order, its
    `HeuristicSolution` -- bit for bit what `heuristic` gives for it alone -- or the exception `heuristic` would have raised for it
    (the other tables are still solved).  `row_limits` / `allow_mutations`: per table, or one value for all.  A failure of the
    call itself (no device, a CUDA error) raises.  `with_stats`: also returns (per-table stats, totals of the call)."""
    keep, pp, sp, rl, am, status, errs, errlen, sols = heuristic_arguments(problems, row_limits, allow_mutations)
    n = len(sols)
    stats, total = (CStats * max(n, 1))(), CStats()
    rc = lib().whmec_heuristic_batch(pp, sp, rl, am, n, device, status, errs, errlen, stats, C.byref(total))
    if rc != 0:
        message = errs.raw[:errlen].split(b"\0", 1)[0].decode() if n else ""
        raise_for(rc, message or "whmec_heuristic_batch: invalid arguments")
    out = heuristic_results(keep, status, errs, errlen, sols)
    if with_stats:
        return out, ([stats[t].as_dict() for t in range(n)], total.as_dict())
    return out


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


class GenotypeSegment:
    """A run of whole chains of a pedigree genotyping table on one GPU (`whmec_genotype_segment_*`, include/whmec.h): the unit
    `multigpu.genotype_sharded` spreads over the ranks when T > 1.  `continues`: the segment does not start the table;
    `continued`: it does not end it.  `stats` holds the statistics of the last `transfer()` / `run()`."""

    def __init__(self, prob: FlatProblem, continues: bool, continued: bool, device: int = 0):
        self.prob = prob
        self.T = 4 ** prob.n_trios
        self.stats: dict = {}
        self._h = C.c_void_p()
        cp = prob.as_c()
        err = C.create_string_buffer(512)
        rc = lib().whmec_genotype_segment_create(C.byref(cp), device, int(bool(continues)), int(bool(continued)), C.byref(self._h), err, len(err))
        raise_for(rc, err.value.decode())

    @staticmethod
    def _ptr(a):
        return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))

    def transfer(self) -> np.ndarray:
        """The T x T transfer matrix: row u is the segment's forward output for the input e_u."""
        m = np.zeros((self.T, self.T), np.float64)
        st, err = CStats(), C.create_string_buffer(512)
        raise_for(lib().whmec_genotype_segment_transfer(self._h, self._ptr(m), C.byref(st), err, len(err)), err.value.decode())
        self.stats = st.as_dict()
        return m

    def run(self, alpha: Optional[np.ndarray] = None, beta: Optional[np.ndarray] = None) -> np.ndarray:
        """Likelihoods [n_ind, segment columns, 3] from the true forward input `alpha` and backward input `beta` (T each)."""
        out = np.zeros((self.prob.n_ind, self.prob.n_cols, 3), np.float64)
        a = None if alpha is None else np.ascontiguousarray(alpha, np.float64)
        b = None if beta is None else np.ascontiguousarray(beta, np.float64)
        st, err = CStats(), C.create_string_buffer(512)
        raise_for(lib().whmec_genotype_segment_run(self._h, self._ptr(a), self._ptr(b), self._ptr(out), C.byref(st), err, len(err)),
                  err.value.decode())
        self.stats = st.as_dict()
        return out

    def close(self) -> None:
        if self._h:
            lib().whmec_genotype_segment_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def read_sort_key(name: str, source_id: int) -> int:
    b = name.encode("utf-8")
    return int(lib().whmec_read_sort_key(b, len(b), source_id))
