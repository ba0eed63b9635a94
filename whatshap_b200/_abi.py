"""ctypes mirror of include/whmec.h plus numpy-backed containers for its arrays.

`FlatProblem` is the flat (CSR) form of one `PedigreeDPTable(...)` call — what the reference
holds as ReadSet / Pedigree / recombcost objects (whatshap/core.pyx:364-376) — and
`FlatSolution` holds everything the reference object can be asked for afterwards
(core.pyx:381-416).  Nothing here computes anything; it only describes memory.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

WHMEC_OK = 0
WHMEC_ERR_MENDELIAN = 1
WHMEC_ERR_INPUT = 2
WHMEC_ERR_CUDA = 3
WHMEC_ERR_UNSUPPORTED = 4
GT_OTHER = 255

_u8p = C.POINTER(C.c_uint8)
_u32p = C.POINTER(C.c_uint32)
_u64p = C.POINTER(C.c_uint64)
_f64p = C.POINTER(C.c_double)


class CProblem(C.Structure):
    _fields_ = [
        ("n_cols", C.c_uint32),
        ("positions", _u32p),
        ("n_reads", C.c_uint32),
        ("read_off", _u64p),
        ("ent_col", _u32p),
        ("ent_allele", _u8p),
        ("ent_phred", _u32p),
        ("read_ind", _u32p),
        ("recombcost", _u32p),
        ("n_ind", C.c_uint32),
        ("n_trios", C.c_uint32),
        ("trios", _u32p),
        ("distrust", C.c_uint32),
        ("gt", _u8p),
        ("gl", _f64p),
    ]


class CSolution(C.Structure):
    _fields_ = [
        ("cost", C.c_uint32),
        ("path_index", _u32p),
        ("path_tv", _u32p),
        ("partition", _u8p),
        ("sr_allele", _u8p),
        ("sr_quality", _u32p),
    ]


class CHeuristicSolution(C.Structure):
    """whmec_heuristic_solution (include/whmec.h)."""

    _fields_ = [
        ("score", C.c_float),
        ("n_samples", C.c_uint32),
        ("partition", _u8p),
        ("transmission", _u32p),
        ("haplotypes", C.POINTER(C.c_int8)),
        ("mutated", _u8p),
    ]


class HeuristicSolution:
    """Host arrays behind a whmec_heuristic_solution."""

    def __init__(self, n_cols: int, n_reads: int, n_ind: int):
        self.score = 0.0
        self.n_samples = 0
        self.partition = np.zeros(n_reads, np.uint8)
        self.transmission = np.zeros(n_cols, np.uint32)
        self.haplotypes = np.full((n_ind, 2, n_cols), -1, np.int8)
        self.mutated = np.zeros((n_ind, 2, n_cols), np.uint8)

    def as_c(self) -> "CHeuristicSolution":
        return CHeuristicSolution(0.0, 0, self.partition.ctypes.data_as(_u8p), self.transmission.ctypes.data_as(_u32p),
                                  self.haplotypes.ctypes.data_as(C.POINTER(C.c_int8)), self.mutated.ctypes.data_as(_u8p))

    def same_as(self, other: "HeuristicSolution") -> bool:
        return (self.n_samples == other.n_samples and self.score == other.score and np.array_equal(self.partition, other.partition)
                and np.array_equal(self.transmission, other.transmission)
                and np.array_equal(self.haplotypes[: self.n_samples], other.haplotypes[: self.n_samples])
                and np.array_equal(self.mutated[: self.n_samples], other.mutated[: self.n_samples]))


class CStats(C.Structure):
    _fields_ = [
        ("cells", C.c_uint64),
        ("algorithmic_bytes", C.c_uint64),
        ("backptr_bytes", C.c_uint64),
        ("state_bytes", C.c_uint64),
        ("kernel_launches", C.c_uint32),
        ("n_chains", C.c_uint32),
        ("max_active", C.c_uint32),
        ("transmissions", C.c_uint32),
        ("sweep_ms", C.c_float),
        ("h2d_ms", C.c_float),
        ("d2h_ms", C.c_float),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
        ("path_kind", C.c_uint32),
        ("reserved", C.c_uint32),
    ]

    def as_dict(self) -> dict:
        return {name: getattr(self, name) for name, _ in self._fields_ if name != "reserved"}


def _ptr(a: Optional[np.ndarray], ctype):
    if a is None:
        return C.cast(None, C.POINTER(ctype))
    return a.ctypes.data_as(C.POINTER(ctype))


def _arr(x, dtype, n: Optional[int] = None) -> np.ndarray:
    a = np.ascontiguousarray(x, dtype=dtype)
    if n is not None and a.size != n:
        raise ValueError(f"expected {n} elements, got {a.size}")
    return a


@dataclass
class FlatProblem:
    """Flat form of one DP instance; see `whmec_problem` in include/whmec.h."""

    positions: np.ndarray          # u32 [n_cols]
    read_off: np.ndarray           # u64 [n_reads+1]
    ent_col: np.ndarray            # u32 [nnz]
    ent_allele: np.ndarray         # u8  [nnz]
    ent_phred: np.ndarray          # u32 [nnz]
    read_ind: np.ndarray           # u32 [n_reads]
    recombcost: np.ndarray         # u32 [n_cols]
    n_ind: int = 1
    trios: np.ndarray = field(default_factory=lambda: np.zeros(0, np.uint32))  # u32 [3*n_trios]
    distrust: bool = False
    gt: Optional[np.ndarray] = None  # u8 [n_ind, n_cols]
    gl: Optional[np.ndarray] = None  # f64 [n_ind, n_cols, 3]

    def __post_init__(self):
        self.positions = _arr(self.positions, np.uint32)
        n = self.positions.size
        self.read_off = _arr(self.read_off, np.uint64)
        nnz = int(self.read_off[-1]) if self.read_off.size else 0
        self.ent_col = _arr(self.ent_col, np.uint32, nnz)
        self.ent_allele = _arr(self.ent_allele, np.uint8, nnz)
        self.ent_phred = _arr(self.ent_phred, np.uint32, nnz)
        self.read_ind = _arr(self.read_ind, np.uint32, self.read_off.size - 1)
        rc = np.asarray(self.recombcost, dtype=np.uint32)
        if rc.size < n:
            # the reference indexes recombcost[column] (pedigreedptable.cpp:291); shorter lists are a caller bug
            raise ValueError("recombcost shorter than the number of columns")
        self.recombcost = _arr(rc[:n] if rc.size > n else rc, np.uint32, n)
        self.trios = _arr(self.trios, np.uint32)
        if self.gt is None:
            self.gt = np.full((self.n_ind, n), GT_OTHER, np.uint8)
        self.gt = _arr(self.gt, np.uint8, self.n_ind * n).reshape(self.n_ind, n)
        if self.gl is not None:
            self.gl = _arr(self.gl, np.float64, self.n_ind * n * 3).reshape(self.n_ind, n, 3)

    @property
    def n_cols(self) -> int:
        return int(self.positions.size)

    @property
    def n_reads(self) -> int:
        return int(self.read_ind.size)

    @property
    def n_trios(self) -> int:
        return int(self.trios.size // 3)

    def as_c(self) -> CProblem:
        p = CProblem()
        p.n_cols = self.n_cols
        p.positions = _ptr(self.positions, C.c_uint32)
        p.n_reads = self.n_reads
        p.read_off = _ptr(self.read_off, C.c_uint64)
        p.ent_col = _ptr(self.ent_col, C.c_uint32)
        p.ent_allele = _ptr(self.ent_allele, C.c_uint8)
        p.ent_phred = _ptr(self.ent_phred, C.c_uint32)
        p.read_ind = _ptr(self.read_ind, C.c_uint32)
        p.recombcost = _ptr(self.recombcost, C.c_uint32)
        p.n_ind = self.n_ind
        p.n_trios = self.n_trios
        p.trios = _ptr(self.trios, C.c_uint32)
        p.distrust = 1 if self.distrust else 0
        p.gt = _ptr(self.gt, C.c_uint8)
        p.gl = _ptr(self.gl, C.c_double)
        return p

    def slice_columns(self, lo: int, hi: int) -> "FlatProblem":
        """Sub-problem over columns [lo, hi); valid only if no read crosses the cut."""
        first = self.ent_col[self.read_off[:-1].astype(np.int64)] if self.n_reads else np.zeros(0, np.uint32)
        sel = np.nonzero((first >= lo) & (first < hi))[0]
        if sel.size:
            r0, r1 = int(sel[0]), int(sel[-1]) + 1
            assert sel.size == r1 - r0
        else:
            r0 = r1 = 0
        e0, e1 = int(self.read_off[r0]), int(self.read_off[r1])
        if e1 > e0 and int(self.ent_col[e0:e1].max()) >= hi:
            raise ValueError("a read crosses the requested cut")
        return FlatProblem(
            positions=self.positions[lo:hi],
            read_off=self.read_off[r0 : r1 + 1] - self.read_off[r0],
            ent_col=self.ent_col[e0:e1] - np.uint32(lo),
            ent_allele=self.ent_allele[e0:e1],
            ent_phred=self.ent_phred[e0:e1],
            read_ind=self.read_ind[r0:r1],
            recombcost=self.recombcost[lo:hi],
            n_ind=self.n_ind,
            trios=self.trios,
            distrust=self.distrust,
            gt=self.gt[:, lo:hi],
            gl=None if self.gl is None else self.gl[:, lo:hi],
        )


@dataclass
class FlatSolution:
    n_cols: int
    n_reads: int
    n_ind: int
    cost: int = 0
    path_index: np.ndarray = None
    path_tv: np.ndarray = None
    partition: np.ndarray = None
    sr_allele: np.ndarray = None   # [n_ind, 2, n_cols]
    sr_quality: np.ndarray = None  # [n_ind, n_cols]

    def __post_init__(self):
        n, m, i = self.n_cols, self.n_reads, self.n_ind
        self.path_index = np.zeros(n, np.uint32)
        self.path_tv = np.zeros(n, np.uint32)
        self.partition = np.zeros(m, np.uint8)
        self.sr_allele = np.zeros((i, 2, n), np.uint8)
        self.sr_quality = np.zeros((i, n), np.uint32)

    def as_c(self) -> CSolution:
        s = CSolution()
        s.cost = 0
        s.path_index = _ptr(self.path_index, C.c_uint32)
        s.path_tv = _ptr(self.path_tv, C.c_uint32)
        s.partition = _ptr(self.partition, C.c_uint8)
        s.sr_allele = _ptr(self.sr_allele, C.c_uint8)
        s.sr_quality = _ptr(self.sr_quality, C.c_uint32)
        return s

    def same_as(self, other: "FlatSolution") -> bool:
        return (
            self.cost == other.cost
            and np.array_equal(self.path_index, other.path_index)
            and np.array_equal(self.path_tv, other.path_tv)
            and np.array_equal(self.partition, other.partition)
            and np.array_equal(self.sr_allele, other.sr_allele)
            and np.array_equal(self.sr_quality, other.sr_quality)
        )

    def diff(self, other: "FlatSolution") -> str:
        out = []
        if self.cost != other.cost:
            out.append(f"cost {self.cost} != {other.cost}")
        for name in ("path_index", "path_tv", "partition", "sr_allele", "sr_quality"):
            a, b = getattr(self, name), getattr(other, name)
            if not np.array_equal(a, b):
                bad = np.argwhere(a != b)
                out.append(f"{name}: {len(bad)} mismatches, first at {bad[0].tolist()}: {a[tuple(bad[0])]} != {b[tuple(bad[0])]}")
        return "; ".join(out) or "identical"


class MendelianConflict(RuntimeError):
    """RuntimeError('Error: Mendelian conflict') — same text as pedigreedptable.cpp:302."""


class Unsupported(RuntimeError):
    """WHMEC_ERR_UNSUPPORTED: the problem is outside what this build handles (include/whmec.h)."""


def raise_for(rc: int, msg: str):
    """Map a C-ABI return code to the exception the reference would raise (cpp.pxd `except +`)."""
    if rc == WHMEC_OK:
        return
    if rc == WHMEC_ERR_MENDELIAN:
        raise MendelianConflict(msg or "Error: Mendelian conflict")
    if rc == WHMEC_ERR_INPUT:
        raise RuntimeError(msg or "invalid input")
    if rc == WHMEC_ERR_CUDA:
        raise RuntimeError(f"CUDA failure: {msg}")
    if rc == WHMEC_ERR_UNSUPPORTED:
        raise Unsupported(f"unsupported problem: {msg}")
    raise RuntimeError(f"whmec error {rc}: {msg}")


class CRealignInput(C.Structure):
    """whmec_realign_input: alignments, variants, restricted genotypes, reference and costs of one whmec_realign call."""
    _fields_ = [
        ("n_alignments", C.c_uint32),
        ("reference_start", C.POINTER(C.c_int32)),
        ("cigar_off", _u64p),
        ("cigar_op", _u8p),
        ("cigar_len", C.POINTER(C.c_int32)),
        ("query_off", _u64p),
        ("query", _u8p),
        ("n_variants", C.c_uint32),
        ("position", C.POINTER(C.c_int32)),
        ("allele_first", _u32p),
        ("allele_off", _u64p),
        ("allele_bytes", _u8p),
        ("restrict_off", _u64p),
        ("restrict_allele", C.POINTER(C.c_int32)),
        ("reference", _u8p),
        ("reference_len", C.c_uint64),
        ("overhang", C.c_int32),
        ("affine", C.c_int32),
        ("gap_start", C.c_int32),
        ("gap_extend", C.c_int32),
        ("mismatch", C.c_double),
    ]


class CRealignOutput(C.Structure):
    """whmec_realign_output: per alignment (CSR) the calls (variant index, allele, quality); the library owns the arrays."""
    _fields_ = [
        ("call_off", _u64p),
        ("variant", _u32p),
        ("allele", C.POINTER(C.c_int32)),
        ("quality", C.POINTER(C.c_int64)),
    ]


class CRealignStats(C.Structure):
    _fields_ = [
        ("items", C.c_uint64),
        ("jobs", C.c_uint64),
        ("short_jobs", C.c_uint64),
        ("long_jobs", C.c_uint64),
        ("long_items", C.c_uint64),
        ("cells", C.c_uint64),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
        ("chunks", C.c_uint32),
        ("kernel_launches", C.c_uint32),
        ("device_ms", C.c_float),
        ("plan_ms", C.c_float),
    ]

    def as_dict(self) -> dict:
        return {name: getattr(self, name) for name, _ in self._fields_}


class CQueryQualities(C.Structure):
    """whmec_query_qualities: per alignment (CSR) its query_qualities, and which alignments lack query_sequence or cigartuples."""
    _fields_ = [
        ("qual_off", _u64p),
        ("qual", _u8p),
        ("missing", _u8p),
    ]


class CKmerCosts(C.Structure):
    """whmec_kmer_costs: the sorted costs table of k-mer realignment, keys (ref k-mer << 32 | read k-mer, 0 for -5)."""
    _fields_ = [
        ("n", C.c_uint64),
        ("key", _u64p),
        ("cost", C.POINTER(C.c_float)),
    ]


class CKmeraldParams(C.Structure):
    """whmec_kmerald_params: k-mer size, gap penalty, window, costs and each variant's alternative_allele (CSR)."""
    _fields_ = [
        ("kmer_size", C.c_int32),
        ("gap_penalty", C.c_float),
        ("window", C.c_int32),
        ("costs", C.POINTER(CKmerCosts)),
        ("alt_off", _u64p),
        ("alt_bytes", _u8p),
        ("has_alt", _u8p),
    ]


class CLearnInput(C.Structure):
    """whmec_learn_input: reference, alignments, variant list and state, k, window and the popped columns of one whmec_learn call."""
    _fields_ = [
        ("reference", _u8p),
        ("reference_len", C.c_uint64),
        ("n_alignments", C.c_uint32),
        ("reference_start", C.POINTER(C.c_int32)),
        ("cigar_off", _u64p),
        ("cigar_op", _u8p),
        ("cigar_len", C.POINTER(C.c_int32)),
        ("query_off", _u64p),
        ("query", _u8p),
        ("n_variants", C.c_uint32),
        ("variant_pos", C.POINTER(C.c_int32)),
        ("variant_len", C.POINTER(C.c_int32)),
        ("first_variant", C.c_uint32),
        ("k", C.c_int32),
        ("window", C.c_int32),
        ("final", C.c_int32),
        ("col_lo", C.c_int64),
        ("col_hi", C.c_int64),
        ("floor", C.POINTER(C.c_int32)),
    ]


class CLearnOutput(C.Structure):
    """whmec_learn_output: rows [n_rows][4] (column, reference k-mer, read k-mer, count) and the variant list's next front."""
    _fields_ = [
        ("n_rows", C.c_uint64),
        ("rows", C.POINTER(C.c_int32)),
        ("next_variant", C.c_uint32),
    ]


class CLearnStats(C.Structure):
    _fields_ = [
        ("alignments", C.c_uint64),
        ("kmers", C.c_uint64),
        ("kept", C.c_uint64),
        ("distinct", C.c_uint64),
        ("rows", C.c_uint64),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
        ("chunks", C.c_uint32),
        ("kernel_launches", C.c_uint32),
        ("device_ms", C.c_float),
        ("plan_ms", C.c_float),
    ]

    def as_dict(self) -> dict:
        return {name: getattr(self, name) for name, _ in self._fields_}


class CHaplotagInput(C.Structure):
    """whmec_haplotag_input: every sample's phase table and reads (entries as CSR) of one whmec_haplotag call."""
    _fields_ = [
        ("n_samples", C.c_uint32),
        ("phase_off", _u64p),
        ("phase_pos", C.POINTER(C.c_int64)),
        ("phase_block", C.POINTER(C.c_int64)),
        ("allele_off", _u64p),
        ("allele", C.POINTER(C.c_int32)),
        ("n_reads", C.c_uint32),
        ("read_off", _u64p),
        ("entry_pos", C.POINTER(C.c_int64)),
        ("entry_allele", C.POINTER(C.c_int32)),
        ("entry_quality", C.POINTER(C.c_int32)),
        ("read_sample", C.POINTER(C.c_uint32)),
        ("read_repr", C.POINTER(C.c_int64)),
        ("read_bx", C.POINTER(C.c_int64)),
        ("reference_start", C.POINTER(C.c_int64)),
        ("ploidy", C.c_int64),
        ("linked_read_cutoff", C.c_int64),
    ]


class CHaplotagOutput(C.Structure):
    """whmec_haplotag_output: caller-allocated [n_reads] arrays and the first error."""
    _fields_ = [
        ("group", C.POINTER(C.c_int64)),
        ("n_blocks", C.POINTER(C.c_int32)),
        ("block", C.POINTER(C.c_int64)),
        ("haplotype", C.POINTER(C.c_int32)),
        ("quality", C.POINTER(C.c_int64)),
        ("error_kind", C.c_int32),
        ("error_read", C.c_int64),
        ("error_entry", C.c_int64),
    ]


class CHaplotagStats(C.Structure):
    _fields_ = [
        ("entries", C.c_uint64),
        ("groups", C.c_uint64),
        ("keys", C.c_uint64),
        ("runs", C.c_uint64),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
        ("chunks", C.c_uint32),
        ("kernel_launches", C.c_uint32),
        ("device_ms", C.c_float),
        ("plan_ms", C.c_float),
    ]

    def as_dict(self) -> dict:
        return {name: getattr(self, name) for name, _ in self._fields_}
