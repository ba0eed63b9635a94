"""Allele detection by re-alignment on the GPU, for many alignments in one call.

`detect_alleles` gives, per alignment, the list of (variant index, allele, quality) that WhatsHap's
`ReadSetReader.detect_alleles_by_alignment(variants, restricted_genotypes, 0, alignment, reference, overhang, use_affine,
gap_start, gap_extend, default_mismatch)` yields, in the same order (whatshap/variants.py:599-912): the host walks every CIGAR
against the variant list, the device aligns each covered variant's query window against its padded alleles
(`whmec_realign`, DESIGN §4.11).  `edit_distances` and `edit_distances_affine_gap` are `whatshap.align.edit_distance` and
`edit_distance_affine_gap` (with one mismatch cost for every query position) over many pairs.

With `use_kmerald=True` (`whatshap genotype --use-kmerald`), `detect_alleles` is detect_alleles_by_alignment(...,
use_kmerald=True, kmerald_costs, kmer_size, kmerald_gappenalty, kmerald_window): each query window (kmerald_window for the
overhang) and the padded reference and alternative alleles are cut into k-mers (`enumerate_all_kmers`) and aligned with
`kmer_align` in float32 on the device (`whmec_realign_kmerald`, DESIGN §4.12); the costs are a `KmerCosts` table, packed once
and reusable across calls.  `kmer_distances` is `kmer_align` over many pairs of strings.

With `reference=None` (`whatshap phase --no-reference`, `whatshap haplotag --no-reference`), `detect_alleles` is
_alignments_to_reads without a reference: per alignment, `_detect_alleles(normalized, var_progress, 0, alignment)`
(whatshap/_variants.pyx:84-298) over the normalized variants that `detect_non_overlapping_variants` keeps, reading the query
bases and `query_qualities` at the CIGAR's insertions, deletions and matches (`whmec_detect_alleles_cigar`, DESIGN §4.14); the
re-alignment and k-mer options are not used.  For alignments in non-decreasing `reference_start` order the reference's running
index gives the same answer as starting at 0.  Where that code raises (an operation outside 0..8, a base or quality index past the
end of the query, a missing query sequence or CIGAR, a variant without alternatives), the call raises ValueError naming the first
such alignment (or the variant) and the reference's exception.

Where the reference raises (an unknown CIGAR operation, a failed window assert, a restricted genotype that leaves no allele,
in k-mer mode a covered multiallelic variant, which has no `alternative_allele`), the call raises ValueError naming the first
such alignment and variant.  Inputs the reference would only reject later are rejected up front: affine mode without its three
costs, a negative overhang or window, a CIGAR without a query sequence, fewer restricted genotypes than variants, k-mer mode
without costs, a k-mer size outside 1..15.
"""
from __future__ import annotations

import csv
import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._abi import WHMEC_ERR_INPUT, CKmeraldParams, CKmerCosts, CQueryQualities, CRealignInput, CRealignOutput, CRealignStats, raise_for

Call = Tuple[int, int, int]


def _bytes(s) -> bytes:
    return s.encode() if isinstance(s, str) else bytes(s)


def _ptr(a: Optional[np.ndarray], ctype):
    return C.cast(None, C.POINTER(ctype)) if a is None else a.ctypes.data_as(C.POINTER(ctype))


def _csr(chunks: Sequence[bytes]) -> Tuple[np.ndarray, np.ndarray]:
    off = np.zeros(len(chunks) + 1, np.uint64)
    if chunks:
        np.cumsum(np.fromiter(map(len, chunks), np.uint64, len(chunks)), out=off[1:])
    buf = np.frombuffer(b"".join(chunks), np.uint8) if off[-1] else np.zeros(1, np.uint8)
    return off, buf


def _int32(values, what: str) -> np.ndarray:
    a = np.asarray(values, dtype=np.int64)
    if a.size and (a.min() < -(2**31) or a.max() >= 2**31):
        raise ValueError(f"{what} outside the 32-bit range of the reference's C ints")
    return a.astype(np.int32)


def pack_input(alignments, variants, reference, restricted_genotypes=None, overhang=10, affine=False, gap_start=None,
               gap_extend=None, default_mismatch=None):
    """(whmec_realign_input, the arrays it points into): the flat form of one detect_alleles call."""
    if overhang < 0:
        raise ValueError("overhang must be >= 0")
    if affine and (gap_start is None or gap_extend is None or default_mismatch is None):
        raise ValueError("affine realignment needs gap_start, gap_extend and default_mismatch")
    keep = []
    n = len(alignments)
    cigars = [a.cigartuples or () for a in alignments]
    queries = []
    for k, (a, cg) in enumerate(zip(alignments, cigars)):
        seq = a.query_sequence
        if seq is None and cg:
            raise ValueError(f"alignment {k} has a CIGAR but no query sequence")
        queries.append(_bytes(seq) if seq is not None else b"")
    starts = _int32([a.reference_start for a in alignments], "reference_start")
    cigar_off = np.zeros(n + 1, np.uint64)
    if n:
        np.cumsum(np.fromiter(map(len, cigars), np.uint64, n), out=cigar_off[1:])
    flat = np.array([x for cg in cigars for x in cg], dtype=np.int64).reshape(-1, 2)
    ops = flat[:, 0]
    cigar_op = np.where((ops >= 0) & (ops <= 254), ops, 255).astype(np.uint8)
    cigar_len = _int32(flat[:, 1], "CIGAR length")
    query_off, query = _csr(queries)
    positions = _int32([v.position for v in variants], "variant position")
    alleles, first = [], [0]
    for v in variants:
        alleles.append(_bytes(v.reference_allele))
        alleles.extend(_bytes(x) for x in v.get_alt_allele_list())
        first.append(len(alleles))
    allele_first = np.array(first, np.uint32)
    allele_off, allele_bytes = _csr(alleles)
    r_off = r_all = None
    if restricted_genotypes:
        if len(restricted_genotypes) < len(variants):
            raise ValueError("restricted_genotypes has fewer entries than variants")
        vecs = [list(restricted_genotypes[i].as_vector()) for i in range(len(variants))]
        r_off = np.zeros(len(vecs) + 1, np.uint64)
        if vecs:
            np.cumsum(np.fromiter(map(len, vecs), np.uint64, len(vecs)), out=r_off[1:])
        r_all = np.clip(np.array([x for g in vecs for x in g] or [0], np.int64), -1, 2**31 - 1).astype(np.int32)
    ref = np.frombuffer(_bytes(reference), np.uint8) if len(reference) else np.zeros(1, np.uint8)
    keep += [starts, cigar_off, cigar_op, cigar_len, query_off, query, positions, allele_first, allele_off, allele_bytes, r_off, r_all, ref]
    ci = CRealignInput(
        n, _ptr(starts, C.c_int32), _ptr(cigar_off, C.c_uint64), _ptr(cigar_op, C.c_uint8), _ptr(cigar_len, C.c_int32),
        _ptr(query_off, C.c_uint64), _ptr(query, C.c_uint8), len(variants), _ptr(positions, C.c_int32), _ptr(allele_first, C.c_uint32),
        _ptr(allele_off, C.c_uint64), _ptr(allele_bytes, C.c_uint8), _ptr(r_off, C.c_uint64), _ptr(r_all, C.c_int32),
        _ptr(ref, C.c_uint8), len(reference), int(overhang), int(bool(affine)),
        int(gap_start) if affine else 0, int(gap_extend) if affine else 0, float(default_mismatch) if affine else 0.0)
    return ci, keep


def pack_cigar_input(alignments, variants):
    """(whmec_realign_input, whmec_query_qualities, the arrays they point into) of one detect_alleles call without a reference."""
    n = len(alignments)
    cigars, queries, quals = [], [], []
    missing = np.zeros(max(n, 1), np.uint8)
    for k, a in enumerate(alignments):
        cg, seq, qq = a.cigartuples, a.query_sequence, getattr(a, "query_qualities", None)
        missing[k] = (seq is None) | (cg is None) << 1
        cigars.append(cg or ())
        queries.append(_bytes(seq) if seq is not None else b"")
        quals.append(bytes(qq) if qq is not None and len(qq) else b"")
    starts = _int32([a.reference_start for a in alignments], "reference_start")
    cigar_off = np.zeros(n + 1, np.uint64)
    if n:
        np.cumsum(np.fromiter(map(len, cigars), np.uint64, n), out=cigar_off[1:])
    flat = np.array([x for cg in cigars for x in cg], dtype=np.int64).reshape(-1, 2)
    ops = flat[:, 0]
    cigar_op = np.where((ops >= 0) & (ops <= 254), ops, 255).astype(np.uint8)
    cigar_len = _int32(flat[:, 1], "CIGAR length")
    query_off, query = _csr(queries)
    qual_off, qual = _csr(quals)
    positions = _int32([v.position for v in variants], "variant position")
    alleles, first = [], [0]
    for v in variants:
        alleles.append(_bytes(v.reference_allele))
        alleles.extend(_bytes(x) for x in v.get_alt_allele_list())
        first.append(len(alleles))
    allele_first = np.array(first, np.uint32)
    allele_off, allele_bytes = _csr(alleles)
    keep = [starts, cigar_off, cigar_op, cigar_len, query_off, query, qual_off, qual, missing, positions, allele_first, allele_off, allele_bytes]
    none8 = C.cast(None, C.POINTER(C.c_uint8))
    ci = CRealignInput(
        n, _ptr(starts, C.c_int32), _ptr(cigar_off, C.c_uint64), _ptr(cigar_op, C.c_uint8), _ptr(cigar_len, C.c_int32),
        _ptr(query_off, C.c_uint64), _ptr(query, C.c_uint8), len(variants), _ptr(positions, C.c_int32), _ptr(allele_first, C.c_uint32),
        _ptr(allele_off, C.c_uint64), _ptr(allele_bytes, C.c_uint8), C.cast(None, C.POINTER(C.c_uint64)), C.cast(None, C.POINTER(C.c_int32)),
        none8, 0, 0, 0, 0, 0, 0.0)
    cq = CQueryQualities(_ptr(qual_off, C.c_uint64), _ptr(qual, C.c_uint8), _ptr(missing, C.c_uint8))
    return ci, cq, keep


def _calls(L, out, n):
    """The per-alignment call lists of a filled whmec_realign_output, which is released."""
    try:
        off = np.ctypeslib.as_array(out.call_off, (n + 1,)).copy()
        total = int(off[-1])
        if total:
            var = np.ctypeslib.as_array(out.variant, (total,)).tolist()
            al = np.ctypeslib.as_array(out.allele, (total,)).tolist()
            ql = np.ctypeslib.as_array(out.quality, (total,)).tolist()
        else:
            var = al = ql = []
    finally:
        L.whmec_realign_release(C.byref(out))
    calls = list(zip(var, al, ql))
    return [calls[off[k]:off[k + 1]] for k in range(n)]


def _detect_alleles_cigar(alignments, variants, device, stats, library):
    L = library or _lib.lib()
    ci, cq, keep = pack_cigar_input(alignments, variants)
    out, st = CRealignOutput(), CRealignStats()
    err = C.create_string_buffer(1024)
    rc = L.whmec_detect_alleles_cigar(C.byref(ci), C.byref(cq), device, C.byref(out), C.byref(st), err, len(err))
    del keep
    if rc == WHMEC_ERR_INPUT:
        raise ValueError(err.value.decode())
    raise_for(rc, err.value.decode())
    calls = _calls(L, out, len(alignments))
    if stats is not None:
        stats.update(st.as_dict())
    return calls


_KMER_MAX = 2**30  # k-mers of k <= 15 lie in 1 .. 2^30 - 1


def _integral(x):
    try:
        i = int(x)
    except (TypeError, ValueError, OverflowError):
        return None
    return i if i == x else None


class KmerCosts:
    """The costs of `kmer_align`: {(ref k-mer, read k-mer): cost}, with read k-mer -5 for a ref k-mer's default, packed once
    into the sorted table the device searches (keys ref << 32 | read, -5 as 0; costs as float32 of float(value)).  One table
    serves any number of calls.  Keys no k-mer can ever look up are dropped; a value float() rejects raises ValueError."""

    def __init__(self, mapping):
        keys, values = [], []
        for key, value in mapping.items():
            try:
                v = float(value)
            except (TypeError, ValueError) as e:
                raise ValueError(f"kmer costs: the value {value!r} of {key!r} is not a number float() accepts") from e
            try:
                a, b = key
            except (TypeError, ValueError):
                continue
            a, b = _integral(a), _integral(b)
            if a is None or not 1 <= a < _KMER_MAX or b is None:
                continue
            if b == -5:
                b = 0
            elif not 1 <= b < _KMER_MAX:
                continue
            keys.append((a << 32) | b)
            values.append(v)
        key = np.array(keys, np.uint64)
        with np.errstate(over="ignore"):
            cost = np.array(values, np.float64).astype(np.float32)
        order = np.argsort(key, kind="stable")
        self.key, self.cost = np.ascontiguousarray(key[order]), np.ascontiguousarray(cost[order])
        self._c = CKmerCosts(len(self.key), _ptr(self.key if len(self.key) else None, C.c_uint64),
                             _ptr(self.cost if len(self.cost) else None, C.c_float))

    @classmethod
    def read(cls, path) -> "KmerCosts":
        """The costs file as `_alignments_to_reads` reads it: tab-separated `ref k-mer, read k-mer, cost`, the last of repeated
        keys kept."""
        costs = {}
        with open(path) as f:
            for line in csv.reader(f, delimiter="\t"):
                costs[(int(line[0]), int(line[1]))] = line[2]
        return cls(costs)

    def __len__(self) -> int:
        return len(self.key)


def _kmerald_params(costs, kmer_size, gap_penalty, window, variants=None):
    """(whmec_kmerald_params, the objects it points into)."""
    if costs is None:
        raise ValueError("k-mer realignment needs kmerald_costs")
    if not isinstance(costs, KmerCosts):
        costs = KmerCosts(costs)
    k = int(kmer_size)
    if not 1 <= k <= 15:
        raise ValueError("kmer_size must lie in 1..15")
    if window < 0:
        raise ValueError("kmerald_window must be >= 0")
    keep = [costs]
    alt_off = alt = has = None
    if variants is not None:
        alts = [getattr(v, "alternative_allele", None) for v in variants]
        has = np.array([a is not None for a in alts] or [0], np.uint8)
        alt_off, alt = _csr([_bytes(a) if a is not None else b"" for a in alts])
        keep += [alt_off, alt, has]
    params = CKmeraldParams(k, float(gap_penalty), int(window), C.pointer(costs._c), _ptr(alt_off, C.c_uint64), _ptr(alt, C.c_uint8),
                            _ptr(has, C.c_uint8))
    return params, keep


def detect_alleles(alignments, variants, reference, *, restricted_genotypes=None, overhang: int = 10, affine: bool = False,
                   gap_start=None, gap_extend=None, default_mismatch=None, use_kmerald: bool = False, kmerald_costs=None,
                   kmer_size: int = 7, kmerald_gappenalty=40, kmerald_window=25, device: int = 0, stats: Optional[dict] = None,
                   library: Optional[C.CDLL] = None) -> List[List[Call]]:
    """Per alignment, the (variant index, allele, quality) tuples of detect_alleles_by_alignment, in its order.

    alignments: objects with `reference_start`, `cigartuples` and `query_sequence` (a pysam.AlignedSegment qualifies);
    variants: objects with `position`, `reference_allele` and `get_alt_allele_list()` (and, for k-mer mode,
    `alternative_allele`); reference: the chromosome (str or bytes); restricted_genotypes: None or one object with
    `as_vector()` per variant.  use_kmerald: k-mer realignment with kmerald_costs (a `KmerCosts` or the dict `kmer_align`
    takes), kmer_size, kmerald_gappenalty and int(kmerald_window); overhang, affine, its costs and the restricted genotypes
    are then not used.  reference=None: detection from the CIGAR alone (`--no-reference`), reading `query_qualities` where the
    alignment has it; every re-alignment and k-mer option is then not used.  `stats` (a dict) receives the call's counters: items, jobs, short_jobs / long_jobs (one thread / one
    warp per allele alignment), chunks, device_ms.  `library`: another build of the library with the same entry point (tests)."""
    if reference is None:
        return _detect_alleles_cigar(alignments, variants, device, stats, library)
    L = library or _lib.lib()
    if use_kmerald:
        window = int(kmerald_window)
        params, kkeep = _kmerald_params(kmerald_costs, kmer_size, kmerald_gappenalty, window, variants)
        if restricted_genotypes and len(restricted_genotypes) < len(variants):
            raise ValueError("restricted_genotypes has fewer entries than variants")
        ci, keep = pack_input(alignments, variants, reference)
        keep += kkeep
    else:
        ci, keep = pack_input(alignments, variants, reference, restricted_genotypes, overhang, affine, gap_start, gap_extend, default_mismatch)
    out, st = CRealignOutput(), CRealignStats()
    err = C.create_string_buffer(1024)
    if use_kmerald:
        rc = L.whmec_realign_kmerald(C.byref(ci), C.byref(params), device, C.byref(out), C.byref(st), err, len(err))
    else:
        rc = L.whmec_realign(C.byref(ci), device, C.byref(out), C.byref(st), err, len(err))
    if rc == WHMEC_ERR_INPUT:
        raise ValueError(err.value.decode())
    raise_for(rc, err.value.decode())
    calls = _calls(L, out, len(alignments))
    del keep
    if stats is not None:
        stats.update(st.as_dict())
    return calls


def _pairs(queries, targets, mismatch, gap_start, gap_extend, affine, device, stats, library):
    if len(queries) != len(targets):
        raise ValueError("queries and targets differ in length")
    L = library or _lib.lib()
    n = len(queries)
    q_off, q = _csr([_bytes(s) for s in queries])
    t_off, t = _csr([_bytes(s) for s in targets])
    res = np.zeros(max(n, 1), np.int64)
    st = CRealignStats()
    err = C.create_string_buffer(512)
    i64 = C.POINTER(C.c_int64)
    dst = res.ctypes.data_as(i64)
    none = C.cast(None, i64)
    rc = L.whmec_edit_distance_batch(n, _ptr(q_off, C.c_uint64), _ptr(q, C.c_uint8), _ptr(t_off, C.c_uint64), _ptr(t, C.c_uint8),
                                     float(mismatch), int(gap_start), int(gap_extend), none if affine else dst, dst if affine else none,
                                     device, C.byref(st), err, len(err))
    if rc == WHMEC_ERR_INPUT:
        raise ValueError(err.value.decode())
    raise_for(rc, err.value.decode())
    if stats is not None:
        stats.update(st.as_dict())
    return res[:n]


def edit_distances(queries, targets, *, device: int = 0, stats: Optional[dict] = None, library: Optional[C.CDLL] = None) -> np.ndarray:
    """edit_distance(queries[i], targets[i]) (unit costs, align.pyx:16-109) for every i, as int64."""
    return _pairs(queries, targets, 0.0, 0, 0, False, device, stats, library)


def edit_distances_affine_gap(queries, targets, mismatch, gap_start: int = 1, gap_extend: int = 1, *, device: int = 0,
                              stats: Optional[dict] = None, library: Optional[C.CDLL] = None) -> np.ndarray:
    """int(edit_distance_affine_gap(queries[i], targets[i], [mismatch] * len(queries[i]), gap_start, gap_extend)) for every i
    (align.pyx:114-196): the float32 Gotoh recurrence, mismatch as a float32, gap costs as C ints (10.9 -> 10)."""
    return _pairs(queries, targets, mismatch, int(gap_start), int(gap_extend), True, device, stats, library)


def kmer_distances(seqs1, seqs2, costs, gap_penalty=40, kmer_size: int = 7, *, device: int = 0, stats: Optional[dict] = None,
                   library: Optional[C.CDLL] = None) -> np.ndarray:
    """kmer_align(enumerate_all_kmers(seqs1[i], kmer_size), enumerate_all_kmers(seqs2[i], kmer_size), costs, gap_penalty) for
    every i (align.pyx:199-271), as float32; seqs1 are the rows (the reference's alleles), seqs2 the columns (the reads)."""
    if len(seqs1) != len(seqs2):
        raise ValueError("seqs1 and seqs2 differ in length")
    params, keep = _kmerald_params(costs, kmer_size, gap_penalty, 0)
    L = library or _lib.lib()
    n = len(seqs1)
    off1, s1 = _csr([_bytes(s) for s in seqs1])
    off2, s2 = _csr([_bytes(s) for s in seqs2])
    res = np.zeros(max(n, 1), np.float32)
    st = CRealignStats()
    err = C.create_string_buffer(512)
    rc = L.whmec_kmer_align_batch(n, _ptr(off1, C.c_uint64), _ptr(s1, C.c_uint8), _ptr(off2, C.c_uint64), _ptr(s2, C.c_uint8), C.byref(params),
                                  res.ctypes.data_as(C.POINTER(C.c_float)), device, C.byref(st), err, len(err))
    del keep
    if rc == WHMEC_ERR_INPUT:
        raise ValueError(err.value.decode())
    raise_for(rc, err.value.decode())
    if stats is not None:
        stats.update(st.as_dict())
    return res[:n]
