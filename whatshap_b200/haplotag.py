"""Read assignment of `whatshap haplotag` on the GPU.

`prepare_haplotag_information` has the signature and the four results of the reference's function in
`whatshap/cli/haplotag.py`, and `assign_reads` is the array-level call beneath it (`whmec_haplotag`, DESIGN §4.15).  Per
sample, the host walks the reads into groups (a read and the unprocessed reads of its BX tag within `linked_read_cutoff`);
the device sums the qualities of every (group, phase set, haplotype) with a radix sort and picks each group's phase set and
haplotype.

One order is defined where the reference has none: it keeps a group's reads in a set of identity-hashed objects, so the phase
set that a multi-read group's first vote enters first, which decides between phase sets with the same top score, can change
from run to run.  Here a group is visited as its opening read, then its linked reads in ReadSet order, each read's entries in
its own order.

Where the reference raises, the same exception type is raised, for the first offending entry in that order:
AssertionError for an allele other than 0 or 1, KeyError for a position without phase, IndexError for a matching haplotype
index at or beyond `ploidy` (or `ploidy` below 2 when a group has a phase set).  Qualities must fit in int32 (ValueError).
"""
from __future__ import annotations

import ctypes as C
from collections import defaultdict
from dataclasses import dataclass
from typing import NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._abi import WHMEC_ERR_INPUT, CHaplotagInput, CHaplotagOutput, CHaplotagStats, raise_for

#: the sub-alignment id of a primary alignment (whatshap.variants.PRIMARY_DEFAULT_SUB_ALIGNMENT_ID)
PRIMARY_DEFAULT_SUB_ALIGNMENT_ID = "____1"

_INT32 = (-(1 << 31), (1 << 31) - 1)


@dataclass(frozen=True)
class ReadAlignmentRepresentation:
    read_name: str
    chromosome: str
    is_supplementary: bool
    sub_alignment_id: str


@dataclass(frozen=True)
class PrimaryInfo:
    reference_start: int
    reference_end: int
    is_reverse: bool


def representation(name: str, chromosome: str, is_supplementary: bool, sub_alignment_id: str, as_primary: bool = False) -> tuple:
    """The fields of the reference's `read_representation` as a tuple.  The name loses as many characters as the read's own
    sub-alignment id has whenever it ends with the id in use, so an empty id turns every name into ''."""
    sub = PRIMARY_DEFAULT_SUB_ALIGNMENT_ID if as_primary else sub_alignment_id
    if name.endswith(sub):
        name = name[: -len(sub_alignment_id)]
    return name, chromosome, False if as_primary else bool(is_supplementary), sub


class _Reads:
    """One ReadSet's reads as columns: entries as CSR, and per read its metadata."""

    def __init__(self, readset):
        from .core import ReadSet

        if isinstance(readset, ReadSet):
            lens, _, self.pos, self.allele, self.quality = readset._flat_columns()
            self.off = np.zeros(len(lens) + 1, np.int64)
            np.cumsum(lens, out=self.off[1:])
            reads = readset._reads
            self.meta = [(r._name, r._chromosome, r._is_supplementary, r._sub_alignment_id, r._BX_tag, r._reference_start,
                          r._reference_end, r._is_reverse) for r in reads]
        else:  # the reference's whatshap.core.ReadSet (or any object with its Read interface)
            from .adapters import _readset_to_csr

            self.off, self.pos, self.allele, self.quality, _, _ = _readset_to_csr(readset)
            self.meta = [(r.name, r.chromosome, bool(r.is_supplementary), r.sub_alignment_id, r.BX_tag if r.has_BX_tag() else "",
                          int(r.reference_start), int(r.reference_end), bool(r.is_reverse)) for r in readset]


class Assignment(NamedTuple):
    """Per read of all samples, in order: the group's opening read (-1 for a skipped read), and at opening reads the number
    of phase sets, the chosen phase set, the haplotype (-1: not tagged) and the quality.  sample_off[s] is sample s's first
    read; reprs holds every read's representation fields."""
    group: np.ndarray
    n_blocks: np.ndarray
    block: np.ndarray
    haplotype: np.ndarray
    quality: np.ndarray
    sample_off: np.ndarray
    reprs: list


def _phase_arrays(tables):
    """tables: per sample {position: (block id, phase tuple)} -> phase_off, positions, blocks, allele_off, alleles."""
    offs, pos, blocks, lens, alleles = [0], [], [], [], []
    for table in tables:
        for p in sorted(table):
            block, phase = table[p]
            pos.append(int(p))
            blocks.append(int(block))
            lens.append(len(phase))
            alleles.extend(int(a) if isinstance(a, (int, np.integer)) and _INT32[0] <= a <= _INT32[1] else -1 for a in phase)
        offs.append(len(pos))
    allele_off = np.zeros(len(lens) + 1, np.uint64)
    np.cumsum(np.array(lens, np.uint64), out=allele_off[1:])
    return (np.array(offs, np.uint64), np.array(pos, np.int64), np.array(blocks, np.int64), allele_off, np.array(alleles, np.int32))


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None and len(a) else None


def _assign(columns: Sequence[_Reads], tables, ploidy, ignore_linked_read, linked_read_cutoff, device, stats, library) -> Assignment:
    L = library or _lib.lib()
    n = sum(len(c.meta) for c in columns)
    sample_off = np.zeros(len(columns) + 1, np.int64)
    np.cumsum([len(c.meta) for c in columns], out=sample_off[1:])
    read_off = np.zeros(n + 1, np.uint64)
    if n:
        np.cumsum(np.concatenate([np.diff(c.off) for c in columns]).astype(np.uint64), out=read_off[1:])
    cat = lambda name: np.concatenate([getattr(c, name) for c in columns]) if columns else np.zeros(0, np.int64)
    pos, allele, quality = cat("pos").astype(np.int64), cat("allele"), cat("quality")
    if len(quality) and (quality.min() < _INT32[0] or quality.max() > _INT32[1]):
        raise ValueError("an entry quality lies outside int32")
    allele = np.where((allele >= _INT32[0]) & (allele <= _INT32[1]), allele, -1).astype(np.int32)
    quality = quality.astype(np.int32)
    read_sample = np.repeat(np.arange(len(columns), dtype=np.uint32), np.diff(sample_off))
    reprs, ids, bx_ids = [], {}, {}
    read_repr = np.empty(n, np.int64)
    read_bx = np.full(n, -1, np.int64)
    starts = np.empty(n, np.int64)
    i = 0
    for c in columns:
        for name, chrom, supp, sub, bx, start, _, _ in c.meta:
            key = representation(name, chrom, supp, sub)
            reprs.append(key)
            read_repr[i] = ids.setdefault(key, len(ids))
            if bx and not ignore_linked_read:
                read_bx[i] = bx_ids.setdefault(bx, len(bx_ids))
            starts[i] = start
            i += 1
    phase_off, ppos, pblock, allele_off, palleles = _phase_arrays(tables)
    out_arrays = (np.empty(n, np.int64), np.empty(n, np.int32), np.empty(n, np.int64), np.empty(n, np.int32), np.empty(n, np.int64))
    ci = CHaplotagInput(
        len(columns), _p(phase_off, C.c_uint64), _p(ppos, C.c_int64), _p(pblock, C.c_int64), _p(allele_off, C.c_uint64),
        _p(palleles, C.c_int32), n, _p(read_off, C.c_uint64), _p(pos, C.c_int64), _p(allele, C.c_int32), _p(quality, C.c_int32),
        _p(read_sample, C.c_uint32), _p(read_repr, C.c_int64), _p(read_bx, C.c_int64), _p(starts, C.c_int64), int(ploidy),
        int(linked_read_cutoff))
    out = CHaplotagOutput(*(_p(a, t) for a, t in zip(out_arrays, (C.c_int64, C.c_int32, C.c_int64, C.c_int32, C.c_int64))))
    st = CHaplotagStats()
    err = C.create_string_buffer(1024)
    rc = L.whmec_haplotag(C.byref(ci), device, C.byref(out), C.byref(st), err, len(err))
    if rc == WHMEC_ERR_INPUT:
        raise ValueError(err.value.decode())
    raise_for(rc, err.value.decode())
    if stats is not None:
        stats.update(st.as_dict())
    if out.error_kind:
        r, e = int(out.error_read), int(out.error_entry)
        s = int(np.searchsorted(sample_off, r, side="right") - 1)
        where = f"read {reprs[r][0]!r} of sample {s}"
        if out.error_kind == 1:
            raise AssertionError(f"{where}: entry {e} has an allele other than 0 or 1")
        if out.error_kind == 2:
            raise KeyError(int(pos[int(read_off[r]) + e]))
        if e < 0:
            raise IndexError(f"{where}: ploidy {ploidy} has no second-best haplotype")
        raise IndexError(f"{where}: entry {e} matches a haplotype index at or beyond ploidy {ploidy}")
    return Assignment(*out_arrays, sample_off, reprs)


def assign_reads(samples, ploidy: int, *, ignore_linked_read: bool = False, linked_read_cutoff: int = 50000, device: int = 0,
                 stats: Optional[dict] = None, library: Optional[C.CDLL] = None) -> Assignment:
    """Groups and haplotype choices of the reads of every (ReadSet, phase table) in `samples`, in one call.  A phase table maps a
    position to (block id, phase tuple), as the reference's `get_variant_information` builds it.  `stats` (a dict) receives
    the call's counters: entries, groups, keys, runs, h2d_bytes, d2h_bytes, chunks, kernel_launches, device_ms, plan_ms.
    `library`: another build of the library with the same entry point (tests)."""
    samples = list(samples)
    return _assign([_Reads(rs) for rs, _ in samples], [t for _, t in samples], ploidy, ignore_linked_read, linked_read_cutoff, device,
                   stats, library)


def variant_information(variant_table, sample) -> Tuple[dict, list]:
    """(position -> (block id, phase tuple), heterozygous variants) of a sample's phased records; the later of two records at
    a position wins."""
    table, variants = {}, []
    for v, gt, phase in zip(variant_table.variants, variant_table.genotypes_of(sample), variant_table.phases_of(sample)):
        if phase is None or phase.block_id is None:
            continue
        table[v.position] = (int(phase.block_id), phase.phase)
        if not gt.is_homozygous():
            variants.append(v)
    return table, variants


def _prepare(repr_cls, info_cls, variant_table, shared_samples, phased_input_reader, regions, ignore_linked_read, linked_read_cutoff,
             ploidy, device=0, stats=None, library=None):
    tables, columns = [], []
    for sample in shared_samples:
        table, variants = variant_information(variant_table, sample)
        read_set, _ = phased_input_reader.read(variant_table.chromosome, variants, sample, regions=regions)
        tables.append(table)
        columns.append(_Reads(read_set))
    a = _assign(columns, tables, ploidy, ignore_linked_read, linked_read_cutoff, device, stats, library)
    bx_to_haplotype = defaultdict(list)
    read_to_haplotype, primary_info_by_repr = {}, {}
    n_multiple_phase_sets = 0
    group, n_blocks, block, haplotype, quality = (x.tolist() for x in (a.group, a.n_blocks, a.block, a.haplotype, a.quality))
    order = np.argsort(a.group, kind="stable").tolist()  # members by group, each group's in read order
    first = {}
    for j, r in enumerate(order):
        if group[r] >= 0:
            first.setdefault(group[r], j)
    reprs = [repr_cls(*k) for k in a.reprs]
    for s, c in enumerate(columns):
        base = int(a.sample_off[s])
        for name, chrom, supp, sub, _, start, end, rev in c.meta:
            if not supp:
                primary_info_by_repr[repr_cls(*representation(name, chrom, supp, sub, as_primary=True))] = info_cls(start, end, rev)
        for i, (_, _, _, _, bx, start, _, _) in enumerate(c.meta):
            r = base + i
            if group[r] != r or not n_blocks[r]:
                continue
            if n_blocks[r] > 1:
                n_multiple_phase_sets += 1
            if haplotype[r] < 0:
                continue
            value = (haplotype[r], quality[r], block[r])
            if not ignore_linked_read and bx:
                bx_to_haplotype[bx].append((start, haplotype[r], block[r]))
            j = first[r]
            while j < len(order) and group[order[j]] == r:
                read_to_haplotype[reprs[order[j]]] = value
                j += 1
    return bx_to_haplotype, read_to_haplotype, n_multiple_phase_sets, primary_info_by_repr


def prepare_haplotag_information(variant_table, shared_samples, phased_input_reader, regions, ignore_linked_read, linked_read_cutoff,
                                 ploidy, supplementary_strategy=None, *, device: int = 0, stats: Optional[dict] = None,
                                 library: Optional[C.CDLL] = None):
    """(BX tag -> [(reference_start, haplotype, phase set)] as a defaultdict(list), ReadAlignmentRepresentation -> (haplotype,
    quality, phase set), the number of groups with several phase sets, ReadAlignmentRepresentation -> PrimaryInfo) as the
    reference's function returns them, with one device call for all samples.  supplementary_strategy is accepted and, as in the
    reference, unused."""
    return _prepare(ReadAlignmentRepresentation, PrimaryInfo, variant_table, shared_samples, phased_input_reader, regions,
                    ignore_linked_read, linked_read_cutoff, ploidy, device, stats, library)
