"""Read merging of `whatshap phase --merge-reads` on the GPU.

`ReadMerger` has the constructor and the `merge` of the reference's class in `whatshap/merge.py`, and `merge_reads` is the
array-level call beneath it (`whmec_merge_reads`, DESIGN §4.17).  Read j is compared with every later read i it still overlaps
in the reference's sliding queue (end_j = begin_j + number of entries > begin_k for every k in (j, i]); the device counts the
matches and mismatches of each pair from bit-packed alleles and joins the reads of each blue component.  Where not-blue edges
can exist (thr_diff + thr_neg_diff <= 0), the blue edges come back to the host, which removes edges as the reference does
with networkx's bidirectional BFS.  A component of two reads or more becomes one read named after its least member: per
position the qualities of each allele summed, allele 0 when z0 >= z1, quality |z1 - z0|, positions ascending.

Errors are the reference's: ValueError or ZeroDivisionError from the thresholds, then per readset IndexError for an empty read
or AssertionError for an allele other than 0 or 1, the first offending read deciding.  Positions and qualities must fit in int32
(the reference's Read holds C ints); others are refused with ValueError.
"""
from __future__ import annotations

import ctypes as C
import logging
from abc import ABC, abstractmethod
from array import array
from math import log
from typing import NamedTuple, Optional, Sequence

import numpy as np

from . import _lib
from ._abi import WHMEC_ERR_INPUT, CMergeInput, CMergeOutput, CMergeStats, raise_for

logger = logging.getLogger(__name__)

_INT32 = (-(1 << 31), (1 << 31) - 1)
_CLAMP = 1 << 62  # beyond any count of matches: thresholds past it decide the same


class Merged(NamedTuple):
    """One readset merged: the output reads as the input read each stands for (a singleton or a component's least member, in
    input order) with their entries as CSR, and the representative of every input read (itself for a singleton)."""
    read: np.ndarray
    entry_off: np.ndarray
    position: np.ndarray
    allele: np.ndarray
    quality: np.ndarray
    representative: np.ndarray


def thresholds(error_rate, positive_threshold, negative_threshold):
    """(thr_diff, thr_neg_diff) as the reference computes them, raising its errors (ValueError, ZeroDivisionError)."""
    base = (1 - error_rate) / (error_rate / 3)
    return 1 + int(log(positive_threshold, base)), 1 + int(log(negative_threshold, base))


def _columns(readset):
    """(read_off, position, allele, quality) of this package's ReadSet or any ReadSet-like object."""
    from .core import ReadSet

    if isinstance(readset, ReadSet):
        lens, _, pos, allele, quality = readset._flat_columns()
        off = np.zeros(len(lens) + 1, np.int64)
        np.cumsum(lens, out=off[1:])
        return off, pos, allele, quality
    from .adapters import _bridge_for, _readset_to_csr

    off, pos, allele, quality, _, _ = _readset_to_csr(readset)
    if _bridge_for(readset) is not None:  # the bridge hands the C ints of the qualities over as uint32
        quality = quality.astype(np.uint32).view(np.int32).astype(np.int64)
    return off, pos, allele, quality


def _int32(values, what):
    if len(values) and (values.min() < _INT32[0] or values.max() > _INT32[1]):
        raise ValueError(f"an entry {what} lies outside int32")
    return values.astype(np.int32)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None and len(a) else None


def merge_reads(readsets: Sequence, error_rate=0.15, max_error_rate=0.25, positive_threshold=1000000, negative_threshold=1000, *,
                device: int = 0, stats: Optional[dict] = None, library=None) -> list:
    """Merge every readset of `readsets` in one call; returns one `Merged` per readset.  Raises the reference's exception for
    the first readset that has an offending read."""
    thr_diff, thr_neg_diff = thresholds(error_rate, positive_threshold, negative_threshold)
    cols = [_columns(rs) for rs in readsets]
    n_reads = [len(c[0]) - 1 for c in cols]
    set_off = np.zeros(len(cols) + 1, np.uint64)
    np.cumsum(np.array(n_reads, np.uint64), out=set_off[1:])
    read_off = np.zeros(int(set_off[-1]) + 1, np.uint64)
    if int(set_off[-1]):
        np.cumsum(np.concatenate([np.diff(c[0]) for c in cols]).astype(np.uint64), out=read_off[1:])
    cat = lambda k: np.concatenate([np.asarray(c[k], np.int64) for c in cols]) if cols else np.zeros(0, np.int64)
    position, quality = _int32(cat(1), "position"), _int32(cat(3), "quality")
    allele = cat(2)
    allele = np.where((allele < 0) | (allele > 1), 2, allele).astype(np.uint8)
    ci = CMergeInput(len(cols), set_off.ctypes.data_as(C.POINTER(C.c_uint64)), read_off.ctypes.data_as(C.POINTER(C.c_uint64)),
                     _p(position, C.c_int32), _p(allele, C.c_uint8), _p(quality, C.c_int32),
                     max(-_CLAMP, min(_CLAMP, thr_diff)), max(-_CLAMP, min(_CLAMP, thr_neg_diff)), float(max_error_rate))
    ns = max(len(cols), 1)
    error_kind, error_read = np.zeros(ns, np.int32), np.zeros(ns, np.uint64)
    representative = np.zeros(max(int(set_off[-1]), 1), np.int64)
    out_off = np.zeros(len(cols) + 1, np.uint64)
    out = CMergeOutput(_p(error_kind, C.c_int32), _p(error_read, C.c_uint64), _p(representative, C.c_int64),
                       out_off.ctypes.data_as(C.POINTER(C.c_uint64)))
    st = CMergeStats()
    err = C.create_string_buffer(1024)
    L = library or _lib.lib()
    rc = L.whmec_merge_reads(C.byref(ci), device, C.byref(out), C.byref(st), err, len(err))
    if rc == WHMEC_ERR_INPUT:
        raise ValueError(err.value.decode())
    raise_for(rc, err.value.decode())
    try:
        n = int(out.n_out)
        arr = lambda ptr, count, dt: np.ctypeslib.as_array(ptr, (count,)).astype(dt, copy=True) if count else np.zeros(0, dt)
        read = arr(out.out_read, n, np.int64)
        entry_off = arr(out.out_entry_off, n + 1, np.int64)
        ne = int(entry_off[-1])
        pos, al, q = arr(out.out_position, ne, np.int64), arr(out.out_allele, ne, np.int64), arr(out.out_quality, ne, np.int64)
    finally:
        L.whmec_merge_reads_release(C.byref(out))
    if stats is not None:
        stats.update(st.as_dict())
    for s in range(len(cols)):
        if error_kind[s]:
            raise (IndexError("Index out of bounds: 0") if error_kind[s] == 1 else AssertionError())
    result = []
    for s in range(len(cols)):
        a, b = int(out_off[s]), int(out_off[s + 1])
        e0, e1 = int(entry_off[a]), int(entry_off[b])
        result.append(Merged(read[a:b], entry_off[a:b + 1] - e0, pos[e0:e1], al[e0:e1], q[e0:e1],
                             representative[int(set_off[s]):int(set_off[s + 1])].copy()))
    return result


def _own_readset(m: Merged):
    """This package's ReadSet of the merged reads, filled from the arrays (one Read object per output read)."""
    from .core import ReadSet, Read, _typed

    rs = ReadSet()
    off = m.entry_off.tolist()
    pos, allele, quality = (np.ascontiguousarray(a, np.int64) for a in (m.position, m.allele, m.quality))
    for k, r in enumerate(m.read.tolist()):
        read = Read(f"read{r}")
        a, b = off[k], off[k + 1]
        read._pos.frombytes(pos[a:b].tobytes())
        read._allele.frombytes(allele[a:b].tobytes())
        read._quality.frombytes(quality[a:b].tobytes())
        read._owner = rs
        rs._by_name[(read._name, 0)] = k
        rs._reads.append(read)
    n = len(rs._reads)
    rs._columns = [_typed(np.diff(m.entry_off)), array("q", bytes(8 * n)), _typed(pos), _typed(allele), _typed(quality)]
    return rs


def _foreign_readset(m: Merged, Read, ReadSet):
    """A ReadSet of another module's classes (the reference's), built per entry through add_variant."""
    rs = ReadSet()
    off, pos, allele, quality = m.entry_off.tolist(), m.position.tolist(), m.allele.tolist(), m.quality.tolist()
    for k, r in enumerate(m.read.tolist()):
        read = Read(f"read{r}")
        for x in range(off[k], off[k + 1]):
            read.add_variant(pos[x], allele[x], quality[x])
        rs.add(read)
    return rs


def _merge(params, readset, build, log, device, stats, library):
    error_rate, max_error_rate, thr, thr_neg = params
    log.info("Merging %d reads with error rate %.2f, maximum error rate %.2f, positive threshold %d and negative threshold %d ...",
             len(readset), error_rate, max_error_rate, thr, thr_neg)
    (m,) = merge_reads([readset], error_rate, max_error_rate, thr, thr_neg, device=device, stats=stats, library=library)
    merged = build(m)
    log.info("... after merging: merged %d reads into %d reads", len(readset), len(merged))
    return merged


class ReadMergerBase(ABC):
    @abstractmethod
    def merge(self, readset):
        pass


class DoNothingReadMerger(ReadMergerBase):
    def merge(self, readset):
        return readset


class ReadMerger(ReadMergerBase):
    """The reference's ReadMerger(error_rate, max_error_rate, positive_threshold, negative_threshold) on the GPU; `merge`
    returns this package's ReadSet.  `stats`, when a dict, receives the counters of the last call."""

    def __init__(self, error_rate, max_error_rate, positive_threshold, negative_threshold, *, device: int = 0,
                 stats: Optional[dict] = None, library=None):
        self._params = (error_rate, max_error_rate, positive_threshold, negative_threshold)
        self._device, self._stats, self._library = device, stats, library

    def merge(self, readset):
        return _merge(self._params, readset, _own_readset, logger, self._device, self._stats, self._library)
