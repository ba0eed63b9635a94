"""K-mer pair counts of `whatshap learn` on the GPU.

`count_kmer_pairs` gives the rows (column, reference k-mer, read k-mer, count) that WhatsHap's `Caller` (src/caller.cpp, driven
by `whatshap.cli.learn.run_learn`) writes for a chromosome's reads, in one call (`whmec_learn`, DESIGN §4.13): the host walks
every CIGAR and cuts the columns into chunks; the device emits one key per counted k-mer, sorts and run-length encodes the keys
and attaches the reference k-mers.  `write_counts` writes rows as the reference does (`%d\\t%d\\t%d\\t%d\\n`).

`Caller` is a swap-in for the reference's class with the same interface, so that `whatshap.cli.learn.Caller = Caller` runs an
unchanged `run_learn`.  Two differences, neither of which changes the file `run_learn` writes:

- Within a column the reference writes its rows in the iteration order of a `std::unordered_map`; here they ascend by read
  k-mer.  The columns, and the set of rows of each column, are the reference's.
- The reference writes the columns an `add_read` completes during that call.  `Caller` buffers the reads and writes those
  columns later, to the file each was due to: when the buffered query bytes pass `Caller.buffer_bytes` (the columns complete
  so far), at `final_pop`, when the next `Caller` is constructed or `all_variants` is called (the columns the reference had
  written for this one), and when the object is collected or the interpreter exits.  Lines therefore arrive in batches, in the
  reference's order.

Inputs on which the reference aborts or reads out of bounds raise ValueError instead: k outside 1..15, a reference shorter than
k, an empty variant list, a read without a k-mer, P, B or an unknown CIGAR operation of non-zero length (or the end of the CIGAR)
while query bytes remain, pos + k - 1 or a k-mer column beyond the reference, positions outside int32.  A `Caller` raises them
when it writes the read's columns, naming the read by its `add_read` ordinal.
"""
from __future__ import annotations

import ctypes as C
import os
import re
import weakref
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._abi import WHMEC_ERR_INPUT, CLearnInput, CLearnOutput, CLearnStats, raise_for
from .realign import _bytes, _csr, _int32, _ptr


def _alignment(a):
    if isinstance(a, tuple):
        return a
    pos = a.pos if hasattr(a, "pos") else a.reference_start
    return pos, a.cigartuples, a.query_alignment_sequence


def count_kmer_pairs(alignments, variants, reference, k: int = 7, window: int = 25, *, first_variant: int = 0, final: bool = True,
                     columns: Optional[Tuple[int, int]] = None, floors: Optional[Sequence[int]] = None, device: int = 0,
                     stats: Optional[dict] = None, library: Optional[C.CDLL] = None) -> Tuple[np.ndarray, int]:
    """(rows, next variant offset): the rows one reference `Caller(reference, k, window)` writes for `alignments` added in order,
    as an (n, 4) int32 array of column, reference k-mer, read k-mer and count, ascending by column and then by read k-mer.

    alignments: objects with `pos` (or `reference_start`), `cigartuples` and `query_alignment_sequence` (a pysam.AlignedSegment
    qualifies), or (pos, cigartuples, query) tuples.  variants: the (position, len(REF)) list `run_learn` hands to
    `all_variants`, every chromosome's, and first_variant the list's front before this chromosome (the returned offset is the
    next chromosome's).  final: the chromosome's columns up to its end (`final_pop`); otherwise only those the reads completed
    (a `Caller` that `run_learn` abandons for the next chromosome).  columns (lo, hi) and floors (one per alignment: the last
    column popped before it was added) serve a caller that hands the reads over in parts.  `stats` (a dict) receives the call's
    counters: alignments, kmers, kept, distinct, rows, chunks, kernel_launches, device_ms, plan_ms, h2d_bytes, d2h_bytes.
    `library`: another build of the library with the same entry point (tests)."""
    k = int(k)
    if not 1 <= k <= 15:
        raise ValueError("k must lie in 1..15")
    if not len(variants):
        raise ValueError("the variant list is empty (the reference reads its front)")
    L = library or _lib.lib()
    alns = [_alignment(a) for a in alignments]
    n = len(alns)
    cigars = [cg or () for _, cg, _ in alns]
    starts = _int32([p for p, _, _ in alns], "alignment position")
    cigar_off = np.zeros(n + 1, np.uint64)
    if n:
        np.cumsum(np.fromiter(map(len, cigars), np.uint64, n), out=cigar_off[1:])
    flat = np.array([x for cg in cigars for x in cg], dtype=np.int64).reshape(-1, 2)
    ops = flat[:, 0]
    cigar_op = np.where((ops >= 0) & (ops <= 254), ops, 255).astype(np.uint8)
    cigar_len = _int32(flat[:, 1], "CIGAR length")
    query_off, query = _csr([_bytes(q) if q is not None else b"" for _, _, q in alns])
    var = np.asarray(variants, dtype=np.int64).reshape(-1, 2)
    vpos, vlen = _int32(var[:, 0], "variant position"), _int32(var[:, 1], "variant length")
    ref = np.frombuffer(_bytes(reference), np.uint8) if len(reference) else np.zeros(1, np.uint8)
    fl = None if floors is None else _int32(floors, "floor")
    lo, hi = (0, 0) if columns is None else (int(columns[0]), int(columns[1]))
    if columns is not None and lo <= 0:
        raise ValueError("columns must start at a positive column")
    ci = CLearnInput(
        _ptr(ref, C.c_uint8), len(reference), n, _ptr(starts, C.c_int32), _ptr(cigar_off, C.c_uint64), _ptr(cigar_op, C.c_uint8),
        _ptr(cigar_len, C.c_int32), _ptr(query_off, C.c_uint64), _ptr(query, C.c_uint8), len(vpos), _ptr(vpos, C.c_int32),
        _ptr(vlen, C.c_int32), int(first_variant), k, int(window), int(bool(final)), lo, hi, _ptr(fl, C.c_int32))
    out, st = CLearnOutput(), CLearnStats()
    err = C.create_string_buffer(1024)
    rc = L.whmec_learn(C.byref(ci), device, C.byref(out), C.byref(st), err, len(err))
    if rc == WHMEC_ERR_INPUT:
        raise ValueError(err.value.decode())
    raise_for(rc, err.value.decode())
    try:
        rows = np.ctypeslib.as_array(out.rows, (int(out.n_rows), 4)).copy() if out.n_rows else np.zeros((0, 4), np.int32)
        nxt = int(out.next_variant)
    finally:
        L.whmec_learn_release(C.byref(out))
    if stats is not None:
        stats.update(st.as_dict())
    return rows, nxt


def write_counts(path, rows: np.ndarray, append: bool = True, *, library: Optional[C.CDLL] = None) -> None:
    """Writes rows (an (n, 4) integer array) as the reference does, one `column\\tref k-mer\\tread k-mer\\tcount` line each,
    appending to path or replacing it."""
    L = library or _lib.lib()
    rows = np.ascontiguousarray(rows, dtype=np.int32).reshape(-1, 4)
    out = CLearnOutput(len(rows), _ptr(rows if len(rows) else None, C.c_int32), 0)
    err = C.create_string_buffer(1024)
    rc = L.whmec_learn_write(os.fsencode(path), C.byref(out), int(bool(append)), err, len(err))
    if rc == WHMEC_ERR_INPUT:
        raise OSError(err.value.decode())
    raise_for(rc, err.value.decode())


# all_variants' list and its front, process-wide as the reference's globals, and the state of the Caller constructed last
_variants: List[Tuple[int, int]] = []
_front = 0
_pending: Optional["_State"] = None

_REF_OPS = frozenset((0, 2, 3, 7, 8))  # M D N = X: the operations that advance pos


class _State:
    """What one Caller has buffered: reads not yet complete, the columns written so far and the files the pops since then go to."""

    def __init__(self, reference, k, window, library, device):
        self.reference, self.k, self.window, self.library, self.device = reference, k, window, library, device
        self.written = k - 1  # columns <= written are in their files
        self.top = k - 1      # the last column the reference has popped
        self.reads = []       # [ordinal, pos, cigar, query, floor, last column it can reach]
        self.bytes = 0
        self.n_added = 0
        self.files = []       # [(last column, outfile)] of the pops after `written`, in order


def _flush(state: _State, hi: int) -> None:
    """Writes columns state.written + 1 .. hi to their files, and forgets the reads that end before hi."""
    global _front
    rows = np.zeros((0, 4), np.int32)
    if hi > state.written:
        reads = state.reads
        try:
            rows, _front = count_kmer_pairs([(r[1], r[2], r[3]) for r in reads], _variants, state.reference, state.k, state.window,
                                            first_variant=_front, columns=(state.written + 1, hi), floors=[r[4] for r in reads],
                                            device=state.device, library=state.library)
        except ValueError as e:  # nothing of this Caller is written after a refusal (the reference aborts)
            state.reads, state.files, state.written = [], [], state.top
            m = re.match(r"alignment (\d+): (.*)", str(e), re.S)
            if m:
                raise ValueError(f"read {reads[int(m.group(1))][0]} of this Caller: {m.group(2)}") from None
            raise
    bounds = np.array([c for c, _ in state.files], np.int64)
    cut = np.searchsorted(rows[:, 0], bounds, side="right")
    start = 0
    for (_, path), end in zip(state.files, cut):
        write_counts(path, rows[start:end], append=True, library=state.library)
        start = end
    state.files = []
    state.written = max(state.written, hi)
    state.reads = [r for r in state.reads if r[5] > hi]
    state.bytes = sum(len(r[3]) for r in state.reads)


def _abandon(state: Optional[_State]) -> None:
    """The columns the reference had written for a Caller that gets no more calls."""
    if state is not None and (state.top > state.written or state.files):
        _flush(state, state.top)


class Caller:
    """Swap-in for the reference's `whatshap.core.Caller(reference, k, window)`: `all_variants`, `add_read`, `final_pop` and
    `finish` write the same lines to the same files (see the module docstring for when, and for the order within a column)."""

    #: query bytes a Caller buffers before it writes the columns complete so far
    buffer_bytes = 64 << 20

    def __init__(self, reference, k: int, window: int, *, device: int = 0, library: Optional[C.CDLL] = None):
        global _pending
        k = int(k)
        if not 1 <= k <= 15:
            raise ValueError("k must lie in 1..15")
        reference = _bytes(reference)
        if len(reference) < k:
            raise ValueError("the reference is shorter than k")
        _abandon(_pending)
        self._state = _State(reference, k, int(window), library, device)
        _pending = self._state
        weakref.finalize(self, _abandon, self._state)

    def all_variants(self, variants) -> None:
        """Sets the process-wide variant list [(position, len(REF))], its front at the first."""
        global _variants, _front
        _abandon(_pending)
        _variants = [(int(p), int(n)) for p, n in variants]
        _front = 0

    def add_read(self, pos: int, cigartuples, query, outfile) -> None:
        s = self._state
        cigar = [(int(op), int(n)) for op, n in cigartuples]
        query = _bytes(query)
        span = sum(n for op, n in cigar if op in _REF_OPS)
        s.reads.append([s.n_added, int(pos), cigar, query, s.top, int(pos) + span + 1])
        s.n_added += 1
        s.bytes += len(query)
        s.top = max(s.top, int(pos) + s.k - 1)
        self._pop(s.top, outfile)
        if s.bytes > self.buffer_bytes:
            _flush(s, s.top)

    def final_pop(self, outfile) -> None:
        s = self._state
        s.top = max(s.top, len(s.reference))
        self._pop(len(s.reference), outfile)
        _flush(s, s.top)

    def finish(self) -> None:
        pass

    def _pop(self, hi: int, outfile) -> None:
        files = self._state.files
        if files and files[-1][1] == outfile:
            files[-1] = (max(files[-1][0], hi), outfile)
        else:
            files.append((max(hi, files[-1][0] if files else self._state.written), outfile))
