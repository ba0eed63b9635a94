"""Votes of `whatshap haplotagphase` on the GPU.

`compute_votes` and `consensus` have the signatures and the results of the reference's functions in
`whatshap/cli/haplotagphase.py`, and `vote` is the array-level call beneath them (`whmec_haplotagphase`, DESIGN §4.16).  Per
sample, every entry of a read with usable HP and PS tags at a heterozygous position adds its quality to the key
(PS_tag - 1, (HP_tag - 1) ^ allele_to_id[position][allele]) of its position; the device sums the keys with a radix sort, picks each
position's best key (ties: the key inserted first) and orders positions and keys as the reference's dicts hold them.

Where the reference raises, the same exception type is raised, for what it meets first: KeyError in the vote (a position
missing from `is_homozygous`, an allele missing from `allele_to_id`, or an id other than 0 or 1), then ZeroDivisionError (a
position whose keys sum to 0) or KeyError (`id_to_allele`) in the consensus, positions in vote order.  Qualities must fit in
int32, and a position whose best score or total reaches 2^53 in magnitude is refused with ValueError, so that score / total is
the double Python computes.
"""
from __future__ import annotations

import ctypes as C
import logging
from typing import Iterable, NamedTuple, Optional

import numpy as np

from . import _lib
from ._abi import WHMEC_ERR_INPUT, CHaplotagphaseInput, CHaplotagphaseOutput, CHaplotagphaseStats, raise_for

logger = logging.getLogger(__name__)

_INT32 = (-(1 << 31), (1 << 31) - 1)
_HOMOZYGOUS, _PHASED, _SNV = 1, 2, 4
_ZERO_DIVISION, _KEY_ID, _TOO_LARGE, _EMPTY = 1, 2, 3, 4


class Sample(NamedTuple):
    """One sample's input to `vote`, keyed by position as `run_haplotagphase` builds it: `homozygous` (position -> bool),
    `allele_to_id` and `id_to_allele` (position -> {allele: id} / {id: allele}, records at one position merged), `phased`
    (position -> phase, None when unphased) and `is_snv` (position -> bool)."""
    reads: object
    homozygous: dict
    allele_to_id: dict
    id_to_allele: dict
    phased: dict
    is_snv: dict


class Votes(NamedTuple):
    """One sample's votes, positions in the order reads first reached them: the best key (phase_set, haplotype) with its score
    and the total of all keys, whether the consensus keeps the position and the alleles id_to_allele[h], id_to_allele[1 - h]
    of a kept one; the keys (key_ps[j], j % 2) with key_score[j] for j in key_off[i] .. key_off[i + 1] in insertion order; and
    the reads skipped for HP_tag > 2."""
    position: np.ndarray
    phase_set: np.ndarray
    haplotype: np.ndarray
    score: np.ndarray
    total: np.ndarray
    kept: np.ndarray
    allele: np.ndarray
    error: np.ndarray
    key_off: np.ndarray
    key_ps: np.ndarray
    key_score: np.ndarray
    skipped: int

    def as_dict(self) -> dict:
        """The votes as compute_votes returns them: position -> {(ps, h): score} in insertion order."""
        pos, off, ps, sc = self.position.tolist(), self.key_off.tolist(), self.key_ps.tolist(), self.key_score.tolist()
        return {p: {(ps[j], j & 1): sc[j] for j in range(off[i], off[i + 1])} for i, p in enumerate(pos)}


class VoteDict(dict):
    """compute_votes' result: equal to the reference's dict, carrying the device's choice per position (`choices`: the arrays
    of `Votes` in the dict's order) for `consensus`.  The choices describe the dict as returned; a caller who changes its
    scores afterwards should pass a plain dict(...) copy."""
    __slots__ = ("choices",)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None and len(a) else None


def _read_columns(reads):
    """(read_off, pos, allele, quality, HP_tag, PS_tag) of a ReadSet (this package's or the reference's) or a list of reads."""
    from .core import ReadSet

    if isinstance(reads, ReadSet):
        lens, _, pos, allele, quality = reads._flat_columns()
        off = np.zeros(len(lens) + 1, np.int64)
        np.cumsum(lens, out=off[1:])
        rs = reads._reads
        hp = np.array([r._HP_tag for r in rs], np.int64)
        ps = np.array([r._PS_tag for r in rs], np.int64)
    else:
        from .adapters import _readset_to_csr

        off, pos, allele, quality, _, _ = _readset_to_csr(reads)
        hp = np.array([int(r.HP_tag) for r in reads], np.int64)
        ps = np.array([int(r.PS_tag) for r in reads], np.int64)
    return off, pos, allele, quality, hp, ps


def _pairs(d) -> list:
    return [(int(k), int(v)) for k, v in d.items()]


def _tables(samples):
    """Positions, flags and the two pair tables of every sample: (pos_off, pos, flags, a2i_off, a2i, i2a_off, i2a)."""
    pos_off, pos, flags, a2i_len, a2i, i2a_len, i2a = [0], [], [], [], [], [], []
    for positions, flag_of, a2i_of, i2a_of in samples:
        for p in positions:
            pos.append(int(p))
            flags.append(flag_of(p))
            pa, pi = a2i_of(p), i2a_of(p)
            a2i_len.append(len(pa))
            a2i.extend(pa)
            i2a_len.append(len(pi))
            i2a.extend(pi)
        pos_off.append(len(pos))

    def csr(lens, pairs):
        off = np.zeros(len(lens) + 1, np.uint64)
        np.cumsum(np.array(lens, np.uint64), out=off[1:])
        arr = np.array(pairs, np.int64).reshape(-1, 2)
        return off, np.ascontiguousarray(arr[:, 0]), np.ascontiguousarray(arr[:, 1])

    return (np.array(pos_off, np.uint64), np.array(pos, np.int64), np.array(flags, np.uint8)) + csr(a2i_len, a2i) + csr(i2a_len, i2a)


def _call(tables, n_samples, reads=None, runs=None, gap_threshold=70, only_indels=False, device=0, stats=None, library=None):
    """One whmec_haplotagphase call; returns [Votes] per sample and per sample (entry error kind, entry index)."""
    L = library or _lib.lib()
    pos_off, pos, flags, a2i_off, a2i_a, a2i_i, i2a_off, i2a_i, i2a_a = tables
    ci = CHaplotagphaseInput(n_samples, _p(pos_off, C.c_uint64), _p(pos, C.c_int64), _p(flags, C.c_uint8), _p(a2i_off, C.c_uint64),
                             _p(a2i_a, C.c_int64), _p(a2i_i, C.c_int64), _p(i2a_off, C.c_uint64), _p(i2a_i, C.c_int64), _p(i2a_a, C.c_int64))
    ci.gap_threshold, ci.only_indels = float(gap_threshold), int(bool(only_indels))
    keep = []
    if reads is not None:
        read_sample, hp, ps, off, epos, eallele, equal = reads
        keep += [read_sample, hp, ps, off, epos, eallele, equal]
        ci.n_reads = len(read_sample)
        ci.read_sample, ci.read_hp, ci.read_ps = _p(read_sample, C.c_uint32), _p(hp, C.c_int64), _p(ps, C.c_int64)
        ci.read_off = _p(off, C.c_uint64)
        ci.entry_pos, ci.entry_allele, ci.entry_quality = _p(epos, C.c_int64), _p(eallele, C.c_int64), _p(equal, C.c_int32)
    else:
        rsample, rpos, roff, rps, rh, rscore = runs
        keep += [rsample, rpos, roff, rps, rh, rscore]
        ci.n_runs_pos = len(rsample)
        ci.runs_sample, ci.runs_pos = _p(rsample, C.c_uint32), _p(rpos, C.c_int64)
        ci.run_off = roff.ctypes.data_as(C.POINTER(C.c_uint64))  # (never NULL: it selects the runs form)
        ci.run_ps, ci.run_h, ci.run_score = _p(rps, C.c_int64), _p(rh, C.c_int64), _p(rscore, C.c_int64)
    voted_off = np.zeros(n_samples + 1, np.uint64)
    skipped = np.zeros(max(n_samples, 1), np.uint64)
    entry_error = np.zeros(max(n_samples, 1), np.int32)
    entry_error_at = np.zeros(max(n_samples, 1), np.uint64)
    out = CHaplotagphaseOutput(voted_off.ctypes.data_as(C.POINTER(C.c_uint64)), _p(skipped, C.c_uint64), _p(entry_error, C.c_int32),
                               _p(entry_error_at, C.c_uint64))
    st = CHaplotagphaseStats()
    err = C.create_string_buffer(1024)
    rc = L.whmec_haplotagphase(C.byref(ci), device, C.byref(out), C.byref(st), err, len(err))
    if rc == WHMEC_ERR_INPUT:
        raise ValueError(err.value.decode())
    raise_for(rc, err.value.decode())
    try:
        n = int(out.n_voted)
        nk = int(out.key_off[n]) if n else 0
        arr = lambda ptr, count, dt: np.ctypeslib.as_array(ptr, (count,)).astype(dt, copy=True) if count else np.zeros(0, dt)
        cols = dict(position=arr(out.voted_pos, n, np.int64), phase_set=arr(out.phase_set, n, np.int64), haplotype=arr(out.haplotype, n, np.int64),
                    score=arr(out.score, n, np.int64), total=arr(out.total, n, np.int64), kept=arr(out.kept, n, bool),
                    allele=arr(out.allele, 2 * n, np.int64).reshape(n, 2), error=arr(out.error, n, np.int32),
                    key_off=arr(out.key_off, n + 1, np.int64) if n else np.zeros(1, np.int64), key_ps=arr(out.key_ps, nk, np.int64),
                    key_score=arr(out.key_score, nk, np.int64))
    finally:
        L.whmec_haplotagphase_release(C.byref(out))
    if stats is not None:
        stats.update(st.as_dict())
    result = []
    for s in range(n_samples):
        a, b = int(voted_off[s]), int(voted_off[s + 1])
        ko = cols["key_off"][a:b + 1]
        result.append(Votes(*(cols[k][a:b] for k in ("position", "phase_set", "haplotype", "score", "total", "kept", "allele", "error")),
                            ko - ko[0], cols["key_ps"][ko[0]:ko[-1]], cols["key_score"][ko[0]:ko[-1]], int(skipped[s])))
    return result, [(int(entry_error[s]), int(entry_error_at[s])) for s in range(n_samples)]


def _pack_reads(columns):
    """The reads of every sample as the vote form's arrays."""
    counts = [len(c[0]) - 1 for c in columns]
    read_sample = np.repeat(np.arange(len(columns), dtype=np.uint32), counts)
    off = np.zeros(sum(counts) + 1, np.uint64)
    if counts and sum(counts):
        np.cumsum(np.concatenate([np.diff(c[0]) for c in columns]).astype(np.uint64), out=off[1:])
    cat = lambda i, dt: np.concatenate([np.asarray(c[i], np.int64) for c in columns]).astype(dt) if columns else np.zeros(0, dt)
    quality = cat(3, np.int64)
    if len(quality) and (quality.min() < _INT32[0] or quality.max() > _INT32[1]):
        raise ValueError("an entry quality lies outside int32")
    return read_sample, cat(4, np.int64), cat(5, np.int64), off, cat(1, np.int64), cat(2, np.int64), quality.astype(np.int32)


def _raise_entry_error(kind, at, reads_packed, allele_to_id):
    _, hp, ps, off, epos, eallele, _ = reads_packed
    r = int(np.searchsorted(off, at, side="right") - 1)
    p, a = int(epos[at]), int(eallele[at])
    if kind == 1:
        raise KeyError(p)
    if kind == 2:
        raise KeyError(a)
    raise KeyError((int(ps[r]) - 1, (int(hp[r]) - 1) ^ allele_to_id[p][a]))


def _raise_choice_error(code, pos, h, id_to_allele):
    if code == _ZERO_DIVISION:
        raise ZeroDivisionError("division by zero")
    if code == _TOO_LARGE:
        raise ValueError(f"position {pos}: a vote score or total reaches 2^53, beyond an exact double quotient")
    if code == _EMPTY:
        raise IndexError("list index out of range")
    if code == _KEY_ID:
        id_to_allele[pos][h]
        id_to_allele[pos][1 - h]
        raise KeyError(1 - h)  # (not reached: one of the lookups raises)


def _sample_table(s: Sample):
    positions = sorted(s.homozygous)
    is_snv = s.is_snv or {}
    flag = lambda p: ((_HOMOZYGOUS if s.homozygous[p] else 0) | (_PHASED if s.phased.get(p) is not None else 0) |
                      (_SNV if is_snv.get(p, False) else 0))
    return positions, flag, lambda p: _pairs(s.allele_to_id.get(p, {})), lambda p: _pairs(s.id_to_allele.get(p, {}))


def vote(samples: Iterable[Sample], *, gap_threshold=70, only_indels: bool = False, device: int = 0, stats: Optional[dict] = None,
         library: Optional[C.CDLL] = None) -> list:
    """Votes and consensus choices of every sample in one call: one `Votes` per sample.  The first exception the reference's
    `compute_votes` and `consensus` would raise, sample after sample, is raised.  `stats` (a dict) receives the call's counters:
    entries, positions, records, h2d_bytes, d2h_bytes, chunks, kernel_launches, device_ms, plan_ms.  `library`: another build
    of the library with the same entry point (tests)."""
    samples = list(samples)
    packed = _pack_reads([_read_columns(s.reads) for s in samples])
    res, errors = _call(_tables([_sample_table(s) for s in samples]), len(samples), reads=packed, gap_threshold=gap_threshold,
                        only_indels=only_indels, device=device, stats=stats, library=library)
    for s, (v, (kind, at)) in enumerate(zip(res, errors)):
        if kind:
            _raise_entry_error(kind, at, packed, samples[s].allele_to_id)
        bad = np.flatnonzero(v.error)
        if len(bad):
            i = int(bad[0])
            _raise_choice_error(int(v.error[i]), int(v.position[i]), int(v.haplotype[i]), samples[s].id_to_allele)
    return res


def _compute_votes(is_homozygous, reads, allele_to_id, log, device=0, stats=None, library=None) -> VoteDict:
    positions = sorted(is_homozygous)
    table = (positions, lambda p: _HOMOZYGOUS if is_homozygous[p] else 0, lambda p: _pairs(allele_to_id.get(p, {})), lambda p: [])
    packed = _pack_reads([_read_columns(reads)])
    # the choice alone: nothing passes a gap threshold of +inf, so no position needs id_to_allele here
    (v,), ((kind, at),) = _call(_tables([table]), 1, reads=packed, gap_threshold=float("inf"), device=device, stats=stats, library=library)
    if kind:
        _raise_entry_error(kind, at, packed, allele_to_id)
    if v.skipped > 0:
        log.warning(f"{v.skipped} reads were skipped due incorrect HP. The haplotagphase command supports only a diploid input")
    out = VoteDict(v.as_dict())
    out.choices = v
    return out


def _consensus(variant_cls, only_indels, gap_threshold, cut_homopolymers, refseq, change, phased, votes, id_to_allele, device=0,
               stats=None, library=None):
    # cut_homopolymers and refseq are accepted and not read: the reference's filter counts a homopolymer up to cut_homopolymers
    # bases and then drops the position only when the count exceeds cut_homopolymers, which it never does.
    carried = isinstance(votes, VoteDict) and getattr(votes, "choices", None) is not None and len(votes.choices.position) == len(votes)
    if carried:
        v = votes.choices
    else:
        positions = list(votes)
        rpos, roff, rps, rh, rscore = [], [0], [], [], []
        for p in positions:
            for (ps, h), score in votes[p].items():
                rps.append(ps), rh.append(h), rscore.append(score)
            roff.append(len(rps))
        rps, rh, rscore = (np.array(x, dtype=object) for x in (rps, rh, rscore))
        for name, a, lim in (("phase set", rps, 1 << 62), ("haplotype", rh, 1 << 62), ("score", rscore, 1 << 63)):
            if len(a) and (min(a) < -lim or max(a) >= lim):
                raise ValueError(f"a vote's {name} lies outside the range of whmec_haplotagphase")
        flag = lambda p: (_PHASED if phased[p] is not None else 0) | (
            _SNV if only_indels and phased[p] is None and change[p].is_snv() else 0)
        table = (sorted(positions), flag, lambda p: [], lambda p: _pairs(id_to_allele.get(p, {})))
        runs = (np.zeros(len(positions), np.uint32), np.array(positions, np.int64), np.array(roff, np.uint64),
                rps.astype(np.int64), rh.astype(np.int64), rscore.astype(np.int64))
        (v,), _ = _call(_tables([table]), 1, runs=runs, gap_threshold=gap_threshold, only_indels=only_indels, device=device, stats=stats,
                        library=library)
    positions, ps, h, score, total = (x.tolist() for x in (v.position, v.phase_set, v.haplotype, v.score, v.total))
    error, kept, allele = v.error.tolist(), v.kept.tolist(), v.allele.tolist()
    components, chosen = {}, []
    for i, pos in enumerate(positions):
        if error[i] and error[i] != _KEY_ID:
            _raise_choice_error(error[i], pos, h[i], id_to_allele)
        components[pos] = ps[i]
        if carried:
            if phased[pos] is None:
                if 100 * (score[i] / total[i]) < gap_threshold:
                    continue
                if only_indels and change[pos].is_snv():
                    continue
            chosen.append((pos, id_to_allele[pos][h[i]], id_to_allele[pos][1 - h[i]], score[i]))
        elif kept[i]:
            if error[i] == _KEY_ID:
                _raise_choice_error(error[i], pos, h[i], id_to_allele)
            chosen.append((pos, allele[i][0], allele[i][1], score[i]))
    chosen.sort(key=lambda c: c[0])
    super_reads = [[variant_cls(p, allele=a0, quality=q) for p, a0, _, q in chosen], [variant_cls(p, allele=a1, quality=q) for p, _, a1, q in chosen]]
    return super_reads, components


def compute_votes(is_homozygous, reads, allele_to_id, *, device: int = 0, stats: Optional[dict] = None, library: Optional[C.CDLL] = None):
    """The reference's compute_votes: position -> {(ps, h): score}, positions and keys in insertion order, as a `VoteDict` that
    also carries the device's choice per position.  Reads skipped for HP_tag > 2 are counted in a warning of this module's
    logger."""
    return _compute_votes(is_homozygous, reads, allele_to_id, logger, device, stats, library)


def consensus(only_indels, gap_threshold, cut_homopolymers, refseq, change, phased, votes, id_to_allele, *, device: int = 0,
              stats: Optional[dict] = None, library: Optional[C.CDLL] = None):
    """The reference's consensus: ([super-read 0, super-read 1] as lists of `Variant` sorted by position, position -> phase set).
    A `VoteDict` from `compute_votes` is decided by the choices it carries; any other mapping goes to the device as runs in its
    own key order."""
    from .variant import Variant

    return _consensus(Variant, only_indels, gap_threshold, cut_homopolymers, refseq, change, phased, votes, id_to_allele, device, stats,
                      library)
