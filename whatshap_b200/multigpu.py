"""Sharding of DP-independent blocks across the GPUs of one box (SURVEY.md §8(e)).

For a single individual (T = 1) the DP decomposes exactly at columns that no read spans: cost adds,
partitioning / super-reads concatenate, tie-breaks are unaffected (a constant offset changes no `<`).
Runs of those blocks are the parts of the table (`plan_parts`), solved with no exchange between them and merged in column
order.  Pedigrees (T > 1) couple the blocks through the transmission vector: every part is a SEGMENT of the table
(`whmec_segment_*`) and the parts exchange T x T transfer matrices and exit tables, bit-identical to the single-GPU solve.
Genotyping (the forward-backward DP) cuts a single individual by chains and a pedigree into segments
(`whmec_genotype_segment_*`) that exchange T x T transfer matrices of doubles, folded into every segment's true forward and
backward inputs (DESIGN §4.5).

Each scheme is written once (`_phasing_segments`, `_genotype_segments`, and `_run_parts` for runs of blocks and for the
whole table) and runs on one of three executors: `_Local` (every part in one process on one device, in column order:
`solve_pedigree_segments`, `genotype_pedigree_segments`), `_Threads` (one host thread per device in one process:
`solve_on_devices`, `genotype_on_devices`, which `core`'s tables and the swap-in classes of `adapters` reach through
`solve_table` / `genotype_table` when given `devices` or when WHMEC_DEVICES is set) and `_Ranks` (one process per GPU,
`torch.distributed` over NCCL: `solve_sharded`, `genotype_sharded`).  DESIGN §6.

The reference has no counterpart (single process, `whatshap/cli/phase.py:604-610` runs one
PedigreeDPTable per chromosome x family).
"""
from __future__ import annotations

import os
import time
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from . import _wire
from ._abi import FlatProblem, FlatSolution, Unsupported


def _read_spans(prob: FlatProblem) -> Tuple[np.ndarray, np.ndarray]:
    """(first column, last column) of every read, int64."""
    starts = prob.read_off[:-1].astype(np.int64)
    ends = prob.read_off[1:].astype(np.int64) - 1
    return prob.ent_col[starts].astype(np.int64), prob.ent_col[ends].astype(np.int64)


def independent_blocks(prob: FlatProblem, spans=None) -> List[Tuple[int, int]]:
    """Maximal column ranges [lo, hi) that no read crosses (chains of the DP)."""
    n = prob.n_cols
    if n == 0:
        return []
    span = np.zeros(n + 2, np.int64)
    if prob.n_reads:
        first, last = spans if spans is not None else _read_spans(prob)
        span += np.bincount(first + 1, minlength=n + 2) - np.bincount(last + 1, minlength=n + 2)
    crossing = np.cumsum(span)[1:n]  # crossing[k-1] > 0: some read is active in columns k-1 and k
    cuts = [0] + (np.nonzero(crossing == 0)[0] + 1).tolist() + [n]
    return list(zip(cuts[:-1], cuts[1:]))


def block_work(prob: FlatProblem, blocks: Sequence[Tuple[int, int]], spans=None) -> np.ndarray:
    """DP cells per block, sum_k 2^{a_k} (the quantity the sweep time is proportional to)."""
    n = prob.n_cols
    cov = np.zeros(n + 1, np.int64)
    if prob.n_reads:
        first, last = spans if spans is not None else _read_spans(prob)
        cov += np.bincount(first, minlength=n + 1) - np.bincount(last + 1, minlength=n + 1)
    a = np.cumsum(cov)[:n]
    cells = np.exp2(np.minimum(a, 40).astype(np.float64))
    prefix = np.concatenate([[0.0], np.cumsum(cells)])
    if not len(blocks):
        return np.zeros(0)
    bounds = np.asarray(blocks, np.int64)
    return prefix[bounds[:, 1]] - prefix[bounds[:, 0]]


def assign_blocks(work: np.ndarray, world: int) -> List[List[int]]:
    """Longest-processing-time-first assignment of blocks to ranks."""
    order = np.argsort(-work, kind="stable")
    load = np.zeros(world)
    shares: List[List[int]] = [[] for _ in range(world)]
    for b in order:
        r = int(np.argmin(load))
        shares[r].append(int(b))
        load[r] += work[b]
    for s in shares:
        s.sort()
    return shares


def merge_block_solutions(prob: FlatProblem, blocks, solutions, cost: Optional[int] = None) -> FlatSolution:
    """Concatenate per-block results in column order; costs add (T = 1) unless `cost` is given."""
    out = FlatSolution(prob.n_cols, prob.n_reads, prob.n_ind)
    first = prob.ent_col[prob.read_off[:-1].astype(np.int64)] if prob.n_reads else np.zeros(0, np.uint32)
    total = 0
    for (lo, hi), sol in zip(blocks, solutions):
        total += int(sol.cost)
        out.path_index[lo:hi] = sol.path_index
        out.path_tv[lo:hi] = sol.path_tv
        out.sr_allele[:, :, lo:hi] = sol.sr_allele
        out.sr_quality[:, lo:hi] = sol.sr_quality
        reads = np.nonzero((first >= lo) & (first < hi))[0]
        out.partition[reads] = sol.partition
    out.cost = (total if cost is None else cost) & 0xFFFFFFFF
    return out


UMAX = 0xFFFFFFFF


def contiguous_shares(work: np.ndarray, world: int) -> List[Tuple[int, int]]:
    """Cut the block sequence into `world` contiguous runs [b0, b1) minimising the largest run's work
    (a run may be empty when there are fewer blocks than ranks)."""
    work = np.asarray(work, np.float64)
    n = len(work)
    from bisect import bisect_right

    pre = [0.0] + np.cumsum(work).tolist()  # the loads are sums of powers of two: exact in float64 for any realistic table

    def runs_for(limit):  # greedy: fewest runs with no run above `limit` (a block heavier than the limit is a run of its own)
        cuts, s = [0], 0
        while s < n:
            e = max(bisect_right(pre, pre[s] + limit) - 1, s + 1)  # largest e with load(s, e) <= limit, at least one block
            s = min(e, n)
            cuts.append(s)
            if len(cuts) > world + 2:  # already more runs than ranks: the caller only compares with `world`
                cuts[-1] = n
                return cuts
        return cuts

    lo, hi = (float(work.max()) if n else 0.0), float(work.sum())
    for _ in range(48):  # bisection on the largest run (the classic linear-partition bound)
        mid = (lo + hi) / 2
        if len(runs_for(mid)) - 1 <= world:
            hi = mid
        else:
            lo = mid
    cuts = runs_for(hi * (1 + 1e-9))  # the bisection ends a rounding error below a feasible limit at worst
    if len(cuts) - 1 > world:
        cuts = cuts[:world] + [n]
    runs = [(cuts[i], cuts[i + 1]) for i in range(len(cuts) - 1) if cuts[i + 1] > cuts[i]]
    prefix = np.concatenate([[0.0], np.cumsum(work)])
    load = lambda run: prefix[run[1]] - prefix[run[0]]
    while len(runs) < world:  # idle ranks left: halve the heaviest run that still has two blocks
        candidates = [r for r in runs if r[1] - r[0] >= 2]
        if not candidates:
            break
        a, b = max(candidates, key=load)
        mid = min(range(a + 1, b), key=lambda m: max(prefix[m] - prefix[a], prefix[b] - prefix[m]))
        runs[runs.index((a, b))] = (a, mid)
        runs.append((mid, b))
        runs.sort()
    runs += [(n, n)] * (world - len(runs))  # more ranks than blocks: the rest hold nothing
    return runs


def minplus(vec: np.ndarray, matrix: np.ndarray) -> np.ndarray:
    """out[i] = min_u vec[u] + matrix[u, i] over u32 with 0xFFFFFFFF as +inf (the fold of
    `ped_prefix_kernel`, whatshap_b200/csrc/whmec.cu)."""
    v = vec.astype(np.uint64)[:, None]
    m = matrix.astype(np.uint64)
    s = v + m
    s[(v == UMAX) | (m == UMAX)] = UMAX
    return s.min(axis=0).astype(np.uint32)


def segment_inputs(matrices: Sequence[Optional[np.ndarray]]) -> List[Optional[np.ndarray]]:
    """True input vector of every segment from the segments' transfer matrices (None: rank without
    columns).  The first segment ignores its input: all rows of its matrix are its output."""
    inputs: List[Optional[np.ndarray]] = []
    vec = None
    for m in matrices:
        if m is None:
            inputs.append(None)
            continue
        inputs.append(vec)
        vec = m[0].copy() if vec is None else minplus(vec, m)
    return inputs


def segment_entries(exits: Sequence[Optional[np.ndarray]]) -> List[Optional[int]]:
    """Transmission value the backtrace enters every segment with, right to left; -1 for the segment
    that ends the table (it starts at the optimum and reports the same exit for every value)."""
    entries: List[Optional[int]] = [None] * len(exits)
    entry = -1
    for s in range(len(exits) - 1, -1, -1):
        if exits[s] is None:
            continue
        entries[s] = entry
        entry = int(exits[s][max(entry, 0)])
    return entries


def segment_ranges(prob: FlatProblem, world: int) -> List[Optional[Tuple[int, int]]]:
    """Column range [lo, hi) of every rank's segment (None: no columns for that rank)."""
    blocks = independent_blocks(prob)
    shares = contiguous_shares(block_work(prob, blocks), world)
    return [(blocks[b0][0], blocks[b1 - 1][1]) if b1 > b0 else None for b0, b1 in shares]


def plan_parts(prob: FlatProblem, world: int, genotype: bool = False, spans=None
               ) -> Tuple[str, List[Optional[Tuple[int, int]]]]:
    """How a table is cut over `world` devices, for every driver (`solve_sharded`, `genotype_sharded`, `solve_on_devices`,
    `genotype_on_devices`).  Returns (mode, ranges):
      "whole"    -- the table on one device (ranges empty): no columns, or a pedigree of one chain, or one device for a pedigree;
      "blocks"   -- a single individual (T = 1): device i takes a contiguous run of whole chains with about 1 / world of the DP cells;
      "segments" -- a pedigree of two chains or more: device i holds a segment of the table (`segment_ranges`).
    `ranges[i]` is device i's column range [lo, hi), None when it holds no columns.  Genotyping also runs a single individual
    whole on one device instead of as one run of blocks.  `spans`: the reads' column spans (`_read_spans`) if known."""
    if prob.n_cols == 0 or (genotype and world == 1):
        return "whole", []
    blocks = independent_blocks(prob, spans)
    if prob.n_trios > 0:  # transmission vectors couple the chains: segments of the table, or the whole table on one device
        return ("segments", segment_ranges(prob, world)) if world > 1 and len(blocks) > 1 else ("whole", [])
    runs = contiguous_shares(block_work(prob, blocks, spans), world)
    return "blocks", [(blocks[b0][0], blocks[b1 - 1][1]) if b1 > b0 else None for b0, b1 in runs]


def _scaled(vec: np.ndarray) -> np.ndarray:
    """`vec` divided by its largest entry; unchanged when every entry is 0 (gl_scale_host)."""
    top = float(vec.max()) if vec.size else 0.0
    return vec / top if top > 0.0 else vec


def genotype_segment_inputs(matrices: Sequence[Optional[np.ndarray]]) -> Tuple[List[Optional[np.ndarray]], List[Optional[np.ndarray]]]:
    """True forward input (alpha) and backward input (beta) of every genotyping segment from the segments' T x T transfer
    matrices (None: rank without columns; it gets None for both).  The first segment ignores its input: any row of its
    matrix is its output.  The last segment's matrix holds the mass it leaves at every transmission value, so its row sums
    are the backward vector in front of it.  Left to right alpha_{s+1} = alpha_s . M_s, right to left beta_s = M_{s+1} .
    beta_{s+1}; every vector is divided by its largest entry (a positive factor cancels in the per-column normalisation).
    alpha is None for the first segment, beta for the last."""
    active = [s for s, m in enumerate(matrices) if m is not None]
    alphas: List[Optional[np.ndarray]] = [None] * len(matrices)
    betas: List[Optional[np.ndarray]] = [None] * len(matrices)
    vec = None
    for s in active:
        alphas[s] = vec
        m = np.asarray(matrices[s], np.float64)
        vec = _scaled(m[0].copy() if vec is None else vec @ m)
    vec = None
    for s in reversed(active):
        betas[s] = vec
        m = np.asarray(matrices[s], np.float64)
        vec = _scaled(m @ (np.ones(m.shape[1]) if vec is None else vec))
    return alphas, betas


# ---- the schemes and their executors ------------------------------------------------------------------------------
#
# A table cut by `plan_parts` runs as parts in column order, phase by phase.  An executor runs one phase over every part and
# returns one result per part (None for a part without columns): after a shared phase every participant holds every part's
# result, after the others only the part's owner does.  `_Local` runs the parts one after another in one process, `_Threads`
# on one host thread per device, `_Ranks` one part per rank of a process group.  The segment schemes of the two DPs
# (`_phasing_segments`, `_genotype_segments`) and the runs of blocks or of the whole table (`_run_parts`) are written once
# against that interface; a segment refused as unsupported sends the whole table to the first device, except on `_Local`,
# which raises the refusal.


class _Local:
    """One process, one device: the parts in column order, an error or a refusal raised at once."""

    def __init__(self, prob: FlatProblem, ranges):
        self.prob, self.n_cols, self.ranges = prob, prob.n_cols, list(ranges)

    def piece(self, i: int) -> FlatProblem:
        """Part i's columns of the table."""
        r = self.ranges[i]
        return self.prob if r == (0, self.n_cols) else self.prob.slice_columns(*r)

    def on(self, i: int) -> tuple:
        """The trailing arguments that put a call on part i's device (none: this process's current device)."""
        return ()

    def run(self, step, name: str, share=None, then: Optional[str] = None) -> list:
        """`step(i)` for every part i with columns.  `share` = (dtype, number of T-long dimensions) of a result every
        participant receives; `name` (and `then`, after the exchange of a shared result) name the phase's times."""
        return [None if r is None else step(i) for i, r in enumerate(self.ranges)]

    def close(self, segs) -> None:
        for sg in segs:
            if sg is not None:
                sg.close()

    def collect(self, done: list, codec, name: str) -> Optional[list]:
        """Every part's result where the table is assembled; None on the other ranks.  `codec` = (encode, decode) of a result
        that travels between ranks."""
        return done

    def mark(self, name: str) -> None:
        pass

    def whole(self) -> None:
        """From here on the table is one part, on the first device (rank 0)."""
        self.ranges = [(0, self.n_cols)] + [None] * (len(self.ranges) - 1)


def _run_on_devices(devices: Sequence[int], jobs: Sequence[Optional[Callable[[], object]]]) -> Tuple[list, list]:
    """Runs `jobs[i]()` (None: nothing to do) on the host thread of `devices[i]`, one thread per distinct device, so that
    all devices work at once; the jobs of one device run one after another in list order (two plans created at once on one
    device would each size their arena from the same free HBM).  Returns (results, errors), one entry per job, after every
    thread has been joined."""
    import threading

    results: list = [None] * len(jobs)
    errors: list = [None] * len(jobs)
    lanes: dict = {}
    for i, d in enumerate(devices):
        lanes.setdefault(d, []).append(i)

    def lane(indices):
        for i in indices:
            if jobs[i] is not None:
                try:
                    results[i] = jobs[i]()
                except Exception as e:  # noqa: BLE001 - raised on the calling thread, lowest column first
                    errors[i] = e

    threads = [threading.Thread(target=lane, args=(indices,), name="whmec-device-%d" % d) for d, indices in lanes.items()]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    return results, errors


def _raise_first(errors: Sequence[Optional[BaseException]], refusals_last: bool) -> None:
    """Raises the error of the part with the lowest column (the parts are in column order); with `refusals_last` a refusal
    (Unsupported) only when no part failed otherwise."""
    for e in sorted((e for e in errors if e is not None), key=lambda e: refusals_last and isinstance(e, Unsupported)):
        raise e


class _Threads(_Local):
    """One process, part i on `devices[i]`, one host thread per distinct device (`_run_on_devices`).  An error is raised after
    every thread has been joined: that of the part with the lowest column, where `refusals_last` (segment mode) puts the
    refusals after every other error."""

    def __init__(self, prob: FlatProblem, ranges, devices: List[int], refusals_last: bool):
        super().__init__(prob, ranges or [None] * len(devices))
        self.devices, self.refusals_last = devices, refusals_last

    def on(self, i: int) -> tuple:
        return (self.devices[i],)

    def run(self, step, name: str, share=None, then: Optional[str] = None) -> list:
        done, errors = _run_on_devices(self.devices, [None if r is None else (lambda i=i: step(i)) for i, r in enumerate(self.ranges)])
        _raise_first(errors, self.refusals_last)
        return done

    def close(self, segs) -> None:
        _run_on_devices(self.devices, [None if sg is None else sg.close for sg in segs])  # on the segment's own device thread


_MODES = ("whole", "blocks", "segments")


class _Ranks(_Local):
    """One process per rank of `comm`, rank r holding part r.  Rank 0 cuts `prob` (`plan_parts`) and scatters to every rank one
    row: the header [mode, n_cols, lo_0, hi_0, lo_1, hi_1, ...] (lo = hi: no columns) and the rank's columns
    (`_wire.encode_problem_slices`, written straight into the page-locked send buffer).  Every phase ends in one `all_status`
    that carries the shared results, so an error on one rank is raised on every rank, and a refusal as Unsupported on every
    rank.  The results are gathered to rank 0.  `times` (the caller's `timings` if given) receives the ms of every phase."""

    def __init__(self, comm, prob: Optional[FlatProblem], genotype: bool, timings: Optional[dict]):
        self.comm, self.prob, self.rank = comm, prob, comm.rank
        self.times = timings if timings is not None else {}
        self.T = None
        self._t = time.perf_counter()
        rows = None
        if self.rank == 0:
            mode, ranges = plan_parts(prob, comm.world, genotype, spans=_read_spans(prob) if prob.n_reads else None)
            ranges = ranges or [None] * comm.world
            head = np.array([_MODES.index(mode), prob.n_cols] + [x for r in ranges for x in (r or (0, 0))], np.int64).view(np.uint8)
            rows = [[head] + ([enc] if enc is not None else []) for enc in _wire.encode_problem_slices(prob, ranges)]
        self.mark("cut + encode")
        pieces = _wire.separate(comm.scatter_rows(rows))
        head = pieces[0].view(np.int64)
        self.mode, self.n_cols = _MODES[int(head[0])], int(head[1])
        self.ranges = [None if lo == hi else (int(lo), int(hi)) for lo, hi in head[2:].reshape(-1, 2)]
        self.mine = _wire.decode_problem(pieces[1])[0] if len(pieces) > 1 else None
        self.mark("scatter")

    def piece(self, i: int) -> FlatProblem:
        return self.prob if self.prob is not None and self.ranges[i] == (0, self.n_cols) else self.mine

    def run(self, step, name: str, share=None, then: Optional[str] = None) -> list:
        result, status = None, (0, "")
        if self.ranges[self.rank] is not None:
            try:
                result = step(self.rank)
            except Exception as e:  # noqa: BLE001 - reported to every rank below
                status = _wire.status_of(e)
        if then:
            self.mark(name)
        if share is None:
            states = self.comm.all_status(*status)
        else:
            dtype, dims = share
            if self.T is None:  # ranks without columns do not know T
                self.T = max(self.comm.lengths(4 ** self.mine.n_trios if self.mine is not None else 0))
            states = self.comm.all_status(*status, payload=None if result is None else np.ascontiguousarray(result, dtype),
                                          payload_width=np.dtype(dtype).itemsize * self.T ** dims)
        self.mark(then or name)
        if _wire.raise_first_error(states, name):
            raise Unsupported(next(text for kind, text, _ in states if kind == 1))
        if share is None:
            return [result if r == self.rank else None for r in range(len(self.ranges))]
        return [None if pl is None else pl.view(dtype).reshape((self.T,) * dims).copy() for _, _, pl in states]

    def collect(self, done: list, codec, name: str) -> Optional[list]:
        if any(self.ranges[1:]):  # (else only rank 0 holds columns: the whole table, nothing to gather)
            mine = done[self.rank]
            rows = self.comm.gather_rows(codec[0](mine) if mine is not None else np.zeros(0, np.uint8))
            done = None if rows is None else [codec[1](row) if row.size else None for row in rows]
        self.mark(name)
        return done if self.rank == 0 else None

    def mark(self, name: str) -> None:
        now = time.perf_counter()
        self.times[name] = (now - self._t) * 1e3
        self._t = now


def _current(fn):
    """`fn(..., device=d)` on this process's current CUDA device d."""
    import torch

    device = torch.cuda.current_device()
    return lambda *args: fn(*args, device=device)


def _run_parts(ex: _Local, mode: str, solver, segments) -> Tuple[list, str]:
    """Every part's result and the mode that ran: `segments()` in segment mode, else `solver(part, *device)` on every run of
    blocks, or on the whole table (whole mode, and segment mode when some segment is refused as unsupported in any phase)."""
    if mode == "segments":
        try:
            return segments(), mode
        except Unsupported:  # no part may leave its columns empty
            mode = "whole"
    if mode == "whole":
        ex.whole()
    return ex.run(lambda i: solver(ex.piece(i), *ex.on(i)), "solve"), mode


def _phasing_segments(ex: _Local, factory) -> list:
    """The phasing segments of `ex`: create (`factory(slice, continues, *device)`), transfer (T x T, shared), `segment_inputs`,
    sweep, exits (shared), `segment_entries`, finish.  Returns every part's (solution, statistics)."""
    segs: list = [None] * len(ex.ranges)
    last = max(i for i, r in enumerate(ex.ranges) if r is not None)

    def create(i):
        segs[i] = factory(ex.piece(i), ex.ranges[i][0] > 0, *ex.on(i))

    try:
        ex.run(create, "create")
        inputs = segment_inputs(ex.run(lambda i: segs[i].transfer(), "transfer", (np.uint32, 2), then="gather matrices"))
        ex.run(lambda i: segs[i].sweep(inputs[i]), "sweep")
        entries = segment_entries(ex.run(lambda i: segs[i].exits(i == last), "exits + gather", (np.uint32, 1)))
        return ex.run(lambda i: (segs[i].finish(entries[i]), _segment_stats(segs[i])), "finish")
    finally:
        ex.close(segs)


def _merged(ex: _Local, prob: FlatProblem, done: list, mode: str) -> Tuple[Optional[FlatSolution], Optional[list]]:
    """The parts' solutions merged in column order, and every part's statistics; (None, None) on ranks other than 0.  The
    last segment's cost is the table's; the costs of runs of blocks add."""
    parts = ex.collect(done, _SOLUTIONS, "gather results" if mode == "segments" else "gather")
    if parts is None:
        return None, None
    held = [(r, p[0]) for r, p in zip(ex.ranges, parts) if p is not None]
    sol = merge_block_solutions(prob, [r for r, _ in held], [s for _, s in held], cost=int(held[-1][1].cost) if mode == "segments" else None)
    if mode != "segments":
        ex.mark("merge")
    return sol, [None if p is None else dict(p[1] or {}) for p in parts]


def _genotype_segments(ex: _Local, factory) -> list:
    """The genotyping segments of `ex`: create (`factory(slice, continues, continued, *device)`), transfer (T x T, shared),
    `genotype_segment_inputs`, run.  Returns every part's (likelihoods, {"transfer": statistics, "run": statistics})."""
    segs: list = [None] * len(ex.ranges)

    def create(i):
        lo, hi = ex.ranges[i]
        segs[i] = factory(ex.piece(i), lo > 0, hi < ex.n_cols, *ex.on(i))

    try:
        ex.run(create, "create")
        alphas, betas = genotype_segment_inputs(ex.run(lambda i: segs[i].transfer(), "transfer", (np.float64, 2)))
        transfers = [_segment_stats(sg) for sg in segs]
        return ex.run(lambda i: (segs[i].run(alphas[i], betas[i]), {"transfer": transfers[i], "run": _segment_stats(segs[i])}), "run")
    finally:
        ex.close(segs)


def _likelihoods(ex: _Local, prob: FlatProblem, done: list) -> Tuple[Optional[np.ndarray], Optional[list]]:
    """The parts' likelihoods written into [n_ind, n_cols, 3], and every part's statistics; (None, None) on ranks other than 0."""
    parts = ex.collect(done, _LIKELIHOODS, "gather")
    if parts is None:
        return None, None
    out = np.zeros((prob.n_ind, prob.n_cols, 3), np.float64)
    for r, p in zip(ex.ranges, parts):
        if p is not None:
            out[:, r[0]:r[1], :] = np.reshape(p[0], (prob.n_ind, r[1] - r[0], 3))
    return out, [None if p is None else dict(p[1] or {}) for p in parts]


_SOLUTIONS = (lambda part: _wire.encode_solution(part[0]), lambda row: (_wire.decode_solution(row)[0], None))
_LIKELIHOODS = (lambda part: np.ascontiguousarray(part[0], np.float64).reshape(-1).view(np.uint8), lambda row: (row.view(np.float64), None))


def solve_pedigree_segments(prob: FlatProblem, n_segments: int, segment_factory=None) -> FlatSolution:
    """The multi-GPU pedigree scheme with all `n_segments` segments driven by ONE process on one
    device, in the order the ranks would run them -- the single-GPU check of `whmec_segment_*`
    (tests/test_gpu_sharded.py) and of this module's folding logic."""
    from . import _lib

    ex = _Local(prob, segment_ranges(prob, n_segments))
    return _merged(ex, prob, _phasing_segments(ex, segment_factory or _current(_lib.Segment)), "segments")[0]


def solve_sharded(prob: Optional[FlatProblem], solver: Optional[Callable[[FlatProblem], FlatSolution]] = None,
                  group=None, segment_factory=None, comm=None, timings: Optional[dict] = None) -> Optional[FlatSolution]:
    """Solve `prob` (given on rank 0; other ranks pass None) on all ranks of `group`.

    Rank 0 cuts the problem and SCATTERS the pieces — a rank receives only the columns and reads it works on (the
    "trivial broadcast of the block list" of the north_star, without shipping every rank the whole ReadSet): the blocks of
    its share for a single individual, its segment of the table for a pedigree.  The pieces travel as flat byte rows through
    tensor collectives (`_wire`), the per-block results come back the same way.  Returns the merged solution on rank 0 and
    None elsewhere; an error on any rank is raised on every rank, and so is a refusal (Unsupported) of a run of blocks or of
    the whole table.  A pedigree of one chain runs on rank 0's GPU, as does the whole table when any rank's segment is refused
    as unsupported in any phase.  `solver` / `segment_factory` default to the CUDA path on this rank's current device; tests
    inject CPU stand-ins to exercise the sharding logic with gloo.  `timings` (optional dict) receives this rank's per-phase
    wall times in ms."""
    from . import _lib

    if solver is None:
        solve = _current(_lib.solve)
        solver = lambda p: solve(p)[0]  # noqa: E731
    ex = _Ranks(comm or _wire.Comm(group), prob, False, timings)
    done, mode = _run_parts(ex, ex.mode, lambda p: (solver(p), None), lambda: _phasing_segments(ex, segment_factory or _current(_lib.Segment)))
    sol = _merged(ex, prob, done, mode)[0]
    if ex.rank == 0 and mode == "segments" and os.environ.get("WHMEC_TIMING"):
        print("[whmec] pedigree segments, rank 0: " + ", ".join("%s %.1f ms" % kv for kv in list(ex.times.items())[2:]), flush=True)
    return sol


def genotype_pedigree_segments(prob: FlatProblem, n_segments: int, segment_factory=None) -> np.ndarray:
    """The multi-GPU pedigree genotyping scheme with all `n_segments` segments driven by ONE process on one device, in the
    order the ranks would run them: transfer matrices, the fold, then every segment's run.  Returns [n_ind, n_cols, 3]."""
    from . import _lib

    ex = _Local(prob, segment_ranges(prob, n_segments))
    return _likelihoods(ex, prob, _genotype_segments(ex, segment_factory or _current(_lib.GenotypeSegment)))[0]


def genotype_sharded(prob: Optional[FlatProblem], solver: Optional[Callable[[FlatProblem], np.ndarray]] = None,
                     group=None, comm=None, segment_factory=None) -> Optional[np.ndarray]:
    """Genotype likelihoods (`whmec_genotype`, the reference's GenotypeDPTable) of `prob` (given on rank 0; other ranks
    pass None) on all ranks of `group`; returns [n_ind, n_cols, 3] on rank 0, None elsewhere.

    Without transmission values every DP-independent chain is a forward-backward table of its own (a chain boundary hands
    over one number, which cancels in each column's normalisation), so a single individual shards like the phasing DP:
    every rank takes a contiguous run of whole chains balanced by DP cells, no collective on the data path, likelihoods
    gathered on rank 0.  A pedigree with two chains or more is cut into segments of whole chains (`segment_ranges`), one
    per rank: one all-gather of the T x T transfer matrices, the fold (`genotype_segment_inputs`), every rank runs its
    segment, likelihoods gathered on rank 0.  A pedigree of one chain runs on rank 0's GPU, as does the whole table when
    any rank's segment is refused as unsupported in any phase.  A refusal of the table on one GPU is raised as Unsupported on
    every rank.  `solver` / `segment_factory` default to the CUDA path on this rank's
    current device.  Errors are raised on every rank."""
    from . import _lib

    if solver is None:
        genotype = _current(_lib.genotype)
        solver = lambda p: genotype(p)[0]  # noqa: E731
    ex = _Ranks(comm or _wire.Comm(group), prob, True, None)
    done, _ = _run_parts(ex, ex.mode, lambda p: (solver(p), None), lambda: _genotype_segments(ex, segment_factory or _current(_lib.GenotypeSegment)))
    return _likelihoods(ex, prob, done)[0]


# ---- one process, several devices ---------------------------------------------------------------------------------
#
# The same cuts and schemes as the distributed drivers above, for a caller that is a single process (`whatshap phase` and
# `whatshap genotype` build one table at a time): one host thread per distinct device runs that device's parts through the
# C ABI, which is re-entrant, sets the device on the calling thread and releases the GIL (ctypes); the folds between
# phases run on the calling thread.

ENV_DEVICES = "WHMEC_DEVICES"


def _segment_stats(seg) -> dict:
    st = getattr(seg, "stats", None)  # `_lib.Segment.stats()`, `_lib.GenotypeSegment.stats` (its last call)
    return dict(st() if callable(st) else st or {})


def _part_stats(mode: str, devices: Sequence[int], ranges, stats) -> dict:
    return {"mode": mode, "devices": list(devices),
            "parts": [{"device": d, "columns": r, "stats": st} for d, r, st in zip(devices, ranges, stats) if r is not None]}


def solve_on_devices(prob: FlatProblem, devices: Sequence[int], solver=None, segment_factory=None) -> Tuple[FlatSolution, dict]:
    """`solve_sharded` in one process: one part of `prob` per entry of `devices`, in column order (`plan_parts`); the
    same solution as `whmec_solve` on one device.  A single individual is cut into runs of whole chains, each solved by
    `solver(part, device)`; a pedigree of two chains or more into segments of the table, driven phase by phase (create,
    transfer, `segment_inputs`, sweep, exits, `segment_entries`, finish, `merge_block_solutions`).  Runs whole on
    `devices[0]`: a pedigree of one chain, a problem without columns, and a table some segment of which is refused as
    unsupported while it is created or run.  An error is raised after every part has stopped and every segment is closed:
    that of the part with the lowest column (a refusal only when the whole table is refused too).  A device may repeat:
    its parts run one after another.  `solver(prob, device) -> (FlatSolution, stats)` defaults to `_lib.solve`,
    `segment_factory(prob, continues, device)` to `_lib.Segment`.  Returns (solution, stats): the mode, the devices and
    every part's device, column range and statistics."""
    from . import _lib

    devices = [int(d) for d in devices]
    mode, ranges = plan_parts(prob, len(devices))
    ex = _Threads(prob, ranges, devices, mode == "segments")
    done, mode = _run_parts(ex, mode, solver or _lib.solve, lambda: _phasing_segments(ex, segment_factory or _lib.Segment))
    sol, stats = _merged(ex, prob, done, mode)
    return sol, _part_stats(mode, devices, ex.ranges, stats)


def genotype_on_devices(prob: FlatProblem, devices: Sequence[int], solver=None, segment_factory=None) -> Tuple[np.ndarray, dict]:
    """`genotype_sharded` in one process: likelihoods [n_ind, n_cols, 3] with one part of `prob` per entry of `devices`, in
    column order (`plan_parts`).  A single individual is cut into runs of whole chains, each genotyped by
    `solver(part, device)`; a pedigree of two chains or more into segments of the table (create, transfer,
    `genotype_segment_inputs`, run).  Runs whole on `devices[0]`: one device, a pedigree of one chain, a problem without
    columns, and a table some segment of which is refused as unsupported while it is created, transferred or run.  Errors,
    repeated devices and the result's statistics as in `solve_on_devices`.  `solver(prob, device) -> (likelihoods, stats)`
    defaults to `_lib.genotype`, `segment_factory(prob, continues, continued, device)` to `_lib.GenotypeSegment`."""
    from . import _lib

    devices = [int(d) for d in devices]
    mode, ranges = plan_parts(prob, len(devices), genotype=True)
    ex = _Threads(prob, ranges, devices, mode == "segments")
    done, mode = _run_parts(ex, mode, solver or _lib.genotype, lambda: _genotype_segments(ex, segment_factory or _lib.GenotypeSegment))
    out, stats = _likelihoods(ex, prob, done)
    return out, _part_stats(mode, devices, ex.ranges, stats)



def parse_devices(text: str) -> List[int]:
    """The CUDA ordinals of a WHMEC_DEVICES value ("0,1,2,3"); ValueError naming the variable when it is malformed."""
    items = [t.strip() for t in text.split(",")]
    if not all(t.isascii() and t.isdigit() for t in items):
        raise ValueError("%s=%r: expected comma-separated CUDA device ordinals, e.g. 0,1,2,3" % (ENV_DEVICES, text))
    return [int(t) for t in items]


def table_devices(device: int = 0, devices: Optional[Sequence[int]] = None) -> Optional[List[int]]:
    """The devices one table runs on: `devices`, else the ordinals of WHMEC_DEVICES, else None (the table runs on `device`
    alone, as before there was a choice).  A non-default `device` is kept over WHMEC_DEVICES: code that names a device
    runs there.  ValueError for both a non-default `device` and `devices`, an empty list, a malformed WHMEC_DEVICES and an
    ordinal that is not a visible CUDA device."""
    import os

    from . import _lib

    if devices is not None and device != 0:
        raise ValueError("give either device=%r or devices=%r, not both" % (device, devices))
    if devices is None:
        text = os.environ.get(ENV_DEVICES, "").strip()
        if not text or device != 0:
            return None
        devices = parse_devices(text)
    chosen = list(devices)
    if not chosen:
        raise ValueError("devices: expected at least one CUDA device ordinal")
    count = None
    for d in chosen:
        if isinstance(d, bool) or not isinstance(d, (int, np.integer)) or d < 0:
            raise ValueError("device ordinal %r is not a non-negative integer" % (d,))
        count = _lib.device_count() if count is None else count
        if d >= count:
            raise ValueError("device ordinal %d is not a visible CUDA device (%d visible)" % (d, count))
    return [int(d) for d in chosen]


def solve_table(prob: FlatProblem, device: int = 0, devices: Optional[Sequence[int]] = None) -> Tuple[FlatSolution, dict]:
    """What `core.PedigreeDPTable` and the swap-in class of `adapters` run: `_lib.solve` on `device`, or
    `solve_on_devices` over `devices` / WHMEC_DEVICES (`table_devices`)."""
    from . import _lib

    chosen = table_devices(device, devices)
    return _lib.solve(prob, device=device) if chosen is None else solve_on_devices(prob, chosen)


def genotype_table(prob: FlatProblem, device: int = 0, devices: Optional[Sequence[int]] = None) -> Tuple[np.ndarray, dict]:
    """What `core.GenotypeDPTable` and the swap-in class of `adapters` run: `_lib.genotype` on `device`, or
    `genotype_on_devices` over `devices` / WHMEC_DEVICES (`table_devices`)."""
    from . import _lib

    chosen = table_devices(device, devices)
    return _lib.genotype(prob, device=device) if chosen is None else genotype_on_devices(prob, chosen)


def _tables(problems: Sequence[FlatProblem], device: int, devices: Optional[Sequence[int]], with_stats: bool, batch, single, weight):
    """The driver of `solve_tables` and `genotype_tables`: `batch(problems, device)` -> (results, (per-table stats, totals)) runs
    a list on one device, `single(problem, device, devices)` -> (result, stats) one table over several devices, and
    `weight(problem)` is the work by which whole tables go to devices (longest-processing-time-first, `assign_blocks`)."""
    problems = list(problems)
    chosen = table_devices(device, devices)
    distinct = sorted(set(chosen)) if chosen is not None else [device]
    out: list = [None] * len(problems)
    stats: list = [{} for _ in problems]
    if len(problems) == 1 and len(distinct) > 1:
        try:
            out[0], stats[0] = single(problems[0], device, devices)
        except RuntimeError as e:  # MendelianConflict, input errors, Unsupported: the table's result
            if str(e).startswith("CUDA failure"):
                raise
            out[0] = e
    elif len(distinct) == 1 or not problems:
        out, (stats, _) = batch(problems, distinct[0])
    else:
        shares = assign_blocks(np.array([weight(p) for p in problems]), len(distinct))
        jobs = [(lambda ids=ids, d=d: batch([problems[i] for i in ids], d)) if ids else None for ids, d in zip(shares, distinct)]
        results, errors = _run_on_devices(distinct, jobs)
        for e in errors:
            if e is not None:
                raise e
        for ids, res in zip(shares, results):
            if res is not None:
                for i, r, st in zip(ids, res[0], res[1][0]):
                    out[i], stats[i] = r, st
    return (out, stats) if with_stats else out


def solve_tables(problems: Sequence[FlatProblem], device: int = 0, devices: Optional[Sequence[int]] = None, with_stats: bool = False):
    """Several tables at once: per table, in input order, its `FlatSolution` or the exception `solve_table` would have raised
    for it (an input error, a Mendelian conflict, a refusal; a failure of the device raises, whatever the length of the list).
    On one device this is `_lib.solve_batch` (tables share the GPU's sweeps).  With `devices` / WHMEC_DEVICES whole tables go
    to devices by longest-processing-time-first on their DP cells sum 2^a * T (`block_work`, `assign_blocks`), one
    `whmec_solve_batch` per device on that device's host thread.  A single table behaves like `solve_table`, including being
    spread over the devices.  `with_stats`: (results, per-table stats) instead."""
    from . import _lib

    return _tables(problems, device, devices, with_stats, lambda ps, d: _lib.solve_batch(ps, device=d, with_stats=True),
                   lambda p, dev, devs: solve_table(p, dev, devs),
                   lambda p: float(block_work(p, [(0, p.n_cols)])[0]) * 4.0 ** p.n_trios)


def genotype_tables(problems: Sequence[FlatProblem], device: int = 0, devices: Optional[Sequence[int]] = None, with_stats: bool = False):
    """Several genotyping tables at once: per table, in input order, its likelihoods [n_ind, n_cols, 3] or the exception
    `genotype_table` would have raised for it (a failure of the device raises, whatever the length of the list).  On one device
    this is `_lib.genotype_batch` (tables share the GPU's launches).  With `devices` / WHMEC_DEVICES whole tables go to devices
    by longest-processing-time-first on sum 2^a * T * 2^P (`block_work`, `assign_blocks`), one `whmec_genotype_batch` per
    device on that device's host thread.  A single table behaves like `genotype_table`, including being spread over the
    devices.  `with_stats`: (results, per-table stats) instead."""
    from . import _lib

    return _tables(problems, device, devices, with_stats, lambda ps, d: _lib.genotype_batch(ps, device=d, with_stats=True),
                   lambda p, dev, devs: genotype_table(p, dev, devs),
                   lambda p: float(block_work(p, [(0, p.n_cols)])[0]) * 4.0 ** p.n_trios * 2.0 ** (2 * (p.n_ind - p.n_trios)))


def heuristic_tables(problems: Sequence[FlatProblem], row_limits=256, allow_mutations=True, device: int = 0,
                     devices: Optional[Sequence[int]] = None, with_stats: bool = False):
    """Several heuristic tables at once: per table, in input order, its `HeuristicSolution` or the exception `_lib.heuristic` would
    have raised for it (a failure of the device raises, whatever the length of the list).  `row_limits` / `allow_mutations`: per
    table, or one value for all.  On one device this is `_lib.heuristic_batch` (one CTA per table).  With `devices` /
    WHMEC_DEVICES whole tables go to devices by longest-processing-time-first on columns x row_limit (`assign_blocks`), one
    `whmec_heuristic_batch` per device on that device's host thread; a single table runs on the first device.  `with_stats`:
    (results, per-table stats) instead."""
    from . import _lib

    problems = list(problems)
    n = len(problems)
    limits = [int(row_limits)] * n if isinstance(row_limits, (int, np.integer)) else [int(r) for r in row_limits]
    allow = [bool(allow_mutations)] * n if isinstance(allow_mutations, (bool, int, np.integer)) else [bool(a) for a in allow_mutations]
    if len(limits) != n or len(allow) != n:
        raise ValueError("row_limits and allow_mutations need one entry per table")

    # the driver sees table positions, so that every table keeps its own row limit and flag
    def batch(ids, d):
        return _lib.heuristic_batch([problems[i] for i in ids], [limits[i] for i in ids], [allow[i] for i in ids], device=d, with_stats=True)

    def single(i, dev, devs):
        chosen = table_devices(dev, devs)
        res, (st, _) = batch([i], chosen[0] if chosen else dev)
        if isinstance(res[0], BaseException):
            raise res[0]
        return res[0], st[0]

    return _tables(list(range(n)), device, devices, with_stats, batch, single,
                   lambda i: float(problems[i].n_cols) * max(1, min(limits[i], 65535)))


def batch_heuristic_objects(cls, tables, setup, device: int, devices: Optional[Sequence[int]], return_exceptions: bool) -> list:
    """The `batch` classmethods of the PedMecHeuristic classes: `setup(obj, args)` does the constructor's work up to the solver
    for one argument tuple `(readset, recombcost, pedigree[, row_limit[, distrust_genotypes[, positions[, allow_mutations[,
    verbosity]]]]])`, then every table's row limit (capped to 0..65535, as the constructor does) and flag go with its problem
    to `heuristic_tables`.  Errors as in `batch_objects`."""
    options: list = []

    def build(obj, args):
        setup(obj, args)
        row_limit = min(max(int(args[3]), 0), 65535) if len(args) > 3 else 256
        options.append((row_limit, bool(args[6]) if len(args) > 6 else True))

    return batch_objects(cls, tables, build, lambda problems: heuristic_tables(problems, [o[0] for o in options], [o[1] for o in options], device,
                                                                               devices, with_stats=True), "_solution", return_exceptions)


def batch_objects(cls, tables, build, run, attr: str, return_exceptions: bool) -> list:
    """The `batch` classmethods of the table classes: one `cls` object per constructor argument tuple of `tables`
    (`build(obj, args)` fills it; an exception it raises takes the table's place), `run(problems)` -> (results, per-table stats or
    None) over the `_problem` of every built object, each result stored in the object's `attr` (and its stats in `stats`) or,
    when it is an exception, in the table's place.  Then `finish_batch`."""
    objs: list = []
    for args in tables:
        try:
            obj = cls.__new__(cls)
            build(obj, args)
            objs.append(obj)
        except Exception as e:  # noqa: BLE001 - reported in the table's place, after the others ran
            objs.append(e)
    good = [i for i, o in enumerate(objs) if not isinstance(o, BaseException)]
    results, stats = run([objs[i]._problem for i in good])
    for n, (i, res) in enumerate(zip(good, results)):
        if isinstance(res, BaseException):
            objs[i] = res
        else:
            setattr(objs[i], attr, res)
            if stats is not None:
                objs[i].stats = stats[n]  # (times are 0: the tables shared their launches)
    finish_batch(objs, return_exceptions)
    return objs


def finish_batch(results: list, return_exceptions: bool) -> None:
    """The error contract of the `batch` classmethods: without `return_exceptions`, the error of the lowest-index failing table."""
    if not return_exceptions:
        for r in results:
            if isinstance(r, BaseException):
                raise r
