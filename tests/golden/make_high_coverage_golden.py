"""Generates tests/golden/high_coverage.npz: single-individual instances at coverage 21-25 and the answers of the UNMODIFIED
reference C++ PedigreeDPTable (oracle/_ref/libwhref.so) on them, in the format of make_golden.py (read by golden_io.load).
Run on a machine with the reference:  python tests/golden/make_high_coverage_golden.py

At these coverages the tile kernel hands the state from panel to panel in small chunks (under 128 bytes, gathered element by
element; 2^13 or 2^14-entry tiles, up to 2^10 tiles per panel), into steady and into non-steady panels, mirrored with km = 0
(even coverage) and km != 0 (odd coverage).  The reference needs tens of nanoseconds per DP cell, too slow to run in the GPU
tests at these sizes, so its answers are stored.  tests/test_high_coverage_golden.py checks with the planner that the
instances still reach those paths; tests/test_gpu_high_coverage.py holds the tile kernel to the stored answers.

Instances
  sliding/c=21..25          one chain each: coverage 21 (the last bulk-copy hand-off: 2^6 producer tiles) up to 25 (cfg4)
  ragged/c=22               600 columns in chains of Geometric(mean 60) length: many chains of one sweep at once
  ties/c=23                 phred 1-2, 10 % interior gaps, about 10 % homozygous sites: tie-heavy, non-steady panels
  irregular/c=23            random spans, blanks and homozygous sites: canonical hand-offs at coverage 23
  one_read_then/c=23        a one-read chain in front of a coverage-23 chain (state buffers of the second chain behind 2 words)

Measured on one 8-core x86-64 machine: 1474 s of the reference's CPU time in all (29 s for coverage 21 x 80 columns, 381 s for
coverage 25 x 60, 467 s for the ragged table; 100-190 ns per DP cell), 7.8 minutes of wall time with 6 worker processes, and
up to 6 GB of memory in one process.
"""
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import PROBLEM_FIELDS, SOLUTION_FIELDS  # noqa: E402
from oracle import checker  # noqa: E402
from whatshap_b200 import synth  # noqa: E402
from whatshap_b200._abi import FlatProblem  # noqa: E402

OUT = os.path.join(HERE, "high_coverage.npz")


def active_reads(prob):
    """Reads active in every column (from the column of a read's first entry to that of its last one)."""
    off = prob.read_off.astype(np.int64)
    first, last = prob.ent_col[off[:-1]].astype(np.int64), prob.ent_col[off[1:] - 1].astype(np.int64)
    starts = np.bincount(first, minlength=prob.n_cols + 1) - np.bincount(last + 1, minlength=prob.n_cols + 1)
    return np.cumsum(starts)[:-1]


def _with_homozygous_sites(prob, rate, seed):
    rng = np.random.default_rng(seed)
    prob.gt = prob.gt.copy()
    prob.gt[0, rng.random(prob.n_cols) < rate] = 0
    return prob


def _one_read_chain_in_front(prob, seed):
    """`prob` behind a two-column chain of one read (columns 0 and 1)."""
    rng = np.random.default_rng(seed)
    n = prob.n_cols + 2
    return FlatProblem(
        positions=(np.arange(n, dtype=np.uint32) + 1) * 1000,
        read_off=np.concatenate([[0], prob.read_off.astype(np.uint64) + 2]).astype(np.uint64),
        ent_col=np.concatenate([[0, 1], prob.ent_col.astype(np.int64) + 2]).astype(np.uint32),
        ent_allele=np.concatenate([rng.integers(0, 2, 2), prob.ent_allele]).astype(np.uint8),
        ent_phred=np.concatenate([rng.integers(1, 41, 2), prob.ent_phred]).astype(np.uint32),
        read_ind=np.zeros(prob.n_reads + 1, np.uint32),
        recombcost=np.concatenate([[0, 49], prob.recombcost]).astype(np.uint32),
        n_ind=1,
        distrust=False,
        gt=np.ones((1, n), np.uint8),
    )


def cases():
    out = []
    for cov, n in ((21, 80), (22, 80), (23, 80), (24, 60), (25, 60)):
        out.append((f"sliding/n={n}/c={cov}", synth.sliding_window(n, cov, block_len=n, seed=2026 + cov)))
    out.append(("ragged/n=600/c=22/mean=60", synth.sliding_window(600, 22, block_len=synth.geometric_blocks(600, 60.0, 22), seed=22)))
    ties = synth.sliding_window(70, 23, block_len=70, seed=300, gap=0.1, max_phred=2)
    out.append(("ties/n=70/c=23/phred<=2/gap/hom", _with_homozygous_sites(ties, 0.1, 0)))
    out.append(("irregular/n=60/c<=23", synth.random_problem(np.random.default_rng(0), 60, 23, "single", max_phred=2, mean_len=24.0,
                                                             gap=0.1, burst=6, hom_rate=0.1)))
    out.append(("one_read_then/n=62/c=23", _one_read_chain_in_front(synth.sliding_window(60, 23, block_len=60, seed=523), seed=1)))
    return out


def _solve(prob):
    t0 = time.process_time()
    sol = checker.reference().solve(prob)
    return sol, time.process_time() - t0


def main(workers):
    assert checker.reference() is not None, "the compiled reference (oracle/_ref) is required: the C restatement is not a reference"
    todo = cases()
    order = sorted(range(len(todo)), key=lambda i: -np.sum(2.0 ** active_reads(todo[i][1])))  # most DP cells first
    with ProcessPoolExecutor(workers) as ex:
        futures = {i: ex.submit(_solve, todo[i][1]) for i in order}
        sols = {i: f.result() for i, f in futures.items()}
    data = {"n": np.array(len(todo))}
    cpu = 0.0
    for i, (label, prob) in enumerate(todo):
        sol, secs = sols[i]
        cpu += secs
        print(f"{label}: cost {sol.cost}, {secs:.1f} s", flush=True)
        data[f"{i}.label"] = np.array(label)
        data[f"{i}.n_ind"] = np.array(prob.n_ind)
        data[f"{i}.distrust"] = np.array(int(prob.distrust))
        for f in PROBLEM_FIELDS:
            v = getattr(prob, f)
            if v is not None:
                data[f"{i}.{f}"] = v
        data[f"{i}.error"] = np.array("")
        data[f"{i}.cost"] = np.array(sol.cost, np.uint32)
        for f in SOLUTION_FIELDS:
            data[f"{i}.{f}"] = getattr(sol, f)
    np.savez_compressed(OUT, **data)
    print(f"{len(todo)} cases -> {OUT}, {os.path.getsize(OUT)} bytes; reference CPU time {cpu:.0f} s")


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 6)
