"""A pedigree's genotyping table split into segments of whole chains (DESIGN §4.5, `whmec_genotype_segment_*`) without a GPU:
the segments' transfer passes and runs are stepped on the host by tests/emul/libwhemul_gl_segment.so (the kernels' per-cell code
and the host plans), the matrices folded by `multigpu.genotype_segment_inputs`.  The segmented likelihoods must agree with the
whole table (emul_genotype) to 1e-11, with the C restatement and the reference's golden vectors to 1e-9 (the tolerance of
test_genotype.py), with NaN (a column of zero mass) in the same places."""
import os
import re
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import emul_genotype
import emul_genotype_segment
from oracle import checker
from test_genotype import golden
from whatshap_b200 import multigpu, synth
from whatshap_b200._abi import Unsupported

TOL_WHOLE = 1e-11
TOL_DEVICE = 1e-9
PEDS = ["trio", "quartet", "three_generations", "trio_child_first", "three_children", "four_children"]


def close(a, b, tol):
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and bool(np.all((np.abs(a - b) <= tol) | np.isnan(a)))


def instance(ped, prior, seed, n_cols=60):
    """A table of several chains; recombination costs 0 (every transmission bit flips) and >= 200 (none does) included."""
    for attempt in range(100):
        rng = np.random.Generator(np.random.PCG64([seed, attempt]))
        prob = synth.genotyping_problem(rng, n_cols, 3 if ped == "four_children" else 4, ped, prior=prior, gap=0.04, mean_len=3.0)
        if len(multigpu.independent_blocks(prob)) >= 4:
            break
    special = rng.random(prob.n_cols)
    prob.recombcost = np.where(special < 0.15, 0, np.where(special > 0.85, rng.integers(200, 400, prob.n_cols), prob.recombcost)).astype(np.uint32)
    return prob


def segmented(prob, n_segments, **kw):
    return multigpu.genotype_pedigree_segments(prob, n_segments, segment_factory=lambda p, a, b: emul_genotype_segment.Segment(p, a, b, **kw))


@pytest.mark.parametrize("ped", PEDS)
@pytest.mark.parametrize("prior", ["uniform", "random", "sparse"])
def test_segments_match_the_whole_table(ped, prior):
    prob = instance(ped, prior, PEDS.index(ped) * 3 + ["uniform", "random", "sparse"].index(prior))
    chains = len(multigpu.independent_blocks(prob))
    assert chains >= 3, chains
    whole, _ = emul_genotype.genotype(prob)
    port = checker.port().genotype(prob)
    assert close(whole, port, TOL_DEVICE)
    for n_segments in sorted({2, 3, 5, chains}):
        got = segmented(prob, n_segments)
        assert close(got, whole, TOL_WHOLE), (ped, prior, n_segments, float(np.nanmax(np.abs(got - whole))))
        assert close(got, port, TOL_DEVICE), (ped, prior, n_segments)


def test_golden_vectors_segmented():
    """The reference's answers for every golden pedigree vector with two chains or more, cut into 2 segments and one per chain."""
    n = 0
    for label, prob, want, _ in golden():
        chains = len(multigpu.independent_blocks(prob))
        if prob.n_trios == 0 or chains < 2:
            continue
        for n_segments in sorted({2, chains}):
            got = segmented(prob, n_segments)
            assert close(got, want, TOL_DEVICE), (label, n_segments, float(np.nanmax(np.abs(got - want))))
        n += 1
    assert n >= 5, n


def test_bounded_segment_runs():
    """A segment whose backward tables exceed the budget runs in memory-bounded mode (beta_in is its last checkpoint) and gives
    what the resident segment gives."""
    prob = instance("quartet", "random", 41, n_cols=90)
    whole = segmented(prob, 3)
    ranges = multigpu.segment_ranges(prob, 3)
    lo, hi = ranges[1]
    assert 0 < lo and hi < prob.n_cols
    seg = emul_genotype_segment.Segment(prob.slice_columns(lo, hi), True, True, budget_doubles=1)
    with pytest.raises(Unsupported, match=r"needs at least \d+ bytes") as e:
        seg.run(np.ones(16), np.ones(16))
    seg.close()
    least = int(re.search(r"needs at least (\d+) bytes", str(e.value)).group(1)) // 8
    seen = set()
    for budget in (least, 2 * least, 4 * least, 1 << 40):
        seg = emul_genotype_segment.Segment(prob.slice_columns(lo, hi), True, True, budget_doubles=budget)
        try:
            mats = []
            for r in ranges:
                s = emul_genotype_segment.Segment(prob.slice_columns(*r), r[0] > 0, r[1] < prob.n_cols)
                mats.append(s.transfer())
                s.close()
            alphas, betas = multigpu.genotype_segment_inputs(mats)
            got = seg.run(alphas[1], betas[1])
            seen.add(seg.stats["segments"])
        finally:
            seg.close()
        assert close(got, whole[:, lo:hi], 1e-12), budget
    assert max(seen) > 1 and min(seen) == 1, seen


def test_founder_symmetry_of_trio_matrices():
    """Swapping a founder's two haplotypes flips its transmission bit: M[u ^ m][i ^ m] = M[u][i] for every mask m."""
    prob = instance("trio", "random", 5)
    ranges = multigpu.segment_ranges(prob, 4)
    checked = 0
    for r in ranges:
        seg = emul_genotype_segment.Segment(prob.slice_columns(*r), r[0] > 0, r[1] < prob.n_cols)
        m = seg.transfer()
        seg.close()
        assert m.max() > 0
        for mask in (1, 2, 3):
            perm = np.arange(4) ^ mask
            assert np.allclose(m[np.ix_(perm, perm)], m, rtol=1e-12, atol=1e-12 * m.max()), (r, mask)
        checked += 1
    assert checked == 4


def test_fold_handles_zero_rows_and_ranks_without_columns():
    rng = np.random.default_rng(3)
    a, b, c = rng.random((3, 4, 4))
    b[1] = 0.0  # an input that leaves no mass
    alphas, betas = multigpu.genotype_segment_inputs([a, None, b, None, c])
    assert alphas[1] is None and betas[1] is None and alphas[3] is None and betas[3] is None
    assert alphas[0] is None and betas[4] is None
    scaled = lambda v: v / v.max()
    assert np.allclose(alphas[2], scaled(a[0])) and np.allclose(alphas[4], scaled(scaled(a[0]) @ b))
    assert np.allclose(betas[2], scaled(c.sum(axis=1))) and np.allclose(betas[0], scaled(b @ scaled(c.sum(axis=1))))
    assert betas[0][1] == 0.0 and np.all(np.isfinite(betas[0]))
    zero = np.zeros((4, 4))  # a segment with no mass at all: the vectors behind it stay 0 instead of turning into NaN
    alphas, betas = multigpu.genotype_segment_inputs([a, zero, c])
    assert np.all(alphas[2] == 0.0) and np.all(betas[0] == 0.0)
    alphas, betas = multigpu.genotype_segment_inputs([None, a, None])
    assert alphas == [None, None, None] and betas == [None, None, None]


def test_misuse_is_refused():
    single = synth.genotyping_problem(np.random.default_rng(1), 20, 4, "single")
    with pytest.raises(Unsupported, match="independent tables"):
        emul_genotype_segment.Segment(single, True, True)
    prob = instance("trio", "random", 9)
    lo, hi = multigpu.segment_ranges(prob, 3)[1]
    seg = emul_genotype_segment.Segment(prob.slice_columns(lo, hi), True, True)
    try:
        with pytest.raises(RuntimeError, match="needs alpha_in"):
            seg.run(None, np.ones(4))
        with pytest.raises(RuntimeError, match="needs beta_in"):
            seg.run(np.ones(4), None)
    finally:
        seg.close()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, ped, out_queue):
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here))
    sys.path.insert(0, here)
    import emul_genotype
    import emul_genotype_segment

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    prob = instance(ped, "random", 17) if rank == 0 else None
    got = multigpu.genotype_sharded(prob, solver=lambda p: emul_genotype.genotype(p)[0], segment_factory=emul_genotype_segment.Segment)
    if rank == 0:
        want = multigpu.genotype_pedigree_segments(prob, world, segment_factory=emul_genotype_segment.Segment)
        out_queue.put((bool(np.array_equal(got, want, equal_nan=True)), len(multigpu.independent_blocks(prob))))
    else:
        assert got is None
    dist.destroy_process_group()


@pytest.mark.parametrize("ped,world", [("trio", 2), ("quartet", 3)])
def test_sharded_equals_single_process(ped, world):
    """Every gloo rank runs its emulated segment; the gathered likelihoods equal the single-process driver's exactly."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, ped, q)) for r in range(world)]
    for p in procs:
        p.start()
    same, chains = q.get(timeout=180)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert same and chains > world


def _unsupported_worker(rank, world, port, where, out_queue):
    """Rank 1's segment refuses as unsupported in `where` (its run finds no room for its backward tables, or its transfer pass is
    refused); `whole_too`: the whole table is refused as well, as the single-GPU call would refuse it."""
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here))
    sys.path.insert(0, here)
    import emul_genotype
    import emul_genotype_segment

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)

    class Refusing(emul_genotype_segment.Segment):
        def transfer(self):
            if where == "transfer":
                raise Unsupported("unsupported problem: transfer refused")
            return super().transfer()

    def factory(p, continues, continued):
        if rank != 1:
            return emul_genotype_segment.Segment(p, continues, continued)
        return Refusing(p, continues, continued, budget_doubles=1 if where.startswith("run") else 1 << 62)

    def solver(p):
        if where == "run_whole_too":
            raise Unsupported("unsupported problem: whole table refused")
        return emul_genotype.genotype(p)[0]

    prob = instance("trio", "random", 17) if rank == 0 else None
    try:
        got = multigpu.genotype_sharded(prob, solver=solver, segment_factory=factory)
    except Unsupported as e:
        out_queue.put((rank, "raised", str(e)))
    else:
        if rank == 0:
            out_queue.put((rank, bool(np.array_equal(got, emul_genotype.genotype(prob)[0], equal_nan=True)), ""))
        else:
            out_queue.put((rank, got is None, ""))
    dist.destroy_process_group()


@pytest.mark.parametrize("where", ["run", "transfer", "run_whole_too"])
def test_unsupported_segment_falls_back_to_the_whole_table(where):
    """A segment refused as unsupported on one rank never leaves its columns empty: every rank falls back to the whole table on
    rank 0, which gives the whole table's likelihoods or raises the single-GPU call's refusal on every rank."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_unsupported_worker, args=(r, 2, port, where, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = sorted(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    if where == "run_whole_too":
        assert all(r[1] == "raised" and "whole table refused" in r[2] for r in results), results
    else:
        assert all(r[1] is True for r in results), results


def test_long_segments_with_batched_inputs():
    """T = 64: the transfer pass runs 4 batches of 16 inputs, each with its own scale per column, over segments of hundreds of
    columns; the products of those scales put the batches' rows on one scale without losing precision."""
    prob = instance("three_children", "random", 23, n_cols=1200)
    chains = len(multigpu.independent_blocks(prob))
    assert chains >= 3, chains
    whole, _ = emul_genotype.genotype(prob)
    for n_segments in (2, 3):
        got = segmented(prob, n_segments)
        assert close(got, whole, TOL_WHOLE), (n_segments, float(np.nanmax(np.abs(got - whole))))
