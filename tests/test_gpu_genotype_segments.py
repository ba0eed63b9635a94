"""A pedigree's genotyping table split into segments of whole chains on the GPU (DESIGN §4.5, `whmec_genotype_segment_*`):
every segment on cuda:0, driven by `multigpu.genotype_pedigree_segments` in one process or by `genotype_sharded` over gloo
ranks that share the device.  The likelihoods must agree with `whmec_genotype` on the whole table, with the C restatement and
with the reference's golden vectors to 1e-9 (the double atomicAdd makes even two whole-table runs differ in the last bits)."""
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import emul_genotype_segment
from oracle import checker
from test_genotype import golden
from test_genotype_segments import PEDS, instance
from whatshap_b200 import _lib, multigpu, synth

pytestmark = pytest.mark.gpu

TOL = 1e-9
HOOK = "WHMEC_GENOTYPE_ARENA_BUDGET"


def close(a, b):
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and bool(np.all((np.abs(a - b) <= TOL) | np.isnan(a)))


def trio_problem(cols, c_per_sample, block_len, seed):
    rng = np.random.default_rng(seed)
    prob = synth.trio(cols, c_per_sample, block_len=block_len, seed=seed)
    prob.gl = rng.random((3, prob.n_cols, 3)) + 0.05
    prob.gl /= prob.gl.sum(axis=2, keepdims=True)
    prob.recombcost = rng.integers(0, 30, prob.n_cols).astype(np.uint32)
    prob.distrust = True
    return prob


@pytest.fixture(autouse=True)
def no_hook(monkeypatch):
    monkeypatch.delenv(HOOK, raising=False)


@pytest.mark.parametrize("n_segments", [2, 3, 8])
def test_trio_matches_the_whole_table_and_the_restatement(n_segments):
    prob = trio_problem(600, 3, 40, 1)
    whole, _ = _lib.genotype(prob)
    got = multigpu.genotype_pedigree_segments(prob, n_segments)
    assert close(got, whole), float(np.nanmax(np.abs(got - whole)))
    assert close(got, checker.best().genotype(prob))


def test_cfg5_shaped_trio():
    """15 reads per column, 4 000 columns (8 chains of 500), random priors."""
    prob = trio_problem(4000, 5, 500, 2)
    whole, _ = _lib.genotype(prob)
    for n_segments in (2, 3, 8):
        got = multigpu.genotype_pedigree_segments(prob, n_segments)
        assert close(got, whole), (n_segments, float(np.nanmax(np.abs(got - whole))))


@pytest.mark.parametrize("ped", PEDS)
def test_random_pedigrees(ped):
    """T = 64 and T = 256 take the transfer pass in batches of 16 inputs, put on one scale afterwards."""
    for prior in ("uniform", "random", "sparse"):
        prob = instance(ped, prior, PEDS.index(ped) * 3 + ["uniform", "random", "sparse"].index(prior))
        whole, _ = _lib.genotype(prob)
        want = checker.best().genotype(prob)
        chains = len(multigpu.independent_blocks(prob))
        for n_segments in sorted({2, 3, chains}):
            got = multigpu.genotype_pedigree_segments(prob, n_segments)
            assert close(got, whole) and close(got, want), (ped, prior, n_segments, float(np.nanmax(np.abs(got - whole))))
        # the device's transfer matrices are the emulation's, up to the order of the atomic additions
        r = multigpu.segment_ranges(prob, 3)[1]
        sub = prob.slice_columns(*r)
        dev = _lib.GenotypeSegment(sub, True, r[1] < prob.n_cols)
        emu = emul_genotype_segment.Segment(sub, True, r[1] < prob.n_cols)
        try:
            m, e = dev.transfer(), emu.transfer()
            assert np.allclose(m / m.max(), e / e.max(), rtol=1e-12, atol=1e-13), (ped, prior)
            T = 4 ** prob.n_trios
            assert dev.stats["kernel_launches"] == sub.n_cols * (2 if T <= 16 else 3) * max(1, T // 16)
        finally:
            dev.close()
            emu.close()


def test_golden_vectors_segmented():
    n = 0
    for label, prob, want, _ in golden():
        chains = len(multigpu.independent_blocks(prob))
        if prob.n_trios == 0 or chains < 2:
            continue
        for n_segments in sorted({2, chains}):
            got = multigpu.genotype_pedigree_segments(prob, n_segments)
            assert close(got, want), (label, n_segments, float(np.nanmax(np.abs(got - want))))
        n += 1
    assert n >= 5, n


def test_bounded_segment(monkeypatch):
    """A segment run under a budget below its backward tables takes the memory-bounded mode: same likelihoods, less memory."""
    prob = trio_problem(600, 3, 40, 3)
    ranges = multigpu.segment_ranges(prob, 3)
    mats = []
    for r in ranges:
        seg = _lib.GenotypeSegment(prob.slice_columns(*r), r[0] > 0, r[1] < prob.n_cols)
        mats.append(seg.transfer())
        seg.close()
    alphas, betas = multigpu.genotype_segment_inputs(mats)
    seg = _lib.GenotypeSegment(prob.slice_columns(*ranges[1]), True, True)
    try:
        resident = seg.run(alphas[1], betas[1])
        st = seg.stats
        monkeypatch.setenv(HOOK, str(st["backptr_bytes"] // 4))
        bounded = seg.run(alphas[1], betas[1])
        st2 = seg.stats
    finally:
        seg.close()
    assert close(bounded, resident), float(np.nanmax(np.abs(bounded - resident)))
    assert st2["backptr_bytes"] < st["backptr_bytes"] and st2["kernel_launches"] > st["kernel_launches"], (st, st2)
    whole, _ = _lib.genotype(prob)
    lo, hi = ranges[1]
    assert close(bounded, whole[:, lo:hi])


def test_misuse_is_refused():
    from whatshap_b200._abi import Unsupported

    with pytest.raises(Unsupported, match="independent tables"):
        _lib.GenotypeSegment(synth.genotyping_problem(np.random.default_rng(1), 20, 4, "single"), True, True)
    prob = trio_problem(120, 3, 40, 4)
    seg = _lib.GenotypeSegment(prob.slice_columns(40, 80), True, True)
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


def _worker(rank, world, port, out_queue):
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here))
    sys.path.insert(0, here)
    import torch

    torch.cuda.set_device(0)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    prob = trio_problem(600, 3, 40, 5) if rank == 0 else None
    got = multigpu.genotype_sharded(prob)
    if rank == 0:
        want = multigpu.genotype_pedigree_segments(prob, world)
        out_queue.put((bool(close(got, want)), float(np.nanmax(np.abs(got - want)))))
    else:
        assert got is None
    dist.destroy_process_group()


def test_two_ranks_on_one_device():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    same, diff = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert same, diff
