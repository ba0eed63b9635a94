"""Refusals and clean-up of the multi-GPU schemes without a GPU.  Phasing over gloo ranks, with the CPU checker and the emulated
segments standing in for the per-rank CUDA calls: a refused run of blocks or whole table is raised as Unsupported on every
rank, and a segment refused in any phase sends every rank to the whole table on rank 0, as the genotyping and one-process
drivers do.  One process: `solve_pedigree_segments` closes the segments it has created when a later one cannot be created."""
import os
import socket

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import emul_segment
from oracle import checker
from whatshap_b200 import multigpu, synth
from whatshap_b200._abi import Unsupported


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _refusing_worker(rank, world, port, where, out_queue):
    """Rank `refuser` refuses as unsupported in `where`: its run of blocks ("blocks"), the whole table ("whole", rank 0), or its
    segment's transfer or exits pass."""
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here))
    sys.path.insert(0, here)
    from emul_segment import EmulSegment
    from oracle import checker

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    refuser = 0 if where == "whole" else 1

    class Refusing(EmulSegment):
        def transfer(self):
            if where == "transfer":
                raise Unsupported("unsupported problem: transfer refused")
            return super().transfer()

        def exits(self, is_last):
            if where == "exits":
                raise Unsupported("unsupported problem: exits refused")
            return super().exits(is_last)

    def solver(p):
        if where in ("blocks", "whole") and rank == refuser:
            raise Unsupported("unsupported problem: %s refused" % where)
        return checker.best().solve(p)

    prob = None
    if rank == 0:
        prob = {"blocks": lambda: synth.sliding_window(120, 6, block_len=20, seed=5, gap=0.1),
                "whole": lambda: synth.trio(30, 2, block_len=30, seed=3)}.get(where, lambda: synth.trio(40, 2, block_len=10, seed=6))()
    try:
        sol = multigpu.solve_sharded(prob, solver=solver, segment_factory=Refusing if rank == refuser else EmulSegment)
    except Unsupported as e:
        out_queue.put((rank, "raised", str(e)))
    else:
        if rank == 0:
            want = checker.best().solve(prob)
            out_queue.put((rank, bool(sol.same_as(want)), sol.diff(want)))
        else:
            out_queue.put((rank, sol is None, ""))
    dist.destroy_process_group()


@pytest.mark.parametrize("where", ["blocks", "whole", "transfer", "exits"])
def test_phasing_ranks_raise_or_fall_back_on_a_refusal(where):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_refusing_worker, args=(r, 2, port, where, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = sorted(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    if where in ("blocks", "whole"):
        assert all(r[1] == "raised" and "%s refused" % where in r[2] for r in results), results
    else:
        assert all(r[1] is True for r in results), results


def test_local_segments_are_closed_when_a_create_fails():
    prob = synth.trio(120, 2, block_len=10, seed=6)
    ranges = multigpu.segment_ranges(prob, 4)
    assert all(r is not None for r in ranges)
    opened, closed = [], []

    class Failing(emul_segment.EmulSegment):
        def __init__(self, p, continues):
            if len(opened) == 2:
                raise RuntimeError("no third segment")
            super().__init__(p, continues)
            opened.append(self)

        def close(self):
            closed.append(self)
            super().close()

    with pytest.raises(RuntimeError, match="^no third segment$"):
        multigpu.solve_pedigree_segments(prob, 4, Failing)
    assert len(opened) == 2 and sorted(map(id, closed)) == sorted(map(id, opened))
    assert multigpu.solve_pedigree_segments(prob, 4, emul_segment.EmulSegment).same_as(checker.best().solve(prob))
