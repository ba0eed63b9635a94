"""Pedigree genotyping split into segments of whole chains (DESIGN §4.5, `whmec_genotype_segment_*`) against the whole table.

  python scripts/genotype_segments.py [--cols 20000] [--reps 3] [--out FILE]
  torchrun --nproc-per-node N scripts/genotype_segments.py      (N > 1 GPUs: also genotype_sharded over NCCL)

A cfg5-shaped trio genotyping problem (`synth.trio(cols, 5)`: 15 reads per column, chains of 500 columns; random priors,
phred-scaled recombination costs).  On one GPU: the whole table (`whmec_genotype`), then 2, 4 and 8 segments, all on this GPU
one after the other.  For each segment: device time and launches of its transfer pass and of its run (median of --reps), and
the largest absolute difference of the segmented likelihoods from the whole table's.  `max(transfer) + max(run)` is a
PROJECTION of what N GPUs would take (no communication, no host work), not a multi-GPU measurement.  Under torchrun with
N > 1 ranks the script also times `multigpu.genotype_sharded` (wall time on rank 0) against the single-GPU call.

Prints one JSON line per measurement, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whatshap_b200 import _lib, multigpu, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def problem(cols, seed=20250935):
    rng = np.random.default_rng(seed)
    prob = synth.trio(cols, 5, seed=seed)
    prob.gl = rng.random((3, prob.n_cols, 3)) + 0.05
    prob.gl /= prob.gl.sum(axis=2, keepdims=True)
    prob.recombcost = rng.integers(0, 30, prob.n_cols).astype(np.uint32)
    prob.distrust = True
    return prob


def median(xs):
    return sorted(xs)[len(xs) // 2]


def emit(out, rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def one_gpu(prob, a, hw, device):
    times, whole, st = [], None, None
    _lib.genotype(prob, device=device)  # warm-up: module load, memory pool
    for _ in range(a.reps):
        whole, st = _lib.genotype(prob, device=device)
        times.append(st["sweep_ms"])
    emit(a.out, dict(hw, case="cfg5-shaped trio genotyping", cols=a.cols, segments=1, device_ms=round(median(times), 3),
                     launches=st["kernel_launches"]))
    for n_segments in (2, 4, 8):
        ranges = [r for r in multigpu.segment_ranges(prob, n_segments) if r is not None]
        segs = [_lib.GenotypeSegment(prob.slice_columns(*r), r[0] > 0, r[1] < prob.n_cols, device=device) for r in ranges]
        try:
            tr = [[] for _ in segs]
            run = [[] for _ in segs]
            got = np.zeros_like(whole)
            for _ in range(a.reps):
                mats = []
                for s, sg in enumerate(segs):
                    mats.append(sg.transfer())
                    tr[s].append((sg.stats["sweep_ms"], sg.stats["kernel_launches"]))
                alphas, betas = multigpu.genotype_segment_inputs(mats)
                for s, (sg, r) in enumerate(zip(segs, ranges)):
                    got[:, r[0]:r[1]] = sg.run(alphas[s], betas[s])
                    run[s].append((sg.stats["sweep_ms"], sg.stats["kernel_launches"]))
        finally:
            for sg in segs:
                sg.close()
        per = [{"cols": [int(r[0]), int(r[1])], "transfer_ms": round(median([t for t, _ in tr[s]]), 3), "transfer_launches": tr[s][0][1],
                "run_ms": round(median([t for t, _ in run[s]]), 3), "run_launches": run[s][0][1]} for s, r in enumerate(ranges)]
        emit(a.out, dict(hw, case="cfg5-shaped trio genotyping", cols=a.cols, segments=len(ranges), per_segment=per,
                         projection_ms=round(max(p["transfer_ms"] for p in per) + max(p["run_ms"] for p in per), 3),
                         projection="max(transfer) + max(run): segments timed one after the other on one GPU, not a multi-GPU measurement",
                         max_abs_diff=float(np.nanmax(np.abs(got - whole)))))


def sharded(prob, a, hw):
    import torch
    import torch.distributed as dist

    rank = int(os.environ["RANK"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl")
    world = dist.get_world_size()
    from whatshap_b200 import _wire

    comm = _wire.Comm()
    comm.warm_up()
    mine = prob if rank == 0 else None
    multigpu.genotype_sharded(mine, comm=comm)  # warm-up
    walls = []
    got = None
    for _ in range(a.reps):
        dist.barrier()
        t0 = time.perf_counter()
        got = multigpu.genotype_sharded(mine, comm=comm)
        walls.append((time.perf_counter() - t0) * 1e3)
    if rank == 0:
        single = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            whole, _ = _lib.genotype(prob, device=torch.cuda.current_device())
            single.append((time.perf_counter() - t0) * 1e3)
        emit(a.out, dict(hw, case="cfg5-shaped trio genotyping, genotype_sharded over NCCL", cols=a.cols, ranks=world,
                         sharded_wall_ms=round(median(walls), 3), single_gpu_wall_ms=round(median(single), 3),
                         max_abs_diff=float(np.nanmax(np.abs(got - whole)))))
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cols", type=int, default=20_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert _lib.device_count() > 0, "needs a CUDA device"
    hw = card()
    os.environ.pop("WHMEC_GENOTYPE_ARENA_BUDGET", None)
    prob = problem(a.cols)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        sharded(prob, a, hw)
    else:
        one_gpu(prob, a, hw, 0)


if __name__ == "__main__":
    main()
